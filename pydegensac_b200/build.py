"""In-tree build of the native pieces (sm_90a, H100, only).

    python -m pydegensac_b200.build          # CUDA library + pybind11 module (+ oracle builds)

Artifacts (git-ignored):
    pydegensac_b200/libdegensac_b200.so                  C ABI + sm_90a kernels (nvcc cross-compiles without a GPU)
    pydegensac_b200/pydegensac.<abi>.so                  pybind11 surface (findHomography_, findFundamentalMatrix_)
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdegensac_b200.so")
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
              "--shared", "-Xcompiler", "-fPIC"]


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def _csrc_files():
    out = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    out.append(os.path.join(ROOT, "include", "degensac_b200.h"))
    return out


def build_cuda(force=False, verbose=False):
    src = os.path.join(CSRC, "degensac_b200.cu")
    src2 = os.path.join(CSRC, "frontend.cu")      # matcher / pose / QR null space (the steps either side of the path)
    src3 = os.path.join(CSRC, "absolute_pose.cu")  # P3P RANSAC: registering a view against known 3D points
    src4 = os.path.join(CSRC, "triangulate.cu")    # multi-view triangulation of tracks across registered views
    src5 = os.path.join(CSRC, "bundle_adjust.cu")  # bundle adjustment of registered views and their tracks
    src6 = os.path.join(CSRC, "tracks.cu")         # tracks from verified pairwise matches (union-find over keypoints)
    src7 = os.path.join(CSRC, "bundle_adjust_pcg.cu")  # bundle adjustment of any number of cameras (PCG on Schur)
    src8 = os.path.join(CSRC, "bundle_adjust_intrinsics.cu")  # bundle adjustment with intrinsics, undistortion
    src9 = os.path.join(CSRC, "rotation_averaging.cu")  # world rotations of many views from their relative rotations
    src10 = os.path.join(CSRC, "global_positioning.cu")  # the views' centres and the tracks' points from the rotations
    src11 = os.path.join(CSRC, "view_graph_calibration.cu")  # the groups' focal lengths from the pairs' F
    src12 = os.path.join(CSRC, "essential.cu")     # five-point RANSAC: relative pose of calibrated pairs
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest(_csrc_files()):
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, src, src2, src3, src4, src5, src6,
                                                                                 src7, src8, src9, src10, src11, src12]
    subprocess.check_call(cmd)
    return LIB


def pybind_target():
    return os.path.join(HERE, "pydegensac" + sysconfig.get_config_var("EXT_SUFFIX"))


def build_pybind(force=False):
    import pybind11
    src = os.path.join(CSRC, "pybind_module.cpp")
    out = pybind_target()
    if not force and os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(src), os.path.getmtime(LIB)):
        return out
    cmd = ["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-fvisibility=hidden",
           "-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"], src, "-o", out,
           "-L" + HERE, "-ldegensac_b200", "-Wl,-rpath,$ORIGIN"]
    subprocess.check_call(cmd)
    return out


LEGACY = os.path.join(HERE, "libdegensac_b200_legacy.so")


def build_legacy(force=False):
    """The reference's own C entry points (include/degensac_legacy.h) over the C ABI."""
    src = os.path.join(CSRC, "legacy_shim.cpp")
    if not force and os.path.exists(LEGACY) and os.path.getmtime(LEGACY) >= max(os.path.getmtime(src), os.path.getmtime(LIB)):
        return LEGACY
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", src, "-o", LEGACY, "-L" + HERE,
                           "-ldegensac_b200", "-Wl,-rpath,$ORIGIN"])
    return LEGACY


def build_all(force=False, verbose=False):
    build_cuda(force, verbose)
    build_pybind(force)
    build_legacy(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built", LIB)
    print("built", pybind_target())
