"""CTAs per SM of ransac_pairs_kernel<KIND> at given CTA widths, from the driver's occupancy query.

    cuobjdump -xelf degensac_b200.sm_90a.cubin pydegensac_b200/libdegensac_b200.so
    python tools/occupancy.py degensac_b200.sm_90a.cubin SMEM_BYTES THREADS...

SMEM_BYTES is the launch's dynamic shared memory (the block scratch rounded up to 128 B: 15 936 B in the default build).
Needs a GPU; loads the cubin through the driver API, so it sees the registers and stack of the shipped binary."""
import ctypes
import re
import sys


def main():
    cubin, smem = sys.argv[1], int(sys.argv[2])
    threads = [int(t) for t in sys.argv[3:]]
    cu = ctypes.CDLL("libcuda.so.1")

    def ck(r, what):
        if r != 0:
            raise RuntimeError("%s: CUresult %d" % (what, r))

    ck(cu.cuInit(0), "cuInit")
    dev, ctx, mod = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_void_p()
    ck(cu.cuDeviceGet(ctypes.byref(dev), 0), "cuDeviceGet")
    ck(cu.cuDevicePrimaryCtxRetain(ctypes.byref(ctx), dev), "cuDevicePrimaryCtxRetain")
    ck(cu.cuCtxSetCurrent(ctx), "cuCtxSetCurrent")
    data = open(cubin, "rb").read()
    ck(cu.cuModuleLoadData(ctypes.byref(mod), ctypes.c_char_p(data)), "cuModuleLoadData")
    for kind in (b"0", b"1", b"2"):
        m = re.search(rb"_ZN\w*ransac_pairs_kernelILi" + kind + rb"EEEvNS_9BatchArgsE", data)
        if not m:
            continue
        f, regs = ctypes.c_void_p(), ctypes.c_int()
        ck(cu.cuModuleGetFunction(ctypes.byref(f), mod, m.group(0)), "cuModuleGetFunction")
        ck(cu.cuFuncSetAttribute(f, 8, smem), "max dynamic shared memory")   # CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES
        ck(cu.cuFuncGetAttribute(ctypes.byref(regs), 4, f), "registers")      # CU_FUNC_ATTRIBUTE_NUM_REGS
        for t in threads:
            n = ctypes.c_int()
            ck(cu.cuOccupancyMaxActiveBlocksPerMultiprocessor(ctypes.byref(n), f, t, ctypes.c_size_t(smem)), "occupancy")
            print("kernel<%s> regs %d threads %d smem %d -> %d CTAs/SM" % (kind.decode(), regs.value, t, smem, n.value))
    cu.cuDevicePrimaryCtxRelease(dev)


if __name__ == "__main__":
    main()
