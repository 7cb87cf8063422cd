"""ctypes binding of the C ABI (include/degensac_b200.h) -- used for the batched entry points.

The library is the product: if libdegensac_b200.so is missing or no CUDA device is visible, calls raise.
There is no CPU fallback anywhere in this package.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libdegensac_b200.so")
_lib = None
FLAG_FINAL_LSQ = 1   # DGB200_FLAG_FINAL_LSQ
GUIDE_F, GUIDE_H = 0, 1   # DGB200_GUIDE_F, DGB200_GUIDE_H


class EngineUnavailable(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIBPATH):
            raise EngineUnavailable(
                "pydegensac_b200: %s is missing - build it with `python -m pydegensac_b200.build` "
                "(the engine is CUDA-only; there is no CPU fallback)" % _LIBPATH)
        L = ctypes.CDLL(_LIBPATH)
        dp = ctypes.POINTER(ctypes.c_double)
        u8 = ctypes.POINTER(ctypes.c_uint8)
        i32 = ctypes.POINTER(ctypes.c_int32)
        u64 = ctypes.POINTER(ctypes.c_uint64)
        ci, cd = ctypes.c_int, ctypes.c_double
        L.dgb200_find_fundamental_batch.argtypes = [dp, dp, ci, ci, ci, cd, cd, ci, ci, ci, cd, ci, u64, dp, u8, i32]
        L.dgb200_find_homography_batch.argtypes = [dp, dp, ci, ci, ci, cd, cd, ci, ci, ci, cd, u64, dp, u8, i32]
        vp = ctypes.c_void_p
        L.dgb200_find_fundamental_batch_dev.argtypes = [vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, ci, vp, vp, vp, vp, vp]
        L.dgb200_find_homography_batch_dev.argtypes = [vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, vp, vp, vp, vp, vp]
        cu = ctypes.c_uint
        L.dgb200_find_fundamental_batch_ex.argtypes = [dp, dp, ci, ci, ci, cd, cd, ci, ci, ci, cd, ci, u64, dp, u8, i32, cu]
        L.dgb200_find_homography_batch_ex.argtypes = [dp, dp, ci, ci, ci, cd, cd, ci, ci, ci, cd, u64, dp, u8, i32, cu]
        L.dgb200_find_fundamental_batch_dev_ex.argtypes = [vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, ci, vp, vp, vp, vp, vp, cu]
        L.dgb200_find_homography_batch_dev_ex.argtypes = [vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, vp, vp, vp, vp, vp, cu]
        L.dgb200_find_fundamental_ragged.argtypes = [dp, dp, i32, ci, ci, cd, cd, ci, ci, ci, cd, ci, u64, dp, u8, i32]
        L.dgb200_find_homography_ragged.argtypes = [dp, dp, i32, ci, ci, cd, cd, ci, ci, ci, cd, u64, dp, u8, i32]
        L.dgb200_find_fundamental_ragged_dev.argtypes = [vp, vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, ci, vp, vp, vp, vp, vp]
        L.dgb200_find_homography_ragged_dev.argtypes = [vp, vp, vp, ci, ci, ci, cd, cd, ci, ci, ci, cd, vp, vp, vp, vp, vp]
        L.dgb200_find_homography_2el_batch.argtypes = [dp, ci, ci, cd, cd, ci, u64, dp, u8, i32]
        L.dgb200_find_homography_2el_batch_dev.argtypes = [vp, ci, ci, cd, cd, ci, vp, vp, vp, vp, vp]
        L.dgb200_match_workspace_bytes.restype = ctypes.c_size_t
        L.dgb200_match_workspace_bytes.argtypes = [ci, ci]
        L.dgb200_match_descriptors_dev.argtypes = [vp, ci, vp, ci, ci, ctypes.c_float, ci, vp, vp, ci, vp, vp, vp, vp, ci, ci, vp, vp, vp]
        L.dgb200_match_batch_workspace_bytes.restype = ctypes.c_size_t
        L.dgb200_match_batch_workspace_bytes.argtypes = [i32, ci, i32, ci]
        L.dgb200_match_descriptors_batch_dev.argtypes = [vp, i32, ci, ci, i32, ci, ctypes.c_float, ci, vp, ci, vp, vp, vp, vp,
                                                         ci, ci, vp, vp, vp]
        L.dgb200_match_binary_descriptors_dev.argtypes = [vp, ci, vp, ci, ci, cd, ci, vp, vp, ci, vp, vp, vp, vp, ci, ci, vp,
                                                          vp, vp]
        L.dgb200_match_binary_descriptors_batch_dev.argtypes = [vp, i32, ci, ci, i32, ci, cd, ci, vp, ci, vp, vp, vp, vp,
                                                                ci, ci, vp, vp, vp]
        L.dgb200_match_descriptors_guided_batch_dev.argtypes = [vp, i32, ci, ci, i32, ci, vp, ci, cd, ctypes.c_float, ci,
                                                                vp, ci, vp, vp, vp, vp, ci, ci, vp, vp, vp]
        L.dgb200_match_binary_descriptors_guided_batch_dev.argtypes = [vp, i32, ci, ci, i32, ci, vp, ci, cd, cd, ci, vp,
                                                                       ci, vp, vp, vp, vp, ci, ci, vp, vp, vp]
        L.dgb200_pose_from_fundamental_batch_dev.argtypes =[vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, vp, vp, vp, vp]
        L.dgb200_pose_from_fundamental_ragged_dev.argtypes = [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, vp, vp, vp, vp, vp, vp,
                                                              vp, vp, vp]
        L.dgb200_pose_from_homography_ragged_dev.argtypes = [vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, vp, vp, vp, vp, vp,
                                                             vp, vp, vp, vp, vp, vp]
        L.dgb200_refine_pose_ragged_dev.argtypes = [vp, vp, vp, vp, ci, vp, vp, vp, ci, ci, ci, vp, ci, cd, vp, vp, vp, vp,
                                                    vp, vp, vp, vp, vp]
        L.dgb200_refine_homography_ragged_dev.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, ci, cd, vp, vp, vp, vp, vp, vp,
                                                          vp]
        L.dgb200_refine_fundamental_ragged_dev.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, ci, cd, vp, vp, vp, vp, vp,
                                                           vp, vp]
        L.dgb200_find_absolute_pose_ragged_dev.argtypes = [vp, vp, vp, ci, vp, ci, ci, vp, cd, cd, ci, ci, vp, vp, vp,
                                                           vp, vp, vp, vp, vp, vp]
        L.dgb200_absolute_pose_last_error.restype = ctypes.c_char_p
        L.dgb200_find_essential_ragged_dev.argtypes = [vp, vp, vp, vp, ci, vp, ci, ci, vp, cd, cd, ci, ci, vp, vp, vp,
                                                       vp, vp, vp, vp, vp, vp]
        L.dgb200_essential_last_error.restype = ctypes.c_char_p
        L.dgb200_triangulate_tracks_ragged_dev.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, cd, cd, cd, ci, ci,
                                                           vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.dgb200_triangulate_last_error.restype = ctypes.c_char_p
        L.dgb200_bundle_adjust_ragged_dev.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, vp, i32, ci, ci, cd, ci,
                                                      cd, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.dgb200_bundle_adjust_last_error.restype = ctypes.c_char_p
        L.dgb200_bundle_adjust_pcg_ragged_dev.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, vp, i32, ci, ci, cd,
                                                          ci, cd, ci, cd, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        L.dgb200_bundle_adjust_pcg_last_error.restype = ctypes.c_char_p
        L.dgb200_bundle_adjust_intrinsics_ragged_dev.argtypes = [vp, vp, vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, vp, i32,
                                                                 ci, i32, ci, ci, ci, cd, ci, cd, ci, cd, vp, vp, vp,
                                                                 vp, vp, vp, vp, vp, vp, vp, vp]
        L.dgb200_bundle_adjust_intrinsics_last_error.restype = ctypes.c_char_p
        L.dgb200_undistort_points_dev.argtypes = [vp, vp, ci, vp, ci, vp, ci, vp, vp]
        L.dgb200_undistort_last_error.restype = ctypes.c_char_p
        L.dgb200_build_tracks_ragged_dev.argtypes = [i32, ci, i32, ci, vp, vp, vp, ci, vp, vp, ci, vp, vp, vp, vp, vp, vp,
                                                     vp]
        L.dgb200_tracks_last_error.restype = ctypes.c_char_p
        L.dgb200_average_rotations_dev.argtypes = [i32, ci, ci, vp, vp, vp, cd, ci, ci, cd, ci, cd, vp, vp, vp, vp, vp,
                                                   vp]
        L.dgb200_rotation_averaging_last_error.restype = ctypes.c_char_p
        L.dgb200_global_positioning_ragged_dev.argtypes = [vp, vp, vp, vp, ci, ci, vp, ci, ci, vp, ctypes.c_uint64, cd,
                                                           cd, ci, cd, ci, cd, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                                           vp]
        L.dgb200_global_positioning_last_error.restype = ctypes.c_char_p
        L.dgb200_calibrate_view_graph_dev.argtypes = [i32, ci, ci, vp, vp, vp, vp, ci, cd, cd, cd, ci, ci, cd, vp, vp,
                                                      vp, vp, vp, vp, vp, vp, vp, vp]
        L.dgb200_view_graph_calibration_last_error.restype = ctypes.c_char_p
        L.dgb200_nullspace_qr7x9_batch_dev.argtypes = [vp, vp, vp, ci, vp]
        L.dgb200_frontend_last_error.restype = ctypes.c_char_p
        L.dgb200_last_error.restype = ctypes.c_char_p
        L.dgb200_kernel_launches.restype = ctypes.c_longlong
        L.dgb200_last_kernel_ms.restype = ctypes.c_double
        _lib = L
    return _lib


def _raise(rc):
    msg = lib().dgb200_last_error().decode()
    if rc in (-1, -2, -3):
        raise ValueError(msg)
    raise EngineUnavailable("degensac_b200: " + msg)


def _p(a, t):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _prep(pts1, pts2):
    p1 = np.ascontiguousarray(pts1, dtype=np.float64)
    p2 = np.ascontiguousarray(pts2, dtype=np.float64)
    if p1.ndim == 2:
        p1, p2 = p1[None], p2[None]
    if p1.ndim != 3 or p1.shape != p2.shape:
        raise ValueError("expected two arrays of shape [P,N,2] or [P,N,6] with equal shapes")
    return p1, p2


def _seeds(seeds, P):
    if seeds is None:
        return None
    s = np.ascontiguousarray(np.broadcast_to(np.asarray(seeds, dtype=np.uint64), (P,)))
    return s


def fundamental_batch(pts1, pts2, px_th, conf, max_iters, error_type, sym_check, laf_coef, degen_check, seeds, flags=0):
    p1, p2 = _prep(pts1, pts2)
    P, N, dim = p1.shape
    F = np.zeros((P, 3, 3), dtype=np.float64)
    mask = np.zeros((P, N), dtype=np.uint8)
    stats = np.zeros((P, 4), dtype=np.int32)
    s = _seeds(seeds, P)
    rc = lib().dgb200_find_fundamental_batch_ex(_p(p1, ctypes.c_double), _p(p2, ctypes.c_double), P, N, dim,
                                                float(px_th), float(conf), int(max_iters), int(error_type),
                                                int(bool(sym_check)), float(laf_coef), int(bool(degen_check)),
                                                _p(s, ctypes.c_uint64) if s is not None else None,
                                                _p(F, ctypes.c_double), _p(mask, ctypes.c_uint8), _p(stats, ctypes.c_int32),
                                                int(flags))
    if rc != 0:
        _raise(rc)
    return F, mask.view(np.bool_), stats


def homography_batch(pts1, pts2, px_th, conf, max_iters, error_type, sym_check, laf_coef, seeds, flags=0):
    p1, p2 = _prep(pts1, pts2)
    P, N, dim = p1.shape
    H = np.zeros((P, 3, 3), dtype=np.float64)
    mask = np.zeros((P, N), dtype=np.uint8)
    stats = np.zeros((P, 4), dtype=np.int32)
    s = _seeds(seeds, P)
    rc = lib().dgb200_find_homography_batch_ex(_p(p1, ctypes.c_double), _p(p2, ctypes.c_double), P, N, dim,
                                               float(px_th), float(conf), int(max_iters), int(error_type),
                                               int(bool(sym_check)), float(laf_coef),
                                               _p(s, ctypes.c_uint64) if s is not None else None,
                                               _p(H, ctypes.c_double), _p(mask, ctypes.c_uint8), _p(stats, ctypes.c_int32),
                                               int(flags))
    if rc != 0:
        _raise(rc)
    return H, mask.view(np.bool_), stats


def _ragged_prep(list1, list2):
    if len(list1) != len(list2) or len(list1) == 0:
        raise ValueError("expected two equally long, non-empty lists of [n_i, dim] arrays")
    a1 = [np.ascontiguousarray(a, dtype=np.float64) for a in list1]
    a2 = [np.ascontiguousarray(a, dtype=np.float64) for a in list2]
    dim = a1[0].shape[1] if a1[0].ndim == 2 else -1
    for x, y in zip(a1, a2):
        if x.ndim != 2 or x.shape != y.shape or x.shape[1] != dim:
            raise ValueError("every pair needs two arrays of equal shape [n_i, dim] with the same dim across the batch")
    offsets = np.zeros(len(a1) + 1, dtype=np.int32)
    offsets[1:] = np.cumsum([x.shape[0] for x in a1])
    return np.concatenate(a1, 0), np.concatenate(a2, 0), offsets, dim


def fundamental_ragged(list1, list2, px_th, conf, max_iters, error_type, sym_check, laf_coef, degen_check, seeds):
    """Ragged batch: lists of [n_i, dim] arrays.  Returns (F [P,3,3], list of bool masks, stats [P,4])."""
    p1, p2, offsets, dim = _ragged_prep(list1, list2)
    P = len(offsets) - 1
    F = np.zeros((P, 3, 3), dtype=np.float64)
    mask = np.zeros(int(offsets[-1]), dtype=np.uint8)
    stats = np.zeros((P, 4), dtype=np.int32)
    s = _seeds(seeds, P)
    rc = lib().dgb200_find_fundamental_ragged(_p(p1, ctypes.c_double), _p(p2, ctypes.c_double), _p(offsets, ctypes.c_int32),
                                              P, dim, float(px_th), float(conf), int(max_iters), int(error_type),
                                              int(bool(sym_check)), float(laf_coef), int(bool(degen_check)),
                                              _p(s, ctypes.c_uint64) if s is not None else None,
                                              _p(F, ctypes.c_double), _p(mask, ctypes.c_uint8), _p(stats, ctypes.c_int32))
    if rc != 0:
        _raise(rc)
    mb = mask.view(np.bool_)
    return F, [mb[offsets[i]:offsets[i + 1]] for i in range(P)], stats


def homography_ragged(list1, list2, px_th, conf, max_iters, error_type, sym_check, laf_coef, seeds):
    """Ragged batch: lists of [n_i, dim] arrays.  Returns (RAW H [P,3,3], list of bool masks, stats [P,4])."""
    p1, p2, offsets, dim = _ragged_prep(list1, list2)
    P = len(offsets) - 1
    H = np.zeros((P, 3, 3), dtype=np.float64)
    mask = np.zeros(int(offsets[-1]), dtype=np.uint8)
    stats = np.zeros((P, 4), dtype=np.int32)
    s = _seeds(seeds, P)
    rc = lib().dgb200_find_homography_ragged(_p(p1, ctypes.c_double), _p(p2, ctypes.c_double), _p(offsets, ctypes.c_int32),
                                             P, dim, float(px_th), float(conf), int(max_iters), int(error_type),
                                             int(bool(sym_check)), float(laf_coef),
                                             _p(s, ctypes.c_uint64) if s is not None else None,
                                             _p(H, ctypes.c_double), _p(mask, ctypes.c_uint8), _p(stats, ctypes.c_int32))
    if rc != 0:
        _raise(rc)
    mb = mask.view(np.bool_)
    return H, [mb[offsets[i]:offsets[i + 1]] for i in range(P)], stats


def fundamental_batch_dev(d_p1, d_p2, P, N, dim, px_th, conf, max_iters, error_type, sym_check, laf_coef, degen_check,
                          d_seeds, d_F, d_mask, d_stats, stream=0, flags=0):
    """Device-pointer flavour: all d_* are integer device addresses (e.g. torch.Tensor.data_ptr())."""
    rc = lib().dgb200_find_fundamental_batch_dev_ex(d_p1, d_p2, P, N, dim, float(px_th), float(conf), int(max_iters),
                                                    int(error_type), int(bool(sym_check)), float(laf_coef),
                                                    int(bool(degen_check)), d_seeds, d_F, d_mask, d_stats, stream,
                                                    int(flags))
    if rc != 0:
        _raise(rc)


def homography_batch_dev(d_p1, d_p2, P, N, dim, px_th, conf, max_iters, error_type, sym_check, laf_coef, d_seeds,
                         d_H, d_mask, d_stats, stream=0, flags=0):
    rc = lib().dgb200_find_homography_batch_dev_ex(d_p1, d_p2, P, N, dim, float(px_th), float(conf), int(max_iters),
                                                   int(error_type), int(bool(sym_check)), float(laf_coef), d_seeds, d_H,
                                                   d_mask, d_stats, stream, int(flags))
    if rc != 0:
        _raise(rc)


def fundamental_ragged_dev(d_p1, d_p2, d_offsets, P, n_max, dim, px_th, conf, max_iters, error_type, sym_check, laf_coef,
                           degen_check, d_seeds, d_F, d_mask, d_stats, stream=0):
    """Device-pointer ragged batch: pair p owns rows d_offsets[p] .. d_offsets[p+1]-1 (int32 device array)."""
    rc = lib().dgb200_find_fundamental_ragged_dev(d_p1, d_p2, d_offsets, P, int(n_max), dim, float(px_th), float(conf),
                                                  int(max_iters), int(error_type), int(bool(sym_check)), float(laf_coef),
                                                  int(bool(degen_check)), d_seeds, d_F, d_mask, d_stats, stream)
    if rc != 0:
        _raise(rc)


def homography_ragged_dev(d_p1, d_p2, d_offsets, P, n_max, dim, px_th, conf, max_iters, error_type, sym_check, laf_coef,
                          d_seeds, d_H, d_mask, d_stats, stream=0):
    rc = lib().dgb200_find_homography_ragged_dev(d_p1, d_p2, d_offsets, P, int(n_max), dim, float(px_th), float(conf),
                                                 int(max_iters), int(error_type), int(bool(sym_check)), float(laf_coef),
                                                 d_seeds, d_H, d_mask, d_stats, stream)
    if rc != 0:
        _raise(rc)


def homography_2el_batch(u10, px_th, conf, max_iters, seeds):
    """ransacH2el over a batch: u10 [P,N,10] rows (x', y', a', b', c', x, y, a, b, c) -> raw H [P,3,3], mask, stats."""
    u = np.ascontiguousarray(u10, dtype=np.float64)
    if u.ndim == 2:
        u = u[None]
    if u.ndim != 3 or u.shape[2] != 10:
        raise ValueError("u10 should be an array with dims [n,10] or [P,n,10]")
    P, N, _ = u.shape
    H = np.zeros((P, 3, 3), dtype=np.float64)
    mask = np.zeros((P, N), dtype=np.uint8)
    stats = np.zeros((P, 4), dtype=np.int32)
    s = _seeds(seeds, P)
    rc = lib().dgb200_find_homography_2el_batch(_p(u, ctypes.c_double), P, N, float(px_th), float(conf), int(max_iters),
                                                _p(s, ctypes.c_uint64) if s is not None else None,
                                                _p(H, ctypes.c_double), _p(mask, ctypes.c_uint8), _p(stats, ctypes.c_int32))
    if rc != 0:
        _raise(rc)
    return H, mask.view(np.bool_), stats


def homography_2el_batch_dev(d_u10, P, N, px_th, conf, max_iters, d_seeds, d_H, d_mask, d_stats, stream=0):
    rc = lib().dgb200_find_homography_2el_batch_dev(d_u10, P, N, float(px_th), float(conf), int(max_iters), d_seeds, d_H,
                                                    d_mask, d_stats, stream)
    if rc != 0:
        _raise(rc)


def kernel_launches():
    return int(lib().dgb200_kernel_launches())


def last_kernel_ms():
    return float(lib().dgb200_last_kernel_ms())
