"""Python API of the reference (src/pydegensac/utils.py:15-146), same names, arguments, defaults,
validation and return conventions, on top of the CUDA engine.

Additive: `seed=None` on both functions (the reference seeds libc rand() from time(NULL) inside the C
core and cannot be made reproducible); batched entry points `findFundamentalMatrixBatch` /
`findHomographyBatch` for [P,N,2] stacks of independent image pairs.
"""
import math
import os
import warnings

import numpy as np

try:
    import cv2
    OPENCV_HERE = True
except Exception:  # pragma: no cover
    OPENCV_HERE = False

error_type_dict_homography = {"sampson": 0,
                              "symm_sq_max": 1,
                              "symm_max": 2,
                              "symm_sq_sum": 3,
                              "symm_sum": 4}

error_type_dict_fundamental = {"sampson": 0,
                               "symm_epipolar": 1}


def _native():
    """The pybind11 module (bindings.cpp surface). Import lazily so that the pure-Python validation layer can
    be exercised without the native build; any compute call without it raises loudly."""
    from . import _cabi
    _cabi.lib()  # raises EngineUnavailable with build instructions if the CUDA library is missing
    from . import pydegensac as native
    return native


def convert_cv2_kpts_to_xyA(kps):
    """cv2.KeyPoint list -> [N,6] (x, y, a11, a12, a21, a22)   (reference utils.py:24-41)."""
    num = len(kps)
    out = np.zeros((num, 6)).astype(np.float64)
    for i, kp in enumerate(kps):
        out[i, :2] = kp.pt
        s = kp.size
        a = kp.angle
        cos = math.cos(a * math.pi / 180.0)
        sin = math.sin(a * math.pi / 180.0)
        out[i, 2] = s * cos
        out[i, 3] = s * sin
        out[i, 4] = -s * sin
        out[i, 5] = s * cos
    return out


def convert_and_check(kps1):
    """Input validation of the reference (utils.py:43-71)."""
    if type(kps1) is np.ndarray:
        sh = kps1.shape
        err_message = ValueError("Keypoints should be list of cv2.KeyPoint or numpy.array [Nx2] or [Nx6]. N>=4 "
                                 "Got shape of {} with shape instead".format(str(sh)))
        if len(sh) != 2:
            raise err_message
        num, dim = sh
        if (dim != 2) and (dim != 6):
            raise err_message
        if num < 4:
            raise err_message
        out = kps1.astype(np.float64)
    elif type(kps1) is list:
        if OPENCV_HERE:
            if type(kps1[0]) is not cv2.KeyPoint:
                raise ValueError("Keypoints should be list of cv2.KeyPoint or numpy.array [Nx2] or [Nx6]. N>=4 "
                                 "Got input of list of type {}".format(str(type(kps1[0]))))
            out = convert_cv2_kpts_to_xyA(kps1)
        else:
            raise ValueError("Cannot import cv2. Please, install or pass np.arrays instead")
    else:
        raise ValueError("Keypoints should be list of cv2.KeyPoint or numpy.array [Nx2] or [Nx6]. N>=4 "
                         "Got input of type {}".format(str(type(kps1))))
    return out


def _seed_value(seed):
    if seed is None:
        return int.from_bytes(os.urandom(8), "little")
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def _error_type(error_type, table):
    try:
        return table[error_type.lower()]
    except Exception:
        raise ValueError("Error type should be on of {}. Got {} instead".format(list(table.keys()), error_type))


def findHomography(pts1_,
                   pts2_,
                   px_th=1.0,
                   conf=0.999,
                   max_iters=50000,
                   laf_consistensy_coef=-1.0,
                   error_type="sampson",
                   symmetric_error_check=True,
                   seed=None):
    """Reference utils.py:74-109. Returns (H 3x3 in OpenCV convention x2 ~ H x1, mask)."""
    pts1 = convert_and_check(pts1_)
    pts2 = convert_and_check(pts2_)
    n, dim = pts1.shape
    n2, dim2 = pts2.shape
    assert (n == n2) and (dim == dim2)
    if dim == 2 and laf_consistensy_coef > 0:
        warnings.warn('You set laf_consistensy_coef, but provided only (x,y) keypoints. Skipping LAF check')
        laf_consistensy_coef = 0
    error_type_int = _error_type(error_type, error_type_dict_homography)
    laf_consistensy_coef = max(0, laf_consistensy_coef)
    H, mask = _native().findHomography_(pts1, pts2, px_th, conf, max_iters, error_type_int, symmetric_error_check,
                                        laf_consistensy_coef, _seed_value(seed))
    if np.abs(H).sum() == 0:
        # If we haven`t found any good model, output zeros
        mask = [False] * len(mask)
        return H, mask
    H_out = np.linalg.inv(H.T)
    return H_out, mask


def findFundamentalMatrix(pts1_,
                          pts2_,
                          px_th=0.5,
                          conf=0.9999,
                          max_iters=100000,
                          laf_consistensy_coef=-1.0,
                          error_type="sampson",
                          symmetric_error_check=True,
                          enable_degeneracy_check=True,
                          seed=None):
    """Reference utils.py:111-146. Returns (F 3x3 with x2^T F x1 = 0, mask)."""
    pts1 = convert_and_check(pts1_)
    pts2 = convert_and_check(pts2_)
    n, dim = pts1.shape
    n2, dim2 = pts2.shape
    assert (n == n2) and (dim == dim2)
    if dim == 2 and laf_consistensy_coef > 0:
        warnings.warn('You set laf_consistensy_coef, but provided only (x,y) keypoints. Skipping LAF check')
        laf_consistensy_coef = 0
    error_type_int = _error_type(error_type, error_type_dict_fundamental)
    laf_consistensy_coef = max(0, laf_consistensy_coef)
    F, mask = _native().findFundamentalMatrix_(pts1, pts2, px_th, conf, max_iters, error_type_int,
                                               symmetric_error_check, laf_consistensy_coef, enable_degeneracy_check,
                                               _seed_value(seed))
    if np.abs(F).sum() == 0:
        # If we haven`t found any good model, output zeros
        mask = [False] * n
    return F, mask


def _opencv_convention(Hraw):
    """[P,3,3] raw core outputs (column-major, image 2 -> image 1) -> inv(H^T) per pair as utils.py:108 of the reference
    does for one; a zero model (nothing found) stays zero.  One batched LAPACK call instead of P Python-level ones."""
    H = np.zeros_like(Hraw)
    found = np.abs(Hraw).reshape(Hraw.shape[0], -1).sum(axis=1) != 0
    if found.any():
        H[found] = np.linalg.inv(np.transpose(Hraw[found], (0, 2, 1)))
    return H


def _batch_seeds(seeds, P):
    if seeds is None:
        base = _seed_value(None)
        return (np.arange(P, dtype=np.uint64) + np.uint64(base & 0x7FFFFFFFFFFFFFFF))
    return seeds


def _is_ragged(pts):
    """A list/tuple of per-pair arrays (possibly of different lengths) rather than one [P,N,dim] array."""
    return isinstance(pts, (list, tuple)) and len(pts) > 0 and np.ndim(pts[0]) == 2


def _batch_laf(coef, p1):
    """The single-pair API's treatment of laf_consistensy_coef (utils.py:87-89, 116): dropped with a warning for
    (x, y)-only keypoints, clamped at 0."""
    if p1.shape[-1] == 2 and coef > 0:
        warnings.warn('You set laf_consistensy_coef, but provided only (x,y) keypoints. Skipping LAF check')
        coef = 0
    return max(0, coef)


def findFundamentalMatrixBatch(pts1, pts2, px_th=0.5, conf=0.9999, max_iters=100000, error_type="sampson",
                               symmetric_error_check=True, enable_degeneracy_check=True, seeds=None,
                               return_stats=False, laf_consistensy_coef=-1.0, final_lsq=False, offsets=None, n_max=None):
    """Batched findFundamentalMatrix over P independent pairs: pts [P,N,2] (or [P,N,6] with local affine shapes)
    -> (F [P,3,3], mask [P,N] bool).  Pairs without a model get an all-zero F and an all-False mask row.
    RAGGED batches: pass two lists of [n_i, 2] (or [n_i, 6]) arrays -> (F [P,3,3], list of P bool masks); one kernel
    launch, same results as one call per pair with the same seed.
    CUDA tensors (torch, or any DLPack exporter) stay on the device: see pydegensac_b200.tensor_api.
    final_lsq=True: the reference's compile-time __FINAL_LSQ__ polish (exp_ranF.c:1701-1705).
    offsets=, n_max=: a ragged batch resident on the device (tensor_api; CUDA tensors only), e.g. the output of
    matching.match_descriptors_batch."""
    from . import _cabi
    if not isinstance(pts1, (np.ndarray, list, tuple)):
        from . import tensor_api
        if tensor_api.is_device_tensor(pts1):
            return tensor_api.findFundamentalMatrixBatch(pts1, pts2, px_th, conf, max_iters, error_type,
                                                         symmetric_error_check, enable_degeneracy_check, seeds,
                                                         return_stats, laf_consistensy_coef, final_lsq,
                                                         offsets=offsets, n_max=n_max)
    if offsets is not None:
        raise ValueError("offsets= takes CUDA tensors only")
    et = _error_type(error_type, error_type_dict_fundamental)
    if _is_ragged(pts1):
        F, masks, stats = _cabi.fundamental_ragged(pts1, pts2, px_th, conf, max_iters, et, symmetric_error_check,
                                                   _batch_laf(laf_consistensy_coef, np.asarray(pts1[0])),
                                                   enable_degeneracy_check, _batch_seeds(seeds, len(pts1)))
        return (F, masks, stats) if return_stats else (F, masks)
    p1 = np.asarray(pts1)
    F, mask, stats = _cabi.fundamental_batch(pts1, pts2, px_th, conf, max_iters, et, symmetric_error_check,
                                             _batch_laf(laf_consistensy_coef, p1),
                                             enable_degeneracy_check, _batch_seeds(seeds, p1.shape[0]),
                                             flags=_cabi.FLAG_FINAL_LSQ if final_lsq else 0)
    return (F, mask, stats) if return_stats else (F, mask)


def findHomographyBatch(pts1, pts2, px_th=1.0, conf=0.999, max_iters=50000, error_type="sampson",
                        symmetric_error_check=True, seeds=None, return_stats=False, laf_consistensy_coef=-1.0,
                        final_lsq=False, offsets=None, n_max=None):
    """Batched findHomography: pts [P,N,2] (or [P,N,6]) -> (H [P,3,3] OpenCV convention, mask [P,N] bool).
    RAGGED batches: two lists of [n_i, 2] (or [n_i, 6]) arrays -> (H [P,3,3], list of P bool masks).
    CUDA tensors stay on the device (pydegensac_b200.tensor_api); final_lsq: __FINAL_LSQ__ (exp_ranH.c:866-870).
    offsets=, n_max=: a ragged batch resident on the device (CUDA tensors only)."""
    from . import _cabi
    if not isinstance(pts1, (np.ndarray, list, tuple)):
        from . import tensor_api
        if tensor_api.is_device_tensor(pts1):
            return tensor_api.findHomographyBatch(pts1, pts2, px_th, conf, max_iters, error_type, symmetric_error_check,
                                                  seeds, return_stats, laf_consistensy_coef, final_lsq,
                                                  offsets=offsets, n_max=n_max)
    if offsets is not None:
        raise ValueError("offsets= takes CUDA tensors only")
    et = _error_type(error_type, error_type_dict_homography)
    if _is_ragged(pts1):
        Hraw, masks, stats = _cabi.homography_ragged(pts1, pts2, px_th, conf, max_iters, et, symmetric_error_check,
                                                     _batch_laf(laf_consistensy_coef, np.asarray(pts1[0])),
                                                     _batch_seeds(seeds, len(pts1)))
        H = _opencv_convention(Hraw)
        return (H, masks, stats) if return_stats else (H, masks)
    p1 = np.asarray(pts1)
    Hraw, mask, stats = _cabi.homography_batch(pts1, pts2, px_th, conf, max_iters, et, symmetric_error_check,
                                               _batch_laf(laf_consistensy_coef, p1), _batch_seeds(seeds, p1.shape[0]),
                                               flags=_cabi.FLAG_FINAL_LSQ if final_lsq else 0)
    H = _opencv_convention(Hraw)
    return (H, mask, stats) if return_stats else (H, mask)


def laf_to_ellipse_frame(xyA):
    """[N,6] rows (x, y, a11, a12, a21, a22) (convert_cv2_kpts_to_xyA) -> [N,5] rows (x, y, a, b, c): the SAME ellipse
    A * unit-circle written as the lower-triangular frame [a 0; b c] with a, c > 0 that ransacH2el takes (ranH2el.h:4,
    getTransf ranH2el.c:211-231).  A = L Q with Q a rotation: L L^T = A A^T (Cholesky)."""
    k = np.asarray(xyA, dtype=np.float64)
    if k.ndim != 2 or k.shape[1] != 6:
        raise ValueError("expected [N,6] rows (x, y, a11, a12, a21, a22)")
    a11, a12, a21, a22 = k[:, 2], k[:, 3], k[:, 4], k[:, 5]
    s11 = a11 * a11 + a12 * a12
    s21 = a21 * a11 + a22 * a12
    s22 = a21 * a21 + a22 * a22
    a = np.sqrt(s11)
    b = s21 / a
    c = np.sqrt(np.maximum(s22 - b * b, 0.0))
    return np.stack([k[:, 0], k[:, 1], a, b, c], axis=1)


def findHomographyFromEllipses(frames1, frames2, px_th=1.0, conf=0.999, max_iters=50000, seed=None, seeds=None,
                               return_stats=False):
    """Homography from correspondences of local elliptical features, two correspondences per sample: the reference
    core's ransacH2el (ranH2el.c:19), which the reference never bound to Python.
    frames1, frames2: [N,5] (or [P,N,5]) rows (x, y, a, b, c) -- centre and lower-triangular frame [a 0; b c] of the
    feature in image 1 / image 2 (`laf_to_ellipse_frame` converts [N,6] keypoints).  px_th bounds the Sampson error of
    the centres (th = px_th^2).  Returns (H, mask) in the findHomography convention: H maps image 1 -> image 2."""
    from . import _cabi
    f1 = np.asarray(frames1, dtype=np.float64)
    f2 = np.asarray(frames2, dtype=np.float64)
    if f1.shape != f2.shape or f1.ndim not in (2, 3) or f1.shape[-1] != 5:
        raise ValueError("frames1, frames2 should be arrays with dims [n,5] (x, y, a, b, c)")
    single = f1.ndim == 2
    if single:
        f1, f2 = f1[None], f2[None]
    P = f1.shape[0]
    if seeds is None:
        seeds = np.full(P, _seed_value(seed), dtype=np.uint64) if single else _batch_seeds(None, P)
    u10 = np.concatenate([f1, f2], axis=2)
    Hraw, mask, stats = _cabi.homography_2el_batch(u10, px_th, conf, max_iters, seeds)
    H = _opencv_convention(Hraw)
    if single:
        H, mask, stats = H[0], mask[0], stats[0]
    return (H, mask, stats) if return_stats else (H, mask)
