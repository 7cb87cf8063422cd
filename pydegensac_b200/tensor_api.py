"""Device-resident entry points: correspondences that already live in GPU memory (torch CUDA tensors, or anything that
speaks DLPack -- CuPy, JAX, Numba device arrays) go straight into the RANSAC kernel and the results stay on the device.

This is SURVEY.md section 8(f).3 "the step before the path": the reference's pipeline builds `src_pts/dst_pts` on the
host from cv2 matches (examples/simple-example.py:26-27, 46-53); here a GPU matcher (pydegensac_b200.matching) or any
other GPU front-end hands its [N,2] tensors over without a host round trip.

    F, mask = findFundamentalMatrixBatch(pts1, pts2, 1.0, 0.9999, 10000)        # pts: [P,N,2] cuda float64 tensors
    H, mask = findHomographyBatch(pts1, pts2, 3.0)                              # H in OpenCV convention (x2 ~ H x1)

Arguments, defaults and conventions are those of `pydegensac_b200.utils` (which dispatches here when it is given CUDA
tensors); outputs are torch tensors on the inputs' device.  Asynchronous with respect to the host: the kernel is
enqueued on the current torch stream.
"""
import numpy as np

from . import _cabi
from .utils import (_error_type, _batch_laf, _seed_value, error_type_dict_fundamental, error_type_dict_homography)


def _torch():
    import torch
    return torch


def is_device_tensor(x):
    """True for a torch CUDA tensor or a non-torch object exporting DLPack from a CUDA device."""
    try:
        torch = _torch()
    except ImportError:   # pragma: no cover
        return False
    if isinstance(x, torch.Tensor):
        return x.is_cuda
    if isinstance(x, (np.ndarray, list, tuple)):
        return False
    if hasattr(x, "__dlpack__") and hasattr(x, "__dlpack_device__"):
        try:
            return int(x.__dlpack_device__()[0]) == 2      # kDLCUDA
        except Exception:
            return False
    return False


def as_device_f64(x):
    """[P,N,dim] (or [N,dim]) contiguous float64 CUDA tensor from a torch tensor / DLPack object; no host copy."""
    torch = _torch()
    t = x if isinstance(x, torch.Tensor) else torch.from_dlpack(x)
    if not t.is_cuda:
        raise ValueError("expected a CUDA tensor")
    if t.dim() == 2:
        t = t[None]
    if t.dim() != 3 or t.shape[2] not in (2, 6):
        raise ValueError("expected correspondences of shape [P,N,2] or [P,N,6]")
    return t.to(torch.float64).contiguous()


def _seeds_tensor(seeds, P, device):
    torch = _torch()
    if seeds is None:
        base = _seed_value(None) & 0x3FFFFFFFFFFFFFFF
        return torch.arange(P, dtype=torch.int64, device=device) + base
    if isinstance(seeds, torch.Tensor):
        return seeds.to(device=device, dtype=torch.int64).contiguous()
    s = np.ascontiguousarray(np.broadcast_to(np.asarray(seeds, dtype=np.uint64), (P,)))
    return torch.from_numpy(s.view(np.int64).copy()).to(device)


def _launch(kind, p1, p2, px_th, conf, max_iters, et, sym, laf, degen, seeds, flags=0):
    torch = _torch()
    if p1.shape != p2.shape or p1.device != p2.device:
        raise ValueError("pts1 and pts2 must have the same shape and device")
    P, N, dim = p1.shape
    dev = p1.device
    with torch.cuda.device(dev):
        _cabi.lib().dgb200_set_device(dev.index if dev.index is not None else torch.cuda.current_device())
        model = torch.zeros((P, 3, 3), dtype=torch.float64, device=dev)
        mask = torch.zeros((P, N), dtype=torch.uint8, device=dev)
        stats = torch.zeros((P, 4), dtype=torch.int32, device=dev)
        ds = _seeds_tensor(seeds, P, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        if kind == 0:
            _cabi.fundamental_batch_dev(p1.data_ptr(), p2.data_ptr(), P, N, dim, px_th, conf, max_iters, et, sym, laf,
                                        degen, ds.data_ptr(), model.data_ptr(), mask.data_ptr(), stats.data_ptr(), stream,
                                        flags=flags)
        else:
            _cabi.homography_batch_dev(p1.data_ptr(), p2.data_ptr(), P, N, dim, px_th, conf, max_iters, et, sym, laf,
                                       ds.data_ptr(), model.data_ptr(), mask.data_ptr(), stats.data_ptr(), stream,
                                       flags=flags)
        # the inputs must outlive the asynchronous kernel: tie them to the stream
        for t in (p1, p2, ds):
            t.record_stream(torch.cuda.current_stream(dev))
    return model, mask, stats


def _launch_ragged(kind, pts1, pts2, offsets, n_max, px_th, conf, max_iters, et, sym, laf_coef, degen, seeds, final_lsq):
    """Ragged batch on the device: pts [rows, 2|6] CUDA tensors, pair p owns rows offsets[p] .. offsets[p+1]-1
    (offsets: int32 CUDA tensor [P+1], e.g. from matching.match_descriptors_batch; n_max: a host int >= every pair's
    length).  Nothing is read back: the kernel skips pairs that are too short or longer than n_max (zero model, False
    mask rows, zero stats).  Returns (model [P,3,3], mask [rows] uint8, stats [P,4])."""
    torch = _torch()
    if final_lsq:
        raise ValueError("final_lsq is not available with offsets=")
    if n_max is None:
        raise ValueError("offsets= needs n_max, the largest pair's row count (reading it from the device would synchronise)")
    if not (isinstance(offsets, torch.Tensor) and offsets.is_cuda and offsets.dim() == 1 and offsets.shape[0] >= 2):
        raise ValueError("offsets must be a CUDA tensor [P+1]")
    p1 = pts1 if isinstance(pts1, torch.Tensor) else torch.from_dlpack(pts1)
    p2 = pts2 if isinstance(pts2, torch.Tensor) else torch.from_dlpack(pts2)
    if not p1.is_cuda or p1.dim() != 2 or p1.shape[1] not in (2, 6) or p1.shape != p2.shape or p1.device != p2.device \
            or offsets.device != p1.device:
        raise ValueError("with offsets=, pts1 and pts2 must be CUDA tensors [rows, 2] or [rows, 6] on the offsets' device")
    p1, p2 = p1.to(torch.float64).contiguous(), p2.to(torch.float64).contiguous()
    off = offsets.to(torch.int32).contiguous()
    P = int(off.shape[0]) - 1
    rows, dim = int(p1.shape[0]), int(p1.shape[1])
    laf = _batch_laf(laf_coef, p1)
    n_max = max(int(n_max), 8 if kind == 0 else 4)   # the slabs need room for one minimal sample; shorter pairs are skipped
    dev = p1.device
    with torch.cuda.device(dev):
        _cabi.lib().dgb200_set_device(dev.index if dev.index is not None else torch.cuda.current_device())
        model = torch.zeros((P, 3, 3), dtype=torch.float64, device=dev)
        mask = torch.zeros(max(rows, 1), dtype=torch.uint8, device=dev)
        stats = torch.zeros((P, 4), dtype=torch.int32, device=dev)
        ds = _seeds_tensor(seeds, P, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        args = (p1.data_ptr(), p2.data_ptr(), off.data_ptr(), P, n_max, dim, px_th, conf, max_iters, et, sym, laf)
        if kind == 0:
            _cabi.fundamental_ragged_dev(*args, degen, ds.data_ptr(), model.data_ptr(), mask.data_ptr(), stats.data_ptr(),
                                         stream)
        else:
            _cabi.homography_ragged_dev(*args, ds.data_ptr(), model.data_ptr(), mask.data_ptr(), stats.data_ptr(), stream)
    return model, mask[:rows], stats


def _opencv_convention_nosync(Hraw):
    """inv(H.T) per pair on the device without reading anything back: all-zero and singular models give all-zero H."""
    torch = _torch()
    Ht = Hraw.transpose(1, 2)
    good = (Hraw.abs().sum(dim=(1, 2)) != 0) & (torch.linalg.det(Ht).abs() > 0)
    eye = torch.eye(3, dtype=Hraw.dtype, device=Hraw.device).expand_as(Ht)
    inv, _ = torch.linalg.inv_ex(torch.where(good[:, None, None], Ht, eye))
    return torch.where(good[:, None, None], inv, torch.zeros_like(inv))


def findFundamentalMatrixBatch(pts1, pts2, px_th=0.5, conf=0.9999, max_iters=100000, error_type="sampson",
                               symmetric_error_check=True, enable_degeneracy_check=True, seeds=None,
                               return_stats=False, laf_consistensy_coef=-1.0, final_lsq=False, offsets=None, n_max=None):
    """Device-resident batched findFundamentalMatrix: CUDA tensors in, CUDA tensors out
    (F [P,3,3] float64, mask [P,N] bool[, stats [P,4] int32]).
    offsets= (int32 CUDA [P+1]) with n_max: a ragged batch, pts [rows, 2|6] -> mask [rows] bool aligned with pts."""
    et = _error_type(error_type, error_type_dict_fundamental)
    if offsets is not None:
        F, mask, stats = _launch_ragged(0, pts1, pts2, offsets, n_max, float(px_th), float(conf), int(max_iters), et,
                                        bool(symmetric_error_check), laf_consistensy_coef, bool(enable_degeneracy_check),
                                        seeds, final_lsq)
        mask = mask.view(_torch().bool)
        return (F, mask, stats) if return_stats else (F, mask)
    p1, p2 = as_device_f64(pts1), as_device_f64(pts2)
    laf = _batch_laf(laf_consistensy_coef, p1)
    F, mask, stats = _launch(0, p1, p2, float(px_th), float(conf), int(max_iters), et, bool(symmetric_error_check), laf,
                             bool(enable_degeneracy_check), seeds, flags=_cabi.FLAG_FINAL_LSQ if final_lsq else 0)
    mask = mask.view(_torch().bool)
    return (F, mask, stats) if return_stats else (F, mask)


def findHomographyBatch(pts1, pts2, px_th=1.0, conf=0.999, max_iters=50000, error_type="sampson",
                        symmetric_error_check=True, seeds=None, return_stats=False, laf_consistensy_coef=-1.0,
                        final_lsq=False, offsets=None, n_max=None):
    """Device-resident batched findHomography: H [P,3,3] in the OpenCV convention (x2 ~ H x1; the core's raw
    column-major image2->image1 model is inverted/transposed on the device, utils.py:108), mask [P,N] bool.
    offsets= (int32 CUDA [P+1]) with n_max: a ragged batch, pts [rows, 2|6] -> mask [rows] bool aligned with pts."""
    torch = _torch()
    et = _error_type(error_type, error_type_dict_homography)
    if offsets is not None:
        Hraw, mask, stats = _launch_ragged(1, pts1, pts2, offsets, n_max, float(px_th), float(conf), int(max_iters), et,
                                           bool(symmetric_error_check), laf_consistensy_coef, False, seeds, final_lsq)
        H = _opencv_convention_nosync(Hraw)
        mask = mask.view(torch.bool)
        return (H, mask, stats) if return_stats else (H, mask)
    p1, p2 = as_device_f64(pts1), as_device_f64(pts2)
    laf = _batch_laf(laf_consistensy_coef, p1)
    Hraw, mask, stats = _launch(1, p1, p2, float(px_th), float(conf), int(max_iters), et, bool(symmetric_error_check),
                                laf, False, seeds, flags=_cabi.FLAG_FINAL_LSQ if final_lsq else 0)
    ok = Hraw.abs().sum(dim=(1, 2)) != 0
    H = torch.zeros_like(Hraw)
    if bool(ok.any()):
        # inv(H.T) per pair; singular models (the reference raises LinAlgError) are reported as all-zero
        Ht = Hraw.transpose(1, 2)
        det = torch.linalg.det(Ht)
        good = ok & (det.abs() > 0)
        if bool(good.any()):
            H[good] = torch.linalg.inv(Ht[good])
    mask = mask.view(torch.bool)
    return (H, mask, stats) if return_stats else (H, mask)
