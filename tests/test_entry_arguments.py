"""The argument checks of the public entry points, message for message.  Python: every public function of
matching.py, one malformed argument per case, with the exact ValueError text; "well-formed but on the host" is one of
the cases, so these run without a GPU.  C: the five ragged pose and refine entry points of the front end, with the
exact message and return code of every refused case, through fake pointers that are never dereferenced."""
import ctypes
import math
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def _torch():
    return pytest.importorskip("torch")


def _raises(fn, args, message):
    with pytest.raises(ValueError) as e:
        fn(**args)
    assert str(e.value) == message


# ------------------------------------------------------------------------------------------------ Python
def _pair_inputs(torch, model):
    f64 = torch.float64
    return {model: torch.zeros((2, 3, 3), dtype=f64), "pts1": torch.zeros((10, 2), dtype=f64),
            "pts2": torch.zeros((10, 2), dtype=f64), "offsets": torch.tensor([0, 4, 10], dtype=torch.int32)}


def _model_cases(torch, m):
    """the cases of a [P,3,3] model named m, its rows, offsets and mask, in the order the checks run"""
    f64, i32 = torch.float64, torch.int32
    return [
        ({m: np.zeros((2, 3, 3))}, "%s must be a torch tensor" % m),
        ({"pts1": np.zeros((10, 2))}, "pts1 must be a torch tensor"),
        ({"pts2": [[0.0, 0.0]] * 10}, "pts2 must be a torch tensor"),
        ({"offsets": np.array([0, 4, 10], np.int32)}, "offsets must be a torch tensor"),
        ({"mask": np.ones(10, bool)}, "mask must be a torch tensor"),
        ({m: torch.zeros((2, 8), dtype=f64)}, "%s must be [P,3,3] or [P,9] with P >= 1, not [2, 8]" % m),
        ({m: torch.zeros((0, 9), dtype=f64)}, "%s must be [P,3,3] or [P,9] with P >= 1, not [0, 9]" % m),
        ({m: torch.zeros(9, dtype=f64)}, "%s must be [P,3,3] or [P,9] with P >= 1, not [9]" % m),
        ({m: torch.zeros((2, 3, 3, 1), dtype=f64)}, "%s must be [P,3,3] or [P,9] with P >= 1, not [2, 3, 3, 1]" % m),
        ({"pts1": torch.zeros((10, 1), dtype=f64), "pts2": torch.zeros((10, 1), dtype=f64)},
         "pts1 and pts2 must be [rows, 2|6] tensors of one shape"),
        ({"pts2": torch.zeros((9, 2), dtype=f64)}, "pts1 and pts2 must be [rows, 2|6] tensors of one shape"),
        ({"pts1": torch.zeros(10, dtype=f64)}, "pts1 and pts2 must be [rows, 2|6] tensors of one shape"),
        ({"offsets": torch.tensor([0, 10], dtype=i32)}, "offsets must be [P+1] = [3], not [2]"),
        ({"offsets": torch.tensor([[0, 4, 10]], dtype=i32)}, "offsets must be [P+1] = [3], not [1, 3]"),
        ({"offsets": torch.tensor([0, 4, 10])}, "offsets must be int32, not torch.int64"),
        ({m: torch.zeros((2, 9), dtype=torch.int64)}, "%s must be a floating tensor, not torch.int64" % m),
        ({"pts1": torch.zeros((10, 2), dtype=torch.int64)}, "pts1 must be a floating tensor, not torch.int64"),
        ({"pts2": torch.zeros((10, 2), dtype=i32)}, "pts2 must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(9, dtype=torch.bool)}, "mask must be [rows] = [10], not [9]"),
        ({"mask": torch.ones((10, 1), dtype=torch.bool)}, "mask must be [rows] = [10], not [10, 1]"),
        ({"mask": torch.ones(10, dtype=i32)}, "mask must be bool or uint8, not torch.int32"),
        ({"mask": torch.ones(9, dtype=i32)}, "mask must be [rows] = [10], not [9]"),
        ({m: torch.zeros((2, 8), dtype=torch.int64)}, "%s must be [P,3,3] or [P,9] with P >= 1, not [2, 8]" % m),
        ({"offsets": torch.tensor([0, 10])}, "offsets must be [P+1] = [3], not [2]"),
    ]


def _k_cases(torch):
    f64 = torch.float64
    return [
        ({"K1": np.eye(3)}, "K1 must be a torch tensor"),
        ({"K2": None}, "K2 must be a torch tensor"),
        ({"K1": torch.eye(4, dtype=f64)}, "K1 must be [3,3] or [P,3,3] with P = 2, not [4, 4]"),
        ({"K2": torch.zeros((3, 3, 3), dtype=f64)}, "K2 must be [3,3] or [P,3,3] with P = 2, not [3, 3, 3]"),
        ({"K1": torch.eye(3, dtype=torch.int32)}, "K1 must be a floating tensor, not torch.int32"),
        ({"K2": torch.eye(3, dtype=torch.int64)}, "K2 must be a floating tensor, not torch.int64"),
        ({"K1": torch.eye(4, dtype=torch.int32), "offsets": torch.tensor([0, 10])},
         "K1 must be [3,3] or [P,3,3] with P = 2, not [4, 4]"),
    ]


def _pose_ragged(model):
    torch = _torch()
    f64 = torch.float64
    good = dict(_pair_inputs(torch, model), K1=torch.eye(3, dtype=f64), K2=torch.eye(3, dtype=f64).repeat(2, 1, 1))
    cases = _model_cases(torch, model) + _k_cases(torch) + [
        ({}, "%s, K1, K2, pts1, pts2, offsets and mask must be CUDA tensors on one device" % model),
        ({"mask": torch.ones(10, dtype=torch.uint8)},
         "%s, K1, K2, pts1, pts2, offsets and mask must be CUDA tensors on one device" % model),
    ]
    return good, cases


def test_pose_from_fundamental_ragged_messages():
    from pydegensac_b200.matching import pose_from_fundamental_ragged
    good, cases = _pose_ragged("F")
    for kw, msg in cases:
        _raises(pose_from_fundamental_ragged, dict(good, **kw), msg)


def test_pose_from_homography_ragged_messages():
    from pydegensac_b200.matching import pose_from_homography_ragged
    good, cases = _pose_ragged("H")
    for kw, msg in cases:
        _raises(pose_from_homography_ragged, dict(good, **kw), msg)


def _scalar_cases():
    return [
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"max_iters": -2.7}, "max_iters must not be negative, not -2"),
        ({"px_th": -0.5}, "px_th must be a non-negative number, not -0.5"),
        ({"px_th": float("nan")}, "px_th must be a non-negative number, not nan"),
        ({"px_th": -0.5, "max_iters": -1}, "max_iters must not be negative, not -1"),
    ]


def test_refine_pose_ragged_messages():
    torch = _torch()
    from pydegensac_b200.matching import refine_pose_ragged
    f64 = torch.float64
    good = dict(_pair_inputs(torch, "R"), t=torch.ones((2, 3), dtype=f64), K1=torch.eye(3, dtype=f64),
                K2=torch.eye(3, dtype=f64))
    host = "R, t, K1, K2, pts1, pts2, offsets and mask must be CUDA tensors on one device"
    cases = _model_cases(torch, "R") + _k_cases(torch) + _scalar_cases() + [
        ({"t": np.ones((2, 3))}, "t must be a torch tensor"),
        ({"t": torch.ones((3, 3), dtype=f64)}, "t must be [P,3] = [2,3], not [3, 3]"),
        ({"t": torch.ones(6, dtype=f64)}, "t must be [P,3] = [2,3], not [6]"),
        ({"t": torch.ones((2, 3), dtype=torch.int32)}, "t must be a floating tensor, not torch.int32"),
        ({"t": torch.ones(6, dtype=f64), "pts2": torch.zeros((9, 2), dtype=f64)}, "t must be [P,3] = [2,3], not [6]"),
        ({"mask": torch.ones(9, dtype=torch.bool), "max_iters": -1}, "mask must be [rows] = [10], not [9]"),
        ({"px_th": 1.0}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(refine_pose_ragged, dict(good, **kw), msg)


@pytest.mark.parametrize("model", ["H", "F"])
def test_refine_model_ragged_messages(model):
    torch = _torch()
    from pydegensac_b200 import matching
    fn = matching.refine_homography_ragged if model == "H" else matching.refine_fundamental_ragged
    good = _pair_inputs(torch, model)
    host = "%s, pts1, pts2, offsets and mask must be CUDA tensors on one device" % model
    cases = _model_cases(torch, model) + _scalar_cases() + [
        ({"mask": torch.ones(9, dtype=torch.bool), "max_iters": -1}, "mask must be [rows] = [10], not [9]"),
        ({"px_th": 2.0, "mask": torch.ones(10, dtype=torch.bool)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(fn, dict(good, **kw), msg)


def test_find_absolute_pose_ragged_messages():
    torch = _torch()
    from pydegensac_b200.matching import find_absolute_pose_ragged
    f64, i32 = torch.float64, torch.int32
    good = dict(pts2d=torch.zeros((10, 2), dtype=f64), pts3d=torch.zeros((10, 3), dtype=f64),
                K=torch.eye(3, dtype=f64), offsets=torch.tensor([0, 4, 10], dtype=i32))
    host = "pts2d, pts3d, K, offsets and mask must be CUDA tensors on one device"
    cases = [
        ({"pts2d": np.zeros((10, 2))}, "pts2d must be a torch tensor"),
        ({"pts3d": None}, "pts3d must be a torch tensor"),
        ({"K": np.eye(3)}, "K must be a torch tensor"),
        ({"offsets": [0, 4, 10]}, "offsets must be a torch tensor"),
        ({"mask": np.ones(10, bool)}, "mask must be a torch tensor"),
        ({"offsets": torch.tensor([0], dtype=i32)}, "offsets must be [P+1] with P >= 1, not [1]"),
        ({"offsets": torch.tensor([[0, 4, 10]], dtype=i32)}, "offsets must be [P+1] with P >= 1, not [1, 3]"),
        ({"offsets": torch.tensor([0, 4, 10])}, "offsets must be int32, not torch.int64"),
        ({"offsets": torch.tensor([0])}, "offsets must be [P+1] with P >= 1, not [1]"),
        ({"pts2d": torch.zeros((10, 3), dtype=f64)}, "pts2d must be [rows,2], not [10, 3]"),
        ({"pts2d": torch.zeros(10, dtype=f64)}, "pts2d must be [rows,2], not [10]"),
        ({"pts3d": torch.zeros((9, 3), dtype=f64)}, "pts3d must be [rows,3] = [10,3], not [9, 3]"),
        ({"pts3d": torch.zeros((10, 2), dtype=f64)}, "pts3d must be [rows,3] = [10,3], not [10, 2]"),
        ({"K": torch.eye(4, dtype=f64)}, "K must be [3,3] or [P,3,3] with P = 2, not [4, 4]"),
        ({"K": torch.eye(3, dtype=f64).repeat(3, 1, 1)}, "K must be [3,3] or [P,3,3] with P = 2, not [3, 3, 3]"),
        ({"pts2d": torch.zeros((10, 2), dtype=i32)}, "pts2d must be a floating tensor, not torch.int32"),
        ({"pts3d": torch.zeros((10, 3), dtype=torch.int64)}, "pts3d must be a floating tensor, not torch.int64"),
        ({"K": torch.eye(3, dtype=i32)}, "K must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(9, dtype=torch.bool)}, "mask must be [rows] = [10], not [9]"),
        ({"mask": torch.ones(10, dtype=i32)}, "mask must be bool or uint8, not torch.int32"),
        ({"px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"px_th": -1.0}, "px_th must be a positive number, not -1.0"),
        ({"px_th": float("inf")}, "px_th must be a positive number, not inf"),
        ({"px_th": float("nan")}, "px_th must be a positive number, not nan"),
        ({"conf": 0.0}, "conf must lie in (0, 1], not 0.0"),
        ({"conf": 1.5}, "conf must lie in (0, 1], not 1.5"),
        ({"conf": float("nan")}, "conf must lie in (0, 1], not nan"),
        ({"max_iters": 0}, "max_iters must be at least 1, not 0"),
        ({"refine_iters": -1}, "refine_iters must not be negative, not -1"),
        ({"refine_iters": -1, "px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"max_iters": 0, "conf": 2.0}, "conf must lie in (0, 1], not 2.0"),
        ({"mask": torch.ones(10, dtype=torch.bool)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(find_absolute_pose_ragged, dict(good, **kw), msg)


def _track_inputs(torch):
    f64, i32 = torch.float64, torch.int32
    return dict(cams=torch.zeros(10, dtype=i32), pts=torch.zeros((10, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(4, 1, 1), t=torch.zeros((4, 3), dtype=f64), K=torch.eye(3, dtype=f64),
                offsets=torch.tensor([0, 4, 10], dtype=i32))


def _track_cases(torch):
    """the cases triangulate_tracks_ragged and bundle_adjust_ragged share, in the order the checks run"""
    f64, i32 = torch.float64, torch.int32
    return [
        ({"cams": np.zeros(10, np.int32)}, "cams must be a torch tensor"),
        ({"pts": np.zeros((10, 2))}, "pts must be a torch tensor"),
        ({"R": np.eye(3)}, "R must be a torch tensor"),
        ({"t": None}, "t must be a torch tensor"),
        ({"K": np.eye(3)}, "K must be a torch tensor"),
        ({"offsets": [0, 4, 10]}, "offsets must be a torch tensor"),
        ({"mask": np.ones(10, bool)}, "mask must be a torch tensor"),
        ({"offsets": torch.tensor([0], dtype=i32)}, "offsets must be [T+1] with T >= 1, not [1]"),
        ({"offsets": torch.tensor([[0, 4, 10]], dtype=i32)}, "offsets must be [T+1] with T >= 1, not [1, 3]"),
        ({"offsets": torch.tensor([0, 4, 10])}, "offsets must be int32, not torch.int64"),
        ({"cams": torch.zeros(10, dtype=torch.int64)}, "cams must be int32, not torch.int64"),
        ({"cams": torch.zeros(10, dtype=f64), "offsets": torch.tensor([0, 4, 10])},
         "offsets must be int32, not torch.int64"),
        ({"pts": torch.zeros((10, 3), dtype=f64)}, "pts must be [obs,2], not [10, 3]"),
        ({"pts": torch.zeros(10, dtype=f64)}, "pts must be [obs,2], not [10]"),
        ({"cams": torch.zeros(9, dtype=i32)}, "cams must be [obs] = [10], not [9]"),
        ({"R": torch.eye(3, dtype=f64)}, "R must be [C,3,3] with C >= 1, not [3, 3]"),
        ({"R": torch.zeros((0, 3, 3), dtype=f64)}, "R must be [C,3,3] with C >= 1, not [0, 3, 3]"),
        ({"R": torch.zeros((4, 9), dtype=f64)}, "R must be [C,3,3] with C >= 1, not [4, 9]"),
        ({"t": torch.zeros((3, 3), dtype=f64)}, "t must be [C,3] = [4,3], not [3, 3]"),
        ({"K": torch.eye(3, dtype=f64).repeat(3, 1, 1)}, "K must be [3,3] or [C,3,3] with C = 4, not [3, 3, 3]"),
        ({"pts": torch.zeros((10, 2), dtype=i32)}, "pts must be a floating tensor, not torch.int32"),
        ({"R": torch.eye(3, dtype=i32).repeat(4, 1, 1)}, "R must be a floating tensor, not torch.int32"),
        ({"t": torch.zeros((4, 3), dtype=torch.int64)}, "t must be a floating tensor, not torch.int64"),
        ({"K": torch.eye(3, dtype=i32)}, "K must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(9, dtype=torch.bool)}, "mask must be [obs] = [10], not [9]"),
        ({"mask": torch.ones(10, dtype=i32)}, "mask must be bool or uint8, not torch.int32"),
        ({"px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"px_th": float("nan")}, "px_th must be a positive number, not nan"),
        ({"px_th": float("inf")}, "px_th must be a positive number, not inf"),
    ]


def test_triangulate_tracks_ragged_messages():
    torch = _torch()
    from pydegensac_b200.matching import triangulate_tracks_ragged
    good = _track_inputs(torch)
    host = "cams, pts, R, t, K, offsets and mask must be CUDA tensors on one device"
    cases = _track_cases(torch) + [
        ({"max_iters": -1, "px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"min_angle": -0.1}, "min_angle must lie in [0, pi), not -0.1"),
        ({"min_angle": math.pi}, "min_angle must lie in [0, pi), not %r" % math.pi),
        ({"conf": 0.0}, "conf must lie in (0, 1], not 0.0"),
        ({"conf": 1.01}, "conf must lie in (0, 1], not 1.01"),
        ({"max_iters": 0}, "max_iters must be at least 1, not 0"),
        ({"refine_iters": -1}, "refine_iters must not be negative, not -1"),
        ({"refine_iters": -1, "conf": 0.0}, "conf must lie in (0, 1], not 0.0"),
        ({"mask": torch.ones(10, dtype=torch.uint8)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(triangulate_tracks_ragged, dict(good, **kw), msg)


def test_bundle_adjust_ragged_messages():
    torch = _torch()
    from pydegensac_b200.matching import bundle_adjust_ragged
    f64 = torch.float64
    good = dict(_track_inputs(torch), X=torch.zeros((2, 3), dtype=f64))
    host = "cams, pts, R, t, K, offsets, X and mask must be CUDA tensors on one device"
    cases = _track_cases(torch) + [
        ({"X": np.zeros((2, 3))}, "X must be a torch tensor"),
        ({"X": torch.zeros((3, 3), dtype=f64)}, "X must be [T,3] = [2,3], not [3, 3]"),
        ({"X": torch.zeros((2, 3), dtype=torch.int64)}, "X must be a floating tensor, not torch.int64"),
        ({"X": torch.zeros((2, 3), dtype=torch.int64), "K": torch.eye(3, dtype=torch.int32)},
         "K must be a floating tensor, not torch.int32"),
        ({"free": [1, 1]}, "free holds a camera twice"),
        ({"free": [4]}, "free holds a camera index outside [0, 4)"),
        ({"free": [-1]}, "free holds a camera index outside [0, 4)"),
        ({"free": list(range(65))}, "free holds 65 cameras, more than 64"),
        ({"free": "x"}, "free must be a host sequence of camera indices"),
        ({"R": torch.eye(3, dtype=f64).repeat(66, 1, 1), "t": torch.zeros((66, 3), dtype=f64)},
         "free=None frees 65 cameras, more than 64: pass an explicit free list"),
        ({"scale_gauge": 0}, "scale_gauge 0 is not one of the free cameras"),
        ({"scale_gauge": "first"}, "scale_gauge must be 'auto', None or a camera of free, not 'first'"),
        ({"free": [0, 1, 2, 3], "scale_gauge": 1}, "scale_gauge needs a held camera: every camera is free"),
        ({"loss_scale": 0.0}, "loss_scale must be a positive number or None, not 0.0"),
        ({"loss_scale": float("nan")}, "loss_scale must be a positive number or None, not nan"),
        ({"loss_scale": float("inf")}, "loss_scale must be a positive number or None, not inf"),
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"max_iters": -1, "px_th": 0.0}, "max_iters must not be negative, not -1"),
        ({"max_iters": 0, "scale_gauge": None, "loss_scale": 1.0}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(bundle_adjust_ragged, dict(good, **kw), msg)


def test_pose_from_fundamental_messages():
    torch = _torch()
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200.matching import pose_from_fundamental
    f64 = torch.float64
    good = dict(F=torch.zeros((2, 3, 3), dtype=f64), K1=torch.eye(3, dtype=f64), K2=torch.eye(3, dtype=f64),
                pts1=torch.zeros((2, 8, 2), dtype=f64), pts2=torch.zeros((2, 8, 2), dtype=f64))
    _raises(pose_from_fundamental, good, "Expected a cuda device, but got: cpu")


def test_match_descriptors_messages():
    torch = _torch()
    from pydegensac_b200.matching import match_descriptors
    d = torch.zeros((5, 8))
    b = torch.zeros((5, 32), dtype=torch.uint8)
    cases = [
        (dict(desc1=d, desc2=d, norm="l1"), "norm must be 'l2' or 'hamming', not 'l1'"),
        (dict(desc1=d, desc2=d), "expected two CUDA descriptor tensors [n1,D], [n2,D] on the same device"),
        (dict(desc1=d, desc2=torch.zeros((5, 4))),
         "expected two CUDA descriptor tensors [n1,D], [n2,D] on the same device"),
        (dict(desc1=d, desc2=d, norm="hamming"),
         "norm='hamming' takes uint8 descriptor tensors [n, B] (the layout cv2 returns)"),
        (dict(desc1=b, desc2=b[0], norm="hamming"), "expected binary descriptor tensors [n, B]"),
        (dict(desc1=b, desc2=b[:, :16], norm="hamming"),
         "binary descriptors of one call must all have the same length in bytes"),
        (dict(desc1=b[:, :0], desc2=b[:, :0], norm="hamming"), "binary descriptors must be 1 to 256 bytes long, not 0"),
        (dict(desc1=b, desc2=b, norm="hamming"), "expected CUDA descriptor tensors on one device"),
    ]
    for kw, msg in cases:
        _raises(match_descriptors, kw, msg)


def test_match_descriptors_batch_and_guided_messages():
    torch = _torch()
    from pydegensac_b200.matching import batch_layout, match_descriptors_batch, match_descriptors_guided
    d = [torch.zeros((5, 8)), torch.zeros((6, 8))]
    kps = [torch.zeros((5, 2)), torch.zeros((6, 2))]
    pairs = [[0, 1]]
    models = np.zeros((1, 9))
    batch = [
        (dict(descs=d, pairs=pairs, norm="x"), "norm must be 'l2' or 'hamming', not 'x'"),
        (dict(descs=[], pairs=pairs), "expected a non-empty list of descriptor tensors"),
        (dict(descs=d, pairs=pairs), "expected CUDA descriptor tensors [n_i, D] with one D, on one device"),
        (dict(descs=[torch.zeros((5, 8), dtype=torch.float32)] * 2, pairs=pairs, norm="hamming"),
         "norm='hamming' takes uint8 descriptor tensors [n, B] (the layout cv2 returns)"),
    ]
    for kw, msg in batch:
        _raises(match_descriptors_batch, kw, msg)
    guided = [
        (dict(guide="E"), "guide must be 'F' or 'H', not 'E'"),
        (dict(px_th=-1.0), "px_th must be a non-negative number, not -1.0"),
        (dict(px_th=float("nan"), guide="X"), "guide must be 'F' or 'H', not 'X'"),
        (dict(norm="l1"), "norm must be 'l2' or 'hamming', not 'l1'"),
        (dict(kps=None), "guided matching needs the keypoints of every image (kps)"),
        (dict(models=np.zeros((2, 9))), "models must be [P,3,3] or [P,9] with P = 1 pairs, not [2, 9]"),
        (dict(models=torch.zeros((1, 8))), "models must be [P,3,3] or [P,9] with P = 1 pairs, not [1, 8]"),
        (dict(), "expected CUDA descriptor tensors [n_i, D] with one D, on one device"),
    ]
    for kw, msg in guided:
        _raises(match_descriptors_guided, dict(dict(descs=d, pairs=pairs, kps=kps, models=models, px_th=1.0), **kw),
                msg)
    layout = [
        (dict(counts=[5, 6], pairs=[0, 1]), "pairs must be a non-empty [P,2] array of (query image, train image)"),
        (dict(counts=[5, 6], pairs=np.zeros((0, 2))),
         "pairs must be a non-empty [P,2] array of (query image, train image)"),
        (dict(counts=[5, 6], pairs=[[0, 2]]), "pairs: image index out of range"),
        (dict(counts=[5, 6], pairs=[[-1, 1]]), "pairs: image index out of range"),
    ]
    for kw, msg in layout:
        _raises(batch_layout, kw, msg)


# ------------------------------------------------------------------------------------------------ C
FAKE = ctypes.c_void_p(256)      # never dereferenced: every case is refused on the host


def _lib():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    return _cabi.lib()


def _c_cases(call, L, required, row, refine):
    """every refused case of a ragged pose or refine entry point, with its message: call(n_pairs, rows, dim, max_iters,
    px_th, null) calls it with the buffers named in `null` null and the others fake"""
    sizes = "need n_pairs >= 1, rows >= 0 and dim >= 2"
    cases = [(dict(null={k}), "null buffer") for k in required]
    cases += [(dict(null={k}), "null row buffer") for k in row]
    cases += [
        (dict(null={required[0]}, n_pairs=0, rows=-1), "null buffer"),
        (dict(null={row[0]}, n_pairs=0, dim=1), "null row buffer"),
        (dict(null=set(row), rows=-1), sizes),
        (dict(n_pairs=0), sizes), (dict(n_pairs=-1), sizes), (dict(rows=-1), sizes),
        (dict(dim=1), sizes), (dict(dim=0), sizes), (dict(dim=-2), sizes),
    ]
    if refine:
        cases += [
            (dict(max_iters=-1), "max_iters must not be negative"),
            (dict(max_iters=-1, dim=1), sizes),
            (dict(px_th=-1.0), "px_th must be a non-negative number"),
            (dict(px_th=float("nan")), "px_th must be a non-negative number"),
            (dict(px_th=float("nan"), max_iters=-1), "max_iters must not be negative"),
        ]
    for kw, msg in cases:
        kw = dict(dict(n_pairs=3, rows=10, dim=2, max_iters=10, px_th=1.0, null=()), **kw)
        assert call(**kw) == -1, kw
        assert L.dgb200_frontend_last_error().decode() == msg, kw


def _buffers(names, null):
    return {k: (None if k in null else FAKE) for k in names}


@pytest.mark.parametrize("model", ["F", "H"])
def test_pose_ragged_c_messages(model):
    L = _lib()
    names = ["M", "K1", "K2", "x1y1", "x2y2", "offsets", "mask", "R", "t", "plane", "good", "rotation_only", "points",
             "in_front", "angle", "median"]

    def call(n_pairs, rows, dim, max_iters, px_th, null):
        b = _buffers(names, null)
        if model == "F":
            return L.dgb200_pose_from_fundamental_ragged_dev(
                b["M"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"], n_pairs, rows, dim, b["mask"], b["R"],
                b["t"], b["good"], b["points"], b["in_front"], b["angle"], b["median"], None)
        return L.dgb200_pose_from_homography_ragged_dev(
            b["M"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"], n_pairs, rows, dim, b["mask"], b["R"],
            b["t"], b["plane"], b["good"], b["rotation_only"], b["points"], b["in_front"], b["angle"], b["median"], None)

    required = ["M", "K1", "K2", "offsets", "R", "t", "median"] + (["plane", "rotation_only"] if model == "H" else [])
    _c_cases(call, L, required, ["x1y1", "x2y2", "points", "in_front", "angle"], refine=False)


def test_refine_pose_ragged_c_messages():
    L = _lib()
    names = ["R", "t", "K1", "K2", "x1y1", "x2y2", "offsets", "mask", "R_out", "t_out", "F_out", "cost0", "cost",
             "n_used", "iters", "inliers"]

    def call(n_pairs, rows, dim, max_iters, px_th, null):
        b = _buffers(names, null)
        return L.dgb200_refine_pose_ragged_dev(b["R"], b["t"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"],
                                               n_pairs, rows, dim, b["mask"], max_iters, ctypes.c_double(px_th),
                                               b["R_out"], b["t_out"], b["F_out"], b["cost0"], b["cost"], b["n_used"],
                                               b["iters"], b["inliers"], None)

    _c_cases(call, L, ["R", "t", "K1", "K2", "offsets", "R_out", "t_out", "F_out", "cost"], ["x1y1", "x2y2"],
             refine=True)


@pytest.mark.parametrize("model", ["H", "F"])
def test_refine_model_ragged_c_messages(model):
    L = _lib()
    fn = L.dgb200_refine_homography_ragged_dev if model == "H" else L.dgb200_refine_fundamental_ragged_dev
    names = ["M", "x1y1", "x2y2", "offsets", "mask", "M_out", "cost0", "cost", "n_used", "iters", "inliers"]

    def call(n_pairs, rows, dim, max_iters, px_th, null):
        b = _buffers(names, null)
        return fn(b["M"], b["x1y1"], b["x2y2"], b["offsets"], n_pairs, rows, dim, b["mask"], max_iters,
                  ctypes.c_double(px_th), b["M_out"], b["cost0"], b["cost"], b["n_used"], b["iters"], b["inliers"], None)

    _c_cases(call, L, ["M", "offsets", "M_out", "cost"], ["x1y1", "x2y2"], refine=True)
