"""GPU front-end of the RANSAC path (SURVEY.md section 8(f).3): descriptor matching on the device.

Replaces the host-side matching of the reference's pipeline -- `cv2.BFMatcher().knnMatch(descs1, descs2, k=2)` followed
by the SNN ratio test `m.distance < 0.9 * n.distance` (examples/simple-example.py:46-53) -- with a CUDA kernel whose
output, two [N,2] float64 CUDA tensors, is what `findFundamentalMatrixBatch / findHomographyBatch` take: keypoints and
descriptors go in, models and masks come out, nothing visits the host in between.

    idx1, idx2, pts1, pts2 = match_descriptors(desc1, desc2, kp1, kp2, ratio=0.9)
    F, mask = pydegensac_b200.findFundamentalMatrixBatch(pts1[None], pts2[None], 0.5, 0.999, 50000)

Binary descriptors (ORB, AKAZE, BRISK, FREAK: uint8 [n, B]) by Hamming distance, as cv2.NORM_HAMMING:

    idx1, idx2, pts1, pts2 = match_descriptors(orb1, orb2, kp1, kp2, ratio=0.9, norm="hamming")

Many image pairs at once (one matcher call, one RANSAC launch, no host read in between):

    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    F, mask = pydegensac_b200.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, offsets=m.offsets,
                                                         n_max=m.n_max)

Guided re-match with the models found (candidates: the train keypoints within px_th of the epipolar line / transfer):

    g = match_descriptors_guided(descs, pairs, kps, F, 1.0, guide="F")

Relative pose, triangulated points and parallax angles of the ragged result, still without a host read:

    pose = pose_from_fundamental_ragged(F, K1, K2, m.pts1, m.pts2, m.offsets, mask)

The pose refined on its inliers (Levenberg-Marquardt on the Sampson error), with the calibrated F for a guided re-match:

    fine = refine_pose_ragged(pose.R, pose.t, K1, K2, m.pts1, m.pts2, m.offsets, pose.in_front)

The H branch (planar scenes, pure rotations): pose and scene plane from H, the best two of its decompositions:

    H, hmask = pydegensac_b200.findHomographyBatch(m.pts1, m.pts2, 2.0, 0.999, 10000, offsets=m.offsets, n_max=m.n_max)
    hpose = pose_from_homography_ragged(H, K1, K2, m.pts1, m.pts2, m.offsets, hmask)

H refined on its inliers first (Levenberg-Marquardt on the Sampson error of the H RANSAC's inlier rule):

    fine_h = refine_homography_ragged(H, m.pts1, m.pts2, m.offsets, hmask, px_th=2.0)

F refined on its inliers when the intrinsics are unknown (Levenberg-Marquardt on the Sampson error over the rank-2
matrices), then the guided re-match in the band of the refined F:

    fine_f = refine_fundamental_ragged(F, m.pts1, m.pts2, m.offsets, mask, px_th=1.0)
    g = match_descriptors_guided(descs, pairs, kps, fine_f.F, 1.0, guide="F")

Calibrated pairs verified by the five-point solver instead of the 7-point F (essential-matrix RANSAC,
cv2.findEssentialMat); its F goes on to the pose:

    ess = find_essential_ragged(m.pts1, m.pts2, K1, K2, m.offsets, px_th=1.0)
    pose = pose_from_fundamental_ragged(ess.F, K1, K2, m.pts1, m.pts2, m.offsets, ess.mask)

A further view registered against the triangulated points (P3P RANSAC on 2D-3D correspondences, cv2.solvePnPRansac):

    view = find_absolute_pose_ragged(pts2d, pts3d, K, offsets, mask=valid, px_th=2.0)

Tracks triangulated across the registered views (two-ray midpoint RANSAC with local optimisation on each track):

    tr = triangulate_tracks_ragged(cams, pts, R, t, K, offsets, mask=observed, px_th=2.0)

Cameras and points refined jointly (bundle adjustment, Levenberg-Marquardt with the Schur complement), view 0 held:

    ba = bundle_adjust_ragged(cams, pts, R, t, K, offsets, tr.X, mask=tr.mask, free=[1, 2], scale_gauge=1)

The tracks themselves, built from the verified matches of many pairs (union-find over the keypoints of all images):

    ts = build_tracks_ragged(counts, pairs, m.idx1, m.idx2, m.offsets, mask, kps=kps)
    tr = triangulate_tracks_ragged(ts.cams, ts.pts, R, t, K, ts.offsets, px_th=2.0)

A world rotation for every view from the relative rotations of the verified pairs (rotation averaging over the view
graph: a maximum-spanning-tree start ranked by the pairs' support, then robust IRLS); the translations are not estimated:

    ra = average_rotations(pairs, fine.R, n_views, weights=pose.good)

Before that, for images whose intrinsics are not known, each camera group's focal length from the pairs' fundamental
matrices (view-graph calibration: robust Levenberg-Marquardt on the Kruppa residuals); its inliers gate the rotations:

    cal = calibrate_view_graph(pairs, F, groups, intrinsics)
"""
import collections
import ctypes
import math

import numpy as np

from . import _cabi

kTQ = 32   # query descriptors per 2-NN work item (frontend.cu)

BatchLayout = collections.namedtuple("BatchLayout", "tile_prefix row_prefix col_prefix capacity n_max")
BatchMatches = collections.namedtuple("BatchMatches", "idx1 idx2 pts1 pts2 offsets n_max")
RaggedPose = collections.namedtuple("RaggedPose", "R t good points in_front angle median_angle")
RefinedPose = collections.namedtuple("RefinedPose", "R t F cost0 cost n_used iters inliers")
RefinedHomography = collections.namedtuple("RefinedHomography", "H cost0 cost n_used iters inliers")
RefinedFundamental = collections.namedtuple("RefinedFundamental", "F cost0 cost n_used iters inliers")
AbsolutePose = collections.namedtuple("AbsolutePose", "R t mask n_inliers iters cost0 cost")
EssentialMatrix = collections.namedtuple("EssentialMatrix", "E F mask n_inliers iters cost0 cost")
Tracks = collections.namedtuple("Tracks", "X mask n_inliers iters cost0 cost angle")
BundleAdjustment = collections.namedtuple("BundleAdjustment", "R t X mask cost0 cost iters n_used")
BundleAdjustmentPCG = collections.namedtuple("BundleAdjustmentPCG", "R t X mask cost0 cost iters n_used cg_iters")
BundleAdjustmentIntrinsics = collections.namedtuple("BundleAdjustmentIntrinsics",
                                                    "R t X intrinsics mask cost0 cost iters n_used cg_iters")
TrackSet = collections.namedtuple("TrackSet", "offsets cams kp pts track_of stats")
RotationAveraging = collections.namedtuple("RotationAveraging", "R component residual iters cg_iters")
ViewGraphCalibration = collections.namedtuple("ViewGraphCalibration",
                                              "intrinsics refined error inliers cost0 cost iters n_used cg_iters")
GlobalPositioning = collections.namedtuple("GlobalPositioning",
                                           "t X component angle inliers cost0 cost iters n_used cg_iters")
HomographyPose = collections.namedtuple("HomographyPose",
                                        "R t plane good rotation_only points in_front angle median_angle")


def batch_layout(counts, pairs):
    """Work layout of a matcher batch, from the descriptor counts of the images and the [P,2] pair table
    (query image, train image) -- what dgb200_match_descriptors_batch_dev derives on the host:
    tile_prefix [P+1]: first 2-NN work item of each pair (ceil(n1/32) items; none for a pair whose query image has no
    descriptors or whose train image has fewer than 2); row_prefix [P+1]: first output row a pair may use (prefix of the
    query counts); col_prefix [P+1]: the pair's col_best segment (prefix of the train counts); capacity = row_prefix[P];
    n_max = the largest query-image count over the pairs (an upper bound on any pair's match count)."""
    c = np.asarray(counts, dtype=np.int64)
    pr = _check_pair_table(pairs, len(c))
    n1, n2 = c[pr[:, 0]], c[pr[:, 1]]
    tiles = np.where((n1 >= 1) & (n2 >= 2), (n1 + kTQ - 1) // kTQ, 0)

    def prefix(x):
        out = np.zeros(len(x) + 1, dtype=np.int64)
        np.cumsum(x, out=out[1:])
        return out
    rows = prefix(n1)
    return BatchLayout(prefix(tiles), rows, prefix(n2), int(rows[-1]), int(n1.max()))


def _check_pair_table(pairs, n_images):
    """a host [P,2] table of (query image, train image) with P >= 1 and indices in [0, n_images); returns it as int64"""
    pr = np.asarray(pairs, dtype=np.int64)
    if pr.ndim != 2 or pr.shape[1] != 2 or pr.shape[0] < 1:
        raise ValueError("pairs must be a non-empty [P,2] array of (query image, train image)")
    if pr.min() < 0 or pr.max() >= n_images:
        raise ValueError("pairs: image index out of range")
    return pr


def _check_norm(norm):
    if norm not in ("l2", "hamming"):
        raise ValueError("norm must be 'l2' or 'hamming', not %r" % (norm,))
    return norm == "hamming"


def _binary_words(descs):
    """uint8 CUDA tensors [n_i, B] (one B in [1, 256]) -> one int32 tensor [sum n_i, W] of their rows, zero-padded to
    W = ceil(B / 16) * 4 32-bit words (padding changes no Hamming distance; 16-byte rows keep the bulk copies)."""
    import torch
    dev = descs[0].device
    if any(d.dtype != torch.uint8 for d in descs):
        raise ValueError("norm='hamming' takes uint8 descriptor tensors [n, B] (the layout cv2 returns)")
    if any(d.dim() != 2 for d in descs):
        raise ValueError("expected binary descriptor tensors [n, B]")
    B = int(descs[0].shape[1])
    if any(int(d.shape[1]) != B for d in descs):
        raise ValueError("binary descriptors of one call must all have the same length in bytes")
    if not 1 <= B <= 256:
        raise ValueError("binary descriptors must be 1 to 256 bytes long, not %d" % B)
    if dev.type != "cuda" or any(d.device != dev for d in descs):
        raise ValueError("expected CUDA descriptor tensors on one device")
    W = (B + 15) // 16 * 4
    rows = torch.zeros((sum(int(d.shape[0]) for d in descs), 4 * W), dtype=torch.uint8, device=dev)
    rows[:, :B] = torch.cat(descs, 0)
    return rows.view(torch.int32)


# ------------------------------------------------------------------------------------------------ argument checks
# Each helper raises the ValueError of one rule that the entry points share; a wrapper runs them in its own order.
def _check_tensors(named, mask):
    """named: (name, value) pairs of the required tensor arguments; mask: the optional one"""
    import torch
    for nm, x in named + ((("mask", mask),) if mask is not None else ()):
        if not isinstance(x, torch.Tensor):
            raise ValueError("%s must be a torch tensor" % nm)


def _check_model(name, M):
    """a [P,3,3] or [P,9] model tensor; returns P"""
    if M.dim() not in (2, 3) or M.shape[0] < 1 or tuple(M.shape[1:]) not in ((3, 3), (9,)):
        raise ValueError("%s must be [P,3,3] or [P,9] with P >= 1, not %s" % (name, list(M.shape)))
    return int(M.shape[0])


def _check_points(pts1, pts2):
    """the [rows, 2|6] correspondence rows; returns (rows, dim)"""
    if pts1.dim() != 2 or pts1.shape[1] < 2 or pts2.shape != pts1.shape:
        raise ValueError("pts1 and pts2 must be [rows, 2|6] tensors of one shape")
    return int(pts1.shape[0]), int(pts1.shape[1])


def _check_shape(name, x, letter, shape):
    """x of exactly `shape`, whose first dimension is called `letter` in the message"""
    if tuple(x.shape) != shape:
        raise ValueError("%s must be [%s] = [%s], not %s" % (name, ",".join((letter,) + tuple(map(str, shape[1:]))),
                                                          ",".join(map(str, shape)), list(x.shape)))


def _check_columns(name, x, letter, cols):
    """x of shape [rows, cols], the rows called `letter` in the message; returns rows"""
    if x.dim() != 2 or x.shape[1] != cols:
        raise ValueError("%s must be [%s,%d], not %s" % (name, letter, cols, list(x.shape)))
    return int(x.shape[0])


def _check_K(name, K, letter, n):
    """intrinsics [3,3] shared or [n,3,3], one per pair or camera (`letter`)"""
    if tuple(K.shape) not in ((3, 3), (n, 3, 3)):
        raise ValueError("%s must be [3,3] or [%s,3,3] with %s = %d, not %s" % (name, letter, letter, n, list(K.shape)))


def _check_int32(name, x):
    import torch
    if x.dtype != torch.int32:
        raise ValueError("%s must be int32, not %s" % (name, x.dtype))


def _check_offsets(offsets, letter, n=None):
    """int32 offsets [n+1] for a given n, or [N+1] with N >= 1 (N called `letter`); returns N"""
    if n is not None:
        if tuple(offsets.shape) != (n + 1,):
            raise ValueError("offsets must be [%s+1] = [%d], not %s" % (letter, n + 1, list(offsets.shape)))
    elif offsets.dim() != 1 or offsets.shape[0] < 2:
        raise ValueError("offsets must be [%s+1] with %s >= 1, not %s" % (letter, letter, list(offsets.shape)))
    _check_int32("offsets", offsets)
    return int(offsets.shape[0]) - 1


def _check_floating(named):
    for nm, x in named:
        if not x.is_floating_point():
            raise ValueError("%s must be a floating tensor, not %s" % (nm, x.dtype))


def _check_mask(mask, letter, rows):
    """an optional row mask [rows], bool or uint8"""
    import torch
    if mask is not None:
        _check_shape("mask", mask, letter, (rows,))
        if mask.dtype not in (torch.bool, torch.uint8):
            raise ValueError("mask must be bool or uint8, not %s" % mask.dtype)


def _check_count(name, value, least):
    """an iteration bound: an int >= least (0 or 1)"""
    value = int(value)
    if value < least:
        raise ValueError("%s must not be negative, not %d" % (name, value) if least == 0 else
                         "%s must be at least %d, not %d" % (name, least, value))
    return value


def _check_px_th(px_th, positive):
    """a pixel threshold: finite and > 0 (positive) or >= 0"""
    px_th = float(px_th)
    if not (0.0 < px_th < float("inf") if positive else px_th >= 0.0):
        raise ValueError("px_th must be a %s number, not %r" % ("positive" if positive else "non-negative", px_th))
    return px_th


def _check_conf(conf):
    conf = float(conf)
    if not 0.0 < conf <= 1.0:
        raise ValueError("conf must lie in (0, 1], not %r" % (conf,))
    return conf


def _check_device(named, mask):
    """the one CUDA device of the tensors of _check_tensors"""
    dev = named[0][1].device
    if dev.type != "cuda" or any(x.device != dev for _, x in named) or (mask is not None and mask.device != dev):
        raise ValueError("%s and mask must be CUDA tensors on one device" % ", ".join(nm for nm, _ in named))
    return dev


def _f64(*xs):
    import torch
    return tuple(x.to(torch.float64).contiguous() for x in xs)


def _mask_u8(mask):
    import torch
    return mask.contiguous().view(torch.uint8) if mask is not None else None


def _rows_out(n, dev):
    """a uint8 row output [n] (never a zero-sized allocation, which would pass a null pointer)"""
    import torch
    return torch.empty(max(n, 1), dtype=torch.uint8, device=dev)[:n]


def _call(fn, last_error, dev, *args):
    """fn(*args, stream) on device dev and its current stream, tensors passed by their data pointers and None as a
    null pointer; a nonzero return code raises ValueError with the message of last_error()"""
    import torch
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        rc = fn(*args, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    if rc != 0:
        raise ValueError(last_error().decode())


def match_descriptors(desc1, desc2, kp1=None, kp2=None, ratio=0.9, mutual=False, norm="l2"):
    """Two-nearest-neighbour matching + SNN ratio test (+ optional mutual nearest-neighbour check).

    norm="l2": squared L2.  desc1 [n1,D], desc2 [n2,D]: CUDA tensors (any float dtype; computed in float32), D a
    multiple of 4, <= 256; a query is accepted when d1 < ratio^2 * d2 (FP32, on the squared distances).
    norm="hamming": binary descriptors (ORB 32 bytes, AKAZE 61, BRISK/FREAK 64) as uint8 CUDA tensors [n1,B], [n2,B]
    with B in [1, 256]; the distance is the number of differing bits and a query is accepted when
    float64(d1) < ratio * float64(d2) -- what cv2.BFMatcher(cv2.NORM_HAMMING).knnMatch(k=2) and the ratio test
    `m.distance < ratio * n.distance` accept.
    kp1 [n1,>=2], kp2 [n2,>=2]: optional keypoint coordinate tensors (first two columns x, y; six columns carry the
    local affine shape through for the LAF check).
    Returns (idx1, idx2) int64 CUDA tensors of the accepted matches in ascending query order, plus (pts1, pts2) float64
    [N,2] (or [N,6]) CUDA tensors when keypoints were given."""
    import torch
    hamming = _check_norm(norm)
    if hamming:
        words = _binary_words([desc1, desc2])     # one allocation; desc2's rows start 16-byte aligned
        d1, d2 = words[:desc1.shape[0]], words[desc1.shape[0]:]
    else:
        d1 = desc1.to(torch.float32).contiguous()
        d2 = desc2.to(torch.float32).contiguous()
    if d1.dim() != 2 or d2.dim() != 2 or d1.shape[1] != d2.shape[1] or not d1.is_cuda or d1.device != d2.device:
        raise ValueError("expected two CUDA descriptor tensors [n1,D], [n2,D] on the same device")
    n1, D = d1.shape
    n2 = d2.shape[0]
    dev = d1.device
    L = _cabi.lib()
    mq = torch.empty(n1, dtype=torch.int32, device=dev)
    mt = torch.empty(n1, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.empty(int(L.dgb200_match_workspace_bytes(n1, n2)), dtype=torch.uint8, device=dev)
    k1 = k2 = x1 = x2 = None
    kp_dim = out_dim = 0
    if kp1 is not None:
        k1 = kp1.to(device=dev, dtype=torch.float64).contiguous()
        k2 = kp2.to(device=dev, dtype=torch.float64).contiguous()
        if k1.shape[0] != n1 or k2.shape[0] != n2 or k1.shape[1] != k2.shape[1] or k1.shape[1] < 2:
            raise ValueError("keypoint tensors must be [n1,k], [n2,k] with k >= 2")
        kp_dim = int(k1.shape[1])
        out_dim = 6 if kp_dim >= 6 else 2
        x1 = torch.empty((n1, out_dim), dtype=torch.float64, device=dev)
        x2 = torch.empty((n1, out_dim), dtype=torch.float64, device=dev)
    fn = L.dgb200_match_binary_descriptors_dev if hamming else L.dgb200_match_descriptors_dev
    _call(fn, L.dgb200_frontend_last_error, dev, d1, n1, d2, n2, D, ratio, int(bool(mutual)), k1, k2, kp_dim, mq, mt,
          x1, x2, out_dim, n1, cnt, ws)
    n = int(cnt.item())          # the one host read of the front-end: how many tentatives there are
    out = (mq[:n].long(), mt[:n].long())
    if x1 is not None:
        out = out + (x1[:n], x2[:n])
    return out


def pose_from_fundamental(F, K1, K2, pts1, pts2, mask=None):
    """Relative pose from fundamental matrices: E = K2^T F K1, SVD, cheirality vote over the inliers.

    F [P,3,3], pts [P,N,2] (float64 CUDA tensors), K1/K2 [3,3] or [P,3,3], mask [P,N] bool/uint8 or None.
    Returns R [P,3,3], t [P,3] (unit length; x2 ~ R x1 + t), good [P] int32 (correspondences in front of both cameras)."""
    import torch
    dev = F.device
    Fc = F.to(torch.float64).contiguous().view(-1, 9)
    P = Fc.shape[0]
    p1 = pts1.to(torch.float64).contiguous()
    p2 = pts2.to(torch.float64).contiguous()
    if p1.dim() == 2:
        p1, p2 = p1[None], p2[None]
    N, dim = int(p1.shape[1]), int(p1.shape[2])
    K1c = K1.to(device=dev, dtype=torch.float64).contiguous()
    K2c = K2.to(device=dev, dtype=torch.float64).contiguous()
    per_pair = 1 if K1c.dim() == 3 else 0
    m = None
    if mask is not None:
        m = mask.to(device=dev, dtype=torch.uint8).contiguous()
    L = _cabi.lib()
    R = torch.empty((P, 3, 3), dtype=torch.float64, device=dev)
    t = torch.empty((P, 3), dtype=torch.float64, device=dev)
    good = torch.empty(P, dtype=torch.int32, device=dev)
    _call(L.dgb200_pose_from_fundamental_batch_dev, L.dgb200_frontend_last_error, dev, Fc, K1c, K2c, per_pair, p1, p2,
          m, P, N, dim, R, t, good)
    return R, t, good


def _ragged_pose_inputs(model, name, K1, K2, pts1, pts2, offsets, mask):
    """Checks the inputs of a ragged pose call (a [P,3,3] or [P,9] model named `name`, K, rows, offsets, mask) and returns
    them ready for the C ABI: (P, rows, dim, device, per_pair, model, K1, K2, pts1, pts2, offsets, mask or None)."""
    named = ((name, model), ("K1", K1), ("K2", K2), ("pts1", pts1), ("pts2", pts2), ("offsets", offsets))
    _check_tensors(named, mask)
    P = _check_model(name, model)
    rows, dim = _check_points(pts1, pts2)
    _check_K("K1", K1, "P", P)
    _check_K("K2", K2, "P", P)
    _check_offsets(offsets, "P", P)
    _check_floating(named[:5])
    _check_mask(mask, "rows", rows)
    dev = _check_device(named, mask)
    per_pair = K1.dim() == 3 or K2.dim() == 3
    if per_pair:
        K1, K2 = K1.expand(P, 3, 3), K2.expand(P, 3, 3)
    return (P, rows, dim, dev, int(per_pair)) + _f64(model, K1, K2, pts1, pts2) + (offsets.contiguous(), _mask_u8(mask))


def pose_from_fundamental_ragged(F, K1, K2, pts1, pts2, offsets, mask=None):
    """pose_from_fundamental over a ragged batch, with the triangulated points and parallax angles of every row.

    The inputs are what the ragged pipeline produces (match_descriptors_batch, then findFundamentalMatrixBatch with
    offsets=), all CUDA tensors on one device: F [P,3,3] or [P,9] (x2^T F x1 = 0), K1 / K2 [3,3] or [P,3,3], pts1 /
    pts2 [rows, 2|6] (columns 0-1 are the pixel coordinates), offsets int32 [P+1] (pair p owns rows
    offsets[p] .. offsets[p+1]-1), mask [rows] bool / uint8 or None (every row).  Floating inputs are used in float64.
    Per pair, R, t and good are what pose_from_fundamental returns for the pair alone.  Per row, under the chosen pose:
    points [rows,3] the midpoint of the two rays' closest points, in camera 1's frame and units of the baseline
    (|t| = 1); in_front [rows] bool, mask and both depths positive (good is the pair's count of it); angle [rows] the
    parallax angle between the rays in radians.  median_angle [P] is the median angle of the pair's in-front rows (NaN
    when there is none): COLMAP-style tools keep pairs whose median parallax is large enough.  A pair whose F is all zero
    (no model found) or holds a NaN gets R = t = 0, good = 0, NaN points and angles, no in-front row and a NaN median.
    Returns RaggedPose(R, t, good, points, in_front, angle, median_angle); asynchronous, nothing is read back."""
    import torch
    P, rows, dim, dev, per_pair, Fc, K1c, K2c, p1, p2, off, m = _ragged_pose_inputs(F, "F", K1, K2, pts1, pts2,
                                                                                    offsets, mask)
    f64 = torch.float64
    L = _cabi.lib()
    R = torch.empty((P, 3, 3), dtype=f64, device=dev)
    t = torch.empty((P, 3), dtype=f64, device=dev)
    good = torch.empty(P, dtype=torch.int32, device=dev)
    points = torch.empty((rows, 3), dtype=f64, device=dev)
    in_front = torch.empty(rows, dtype=torch.uint8, device=dev)
    angle = torch.empty(rows, dtype=f64, device=dev)
    median = torch.empty(P, dtype=f64, device=dev)
    _call(L.dgb200_pose_from_fundamental_ragged_dev, L.dgb200_frontend_last_error, dev, Fc, K1c, K2c, per_pair, p1,
          p2, off, P, rows, dim, m, R, t, good, points, in_front, angle, median)
    return RaggedPose(R, t, good, points, in_front.view(torch.bool), angle, median)


def pose_from_homography_ragged(H, K1, K2, pts1, pts2, offsets, mask=None):
    """Relative pose and scene plane from homographies over a ragged batch: the H branch's counterpart of
    pose_from_fundamental_ragged, for planar scenes (F undetermined) and pure rotations (no F).

    The inputs are what the ragged pipeline produces (match_descriptors_batch, then findHomographyBatch with offsets=),
    all CUDA tensors on one device: H [P,3,3] or [P,9] (x2 ~ H x1, OpenCV convention), K1 / K2 [3,3] or [P,3,3], pts1 /
    pts2 [rows, 2|6], offsets int32 [P+1], mask [rows] bool / uint8 or None (every row); floating inputs are used in
    float64.  Per pair, Hn = K2^-1 H K1 is scaled to a middle singular value of 1 and det > 0.  When
    max |Hn^T Hn - I| < 1e-3 the pair is a pure rotation: one candidate, the rotation nearest to Hn, t = 0.  Otherwise
    Hn = R + t' n^T has the four solutions of cv2.decomposeHomographyMat, in its order (Malis & Vargas).  The rows with
    mask set vote (both depths positive; x1 . R^T x2 > 0 for a rotation): candidate 0 has the most votes, candidate 1
    the most among the rest, ties to the earlier solution.  Two views of a plane often leave both with equal votes, so
    candidate 1 is returned for callers with a prior (ground-plane normal, a third view).
    Returns HomographyPose(R, t, plane, good, rotation_only, points, in_front, angle, median_angle):
    R [P,2,3,3]; t [P,2,3] unit length, x2 ~ R x1 + t (candidate 0 goes straight into refine_pose_ragged);
    plane [P,2,4] (n, d), the plane n^T X = d in camera 1's frame and baseline units, d > 0; good [P,2] int32 the votes;
    rotation_only [P] bool.  Per row, under candidate 0 and as pose_from_fundamental_ragged defines them: points [rows,3],
    in_front [rows] bool, angle [rows]; median_angle [P].  A pure rotation has t = 0 and a NaN plane in candidate 0,
    R = t = 0, a NaN plane and good 0 in candidate 1, NaN points and in_front = mask and x1 . R^T x2 > 0; its
    median_angle is what COLMAP-style code compares with a threshold to call a pair panoramic.  A pair whose H is all zero
    (no model found) or holds a NaN gets zero R and t, NaN planes, good 0, NaN rows and a NaN median.  Asynchronous,
    nothing is read back."""
    import torch
    P, rows, dim, dev, per_pair, Hc, K1c, K2c, p1, p2, off, m = _ragged_pose_inputs(H, "H", K1, K2, pts1, pts2,
                                                                                    offsets, mask)
    f64 = torch.float64
    L = _cabi.lib()
    R = torch.empty((P, 2, 3, 3), dtype=f64, device=dev)
    t = torch.empty((P, 2, 3), dtype=f64, device=dev)
    plane = torch.empty((P, 2, 4), dtype=f64, device=dev)
    good = torch.empty((P, 2), dtype=torch.int32, device=dev)
    rotation_only = torch.empty(P, dtype=torch.uint8, device=dev)
    points = torch.empty((rows, 3), dtype=f64, device=dev)
    in_front = torch.empty(rows, dtype=torch.uint8, device=dev)
    angle = torch.empty(rows, dtype=f64, device=dev)
    median = torch.empty(P, dtype=f64, device=dev)
    _call(L.dgb200_pose_from_homography_ragged_dev, L.dgb200_frontend_last_error, dev, Hc, K1c, K2c, per_pair, p1,
          p2, off, P, rows, dim, m, R, t, plane, good, rotation_only, points, in_front, angle, median)
    return HomographyPose(R, t, plane, good, rotation_only.view(torch.bool), points, in_front.view(torch.bool), angle,
                          median)


def refine_pose_ragged(R, t, K1, K2, pts1, pts2, offsets, mask=None, max_iters=10, px_th=None):
    """Refine the relative pose of every pair of a ragged batch on its inliers: Levenberg-Marquardt on the Sampson error.

    pose_from_fundamental_ragged takes its pose from an uncalibrated F; this step minimises, per pair, the sum of the
    squared pixel-domain Sampson residuals of F = K2^-T [t]x R K1^-1 over the rows with mask set -- the residual of the
    RANSAC's inlier rule -- over the five degrees of freedom of (R, t), |t| = 1, starting from the pose given.
    All inputs are CUDA tensors on one device: R [P,3,3] or [P,9], t [P,3] (x2 ~ R x1 + t), K1 / K2 [3,3] or [P,3,3],
    pts1 / pts2 [rows, 2|6], offsets int32 [P+1], mask [rows] bool / uint8 or None (every row), as
    pose_from_fundamental_ragged takes and returns them; floating inputs are used in float64.  The intended call is
    refine_pose_ragged(pose.R, pose.t, K1, K2, m.pts1, m.pts2, m.offsets, pose.in_front): the RANSAC's inliers that
    triangulate in front of both cameras.  max_iters bounds the trial steps per pair (schedule: include/degensac_b200.h).
    Returns RefinedPose(R, t, F, cost0, cost, n_used, iters, inliers): R [P,3,3], t [P,3] refined; F [P,3,3] the
    calibrated fundamental matrix of (R, t), unit Frobenius norm (x2^T F x1 = 0), the model match_descriptors_guided(...,
    guide="F") takes; cost0 / cost [P] the sum of squared residuals (px^2) before and after, cost <= cost0; n_used [P]
    int32 the rows used; iters [P] int32 the trial steps taken; inliers [rows] bool, with px_th given: Sampson residual
    of the refined F at most px_th^2 for every row, masked or not (None without px_th).  A pair with fewer than 6 rows
    used keeps its pose (iters 0); a pair whose R is all zero or holds a NaN (no model) gets R = t = F = 0, NaN costs and
    no inliers.  The result of a pair does not depend on the batch it is in.  Asynchronous, nothing is read back."""
    import torch
    named = (("R", R), ("t", t), ("K1", K1), ("K2", K2), ("pts1", pts1), ("pts2", pts2), ("offsets", offsets))
    _check_tensors(named, mask)
    P = _check_model("R", R)
    _check_shape("t", t, "P", (P, 3))
    rows, dim = _check_points(pts1, pts2)
    _check_K("K1", K1, "P", P)
    _check_K("K2", K2, "P", P)
    _check_offsets(offsets, "P", P)
    _check_floating(named[:6])
    _check_mask(mask, "rows", rows)
    max_iters = _check_count("max_iters", max_iters, 0)
    if px_th is not None:
        px_th = _check_px_th(px_th, False)
    dev = _check_device(named, mask)
    per_pair = K1.dim() == 3 or K2.dim() == 3
    if per_pair:
        K1, K2 = K1.expand(P, 3, 3), K2.expand(P, 3, 3)
    Rc, tc, K1c, K2c, p1, p2 = _f64(R, t, K1, K2, pts1, pts2)
    off, m = offsets.contiguous(), _mask_u8(mask)
    f64 = torch.float64
    L = _cabi.lib()
    Ro = torch.empty((P, 3, 3), dtype=f64, device=dev)
    to = torch.empty((P, 3), dtype=f64, device=dev)
    Fo = torch.empty((P, 3, 3), dtype=f64, device=dev)
    cost0 = torch.empty(P, dtype=f64, device=dev)
    cost = torch.empty(P, dtype=f64, device=dev)
    n_used = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    inl = _rows_out(rows, dev) if px_th is not None else None
    _call(L.dgb200_refine_pose_ragged_dev, L.dgb200_frontend_last_error, dev, Rc, tc, K1c, K2c, int(per_pair), p1, p2,
          off, P, rows, dim, m, max_iters, px_th if px_th is not None else 0.0, Ro, to, Fo, cost0, cost, n_used, iters,
          inl)
    return RefinedPose(Ro, to, Fo, cost0, cost, n_used, iters, inl.view(torch.bool) if inl is not None else None)


def refine_homography_ragged(H, pts1, pts2, offsets, mask=None, max_iters=10, px_th=None):
    """Refine the homography of every pair of a ragged batch on its inliers: Levenberg-Marquardt on the Sampson error.

    findHomographyBatch returns the local optimisation's iterated algebraic (DLT) fit, which minimises no geometric
    error; this step minimises, per pair, the sum of the engine's Sampson errors over the rows with mask set -- the
    residual of the H RANSAC's default inlier rule (error_type="sampson", px^2) -- over the 8 degrees of freedom of H,
    starting from the H given, as cv2.findHomography polishes its result.  All inputs are CUDA tensors on one device:
    H [P,3,3] or [P,9] (x2 ~ H x1, what findHomographyBatch returns), pts1 / pts2 [rows, 2|6] (columns 0-1 are the
    pixel coordinates), offsets int32 [P+1], mask [rows] bool / uint8 or None (every row); floating inputs are used in
    float64.  The intended call is refine_homography_ragged(H, m.pts1, m.pts2, m.offsets, hmask, px_th=...), straight
    from the ragged findHomographyBatch.  max_iters bounds the trial steps per pair (schedule: include/degensac_b200.h).
    Returns RefinedHomography(H, cost0, cost, n_used, iters, inliers): H [P,3,3] refined, unit Frobenius norm, det > 0
    (what pose_from_homography_ragged and match_descriptors_guided(..., guide="H") take); cost0 / cost [P] the summed
    Sampson error (px^2) before and after, cost <= cost0; n_used [P] int32 the rows used; iters [P] int32 the trial steps
    taken; inliers [rows] bool, with px_th given: Sampson error of the refined H at most px_th^2 for every row, masked or
    not (None without px_th).  A pair with fewer than 5 rows used keeps its H (normalised; iters 0); a pair whose H is
    all zero, holds a NaN or is singular (no model) gets H = 0, NaN costs and no inliers.  The result of a pair does not
    depend on the batch it is in.  Asynchronous, nothing is read back."""
    Ho, cost0, cost, n_used, iters, inl = _refine_model_ragged("H", "dgb200_refine_homography_ragged_dev", H, pts1, pts2,
                                                               offsets, mask, max_iters, px_th)
    return RefinedHomography(Ho, cost0, cost, n_used, iters, inl)


def refine_fundamental_ragged(F, pts1, pts2, offsets, mask=None, max_iters=10, px_th=None):
    """Refine the fundamental matrix of every pair of a ragged batch on its inliers: Levenberg-Marquardt on the Sampson
    error over the rank-2 matrices, for pairs whose intrinsics are unknown.

    findFundamentalMatrixBatch returns the local optimisation's iterated, weighted algebraic fit with a rank-2
    projection, which minimises no geometric error; this step minimises, per pair, the sum of the Sampson errors over
    the rows with mask set -- the residual of the F RANSAC's default inlier rule (error_type="sampson", px^2) -- over the
    7 degrees of freedom of F, starting from the F given, as cv2.findFundamentalMat polishes its result.  All inputs are
    CUDA tensors on one device: F [P,3,3] or [P,9] (x2^T F x1 = 0, what findFundamentalMatrixBatch returns), pts1 / pts2
    [rows, 2|6] (columns 0-1 are the pixel coordinates), offsets int32 [P+1], mask [rows] bool / uint8 or None (every
    row); floating inputs are used in float64.  The intended call is refine_fundamental_ragged(F, m.pts1, m.pts2,
    m.offsets, mask, px_th=...), straight from the ragged findFundamentalMatrixBatch.  max_iters bounds the trial steps
    per pair (schedule: include/degensac_b200.h).  Returns RefinedFundamental(F, cost0, cost, n_used, iters, inliers):
    F [P,3,3] refined, rank 2, unit Frobenius norm, signed so that its inner product with the F given is not negative
    (what match_descriptors_guided(..., guide="F") and pose_from_fundamental_ragged take); cost0 / cost [P] the summed
    Sampson error (px^2) at the start point (the F given, projected to rank 2 if it is not) and after, cost <= cost0;
    n_used [P] int32 the rows used; iters [P] int32 the trial steps taken; inliers [rows] bool, with px_th given:
    Sampson error of the refined F at most px_th^2 for every row, masked or not (None without px_th).  A pair with fewer
    than 8 rows used keeps its F (normalised; iters 0); a pair whose F is all zero or not finite (no model) gets F = 0,
    NaN costs and no inliers.  The result of a pair does not depend on the batch it is in.  Asynchronous, nothing is
    read back."""
    Fo, cost0, cost, n_used, iters, inl = _refine_model_ragged("F", "dgb200_refine_fundamental_ragged_dev", F, pts1,
                                                               pts2, offsets, mask, max_iters, px_th)
    return RefinedFundamental(Fo, cost0, cost, n_used, iters, inl)


def _refine_model_ragged(name, entry, M, pts1, pts2, offsets, mask, max_iters, px_th):
    """The checks and the call of a refinement of one 3 x 3 model per pair (H or F, by `name`) through the C entry
    point `entry`: the refined models [P,3,3], cost0, cost, n_used, iters and the inlier rows (None without px_th)."""
    import torch
    named = ((name, M), ("pts1", pts1), ("pts2", pts2), ("offsets", offsets))
    _check_tensors(named, mask)
    P = _check_model(name, M)
    rows, dim = _check_points(pts1, pts2)
    _check_offsets(offsets, "P", P)
    _check_floating(named[:3])
    _check_mask(mask, "rows", rows)
    max_iters = _check_count("max_iters", max_iters, 0)
    if px_th is not None:
        px_th = _check_px_th(px_th, False)
    dev = _check_device(named, mask)
    Mc, p1, p2 = _f64(M, pts1, pts2)
    off, m = offsets.contiguous(), _mask_u8(mask)
    f64 = torch.float64
    L = _cabi.lib()
    Mo = torch.empty((P, 3, 3), dtype=f64, device=dev)
    cost0 = torch.empty(P, dtype=f64, device=dev)
    cost = torch.empty(P, dtype=f64, device=dev)
    n_used = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    inl = _rows_out(rows, dev) if px_th is not None else None
    _call(getattr(L, entry), L.dgb200_frontend_last_error, dev, Mc, p1, p2, off, P, rows, dim, m, max_iters,
          px_th if px_th is not None else 0.0, Mo, cost0, cost, n_used, iters, inl)
    return Mo, cost0, cost, n_used, iters, inl.view(torch.bool) if inl is not None else None


def find_absolute_pose_ragged(pts2d, pts3d, K, offsets, mask=None, px_th=2.0, conf=0.999, max_iters=10000, seeds=None,
                              refine_iters=10):
    """Register views against known 3D points: P3P MSAC-RANSAC with local optimisation over a ragged batch of 2D-3D
    correspondences, the batched, device-resident counterpart of cv2.solvePnPRansac.

    All inputs are CUDA tensors on one device: pts2d [rows,2] pixels in the view being registered, pts3d [rows,3]
    points in the world frame (e.g. the `points` of pose_from_fundamental_ragged, gathered onto the view's matches),
    K [3,3] or [P,3,3], offsets int32 [P+1] (pair p owns rows offsets[p] .. offsets[p+1]-1), mask [rows] bool / uint8 or
    None (every row): the rows that may be used (e.g. `in_front`).  Floating inputs are used in float64.  A row is
    usable when it is in the mask and its five coordinates are finite; a pair needs 4 usable rows.  px_th: the inlier
    threshold on the reprojection error in pixels (> 0); conf in (0, 1]; max_iters >= 1 bounds the RANSAC iterations;
    seeds: the seed of each pair's sample stream, as findFundamentalMatrixBatch takes it; refine_iters >= 0 bounds the
    trial steps of each Levenberg-Marquardt round of the local optimisation (0 skips it).  The estimator, its stopping
    rule and its local optimisation are specified in include/degensac_b200.h.
    Returns AbsolutePose(R, t, mask, n_inliers, iters, cost0, cost): R [P,3,3], t [P,3] with x ~ K (R X + t) (OpenCV's
    solvePnP convention); mask [rows] bool the inliers of the returned pose; n_inliers [P] int32; iters [P] int32 the
    RANSAC iterations drawn; cost0 [P] the MSAC cost sum min(e^2, px_th^2) of the best RANSAC pose and cost [P] that of
    the returned pose after local optimisation (cost <= cost0).  A pair without a model (fewer than 4 usable rows, no
    pose found, malformed offsets) gets R = t = 0, no inliers and NaN costs.  The result of a pair does not depend on
    the batch it is in.  Asynchronous, nothing is read back."""
    import torch
    from .tensor_api import _seeds_tensor
    named = (("pts2d", pts2d), ("pts3d", pts3d), ("K", K), ("offsets", offsets))
    _check_tensors(named, mask)
    P = _check_offsets(offsets, "P")
    rows = _check_columns("pts2d", pts2d, "rows", 2)
    _check_shape("pts3d", pts3d, "rows", (rows, 3))
    _check_K("K", K, "P", P)
    _check_floating(named[:3])
    _check_mask(mask, "rows", rows)
    px_th = _check_px_th(px_th, True)
    conf = _check_conf(conf)
    max_iters = _check_count("max_iters", max_iters, 1)
    refine_iters = _check_count("refine_iters", refine_iters, 0)
    dev = _check_device(named, mask)
    if isinstance(seeds, torch.Tensor) and seeds.is_cuda and seeds.device != dev:
        raise ValueError("seeds must be on the device of pts2d")
    x, X, Kc = _f64(pts2d, pts3d, K)
    off, m = offsets.contiguous(), _mask_u8(mask)
    ds = _seeds_tensor(seeds, P, dev)
    if tuple(ds.shape) != (P,):
        raise ValueError("seeds must hold one seed per pair (%d), not %s" % (P, list(ds.shape)))
    f64 = torch.float64
    L = _cabi.lib()
    R = torch.empty((P, 3, 3), dtype=f64, device=dev)
    t = torch.empty((P, 3), dtype=f64, device=dev)
    mo = _rows_out(rows, dev)
    n_inl = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    cost0 = torch.empty(P, dtype=f64, device=dev)
    cost = torch.empty(P, dtype=f64, device=dev)
    _call(L.dgb200_find_absolute_pose_ragged_dev, L.dgb200_absolute_pose_last_error, dev, x, X, Kc, int(Kc.dim() == 3),
          off, P, rows, m, px_th, conf, max_iters, refine_iters, ds, R, t, mo, n_inl, iters, cost0, cost)
    return AbsolutePose(R, t, mo.view(torch.bool), n_inl, iters, cost0, cost)


def find_essential_ragged(pts1, pts2, K1, K2, offsets, mask=None, px_th=1.0, conf=0.999, max_iters=10000, seeds=None,
                          refine_iters=10):
    """Verify calibrated image pairs: five-point MSAC-RANSAC with local optimisation over a ragged batch of
    correspondences, the batched, device-resident counterpart of cv2.findEssentialMat.

    All inputs are CUDA tensors on one device: pts1 / pts2 [rows, 2|6] (columns 0-1 are the pixel coordinates, as
    match_descriptors_batch returns them), K1 / K2 [3,3] or [P,3,3], offsets int32 [P+1] (pair p owns rows
    offsets[p] .. offsets[p+1]-1), mask [rows] bool / uint8 or None (every row): the rows that may be used.  Floating
    inputs are used in float64.  A row is usable when it is in the mask and its four coordinates are finite; a pair
    needs 5 usable rows.  px_th: the inlier threshold on the Sampson error in pixels (> 0), the F RANSAC's rule;
    conf in (0, 1]; max_iters >= 1 bounds the RANSAC iterations; seeds: the seed of each pair's sample stream, as
    findFundamentalMatrixBatch takes it; refine_iters >= 0 bounds the trial steps of each Levenberg-Marquardt round of
    the local optimisation over (R, t) (0 skips it).  The estimator, its stopping rule and its local optimisation are
    specified in include/degensac_b200.h.
    Returns EssentialMatrix(E, F, mask, n_inliers, iters, cost0, cost): E [P,3,3] at unit Frobenius norm
    (x2n^T E x1n = 0 for the normalised coordinates K^-1 [x, y, 1]); F [P,3,3] = K2^-T E K1^-1 at unit norm, what
    pose_from_fundamental_ragged, refine_pose_ragged and match_descriptors_guided(..., guide="F") take; mask [rows] bool
    the inliers of the returned model; n_inliers [P] int32; iters [P] int32 the RANSAC iterations drawn; cost0 [P] the
    MSAC cost sum min(e^2, px_th^2) of the best RANSAC model and cost [P] that of the returned model after local
    optimisation (cost <= cost0).  A pair without a model (fewer than 5 usable rows, no solution found, malformed
    offsets) gets E = F = 0, no inliers and NaN costs.  The result of a pair does not depend on the batch it is in.
    Asynchronous, nothing is read back."""
    import torch
    from .tensor_api import _seeds_tensor
    named = (("pts1", pts1), ("pts2", pts2), ("K1", K1), ("K2", K2), ("offsets", offsets))
    _check_tensors(named, mask)
    P = _check_offsets(offsets, "P")
    rows, dim = _check_points(pts1, pts2)
    _check_K("K1", K1, "P", P)
    _check_K("K2", K2, "P", P)
    _check_floating(named[:4])
    _check_mask(mask, "rows", rows)
    px_th = _check_px_th(px_th, True)
    conf = _check_conf(conf)
    max_iters = _check_count("max_iters", max_iters, 1)
    refine_iters = _check_count("refine_iters", refine_iters, 0)
    dev = _check_device(named, mask)
    if isinstance(seeds, torch.Tensor) and seeds.is_cuda and seeds.device != dev:
        raise ValueError("seeds must be on the device of pts1")
    per_pair = K1.dim() == 3 or K2.dim() == 3
    if per_pair:
        K1, K2 = K1.expand(P, 3, 3), K2.expand(P, 3, 3)
    x1, x2, K1c, K2c = _f64(pts1[:, :2], pts2[:, :2], K1, K2)
    off, m = offsets.contiguous(), _mask_u8(mask)
    ds = _seeds_tensor(seeds, P, dev)
    if tuple(ds.shape) != (P,):
        raise ValueError("seeds must hold one seed per pair (%d), not %s" % (P, list(ds.shape)))
    f64 = torch.float64
    L = _cabi.lib()
    E = torch.empty((P, 3, 3), dtype=f64, device=dev)
    F = torch.empty((P, 3, 3), dtype=f64, device=dev)
    mo = _rows_out(rows, dev)
    n_inl = torch.empty(P, dtype=torch.int32, device=dev)
    iters = torch.empty(P, dtype=torch.int32, device=dev)
    cost0 = torch.empty(P, dtype=f64, device=dev)
    cost = torch.empty(P, dtype=f64, device=dev)
    _call(L.dgb200_find_essential_ragged_dev, L.dgb200_essential_last_error, dev, x1, x2, K1c, K2c, int(per_pair), off,
          P, rows, m, px_th, conf, max_iters, refine_iters, ds, E, F, mo, n_inl, iters, cost0, cost)
    return EssentialMatrix(E, F, mo.view(torch.bool), n_inl, iters, cost0, cost)


def _check_tracks(cams, pts, R, t, K, offsets):
    """the track layout of triangulate_tracks_ragged and bundle_adjust_ragged; returns (T, obs, C)"""
    T = _check_offsets(offsets, "T")
    _check_int32("cams", cams)
    obs = _check_columns("pts", pts, "obs", 2)
    _check_shape("cams", cams, "obs", (obs,))
    if R.dim() != 3 or R.shape[0] < 1 or tuple(R.shape[1:]) != (3, 3):
        raise ValueError("R must be [C,3,3] with C >= 1, not %s" % list(R.shape))
    C = int(R.shape[0])
    _check_shape("t", t, "C", (C, 3))
    _check_K("K", K, "C", C)
    return T, obs, C


def triangulate_tracks_ragged(cams, pts, R, t, K, offsets, mask=None, px_th=2.0, min_angle=math.radians(1.5),
                              conf=0.999, max_iters=1000, seeds=None, refine_iters=10):
    """Triangulate tracks across registered views: two-ray midpoint MSAC-RANSAC with local optimisation over a ragged
    batch of tracks, each a list of observations (camera index, pixel) of one scene point.

    All inputs are CUDA tensors on one device: cams int32 [obs] the camera of each observation, pts [obs,2] its pixel,
    R [C,3,3] and t [C,3] the cameras' poses, world to camera with x ~ K (R X + t) (what find_absolute_pose_ragged
    returns; a camera whose R, t are not finite or whose det R <= 0.5, such as the R = t = 0 of a view that was not
    registered, is skipped), K [3,3] or [C,3,3], offsets int32 [T+1] (track j owns observations offsets[j] ..
    offsets[j+1]-1), mask [obs] bool / uint8 or None (every row): the observations that may be used.  A fixed-width
    layout (one slot per view, mask = observed) is a valid input.  Floating inputs are used in float64.  px_th: the
    inlier threshold on the reprojection error in pixels (> 0); min_angle in [0, pi): the smallest angle between the
    two rays of a hypothesis, in radians; conf in (0, 1]; max_iters >= 1 bounds the hypotheses per track (a track
    whose pairs are no more than max_iters tries every pair, in order); seeds: the seed of each track's sample stream,
    as findFundamentalMatrixBatch takes it; refine_iters >= 0 bounds the trial steps of each Levenberg-Marquardt round
    of the local optimisation (0 skips it).  The estimator is specified in include/degensac_b200.h.
    Returns Tracks(X, mask, n_inliers, iters, cost0, cost, angle): X [T,3] the points in the world frame; mask [obs]
    bool the inliers of the returned point; n_inliers [T] int32; iters [T] int32 the hypotheses drawn or enumerated;
    cost0 [T] the MSAC cost sum min(e^2, px_th^2) of the best RANSAC point and cost [T] that of the returned point
    (cost <= cost0); angle [T] the largest triangulation angle at X over pairs of inliers from distinct cameras, in
    radians (0 without such a pair; filter on it as COLMAP does).  A track without a model (fewer than 2 usable
    observations, no hypothesis, malformed offsets) gets X = NaN, no inliers and NaN costs and angle.  The result of a
    track does not depend on the batch it is in.  Asynchronous, nothing is read back."""
    import torch
    from .tensor_api import _seeds_tensor
    named = (("cams", cams), ("pts", pts), ("R", R), ("t", t), ("K", K), ("offsets", offsets))
    _check_tensors(named, mask)
    T, obs, C = _check_tracks(cams, pts, R, t, K, offsets)
    _check_floating(named[1:5])
    _check_mask(mask, "obs", obs)
    px_th, min_angle = _check_px_th(px_th, True), float(min_angle)
    if not 0.0 <= min_angle < math.pi:
        raise ValueError("min_angle must lie in [0, pi), not %r" % (min_angle,))
    conf = _check_conf(conf)
    max_iters = _check_count("max_iters", max_iters, 1)
    refine_iters = _check_count("refine_iters", refine_iters, 0)
    dev = _check_device(named, mask)
    if isinstance(seeds, torch.Tensor) and seeds.is_cuda and seeds.device != dev:
        raise ValueError("seeds must be on the device of pts")
    x, Rc, tc, Kc = _f64(pts, R, t, K)
    cm, off, m = cams.contiguous(), offsets.contiguous(), _mask_u8(mask)
    ds = _seeds_tensor(seeds, T, dev)
    if tuple(ds.shape) != (T,):
        raise ValueError("seeds must hold one seed per track (%d), not %s" % (T, list(ds.shape)))
    f64 = torch.float64
    L = _cabi.lib()
    X = torch.empty((T, 3), dtype=f64, device=dev)
    mo = _rows_out(obs, dev)
    n_inl = torch.empty(T, dtype=torch.int32, device=dev)
    iters = torch.empty(T, dtype=torch.int32, device=dev)
    cost0 = torch.empty(T, dtype=f64, device=dev)
    cost = torch.empty(T, dtype=f64, device=dev)
    angle = torch.empty(T, dtype=f64, device=dev)
    _call(L.dgb200_triangulate_tracks_ragged_dev, L.dgb200_triangulate_last_error, dev, cm, x, Rc, tc, Kc,
          int(Kc.dim() == 3), C, off, T, obs, m, px_th, min_angle, conf, max_iters, refine_iters, ds, X, mo, n_inl,
          iters, cost0, cost, angle)
    return Tracks(X, mo.view(torch.bool), n_inl, iters, cost0, cost, angle)


BA_MAX_FREE = 64   # free cameras per call at most (the reduced camera system is dense)


def _check_ba_controls(free, scale_gauge, loss_scale, C, max_free=None):
    """free, scale_gauge and loss_scale of the bundle adjustments over C cameras; max_free: the most free cameras
    (None: no limit).  Returns (the free list, the gauge camera or -1, sigma or 0)"""
    if free is None:
        if max_free is not None and C - 1 > max_free:
            raise ValueError("free=None frees %d cameras, more than %d: pass an explicit free list" % (C - 1, max_free))
        free = list(range(1, C))
    free = _host_pairs(free)
    try:
        fr = [int(c) for c in np.asarray(free).reshape(-1)]
    except (TypeError, ValueError):
        raise ValueError("free must be a host sequence of camera indices")
    if max_free is not None and len(fr) > max_free:
        raise ValueError("free holds %d cameras, more than %d" % (len(fr), max_free))
    if len(set(fr)) != len(fr):
        raise ValueError("free holds a camera twice")
    if any(not 0 <= c < C for c in fr):
        raise ValueError("free holds a camera index outside [0, %d)" % C)
    n_held = C - len(fr)
    if isinstance(scale_gauge, str):
        if scale_gauge != "auto":
            raise ValueError("scale_gauge must be 'auto', None or a camera of free, not %r" % (scale_gauge,))
        gauge = fr[0] if n_held == 1 and fr else -1
    elif scale_gauge is None:
        gauge = -1
    else:
        gauge = int(scale_gauge)
        if gauge not in fr:
            raise ValueError("scale_gauge %d is not one of the free cameras" % gauge)
        if n_held == 0:
            raise ValueError("scale_gauge needs a held camera: every camera is free")
    if loss_scale is None:
        sigma = 0.0
    else:
        sigma = float(loss_scale)
        if not 0.0 < sigma < float("inf"):
            raise ValueError("loss_scale must be a positive number or None, not %r" % (loss_scale,))
    return fr, gauge, sigma


def bundle_adjust_ragged(cams, pts, R, t, K, offsets, X, mask=None, free=None, scale_gauge="auto", loss_scale=None,
                         max_iters=50, px_th=2.0):
    """Bundle-adjust registered views and their tracks: Levenberg-Marquardt over the free cameras' poses and the
    tracks' points jointly, the points eliminated by the Schur complement and the reduced camera system solved densely.

    cams, pts, R, t, K, offsets and mask are CUDA tensors on one device, laid out as triangulate_tracks_ragged takes
    them (x ~ K (R X + t); a camera whose R, t are not finite or whose det R <= 0.5 is not registered, and its
    observations are not used).  X [T,3] the tracks' points and mask [obs] (bool / uint8 or None: every row) the
    observations that may be used: the X and mask of triangulate_tracks_ragged feed straight in.  Floating inputs are
    used in float64; the intrinsics are held.
    free: a HOST sequence of at most 64 distinct camera indices whose poses move (control data, as match_descriptors_
    batch's pairs); every other camera is held.  None: every camera but camera 0, a ValueError when that is more than
    64.  scale_gauge: a camera of `free` one of whose translation coordinates is held, which fixes the scale that one
    held camera leaves free (the axis of its largest translation relative to the lowest-index held camera, chosen on
    the device); "auto": free[0] when exactly one camera is held, else None; None: no scale hold.  loss_scale: None for
    the squared pixel error, sigma > 0 for the Cauchy loss sigma^2 log(1 + e^2 / sigma^2).  max_iters >= 0 bounds the
    trial steps.  px_th > 0: the inlier threshold of the output mask, in pixels.  The estimator is specified in
    include/degensac_b200.h.
    Returns BundleAdjustment(R, t, X, mask, cost0, cost, iters, n_used): R [C,3,3], t [C,3] and X [T,3] (held cameras
    and tracks that were not optimised -- fewer than 2 distinct cameras, or a point behind all but one -- bit-identical
    to the input); mask [obs] bool: the usable observations with positive depth and a reprojection error <= px_th at
    the output; cost0, cost: [1] float64 the cost at the start and at the output (cost <= cost0); iters: [1] int32 the
    trial steps; n_used: [1] int32 the observations in the cost.  Asynchronous, nothing is read back."""
    import torch
    named = (("cams", cams), ("pts", pts), ("R", R), ("t", t), ("K", K), ("offsets", offsets), ("X", X))
    _check_tensors(named, mask)
    T, obs, C = _check_tracks(cams, pts, R, t, K, offsets)
    _check_shape("X", X, "T", (T, 3))
    _check_floating(named[1:5] + named[6:])
    _check_mask(mask, "obs", obs)
    fr, gauge, sigma = _check_ba_controls(free, scale_gauge, loss_scale, C, BA_MAX_FREE)
    max_iters = _check_count("max_iters", max_iters, 0)
    px_th = _check_px_th(px_th, True)
    dev = _check_device(named, mask)
    x, Rc, tc, Kc, Xc = _f64(pts, R, t, K, X)
    cm, off, m = cams.contiguous(), offsets.contiguous(), _mask_u8(mask)
    hf = np.ascontiguousarray(fr, dtype=np.int32)
    f64 = torch.float64
    L = _cabi.lib()
    Ro = torch.empty((C, 3, 3), dtype=f64, device=dev)
    to = torch.empty((C, 3), dtype=f64, device=dev)
    Xo = torch.empty((T, 3), dtype=f64, device=dev)
    mo = _rows_out(obs, dev)
    cost0 = torch.empty(1, dtype=f64, device=dev)
    cost = torch.empty(1, dtype=f64, device=dev)
    iters = torch.empty(1, dtype=torch.int32, device=dev)
    n_used = torch.empty(1, dtype=torch.int32, device=dev)
    _call(L.dgb200_bundle_adjust_ragged_dev, L.dgb200_bundle_adjust_last_error, dev, cm, x, Rc, tc, Kc,
          int(Kc.dim() == 3), C, off, T, obs, Xc, m, hf.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(fr), gauge,
          sigma, max_iters, px_th, Ro, to, Xo, mo, cost0, cost, iters, n_used)
    return BundleAdjustment(Ro, to, Xo, mo.view(torch.bool), cost0, cost, iters, n_used)


def bundle_adjust_pcg_ragged(cams, pts, R, t, K, offsets, X, mask=None, free=None, scale_gauge="auto", loss_scale=None,
                             max_iters=50, px_th=2.0, cg_max_iters=100, cg_tol=0.1):
    """Bundle-adjust any number of cameras: the Levenberg-Marquardt of bundle_adjust_ragged, with the reduced camera
    system solved inexactly by conjugate gradients on the implicit Schur complement and a block-Jacobi preconditioner
    (Ceres' ITERATIVE_SCHUR with SCHUR_JACOBI), so that it has no camera limit.  It is a different estimator from
    bundle_adjust_ragged: each trial step is the exact LM step only up to the CG tolerance.

    The arguments are bundle_adjust_ragged's, except: free is a HOST sequence of any number of distinct camera
    indices (None: every camera but camera 0, whatever their number); cg_max_iters >= 1 bounds the CG iterations of
    each trial step, and cg_tol >= 0 stops them once |r| <= cg_tol |b| (0.1, the default, is Ceres' inexact-Newton
    forcing value).  The estimator is specified in include/degensac_b200.h.
    Returns BundleAdjustmentPCG(R, t, X, mask, cost0, cost, iters, n_used, cg_iters): bundle_adjust_ragged's fields and
    cg_iters [1] int32, the CG iterations summed over the trial steps.  Asynchronous, nothing is read back."""
    import torch
    named = (("cams", cams), ("pts", pts), ("R", R), ("t", t), ("K", K), ("offsets", offsets), ("X", X))
    _check_tensors(named, mask)
    T, obs, C = _check_tracks(cams, pts, R, t, K, offsets)
    _check_shape("X", X, "T", (T, 3))
    _check_floating(named[1:5] + named[6:])
    _check_mask(mask, "obs", obs)
    fr, gauge, sigma = _check_ba_controls(free, scale_gauge, loss_scale, C)
    max_iters = _check_count("max_iters", max_iters, 0)
    px_th = _check_px_th(px_th, True)
    cg_max_iters = _check_count("cg_max_iters", cg_max_iters, 1)
    cg_tol = float(cg_tol)
    if not 0.0 <= cg_tol < float("inf"):
        raise ValueError("cg_tol must be a non-negative finite number, not %r" % (cg_tol,))
    dev = _check_device(named, mask)
    x, Rc, tc, Kc, Xc = _f64(pts, R, t, K, X)
    cm, off, m = cams.contiguous(), offsets.contiguous(), _mask_u8(mask)
    hf = np.ascontiguousarray(fr, dtype=np.int32)
    f64 = torch.float64
    L = _cabi.lib()
    Ro = torch.empty((C, 3, 3), dtype=f64, device=dev)
    to = torch.empty((C, 3), dtype=f64, device=dev)
    Xo = torch.empty((T, 3), dtype=f64, device=dev)
    mo = _rows_out(obs, dev)
    cost0 = torch.empty(1, dtype=f64, device=dev)
    cost = torch.empty(1, dtype=f64, device=dev)
    iters = torch.empty(1, dtype=torch.int32, device=dev)
    n_used = torch.empty(1, dtype=torch.int32, device=dev)
    cg_iters = torch.empty(1, dtype=torch.int32, device=dev)
    _call(L.dgb200_bundle_adjust_pcg_ragged_dev, L.dgb200_bundle_adjust_pcg_last_error, dev, cm, x, Rc, tc, Kc,
          int(Kc.dim() == 3), C, off, T, obs, Xc, m, hf.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(fr), gauge,
          sigma, max_iters, px_th, cg_max_iters, cg_tol, Ro, to, Xo, mo, cost0, cost, iters, n_used, cg_iters)
    return BundleAdjustmentPCG(Ro, to, Xo, mo.view(torch.bool), cost0, cost, iters, n_used, cg_iters)


def _check_groups(groups, intrinsics, C):
    """groups int32 [C] and intrinsics [G,5] of the RADIAL model; returns G"""
    _check_int32("groups", groups)
    _check_shape("groups", groups, "C", (C,))
    if intrinsics.dim() != 2 or intrinsics.shape[0] < 1 or intrinsics.shape[1] != 5:
        raise ValueError("intrinsics must be [G,5] with G >= 1, not %s" % list(intrinsics.shape))
    return int(intrinsics.shape[0])


def bundle_adjust_intrinsics_ragged(cams, pts, R, t, groups, intrinsics, offsets, X, mask=None, free=None,
                                    free_groups=None, refine_focal=True, refine_principal_point=False,
                                    refine_distortion=True, scale_gauge="auto", loss_scale=None, max_iters=50,
                                    px_th=2.0, cg_max_iters=100, cg_tol=0.1):
    """Bundle adjustment that also refines the intrinsics: the estimator of bundle_adjust_pcg_ragged over the free
    cameras' poses, the free intrinsics groups and the tracks' points, with COLMAP's RADIAL camera model.

    The camera model: p = R X + t, u = p[:2] / p[2], s = u . u, pixel = f (1 + k1 s + k2 s^2) u + (cx, cy), with the
    intrinsics (f, cx, cy, k1, k2) of the camera's group.  One focal length and no skew, by design; with k1 = k2 = 0 it
    is the pinhole K = [[f, 0, cx], [0, f, cy], [0, 0, 1]] of the other entry points.
    groups: int32 [C] CUDA tensor, the row of intrinsics [G,5] (a floating CUDA tensor) that each camera uses: one group
    for every view of one camera, arange(C) for a camera per view.  A camera whose group index lies outside [0, G), or
    whose group's parameters are not finite or have f <= 0, is treated as an unregistered camera.
    free_groups: a HOST sequence of distinct group indices whose intrinsics move (None: every group).  refine_focal,
    refine_principal_point, refine_distortion: which of f, (cx, cy) and (k1, k2) move in a free group (COLMAP's
    defaults).  A free group without a used observation is passed through.  Observations of held cameras constrain
    their group's intrinsics.  The other arguments are bundle_adjust_pcg_ragged's.  The estimator is specified in
    include/degensac_b200.h.
    Returns BundleAdjustmentIntrinsics(R, t, X, intrinsics, mask, cost0, cost, iters, n_used, cg_iters):
    bundle_adjust_pcg_ragged's fields and intrinsics [G,5] float64 (held groups bit-identical to the input); the mask is
    taken at the refined intrinsics.  Asynchronous, nothing is read back."""
    import torch
    named = (("cams", cams), ("pts", pts), ("R", R), ("t", t), ("groups", groups), ("intrinsics", intrinsics),
             ("offsets", offsets), ("X", X))
    _check_tensors(named, mask)
    T = _check_offsets(offsets, "T")
    _check_int32("cams", cams)
    obs = _check_columns("pts", pts, "obs", 2)
    _check_shape("cams", cams, "obs", (obs,))
    if R.dim() != 3 or R.shape[0] < 1 or tuple(R.shape[1:]) != (3, 3):
        raise ValueError("R must be [C,3,3] with C >= 1, not %s" % list(R.shape))
    C = int(R.shape[0])
    _check_shape("t", t, "C", (C, 3))
    G = _check_groups(groups, intrinsics, C)
    _check_shape("X", X, "T", (T, 3))
    _check_floating((("pts", pts), ("R", R), ("t", t), ("intrinsics", intrinsics), ("X", X)))
    _check_mask(mask, "obs", obs)
    fr, gauge, sigma = _check_ba_controls(free, scale_gauge, loss_scale, C)
    if free_groups is None:
        fg = list(range(G))
    else:
        try:
            fg = [int(g) for g in np.asarray(_host_pairs(free_groups)).reshape(-1)]
        except (TypeError, ValueError):
            raise ValueError("free_groups must be a host sequence of group indices")
        if len(set(fg)) != len(fg):
            raise ValueError("free_groups holds a group twice")
        if any(not 0 <= g < G for g in fg):
            raise ValueError("free_groups holds a group index outside [0, %d)" % G)
    refine = (1 if refine_focal else 0) | (2 if refine_principal_point else 0) | (4 if refine_distortion else 0)
    max_iters = _check_count("max_iters", max_iters, 0)
    px_th = _check_px_th(px_th, True)
    cg_max_iters = _check_count("cg_max_iters", cg_max_iters, 1)
    cg_tol = float(cg_tol)
    if not 0.0 <= cg_tol < float("inf"):
        raise ValueError("cg_tol must be a non-negative finite number, not %r" % (cg_tol,))
    dev = _check_device(named, mask)
    x, Rc, tc, kc, Xc = _f64(pts, R, t, intrinsics, X)
    cm, gr, off, m = cams.contiguous(), groups.contiguous(), offsets.contiguous(), _mask_u8(mask)
    hf = np.ascontiguousarray(fr, dtype=np.int32)
    hg = np.ascontiguousarray(fg, dtype=np.int32)
    f64 = torch.float64
    L = _cabi.lib()
    Ro = torch.empty((C, 3, 3), dtype=f64, device=dev)
    to = torch.empty((C, 3), dtype=f64, device=dev)
    Xo = torch.empty((T, 3), dtype=f64, device=dev)
    ko = torch.empty((G, 5), dtype=f64, device=dev)
    mo = _rows_out(obs, dev)
    cost0 = torch.empty(1, dtype=f64, device=dev)
    cost = torch.empty(1, dtype=f64, device=dev)
    iters = torch.empty(1, dtype=torch.int32, device=dev)
    n_used = torch.empty(1, dtype=torch.int32, device=dev)
    cg_iters = torch.empty(1, dtype=torch.int32, device=dev)
    i32p = ctypes.POINTER(ctypes.c_int32)
    _call(L.dgb200_bundle_adjust_intrinsics_ragged_dev, L.dgb200_bundle_adjust_intrinsics_last_error, dev, cm, x, Rc,
          tc, gr, kc, G, C, off, T, obs, Xc, m, hf.ctypes.data_as(i32p), len(fr), hg.ctypes.data_as(i32p), len(fg),
          refine, gauge, sigma, max_iters, px_th, cg_max_iters, cg_tol, Ro, to, Xo, ko, mo, cost0, cost, iters, n_used,
          cg_iters)
    return BundleAdjustmentIntrinsics(Ro, to, Xo, ko, mo.view(torch.bool), cost0, cost, iters, n_used, cg_iters)


def undistort_points(pts, cams, groups, intrinsics):
    """The pinhole pixels of raw pixels through the RADIAL model of bundle_adjust_intrinsics_ragged.

    pts [obs,2] floating, cams int32 [obs] the camera of each row, groups int32 [C] and intrinsics [G,5] (f, cx, cy, k1,
    k2): CUDA tensors on one device.  Returns float64 [obs,2], f u + (cx, cy) for the undistorted normalised point u of
    each row, which triangulate_tracks_ragged and find_absolute_pose_ragged take with K = [[f, 0, cx], [0, f, cy],
    [0, 0, 1]] of the row's group.  A row whose camera or group index is out of range, whose group's intrinsics are not
    finite or have f <= 0, whose radius lies beyond the first turning point of the distortion, or whose Newton
    iteration does not converge, gives NaN.  Asynchronous, nothing is read back."""
    import torch
    named = (("pts", pts), ("cams", cams), ("groups", groups), ("intrinsics", intrinsics))
    _check_tensors(named, None)
    obs = _check_columns("pts", pts, "obs", 2)
    _check_int32("cams", cams)
    _check_shape("cams", cams, "obs", (obs,))
    _check_int32("groups", groups)
    if groups.dim() != 1 or groups.shape[0] < 1:
        raise ValueError("groups must be [C] with C >= 1, not %s" % list(groups.shape))
    C = int(groups.shape[0])
    G = _check_groups(groups, intrinsics, C)
    _check_floating((("pts", pts), ("intrinsics", intrinsics)))
    dev = _check_device(named, None)
    x, kc = _f64(pts, intrinsics)
    out = torch.empty((obs, 2), dtype=torch.float64, device=dev)
    L = _cabi.lib()
    _call(L.dgb200_undistort_points_dev, L.dgb200_undistort_last_error, dev, x, cams.contiguous(), obs,
          groups.contiguous(), C, kc, G, out)
    return out


def build_tracks_ragged(counts, pairs, idx1, idx2, offsets, mask=None, kps=None, min_length=2):
    """Build tracks from the verified matches of many image pairs: the connected components of the graph whose nodes
    are the keypoints of all images and whose edges are the matches, in the ragged layout that
    triangulate_tracks_ragged and bundle_adjust_ragged take (OpenMVG's TracksBuilder, on the device).

    counts: a HOST sequence of the I images' keypoint counts (the node of keypoint k of image i is sum(counts[:i]) + k;
    at most 2^31 - 1 nodes).  pairs: a HOST [P,2] table of (query image, train image), as match_descriptors_batch
    takes it.  idx1, idx2 (int32 or int64 [rows]), offsets (int32 [P+1]) and mask ([rows] bool / uint8 or None: every
    row) are CUDA tensors on one device: the BatchMatches fields and the ragged RANSAC mask, used as they are (int64
    indices are narrowed on the device, out-of-range values staying out of range).  Row r of pair p = (q, t), with
    offsets[p] <= r < offsets[p+1], joins keypoint idx1[r] of q and idx2[r] of t when the mask is set and both indices
    lie inside their images; a pair whose offsets are not 0 <= offsets[p] <= offsets[p+1] <= rows adds nothing.
    kps: optional list of I CUDA keypoint tensors [n_i, k >= 2]; their x, y (columns 0-1) become the observations'
    pixels.  A component with two keypoints of one image is conflicting and dropped whole; a track needs at least
    min_length (>= 2) keypoints.  Tracks are ordered by their smallest node, a track's observations by node (so by
    image).  The estimator is specified in include/degensac_b200.h.
    Returns TrackSet(offsets, cams, kp, pts, track_of, stats), capacity-sized because the number of tracks T is only
    known on the device (N = sum(counts), T_cap = N // min_length): offsets int32 [T_cap+1] (entries past T repeat the
    observation count: empty tracks, which triangulation and bundle adjustment leave alone); cams int32 [N] the image
    of each observation; kp int32 [N] its keypoint index in that image; pts float64 [N,2] its pixel (None without kps);
    track_of int32 [N] the track of each keypoint or -1; stats int32 [4] (tracks, observations, conflicting
    components, keypoints in them).  Rows past the observations are cams = kp = -1, pts = NaN.  The output depends on
    the set of matches alone, not on their order.  Asynchronous, nothing is read back; trim_tracks cuts it to size."""
    import torch
    if isinstance(counts, torch.Tensor) and counts.is_cuda:
        raise ValueError("counts must be a host sequence: reading a CUDA tensor would synchronise")
    pairs = _host_pairs(pairs)
    cn = np.asarray(counts)
    if cn.ndim != 1 or len(cn) < 1 or not np.issubdtype(cn.dtype, np.integer):
        raise ValueError("counts must be a non-empty host sequence of integer keypoint counts")
    cn = cn.astype(np.int64)
    if cn.min() < 0:
        raise ValueError("counts must not be negative")
    if int(cn.sum()) > 2 ** 31 - 1:
        raise ValueError("counts sum to %d keypoints, more than 2^31 - 1" % int(cn.sum()))
    I = len(cn)
    pr = np.ascontiguousarray(_check_pair_table(pairs, I), dtype=np.int32)
    P = len(pr)
    named = (("idx1", idx1), ("idx2", idx2), ("offsets", offsets))
    _check_tensors(named, mask)
    if idx1.dim() != 1:
        raise ValueError("idx1 must be [rows], not %s" % list(idx1.shape))
    rows = int(idx1.shape[0])
    _check_shape("idx2", idx2, "rows", (rows,))
    for nm, x in named[:2]:
        if x.dtype not in (torch.int32, torch.int64):
            raise ValueError("%s must be int32 or int64, not %s" % (nm, x.dtype))
    _check_offsets(offsets, "P", P)
    _check_mask(mask, "rows", rows)
    min_length = _check_count("min_length", min_length, 2)
    dev = _check_device(named, mask)
    N = int(cn.sum())
    kbank = None
    if kps is not None:
        if len(kps) != I or any(not isinstance(k, torch.Tensor) for k in kps):
            raise ValueError("kps must hold one keypoint tensor per image (%d)" % I)
        if any(k.dim() != 2 or k.shape[0] != c or k.shape[1] < 2 for k, c in zip(kps, cn)):
            raise ValueError("keypoint tensors must be [n_i, k] with k >= 2 and n_i = counts[i]")
        if any(k.device != dev for k in kps):
            raise ValueError("kps must be on the device of idx1")
        _check_floating([("kps", k) for k in kps])
        kbank = torch.cat([k[:, :2].to(torch.float64) for k in kps], 0).contiguous() if N else None
    i1, i2 = ((x if x.dtype == torch.int32 else x.clamp(-1, 2 ** 31 - 1).to(torch.int32)).contiguous()
              for x in (idx1, idx2))
    img_off = np.zeros(I + 1, dtype=np.int32)
    img_off[1:] = np.cumsum(cn)
    i32 = ctypes.POINTER(ctypes.c_int32)
    L = _cabi.lib()
    T_cap = N // min_length
    off_out = torch.empty(T_cap + 1, dtype=torch.int32, device=dev)
    cams = torch.empty(N, dtype=torch.int32, device=dev)
    kp = torch.empty(N, dtype=torch.int32, device=dev)
    pts = torch.empty((N, 2), dtype=torch.float64, device=dev) if kbank is not None else None
    track_of = torch.empty(N, dtype=torch.int32, device=dev)
    stats = torch.empty(4, dtype=torch.int32, device=dev)
    _call(L.dgb200_build_tracks_ragged_dev, L.dgb200_tracks_last_error, dev, img_off.ctypes.data_as(i32), I,
          pr.ctypes.data_as(i32), P, i1, i2, offsets.contiguous(), rows, _mask_u8(mask), kbank, min_length, off_out,
          cams, kp, pts, track_of, stats)
    if kps is not None and pts is None:
        pts = torch.empty((0, 2), dtype=torch.float64, device=dev)
    return TrackSet(off_out, cams, kp, pts, track_of, stats)


def trim_tracks(ts):
    """A TrackSet of build_tracks_ragged cut to its T tracks and their observations: one host read (of stats); the
    tensors returned are views of the ones given."""
    T, n = (int(v) for v in ts.stats[:2].tolist())
    return TrackSet(ts.offsets[:T + 1], ts.cams[:n], ts.kp[:n], ts.pts[:n] if ts.pts is not None else None,
                    ts.track_of, ts.stats)


def calibrate_view_graph(pairs, F, groups, intrinsics, mask=None, loss_scale=1e-2, max_error=1e-2, max_ratio=10.0,
                         max_iters=100, cg_max_iters=500, cg_tol=1e-6):
    """Calibrate the view graph: each camera group's focal length from the fundamental matrices of the verified pairs,
    and the pairs whose F agrees with the result (GLOMAP's view-graph calibration, on the device), for images whose
    intrinsics are not known.

    pairs: a HOST [P,2] table of (i, j) over the C views, as average_rotations takes it.  F: a CUDA float tensor [P,3,3]
    or [P,9] (used in float64) with x_j^T F x_i = 0, what findFundamentalMatrixBatch returns with pts1 from view i and
    pts2 from view j.  groups: int32 [C] CUDA tensor, each view's row of intrinsics; intrinsics: a floating [G,5] CUDA
    tensor of each group's start (f0, cx, cy, k1, k2), the RADIAL row of bundle_adjust_intrinsics_ragged (1.2 max(w, h)
    is a usual f0 without EXIF).  mask: [P] bool / uint8 or None (every pair).
    Each group's f = f0 exp(theta) moves, its principal point is held, k1 and k2 are passed through (F is taken as the
    pinhole F of the pixels given).  An edge is used when i != j, its mask is set, F is finite, both groups' intrinsics
    are finite with f0 > 0 and s2 > 1e-6 s1 for the singular values of K0_j^T F K0_i.  Each used edge has two residuals
    of the simplified Kruppa equations in [-1, 1]; Levenberg-Marquardt from theta = 0 minimises the sum of their Cauchy
    loss of scale loss_scale (0: the squared loss) for at most max_iters trial steps, each solved by Jacobi-
    preconditioned CG over the groups (cg_max_iters, cg_tol).  A group without a used edge keeps theta = 0.  The
    estimator is specified in include/degensac_b200.h.
    Returns ViewGraphCalibration(intrinsics, refined, error, inliers, cost0, cost, iters, n_used, cg_iters):
    intrinsics [G,5] float64, with f refined where 1 / max_ratio <= f / f0 <= max_ratio on a group with a used edge and
    every other row bit-identical to the input; refined [G] bool; error [P] float64 the edge's residual norm at those
    intrinsics (NaN for an edge that is not used); inliers [P] bool, the used edges with error <= max_error, the mask
    that average_rotations takes next; cost0, cost [1] float64; iters, n_used, cg_iters [1] int32.  Asynchronous,
    nothing is read back."""
    import torch
    named = (("F", F), ("groups", groups), ("intrinsics", intrinsics))
    _check_tensors(named, mask)
    _check_int32("groups", groups)
    if groups.dim() != 1 or groups.shape[0] < 1:
        raise ValueError("groups must be [C] with C >= 1, not %s" % list(groups.shape))
    C = int(groups.shape[0])
    G = _check_groups(groups, intrinsics, C)
    pairs = _host_pairs(pairs)
    pr = np.ascontiguousarray(_check_pair_table(pairs, C), dtype=np.int32)
    P = len(pr)
    if _check_model("F", F) != P:
        raise ValueError("F must hold one matrix per pair (%d), not %d" % (P, int(F.shape[0])))
    _check_floating((("F", F), ("intrinsics", intrinsics)))
    _check_mask(mask, "P", P)
    loss_scale, max_error, max_ratio, cg_tol = float(loss_scale), float(max_error), float(max_ratio), float(cg_tol)
    for nm, v in (("loss_scale", loss_scale), ("max_error", max_error), ("cg_tol", cg_tol)):
        if not 0.0 <= v < float("inf"):
            raise ValueError("%s must be a non-negative finite number, not %r" % (nm, v))
    if not 1.0 <= max_ratio < float("inf"):
        raise ValueError("max_ratio must be a finite number >= 1, not %r" % (max_ratio,))
    max_iters = _check_count("max_iters", max_iters, 0)
    cg_max_iters = _check_count("cg_max_iters", cg_max_iters, 1)
    dev = _check_device(named, mask)
    Fc, kc = _f64(F, intrinsics)
    f64, i32 = torch.float64, torch.int32
    L = _cabi.lib()
    ko = torch.empty((G, 5), dtype=f64, device=dev)
    ref = torch.empty(G, dtype=torch.uint8, device=dev)
    err = torch.empty(P, dtype=f64, device=dev)
    inl = torch.empty(P, dtype=torch.uint8, device=dev)
    cost0 = torch.empty(1, dtype=f64, device=dev)
    cost = torch.empty(1, dtype=f64, device=dev)
    iters = torch.empty(1, dtype=i32, device=dev)
    n_used = torch.empty(1, dtype=i32, device=dev)
    cg_iters = torch.empty(1, dtype=i32, device=dev)
    _call(L.dgb200_calibrate_view_graph_dev, L.dgb200_view_graph_calibration_last_error, dev,
          pr.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), P, C, Fc, _mask_u8(mask), groups.contiguous(), kc, G,
          loss_scale, max_error, max_ratio, max_iters, cg_max_iters, cg_tol, ko, ref, err, inl, cost0, cost, iters,
          n_used, cg_iters)
    return ViewGraphCalibration(ko, ref.view(torch.bool), err, inl.view(torch.bool), cost0, cost, iters, n_used,
                                cg_iters)


def average_rotations(pairs, R_rel, n_views, mask=None, weights=None, sigma=math.radians(5.0), l1_iters=5,
                      max_iters=100, step_tol=1e-6, cg_max_iters=500, cg_tol=1e-6):
    """Average the views' rotations over the view graph: a world rotation for each of n_views views from the relative
    rotations of its pairs, as global SfM starts (GLOMAP's rotation averager, on the device).  Translations are neither
    used nor produced.

    pairs: a HOST [P,2] table of (i, j), as match_descriptors_batch takes it.  R_rel: a CUDA float tensor [P,3,3] or
    [P,9] (used in float64) with x_j ~ R_rel[e] x_i, so R_rel[e] ~ R_j R_i^T: what pose_from_fundamental_ragged and
    refine_pose_ragged return for the pair (q, t) = (i, j).  mask: [P] bool / uint8 or None (every edge); weights:
    int32 [P] or None (all 0), the edges' priority in the spanning tree, such as pose.good.  An edge is used when
    i != j, its mask is set, its weight is >= 0 and R_rel is finite with det > 0.5 (a failed pose's R = 0 is not).
    The start is the maximum spanning forest under (weight, then lower edge index) with R = I at each component's
    smallest view; then at most l1_iters iterations of IRLS with L1 weights and at most max_iters with Geman-McClure
    weights of scale sigma (radians), each phase ending once no view moves by more than step_tol radians.  Each
    iteration solves the linearised problem by Jacobi-preconditioned CG, stopped at |r| <= cg_tol |b| or after
    cg_max_iters iterations.  sigma, l1_iters and max_iters default to GLOMAP's values; at 10^4 views and 2 10^5
    edges (tools/rotation_averaging_rate.py) step_tol ends the second phase after 8 iterations with the median error
    at 0.4 deg, below the 1 deg edge noise.  The estimator is specified in include/degensac_b200.h.
    Returns RotationAveraging(R, component, residual, iters, cg_iters): R [n_views,3,3] float64 world to camera, x ~
    K (R X + t) as find_absolute_pose_ragged, triangulate_tracks_ragged and the bundle adjustments take it (NaN for a
    view without a used edge); component int32 [n_views] the smallest view of each view's component, or -1; residual
    [P] float64 the angle of each edge's residual rotation at R, NaN for an edge that is not used; iters int32 [2] the
    iterations of each phase; cg_iters int32 [1] the CG iterations, summed.  Asynchronous, nothing is read back."""
    import torch
    pairs = _host_pairs(pairs)
    n_views = _check_count("n_views", n_views, 1)
    pr = np.ascontiguousarray(_check_pair_table(pairs, n_views), dtype=np.int32)
    P = len(pr)
    named = (("R_rel", R_rel),) + ((("weights", weights),) if weights is not None else ())
    _check_tensors(named, mask)
    if _check_model("R_rel", R_rel) != P:
        raise ValueError("R_rel must hold one rotation per pair (%d), not %d" % (P, int(R_rel.shape[0])))
    _check_floating(named[:1])
    _check_mask(mask, "P", P)
    if weights is not None:
        _check_shape("weights", weights, "P", (P,))
        _check_int32("weights", weights)
    sigma = float(sigma)
    if not 0.0 < sigma < float("inf"):
        raise ValueError("sigma must be a positive number, not %r" % (sigma,))
    l1_iters = _check_count("l1_iters", l1_iters, 0)
    max_iters = _check_count("max_iters", max_iters, 0)
    step_tol, cg_tol = float(step_tol), float(cg_tol)
    if not 0.0 <= step_tol < float("inf"):
        raise ValueError("step_tol must be a non-negative finite number, not %r" % (step_tol,))
    cg_max_iters = _check_count("cg_max_iters", cg_max_iters, 1)
    if not 0.0 <= cg_tol < float("inf"):
        raise ValueError("cg_tol must be a non-negative finite number, not %r" % (cg_tol,))
    dev = _check_device(named, mask)
    Rr = R_rel.to(torch.float64).contiguous()
    w = weights.contiguous() if weights is not None else None
    L = _cabi.lib()
    R = torch.empty((n_views, 3, 3), dtype=torch.float64, device=dev)
    comp = torch.empty(n_views, dtype=torch.int32, device=dev)
    res = torch.empty(P, dtype=torch.float64, device=dev)
    iters = torch.empty(2, dtype=torch.int32, device=dev)
    cg_iters = torch.empty(1, dtype=torch.int32, device=dev)
    _call(L.dgb200_average_rotations_dev, L.dgb200_rotation_averaging_last_error, dev,
          pr.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), P, n_views, Rr, _mask_u8(mask), w, sigma, l1_iters,
          max_iters, step_tol, cg_max_iters, cg_tol, R, comp, res, iters, cg_iters)
    return RotationAveraging(R, comp, res, iters, cg_iters)


def global_positioning_ragged(cams, pts, R, K, offsets, mask=None, seed=0, init_scale=100.0, loss_scale=0.1,
                              max_iters=100, max_angle=math.radians(2.0), cg_max_iters=500, cg_tol=1e-6):
    """Position the views and their tracks from the views' rotations: the centre of every view and the point of every
    track, as global SfM does after rotation averaging (GLOMAP's global positioner with point-to-camera constraints,
    on the device).  Translations are not taken.

    cams, pts, offsets and mask are CUDA tensors on one device in the layout of triangulate_tracks_ragged (the padded
    output of build_tracks_ragged goes in as it is); R [C,3,3] the world-to-camera rotations (what average_rotations
    returns: a view whose R is not finite or whose det R <= 0.5 is not registered); K [3,3] or [C,3,3].  Floating
    inputs are used in float64.  A track is used when its usable observations come from at least 2 distinct views.
    Each observation's ray v = normalise(R^T K^-1 (x, y, 1)) constrains its view's centre c and its track's point X
    through r = d (X - c) - v with a scale d >= 1e-5 of its own; the cost sum rho(|r|^2) uses the Huber loss of scale
    loss_scale (0: the squared error).  Levenberg-Marquardt from a random start (centres and points uniform in
    [-init_scale, init_scale]^3 from the Philox stream of `seed`, every d = 1) runs at most max_iters trial steps, each
    solved by conjugate gradients on the centres (cg_max_iters, cg_tol) once the scales and the points are
    eliminated.  Each component of the view graph has its smallest view at the origin and a free scale.  max_angle: the
    largest angle between an observation's ray and its point, in radians, for `inliers`.  The estimator is specified
    in include/degensac_b200.h.
    Returns GlobalPositioning(t, X, component, angle, inliers, cost0, cost, iters, n_used, cg_iters): t [C,3] float64 =
    -R c, so that (R, t) feeds triangulate_tracks_ragged and bundle_adjust_pcg_ragged (NaN for a view without a used
    observation); X [T,3] (NaN for a track that is not used); component int32 [C] the smallest view of each view's
    component, or -1; angle [obs] float64 (NaN for an observation that is not used); inliers [obs] bool, the used
    observations with angle <= max_angle, the mask that triangulation and bundle adjustment take next; cost0, cost [1]
    float64; iters, n_used, cg_iters [1] int32.  Asynchronous, nothing is read back."""
    import torch
    named = (("cams", cams), ("pts", pts), ("R", R), ("K", K), ("offsets", offsets))
    _check_tensors(named, mask)
    T = _check_offsets(offsets, "T")
    _check_int32("cams", cams)
    obs = _check_columns("pts", pts, "obs", 2)
    _check_shape("cams", cams, "obs", (obs,))
    if R.dim() != 3 or R.shape[0] < 1 or tuple(R.shape[1:]) != (3, 3):
        raise ValueError("R must be [C,3,3] with C >= 1, not %s" % list(R.shape))
    C = int(R.shape[0])
    _check_K("K", K, "C", C)
    _check_floating(named[1:4])
    _check_mask(mask, "obs", obs)
    seed = int(seed)
    if not 0 <= seed < 1 << 64:
        raise ValueError("seed must lie in [0, 2^64), not %d" % seed)
    init_scale, loss_scale, max_angle, cg_tol = float(init_scale), float(loss_scale), float(max_angle), float(cg_tol)
    for nm, v in (("init_scale", init_scale), ("loss_scale", loss_scale), ("max_angle", max_angle)):
        if not 0.0 <= v < float("inf"):
            raise ValueError("%s must be a non-negative finite number, not %r" % (nm, v))
    max_iters = _check_count("max_iters", max_iters, 0)
    cg_max_iters = _check_count("cg_max_iters", cg_max_iters, 1)
    if not 0.0 <= cg_tol < float("inf"):
        raise ValueError("cg_tol must be a non-negative finite number, not %r" % (cg_tol,))
    dev = _check_device(named, mask)
    x, Rc, Kc = _f64(pts, R, K)
    cm, off, m = cams.contiguous(), offsets.contiguous(), _mask_u8(mask)
    f64, i32 = torch.float64, torch.int32
    L = _cabi.lib()
    t = torch.empty((C, 3), dtype=f64, device=dev)
    X = torch.empty((T, 3), dtype=f64, device=dev)
    comp = torch.empty(C, dtype=i32, device=dev)
    ang = torch.empty(max(obs, 1), dtype=f64, device=dev)[:obs]
    inl = _rows_out(obs, dev)
    cost0 = torch.empty(1, dtype=f64, device=dev)
    cost = torch.empty(1, dtype=f64, device=dev)
    iters = torch.empty(1, dtype=i32, device=dev)
    n_used = torch.empty(1, dtype=i32, device=dev)
    cg_iters = torch.empty(1, dtype=i32, device=dev)
    _call(L.dgb200_global_positioning_ragged_dev, L.dgb200_global_positioning_last_error, dev, cm, x, Rc, Kc,
          int(Kc.dim() == 3), C, off, T, obs, m, seed, init_scale, loss_scale, max_iters, max_angle, cg_max_iters,
          cg_tol, t, X, comp, ang, inl, cost0, cost, iters, n_used, cg_iters)
    return GlobalPositioning(t, X, comp, ang, inl.view(torch.bool), cost0, cost, iters, n_used, cg_iters)


def match_descriptors_batch(descs, pairs, kps=None, ratio=0.9, mutual=False, norm="l2"):
    """match_descriptors over many image pairs in one call, output in the ragged layout of the offsets= entry points.

    descs: list of I CUDA tensors [n_i, D] (n_i may be 0; converted to float32 like match_descriptors), or with
    norm="hamming" uint8 tensors [n_i, B] with one B in [1, 256] (the distance and ratio test of match_descriptors).
    pairs: HOST [P,2] int array (numpy / list / CPU tensor) of (query image, train image); reading a CUDA tensor would
    synchronise, so one is refused.  kps: optional list of I tensors [n_i, k] (k >= 2; six columns carry the local
    affine shape through).
    Returns BatchMatches(idx1, idx2, pts1, pts2, offsets, n_max): pair p's matches, in ascending query order, are rows
    offsets[p] .. offsets[p+1]-1 of idx1/idx2 (int64, indices local to each image) and of pts1/pts2 (float64
    [capacity, 2|6], None without kps); offsets is an int32 CUDA tensor [P+1]; n_max is a host int bounding every pair's
    match count.  capacity is the sum of the query images' counts; rows past offsets[P] are unspecified.  A pair whose
    query image is empty or whose train image has fewer than 2 descriptors has no matches.  Asynchronous: nothing is
    read back from the device."""
    hamming = _check_norm(norm)
    pairs = _host_pairs(pairs)
    bank, counts, kbank = _banks(descs, kps, hamming)
    return _match_bank(bank, counts, pairs, kbank, ratio, mutual, hamming)


def match_descriptors_guided(descs, pairs, kps, models, px_th, guide="F", ratio=0.9, mutual=False, norm="l2"):
    """Guided matching: match_descriptors_batch with each pair's candidates restricted by a model of the pair.

    After a first pass (match_descriptors_batch, then findFundamentalMatrixBatch / findHomographyBatch on its ragged
    output), match the descriptors again, counting as candidates of a query only the train keypoints the pair's model
    allows: guide="F" (x_t^T F x_q = 0): the engine's Sampson residual of (query, train) at most px_th^2 -- the
    RANSAC's own inlier rule; guide="H" (x_t ~ H x_q): the query's transfer H x_q within px_th pixels of the train
    keypoint.  The 2-NN, ratio test and mutual check then run among those candidates; a query with one candidate passes
    the ratio test.  Repeated texture defeats the plain ratio test (the second neighbour is a look-alike elsewhere in the
    image); inside the gate the look-alike is usually gone, so many true matches come back.

    descs, pairs, ratio, mutual, norm: as match_descriptors_batch.  kps: list of I keypoint tensors [n_i, k] (k >= 2,
    x and y in the first two columns), required.  models: [P,3,3] or [P,9] float64, row-major, in the pair order of
    `pairs` (what findFundamentalMatrixBatch / findHomographyBatch return); a float64 CUDA tensor on the descriptors'
    device is used in place, other input is uploaded.  A pair whose model is all zeros (no model found) or holds a NaN
    gets no matches.  Returns BatchMatches like match_descriptors_batch; nothing is read back from the device."""
    import torch
    if guide not in ("F", "H"):
        raise ValueError("guide must be 'F' or 'H', not %r" % (guide,))
    px_th = _check_px_th(px_th, False)
    hamming = _check_norm(norm)
    pairs = _host_pairs(pairs)
    if kps is None:
        raise ValueError("guided matching needs the keypoints of every image (kps)")
    P = len(np.asarray(pairs))
    if not isinstance(models, torch.Tensor):
        models = np.array(models, dtype=np.float64)      # (a copy: torch wants a writable array)
    if tuple(models.shape) not in ((P, 9), (P, 3, 3)):
        raise ValueError("models must be [P,3,3] or [P,9] with P = %d pairs, not %s" % (P, list(models.shape)))
    bank, counts, kbank = _banks(descs, kps, hamming)
    dev = bank.device
    if isinstance(models, torch.Tensor) and models.is_cuda and models.device != dev:
        raise ValueError("models must be on the descriptors' device")
    M = torch.as_tensor(models).to(device=dev, dtype=torch.float64).contiguous().view(P, 9)
    return _match_bank(bank, counts, pairs, kbank, ratio, mutual, hamming,
                       guide=(_cabi.GUIDE_F if guide == "F" else _cabi.GUIDE_H), models=M, px_th=px_th)


def _host_pairs(pairs):
    import torch
    if isinstance(pairs, torch.Tensor):
        if pairs.is_cuda:
            raise ValueError("pairs must be a host array: reading a CUDA tensor would synchronise")
        pairs = pairs.numpy()
    return pairs


def _banks(descs, kps, hamming):
    """descriptor bank [R,D] (float32, or binary words), per-image counts and keypoint bank [R,k] float64 (or None)
    of the lists taken by match_descriptors_batch"""
    import torch
    if len(descs) < 1:
        raise ValueError("expected a non-empty list of descriptor tensors")
    dev = descs[0].device
    if hamming:
        ds = descs
        bank = _binary_words(list(ds))
    else:
        ds = [d.to(torch.float32) for d in descs]
        if not dev.type == "cuda" or any(d.dim() != 2 or d.device != dev or d.shape[1] != ds[0].shape[1] for d in ds):
            raise ValueError("expected CUDA descriptor tensors [n_i, D] with one D, on one device")
        bank = torch.cat(ds, 0).contiguous()
    counts = [int(d.shape[0]) for d in ds]
    kbank = None
    if kps is not None:
        if len(kps) != len(ds):
            raise ValueError("kps must hold one keypoint tensor per descriptor tensor")
        ks = [k.to(device=dev, dtype=torch.float64) for k in kps]
        if any(k.dim() != 2 or k.shape[0] != c or k.shape[1] != ks[0].shape[1] for k, c in zip(ks, counts)) \
                or ks[0].shape[1] < 2:
            raise ValueError("keypoint tensors must be [n_i, k] with one k >= 2")
        kbank = torch.cat(ks, 0).contiguous()
    return bank, counts, kbank


def _match_bank(bank, counts, pairs, kbank, ratio, mutual, hamming=False, guide=None, models=None, px_th=0.0):
    """The batched matcher over a descriptor bank [R,D] (any 4-byte alignment) whose image i owns rows
    sum(counts[:i]) .. sum(counts[:i+1])-1: float32 rows, or with `hamming` binary rows of D 32-bit words (D a
    multiple of 4); kbank: keypoint rows of the same images or None.  guide (_cabi.GUIDE_F / GUIDE_H): guided matching
    with models, a float64 CUDA tensor [P,9], and px_th."""
    import torch
    pr = np.ascontiguousarray(np.asarray(pairs), dtype=np.int32)
    lay = batch_layout(counts, pr)
    off = np.zeros(len(counts) + 1, dtype=np.int32)
    np.cumsum(counts, out=off[1:])
    P = pr.shape[0]
    D = int(bank.shape[1])
    dev = bank.device
    L = _cabi.lib()
    i32 = ctypes.POINTER(ctypes.c_int32)
    cap = max(lay.capacity, 1)        # (a zero-sized allocation would pass a null pointer)
    mq = torch.empty(cap, dtype=torch.int32, device=dev)
    mt = torch.empty(cap, dtype=torch.int32, device=dev)
    offsets = torch.empty(P + 1, dtype=torch.int32, device=dev)
    ws = torch.empty(max(int(L.dgb200_match_batch_workspace_bytes(off.ctypes.data_as(i32), len(counts),
                                                                  pr.ctypes.data_as(i32), P)), 1),
                     dtype=torch.uint8, device=dev)
    x1 = x2 = None
    kp_dim = out_dim = 0
    if kbank is not None:
        kp_dim = int(kbank.shape[1])
        out_dim = 6 if kp_dim >= 6 else 2
        x1 = torch.empty((cap, out_dim), dtype=torch.float64, device=dev)
        x2 = torch.empty((cap, out_dim), dtype=torch.float64, device=dev)
    guided = ()
    if guide is None:
        fn = L.dgb200_match_binary_descriptors_batch_dev if hamming else L.dgb200_match_descriptors_batch_dev
    else:
        fn = (L.dgb200_match_binary_descriptors_guided_batch_dev if hamming else
              L.dgb200_match_descriptors_guided_batch_dev)
        guided = (models, int(guide), px_th)
    _call(fn, L.dgb200_frontend_last_error, dev, bank, off.ctypes.data_as(i32), len(counts), D, pr.ctypes.data_as(i32),
          P, *guided, ratio, int(bool(mutual)), kbank, kp_dim, mq, mt, x1, x2, out_dim, cap, offsets, ws)
    return BatchMatches(mq.long(), mt.long(), x1, x2, offsets, lay.n_max)
