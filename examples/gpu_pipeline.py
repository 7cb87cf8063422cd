#!/usr/bin/env python
"""The reference's examples/simple-example.py pipeline with every step after feature extraction on the GPU:

    descriptors + keypoints (CUDA tensors)  ->  2-NN matching + SNN ratio test   (pydegensac_b200.matching, CUDA)
                                            ->  findHomography / findFundamentalMatrix (device-resident tensors)
                                            ->  F refined on the inliers (Sampson error)  (pydegensac_b200.matching)
                                            ->  guided re-match inside F's epipolar band   (pydegensac_b200.matching, CUDA)
                                            ->  relative pose from F                      (pydegensac_b200.matching)
                                            ->  pose refined on the inliers (Sampson error) (pydegensac_b200.matching)
    and the H branch for a planar scene:    ->  findHomographyBatch -> pose and scene plane from H
    and a third view:                       ->  its matches to view 0 carry the two-view points (scatter / gather)
                                            ->  absolute pose by P3P RANSAC                (pydegensac_b200.matching)
                                            ->  3-view tracks triangulated across the registered views
                                            ->  views 1 and 2 and the tracks bundle-adjusted, view 0 held
    and many views:                         ->  every pair matched and verified by the ragged F RANSAC
                                            ->  tracks built from the verified matches   (pydegensac_b200.matching, CUDA)
                                            ->  tracks triangulated with the views' poses
                                            ->  every view's rotation averaged over the view graph (CUDA)
                                            ->  every view's position and every track's point from the rotations
                                            ->  tracks triangulated on the positioning's inliers, bundle-adjusted
    and many views whose focal length is not known:
                                            ->  the camera's focal length from the pairs' F (view-graph calibration)
                                            ->  pose, rotations on the calibration's inlier pairs, positions, tracks
                                            ->  bundle adjustment that also refines the intrinsics

The reference does the matching with cv2.BFMatcher on the host (simple-example.py:46-53) and copies the tentative
correspondences into numpy arrays; here nothing visits the host between the descriptors and the inlier mask.
Feature extraction itself (AKAZE/SIFT) is outside the path: this script synthesises keypoints and descriptors.

    python examples/gpu_pipeline.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pydegensac_b200 as pydegensac
from pydegensac_b200.matching import (average_rotations, build_tracks_ragged, calibrate_view_graph, global_positioning_ragged, bundle_adjust_intrinsics_ragged, bundle_adjust_pcg_ragged,
                                      find_absolute_pose_ragged, undistort_points,
                                      match_descriptors, match_descriptors_batch, trim_tracks,
                                      match_descriptors_guided, pose_from_fundamental, pose_from_fundamental_ragged,
                                      pose_from_homography_ragged, refine_fundamental_ragged, refine_homography_ragged,
                                      refine_pose_ragged, triangulate_tracks_ragged, bundle_adjust_ragged)
from pydegensac_b200.scenes import scene_F, _K, _rot


def synth_features(n_true=1200, n_clutter=800, D=64, seed=0):
    """Two views of one scene: keypoints of scene_F + descriptors that agree (up to noise) on true matches."""
    rng = np.random.default_rng(seed)
    p1, p2, _ = scene_F(n_true, 1.0, seed)
    kp1 = np.r_[p1, rng.uniform(0, 640, (n_clutter, 2))]
    kp2 = np.r_[p2, rng.uniform(0, 640, (n_clutter, 2))]
    base = rng.normal(size=(n_true, D)).astype(np.float32)
    d1 = np.r_[base + 0.2 * rng.normal(size=base.shape).astype(np.float32), rng.normal(size=(n_clutter, D)).astype(np.float32)]
    d2 = np.r_[base + 0.2 * rng.normal(size=base.shape).astype(np.float32), rng.normal(size=(n_clutter, D)).astype(np.float32)]
    perm = rng.permutation(len(kp2))
    return kp1, d1, kp2[perm], d2[perm]


def synth_plane(n=1000, seed=1):
    """Two views of points on a plane (a facade 6 units away, tilted): pixel pairs with 0.3 px noise."""
    rng = np.random.default_rng(seed)
    R, t = _rot("y", -0.15) @ _rot("x", 0.05), np.array([1.0, 0.1, 0.2])
    nrm = np.array([0.2, -0.1, 1.0]) / np.linalg.norm([0.2, -0.1, 1.0])
    xy = np.c_[rng.uniform(-3, 3, n), rng.uniform(-2, 2, n)]
    X = np.c_[xy, (6.0 - xy @ nrm[:2]) / nrm[2]]
    x1, x2 = X @ _K.T, (X @ R.T + t) @ _K.T
    return (x1[:, :2] / x1[:, 2:3] + 0.3 * rng.normal(size=(n, 2)), x2[:, :2] / x2[:, 2:3] + 0.3 * rng.normal(size=(n, 2)))


def synth_views(n_img=3, n_pts=900, n_clutter=300, D=64, seed=3):
    """n_img views of one 3-D scene (view i at R_i = rot_y(0.08 i) rot_x(0.02 i), t_i = (0.6, 0.05, 0.1) i, x ~ K (R_i X +
    t_i)): per view keypoints and descriptors (a shared code per point plus noise, then clutter), (R_i, t_i), the
    points X and per view the index in X of each keypoint (-1 for clutter)"""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-4, 4, n_pts), rng.uniform(-4, 4, n_pts), rng.uniform(2, 12, n_pts)]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    kps, descs, poses, ids = [], [], [], []
    for i in range(n_img):
        R, t = _rot("y", 0.08 * i) @ _rot("x", 0.02 * i), np.array([0.6, 0.05, 0.1]) * i
        x = (X @ R.T + t) @ _K.T
        kp = np.r_[x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_pts, 2)), rng.uniform(0, 640, (n_clutter, 2))]
        d = np.r_[code + 0.15 * rng.normal(size=code.shape).astype(np.float32),
                  rng.normal(size=(n_clutter, D)).astype(np.float32)]
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm]); poses.append((R, t))
        ids.append(np.r_[np.arange(n_pts), np.full(n_clutter, -1)][perm])
    return kps, descs, poses, X, ids


def register_third_view(dev, K):
    """Two-view initialisation on views 0 and 1, then view 2 registered against its points and the tracks of view 0's
    keypoints triangulated across the three views, without a host read"""
    kps, descs, poses, X, ids = synth_views()
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    n0 = len(kps[0])
    m = match_descriptors_batch(dt, [(0, 1)], kt, ratio=0.9, mutual=True)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=[0], offsets=m.offsets,
                                                    n_max=m.n_max)
    pose = pose_from_fundamental_ragged(F, K, K, m.pts1, m.pts2, m.offsets, mask)
    fine = refine_pose_ragged(pose.R, pose.t, K, K, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
    tri = pose_from_fundamental_ragged(fine.F, K, K, m.pts1, m.pts2, m.offsets, fine.inliers)
    # the points (camera 0's frame, baseline units) onto view 0's keypoints through idx1; slot n0 takes the rows past
    # the pair's matches, which are never valid
    live = torch.arange(m.idx1.shape[0], device=dev) < m.offsets[1]
    slot = torch.where(live, m.idx1, n0)
    pts0 = torch.full((n0 + 1, 3), float("nan"), dtype=torch.float64, device=dev).index_put_((slot,), tri.points)
    valid0 = torch.zeros(n0 + 1, dtype=torch.bool, device=dev).index_put_((slot,), tri.in_front & live)
    # view 2 matched against view 0: its keypoints see view 0's points through idx2
    m2 = match_descriptors_batch(dt, [(2, 0)], kt, ratio=0.9, mutual=True)
    live2 = torch.arange(m2.idx2.shape[0], device=dev) < m2.offsets[1]
    src = torch.where(live2, m2.idx2, n0)
    view = find_absolute_pose_ragged(m2.pts1, pts0.index_select(0, src), K, m2.offsets,
                                     valid0.index_select(0, src) & live2, px_th=2.0, seeds=[0])
    (R0, t0), (R1, t1), (R2, t2) = poses
    R20 = R2 @ R0.T
    base = np.linalg.norm(t1 - R1 @ R0.T @ t0)
    Rv, tv = view.R[0].cpu().numpy(), view.t[0].cpu().numpy()
    print("view 2 registered: %d inliers after %d RANSAC iterations, MSAC cost %.2f -> %.2f px^2"
          % (int(view.n_inliers[0]), int(view.iters[0]), float(view.cost0[0]), float(view.cost[0])))
    print("  rotation error %.2e rad, translation error %.2e baselines (against the planted pose)"
          % (np.arccos(np.clip((np.trace(Rv @ R20.T) - 1) / 2, -1, 1)),
             np.linalg.norm(tv - (t2 - R20 @ t0) / base)))
    # 3-slot tracks keyed by view 0's keypoints: the keypoint, its match in view 1 (from the (0, 1) matches) and in
    # view 2 (from the (2, 0) matches); cameras view 0 = (I, 0), view 1 = the refined pose, view 2 = the registered pose
    f64 = torch.float64
    pts = torch.zeros((n0 + 1, 3, 2), dtype=f64, device=dev)
    seen = torch.zeros((n0 + 1, 3), dtype=torch.bool, device=dev)
    pts[:n0, 0] = kt[0].to(f64)
    seen[:n0, 0] = True
    pts[:, 1].index_put_((slot,), m.pts2.to(f64))
    seen[:, 1].index_put_((slot,), live)
    pts[:, 2].index_put_((src,), m2.pts1.to(f64))
    seen[:, 2].index_put_((src,), live2)
    R = torch.stack([torch.eye(3, dtype=f64, device=dev), fine.R[0], view.R[0]])
    t = torch.stack([torch.zeros(3, dtype=f64, device=dev), fine.t[0], view.t[0]])
    cams = torch.arange(3, dtype=torch.int32, device=dev).repeat(n0)
    offsets = torch.arange(0, 3 * n0 + 1, 3, dtype=torch.int32, device=dev)
    tr = triangulate_tracks_ragged(cams, pts[:n0].reshape(-1, 2), R, t, K, offsets, seen[:n0].reshape(-1), px_th=2.0)
    n_in = tr.n_inliers.cpu().numpy()
    ok = (n_in >= 2) & (ids[0] >= 0)
    truth = (X[ids[0][ok]] @ R0.T + t0) / base                # the planted points in camera 0's frame, baseline units
    err = np.linalg.norm(tr.X.cpu().numpy()[ok] - truth, axis=1)
    print("tracks of view 0's %d keypoints: %d triangulated (%d from all three views), median 3D error %.2e baselines "
          "against the planted points" % (n0, int((n_in >= 2).sum()), int((n_in == 3).sum()), float(np.median(err))))
    # bundle adjustment: views 1 and 2 and every track's point refined jointly, view 0 held and one translation
    # coordinate of view 1 held (the scale)
    ba = bundle_adjust_ragged(cams, pts[:n0].reshape(-1, 2), R, t, K, offsets, tr.X, mask=tr.mask, free=[1, 2],
                              scale_gauge=1, loss_scale=1.0)
    Rp = [R1 @ R0.T, R20]

    def rot_err(Rs):
        return sum(np.arccos(np.clip((np.trace(Rs[c].cpu().numpy() @ Rp[c - 1].T) - 1) / 2, -1, 1)) for c in (1, 2))
    # (the planted points are in baseline units: the adjusted scene is scaled back to |t_1| = 1 first)
    err_ba = np.linalg.norm(ba.X.cpu().numpy()[ok] / np.linalg.norm(ba.t[1].cpu().numpy()) - truth, axis=1)
    print("bundle adjustment of views 1 and 2 over %d observations in %d trial steps: cost %.2f -> %.2f" %
          (int(ba.n_used[0]), int(ba.iters[0]), float(ba.cost0[0]), float(ba.cost[0])))
    print("  summed rotation error of views 1 and 2 %.2e -> %.2e rad, median 3D error %.2e -> %.2e baselines"
          % (rot_err(R), rot_err(ba.R), float(np.median(err)), float(np.median(err_ba))))


def tracks_across_views(dev, K, n_img=6):
    """Every pair of n_img views matched and verified in one ragged batch, tracks built from the verified matches and
    triangulated with the views' (planted) poses, without a host read until the report"""
    kps, descs, poses, X, ids = synth_views(n_img=n_img, seed=5)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    pairs = np.array([(i, j) for i in range(n_img) for j in range(i + 1, n_img)], dtype=np.int32)
    m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=list(range(len(pairs))),
                                                    offsets=m.offsets, n_max=m.n_max)
    ts = build_tracks_ragged([len(k) for k in kps], pairs, m.idx1, m.idx2, m.offsets, mask, kps=kt)
    f64 = torch.float64
    R = torch.from_numpy(np.stack([p[0] for p in poses])).to(dev, f64)
    t = torch.from_numpy(np.stack([p[1] for p in poses])).to(dev, f64)
    # the padded layout goes straight in: the empty tracks past the last one get no model
    tr = triangulate_tracks_ragged(ts.cams, ts.pts, R, t, K, ts.offsets, px_th=2.0)
    ex = trim_tracks(ts)                                      # the one host read of the track builder
    off, cams, kp = ex.offsets.cpu().numpy(), ex.cams.cpu().numpy(), ex.kp.cpu().numpy()
    T = len(off) - 1
    pid = np.array([ids[c][k] for c, k in zip(cams, kp)])
    pure = np.array([pid[off[j]] >= 0 and (pid[off[j]:off[j + 1]] == pid[off[j]]).all() for j in range(T)])
    s = ts.stats.cpu().numpy()
    print("%d views, %d pairs: %d tracks of %d observations (longest %d), %.1f %% of them pure; %d conflicting "
          "components (%d keypoints) dropped" % (n_img, len(pairs), T, len(cams), int(np.diff(off).max()),
                                                  100 * pure.mean(), int(s[2]), int(s[3])))
    n_in = tr.n_inliers[:T].cpu().numpy()
    ok = (n_in >= 2) & pure
    err = np.linalg.norm(tr.X[:T].cpu().numpy()[ok] - X[pid[off[:-1]][ok]], axis=1)
    print("  %d tracks triangulated with the planted poses, median 3D error %.2e units" % (int((n_in >= 2).sum()),
                                                                                        float(np.median(err))))


def path_scene(dev, n_img=100, n_pts=20000, D=64, seed=7):
    """n_img views along a path looking at one scene, with keypoints and descriptors on the device, and the pairs of
    each view with its next three.  Returns (rng, planted rotations, planted translations, kps, descs, pairs)"""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-3, 0.3 * n_img + 3, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(4, 10, n_pts)]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    Rs = np.stack([_rot("y", rng.uniform(-0.05, 0.05)) @ _rot("x", rng.uniform(-0.03, 0.03)) for _ in range(n_img)])
    ts = -np.einsum("cij,cj->ci", Rs, np.c_[0.3 * np.arange(n_img), np.zeros((n_img, 2))])
    kps, descs = [], []
    for i in range(n_img):
        q = (X @ Rs[i].T + ts[i]) @ _K.T
        x = q[:, :2] / q[:, 2:3]
        seen = np.flatnonzero((q[:, 2] > 0) & (x[:, 0] > 0) & (x[:, 0] < 640) & (x[:, 1] > 0) & (x[:, 1] < 480))
        kps.append(torch.from_numpy(x[seen] + 0.3 * rng.normal(size=(len(seen), 2))).to(dev))
        descs.append(torch.from_numpy(code[seen] + 0.15 * rng.normal(size=(len(seen), D)).astype(np.float32)).to(dev))
    pairs = np.array([(i, j) for i in range(n_img) for j in range(i + 1, min(i + 4, n_img))], dtype=np.int32)
    return rng, Rs, ts, kps, descs, pairs


def global_adjustment(dev, K, n_img=100, n_pts=20000, D=64, seed=7):
    """n_img views along a path, each matched with its next three and verified in one ragged batch, tracks built and
    triangulated from perturbed planted poses, then one bundle adjustment of every view but view 0 -- more cameras
    than bundle_adjust_ragged takes -- by conjugate gradients on the implicit Schur complement"""
    rng, Rs, ts, kps, descs, pairs = path_scene(dev, n_img, n_pts, D, seed)
    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=list(range(len(pairs))),
                                                    offsets=m.offsets, n_max=m.n_max)
    tk = build_tracks_ragged([len(k) for k in kps], pairs, m.idx1, m.idx2, m.offsets, mask, kps=kps)
    # the start: every view but view 0 rotated by ~2e-3 rad and moved by ~1e-2
    R0, t0 = Rs.copy(), ts.copy()
    for c in range(1, n_img):
        a = 2e-3 * rng.normal(size=3)
        A = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
        th = np.linalg.norm(a)
        R0[c] = (np.eye(3) + np.sin(th) / th * A + (1 - np.cos(th)) / th ** 2 * A @ A) @ Rs[c]
        t0[c] = ts[c] + 1e-2 * rng.normal(size=3)
    f64 = torch.float64
    R, t = torch.from_numpy(R0).to(dev, f64), torch.from_numpy(t0).to(dev, f64)
    tr = triangulate_tracks_ragged(tk.cams, tk.pts, R, t, K, tk.offsets, px_th=3.0)
    gb = bundle_adjust_pcg_ragged(tk.cams, tk.pts, R, t, K, tk.offsets, tr.X, mask=tr.mask, loss_scale=1.0)

    def rot_err(Rx):
        Rx = Rx.cpu().numpy()
        return np.degrees(max(np.arccos(np.clip((np.trace(Rx[c] @ Rs[c].T) - 1) / 2, -1, 1)) for c in range(n_img)))
    n_tr = int(tk.stats[0])
    print("%d views, %d pairs: %d tracks; global bundle adjustment of %d views over %d observations in %d trial steps "
          "(%d CG iterations): cost %.1f -> %.1f" % (n_img, len(pairs), n_tr, n_img - 1, int(gb.n_used[0]),
                                                      int(gb.iters[0]), int(gb.cg_iters[0]), float(gb.cost0[0]),
                                                      float(gb.cost[0])))
    print("  largest rotation error %.2e -> %.2e deg against the planted poses" % (rot_err(R), rot_err(gb.R)))


def view_graph_scene(dev, n_bad=6, seed=11):
    """The path scene of global_adjustment and n_bad long-range pairs (i, i + 40) whose relative rotation will be a
    random one (a wrong pose that passed verification); the random rotations are uploaded here, before the device
    pipeline runs"""
    scene = path_scene(dev)
    n_img = len(scene[1])
    rng = np.random.default_rng(seed)
    first = rng.choice(n_img - 40, n_bad, replace=False)
    bad = np.c_[first, first + 40].astype(np.int32)
    q, _ = np.linalg.qr(rng.normal(size=(n_bad, 3, 3)))
    q *= np.sign(np.linalg.det(q))[:, None, None]
    return scene + (bad, torch.from_numpy(q).to(dev))


def view_graph_rotations(dev, K, scene):
    """Every pair of the scene matched, verified by the ragged F RANSAC, posed and refined; the bad pairs appended with
    their random rotations and a support of 30; then the rotations averaged over the view graph, ranked by the pairs'
    support -- the spanning-tree start alone, and the whole estimator.  No host read."""
    _, Rs, _, kps, descs, pairs, bad, R_bad = scene
    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                    n_max=m.n_max)
    pose = pose_from_fundamental_ragged(F, K, K, m.pts1, m.pts2, m.offsets, mask)
    fine = refine_pose_ragged(pose.R, pose.t, K, K, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
    all_pairs = np.r_[pairs, bad]
    R_rel = torch.cat([fine.R, R_bad])
    good = torch.cat([pose.good, torch.full((len(bad),), 30, dtype=torch.int32, device=dev)])
    start = average_rotations(all_pairs, R_rel, len(Rs), weights=good, l1_iters=0, max_iters=0)
    return start, average_rotations(all_pairs, R_rel, len(Rs), weights=good)


def report_view_graph(scene, out):
    """Prints the largest rotation error of the start and of the result against the planted rotations (the gauge
    aligned at view 0), in degrees, and returns them"""
    Rs, pairs, bad = scene[1], scene[5], scene[6]
    start, ra = out

    def largest(R):
        R = R.cpu().numpy()
        R = R @ (R[0].T @ Rs[0])
        return np.degrees(max(np.arccos(np.clip((np.trace(R[c] @ Rs[c].T) - 1) / 2, -1, 1)) for c in range(len(Rs))))
    e0, e1 = largest(start.R), largest(ra.R)
    res = np.degrees(ra.residual.cpu().numpy())
    print("rotation averaging of %d views over %d verified pairs and %d wrong ones: %s L1 and %s Geman-McClure "
          "iterations (%d CG); residual of the wrong pairs %.1f deg at least, of the others %.3f deg at most"
          % (len(Rs), len(pairs), len(bad), *ra.iters.cpu().tolist(), int(ra.cg_iters[0]), res[len(pairs):].min(),
             np.nanmax(res[:len(pairs)])))
    print("  largest rotation error %.3f deg from the spanning tree, %.3f deg averaged (against the planted rotations)"
          % (e0, e1))
    return e0, e1


def rotations_from_view_graph(dev, K):
    """A world rotation for each of 100 views from the verified relative poses of their pairs, a few wrong pairs
    among them"""
    scene = view_graph_scene(dev)
    report_view_graph(scene, view_graph_rotations(dev, K, scene))



def global_reconstruction_run(dev, K, scene):
    """Global SfM on the path scene with no pose from outside and no host read: every pair matched, verified by the
    ragged F RANSAC, posed and refined; the rotations averaged over the view graph; tracks built from the verified
    matches (their padded layout as it is); the views' positions and the tracks' points from the rotations; the tracks
    triangulated on the positioning's inliers; one bundle adjustment of every view but view 0.  Returns (rotation
    averaging, positioning, triangulation, bundle adjustment)"""
    _, Rs, _, kps, descs, pairs = scene
    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                    n_max=m.n_max)
    pose = pose_from_fundamental_ragged(F, K, K, m.pts1, m.pts2, m.offsets, mask)
    fine = refine_pose_ragged(pose.R, pose.t, K, K, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
    ra = average_rotations(pairs, fine.R, len(Rs), weights=pose.good)
    tk = build_tracks_ragged([len(k) for k in kps], pairs, m.idx1, m.idx2, m.offsets, mask, kps=kps)
    gpos = global_positioning_ragged(tk.cams, tk.pts, ra.R, K, tk.offsets)
    tr = triangulate_tracks_ragged(tk.cams, tk.pts, ra.R, gpos.t, K, tk.offsets, mask=gpos.inliers, px_th=3.0)
    ba = bundle_adjust_pcg_ragged(tk.cams, tk.pts, ra.R, gpos.t, K, tk.offsets, tr.X, mask=tr.mask, loss_scale=1.0)
    return ra, gpos, tr, ba


def similarity_errors(R, t, Rs, ts):
    """The errors against the planted poses after the similarity world_true = s Q world_est + tau that best fits them:
    Q from the rotations (the chordal mean, R_true ~ R_est Q^T: the path's centres lie on a line, so they leave the
    rotation about it open), then s and tau from the centres by least squares.  Returns (centre errors in units of the
    planted scene, rotation errors in degrees)"""
    M = np.einsum("cji,cjk->ik", R, Rs)               # sum R_est^T R_true
    U, _, Vt = np.linalg.svd(M)
    G = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))]) @ Vt
    Ra = R @ G                                         # G = Q^T
    er = np.degrees(np.arccos(np.clip((np.einsum("cij,cij->c", Ra, Rs) - 1.0) / 2.0, -1.0, 1.0)))
    C = -np.einsum("cji,cj->ci", R, t)
    Ct = -np.einsum("cji,cj->ci", Rs, ts)
    A = (C - C.mean(0)) @ G                            # Q (C - mean), row by row
    B = Ct - Ct.mean(0)
    s = np.sum(A * B) / np.sum(A * A)
    ec = np.linalg.norm(s * A - B, axis=1)
    return ec, er


def report_global_reconstruction(scene, out):
    """Prints the centre and rotation errors against the planted poses after positioning and after bundle adjustment,
    and returns the largest of each: (centre after positioning, centre after BA, rotation after BA in degrees)"""
    _, Rs, ts = scene[:3]
    ra, gpos, tr, ba = out
    R = ra.R.cpu().numpy()
    c0, r0 = similarity_errors(R, gpos.t.cpu().numpy(), Rs, ts)
    c1, r1 = similarity_errors(ba.R.cpu().numpy(), ba.t.cpu().numpy(), Rs, ts)
    print("global reconstruction of %d views: positioning in %d trial steps (%d CG), %d of %d observations inliers; "
          "%d tracks triangulated; bundle adjustment in %d trial steps" % (
              len(Rs), int(gpos.iters[0]), int(gpos.cg_iters[0]), int(gpos.inliers.sum()), int(gpos.n_used[0]),
              int((tr.n_inliers >= 2).sum()), int(ba.iters[0])))
    print("  centre error (baseline 0.3): largest %.2e positioned, %.2e adjusted; rotation error: largest %.3f deg "
          "averaged, %.3f deg adjusted" % (c0.max(), c1.max(), r0.max(), r1.max()))
    return c0.max(), c1.max(), r1.max()


def global_reconstruction(dev, K):
    """The path scene's 100 views from descriptors to a bundle-adjusted reconstruction, no poses from outside"""
    scene = path_scene(dev)
    report_global_reconstruction(scene, global_reconstruction_run(dev, K, scene))


def uncalibrated_reconstruction_run(dev, scene, k_start=(768.0, 320.0, 240.0, 0.0, 0.0)):
    """Global SfM on the path scene without K from outside and with no host read: every pair matched and verified by the
    ragged F RANSAC; one camera group's focal length calibrated from the pairs' F, starting from k_start (f0 = 1.2
    max(w, h), the usual guess without EXIF; the planted f is 800); K built from the result on the device; pose and
    refinement with it; the rotations averaged over the calibration's inlier pairs; tracks, positions and triangulation;
    one bundle adjustment that also refines the intrinsics, from the calibrated ones.  Returns (calibration, rotation
    averaging, positioning, triangulation, bundle adjustment)"""
    _, Rs, _, kps, descs, pairs = scene
    f64, i32 = torch.float64, torch.int32
    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    F, mask = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                    n_max=m.n_max)
    groups = torch.zeros(len(Rs), dtype=i32, device=dev)            # one camera took every view
    # filled on the device from Python scalars (a fill, not a copy from the host, which would synchronise)
    k0 = torch.stack([torch.full((), v, dtype=f64, device=dev) for v in k_start]).view(1, 5)
    cal = calibrate_view_graph(pairs, F, groups, k0)
    k = cal.intrinsics[0]
    zero, one = torch.zeros((), dtype=f64, device=dev), torch.ones((), dtype=f64, device=dev)
    K = torch.stack([k[0], zero, k[1], zero, k[0], k[2], zero, zero, one]).view(3, 3)
    pose = pose_from_fundamental_ragged(F, K, K, m.pts1, m.pts2, m.offsets, mask)
    fine = refine_pose_ragged(pose.R, pose.t, K, K, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
    ra = average_rotations(pairs, fine.R, len(Rs), mask=cal.inliers, weights=pose.good)
    tk = build_tracks_ragged([len(k) for k in kps], pairs, m.idx1, m.idx2, m.offsets, mask, kps=kps)
    gpos = global_positioning_ragged(tk.cams, tk.pts, ra.R, K, tk.offsets)
    tr = triangulate_tracks_ragged(tk.cams, tk.pts, ra.R, gpos.t, K, tk.offsets, mask=gpos.inliers, px_th=3.0)
    ba = bundle_adjust_intrinsics_ragged(tk.cams, tk.pts, ra.R, gpos.t, groups, cal.intrinsics, tk.offsets, tr.X,
                                         mask=tr.mask, loss_scale=1.0)
    return cal, ra, gpos, tr, ba


def report_uncalibrated_reconstruction(scene, out, f_true=800.0, f_start=768.0):
    """Prints the focal error at the start, after calibration and after bundle adjustment, and the largest centre and
    rotation errors after bundle adjustment; returns (relative focal error after calibration, after BA, largest centre
    error, largest rotation error in degrees)"""
    _, Rs, ts, _, _, pairs = scene
    cal, ra, gpos, tr, ba = out
    f_cal, f_ba = float(cal.intrinsics[0, 0]), float(ba.intrinsics[0, 0])
    c1, r1 = similarity_errors(ba.R.cpu().numpy(), ba.t.cpu().numpy(), Rs, ts)
    print("uncalibrated reconstruction of %d views: calibration over %d of %d pairs in %d trial steps (%d CG), %d "
          "inlier pairs; bundle adjustment with the intrinsics in %d trial steps"
          % (len(Rs), int(cal.n_used[0]), len(pairs), int(cal.iters[0]), int(cal.cg_iters[0]), int(cal.inliers.sum()),
             int(ba.iters[0])))
    e = [abs(f - f_true) / f_true for f in (f_start, f_cal, f_ba)]
    print("  focal length %.1f -> %.2f calibrated -> %.2f adjusted (planted %.0f: error %.2f %% -> %.3f %% -> %.3f %%);"
          " largest centre error %.2e (baseline 0.3), rotation error %.3f deg"
          % (f_start, f_cal, f_ba, f_true, 100 * e[0], 100 * e[1], 100 * e[2], c1.max(), r1.max()))
    return e[1], e[2], c1.max(), r1.max()


def uncalibrated_reconstruction(dev):
    """The path scene's 100 views from descriptors to a bundle-adjusted reconstruction, with neither K nor poses from
    outside"""
    scene = path_scene(dev)
    report_uncalibrated_reconstruction(scene, uncalibrated_reconstruction_run(dev, scene))


def self_calibration(dev, n_img=20, n_pts=4000, seed=9):
    """Views through a lens with radial distortion (f = 520, k1 = -0.08, k2 = 0.01), known tracks, and a start with a
    focal length 5 % off and no distortion: undistort, triangulate, adjust poses, points and the intrinsics of the one
    camera, then undistort again with the refined intrinsics and re-triangulate"""
    rng = np.random.default_rng(seed)
    k_true = np.array([520.0, 320.0, 240.0, -0.08, 0.01])
    X = np.c_[rng.uniform(-3, 0.3 * n_img + 3, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(4, 10, n_pts)]
    Rs = np.stack([_rot("y", rng.uniform(-0.05, 0.05)) @ _rot("x", rng.uniform(-0.03, 0.03)) for _ in range(n_img)])
    ts = -np.einsum("cij,cj->ci", Rs, np.c_[0.3 * np.arange(n_img), np.zeros((n_img, 2))])
    cams, pts, off = [], [], [0]
    for j in range(n_pts):
        p = np.einsum("cij,j->ci", Rs, X[j]) + ts
        u = p[:, :2] / p[:, 2:]
        s = (u ** 2).sum(1)
        x = (k_true[0] * (1 + s * (k_true[3] + s * k_true[4])))[:, None] * u + k_true[1:3]
        seen = np.flatnonzero((x[:, 0] > 0) & (x[:, 0] < 640) & (x[:, 1] > 0) & (x[:, 1] < 480))
        cams.append(seen)
        pts.append(x[seen] + 0.3 * rng.normal(size=(len(seen), 2)))
        off.append(off[-1] + len(seen))
    f64, i32 = torch.float64, torch.int32
    cams = torch.from_numpy(np.concatenate(cams).astype(np.int32)).to(dev)
    pts = torch.from_numpy(np.concatenate(pts)).to(dev)
    off = torch.tensor(off, dtype=i32, device=dev)
    R, t = torch.from_numpy(Rs).to(dev, f64), torch.from_numpy(ts).to(dev, f64)
    groups = torch.zeros(n_img, dtype=i32, device=dev)                 # one camera for every view
    k0 = k_true.copy()
    k0[0] *= 1.05
    k0[3:] = 0.0
    intr = torch.from_numpy(k0[None]).to(dev)

    def pinhole(k):
        return torch.tensor([[k[0], 0.0, k[1]], [0.0, k[0], k[2]], [0.0, 0.0, 1.0]], dtype=f64, device=dev)

    def triangulate(k):
        und = undistort_points(pts, cams, groups, torch.from_numpy(k[None]).to(dev))
        return triangulate_tracks_ragged(cams, und, R, t, pinhole(k), off, px_th=4.0)

    tr = triangulate(k0)
    sc = bundle_adjust_intrinsics_ragged(cams, pts, R, t, groups, intr, off, tr.X, mask=tr.mask, loss_scale=1.0)
    k1 = sc.intrinsics[0].cpu().numpy()
    tr2 = triangulate(k1)

    def med_err(Xe):
        return float(np.nanmedian(np.linalg.norm(Xe.cpu().numpy() - X, axis=1)))
    print("self-calibration of %d views over %d observations in %d trial steps (%d CG iterations): cost %.1f -> %.1f"
          % (n_img, int(sc.n_used[0]), int(sc.iters[0]), int(sc.cg_iters[0]), float(sc.cost0[0]), float(sc.cost[0])))
    print("  focal error %.2f -> %.3f px, k1 error %.2e -> %.2e; median 3D error %.2e -> %.2e units after "
          "re-triangulation" % (abs(k0[0] - k_true[0]), abs(k1[0] - k_true[0]), abs(k0[3] - k_true[3]),
                                abs(k1[3] - k_true[3]), med_err(tr.X), med_err(tr2.X)))

def main():
    dev = torch.device("cuda:0")
    kp1, d1, kp2, d2 = (torch.from_numpy(a).to(dev) for a in synth_features())
    # SNN ratio test 0.9 as in the reference's example; tentatives stay on the device
    idx1, idx2, pts1, pts2 = match_descriptors(d1, d2, kp1, kp2, ratio=0.9, mutual=True)
    print("tentative correspondences:", len(idx1))
    F, mask = pydegensac.findFundamentalMatrixBatch(pts1[None], pts2[None], 0.5, 0.999, 50000, seeds=[0])
    print("pydegensac_b200 found %d inliers" % int(mask.sum()))
    # F refined on its inliers (Sampson error over the rank-2 matrices, no intrinsics needed), through the ragged entry
    # points with one pair
    offsets = torch.tensor([0, len(idx1)], dtype=torch.int32, device=dev)
    ff = refine_fundamental_ragged(F, pts1, pts2, offsets, mask[0], px_th=1.0)
    print("F refined on %d rows in %d trial steps: summed Sampson error %.3f -> %.3f px^2, %d inliers at 1 px"
          % (int(ff.n_used[0]), int(ff.iters[0]), float(ff.cost0[0]), float(ff.cost[0]), int(ff.inliers.sum())))
    # guided re-match: candidates of a query are the train keypoints within 1 px (Sampson) of its epipolar line under
    # the refined F
    g = match_descriptors_guided([d1, d2], [[0, 1]], [kp1, kp2], ff.F, 1.0, guide="F", ratio=0.9)
    print("tentative correspondences: %d unguided, %d guided by F" % (len(idx1), int(g.offsets[1])))
    K = torch.from_numpy(_K).to(dev)
    R, t, good = pose_from_fundamental(F, K, K, pts1[None], pts2[None], mask)
    print("R =\n", R[0].cpu().numpy(), "\nt =", t[0].cpu().numpy(), " (%d correspondences in front of both cameras)" % int(good[0]))
    # refinement of the pose on the inliers in front of both cameras
    pose = pose_from_fundamental_ragged(F, K, K, pts1, pts2, offsets, mask[0])
    fine = refine_pose_ragged(pose.R, pose.t, K, K, pts1, pts2, offsets, pose.in_front, px_th=0.5)
    print("refined on %d rows in %d trial steps: sum of squared Sampson residuals %.3f -> %.3f px^2, %d inliers at 0.5 px"
          % (int(fine.n_used[0]), int(fine.iters[0]), float(fine.cost0[0]), float(fine.cost[0]), int(fine.inliers.sum())))
    print("R =\n", fine.R[0].cpu().numpy(), "\nt =", fine.t[0].cpu().numpy())
    # the H branch: a planar scene, where F is not determined; pose and plane from H, the two best decompositions
    q1, q2 = (torch.from_numpy(a).to(dev) for a in synth_plane())
    qoff = torch.tensor([0, len(q1)], dtype=torch.int32, device=dev)
    H, hmask = pydegensac.findHomographyBatch(q1, q2, 2.0, 0.999, 10000, seeds=[0], offsets=qoff, n_max=len(q1))
    # H refined on its inliers (Sampson error of the RANSAC's rule), then pose from the refined H
    fh = refine_homography_ragged(H, q1, q2, qoff, hmask, px_th=2.0)
    print("H refined on %d rows in %d trial steps: summed Sampson error %.3f -> %.3f px^2, %d inliers at 2 px"
          % (int(fh.n_used[0]), int(fh.iters[0]), float(fh.cost0[0]), float(fh.cost[0]), int(fh.inliers.sum())))
    hp = pose_from_homography_ragged(fh.H, K, K, q1, q2, qoff, fh.inliers)
    for c, name in enumerate(("chosen", "runner-up")):
        print("H branch, %s pose (%d votes): R =\n" % (name, int(hp.good[0, c])), hp.R[0, c].cpu().numpy(),
              "\nt =", hp.t[0, c].cpu().numpy(), " plane n =", hp.plane[0, c, :3].cpu().numpy(),
              " d = %.3f" % float(hp.plane[0, c, 3]))
    print("median parallax of the chosen pose: %.2f deg" % np.degrees(float(hp.median_angle[0])))
    register_third_view(dev, K)
    tracks_across_views(dev, K)
    global_adjustment(dev, K)
    rotations_from_view_graph(dev, K)
    global_reconstruction(dev, K)
    self_calibration(dev)
    uncalibrated_reconstruction(dev)


if __name__ == "__main__":
    main()
