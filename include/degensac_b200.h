/*
 * degensac_b200.h -- C ABI of the CUDA (sm_90a) LO-RANSAC / DEGENSAC engine (libdegensac_b200.so).
 *
 * Drop-in boundary for the reference's hot path.  Each entry point states the reference interface it
 * replaces; conventions (thresholds, metric numbering, model layout) are those of the reference's
 * binding layer so that a maintainer can rebind `pydegensac.findHomography_/findFundamentalMatrix_`
 * one-to-one (see INTEGRATION.md).  Plain pointers and sizes only: no torch / pybind types.
 *
 * Common conventions
 *   x1y1, x2y2 : row-major [n_pairs][n][dim] float64, dim = 2 (x,y) or 6 (x,y,a11,a12,a21,a22); only
 *                columns 0-1 are correspondences (bindings.cpp:180-197, 391-408).
 *   px_th, conf, max_iters, error_type, sym_check, laf_coef : exactly the arguments of
 *                findFundamentalMatrix_/findHomography_ (bindings.cpp:484-503); thresholds are squared /
 *                scaled inside, as the binding does (bindings.cpp:64-107, 297-318).
 *   seeds      : one uint64 per pair (NULL -> pair index).  The reference seeds libc rand() from
 *                time(NULL) (exp_ranF.c:1277, exp_ranH.c:510); here sampling is a counter-based Philox
 *                stream keyed by (seed, iteration, draw) -> reproducible and order-independent.
 *   model_out  : [n_pairs][9] float64.  F: row-major, x2^T F x1 = 0 (as the reference returns it).
 *                H: RAW core output = column-major, maps image 2 -> image 1, i.e. what
 *                exp_ransacHcustomLAF writes; the Python layer applies inv(H.T) (utils.py:108).
 *                All-zero model = "no model found" (then the mask is all zero, utils.py:104-107,143-145).
 *   mask_out   : [n_pairs][n] uint8 (1 = inlier).
 *   stats_out  : [n_pairs][4] int32 or NULL: {samples drawn, LO runs, plane inliers (F) / 0 (H),
 *                inlier count of the returned model}  (the reference's data_out[0..1], *Ih, return value).
 *   return     : 0 ok; <0 error (DGB200_E_*), message via dgb200_last_error().
 */
#ifndef DEGENSAC_B200_H
#define DEGENSAC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGB200_OK 0
#define DGB200_E_ARG (-1)          /* bad shape: n < 8 (F) / n < 4 (H), dim not 2 or 6 (bindings.cpp:32-47, 267-282) */
#define DGB200_E_METRIC (-2)       /* unknown error_type (bindings.cpp:10-17) */
#define DGB200_E_UNSUPPORTED (-3)  /* a launch switch this build does not support (DGB200_SMEM_TILE without -DDG_SOA_LD=0) */
#define DGB200_E_CUDA (-10)        /* no device / CUDA runtime failure: the engine has no CPU fallback */

/* error_type numbering of the reference (bindings.cpp:10-17) */
#define DGB200_F_SAMPSON 0
#define DGB200_F_SYMM_EPIPOLAR 1
#define DGB200_H_SAMPSON 0
#define DGB200_H_SYMM_SQ_MAX 1
#define DGB200_H_SYMM_MAX 2
#define DGB200_H_SYMM_SQ_SUM 3
#define DGB200_H_SYMM_SUM 4

/* Replaces exp_ransacFcustomLAF (exp_ranF.h:69-74, exp_ranF.c:1244) as called by findFundamentalMatrix_
 * (bindings.cpp:253-467), batched over independent image pairs.  HOST buffers; synchronous (copies in,
 * runs the wave/replay kernel, copies out). */
int dgb200_find_fundamental_batch(const double* x1y1, const double* x2y2, int n_pairs, int n, int dim,
                                  double px_th, double conf, int max_iters, int error_type, int sym_check,
                                  double laf_coef, int degen_check, const uint64_t* seeds,
                                  double* F_out, uint8_t* mask_out, int32_t* stats_out);

/* Replaces exp_ransacHcustomLAF (exp_ranH.h:27-33, exp_ranH.c:470; iter_type 4, oriented constraint on,
 * inlLimit 0) as called by findHomography_ (bindings.cpp:19-251).  HOST buffers; synchronous. */
int dgb200_find_homography_batch(const double* x1y1, const double* x2y2, int n_pairs, int n, int dim,
                                 double px_th, double conf, int max_iters, int error_type, int sym_check,
                                 double laf_coef, const uint64_t* seeds,
                                 double* H_out, uint8_t* mask_out, int32_t* stats_out);

/* Same two paths with DEVICE pointers (inputs already resident in HBM, outputs left in HBM) on a CUDA
 * stream (cudaStream_t passed as void*; NULL = default stream).  Asynchronous: returns after enqueueing.
 * Re-entrant: every launch in flight owns its scratch slabs and work counter (a pool keyed by stream), so calls on
 * different streams -- F and H mixed -- may overlap; calls on one stream are ordered by the stream.  Input pointers
 * need only the natural 8-byte alignment of float64 (16-byte aligned [n,2] inputs are read with 128-bit loads). */
int dgb200_find_fundamental_batch_dev(const double* d_x1y1, const double* d_x2y2, int n_pairs, int n, int dim,
                                      double px_th, double conf, int max_iters, int error_type, int sym_check,
                                      double laf_coef, int degen_check, const uint64_t* d_seeds,
                                      double* d_F_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream);
int dgb200_find_homography_batch_dev(const double* d_x1y1, const double* d_x2y2, int n_pairs, int n, int dim,
                                     double px_th, double conf, int max_iters, int error_type, int sym_check,
                                     double laf_coef, const uint64_t* d_seeds,
                                     double* d_H_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream);

/* Flagged variants.  DGB200_FLAG_FINAL_LSQ = the reference's compile-time option __FINAL_LSQ__ (exp_ranF.h:28-29;
 * exp_ranF.c:1701-1705, exp_ranH.c:866-870): after the loop one more least-squares fit on all inliers of the best
 * model, the inlier mask is derived from the polished model's residuals (SURVEY.md section 8(f).4). */
#define DGB200_FLAG_FINAL_LSQ 1u
int dgb200_find_fundamental_batch_ex(const double* x1y1, const double* x2y2, int n_pairs, int n, int dim,
                                     double px_th, double conf, int max_iters, int error_type, int sym_check,
                                     double laf_coef, int degen_check, const uint64_t* seeds,
                                     double* F_out, uint8_t* mask_out, int32_t* stats_out, unsigned flags);
int dgb200_find_homography_batch_ex(const double* x1y1, const double* x2y2, int n_pairs, int n, int dim,
                                    double px_th, double conf, int max_iters, int error_type, int sym_check,
                                    double laf_coef, const uint64_t* seeds,
                                    double* H_out, uint8_t* mask_out, int32_t* stats_out, unsigned flags);
int dgb200_find_fundamental_batch_dev_ex(const double* d_x1y1, const double* d_x2y2, int n_pairs, int n, int dim,
                                         double px_th, double conf, int max_iters, int error_type, int sym_check,
                                         double laf_coef, int degen_check, const uint64_t* d_seeds,
                                         double* d_F_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream,
                                         unsigned flags);
int dgb200_find_homography_batch_dev_ex(const double* d_x1y1, const double* d_x2y2, int n_pairs, int n, int dim,
                                        double px_th, double conf, int max_iters, int error_type, int sym_check,
                                        double laf_coef, const uint64_t* d_seeds,
                                        double* d_H_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream,
                                        unsigned flags);

/* Ragged batches (SURVEY.md section 8(b), proposal 3): real tentative sets never share n.  The correspondences of all
 * pairs are concatenated ([offsets[n_pairs]][dim] float64); pair p owns rows offsets[p] .. offsets[p+1]-1
 * (offsets[0] = 0, int32, every pair n >= 8 for F / n >= 4 for H); mask_out is concatenated the same way
 * ([offsets[n_pairs]] uint8); models and stats stay [n_pairs][9] / [n_pairs][4].  Same kernel, same results as one
 * call per pair.  HOST buffers; synchronous. */
int dgb200_find_fundamental_ragged(const double* x1y1, const double* x2y2, const int32_t* offsets, int n_pairs, int dim,
                                   double px_th, double conf, int max_iters, int error_type, int sym_check,
                                   double laf_coef, int degen_check, const uint64_t* seeds,
                                   double* F_out, uint8_t* mask_out, int32_t* stats_out);
int dgb200_find_homography_ragged(const double* x1y1, const double* x2y2, const int32_t* offsets, int n_pairs, int dim,
                                  double px_th, double conf, int max_iters, int error_type, int sym_check,
                                  double laf_coef, const uint64_t* seeds,
                                  double* H_out, uint8_t* mask_out, int32_t* stats_out);
/* DEVICE-pointer flavour of the ragged batches (d_offsets in device memory; n_max = the largest pair, it sizes the
 * per-CTA scratch).  Asynchronous on `stream`.  The device offsets are not read on the host (they may come from
 * dgb200_match_descriptors_batch_dev), so the kernel guards every pair once: a pair with fewer than 8 (F) / 4 (H) rows,
 * or more than n_max rows, is not run -- all-zero model, zero stats, its mask rows left as the caller initialised them
 * (zero them first), no access past the pair's rows.  Offsets must start at 0 and stay within the arrays.  n_max itself
 * must be >= 8 (F) / >= 4 (H). */
int dgb200_find_fundamental_ragged_dev(const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets, int n_pairs,
                                       int n_max, int dim, double px_th, double conf, int max_iters, int error_type,
                                       int sym_check, double laf_coef, int degen_check, const uint64_t* d_seeds,
                                       double* d_F_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream);
int dgb200_find_homography_ragged_dev(const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets, int n_pairs,
                                      int n_max, int dim, double px_th, double conf, int max_iters, int error_type,
                                      int sym_check, double laf_coef, const uint64_t* d_seeds,
                                      double* d_H_out, uint8_t* d_mask_out, int32_t* d_stats_out, void* stream);

/* Homography from correspondences of local ELLIPTICAL features: the reference's ransacH2el (ranH2el.c:19-208; no binding
 * in the reference -- the solver its C core carries for two-correspondence samples).  u10: [n_pairs][n][10] rows
 * (x', y', a', b', c', x, y, a, b, c) as ranH2el.h:4 (image 1 first; each local frame the lower-triangular affinity
 * [a 0; b c] at (x, y)).  th = px_th^2 on the Sampson error of the centres, do_lo = 1, inlLimit = 0.  H_out: RAW core
 * output like dgb200_find_homography (column-major; inv(H^T) maps (x', y') -> (x, y)).  stats: {samples, LO runs, 0,
 * inliers of the returned model}. */
int dgb200_find_homography_2el_batch(const double* u10, int n_pairs, int n, double px_th, double conf, int max_iters,
                                     const uint64_t* seeds, double* H_out, uint8_t* mask_out, int32_t* stats_out);
int dgb200_find_homography_2el_batch_dev(const double* d_u10, int n_pairs, int n, double px_th, double conf,
                                         int max_iters, const uint64_t* d_seeds, double* d_H_out, uint8_t* d_mask_out,
                                         int32_t* d_stats_out, void* stream);

/* One pair (what one findFundamentalMatrix_/findHomography_ call does): batch of 1 with one seed. */
int dgb200_find_fundamental(const double* x1y1, const double* x2y2, int n, int dim, double px_th, double conf,
                            int max_iters, int error_type, int sym_check, double laf_coef, int degen_check,
                            uint64_t seed, double* F_out, uint8_t* mask_out, int32_t* stats_out);
int dgb200_find_homography(const double* x1y1, const double* x2y2, int n, int dim, double px_th, double conf,
                           int max_iters, int error_type, int sym_check, double laf_coef,
                           uint64_t seed, double* H_out, uint8_t* mask_out, int32_t* stats_out);

/* ---- the steps either side of the path (SURVEY.md section 8(f).3 / 8(f).4), device-resident, asynchronous on `stream` ----
 *
 * Descriptor matching: replaces the host side of the reference's pipeline, cv2.BFMatcher().knnMatch(descs1, descs2, k=2)
 * + SNN ratio test `m.distance < ratio * n.distance` (examples/simple-example.py:46-53), optionally with a mutual
 * nearest-neighbour check.  d_desc1 [n1][D], d_desc2 [n2][D] float32 (D a multiple of 4, <= 256); accepted matches in
 * ascending query order: d_match_q/d_match_t [capacity] int32, *d_count; when d_x1y1 != NULL the first `out_dim`
 * columns of the keypoint rows d_kp1 [n1][kp_dim], d_kp2 [n2][kp_dim] (float64) are gathered into d_x1y1/d_x2y2
 * [capacity][out_dim] -- exactly the arrays dgb200_find_*_batch_dev take.  d_workspace: dgb200_match_workspace_bytes(). */
size_t dgb200_match_workspace_bytes(int n1, int n2);
int dgb200_match_descriptors_dev(const float* d_desc1, int n1, const float* d_desc2, int n2, int D, float ratio, int mutual,
                                 const double* d_kp1, const double* d_kp2, int kp_dim, int* d_match_q, int* d_match_t,
                                 double* d_x1y1, double* d_x2y2, int out_dim, int capacity, int* d_count, void* d_workspace,
                                 void* stream);
/* Descriptor matching of MANY image pairs in one call: the matcher above over a batch, with its output in the ragged
 * layout that dgb200_find_*_ragged_dev take.
 *   d_bank [R][D] float32: the descriptors of n_images images concatenated; image i owns rows
 *          img_offsets[i] .. img_offsets[i+1]-1 (img_offsets: HOST int32 [n_images+1], starting at 0, non-decreasing).
 *          Any 4-byte alignment (a 16-byte aligned bank is staged with bulk async copies).
 *   pairs  HOST int32 [n_pairs][2] = (query image, train image); an image may appear in many pairs, on either side.
 *   d_kp_bank [R][kp_dim] float64 or NULL: keypoint rows of the same images, gathered like dgb200_match_descriptors_dev.
 * Output: pair p's matches, in ascending query order, are rows d_offsets_out[p] .. d_offsets_out[p+1]-1 of d_match_q,
 * d_match_t (int32, indices local to each image) and, when d_x1y1 != NULL, of d_x1y1 / d_x2y2 [capacity][out_dim];
 * d_offsets_out: DEVICE int32 [n_pairs+1], d_offsets_out[0] = 0.  capacity must be >= the sum over the pairs of the
 * query image's descriptor count (every match of a pair is a distinct query); rows past d_offsets_out[n_pairs] are
 * left unwritten.  A pair whose query image has no descriptors, or whose train image has fewer than 2, gets zero
 * matches.  Malformed metadata (an image index out of range, decreasing offsets, D not a multiple of 4 in [4, 256],
 * capacity too small) returns DGB200_E_ARG before anything is launched.  The image offsets and pair table are read on
 * the host and copied (with the per-pair work layout derived from them) into d_workspace, sized by
 * dgb200_match_batch_workspace_bytes() (0: malformed metadata).  Asynchronous on `stream`, no synchronisation; the
 * host arrays may be freed on return.  Re-entrant: calls with distinct workspaces may run on different streams. */
size_t dgb200_match_batch_workspace_bytes(const int32_t* img_offsets, int n_images, const int32_t* pairs, int n_pairs);
int dgb200_match_descriptors_batch_dev(const float* d_bank, const int32_t* img_offsets, int n_images, int D,
                                       const int32_t* pairs, int n_pairs, float ratio, int mutual, const double* d_kp_bank,
                                       int kp_dim, int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2,
                                       int out_dim, int capacity, int32_t* d_offsets_out, void* d_workspace,
                                       void* stream);
/* Binary descriptors (ORB, AKAZE/MLDB, BRISK, FREAK) by Hamming distance: what cv2.BFMatcher(cv2.NORM_HAMMING)
 * .knnMatch(k=2) + `m.distance < ratio * n.distance` computes.  Each descriptor is a row of n_words 32-bit words
 * (n_words a multiple of 4 in [4, 64]: up to 2048 bits; zero-pad shorter codes, which changes no distance); the distance
 * is the number of differing bits.  Ties at the nearest distance go to the lowest train index, and d2 is the
 * second-smallest distance of the multiset, so two trains tied at the minimum give d2 == d1.  A query is accepted when
 * (double)d1 < ratio * (double)d2 (never on a tie when ratio <= 1); the mutual check is the float matcher's.  Every
 * other argument, the output and the errors are those of the float twin above (malformed input, including n_words
 * outside the allowed set, returns DGB200_E_ARG before any launch).  The workspace does not depend on the descriptor
 * type: dgb200_match_workspace_bytes / dgb200_match_batch_workspace_bytes size it. */
int dgb200_match_binary_descriptors_dev(const uint32_t* d_desc1, int n1, const uint32_t* d_desc2, int n2, int n_words,
                                        double ratio, int mutual, const double* d_kp1, const double* d_kp2, int kp_dim,
                                        int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim,
                                        int capacity, int* d_count, void* d_workspace, void* stream);
int dgb200_match_binary_descriptors_batch_dev(const uint32_t* d_bank, const int32_t* img_offsets, int n_images,
                                              int n_words, const int32_t* pairs, int n_pairs, double ratio, int mutual,
                                              const double* d_kp_bank, int kp_dim, int* d_match_q, int* d_match_t,
                                              double* d_x1y1, double* d_x2y2, int out_dim, int capacity,
                                              int32_t* d_offsets_out, void* d_workspace, void* stream);
/* Guided matching: the batch matchers above with each pair's candidates restricted by a model of the pair, as after a
 * first RANSAC pass (COLMAP's guided matching).  For pair p = (query image q, train image t), d_models + 9 p holds
 * M_p (float64, row-major) and th = px_th * px_th (FP64).  With (xq, yq) = columns 0-1 of q's keypoint row i and
 * (xt, yt) those of t's row j, train descriptor j is a CANDIDATE of query i when
 *   guide = DGB200_GUIDE_F (x_t^T F x_q = 0, what dgb200_find_fundamental_* return): the engine's Sampson residual,
 *     with rxc = (F0 xt + F3 yt) + F6, ryc = (F1 xt + F4 yt) + F7, rwc = (F2 xt + F5 yt) + F8,
 *     rx = (F0 xq + F1 yq) + F2, ry = (F3 xq + F4 yq) + F5, r = (xq rxc + yq ryc) + rwc:
 *     (r r) / (((rxc rxc + ryc ryc) + rx rx) + ry ry) <= th -- the rule that makes a correspondence an inlier of the
 *     RANSAC mask at the same px_th;
 *   guide = DGB200_GUIDE_H (x_t ~ H x_q, OpenCV convention, what dgb200_find_homography_* return):
 *     w = (H6 xq + H7 yq) + H8, px = ((H0 xq + H1 yq) + H2) / w, py = ((H3 xq + H4 yq) + H5) / w,
 *     dx = xt - px, dy = yt - py:  dx dx + dy dy <= th.
 * Every operation is an IEEE double operation in the order written (no fused multiply-add).  A comparison that is not
 * true fails, so an all-zero model (what the RANSAC returns when it finds none), a model with a NaN, or w = 0 with a
 * finite px_th admits no candidate: such a pair gets ZERO matches.  Among its candidates each query keeps the two
 * nearest train descriptors under the matcher's distance (squared L2 in FP32, or Hamming), ties to the lowest train
 * index, d2 = +inf with fewer than two candidates; the ratio test and mutual check are the batch matcher's, so a query
 * with exactly one candidate passes the ratio test for any ratio > 0, and with `mutual` a train's nearest query is taken
 * over the queries whose gate admits it.  Output, ordering, the degenerate-pair rule, capacity, workspace
 * (dgb200_match_batch_workspace_bytes) and errors are those of the batch matchers; in addition a null d_models, a null
 * d_kp_bank or kp_dim < 2 (the gate needs the coordinates even when d_x1y1 is NULL), a guide other than the two below,
 * or a negative or NaN px_th returns DGB200_E_ARG before any launch.  One pair is a batch of one pair over two images. */
#define DGB200_GUIDE_F 0
#define DGB200_GUIDE_H 1
int dgb200_match_descriptors_guided_batch_dev(const float* d_bank, const int32_t* img_offsets, int n_images, int D,
                                              const int32_t* pairs, int n_pairs, const double* d_models, int guide,
                                              double px_th, float ratio, int mutual, const double* d_kp_bank, int kp_dim,
                                              int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2,
                                              int out_dim, int capacity, int32_t* d_offsets_out, void* d_workspace,
                                              void* stream);
int dgb200_match_binary_descriptors_guided_batch_dev(const uint32_t* d_bank, const int32_t* img_offsets, int n_images,
                                                     int n_words, const int32_t* pairs, int n_pairs,
                                                     const double* d_models, int guide, double px_th, double ratio,
                                                     int mutual, const double* d_kp_bank, int kp_dim, int* d_match_q,
                                                     int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim,
                                                     int capacity, int32_t* d_offsets_out, void* d_workspace,
                                                     void* stream);
/* Pose from fundamental matrices: E = K2^T F K1, the four (R, t) candidates of its SVD, cheirality vote over the
 * correspondences with mask != 0 (NULL: all).  d_K1/d_K2: one 3x3 (k_per_pair = 0) or one per pair, row-major.
 * Outputs R [n_pairs][9] row-major, t [n_pairs][3] (unit length, x2 ~ R x1 + t), good [n_pairs] = supporters or NULL.
 * (The reference stops at F; this is the survey's "step after".) */
int dgb200_pose_from_fundamental_batch_dev(const double* d_F, const double* d_K1, const double* d_K2, int k_per_pair,
                                           const double* d_x1y1, const double* d_x2y2, const uint8_t* d_mask, int n_pairs,
                                           int n, int dim, double* d_R_out, double* d_t_out, int32_t* d_good_out,
                                           void* stream);
/* Pose from F over a RAGGED batch, as dgb200_find_fundamental_ragged_dev leaves it: pair p owns rows
 * d_offsets[p] .. d_offsets[p+1]-1 (DEVICE int32 [n_pairs+1], read on the device only) of d_x1y1 / d_x2y2
 * [rows][dim] float64 and d_mask [rows] (NULL: every row).  d_F [n_pairs][9] row-major (x2^T F x1 = 0), K as above.
 * Per pair, the candidates, the vote and the tie rule of the dense entry point, so R, t, good equal a dense call on
 * the pair alone.  Per row r, with x1 = K1^-1 [p1; 1], x2 = K2^-1 [p2; 1] and (l1, l2) the least-squares depths of
 * l1 R x1 + t = l2 x2 under the chosen (R, t):
 *   d_points_out [rows][3]  midpoint 0.5 (l1 x1 + R^T (l2 x2 - t)): camera 1's frame, units of the baseline (|t| = 1);
 *   d_in_front_out [rows]   mask[r] && l1 > 0 && l2 > 0 (so good[p] is the pair's sum of it);
 *   d_angle_out [rows]      parallax angle atan2(|x1 x R^T x2|, x1 . R^T x2) in radians, in [0, pi].
 * d_median_angle_out [n_pairs]: the median of the angles of the pair's in-front rows (the mean of the two middle values
 * for an even count, as np.median), exact for any pair length; NaN when no row is in front.  A pair whose F is all zero
 * (no model) or holds a NaN gets R = t = 0, good = 0, NaN points and angles, in_front = 0 and a NaN median.  Offsets
 * that decrease, are negative or pass `rows` make an empty pair: no row is read or written.  d_mask and d_good_out may
 * be NULL; the row arrays may be NULL when rows = 0; every other buffer is required.  A null required buffer,
 * n_pairs < 1, rows < 0 or dim < 2 returns DGB200_E_ARG before any launch.  Asynchronous on `stream`, one kernel, no
 * workspace. */
int dgb200_pose_from_fundamental_ragged_dev(const double* d_F, const double* d_K1, const double* d_K2, int k_per_pair,
                                            const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets,
                                            int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                            double* d_R_out, double* d_t_out, int32_t* d_good_out,
                                            double* d_points_out, uint8_t* d_in_front_out, double* d_angle_out,
                                            double* d_median_angle_out, void* stream);
/* Pose and scene plane from homographies over a RAGGED batch laid out as above (d_offsets, d_x1y1 / d_x2y2, d_mask,
 * K), for planar scenes and pure rotations, where F is undetermined or does not exist.  d_H [n_pairs][9] row-major,
 * x2 ~ H x1 (OpenCV convention, what dgb200_find_homography_* return).  Per pair, in FP64:
 *   Hn = K2^-1 H K1 divided by its middle singular value, negated when det(Hn) < 0;
 *   max |(Hn^T Hn - I)_ij| < 1e-3: a PURE ROTATION, one candidate R = U V^T (the rotation nearest to Hn), t = 0;
 *   otherwise the four decompositions Hn = R + t' n^T, |n| = 1, of Malis & Vargas (INRIA RR-6303, the analytical
 *   method, as cv2.decomposeHomographyMat) in the order (Ra, t'a, na), (Ra, -t'a, -na), (Rb, t'b, nb), (Rb, -t'b, -nb).
 * Vote over the rows with mask != 0: a row supports (R, t'/|t'|) when the least-squares depths (l1, l2) of
 * l1 R x1 + t = l2 x2 are both positive (the arithmetic of the F entry points), the rotation when x1 . R^T x2 > 0.
 * Candidate 0 has the most votes, candidate 1 the most among the rest; equal votes go to the earlier candidate in the
 * order above.  Two views of a plane often leave two candidates with equal votes: candidate 1 is the one a caller with
 * a prior (the ground-plane normal, a third view) may prefer.  Outputs, for c = 0, 1:
 *   d_R_out [n_pairs][2][9]      row-major, det R = +1;
 *   d_t_out [n_pairs][2][3]      unit length, x2 ~ R x1 + t, in units of the baseline (the convention of
 *                                dgb200_pose_from_fundamental_ragged_dev: candidate 0 goes straight into
 *                                dgb200_refine_pose_ragged_dev);
 *   d_plane_out [n_pairs][2][4]  (n, d): the plane n^T X = d in camera 1's frame, baseline units, d = 1/|t'| > 0;
 *   d_good_out [n_pairs][2]      the votes;
 *   d_rotation_only_out [n_pairs] 1 for a pure rotation.
 * A pure rotation's candidate 0 has t = 0 and a NaN plane; its candidate 1 is R = t = 0, plane NaN, good 0.
 * Per row r under candidate 0, the definitions of dgb200_pose_from_fundamental_ragged_dev: d_points_out (midpoint),
 * d_in_front_out (mask && l1 > 0 && l2 > 0), d_angle_out (parallax), and d_median_angle_out per pair (exact median of
 * the in-front rows' angles, NaN when there is none).  A pure rotation's rows get NaN points and
 * in_front = mask && x1 . R^T x2 > 0; its angles and median are computed as usual (the median is the value that
 * COLMAP-style code compares with a threshold to call a pair panoramic).  A pair whose H is all zero (no model) or
 * holds a NaN gets R = t = 0 and NaN planes for both candidates, good 0, rotation_only 0, NaN points and angles,
 * in_front 0 and a NaN median.  Offsets that decrease, are negative or pass `rows` make an empty pair: no row is read or
 * written.  d_mask and d_good_out may be NULL; the row arrays may be NULL when rows = 0; every other buffer is required.
 * A null required buffer, n_pairs < 1, rows < 0 or dim < 2 returns DGB200_E_ARG before any launch.  Asynchronous on
 * `stream`, one kernel, no workspace; a pair's result does not depend on the batch it is in. */
int dgb200_pose_from_homography_ragged_dev(const double* d_H, const double* d_K1, const double* d_K2, int k_per_pair,
                                           const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets,
                                           int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                           double* d_R_out, double* d_t_out, double* d_plane_out, int32_t* d_good_out,
                                           uint8_t* d_rotation_only_out, double* d_points_out, uint8_t* d_in_front_out,
                                           double* d_angle_out, double* d_median_angle_out, void* stream);
/* Refinement of the relative pose on the inliers, over a RAGGED batch laid out as above (d_offsets, d_x1y1 / d_x2y2,
 * d_mask, K): per pair, Levenberg-Marquardt from (d_R [n_pairs][9] row-major, d_t [n_pairs][3] of unit length; what
 * dgb200_pose_from_fundamental_ragged_dev returns) on the cost C(R, t) = sum of r^2 over the rows with mask != 0, r the
 * pixel-domain Sampson residual of F = K2^-T [t]x R K1^-1, so r^2 is the residual of the RANSAC's inlier rule (px^2).
 * Five local parameters, re-centred at every accepted step: R <- exp([w]x) R, t <- (t + B d) / |t + B d| with B an
 * orthonormal basis of the plane orthogonal to t; analytic Jacobian.  Schedule: lambda = 1e-3; a trial step solves
 * (J^T J + lambda diag(J^T J)) D = -J^T r (a pivot of the 5 x 5 Cholesky factor that is not positive rejects it) and is
 * accepted when its cost is strictly lower (lambda <- max(lambda / 10, 1e-12)), else lambda <- 10 lambda; stops after
 * max_iters trial steps, after a trial step, accepted or not, whose cost differs from the current one by less than
 * 1e-12 of it (converged), or when lambda > 1e8.
 * The sums of a pair are reduced in a fixed order without atomics: its result does not depend on the batch or the run.
 * Outputs per pair: d_R_out [9], d_t_out [3] (det R = +1, |t| = 1); d_F_out [9] = K2^-T [t]x R K1^-1 row-major, scaled
 * to unit Frobenius norm (x2^T F x1 = 0: the model dgb200_match_descriptors_guided_batch_dev takes); d_cost0_out,
 * d_cost_out the cost before and after (cost <= cost0); d_n_used_out the rows with mask != 0; d_iters_out the trial
 * steps taken.  d_inliers_out [rows], when given: f_resid_sampson(F, row) <= px_th^2 with the output F for EVERY row of
 * the pair, masked or not -- the comparison of the RANSAC's mask.
 * Pairs that are not refined: fewer than 6 rows with mask != 0: R, t copied, F built from them, cost0 = cost = their
 * cost, iters = 0.  R all zero, or a NaN in R or t (no model): R = t = F = 0, NaN costs, n_used = iters = 0, inlier rows
 * 0.  Offsets that decrease, are negative or pass `rows`: per-pair outputs as for no model, no row read or written.
 * d_mask, d_cost0_out, d_n_used_out, d_iters_out and d_inliers_out may be NULL; d_x1y1 / d_x2y2 may be NULL when
 * rows = 0; every other buffer is required.  d_R_out / d_t_out may be d_R / d_t (in place).  A null required buffer,
 * n_pairs < 1, rows < 0, dim < 2, max_iters < 0, or d_inliers_out with a negative or NaN px_th returns DGB200_E_ARG
 * before any launch.  Asynchronous on `stream`, one kernel, no workspace. */
int dgb200_refine_pose_ragged_dev(const double* d_R, const double* d_t, const double* d_K1, const double* d_K2,
                                  int k_per_pair, const double* d_x1y1, const double* d_x2y2,
                                  const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                  int max_iters, double px_th,
                                  double* d_R_out, double* d_t_out, double* d_F_out, double* d_cost0_out,
                                  double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                  uint8_t* d_inliers_out, void* stream);
/* Refinement of homographies on their inliers, over a RAGGED batch laid out as above (d_offsets, d_x1y1 / d_x2y2 with
 * only columns 0-1 used, d_mask): per pair, Levenberg-Marquardt from d_H [n_pairs][9] (row-major, x2 ~ H x1: what
 * dgb200_find_homography_* return) on the cost C = sum of h_resid_sampson(G, row) over the rows with mask != 0, where
 * G = H^-1 is the engine's image-2 -> image-1 model (column-major, csrc/hgeom.h).  The per-row value is the residual of
 * the H RANSAC's default inlier rule (px^2), so a refined inlier means what a RANSAC inlier means.
 *   Residuals for the Jacobian: with the algebraic pair e = (r1, r2) and JJ^T = [[A, B], [B, D]] of h_resid_sampson,
 *   z1 = r1 / sqrt(A), z2 = (r2 - (B / sqrt(A)) z1) / sqrt(D - B^2 / A), so |z|^2 = e^T (JJ^T)^-1 e; analytic Jacobian.
 *   Parameters: 8, re-centred at every accepted step, in Hartley-normalised coordinates.  T1, T2 move the masked rows
 *   of each image to their centroid and an RMS distance of sqrt(2); the normalised model M = T1 G T2^-1 / |.|_F moves
 *   as M <- (M + B d) / |M + B d|_F, B (9 x 8) the Householder basis of the plane orthogonal to M.  Residuals are
 *   evaluated in pixels through G = T1^-1 M T2: the normalisation changes the conditioning, not the cost.
 *   Schedule (that of dgb200_refine_pose_ragged_dev): lambda = 1e-3; a trial step solves (J^T J + lambda diag(J^T J))
 *   D = -J^T z (a pivot of the 8 x 8 Cholesky factor that is not positive rejects it) and is accepted when its cost is
 *   strictly lower (lambda <- max(lambda / 10, 1e-12)), else lambda <- 10 lambda; stops after max_iters trial steps,
 *   after a trial step whose cost differs from the current one by less than 1e-12 of it, or when lambda > 1e8.
 * The sums of a pair are reduced in a fixed order without atomics: its result does not depend on the batch or the run.
 * Outputs per pair: d_H_out [9] the refined H (x2 ~ H x1), unit Frobenius norm, det H > 0 (the input H so normalised
 * when no step was accepted); d_cost0_out, d_cost_out the cost before and after (cost <= cost0); d_n_used_out the rows
 * with mask != 0; d_iters_out the trial steps taken.  d_inliers_out [rows], when given: h_resid_sampson(H_out^-1, row)
 * <= px_th^2 for EVERY row of the pair, masked or not -- the comparison of the RANSAC's mask.
 * Pairs that are not refined: fewer than 5 rows with mask != 0: H passed through (normalised as above), cost0 = cost,
 * iters = 0.  H all zero, holding a NaN, or with an inverse that is not finite (no model): H = 0, NaN costs,
 * n_used = iters = 0, inlier rows 0.  Offsets that decrease, are negative or pass `rows`: per-pair outputs as for no
 * model, no row read or written.
 * d_mask, d_cost0_out, d_n_used_out, d_iters_out and d_inliers_out may be NULL; d_x1y1 / d_x2y2 may be NULL when
 * rows = 0; every other buffer is required.  d_H_out may be d_H (in place).  A null required buffer, n_pairs < 1,
 * rows < 0, dim < 2, max_iters < 0, or d_inliers_out with a negative or NaN px_th returns DGB200_E_ARG before any
 * launch.  Asynchronous on `stream`, one kernel, no workspace. */
int dgb200_refine_homography_ragged_dev(const double* d_H, const double* d_x1y1, const double* d_x2y2,
                                        const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                        int max_iters, double px_th, double* d_H_out, double* d_cost0_out,
                                        double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                        uint8_t* d_inliers_out, void* stream);
/* Refinement of fundamental matrices on their inliers, for pairs whose intrinsics are unknown, over a RAGGED batch laid
 * out as above (d_offsets, d_x1y1 / d_x2y2 with only columns 0-1 used, d_mask): per pair, Levenberg-Marquardt from
 * d_F [n_pairs][9] (row-major, x2^T F x1 = 0: what dgb200_find_fundamental_* return) on the cost C = sum of
 * f_resid_sampson(F, row) over the rows with mask != 0 -- the residual of the F RANSAC's default inlier rule (px^2), so
 * a refined inlier means what a RANSAC inlier means.  Gauss-Newton residual r = (p2^T F p1) / sqrt(s), r^2 the Sampson
 * error, independent of the scale of F; analytic Jacobian.
 *   Parameters: 7, re-centred at every accepted step, in Hartley-normalised coordinates, over the rank-2 matrices.
 *   T1, T2 move the masked rows of each image to their centroid and an RMS distance of sqrt(2); the normalised model is
 *   Fn = T2^-T F T1^-1 at unit Frobenius norm, starting from Fn0 = unit(rank2(T2^-T F_in T1^-1)) (F_in itself, up to
 *   rounding, when it has rank 2; a full-rank F_in is projected).  A step is Fn <- unit(rank2(Fn + B d)), rank2 the
 *   projection that zeroes the smallest singular value, and B (9 x 7) an orthonormal basis of the complement of vec(Fn)
 *   and vec(cof Fn) -- the tangent space of the unit-norm rank-2 matrices at Fn -- built by two Householder
 *   reflections, so it has no gauge direction and depends on Fn alone.  Residuals are evaluated in pixels through
 *   F = T2^T Fn T1: the normalisation changes the conditioning, not the cost.
 *   Schedule (that of dgb200_refine_pose_ragged_dev): lambda = 1e-3; a trial step solves (J^T J + lambda diag(J^T J))
 *   D = -J^T r (a pivot of the 7 x 7 Cholesky factor that is not positive rejects it) and is accepted when its cost is
 *   strictly lower (lambda <- max(lambda / 10, 1e-12)), else lambda <- 10 lambda; stops after max_iters trial steps,
 *   after a trial step whose cost differs from the current one by less than 1e-12 of it, or when lambda > 1e8.
 * The sums of a pair are reduced in a fixed order without atomics: its result does not depend on the batch or the run.
 * Outputs per pair: d_F_out [9] the refined F = T2^T Fn T1 (x2^T F x1 = 0, row-major), rank 2, unit Frobenius norm,
 * signed so that <F_out, F_in> >= 0 (the start point so mapped back when no step was accepted); d_cost0_out, d_cost_out
 * the cost at the start point and after (cost <= cost0); d_n_used_out the rows with mask != 0; d_iters_out the trial
 * steps taken.  d_inliers_out [rows], when given: f_resid_sampson(F_out, row) <= px_th^2 for EVERY row of the pair,
 * masked or not -- the comparison of the RANSAC's mask.
 * Pairs that are not refined: fewer than 8 rows with mask != 0: the start point passed through (as above), cost0 = cost,
 * iters = 0.  F all zero or holding a value that is not finite (no model): F = 0, NaN costs, n_used = iters = 0, inlier
 * rows 0.  Offsets that decrease, are negative or pass `rows`: per-pair outputs as for no model, no row read or written.
 * d_mask, d_cost0_out, d_n_used_out, d_iters_out and d_inliers_out may be NULL; d_x1y1 / d_x2y2 may be NULL when
 * rows = 0; every other buffer is required.  d_F_out may be d_F (in place).  A null required buffer, n_pairs < 1,
 * rows < 0, dim < 2, max_iters < 0, or d_inliers_out with a negative or NaN px_th returns DGB200_E_ARG before any
 * launch.  Asynchronous on `stream`, one kernel, no workspace. */
int dgb200_refine_fundamental_ragged_dev(const double* d_F, const double* d_x1y1, const double* d_x2y2,
                                         const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                         int max_iters, double px_th, double* d_F_out, double* d_cost0_out,
                                         double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                         uint8_t* d_inliers_out, void* stream);
/* Absolute pose (registering a view against known 3D points, as cv2.solvePnPRansac) over a RAGGED batch of 2D-3D
 * correspondences: pair p owns rows d_offsets[p] .. d_offsets[p+1]-1 of d_x [rows][2] (pixels in the view) and
 * d_X [rows][3] (world points); K [9] row-major, one for all pairs (k_per_pair = 0) or [n_pairs][9]; the pose found
 * maps x ~ K (R X + t), OpenCV's solvePnP convention.
 *   Usable rows: d_mask[r] != 0 (every row when d_mask is NULL) and five finite coordinates; n of them, listed in row
 *   order.  n < 4: no model.  Sampling and scoring see only the list.
 *   RANSAC: iteration k = 1, 2, ... draws the 3 list entries of the Philox stream's minimal sample of (d_seeds[p], k)
 *   (csrc/rng.h, as the F / H engines) and solves Lambda Twist P3P (Persson & Nordberg, ECCV 2018) in FP64 on the unit
 *   bearings normalize(K^-1 [x, y, 1]): 0 to 4 poses, each with positive depths for its three points; a degenerate
 *   sample gives none and still counts.  A pose's MSAC cost is C = sum over the usable rows of min(e^2, th^2), e^2 the
 *   squared pixel reprojection error and th = px_th; a row whose depth (R X + t)_z is not positive scores th^2.  A row
 *   is an inlier when its depth is positive and e^2 <= th^2.  The best pose is replaced only by a strictly lower cost
 *   (ties keep the earlier iteration and solution).  After iteration k, N_req = min(max_iters, ceil(log(1 - conf) /
 *   log1p(-w^3))), w = inliers(best) / n (max_iters when conf = 1 or there is no best yet, k when w = 1); iteration
 *   k + 1 runs only if k < N_req.  The kernel evaluates waves of iterations side by side and applies this rule in
 *   iteration order, so the result does not depend on the wave width.
 *   Local optimisation, when the best pose has at least 4 inliers and refine_iters > 0: up to 3 rounds of
 *   Levenberg-Marquardt on the inliers (two pixel residuals per row, 6 local parameters R <- exp([w]x) R, t <- t + d,
 *   analytic Jacobian; the schedule of dgb200_refine_pose_ragged_dev with at most refine_iters trial steps, R
 *   re-orthonormalised when an accepted step left |R R^T - I| above 1e-12), each followed by a re-selection of the
 *   inliers; it stops when the inlier set does not change (or has fewer than 4 rows).  Its pose replaces the RANSAC
 *   pose only when its MSAC cost is <= the RANSAC pose's.
 * The sums of a pair are reduced in a fixed order without atomics: its result does not depend on the batch or the run.
 * Outputs per pair: d_R_out [9], d_t_out [3] the pose; d_n_inliers_out its inliers; d_iters_out the RANSAC iterations
 * drawn; d_cost0_out the MSAC cost of the RANSAC pose and d_cost_out that of the output pose (cost <= cost0).
 * d_mask_out [rows]: 1 for the inliers of the output pose, 0 for every other row of the pair.
 * Pairs without a model (n < 4, or no sample gave a pose): R = t = 0, n_inliers = 0, iters the iterations drawn, NaN
 * costs, mask rows 0.  Offsets that decrease, are negative or pass `rows`: the same with iters = 0, no row read or
 * written.  d_mask may be NULL; d_x, d_X and d_mask_out may be NULL when rows = 0; every other buffer is required.
 * A null required buffer, n_pairs < 1, rows < 0, px_th not a positive finite number, conf outside (0, 1],
 * max_iters < 1 or refine_iters < 0 returns DGB200_E_ARG before any launch; the message is
 * dgb200_absolute_pose_last_error()'s.  Asynchronous on `stream`: one kernel and a stream-ordered workspace of 4 bytes
 * per row (cudaMallocAsync / cudaFreeAsync), nothing read back. */
int dgb200_find_absolute_pose_ragged_dev(const double* d_x, const double* d_X, const double* d_K, int k_per_pair,
                                         const int32_t* d_offsets, int n_pairs, int rows, const uint8_t* d_mask,
                                         double px_th, double conf, int max_iters, int refine_iters,
                                         const uint64_t* d_seeds, double* d_R_out, double* d_t_out,
                                         uint8_t* d_mask_out, int32_t* d_n_inliers_out, int32_t* d_iters_out,
                                         double* d_cost0_out, double* d_cost_out, void* stream);
const char* dgb200_absolute_pose_last_error(void);
/* Relative pose of calibrated image pairs (cv2.findEssentialMat for ragged batches): five-point MSAC-RANSAC with
 * local optimisation.  Pair p owns rows d_offsets[p] .. d_offsets[p+1]-1 of d_x1 / d_x2 [rows][2] (pixels in images 1
 * and 2, x2^T F x1 = 0); d_K1 / d_K2 [9] row-major, shared (k_per_pair = 0) or [n_pairs][9] (k_per_pair = 1);
 * d_seeds [n_pairs] the seeds of the pairs' Philox sample streams; d_mask [rows] or NULL (every row).
 *   usable rows: mask != 0 and four finite coordinates, in row order (n of them); n < 5: no model.
 *   iteration k = 1, 2, ...: minimal_sample<5>(seed, k, n) over the usable rows; the five-point solver (Nistér, in
 *   Stewénius' formulation: null space, ten cubic constraints, 10 x 20 elimination, Sturm-isolated real roots of the
 *   degree-10 polynomial refined by a fixed number of bisections, a few Gauss-Newton steps on the constraints) on
 *   K1^-1 [x1, 1] and K2^-1 [x2, 1] gives 0 to 10 essential matrices E (a degenerate sample gives none and still
 *   counts as an iteration).  Each is scored through F = K2^-T E K1^-1 at unit norm: MSAC cost sum min(e^2, px_th^2)
 *   over the usable rows, e^2 the Sampson error in pixels, inlier when e^2 < px_th^2 (the rule of the F RANSAC, so
 *   the two masks compare).  A strictly lower cost replaces the best model.  Iteration k + 1 runs while
 *   k < N_req = min(max_iters, ceil(log(1 - conf) / log1p(-w^5))), w = inliers / n of the best model (max_iters
 *   without a model or with conf = 1; k itself when w = 1).
 *   local optimisation, when refine_iters > 0 and the best model has at least 6 inliers: the start is one
 *   decomposition E ~ [t]x R (any of the four gives +-E, and the Sampson error ignores the sign); up to 3 rounds of
 *   Levenberg-Marquardt over (R, t), |t| = 1, on the inliers (the rows, solve and step of
 *   dgb200_refine_pose_ragged_dev, at most refine_iters trial steps, R re-orthonormalised when an accepted step left
 *   |R R^T - I| above 1e-12), each followed by a re-selection of the inliers under E = [t]x R; it stops when the
 *   inlier set does not change (or has fewer than 6 rows).  Its model replaces the RANSAC model only when its MSAC
 *   cost is <= the RANSAC model's.
 * The sums of a pair are reduced in a fixed order without atomics: its result does not depend on the batch or the run.
 * Outputs per pair: d_E_out [9] the essential matrix at unit norm; d_F_out [9] = K2^-T E K1^-1 at unit norm (what
 * dgb200_pose_from_fundamental_ragged_dev, dgb200_refine_pose_ragged_dev and guided matching take); d_n_inliers_out its
 * inliers; d_iters_out the RANSAC iterations drawn; d_cost0_out the MSAC cost of the RANSAC model and d_cost_out that
 * of the output model (cost <= cost0).  d_mask_out [rows]: 1 for the inliers of the output model, 0 for every other
 * row of the pair.  No R and t are returned: dgb200_pose_from_fundamental_ragged_dev makes the cheirality vote on F.
 * Pairs without a model (n < 5, or no sample gave a solution): E = F = 0, n_inliers = 0, iters the iterations drawn,
 * NaN costs, mask rows 0.  Offsets that decrease, are negative or pass `rows`: the same with iters = 0, no row read or
 * written.  d_mask may be NULL; d_x1, d_x2 and d_mask_out may be NULL when rows = 0; every other buffer is required.
 * A null required buffer, n_pairs < 1, rows < 0, px_th not a positive finite number, conf outside (0, 1],
 * max_iters < 1 or refine_iters < 0 returns DGB200_E_ARG before any launch; the message is
 * dgb200_essential_last_error()'s.  Asynchronous on `stream`: one kernel and a stream-ordered workspace of 4 bytes per
 * row (cudaMallocAsync / cudaFreeAsync), nothing read back. */
int dgb200_find_essential_ragged_dev(const double* d_x1, const double* d_x2, const double* d_K1, const double* d_K2,
                                     int k_per_pair, const int32_t* d_offsets, int n_pairs, int rows,
                                     const uint8_t* d_mask, double px_th, double conf, int max_iters, int refine_iters,
                                     const uint64_t* d_seeds, double* d_E_out, double* d_F_out, uint8_t* d_mask_out,
                                     int32_t* d_n_inliers_out, int32_t* d_iters_out, double* d_cost0_out,
                                     double* d_cost_out, void* stream);
const char* dgb200_essential_last_error(void);
/* Triangulation of tracks across registered views (the step after registering a view in an incremental
 * reconstruction) over a RAGGED batch of tracks: track j owns observations d_offsets[j] .. d_offsets[j+1]-1, each a
 * camera index d_cams [obs] and a pixel d_pts [obs][2].  Camera c has the pose d_R [n_cams][9] (row-major),
 * d_t [n_cams][3], world to camera, so that x ~ K (R X + t) (the convention of dgb200_find_absolute_pose_ragged_dev's
 * output), and K [9], one for all cameras (k_per_camera = 0) or [n_cams][9].  All arithmetic is FP64.
 *   Usable observations: d_mask[r] != 0 (every row when d_mask is NULL), 0 <= d_cams[r] < n_cams, two finite pixel
 *   coordinates, and a registered camera: the 12 entries of (R, t) finite and det R > 0.5 (this rejects the R = t = 0
 *   of a view that could not be registered).  n of them, listed in row order.  n < 2: no model.
 *   World rays: centre C = -R^T t and direction d = R^T normalize(K^-1 [x, y, 1]).
 *   Hypothesis of list entries (i, j): none when both come from one camera; otherwise b = d_i . d_j, w = C_i - C_j,
 *   none when b > cos(min_angle) or 1 - b^2 <= 0 (the triangulation-angle gate, which also rejects parallel rays);
 *   lambda_i = (b (d_j . w) - d_i . w) / (1 - b^2), lambda_j = (d_j . w - b (d_i . w)) / (1 - b^2), none unless both
 *   are > 0; X = ((C_i + lambda_i d_i) + (C_j + lambda_j d_j)) / 2, the midpoint of the common perpendicular (+, -, x,
 *   / and sqrt only, with dots summed left to right, so that every build gives the same bits).  A missing hypothesis
 *   still counts as an iteration.
 *   Iterations: M = n (n - 1) / 2 pairs and K_max = min(M, max_iters).  When M <= max_iters, iteration k = 1, 2, ...
 *   is the k-th pair (i < j) in lexicographic order, (0, 1), (0, 2), ..., (1, 2), ...: short tracks are enumerated
 *   exhaustively and deterministically.  Otherwise iteration k is (i, j) = the Philox stream's minimal sample of 2 of
 *   (d_seeds[j], k) (csrc/rng.h, as the F / H / P3P engines), in draw order.
 *   Score: the MSAC cost sum over the usable observations of min(e^2, th^2), e^2 the squared pixel reprojection error
 *   in the observation's camera and th = px_th; an observation with depth (R X + t)_z <= 0 scores th^2.  It is an
 *   inlier when its depth is > 0 and e^2 <= th^2.  The best point is replaced only by a strictly lower cost.  After
 *   iteration k, N_req = min(K_max, ceil(log(1 - conf) / log1p(-w^2))), w = inliers(best) / n (K_max when conf = 1 or
 *   there is no best yet, k when w = 1); iteration k + 1 runs only if k < N_req.  The kernel evaluates waves of 32
 *   iterations side by side and applies this rule in iteration order, so the result does not depend on the wave width.
 *   Local optimisation, when the best point has at least 2 inliers and refine_iters > 0: up to 3 rounds of
 *   Levenberg-Marquardt on the inliers' pixel residuals over X (X <- X + D, analytic Jacobian; the schedule of
 *   dgb200_refine_pose_ragged_dev with at most refine_iters trial steps), each followed by a re-selection of the
 *   inliers; it stops when the inlier set does not change (or has fewer than 2 rows).  Its point replaces the RANSAC
 *   point only when its MSAC cost is <= the RANSAC point's.
 * A track is one warp and its sums are reduced in a fixed order without atomics: its result does not depend on the
 * batch or the run.  Outputs per track: d_X_out [3] the point; d_n_inliers_out its inliers; d_iters_out the
 * hypotheses drawn or enumerated; d_cost0_out the MSAC cost of the RANSAC point and d_cost_out that of the output point
 * (cost <= cost0); d_angle_out the largest triangulation angle at X, atan2(|a x b|, a . b) with a = X - C_i and
 * b = X - C_j, over pairs of inliers from distinct cameras (0 without such a pair; the caller applies its threshold).
 * d_mask_out [obs]: 1 for the inliers of the output point, 0 for every other row of the track.
 * Tracks without a model (n < 2, or no hypothesis: one camera only, every angle too small, every pair behind a
 * centre): X = NaN, n_inliers = 0, iters the iterations run, NaN costs and angle, mask rows 0.  Offsets that decrease,
 * are negative or pass `obs`: the same with iters = 0, no row read or written.  d_mask may be NULL; d_cams, d_pts and
 * d_mask_out may be NULL when obs = 0; every other buffer is required.  A null required buffer, n_tracks < 1, obs < 0,
 * n_cams < 1, px_th not a positive finite number, min_angle outside [0, pi), conf outside (0, 1], max_iters < 1 or
 * refine_iters < 0 returns DGB200_E_ARG before any launch; the message is dgb200_triangulate_last_error()'s.
 * Asynchronous on `stream`: two kernels (the camera table, then the tracks) and a stream-ordered workspace of
 * 272 bytes per camera and 4 bytes per observation (cudaMallocAsync / cudaFreeAsync), nothing read back. */
int dgb200_triangulate_tracks_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                         const double* d_t, const double* d_K, int k_per_camera, int n_cams,
                                         const int32_t* d_offsets, int n_tracks, int obs, const uint8_t* d_mask,
                                         double px_th, double min_angle, double conf, int max_iters, int refine_iters,
                                         const uint64_t* d_seeds, double* d_X_out, uint8_t* d_mask_out,
                                         int32_t* d_n_inliers_out, int32_t* d_iters_out, double* d_cost0_out,
                                         double* d_cost_out, double* d_angle_out, void* stream);
const char* dgb200_triangulate_last_error(void);
/* Bundle adjustment of registered views and their tracks (the step after registering a view and triangulating its
 * tracks in an incremental reconstruction): Levenberg-Marquardt over the free cameras' poses and the tracks' points
 * jointly.  Tracks and cameras have the layout and convention of dgb200_triangulate_tracks_ragged_dev: track j owns
 * observations d_offsets[j] .. d_offsets[j+1]-1 (camera d_cams [obs], pixel d_pts [obs][2]), camera c has d_R [9],
 * d_t [3] with x ~ K (R X + t) and K [9] (k_per_camera as there); d_X [n_tracks][3] are the tracks' points (the output
 * of the triangulation).  All arithmetic is FP64; the intrinsics are held.
 *   Free and held cameras: h_free [n_free] is a HOST list of 0 to 64 distinct camera indices, copied into the kernels'
 *   parameter block; every other camera is held (its observations constrain the points, its pose does not move).
 *   Usable observations: d_mask[r] != 0 (every row when d_mask is NULL), 0 <= d_cams[r] < n_cams, a registered camera
 *   (the 12 entries of (R, t) finite and det R > 0.5), a finite pixel, a finite X of its track and depth (R X + t)_z > 0
 *   at the start.  A track is optimised when its usable observations come from at least 2 distinct cameras and V_p =
 *   sum w J_X^T J_X over them has a positive Cholesky factor at the start; its usable observations are then used.  Any
 *   other track's X is copied bit for bit and its observations are not used.  A free camera without a used observation
 *   is held and passed through.
 *   Scale gauge: scale_gauge = -1, or a camera g of h_free when a camera outside h_free exists.  With a = the lowest
 *   index outside h_free and c_a = -R_a^T t_a, translation coordinate argmax |t_g + R_g c_a| of g is held (the lower
 *   axis on ties; chosen on the device from the input poses): g's translation relative to a keeps its scale.
 *   Cost C = sum over the used observations of rho(e^2), e^2 the squared pixel reprojection error: rho(s) = s when
 *   loss_scale = 0, else the Cauchy loss sigma^2 log(1 + s / sigma^2) with sigma = loss_scale.  The normal equations
 *   use the IRLS weights w = rho'(e^2) at the linearisation point (no second-order correction).
 *   Parameters: per free camera 6, R <- exp([w]x) R, t <- t + d (the update of the P3P local optimisation), the held
 *   coordinate dropped; per optimised track 3, X <- X + D.  A trial R whose |R R^T - I| exceeds 1e-12 is
 *   re-orthonormalised before it is scored, so the output's cost is the cost reported.
 *   Trial step: U*_a = U_a + lambda diag U_a, V*_p = V_p + lambda diag V_p; the reduced camera system S dc = -(g_c -
 *   sum_p W_p V*_p^-1 g_p), S = U* - sum_p W_p V*_p^-1 W_p^T, is solved by a dense FP64 Cholesky (rows of held
 *   coordinates and of cameras without used observations replaced by identity rows with a zero right-hand side);
 *   dX_p = -V*_p^-1 (g_p + sum_i W_i^T dc_cam(i)).  A non-positive pivot of S or of any V*_p rejects the step, and a
 *   used observation with depth <= 0 at the trial point costs +inf.
 *   Schedule, that of dgb200_refine_pose_ragged_dev: lambda starts at 1e-3; a strictly lower cost accepts the step
 *   and sets lambda <- max(lambda / 10, 1e-12), otherwise lambda <- 10 lambda; it stops after max_iters trial steps,
 *   after a trial step that changes the cost by less than 1e-12 of it, or when lambda > 1e8.
 * Every sum is reduced in a fixed order without atomics: a rerun gives the same bytes.  Outputs: d_R_out [n_cams][9],
 * d_t_out [n_cams][3] (held cameras bit-identical to the input), d_X_out [n_tracks][3] (tracks that were not optimised
 * bit-identical), d_mask_out [obs]: 1 for a usable observation with depth > 0 and e^2 <= px_th^2 at the output, 0 for
 * every other row; d_cost0_out [1] and d_cost_out [1] the cost at the start and at the output (cost <= cost0);
 * d_iters_out [1] the trial steps taken; d_n_used_out [1] the used observations.  Output buffers may alias the
 * inputs.  A track with offsets that decrease, are negative or pass `obs` is not optimised and none of its rows is
 * read.  d_mask may be NULL; d_cams, d_pts and d_mask_out may be NULL when obs = 0.  A null required buffer,
 * n_tracks < 1, obs < 0, n_cams < 1, n_free outside [0, 64], a repeated or out-of-range index in h_free, a scale_gauge
 * that is neither -1 nor in h_free (or with no camera outside h_free), a loss_scale that is neither 0 nor a positive
 * finite number, max_iters < 0 or px_th not a positive finite number returns DGB200_E_ARG before any launch; the
 * message is dgb200_bundle_adjust_last_error()'s.  Asynchronous on `stream`: 6 kernels per trial step and 7 around
 * them, and a stream-ordered workspace (cudaMallocAsync / cudaFreeAsync) of 418 bytes per observation, 180 bytes per
 * track, 468 bytes per camera and 8 (6 n_free)^2 bytes for S; nothing read back. */
int dgb200_bundle_adjust_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R, const double* d_t,
                                    const double* d_K, int k_per_camera, int n_cams, const int32_t* d_offsets,
                                    int n_tracks, int obs, const double* d_X, const uint8_t* d_mask,
                                    const int32_t* h_free, int n_free, int scale_gauge, double loss_scale,
                                    int max_iters, double px_th, double* d_R_out, double* d_t_out, double* d_X_out,
                                    uint8_t* d_mask_out, double* d_cost0_out, double* d_cost_out,
                                    int32_t* d_iters_out, int32_t* d_n_used_out, void* stream);
const char* dgb200_bundle_adjust_last_error(void);
/* Bundle adjustment of any number of cameras (a global bundle adjustment of a whole reconstruction): the estimator of
 * dgb200_bundle_adjust_ragged_dev with the reduced camera system solved inexactly by preconditioned conjugate
 * gradients (PCG) on the Schur complement, which is never formed (Ceres' ITERATIVE_SCHUR with SCHUR_JACOBI).
 * Everything is as there -- the track layout and conventions, the usable and used observations and the optimised
 * tracks, the held and free cameras and scale_gauge with its device-chosen axis, the squared or Cauchy cost with IRLS
 * weights, the parameterisation and the re-orthonormalisation of a trial R, the damping U* = U + lambda diag U and
 * V* = V + lambda diag V, the back-substitution dX_p = -V*_p^-1 (g_p + sum_i W_i^T dc), the schedule, the output mask
 * and the rule that held cameras and tracks that are not optimised are bit-identical to the input -- except:
 *   Free cameras: h_free [n_free] is a HOST list of 0 to n_cams distinct camera indices, copied to the device.
 *   Reduced system: S dc = b with S and b as the dense entry point defines them; the held coordinate and the cameras
 *   without used observations are pinned to 0.  S p = U* p - sum_p W_p V*_p^-1 (W_p^T p) is computed matrix-free.
 *   Preconditioner: block-diagonal, M_a = U*_a - sum_{i in a} W_i V*_p(i)^-1 W_i^T (6 x 6) per active free camera,
 *   the held coordinate's row and column replaced by the identity's, each block Cholesky-factorised once per trial
 *   step.  A non-positive pivot of M or of any V*_p rejects the step (lambda <- 10 lambda).
 *   PCG: x0 = 0, r0 = b, z0 = M^-1 r0, p0 = z0, rho = r . z; b = 0 gives dc = 0.  Each iteration: q = S p, kappa =
 *   p . q; kappa <= 0 or not finite stops (and rejects the step when it is the first iteration); alpha = rho / kappa,
 *   x += alpha p, r -= alpha q; |r|_2 <= cg_tol |b|_2 or cg_max_iters iterations stop; else z = M^-1 r, rho' = r . z,
 *   p = z + (rho' / rho) p, rho = rho'.  dc = x.
 *   cg_max_iters >= 1, cg_tol >= 0 and finite.  d_cg_iters_out [1]: the products q = S p, summed over the trial steps.
 * Every sum is reduced in a fixed order without atomics, the dot products of PCG included, over partitions that do not
 * depend on the launch grid: a rerun gives the same bytes.  A null required buffer (d_cg_iters_out is one), n_free
 * outside [0, n_cams], cg_max_iters < 1 or cg_tol not a non-negative finite number, and every case the dense entry
 * point refuses, returns DGB200_E_ARG before any launch; the message is dgb200_bundle_adjust_pcg_last_error()'s.
 * Asynchronous on `stream`: a copy of h_free, per trial step 6 launches whatever cg_max_iters is (the PCG loop is one
 * cooperative launch sized by the occupancy API) and 10 around them, and a stream-ordered workspace (cudaMallocAsync /
 * cudaFreeAsync) of 426 bytes per observation, 204 bytes per track, 468 bytes per camera, 760 bytes per free camera
 * and 4 bytes per free camera and 4096 observations; nothing read back. */
int dgb200_bundle_adjust_pcg_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                        const double* d_t, const double* d_K, int k_per_camera, int n_cams,
                                        const int32_t* d_offsets, int n_tracks, int obs, const double* d_X,
                                        const uint8_t* d_mask, const int32_t* h_free, int n_free, int scale_gauge,
                                        double loss_scale, int max_iters, double px_th, int cg_max_iters,
                                        double cg_tol, double* d_R_out, double* d_t_out, double* d_X_out,
                                        uint8_t* d_mask_out, double* d_cost0_out, double* d_cost_out,
                                        int32_t* d_iters_out, int32_t* d_n_used_out, int32_t* d_cg_iters_out,
                                        void* stream);
const char* dgb200_bundle_adjust_pcg_last_error(void);
/* Bundle adjustment with intrinsics: the estimator of dgb200_bundle_adjust_pcg_ragged_dev over the free cameras' poses,
 * the free intrinsics groups' parameters and the tracks' points jointly, with the RADIAL camera model (COLMAP's):
 *   camera c of group g = d_groups[c], intrinsics k_g = d_intrinsics[g] = (f, cx, cy, k1, k2) float64 [n_groups][5]:
 *   p = R_c X + t_c, u = (p0 / p2, p1 / p2), s = u . u, pixel = f (1 + k1 s + k2 s^2) u + (cx, cy).
 *   One focal length (no fx != fy), no skew, no tangential terms.  With k1 = k2 = 0 this is the pinhole projection of
 *   the other entry points with K = [[f, 0, cx], [0, f, cy], [0, 0, 1]].
 * Everything is as in dgb200_bundle_adjust_pcg_ragged_dev (usable and used observations, optimised tracks, scale gauge,
 * loss, IRLS weights, LM schedule, PCG stopping rules, outputs, determinism, pass-through), except:
 *   Cameras: a camera whose group index lies outside [0, n_groups), or whose group's parameters are not all finite or
 *   have f <= 0, is treated as an unregistered camera: its observations are not usable.
 *   Free groups: h_free_groups [n_free_groups] is a HOST list of 0 to n_groups distinct group indices, copied to the
 *   device.  refine is a set of DGB200_REFINE_* bits: the coordinates of each free group that move, f (FOCAL), (cx, cy)
 *   (PRINCIPAL_POINT), (k1, k2) (DISTORTION); with refine = 0 no group is free.  The others are pinned.  A free group
 *   without a used observation is pinned whole and passed through.  Observations of held cameras constrain their
 *   group's intrinsics; their poses do not move.
 *   Reduced system: over [free poses (6 each); free groups' intrinsics (5 each)], pinned coordinates with identity rows
 *   and columns and a zero right-hand side.  With J_pose, J_intr, J_X the observations' Jacobians and w their IRLS
 *   weights, U = sum w J^T J over [pose; intrinsics] is not block-diagonal: camera a of group g adds the cross block
 *   E_a = sum_{i in a} w J_pose,i^T J_intr,i.  W_i = w [J_pose,i; J_intr,i]^T J_X,i.  U* = U + lambda diag U over every
 *   kept coordinate, the intrinsics included.  S p = U* p - sum_p W_p V*_p^-1 W_p^T p, matrix-free: per PCG iteration
 *   y_p = V*_p^-1 sum_i (W_pose,i^T p_cam(i) + W_intr,i^T p_grp(i)), q_a = U*_aa p_a + E_a p_g(a) - sum_{i in a}
 *   W_pose,i y, q_g = U*_gg p_g + sum_{a in g} E_a^T p_a - sum_{i in g} W_intr,i y.
 *   Preconditioner (Ceres' SCHUR_JACOBI): block-diagonal over the parameter blocks, the 6 x 6 pose block of the PCG
 *   entry point per free camera and M_g = U*_gg - sum_{i in g} W_intr,i V*^-1 W_intr,i^T (5 x 5, pinned rows and
 *   columns of the identity) per free group; the cross blocks are left out.
 *   Trial step: intrinsics k_g + dk_g for the active free groups; a trial f <= 0 costs +inf, so the step is rejected.
 *   Sums over a group, which may own every observation, are taken over a fixed partition of the group-major list of
 *   its used observations (a stable counting sort) into chunks of 256, each chunk's partial sum in a fixed tree over a
 *   warp and the chunks summed in order: no floating-point atomics, the same bytes for any grid.
 * Outputs: bundle_adjust_pcg's, and d_intrinsics_out [n_groups][5] (held groups and inactive free groups bit-identical
 * to the input); the mask is taken at the refined intrinsics.  Outputs may alias the inputs (R, t, X, intrinsics).
 * A null required buffer (d_groups, d_intrinsics and d_intrinsics_out are), n_groups < 1, n_free_groups outside
 * [0, n_groups], a null h_free_groups with n_free_groups > 0, a free group index out of range or repeated, refine with
 * a bit outside DGB200_REFINE_*, and every case dgb200_bundle_adjust_pcg_ragged_dev refuses, returns DGB200_E_ARG
 * before any launch (the shared checks first, in that entry point's order); the message is
 * dgb200_bundle_adjust_intrinsics_last_error()'s.  Asynchronous on `stream`: copies of h_free and h_free_groups, per
 * trial step at most 8 launches whatever cg_max_iters is (the PCG loop is one cooperative launch sized by the occupancy
 * API) and at most 27 copies, memsets and launches around them, and a stream-ordered workspace (cudaMallocAsync /
 * cudaFreeAsync) of 962 bytes per observation plus 356 per 256 observations, 204 bytes per track, 468 per camera, 84
 * per group, 760 per free camera, 920 per free group, and 4 per 4096 observations times the larger of the free camera
 * and free group counts; nothing is read back. */
#define DGB200_REFINE_FOCAL 1
#define DGB200_REFINE_PRINCIPAL_POINT 2
#define DGB200_REFINE_DISTORTION 4
int dgb200_bundle_adjust_intrinsics_ragged_dev(
    const int32_t* d_cams, const double* d_pts, const double* d_R, const double* d_t, const int32_t* d_groups,
    const double* d_intrinsics, int n_groups, int n_cams, const int32_t* d_offsets, int n_tracks, int obs,
    const double* d_X, const uint8_t* d_mask, const int32_t* h_free, int n_free, const int32_t* h_free_groups,
    int n_free_groups, int refine, int scale_gauge, double loss_scale, int max_iters, double px_th, int cg_max_iters,
    double cg_tol, double* d_R_out, double* d_t_out, double* d_X_out, double* d_intrinsics_out, uint8_t* d_mask_out,
    double* d_cost0_out, double* d_cost_out, int32_t* d_iters_out, int32_t* d_n_used_out, int32_t* d_cg_iters_out,
    void* stream);
const char* dgb200_bundle_adjust_intrinsics_last_error(void);
/* Undistortion through the RADIAL model: d_out [rows][2] float64 = the pinhole pixel f u + (cx, cy) of each raw pixel
 * d_pts [rows][2] of camera d_cams[r] (int32) in group d_groups[c] (int32 [n_cams]), intrinsics d_intrinsics
 * [n_groups][5] as above.  The pinhole pixels feed the entry points that take K = [[f, 0, cx], [0, f, cy], [0, 0, 1]].
 * One thread per row: the undistorted radius rho solves rho (1 + k1 rho^2 + k2 rho^4) = |pixel - c| / f by Newton's
 * method bracketed in [0, the first turning point of the distortion] (a step that leaves the bracket bisects it), at
 * most 50 steps, converged at a relative step of 1e-15.  NaN for a row whose camera or group index is out of range,
 * whose group's intrinsics are not finite or have f <= 0, whose pixel is not finite, whose radius lies at or beyond
 * the image of the turning point, or that does not converge.  A null d_groups or d_intrinsics, a null row buffer with
 * rows > 0, rows < 0, n_cams < 1 or n_groups < 1 returns DGB200_E_ARG (message: dgb200_undistort_last_error());
 * asynchronous on `stream`, one launch, no workspace. */
int dgb200_undistort_points_dev(const double* d_pts, const int32_t* d_cams, int rows, const int32_t* d_groups,
                                int n_cams, const double* d_intrinsics, int n_groups, double* d_out, void* stream);
const char* dgb200_undistort_last_error(void);
/* Tracks from verified pairwise matches (OpenMVG's TracksBuilder): the connected components of the graph whose nodes
 * are the keypoints of all images and whose edges are the verified matches, in the ragged track layout that
 * dgb200_triangulate_tracks_ragged_dev and dgb200_bundle_adjust_ragged_dev take.
 *   Nodes: keypoint k of image i is node g = img_offsets[i] + k; img_offsets [n_images + 1] is a HOST prefix sum of the
 *   images' keypoint counts (img_offsets[0] = 0, not decreasing), N = img_offsets[n_images] nodes.
 *   Edges: pairs [n_pairs][2] is a HOST table of (query image q, train image t), as dgb200_match_descriptors_batch_dev
 *   takes it, and pair p owns rows d_offsets[p] .. d_offsets[p+1]-1 of d_idx1 / d_idx2 (int32 [rows], keypoint
 *   indices local to q and t) and d_mask (uint8 [rows] or NULL: every row), what the batch matcher and the ragged
 *   RANSAC leave.  Pair p is well-formed when 0 <= d_offsets[p] <= d_offsets[p+1] <= rows; a pair that is not adds no
 *   edge and none of its rows is read.  Row r of a well-formed pair is the edge (img_offsets[q] + d_idx1[r],
 *   img_offsets[t] + d_idx2[r]) when d_mask[r] != 0 and both indices lie inside their images; any other row is
 *   ignored.  Self-pairs (q = t) and repeated pairs or rows are allowed.
 *   Tracks: the components of two or more nodes.  A component with two nodes of one image is conflicting and is
 *   dropped whole (OpenMVG's rule); a component that survives with fewer than min_length nodes is dropped.
 *   Order: tracks by their smallest node, the observations of a track by node, which is ascending image order.
 * Outputs, capacity-sized because the number of tracks T is data-dependent (T_cap = N / min_length, rounded down):
 * d_offsets_out int32 [T_cap + 1] (track j owns observations d_offsets_out[j] .. d_offsets_out[j+1]-1; the entries past
 * T repeat the observation count, so they are empty tracks); d_cams_out int32 [N] the image (camera) of each
 * observation and d_kp_out int32 [N] its keypoint index in that image; d_pts_out float64 [N][2] its pixel, copied from
 * d_kp [N][2] (the keypoints' x, y in node order), when both are given; d_track_of_out int32 [N] the track of every
 * node, or -1; d_stats_out int32 [4] = (tracks, observations, conflicting components, nodes in them).  Observation rows
 * past the last track's are written as cams = kp = -1 and pts = NaN, so every byte of the output is specified.
 * Determinism: the hooks of the union-find (csrc/tracks.h) leave each component's smallest node as its root whatever
 * their order; the sizes and conflict counts are integer sums; the slot an atomic cursor gives a node in its track is
 * undone by ranking the track's nodes.  So the output is a function of the edge set alone: permuting the pairs or the
 * rows within a pair, or swapping a pair's direction together with idx1 / idx2, gives the same bytes.
 * d_mask may be NULL; d_idx1 / d_idx2 may be NULL when rows = 0; d_cams_out, d_kp_out and d_track_of_out may be NULL
 * when N = 0.  A null required buffer, n_images < 1, n_pairs < 1, rows < 0, min_length < 2, img_offsets that do not
 * start at 0 or decrease, d_kp without d_pts_out (or the reverse), or a pair image index outside [0, n_images)
 * returns DGB200_E_ARG before any launch; the message is dgb200_tracks_last_error()'s.  Asynchronous on `stream`:
 * two copies of the host tables, 13 kernels and a stream-ordered workspace (cudaMallocAsync / cudaFreeAsync) of 22
 * bytes per node, 16 per pair and 4 per image; nothing is read back. */
int dgb200_build_tracks_ragged_dev(const int32_t* img_offsets, int n_images, const int32_t* pairs, int n_pairs,
                                   const int32_t* d_idx1, const int32_t* d_idx2, const int32_t* d_offsets, int rows,
                                   const uint8_t* d_mask, const double* d_kp, int min_length, int32_t* d_offsets_out,
                                   int32_t* d_cams_out, int32_t* d_kp_out, double* d_pts_out, int32_t* d_track_of_out,
                                   int32_t* d_stats_out, void* stream);
const char* dgb200_tracks_last_error(void);
/* View-graph calibration (GLOMAP's first step, before rotation averaging): each camera group's focal length from the
 * fundamental matrices of the verified pairs, and the pairs whose F does not agree with the result.
 *   Edges: h_pairs [n_pairs][2] is a HOST table of (i, j) over n_views views; d_F float64 [n_pairs][9] row-major with
 *   x_j^T F_e x_i = 0 (what dgb200_find_fundamental_batch returns for pts1 from view i and pts2 from view j, the
 *   convention of dgb200_pose_from_fundamental_ragged_dev); d_mask uint8 [n_pairs] or NULL (every edge).  d_groups
 *   int32 [n_views] the camera group g(v) of each view; d_intrinsics float64 [n_groups][5] each group's start (f0, cx,
 *   cy, k1, k2), the RADIAL row of dgb200_bundle_adjust_intrinsics_ragged_dev; K0 = [[f0, 0, cx], [0, f0, cy],
 *   [0, 0, 1]].  k1 and k2 play no part: F is taken as the pinhole F of the pixels given.
 *   1 Unknowns: theta_g per group, f_g = f0_g exp(theta_g); the principal point is held.
 *   2 Constants of an edge: G = K0_{g(j)}^T F_e K0_{g(i)} scaled to unit Frobenius norm, G = U S V^T by
 *     dg::svd3_onesided with s1 >= s2 >= s3, v1, v2 from V and u_k = G v_k / s_k.  With w(theta) = diag(e^{2 theta},
 *     e^{2 theta}, 1), the simplified Kruppa equations (Hartley, PAMI 1997) compare A = (s1^2 v1^T w_i v1, s1 s2 v1^T
 *     w_i v2, s2^2 v2^T w_i v2) and B = (u2^T w_j u2, -u1^T w_j u2, u1^T w_j u1); A_k = alpha_k e^{2 theta_i} + beta_k
 *     and B_k = gamma_k e^{2 theta_j} + delta_k, 12 constants per edge.
 *   3 Used edge: i != j, both views' groups in [0, n_groups), the mask set, F finite, both groups' intrinsics finite
 *     with f0 > 0, and s2 > 1e-6 s1.
 *   4 Residuals, both in [-1, 1] and unchanged when F is scaled: r1 = (A0 B2 - A2 B0) / (A0 B2 + A2 B0) and r2 =
 *     (A1 / sqrt(A0 A2) - B1 / sqrt(B0 B2)) / 2; both are 0 exactly when the Kruppa equations hold.  The sign of r2
 *     follows the singular vectors' signs; s_e = r1^2 + r2^2 and the steps do not.
 *   5 Cost sum_e rho(s_e), rho the Cauchy loss sig2 log(1 + s / sig2) with sig2 = loss_scale^2 and IRLS weight
 *     1 / (1 + s / sig2) (the bundle adjustments'); loss_scale = 0: the squared loss.
 *   6 Levenberg-Marquardt from theta = 0 with the schedule and stopping rules of dgb200_bundle_adjust_ragged_dev: each
 *     trial step solves (H + lambda diag H) x = -g, H = sum J_e^T w_e J_e and g = sum J_e^T w_e r_e, by Jacobi-
 *     preconditioned CG over the groups with the stopping rules of dgb200_bundle_adjust_pcg_ragged_dev (a first p . q
 *     that is not positive rejects the step).  An edge whose views share a group contributes one column, the sum of its
 *     two.  A group without a used edge is pinned at theta = 0.  A trial point where an edge's s is not finite costs
 *     +inf.
 * Outputs: d_intrinsics_out float64 [n_groups][5]: a group is refined when it has a used edge and 1 / max_ratio <= f
 * / f0 <= max_ratio, and then its row is the input's with f = f0 exp(theta); any other group's row is the input's, bit
 * for bit.  d_refined_out uint8 [n_groups]; d_error_out float64 [n_pairs] sqrt(s_e) at the output intrinsics (NaN for
 * an edge that is not used); d_inliers_out uint8 [n_pairs]: used with error <= max_error; d_cost0_out, d_cost_out
 * float64 [1] the cost at theta = 0 and at the last accepted step; d_iters_out (trial steps), d_n_used_out (used
 * edges), d_cg_iters_out (CG iterations, summed) int32 [1].
 * Determinism: no floating-point atomics; every sum has a fixed order that does not depend on the launch grid (a
 * group's list is summed in chunks of 256 entries, then the chunks in order), so a rerun gives the same bytes.  A null
 * required buffer (d_mask is not), n_views, n_pairs or n_groups < 1, a null h_pairs, a view index outside [0,
 * n_views), loss_scale or max_error not a non-negative finite number, max_ratio not a finite number >= 1, negative
 * max_iters, cg_max_iters < 1 or cg_tol not a non-negative finite number returns DGB200_E_ARG before any CUDA call;
 * the message is dgb200_view_graph_calibration_last_error()'s.  Asynchronous on `stream`: a copy of h_pairs, 9
 * launches, 6 per trial step whatever cg_max_iters is (the CG loop is one cooperative launch sized by the occupancy
 * API; every kernel returns at once once the call has stopped) and 2 for the outputs, with a stream-ordered workspace
 * (cudaMallocAsync / cudaFreeAsync); nothing is read back. */
int dgb200_calibrate_view_graph_dev(const int32_t* h_pairs, int n_pairs, int n_views, const double* d_F,
                                    const uint8_t* d_mask, const int32_t* d_groups, const double* d_intrinsics,
                                    int n_groups, double loss_scale, double max_error, double max_ratio, int max_iters,
                                    int cg_max_iters, double cg_tol, double* d_intrinsics_out, uint8_t* d_refined_out,
                                    double* d_error_out, uint8_t* d_inliers_out, double* d_cost0_out,
                                    double* d_cost_out, int32_t* d_iters_out, int32_t* d_n_used_out,
                                    int32_t* d_cg_iters_out, void* stream);
const char* dgb200_view_graph_calibration_last_error(void);
/* Rotation averaging over a view graph (the first step of global SfM, as GLOMAP's rotation averager): a world rotation
 * for every view from the relative rotations of its verified pairs.  Translations are neither used nor produced.
 *   Edges: h_pairs [n_pairs][2] is a HOST table of (i, j), as dgb200_match_descriptors_batch_dev takes it; d_R_rel
 *   float64 [n_pairs][9] row-major with x_j ~ R_e x_i, so R_e ~ R_j R_i^T (what dgb200_pose_from_fundamental_ragged_dev
 *   returns for the pair (q, t) = (i, j)); d_mask uint8 [n_pairs] or NULL (every edge); d_weights int32 [n_pairs] or
 *   NULL (all 0): each edge's priority in the spanning tree, such as the pose's count of points in front.
 *   1 Valid edge: i != j, the mask set, weight >= 0, R_e finite with det R_e > 0.5 (a failed pose's R = 0 drops out).
 *     A valid R_e whose largest |R R^T - I| entry exceeds 1e-12 is re-orthonormalised (Gram-Schmidt on the rows).
 *   2 Components: the connected components of the valid edges, each rooted at its smallest view.  A view without a
 *     valid edge gets R = NaN and component -1.
 *   3 Start: the maximum spanning forest under the strict order "e before f iff w_e > w_f, or w_e = w_f and e < f"
 *     (unique; Boruvka rounds on the key ((INT32_MAX - w) << 32) | e).  Each root gets R = I; along each tree edge the
 *     child's rotation is its parent's composed with the edge's, R_j = R_e R_i or R_i = R_e^T R_j.
 *   4 Residual of a valid edge: dR_e = R_j^T R_e R_i, r_e = log dR_e, theta_e = |r_e| in [0, pi]: with a = (dR32 -
 *     dR23, dR13 - dR31, dR21 - dR12), theta = atan2(|a|, tr dR - 1), r = theta / (2 sin theta) a, by its Taylor
 *     series below theta = 1e-4; within 1e-3 of pi the axis is the largest-diagonal column of (dR + dR^T) / 2 - cos
 *     theta I, normalised and signed as a.  Finite for every rotation.
 *   5 Linearisation: right perturbations R_v <- R_v exp([w_v]x) (w in the world frame) change r_e by -w_j + w_i to
 *     first order, so each iteration solves min sum_e w_e |w_j - w_i - r_e|^2 with w = 0 at every root: the weighted
 *     graph Laplacian (x) I_3 with each root's row and column replaced by the identity's and its right-hand side 0.
 *     The update R_v <- exp([R_v w_v]x) R_v is re-orthonormalised when it drifts more than 1e-12.
 *   6 Weights: phase 1 (L1, Weiszfeld) w_e = 1 / max(theta_e, 1e-3) for at most l1_iters iterations, then phase 2
 *     (Geman-McClure, rho = sigma^2 theta^2 / (sigma^2 + theta^2)) w_e = (sigma^2 / (sigma^2 + theta_e^2))^2 for at
 *     most max_iters.  A phase ends early once max_v |w_v| <= step_tol after that iteration's update.  With l1_iters =
 *     max_iters = 0 the output is the start.
 *   7 Solve: Jacobi-preconditioned CG over the 3 n_views unknowns (diagonal sum_{e in v} w_e, 1 on roots), with the
 *     stopping rules of dgb200_bundle_adjust_pcg_ragged_dev: x0 = 0; |r| <= cg_tol |b| or cg_max_iters iterations
 *     stop; kappa = p . q <= 0 or not finite stops, and on the first iteration the iteration makes no update and ends
 *     its phase.  S p is matrix-free over a view-major list of the valid edges (ascending edge order within a view).
 * Outputs: d_R_out float64 [n_views][9] world-to-camera (x ~ K (R X + t), the convention of
 * dgb200_find_absolute_pose_ragged_dev, triangulation and bundle adjustment); d_component_out int32 [n_views];
 * d_residual_out float64 [n_pairs] theta_e at the output (NaN for an edge that is not valid); d_iters_out int32 [2]
 * the iterations of each phase; d_cg_iters_out int32 [1] the products S p, summed over the iterations.
 * Determinism: no floating-point atomics; the dot products and per-view sums are taken over partitions that do not
 * depend on the launch grid, so a rerun gives the same bytes.  A null required buffer (d_mask and d_weights are not),
 * n_views < 1, n_pairs < 1, a null h_pairs, a view index outside [0, n_views), sigma not a positive finite number,
 * negative l1_iters or max_iters, step_tol or cg_tol not a non-negative finite number, or cg_max_iters < 1 returns
 * DGB200_E_ARG before any launch; the message is dgb200_rotation_averaging_last_error()'s.  Asynchronous on `stream`:
 * a copy of h_pairs, 5 launches, 3 per Boruvka round, one cooperative launch for the start, 4 per iteration whatever
 * cg_max_iters is (the CG loop is one cooperative launch sized by the occupancy API; every kernel returns at once once
 * the call has stopped) and 2 for the outputs, and a stream-ordered workspace (cudaMallocAsync / cudaFreeAsync) of 146
 * bytes per edge, 308 bytes per view and 4 bytes per view and 2048 edges; nothing is read back. */
int dgb200_average_rotations_dev(const int32_t* h_pairs, int n_pairs, int n_views, const double* d_R_rel,
                                 const uint8_t* d_mask, const int32_t* d_weights, double sigma, int l1_iters,
                                 int max_iters, double step_tol, int cg_max_iters, double cg_tol, double* d_R_out,
                                 int32_t* d_component_out, double* d_residual_out, int32_t* d_iters_out,
                                 int32_t* d_cg_iters_out, void* stream);
const char* dgb200_rotation_averaging_last_error(void);
/* Global positioning (the second step of global SfM, GLOMAP's global positioner with point-to-camera constraints): the
 * views' centres and the tracks' points from the views' rotations and the tracks' rays.  Translations are not taken.
 *   Layout: the tracks of dgb200_triangulate_tracks_ragged_dev (d_cams, d_pts, d_offsets [n_tracks + 1], d_mask or
 *   NULL; the padded output of dgb200_build_tracks_ragged_dev goes in as it is), world-to-camera rotations d_R
 *   [n_cams][9] (what dgb200_average_rotations_dev returns) and K [9] (k_per_camera as there).
 *   1 Registered view: R finite with det R > 0.5.  Usable observation: its mask set, its camera in range and registered,
 *     a finite pixel; its ray v = normalise(R^T K^-1 (x, y, 1)).  Used track: usable observations from at least 2
 *     distinct cameras; its usable observations are then used.  A track with offsets that decrease, are negative or
 *     pass `obs` is not used and none of its rows is read.
 *   2 Components: the connected components of the views over the used tracks; each component's smallest view is its
 *     anchor, whose centre is held at 0.  A view without a used observation is inactive: t = NaN, component -1.  The
 *     result is defined up to a similarity per component (the scale is free, as in GLOMAP).
 *   3 Unknowns: a centre c_i per active view that is not an anchor, a point X_j per used track and a scale d_o per used
 *     observation, d_o >= d_min = 1e-5.
 *   4 Cost C = sum_o rho(|r_o|^2), r_o = d_o (X_j - c_i) - v_o (BATA's pairwise direction error); rho(s) = s when
 *     loss_scale = 0, else the Huber loss of scale delta = loss_scale: s for s <= delta^2, 2 delta sqrt(s) - delta^2
 *     above.  The normal equations use the IRLS weights w = min(1, delta / |r|) at the linearisation point.
 *   5 Start: c_i and X_j uniform in [-init_scale, init_scale]^3, all d = 1, anchors at 0.  Coordinate k of view i is
 *     init_scale (2 u - 1), u = (o[k] + 1/2) 2^-32, o = Philox4x32-10 (csrc/rng.h) of counter (0, i, 0, 0) and key
 *     (seed low 32 bits, seed high 32 bits); track j's uses counter (0, j, 1, 0).
 *   6 Schedule, that of dgb200_bundle_adjust_ragged_dev: Levenberg-Marquardt with lambda from 1e-3, a strictly lower
 *     cost accepts and sets lambda <- max(lambda / 10, 1e-12), otherwise lambda <- 10 lambda; it stops after max_iters
 *     trial steps, a trial step that changes the cost by less than 1e-12 of it, or lambda > 1e8.  Marquardt damping
 *     lambda diag(J^T W J) over every coordinate, the scales included.
 *   7 Trial step by a nested Schur complement.  With a = X - c, u = a / |a|, s = w d^2 and P = I - u u^T / (1 +
 *     lambda), an observation's scale is eliminated (H_dd* = (1 + lambda) w |a|^2), which leaves m = s P in its
 *     centre's and its point's blocks (-m between them) and e = w d (r - u (u . r) / (1 + lambda)) in their gradients
 *     (-e at the centre, +e at the point).  Then each point: V*_j = sum m + lambda sum s I, g_j = sum e, t_j = V*_j^-1
 *     g_j.  The reduced system over the centres that move, S dc = b with S = U* - sum_j W_j V*_j^-1 W_j^T, U*_i = sum
 *     m + lambda sum s I, b_i = sum_{o in i} (e_o - m_o t_j), is solved by PCG with the stopping rules of
 *     dgb200_bundle_adjust_pcg_ragged_dev (x0 = 0; |r| <= cg_tol |b| or cg_max_iters iterations; kappa <= 0 or not
 *     finite stops, and on the first iteration rejects the step) and the block-Jacobi preconditioner M_i = S_ii = U*_i -
 *     sum_j W_ij V*_j^-1 W_ij, W_ij the sum of m over view i's observations of track j (3 x 3, Cholesky); anchors and
 *     inactive views get identity rows.  Back-substitution: dX_j = -t_j + V*_j^-1
 *     sum m dc_i, dd = -(a . r + d a . (dX - dc)) / ((1 + lambda) |a|^2), trial d <- max(d + dd, d_min).  A non-positive
 *     pivot of any V* or M rejects the step.  A used observation with |a| = 0 or not finite at the linearisation point
 *     rejects every step from it (lambda grows until the call stops); at a trial point it costs +inf.
 * Outputs: d_t_out [n_cams][3] = -R c, so that (R, t) goes straight into triangulation and bundle adjustment;
 * d_X_out [n_tracks][3] (NaN for a track that is not used); d_component_out int32 [n_cams] the anchor of each view's
 * component or -1; d_angle_out [obs] the angle between v_o and X_j - c_i at the output, atan2(|v x a|, v . a) (NaN for
 * an observation that is not used); d_inliers_out uint8 [obs]: used and angle <= max_angle; d_cost0_out [1],
 * d_cost_out [1] the cost at the start and at the output; d_iters_out [1] the trial steps; d_n_used_out [1] the used
 * observations; d_cg_iters_out [1] the products S p, summed over the trial steps.
 * Determinism: no floating-point atomics; every sum is taken in a fixed order over partitions that do not depend on the
 * launch grid, so a rerun gives the same bytes.  A null required buffer (d_angle_out and d_inliers_out are when obs >
 * 0), n_tracks < 1, obs < 0, n_cams < 1, loss_scale that is negative or not finite, max_iters < 0 (the shared checks of
 * the bundle adjustments, in their order), init_scale or max_angle not a non-negative finite number, cg_max_iters < 1
 * or cg_tol not a non-negative finite number returns DGB200_E_ARG before any launch; the message is
 * dgb200_global_positioning_last_error()'s.  Asynchronous on `stream`: 4 memsets and 10 launches before the trial
 * steps, 6 launches per trial step whatever cg_max_iters is (the PCG loop is one cooperative launch sized by the
 * occupancy API; every kernel returns at once once the call has stopped) and 3 for the outputs, and a stream-ordered
 * workspace (cudaMallocAsync / cudaFreeAsync) of 161 bytes per observation, 276 bytes per track, 628 bytes per view and
 * 4 bytes per view and 4096 observations; nothing is read back. */
int dgb200_global_positioning_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                         const double* d_K, int k_per_camera, int n_cams, const int32_t* d_offsets,
                                         int n_tracks, int obs, const uint8_t* d_mask, uint64_t seed,
                                         double init_scale, double loss_scale, int max_iters, double max_angle,
                                         int cg_max_iters, double cg_tol, double* d_t_out, double* d_X_out,
                                         int32_t* d_component_out, double* d_angle_out, uint8_t* d_inliers_out,
                                         double* d_cost0_out, double* d_cost_out, int32_t* d_iters_out,
                                         int32_t* d_n_used_out, int32_t* d_cg_iters_out, void* stream);
const char* dgb200_global_positioning_last_error(void);
/* The reference's alternative 7-point null-space solver nullspace_qr7x9 (Ftools.c:594-668, compile-time USE_QR,
 * exp_ranF.c:1346-1349) over `count` systems: d_A [count][7*9] row-major -> d_N [count][2*9], d_rc [count] or NULL. */
int dgb200_nullspace_qr7x9_batch_dev(const double* d_A, double* d_N, int32_t* d_rc, int count, void* stream);
/* Test hook: compares `count` random quotients of the shared-reciprocal division used by the homography Sampson residual
 * (csrc/hgeom.h: h_pinvJ) bit for bit with IEEE division on the device; *h_bad = number of mismatches (must be 0). */
int dgb200_debug_div_check(unsigned long long seed, long long count, unsigned long long* h_bad);
const char* dgb200_frontend_last_error(void);

/* Housekeeping */
int dgb200_version(void);              /* ABI version */
int dgb200_device_count(void);         /* CUDA devices visible (0 or <0: the engine cannot run) */
int dgb200_set_device(int device);     /* device used by subsequent calls of this thread's process */
const char* dgb200_last_error(void);   /* last error message of the calling thread (thread-local storage) */
long long dgb200_kernel_launches(void);/* RANSAC kernels launched so far by this process */
double dgb200_last_kernel_ms(void);    /* device time of the most recent HOST-buffer call's kernel (CUDA events) */
void dgb200_release(void);             /* free cached device buffers */

#ifdef __cplusplus
}
#endif
#endif /* DEGENSAC_B200_H */
