// bundle_adjust_args.h -- the argument checks that the two bundle-adjustment entry points share
// (dgb200_bundle_adjust_ragged_dev in bundle_adjust.cu, dgb200_bundle_adjust_pcg_ragged_dev in bundle_adjust_pcg.cu).
// Host code.
#pragma once
#include <math.h>
#include <stdint.h>

#include <vector>

// The message of the first argument refused, in the order the dense entry point has always checked them, or nullptr.
// null_required / null_obs: a required buffer / an observation buffer (obs > 0) is null.  n_free must lie in
// [0, max_free] (n_free_range: the message otherwise).  On success *gauge_slot is the position of scale_gauge in h_free
// (-1: none) and *held_cam the lowest camera index outside h_free (-1: none).
inline const char* ba_arg_error(bool null_required, bool null_obs, int n_tracks, int obs, int n_cams,
                                const int32_t* h_free, int n_free, int max_free, const char* n_free_range,
                                int scale_gauge, double loss_scale, int max_iters, double px_th, int* gauge_slot,
                                int* held_cam) {
  if (null_required) return "null buffer";
  if (obs > 0 && null_obs) return "null observation buffer";
  if (n_tracks < 1 || obs < 0 || n_cams < 1) return "need n_tracks >= 1, obs >= 0 and n_cams >= 1";
  if (n_free < 0 || n_free > max_free) return n_free_range;
  if (n_free > 0 && !h_free) return "null free-camera list";
  std::vector<unsigned char> is_free((size_t)n_cams, 0);
  *gauge_slot = -1;
  for (int q = 0; q < n_free; ++q) {
    if (h_free[q] < 0 || h_free[q] >= n_cams) return "free camera index out of range";
    if (is_free[h_free[q]]) return "free camera index repeated";
    is_free[h_free[q]] = 1;
    if (h_free[q] == scale_gauge) *gauge_slot = q;
  }
  if (scale_gauge >= 0 && *gauge_slot < 0) return "scale_gauge must be one of the free cameras";
  if (scale_gauge < -1) return "scale_gauge must be a free camera or -1";
  *held_cam = -1;
  for (int c = 0; c < n_cams && *held_cam < 0; ++c)
    if (!is_free[c]) *held_cam = c;
  if (*gauge_slot >= 0 && *held_cam < 0) return "scale_gauge needs a held camera";
  if (!(loss_scale >= 0.0) || !(loss_scale < INFINITY))
    return "loss_scale must be a positive number (or 0 for the trivial loss)";
  if (max_iters < 0) return "max_iters must not be negative";
  if (!(px_th > 0.0) || !(px_th < INFINITY)) return "px_th must be a positive number";
  return nullptr;
}
