// adjust_host.h -- the launch plumbing that the adjustment entry points share (bundle_adjust.cu, bundle_adjust_pcg.cu,
// bundle_adjust_intrinsics.cu, rotation_averaging.cu, global_positioning.cu): the workspace carve, grid sizes, the
// launch chain and the grid of a cooperative launch.  Host code, in the anonymous namespace of the including
// translation unit.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace {

// Lays a workspace's buffers out one after another, each at a 256-byte boundary.  An entry point states its buffers
// once, as a function of a Carve: run from a null base it counts the bytes to allocate, then over the allocation it
// hands out the buffers.
struct Carve {
  char* base;
  size_t bytes = 0;
  template <typename T>
  T* take(size_t count) {
    T* out = base ? (T*)(base + bytes) : nullptr;
    bytes += (sizeof(T) * count + 255) / 256 * 256;
    return out;
  }
};

int blocks(size_t n, int per) { return (int)((n + per - 1) / per); }

// One step of an entry point's launch chain, over its local cudaError_t named launch: the step runs only while every
// step before it succeeded, and its error (a launch's included) is recorded
#define ADJ_LAUNCH(...)                           \
  if (launch == cudaSuccess) {                    \
    __VA_ARGS__;                                  \
    launch = cudaGetLastError();                  \
  }

// The set-up of a cooperative launch: *sms_out the device's SM count, once the device is known to support cooperative
// launches.  Returns nullptr, or the message of the failure with *e its CUDA error (cudaSuccess when there is none).
// The caller then asks the occupancy API itself how many CTAs of its kernel fit on an SM, so that a failure there
// names the kernel; the cooperative grid is that count times *sms_out.
inline const char* coop_sms(int* sms_out, cudaError_t* e) {
#define COOP_CU(call) \
  if ((*e = (call)) != cudaSuccess) return #call
  int dev = 0, sms = 0, coop = 0;
  COOP_CU(cudaGetDevice(&dev));
  COOP_CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  COOP_CU(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
#undef COOP_CU
  if (!coop) return "the device does not support cooperative launches";
  *sms_out = sms;
  return nullptr;
}

}  // namespace
