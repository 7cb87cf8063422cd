// device_util.h -- small device helpers of the ragged pose, registration, triangulation and bundle-adjustment
// kernels.  In the anonymous namespace of the including translation unit, as each kernel source keeps its own.
#pragma once
#include <cuda_runtime.h>

namespace {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000ll); }
__device__ __forceinline__ bool finite(double v) { return fabs(v) < INFINITY; }

// Butterfly sum over the 32 lanes of a full warp: every lane gets the same sum, in a fixed order
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

}  // namespace
