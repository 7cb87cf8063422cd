// entry_error.h -- the error channel of the C entry points (host code; kept out of common.h, which the g++ host
// emulation compiles).  Each translation unit keeps its own thread-local message buffer, read by its own
// dgb200_*_last_error(), and defines in its anonymous namespace
//     thread_local char g_err[N] = "";
//     int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }
// CU(call) returns fail(DGB200_E_CUDA, "call: <CUDA error string>") from the entry point when the call fails.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"

// Writes "what: cudaGetErrorString(e)" (or "what" when e is cudaSuccess) to buf and returns code.
template <size_t N>
inline int set_error(char (&buf)[N], int code, const char* what, cudaError_t e) {
  if (e != cudaSuccess) snprintf(buf, N, "%s: %s", what, cudaGetErrorString(e));
  else snprintf(buf, N, "%s", what);
  return code;
}

#define CU(call)                                                     \
  do {                                                               \
    cudaError_t e__ = (call);                                        \
    if (e__ != cudaSuccess) return fail(DGB200_E_CUDA, #call, e__);  \
  } while (0)
