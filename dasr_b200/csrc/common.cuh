// Shared helpers for the dasr_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/dasr_b200.h"

namespace dasr {

void set_error(const char* fmt, ...);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return DASR_E_LAUNCH;
  }
  return DASR_OK;
}

#define DASR_REQUIRE(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::dasr::set_error(__VA_ARGS__);      \
      return DASR_E_BADARG;                \
    }                                      \
  } while (0)

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }
static inline bool aligned_to(const void* p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

int num_sms();
// programmatic dependent launch of the tensor-core conv kernels (DASR_B200_PDL=0 switches it off)
bool pdl_enabled();

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == DASR_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == DASR_ACT_RELU) return v > 0.f ? v : 0.f;
  return v;
}

__device__ __forceinline__ float bf2f(__nv_bfloat16 v) { return __bfloat162float(v); }

}  // namespace dasr
