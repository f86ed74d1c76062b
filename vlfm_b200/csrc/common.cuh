// Shared helpers for the vlfm_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/vlfm_b200.h"

namespace vlfm {

void set_error(const char* fmt, ...);
void count_launch(unsigned n = 1);

inline int check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return VLFM_E_CUDA;
  }
  return VLFM_OK;
}

#define VLFM_CHECK_LAUNCH(what)                                   \
  do {                                                            \
    int _rc = ::vlfm::check_cuda(cudaGetLastError(), what);       \
    if (_rc != VLFM_OK) return _rc;                               \
  } while (0)

// Programmatic dependent launch (PDL): every kernel of the per-step sequence lets its successor start
// its prologue early (launch_dependents) and waits for its predecessors' memory before touching global
// memory (wait).  Hides launch latency + prologue of the ~400 small kernels of a batch-1 forward.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// "x2" operands (fp32-grade GEMMs on the fp16 tensor path): y = hi + lo / 2048 with hi = fp16(y), lo = fp16((y - hi) * 2048).
// The residual is scaled so that it stays a NORMAL fp16 number of y's magnitude (no subnormal precision loss).
constexpr float X2_SCALE = 2048.f;
__device__ __forceinline__ void split_x2(float y, __half& hi, __half& lo) {
  hi = __float2half_rn(y);
  lo = __float2half_rn((y - __half2float(hi)) * X2_SCALE);
}
__device__ __forceinline__ float ld_cg_f32(const float* p) { return __ldcg(p); }
__device__ __forceinline__ uint32_t ld_cg_u32(const uint32_t* p) { return __ldcg(p); }

}  // namespace vlfm
