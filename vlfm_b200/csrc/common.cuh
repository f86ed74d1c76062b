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

// mbarriers in this CTA's shared memory (the wgmma GEMMs' TMA ring, the batch-1 attention's Q / K / V pieces)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spin = 0; !done; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (spin > (1u << 26)) __trap();  // a protocol bug must fail loudly, never hang the GPU
  }
}

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
// Partial sums of a split residual GEMM, written by the GEMM and added to the residual stream by the LayerNorm launch
// (layernorm_reduce_kernel).  Both sides take the layout from this struct, so they cannot disagree about it.
//   splits > 0: uniform split-K.  Split s stores element (row, col) at s * stride + row * D + col.
//   splits == 0: stream-K over 128 x 128 output tiles.  Tiles are ordered column block first (tile = n_blk * row_tiles + m_blk,
//     so the row tiles that read one weight tile run next to each other) and the (tile, K-block) iterations of all tiles form
//     one sequence, cut into `ctas` contiguous ranges of near-equal length.  CTA c stores the part of tile t it computed (a
//     "segment") in slab c + t: ranges grow monotonically in both c and t, so no two segments share a slab, and
//     ctas + tiles - 1 slabs hold them all.  A slab holds SK_SLAB_ROWS x SK_TILE floats: the tile's 128 rows, then the
//     tail rows (M = 128 q + r, r <= 2) that the last row tile computes on CUDA cores.
constexpr int SK_TILE = 128;
constexpr int SK_SLAB_ROWS = SK_TILE + 2;
constexpr long long SK_SLAB = (long long)SK_SLAB_ROWS * SK_TILE;   // floats
struct SplitK {
  int splits;
  long long stride;                  // uniform split-K: floats between splits
  int ctas, row_tiles, tiles, num_k;  // stream-K
  // first iteration of CTA c (c = ctas: one past the last)
  __host__ __device__ __forceinline__ int sk_begin(int c) const { return (int)((long long)c * tiles * num_k / ctas); }
  // the CTA whose range holds iteration it
  __host__ __device__ __forceinline__ int sk_owner(int it) const { return (int)(((long long)(it + 1) * ctas - 1) / ((long long)tiles * num_k)); }
};

// LayerNorm rows (vit_ops.cu): at most LN_DMAX columns (layernorm_kernel<12>: 12 float4 per lane; layernorm_reduce_kernel: one
// float4 per thread of at most 384).  layernorm_check: the argument checks of every LayerNorm entry point, resid-LN GEMMs included.
constexpr int LN_DMAX = 1536;
int layernorm_check(const char* who, const float* d_x, const float* d_gamma, const float* d_beta, const void* d_out16, const void* d_out16_lo,
                    const float* d_out32, int D, int ldx, int ldo16, int ldo32);

__device__ __forceinline__ float ld_cg_f32(const float* p) { return __ldcg(p); }
__device__ __forceinline__ uint32_t ld_cg_u32(const uint32_t* p) { return __ldcg(p); }

}  // namespace vlfm
