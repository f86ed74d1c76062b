// im2col of the convs that run on the wgmma GEMM (MobileSAM, PointNav, YOLOv7, the GroundingDINO neck): fp16 NHWC rows in, the
// GEMM's A operand out.  The layout is the contract of vlfm_im2col_f16 in include/vlfm_b200.h; vlm/dense.py::conv_rows lays the
// weights out to match.
#include <cuda_fp16.h>

#include "common.cuh"

namespace vlfm {

// One thread writes 8 columns of one row with one 16-byte store.  With VEC (C and ldx multiples of 8, x 16-byte aligned) the 8
// columns lie in one tap and are one 16-byte load; otherwise each column is gathered on its own, with its own tap.  The kernel
// size K is a template argument: with a run-time k, the tap arithmetic made the YOLOv7 convs' im2col measurably slower.
template <bool VEC, int K>
__device__ __forceinline__ void im2col_rows(const __half* __restrict__ x, int ldx, __half* __restrict__ col, int B, int H, int W,
                                            int C, int stride, int Ho, int Wo, int ldk) {
  const int c8 = ldk / 8;
  const long long total = (long long)B * Ho * Wo * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % c8);
    const long long r = i / c8;
    const int ox = (int)(r % Wo), oy = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    const __half* img = x + (size_t)b * H * W * ldx;
    const int col0 = q * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (VEC) {
      if (col0 < K * K * C) {
        const int tap = col0 / C, c = col0 - tap * C;
        const int iy = oy * stride - K / 2 + tap / K, ix = ox * stride - K / 2 + tap % K;
        if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W)
          v = *reinterpret_cast<const uint4*>(img + ((size_t)iy * W + ix) * ldx + c);
      }
    } else {
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cj = col0 + j;
        if (cj >= K * K * C) break;
        const int tap = cj / C, c = cj - tap * C;
        const int iy = oy * stride - K / 2 + tap / K, ix = ox * stride - K / 2 + tap % K;
        if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W)
          w[j / 2] |= (uint32_t)__half_as_ushort(img[((size_t)iy * W + ix) * ldx + c]) << (16 * (j & 1));
      }
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    *reinterpret_cast<uint4*>(col + r * ldk + col0) = v;
  }
}

__global__ void __launch_bounds__(256)
im2col_f16_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ col, int B, int H, int W, int C, int k, int stride,
                  int Ho, int Wo, int ldk, bool vec) {
  if (vec && k == 3) im2col_rows<true, 3>(x, ldx, col, B, H, W, C, stride, Ho, Wo, ldk);
  else if (vec) im2col_rows<true, 1>(x, ldx, col, B, H, W, C, stride, Ho, Wo, ldk);
  else if (k == 3) im2col_rows<false, 3>(x, ldx, col, B, H, W, C, stride, Ho, Wo, ldk);
  else im2col_rows<false, 1>(x, ldx, col, B, H, W, C, stride, Ho, Wo, ldk);
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_im2col_f16(const void* d_x16, int ldx, void* d_col16, int B, int H, int W, int C, int k, int stride, int ldk,
                               void* stream) {
  if (!d_x16 || !d_col16 || B < 1 || H < 1 || W < 1 || C < 1 || (k != 1 && k != 3) || (stride != 1 && stride != 2) || ldx < C ||
      ldk < k * k * C || (ldk & 7) || ((uintptr_t)d_col16 & 15)) {
    set_error("vlfm_im2col_f16: bad argument"); return VLFM_E_INVALID; }
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const bool vec = !(C & 7) && !(ldx & 7) && !((uintptr_t)d_x16 & 15);
  const long long blocks = ((long long)B * Ho * Wo * (ldk / 8) + 255) / 256;
  im2col_f16_kernel<<<(unsigned)(blocks < 132LL * 64 ? blocks : 132LL * 64), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_x16, ldx, (__half*)d_col16, B, H, W, C, k, stride, Ho, Wo, ldk, vec);
  VLFM_CHECK_LAUNCH("im2col_f16_kernel");
  count_launch();
  return VLFM_OK;
}
