// Non-GEMM operators of the GroundingDINO Swin-T backbone (sm_90a).
// Reference call site: vlfm/vlm/grounding_dino.py:52-67 (to_tensor + ImageNet normalise, no resize,
// then groundingdino's Swin-T backbone inside predict()).
//   - swin_patch_im2col_kernel: uint8 HWC -> (x/255 - mean)/std (float32) -> fp16 rows of the 4x4/4
//     patch-embedding GEMM (zero padding to a multiple of 4 AFTER normalisation, as the conv sees it);
//   - swin_window_attention_kernel: (shifted-)window multi-head attention, 7x7 windows, hd=32:
//     gathers q/k/v through the cyclic shift and the pad-to-7 (padded tokens are LayerNorm zeros, so
//     their q/k/v equal the projection bias), adds the relative-position bias and the shift mask
//     (-100 across regions), softmax, PV, scatters back (reverse shift + crop);
//   - swin_patch_merge_kernel: 2x2 neighbourhood gather [x00,x10,x01,x11] with zero padding.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace vlfm {

__global__ void swin_patch_im2col_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W,
                                         int Hp, int Wp, float m0, float m1, float m2, float s0, float s1, float s2) {
  // out [B*Hp*Wp, 48], col = c*16 + ky*4 + kx
  const size_t n = (size_t)B * Hp * Wp * 48;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int col = (int)(i % 48);
    const size_t r = i / 48;
    const int px = (int)(r % Wp), py = (int)((r / Wp) % Hp), b = (int)(r / ((size_t)Wp * Hp));
    const int c = col / 16, ky = (col % 16) / 4, kx = col % 4;
    const int y = py * 4 + ky, x = px * 4 + kx;
    float v = 0.f;
    if (y < H && x < W) {
      const float p = (float)img[(((size_t)b * H + y) * W + x) * 3 + c];
      const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
      v = __fdiv_rn(__fsub_rn(__fdiv_rn(p, 255.f), mean), sd);
    }
    out[i] = __float2half_rn(v);
  }
}

struct WinAttnArgs {
  const __half* qkv;      // [B*H*W, 3C]
  const float* qkv_bias;  // [3C]
  const float* rel_bias;  // [169, heads]
  __half* out;            // [B*H*W, C]
  int H, W, C, heads, shift;
};

constexpr int WS = 7, WT = 49, WHD = 32;
constexpr int WKS = WHD + 8;           // smem row stride (halves): conflict-free fragment loads, 16-byte aligned rows
constexpr int WIN_WARPS = 4;
constexpr int WIN_SMEM_WARP = 3 * 64 * WKS * 2 + 64 * 4 + 64;   // q, k, v tiles + source rows + regions

__device__ __forceinline__ void win_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t win_pack(float a, float b) { __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }

// One warp per (image, window, head).  The 49 window tokens (padded to 64 rows) are gathered through the cyclic shift into
// fp16 shared-memory tiles; S = Q K^T and O = P V run on mma.sync m16n8k16 (fp32 accumulate), relative-position bias,
// shift mask and softmax in registers, 16 query rows at a time.
__global__ void __launch_bounds__(32 * WIN_WARPS)
swin_window_attention_kernel(WinAttnArgs a, int B, int total) {
  extern __shared__ __align__(16) uint8_t win_smem[];
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int item = blockIdx.x * WIN_WARPS + warp;
  if (item >= total) return;
  uint8_t* base = win_smem + (size_t)warp * WIN_SMEM_WARP;
  __half* sQ = reinterpret_cast<__half*>(base);
  __half* sK = sQ + 64 * WKS;
  __half* sV = sK + 64 * WKS;
  int* srow = reinterpret_cast<int*>(sV + 64 * WKS);
  uint8_t* sreg = reinterpret_cast<uint8_t*>(srow + 64);
  const int Hp = (a.H + WS - 1) / WS * WS, Wp = (a.W + WS - 1) / WS * WS;
  const int nwx = Wp / WS, nw = nwx * (Hp / WS);
  const int head = item % a.heads, win = (item / a.heads) % nw, b = item / (a.heads * nw);
  const int wy = win / nwx, wx = win % nwx;
  for (int tk = lane; tk < 64; tk += 32) {
    int row = -2, reg = 0;
    if (tk < WT) {
      const int ty = tk / WS, tx = tk % WS;
      const int y = wy * WS + ty, x = wx * WS + tx;            // coordinates in the shifted, padded frame
      const int ys = (y + a.shift) % Hp, xs = (x + a.shift) % Wp;  // source token (torch.roll by -shift)
      row = (ys < a.H && xs < a.W) ? (b * a.H + ys) * a.W + xs : -1;
      if (a.shift > 0) {
        const int ry = y < Hp - WS ? 0 : (y < Hp - a.shift ? 1 : 2), rx = x < Wp - WS ? 0 : (x < Wp - a.shift ? 1 : 2);
        reg = ry * 3 + rx;
      }
    }
    srow[tk] = row; sreg[tk] = (uint8_t)reg;
  }
  __syncwarp();
  const int C = a.C;
  // gather: 64 rows x 3 matrices x 4 chunks of 16 bytes
  for (int i = lane; i < 64 * 12; i += 32) {
    const int tk = i / 12, rem = i - tk * 12, m = rem >> 2, c = rem & 3;
    const int row = srow[tk];
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (row >= 0) {
      val = __ldg(reinterpret_cast<const uint4*>(a.qkv + (size_t)row * 3 * C + (size_t)m * C + head * WHD + c * 8));
    } else if (row == -1) {   // padded token: LayerNorm output was padded with zeros -> projection = bias (rounded like the GEMM output)
      const float* bp = a.qkv_bias + (size_t)m * C + head * WHD + c * 8;
      val.x = win_pack(bp[0], bp[1]); val.y = win_pack(bp[2], bp[3]); val.z = win_pack(bp[4], bp[5]); val.w = win_pack(bp[6], bp[7]);
    }
    __half* dst = (m == 0 ? sQ : (m == 1 ? sK : sV)) + tk * WKS + c * 8;
    *reinterpret_cast<uint4*>(dst) = val;
  }
  __syncwarp();
  const float scale = 0.17677669529663687f;   // 1/sqrt(32)
  for (int mt = 0; mt < 4; ++mt) {
    const int r_lo = mt * 16 + g, r_hi = r_lo + 8;
    if (mt * 16 >= WT) break;
    uint32_t qa[2][4];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      qa[kk][0] = *reinterpret_cast<const uint32_t*>(sQ + r_lo * WKS + kk * 16 + 2 * t);
      qa[kk][1] = *reinterpret_cast<const uint32_t*>(sQ + r_hi * WKS + kk * 16 + 2 * t);
      qa[kk][2] = *reinterpret_cast<const uint32_t*>(sQ + r_lo * WKS + kk * 16 + 8 + 2 * t);
      qa[kk][3] = *reinterpret_cast<const uint32_t*>(sQ + r_hi * WKS + kk * 16 + 8 + 2 * t);
    }
    float sc[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) { sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f; }
#pragma unroll
    for (int n = 0; n < 7; ++n) {
      const __half* kr = sK + (n * 8 + g) * WKS + 2 * t;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk)
        win_mma(sc[n], qa[kk], *reinterpret_cast<const uint32_t*>(kr + kk * 16), *reinterpret_cast<const uint32_t*>(kr + kk * 16 + 8));
    }
    const int ylo = r_lo / WS, xlo = r_lo % WS, yhi = r_hi / WS, xhi = r_hi % WS;
    const int reg_lo = sreg[r_lo], reg_hi = sreg[r_hi];
    float m_lo = -INFINITY, m_hi = -INFINITY;
#pragma unroll
    for (int n = 0; n < 7; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = n * 8 + 2 * t + (e & 1);
        const bool hi = e >= 2;
        float v = -INFINITY;
        if (col < WT) {
          const int cy = col / WS, cx = col % WS;
          const int dy = (hi ? yhi : ylo) - cy + WS - 1, dx = (hi ? xhi : xlo) - cx + WS - 1;
          v = sc[n][e] * scale;
          if ((hi ? r_hi : r_lo) < WT) v += __ldg(a.rel_bias + (dy * (2 * WS - 1) + dx) * a.heads + head);
          if ((hi ? reg_hi : reg_lo) != sreg[col]) v += -100.f;
        }
        sc[n][e] = v;
      }
      m_lo = fmaxf(m_lo, fmaxf(sc[n][0], sc[n][1])); m_hi = fmaxf(m_hi, fmaxf(sc[n][2], sc[n][3]));
    }
    m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 1)); m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 2));
    m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 1)); m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 2));
    float l_lo = 0.f, l_hi = 0.f;
#pragma unroll
    for (int n = 0; n < 7; ++n) {
      sc[n][0] = __expf(sc[n][0] - m_lo); sc[n][1] = __expf(sc[n][1] - m_lo);
      sc[n][2] = __expf(sc[n][2] - m_hi); sc[n][3] = __expf(sc[n][3] - m_hi);
      l_lo += sc[n][0] + sc[n][1]; l_hi += sc[n][2] + sc[n][3];
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
    float o[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
#pragma unroll
    for (int p = 0; p < 4; ++p) {                     // 16 keys per step; keys 56..63 have zero probability
      uint32_t pa[4];
      pa[0] = win_pack(sc[2 * p][0] * inv_lo, sc[2 * p][1] * inv_lo); pa[1] = win_pack(sc[2 * p][2] * inv_hi, sc[2 * p][3] * inv_hi);
      pa[2] = win_pack(sc[2 * p + 1][0] * inv_lo, sc[2 * p + 1][1] * inv_lo); pa[3] = win_pack(sc[2 * p + 1][2] * inv_hi, sc[2 * p + 1][3] * inv_hi);
      const __half* vr = sV + (p * 16 + (lane & 15)) * WKS;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t b0, b1;
        const uint32_t addr = (uint32_t)__cvta_generic_to_shared(vr + i * 8);
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(addr));
        win_mma(o[i], pa, b0, b1);
      }
    }
    const int row_lo = r_lo < WT ? srow[r_lo] : -2, row_hi = r_hi < WT ? srow[r_hi] : -2;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = head * WHD + i * 8 + 2 * t;
      if (row_lo >= 0) *reinterpret_cast<uint32_t*>(a.out + (size_t)row_lo * C + c) = win_pack(o[i][0], o[i][1]);
      if (row_hi >= 0) *reinterpret_cast<uint32_t*>(a.out + (size_t)row_hi * C + c) = win_pack(o[i][2], o[i][3]);
    }
  }
}

__global__ void swin_patch_merge_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int H, int W, int C) {
  // x [B,H,W,C] -> out [B, H2*W2, 4C]; channel blocks: (0,0), (1,0), (0,1), (1,1) (row offset, col offset)
  pdl_trigger();
  pdl_wait();
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const size_t n = (size_t)B * H2 * W2 * 4 * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % (4 * C));
    const size_t r = i / (4 * C);
    const int x2 = (int)(r % W2), y2 = (int)((r / W2) % H2), b = (int)(r / ((size_t)W2 * H2));
    const int blk = c4 / C, c = c4 % C;
    const int y = 2 * y2 + (blk & 1), xx = 2 * x2 + (blk >> 1);
    out[i] = (y < H && xx < W) ? x[(((size_t)b * H + y) * W + xx) * C + c] : 0.f;
  }
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_swin_patch_im2col(const uint8_t* d_img, void* d_out, int B, int H, int W, const float* h_mean3,
                                      const float* h_std3, void* stream) {
  if (!d_img || !d_out || !h_mean3 || !h_std3 || B < 1) { set_error("vlfm_swin_patch_im2col: bad argument"); return VLFM_E_INVALID; }
  const int Hp = (H + 3) / 4, Wp = (W + 3) / 4;
  size_t n = (size_t)B * Hp * Wp * 48;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  swin_patch_im2col_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_img, (__half*)d_out, B, H, W, Hp, Wp, h_mean3[0], h_mean3[1],
                                                                     h_mean3[2], h_std3[0], h_std3[1], h_std3[2]);
  VLFM_CHECK_LAUNCH("swin_patch_im2col_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_swin_window_attention(const void* d_qkv, const float* d_qkv_bias, const float* d_rel_bias, void* d_out, int B,
                                          int H, int W, int C, int heads, int shift, void* stream) {
  if (!d_qkv || !d_qkv_bias || !d_rel_bias || !d_out || B < 1 || heads < 1 || C != heads * WHD || shift < 0 || shift >= WS) {
    set_error("vlfm_swin_window_attention: bad argument (head_dim must be 32, window 7)"); return VLFM_E_INVALID; }
  WinAttnArgs a{(const __half*)d_qkv, d_qkv_bias, d_rel_bias, (__half*)d_out, H, W, C, heads, shift};
  const int nw = ((H + WS - 1) / WS) * ((W + WS - 1) / WS);
  const long total = (long)B * nw * heads;
  if (total > 0x7fffffffL) { set_error("vlfm_swin_window_attention: too many windows"); return VLFM_E_INVALID; }
  static bool cfg = false;
  if (!cfg) {
    int rc0 = check_cuda(cudaFuncSetAttribute(swin_window_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WIN_WARPS * WIN_SMEM_WARP),
                         "attr(swin_window_attention)");
    if (rc0) return rc0; cfg = true;
  }
  int rc = check_cuda(launch_pdl(swin_window_attention_kernel, dim3((unsigned)((total + WIN_WARPS - 1) / WIN_WARPS)), dim3(32 * WIN_WARPS),
                                 (size_t)WIN_WARPS * WIN_SMEM_WARP, (cudaStream_t)stream, a, B, (int)total),
                      "swin_window_attention_kernel");
  if (rc) return rc;
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_swin_patch_merge(const float* d_x, float* d_out, int B, int H, int W, int C, void* stream) {
  if (!d_x || !d_out || B < 1) { set_error("vlfm_swin_patch_merge: bad argument"); return VLFM_E_INVALID; }
  size_t n = (size_t)B * ((H + 1) / 2) * ((W + 1) / 2) * 4 * C;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  int rc = check_cuda(launch_pdl(swin_patch_merge_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, d_x, d_out, B, H, W, C),
                      "swin_patch_merge_kernel");
  if (rc) return rc;
  count_launch();
  return VLFM_OK;
}
