// Operators of MobileSAM (TinyViT-5M image encoder + box-prompted two-way mask decoder) that no shared kernel covers (sm_90a).
// Reference call site: vlfm/vlm/sam.py:40-57 (SamPredictor.set_image + predict(box=..., multimask_output=False)).
// GEMMs, LayerNorms and the short attentions run on the shared kernels (vlfm_gemm_f16*, vlfm_layernorm, vlfm_attention_f16);
// the engine is vlm/sam_engine.py.
//   - sam_resize_h / sam_resize_v_norm: Pillow-exact separable bilinear resize (ResizeLongestSide(1024)), the fp32 pixel
//     normalisation (true division) and the zero pad to S x S, written as fp16 NHWC;
//   - sam_im2col3x3: fp16 NHWC -> rows of a 3x3 (stride 1 or 2, pad 1) conv GEMM, K zero-padded to ldk;
//   - sam_dwconv3x3: depthwise 3x3 conv with folded BatchNorm and optional GELU (TinyViT MBConv / PatchMerging / local_conv);
//   - sam_add_act: out = act(a + b) (MBConv "add shortcut, then GELU"; plain casts);
//   - sam_window_attention: TinyViT window attention (49- or 196-token windows, head dim 32, |dy|,|dx| bias, the map zero-padded
//     to a window multiple BEFORE the LayerNorm, so padded tokens take part as keys without a mask);
//   - sam_box_tokens: box corners -> random-Fourier positional encoding + corner embeddings, after the iou / mask tokens;
//   - sam_add_pe_f16, sam_decoder_init: decoder operand staging (row-broadcast position embedding, per-box image keys);
//   - sam_t2i_attention: 7 token queries x 4096 image keys, head dim 16, keys split over CTAs in fixed 256-key chunks and merged
//     in chunk order (deterministic: no atomics);
//   - sam_pixel_shuffle2: the 2x2 stride-2 transposed conv's GEMM output [(dy,dx,c) columns] scattered to the 2x map;
//   - sam_mask_logits: second transposed conv's GEMM output -> GELU -> hypernetwork dot product (mask 0 only);
//   - sam_mask_finish: bilinear to S x S, crop to the resized frame, bilinear to (H, W), threshold > 0.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace vlfm {

constexpr int SAM_PREC_BITS = 32 - 8 - 2;   // Pillow's 8-bpc fixed point

__device__ __forceinline__ float sam_gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ uint8_t sam_clip8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

static unsigned grid1d(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  if (b > 132LL * 32) b = 132LL * 32;
  return (unsigned)(b < 1 ? 1 : b);
}

// ---------------------------------------------------------------------------------------------------------- preprocess
__global__ void sam_resize_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ mid, int B, int H, int W, int OW,
                                    const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk, int ksize) {
  const long long n = (long long)B * H * OW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int xo = (int)(i % OW);
    const long long by = i / OW;   // b * H + y
    const int x0 = bounds[2 * xo], cnt = bounds[2 * xo + 1];
    const uint8_t* src = in + (by * W + x0) * 3;
    const int32_t* k = kk + (size_t)xo * ksize;
    int s0 = 1 << (SAM_PREC_BITS - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < cnt; ++t) {
      const int c = k[t];
      s0 += src[3 * t] * c; s1 += src[3 * t + 1] * c; s2 += src[3 * t + 2] * c;
    }
    uint8_t* o = mid + i * 3;
    o[0] = sam_clip8(s0 >> SAM_PREC_BITS); o[1] = sam_clip8(s1 >> SAM_PREC_BITS); o[2] = sam_clip8(s2 >> SAM_PREC_BITS);
  }
}

__global__ void sam_resize_v_norm_kernel(const uint8_t* __restrict__ mid, __half* __restrict__ out, int B, int H, int OH, int OW,
                                         int S, const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk, int ksize,
                                         float m0, float m1, float m2, float s0, float s1, float s2) {
  const long long n = (long long)B * S * S;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % S), y = (int)((i / S) % S), b = (int)(i / ((long long)S * S));
    __half* o = out + i * 3;
    if (y >= OH || x >= OW) {
      o[0] = o[1] = o[2] = __float2half_rn(0.f);
      continue;
    }
    const int y0 = bounds[2 * y], cnt = bounds[2 * y + 1];
    const int32_t* k = kk + (size_t)y * ksize;
    int a0 = 1 << (SAM_PREC_BITS - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < cnt; ++t) {
      const uint8_t* p = mid + (((size_t)b * H + y0 + t) * OW + x) * 3;
      const int c = k[t];
      a0 += p[0] * c; a1 += p[1] * c; a2 += p[2] * c;
    }
    // (x - mean) / std in fp32 with a true division (segment_anything's Sam.preprocess)
    o[0] = __float2half_rn(__fdiv_rn(__fsub_rn((float)sam_clip8(a0 >> SAM_PREC_BITS), m0), s0));
    o[1] = __float2half_rn(__fdiv_rn(__fsub_rn((float)sam_clip8(a1 >> SAM_PREC_BITS), m1), s1));
    o[2] = __float2half_rn(__fdiv_rn(__fsub_rn((float)sam_clip8(a2 >> SAM_PREC_BITS), m2), s2));
  }
}

// ------------------------------------------------------------------------------------------------------- convolutions
__global__ void sam_im2col3x3_kernel(const __half* __restrict__ x, __half* __restrict__ col, int B, int H, int W, int C, int stride,
                                     int Ho, int Wo, int ldk) {
  const long long n = (long long)B * Ho * Wo * ldk;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % ldk);
    const long long r = i / ldk;
    const int xo = (int)(r % Wo), yo = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    __half v = __float2half_rn(0.f);
    if (k < 9 * C) {
      const int tap = k / C, c = k % C;
      const int y = yo * stride - 1 + tap / 3, xx = xo * stride - 1 + tap % 3;
      if (y >= 0 && y < H && xx >= 0 && xx < W) v = x[(((size_t)b * H + y) * W + xx) * C + c];
    }
    col[i] = v;
  }
}

// d_w [9, C] (tap-major, BN folded), d_b [C]; NHWC in / out, fp16 or fp32 each.
__global__ void sam_dwconv3x3_kernel(const void* __restrict__ in, int in_f32, const float* __restrict__ w, const float* __restrict__ bias,
                                     void* __restrict__ out, int out_f32, int B, int H, int W, int C, int stride, int Ho, int Wo,
                                     int gelu) {
  const long long n = (long long)B * Ho * Wo * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int xo = (int)(r % Wo), yo = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int y = yo * stride - 1 + t / 3, x = xo * stride - 1 + t % 3;
      if (y < 0 || y >= H || x < 0 || x >= W) continue;
      const size_t src = (((size_t)b * H + y) * W + x) * C + c;
      const float v = in_f32 ? reinterpret_cast<const float*>(in)[src] : __half2float(reinterpret_cast<const __half*>(in)[src]);
      acc = fmaf(v, w[t * C + c], acc);
    }
    acc += bias[c];
    if (gelu) acc = sam_gelu(acc);
    if (out_f32) reinterpret_cast<float*>(out)[i] = acc;
    else reinterpret_cast<__half*>(out)[i] = __float2half_rn(acc);
  }
}

__global__ void sam_add_act_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out32,
                                   __half* __restrict__ out16, long long n, int gelu) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = a[i];
    if (b) v += b[i];
    if (gelu) v = sam_gelu(v);
    if (out32) out32[i] = v;
    if (out16) out16[i] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------- window attention
constexpr int SAM_HD = 32;

// One CTA per (window, head, image); one thread per window token.  K / V of the window in fp32 shared memory (all threads read
// the same key row: broadcast), softmax online over chunks of one window row (WSZ keys).
template <int WSZ>
__global__ void __launch_bounds__(WSZ == 7 ? 64 : 256)
sam_window_attention_kernel(const __half* __restrict__ qkv, const __half* __restrict__ pad_qkv, const float* __restrict__ bias,
                            __half* __restrict__ out, int H, int W, int C, int heads, float scale) {
  constexpr int N = WSZ * WSZ;
  extern __shared__ float4 sam_win_smem[];
  float* sK = reinterpret_cast<float*>(sam_win_smem);   // [N][32]
  float* sV = sK + N * SAM_HD;                           // [N][32]
  float* sB = sV + N * SAM_HD;                           // [N] bias per |dy|*WSZ+|dx|
  const int nWx = (W + WSZ - 1) / WSZ;
  const int wy = blockIdx.x / nWx, wx = blockIdx.x % nWx, h = blockIdx.y, b = blockIdx.z;
  const int ld = 3 * C;
  for (int e = threadIdx.x; e < N * SAM_HD; e += blockDim.x) {
    const int t = e / SAM_HD, d = e % SAM_HD;
    const int y = wy * WSZ + t / WSZ, x = wx * WSZ + t % WSZ;
    const __half* src = (y < H && x < W) ? qkv + (((size_t)b * H + y) * W + x) * ld : pad_qkv;
    sK[e] = __half2float(src[C + h * SAM_HD + d]);
    sV[e] = __half2float(src[2 * C + h * SAM_HD + d]);
  }
  for (int e = threadIdx.x; e < N; e += blockDim.x) sB[e] = bias[(size_t)h * N + e];
  __syncthreads();
  const int t = threadIdx.x;
  if (t >= N) return;
  const int ty = t / WSZ, tx = t % WSZ;
  const int y = wy * WSZ + ty, x = wx * WSZ + tx;
  if (y >= H || x >= W) return;   // padded queries are cropped away
  const size_t row = ((size_t)b * H + y) * W + x;
  float q[SAM_HD], acc[SAM_HD];
  {
    const __half2* qp = reinterpret_cast<const __half2*>(qkv + row * ld + h * SAM_HD);
#pragma unroll
    for (int d = 0; d < SAM_HD / 2; ++d) { const float2 f = __half22float2(qp[d]); q[2 * d] = f.x; q[2 * d + 1] = f.y; }
  }
#pragma unroll
  for (int d = 0; d < SAM_HD; ++d) acc[d] = 0.f;
  float m = -INFINITY, l = 0.f;
  for (int ky = 0; ky < WSZ; ++ky) {
    const int dy = ky > ty ? ky - ty : ty - ky;
    float s[WSZ];
    float cm = -INFINITY;
#pragma unroll
    for (int kx = 0; kx < WSZ; ++kx) {
      const float4* kr = reinterpret_cast<const float4*>(sK + (ky * WSZ + kx) * SAM_HD);
      float dot = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < SAM_HD / 4; ++d4) {
        const float4 k4 = kr[d4];
        dot = fmaf(q[4 * d4], k4.x, dot); dot = fmaf(q[4 * d4 + 1], k4.y, dot);
        dot = fmaf(q[4 * d4 + 2], k4.z, dot); dot = fmaf(q[4 * d4 + 3], k4.w, dot);
      }
      const int dx = kx > tx ? kx - tx : tx - kx;
      s[kx] = dot * scale + sB[dy * WSZ + dx];
      cm = fmaxf(cm, s[kx]);
    }
    const float mn = fmaxf(m, cm);
    const float corr = __expf(m - mn);
    l *= corr;
#pragma unroll
    for (int d = 0; d < SAM_HD; ++d) acc[d] *= corr;
    m = mn;
#pragma unroll
    for (int kx = 0; kx < WSZ; ++kx) {
      const float p = __expf(s[kx] - m);
      l += p;
      const float4* vr = reinterpret_cast<const float4*>(sV + (ky * WSZ + kx) * SAM_HD);
#pragma unroll
      for (int d4 = 0; d4 < SAM_HD / 4; ++d4) {
        const float4 v4 = vr[d4];
        acc[4 * d4] = fmaf(p, v4.x, acc[4 * d4]); acc[4 * d4 + 1] = fmaf(p, v4.y, acc[4 * d4 + 1]);
        acc[4 * d4 + 2] = fmaf(p, v4.z, acc[4 * d4 + 2]); acc[4 * d4 + 3] = fmaf(p, v4.w, acc[4 * d4 + 3]);
      }
    }
  }
  const float inv = 1.f / l;
  __half2* o = reinterpret_cast<__half2*>(out + row * C + h * SAM_HD);
#pragma unroll
  for (int d = 0; d < SAM_HD / 2; ++d) o[d] = __floats2half2_rn(acc[2 * d] * inv, acc[2 * d + 1] * inv);
}

// ---------------------------------------------------------------------------------------------------- prompt encoder
// tokens[m*7 + 0..4] = fixed[0..4] (iou token, 4 mask tokens); tokens[m*7 + 5 + i] = PE(corner i) + fixed[5 + i].
// The corners follow ResizeLongestSide.apply_boxes (float64 scale, cast to float32) and PositionEmbeddingRandom.
__global__ void sam_box_tokens_kernel(const double* __restrict__ boxes, int M, int H, int W, int newh, int neww, int S,
                                      const float* __restrict__ gauss, const float* __restrict__ fixed, float* __restrict__ tokens,
                                      int D) {
  const int m = blockIdx.x;
  const int half = D / 2;
  float* tok = tokens + (size_t)m * 7 * D;
  for (int e = threadIdx.x; e < 5 * D; e += blockDim.x) tok[e] = fixed[e];
  for (int e = threadIdx.x; e < 2 * half; e += blockDim.x) {
    const int corner = e / half, j = e % half;
    const double sx = (double)neww / (double)W, sy = (double)newh / (double)H;
    const float cx = (float)(boxes[4 * m + 2 * corner] * sx), cy = (float)(boxes[4 * m + 2 * corner + 1] * sy);
    float u = (cx + 0.5f) / (float)S, v = (cy + 0.5f) / (float)S;
    u = 2.f * u - 1.f; v = 2.f * v - 1.f;
    float a = fmaf(v, gauss[half + j], u * gauss[j]);
    a = 6.283185307179586f * a;
    float* t = tok + (size_t)(5 + corner) * D;
    t[j] = sinf(a) + fixed[(5 + corner) * D + j];
    t[half + j] = cosf(a) + fixed[(5 + corner) * D + half + j];
  }
}

__global__ void sam_add_pe_f16_kernel(const float* __restrict__ x, const float* __restrict__ pe, __half* __restrict__ out16,
                                      __half* __restrict__ outp16, long long rows, long long pe_rows, int D) {
  const long long n = rows * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    if (out16) out16[i] = __float2half_rn(v);
    if (outp16) outp16[i] = __float2half_rn(v + pe[((i / D) % pe_rows) * D + i % D]);
  }
}

__global__ void sam_decoder_init_kernel(const float* __restrict__ emb, const int32_t* __restrict__ frame, const float* __restrict__ nomask,
                                        float* __restrict__ keys, int M, int F, long long HW, int D) {
  const long long per = HW * D, n = (long long)M * per;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / per);
    const int f = frame[m];
    const long long r = i % per;
    keys[i] = (f >= 0 && f < F) ? emb[(long long)f * per + r] + nomask[r % D] : __int_as_float(0x7fc00000);
  }
}

// ---------------------------------------------------------------------------------------- token -> image attention
constexpr int T2I_HD = 16, T2I_CHUNK = 256, T2I_MAXQ = 8, T2I_PART = T2I_HD + 2;

// grid (chunks, heads, M), one warp per query (Nq <= 8).  Lane j handles keys j, j+32, ... of the chunk with an online softmax;
// the 32 lane states merge by a fixed butterfly, and the chunk's (max, sum, acc[16]) goes to part[((m*heads+h)*chunks+c)*Nq+q].
__global__ void __launch_bounds__(32 * T2I_MAXQ)
sam_t2i_partial_kernel(const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v, float* __restrict__ part,
                       int heads, int Nq, int Nk, int ldq, int ldk, int ldv, float scale) {
  __shared__ float sK[T2I_CHUNK][T2I_HD], sV[T2I_CHUNK][T2I_HD];
  const int c = blockIdx.x, h = blockIdx.y, m = blockIdx.z, chunks = gridDim.x;
  const int k0 = c * T2I_CHUNK, nk = min(T2I_CHUNK, Nk - k0);
  for (int e = threadIdx.x; e < nk * T2I_HD; e += blockDim.x) {
    const int j = e / T2I_HD, d = e % T2I_HD;
    const size_t r = (size_t)m * Nk + k0 + j;
    sK[j][d] = __half2float(k[r * ldk + h * T2I_HD + d]);
    sV[j][d] = __half2float(v[r * ldv + h * T2I_HD + d]);
  }
  __syncthreads();
  const int w = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (w >= Nq) return;
  float qv[T2I_HD], acc[T2I_HD];
  const __half* qp = q + ((size_t)m * Nq + w) * ldq + h * T2I_HD;
#pragma unroll
  for (int d = 0; d < T2I_HD; ++d) { qv[d] = __half2float(qp[d]) * scale; acc[d] = 0.f; }
  float mx = -INFINITY, l = 0.f;
  for (int j = lane; j < nk; j += 32) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < T2I_HD; ++d) s = fmaf(qv[d], sK[j][d], s);
    const float mn = fmaxf(mx, s);
    const float corr = __expf(mx - mn), p = __expf(s - mn);
    l = l * corr + p;
#pragma unroll
    for (int d = 0; d < T2I_HD; ++d) acc[d] = fmaf(p, sV[j][d], acc[d] * corr);
    mx = mn;
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, mx, off);
    const float mn = fmaxf(mx, mo);
    const float ca = mx == -INFINITY ? 0.f : __expf(mx - mn), cb = mo == -INFINITY ? 0.f : __expf(mo - mn);
    l = l * ca + __shfl_xor_sync(0xffffffffu, l, off) * cb;
#pragma unroll
    for (int d = 0; d < T2I_HD; ++d) acc[d] = acc[d] * ca + __shfl_xor_sync(0xffffffffu, acc[d], off) * cb;
    mx = mn;
  }
  if (lane == 0) {
    float* p = part + ((((size_t)m * heads + h) * chunks + c) * Nq + w) * T2I_PART;
    p[0] = mx; p[1] = l;
#pragma unroll
    for (int d = 0; d < T2I_HD; ++d) p[2 + d] = acc[d];
  }
}

// one thread per (m, q, h, d): merge the chunks in order
__global__ void sam_t2i_merge_kernel(const float* __restrict__ part, __half* __restrict__ o, int M, int heads, int Nq, int chunks, int ldo) {
  const int n = M * Nq * heads * T2I_HD;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int d = i % T2I_HD, h = (i / T2I_HD) % heads, qi = (i / (T2I_HD * heads)) % Nq, m = i / (T2I_HD * heads * Nq);
    float mx = -INFINITY;
    for (int c = 0; c < chunks; ++c) mx = fmaxf(mx, part[((((size_t)m * heads + h) * chunks + c) * Nq + qi) * T2I_PART]);
    float l = 0.f, a = 0.f;
    for (int c = 0; c < chunks; ++c) {
      const float* p = part + ((((size_t)m * heads + h) * chunks + c) * Nq + qi) * T2I_PART;
      const float f = __expf(p[0] - mx);
      l = fmaf(p[1], f, l);
      a = fmaf(p[2 + d], f, a);
    }
    o[((size_t)m * Nq + qi) * ldo + h * T2I_HD + d] = __float2half_rn(a / l);
  }
}

// ------------------------------------------------------------------------------------------------- mask upscaling
// in [B*h*w, 4*C] with column (dy*2+dx)*C + c  ->  out [B, 2h, 2w, C]
__global__ void sam_pixel_shuffle2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int h, int w, int C) {
  const long long n = (long long)B * 4 * h * w * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int X = (int)(r % (2 * w)), Y = (int)((r / (2 * w)) % (2 * h)), b = (int)(r / (4LL * h * w));
    const int y = Y >> 1, x = X >> 1, t = ((Y & 1) << 1) | (X & 1);
    out[i] = in[(((size_t)b * h + y) * w + x) * 4 * C + t * C + c];
  }
}

// logits[m, Y, X] = sum_c hyper[m, c] * GELU(up[m, y, x, (dy,dx,c)])   (C <= 64)
__global__ void sam_mask_logits_kernel(const float* __restrict__ up, const float* __restrict__ hyper, float* __restrict__ logits, int M,
                                       int h, int w, int C) {
  const long long n = (long long)M * 4 * h * w;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(i % (2 * w)), Y = (int)((i / (2 * w)) % (2 * h)), m = (int)(i / (4LL * h * w));
    const int t = ((Y & 1) << 1) | (X & 1);
    const float* u = up + ((((size_t)m * h + (Y >> 1)) * w + (X >> 1)) * 4 + t) * C;
    const float* hy = hyper + (size_t)m * C;
    float s = 0.f;
    for (int c = 0; c < C; ++c) s = fmaf(hy[c], sam_gelu(u[c]), s);
    logits[i] = s;
  }
}

// torch upsample_bilinear2d, align_corners=False: source index and weights of output index `o` for in -> out
struct SamLerp { int i0, i1; float w0, w1; };
__device__ __forceinline__ SamLerp sam_lerp(int o, int in, int out) {
  const float scale = (float)in / (float)out;
  float src = scale * ((float)o + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  SamLerp r;
  r.i0 = (int)src;
  r.i1 = r.i0 + (r.i0 < in - 1 ? 1 : 0);
  r.w1 = src - (float)r.i0;
  r.w0 = 1.f - r.w1;
  return r;
}

// value of the first interpolation (L x L -> S x S) at (Y, X)
__device__ __forceinline__ float sam_up1(const float* __restrict__ low, int L, int S, int Y, int X) {
  const SamLerp a = sam_lerp(Y, L, S), b = sam_lerp(X, L, S);
  return a.w0 * (b.w0 * low[a.i0 * L + b.i0] + b.w1 * low[a.i0 * L + b.i1]) +
         a.w1 * (b.w0 * low[a.i1 * L + b.i0] + b.w1 * low[a.i1 * L + b.i1]);
}

__global__ void sam_mask_finish_kernel(const float* __restrict__ low, uint8_t* __restrict__ out, int M, int L, int S, int newh, int neww,
                                       int H, int W) {
  const long long n = (long long)M * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), m = (int)(i / ((long long)H * W));
    const float* lo = low + (size_t)m * L * L;
    const SamLerp a = sam_lerp(y, newh, H), b = sam_lerp(x, neww, W);
    const float v = a.w0 * (b.w0 * sam_up1(lo, L, S, a.i0, b.i0) + b.w1 * sam_up1(lo, L, S, a.i0, b.i1)) +
                    a.w1 * (b.w0 * sam_up1(lo, L, S, a.i1, b.i0) + b.w1 * sam_up1(lo, L, S, a.i1, b.i1));
    out[i] = v > 0.f ? 1 : 0;
  }
}

}  // namespace vlfm

using namespace vlfm;

#define SAM_LAUNCHED(what)  do { VLFM_CHECK_LAUNCH(what); count_launch(); } while (0)

extern "C" int vlfm_sam_preprocess(const uint8_t* d_img, uint8_t* d_mid, void* d_out, int B, int H, int W, int OH, int OW, int S,
                                   const int32_t* d_hbounds, const int32_t* d_hkk, int hksize, const int32_t* d_vbounds,
                                   const int32_t* d_vkk, int vksize, const float* h_mean3, const float* h_std3, void* stream) {
  if (!d_img || !d_mid || !d_out || !d_hbounds || !d_hkk || !d_vbounds || !d_vkk || !h_mean3 || !h_std3 || B < 1 || H < 1 || W < 1 ||
      OH < 1 || OW < 1 || OH > S || OW > S || hksize < 1 || vksize < 1) {
    set_error("vlfm_sam_preprocess: bad argument"); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  sam_resize_h_kernel<<<grid1d((long long)B * H * OW, 256), 256, 0, st>>>(d_img, d_mid, B, H, W, OW, d_hbounds, d_hkk, hksize);
  SAM_LAUNCHED("sam_resize_h_kernel");
  sam_resize_v_norm_kernel<<<grid1d((long long)B * S * S, 256), 256, 0, st>>>(d_mid, (__half*)d_out, B, H, OH, OW, S, d_vbounds, d_vkk,
                                                                                vksize, h_mean3[0], h_mean3[1], h_mean3[2], h_std3[0],
                                                                                h_std3[1], h_std3[2]);
  SAM_LAUNCHED("sam_resize_v_norm_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_im2col3x3(const void* d_x16, void* d_col16, int B, int H, int W, int C, int stride, int ldk, void* stream) {
  if (!d_x16 || !d_col16 || B < 1 || H < 1 || W < 1 || C < 1 || (stride != 1 && stride != 2) || ldk < 9 * C || (ldk & 7)) {
    set_error("vlfm_sam_im2col3x3: bad argument"); return VLFM_E_INVALID; }
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  sam_im2col3x3_kernel<<<grid1d((long long)B * Ho * Wo * ldk, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_x16, (__half*)d_col16, B, H, W, C, stride, Ho, Wo, ldk);
  SAM_LAUNCHED("sam_im2col3x3_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_dwconv3x3(const void* d_in, int in_f32, const float* d_w, const float* d_b, void* d_out, int out_f32, int B, int H,
                                  int W, int C, int stride, int gelu, void* stream) {
  if (!d_in || !d_w || !d_b || !d_out || B < 1 || H < 1 || W < 1 || C < 1 || (stride != 1 && stride != 2)) {
    set_error("vlfm_sam_dwconv3x3: bad argument"); return VLFM_E_INVALID; }
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  sam_dwconv3x3_kernel<<<grid1d((long long)B * Ho * Wo * C, 256), 256, 0, (cudaStream_t)stream>>>(d_in, in_f32, d_w, d_b, d_out, out_f32,
                                                                                                   B, H, W, C, stride, Ho, Wo, gelu);
  SAM_LAUNCHED("sam_dwconv3x3_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_add_act(const float* d_a, const float* d_b, float* d_out32, void* d_out16, long long n, int gelu, void* stream) {
  if (!d_a || (!d_out32 && !d_out16) || n < 1) { set_error("vlfm_sam_add_act: bad argument"); return VLFM_E_INVALID; }
  sam_add_act_kernel<<<grid1d(n, 256), 256, 0, (cudaStream_t)stream>>>(d_a, d_b, d_out32, (__half*)d_out16, n, gelu);
  SAM_LAUNCHED("sam_add_act_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_window_attention(const void* d_qkv, const void* d_pad_qkv, const float* d_bias, void* d_out, int B, int H, int W,
                                         int C, int heads, int ws, float scale, void* stream) {
  if (!d_qkv || !d_pad_qkv || !d_bias || !d_out || B < 1 || H < 1 || W < 1 || heads < 1 || C != heads * SAM_HD || (ws != 7 && ws != 14)) {
    set_error("vlfm_sam_window_attention: bad argument (head dim 32, window 7 or 14)"); return VLFM_E_INVALID; }
  const int nWy = (H + ws - 1) / ws, nWx = (W + ws - 1) / ws;
  if (B > 65535 || heads > 65535) { set_error("vlfm_sam_window_attention: grid too large"); return VLFM_E_INVALID; }
  const dim3 grid(nWy * nWx, heads, B);
  const size_t smem = ((size_t)2 * ws * ws * SAM_HD + ws * ws) * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  if (ws == 7) {
    sam_window_attention_kernel<7><<<grid, 64, smem, st>>>((const __half*)d_qkv, (const __half*)d_pad_qkv, d_bias, (__half*)d_out, H, W, C,
                                                          heads, scale);
  } else {
    static bool cfg = false;
    if (!cfg) {
      int rc = check_cuda(cudaFuncSetAttribute(sam_window_attention_kernel<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                          "attr(sam_window_attention)");
      if (rc) return rc;
      cfg = true;
    }
    sam_window_attention_kernel<14><<<grid, 256, smem, st>>>((const __half*)d_qkv, (const __half*)d_pad_qkv, d_bias, (__half*)d_out, H, W,
                                                            C, heads, scale);
  }
  SAM_LAUNCHED("sam_window_attention_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_box_tokens(const double* d_boxes, int M, int H, int W, int newh, int neww, int S, const float* d_gauss,
                                   const float* d_fixed, float* d_tokens, int D, void* stream) {
  if (!d_boxes || !d_gauss || !d_fixed || !d_tokens || M < 1 || H < 1 || W < 1 || newh < 1 || neww < 1 || S < 1 || D < 2 || (D & 1)) {
    set_error("vlfm_sam_box_tokens: bad argument"); return VLFM_E_INVALID; }
  sam_box_tokens_kernel<<<M, 256, 0, (cudaStream_t)stream>>>(d_boxes, M, H, W, newh, neww, S, d_gauss, d_fixed, d_tokens, D);
  SAM_LAUNCHED("sam_box_tokens_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_add_pe_f16(const float* d_x, const float* d_pe, void* d_out16, void* d_outp16, long long rows, long long pe_rows,
                                   int D, void* stream) {
  if (!d_x || (!d_out16 && !d_outp16) || (d_outp16 && (!d_pe || pe_rows < 1)) || rows < 1 || D < 1) {
    set_error("vlfm_sam_add_pe_f16: bad argument"); return VLFM_E_INVALID; }
  sam_add_pe_f16_kernel<<<grid1d(rows * D, 256), 256, 0, (cudaStream_t)stream>>>(d_x, d_pe, (__half*)d_out16, (__half*)d_outp16, rows,
                                                                                pe_rows < 1 ? 1 : pe_rows, D);
  SAM_LAUNCHED("sam_add_pe_f16_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_decoder_init(const float* d_emb, const int32_t* d_frame, const float* d_nomask, float* d_keys, int M, int F,
                                     int HW, int D, void* stream) {
  if (!d_emb || !d_frame || !d_nomask || !d_keys || M < 1 || F < 1 || HW < 1 || D < 1) {
    set_error("vlfm_sam_decoder_init: bad argument"); return VLFM_E_INVALID; }
  sam_decoder_init_kernel<<<grid1d((long long)M * HW * D, 256), 256, 0, (cudaStream_t)stream>>>(d_emb, d_frame, d_nomask, d_keys, M, F, HW, D);
  SAM_LAUNCHED("sam_decoder_init_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_t2i_attention(const void* d_q, const void* d_k, const void* d_v, void* d_o, int M, int heads, int Nq, int Nk,
                                      int ldq, int ldk, int ldv, int ldo, float scale, float* d_part, size_t part_floats, void* stream) {
  const int chunks = (Nk + T2I_CHUNK - 1) / T2I_CHUNK;
  if (!d_q || !d_k || !d_v || !d_o || !d_part || M < 1 || heads < 1 || Nq < 1 || Nq > T2I_MAXQ || Nk < 1 || M > 65535 || heads > 65535 ||
      ldq < heads * T2I_HD || ldk < heads * T2I_HD || ldv < heads * T2I_HD || ldo < heads * T2I_HD) {
    set_error("vlfm_sam_t2i_attention: bad argument (head dim 16, Nq <= %d)", T2I_MAXQ); return VLFM_E_INVALID; }
  if (part_floats < (size_t)M * heads * chunks * Nq * T2I_PART) {
    set_error("vlfm_sam_t2i_attention: d_part holds %zu floats, needs %zu", part_floats, (size_t)M * heads * chunks * Nq * T2I_PART);
    return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  sam_t2i_partial_kernel<<<dim3(chunks, heads, M), 32 * T2I_MAXQ, 0, st>>>((const __half*)d_q, (const __half*)d_k, (const __half*)d_v, d_part,
                                                                           heads, Nq, Nk, ldq, ldk, ldv, scale);
  SAM_LAUNCHED("sam_t2i_partial_kernel");
  const int n = M * Nq * heads * T2I_HD;
  sam_t2i_merge_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_part, (__half*)d_o, M, heads, Nq, chunks, ldo);
  SAM_LAUNCHED("sam_t2i_merge_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_pixel_shuffle2(const float* d_in, float* d_out, int B, int h, int w, int C, void* stream) {
  if (!d_in || !d_out || B < 1 || h < 1 || w < 1 || C < 1) { set_error("vlfm_sam_pixel_shuffle2: bad argument"); return VLFM_E_INVALID; }
  sam_pixel_shuffle2_kernel<<<grid1d(4LL * B * h * w * C, 256), 256, 0, (cudaStream_t)stream>>>(d_in, d_out, B, h, w, C);
  SAM_LAUNCHED("sam_pixel_shuffle2_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_mask_logits(const float* d_up, const float* d_hyper, float* d_logits, int M, int h, int w, int C, void* stream) {
  if (!d_up || !d_hyper || !d_logits || M < 1 || h < 1 || w < 1 || C < 1) { set_error("vlfm_sam_mask_logits: bad argument"); return VLFM_E_INVALID; }
  sam_mask_logits_kernel<<<grid1d(4LL * M * h * w, 256), 256, 0, (cudaStream_t)stream>>>(d_up, d_hyper, d_logits, M, h, w, C);
  SAM_LAUNCHED("sam_mask_logits_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_sam_mask_finish(const float* d_low, uint8_t* d_out, int M, int L, int S, int newh, int neww, int H, int W, void* stream) {
  if (!d_low || !d_out || M < 1 || L < 1 || S < 1 || newh < 1 || neww < 1 || newh > S || neww > S || H < 1 || W < 1) {
    set_error("vlfm_sam_mask_finish: bad argument"); return VLFM_E_INVALID; }
  sam_mask_finish_kernel<<<grid1d((long long)M * H * W, 256), 256, 0, (cudaStream_t)stream>>>(d_low, d_out, M, L, S, newh, neww, H, W);
  SAM_LAUNCHED("sam_mask_finish_kernel");
  return VLFM_OK;
}
