// PointNav policy kernels (vlfm/policy/utils/pointnav_policy.py WrappedPointNavResNetPolicy.act: a ResNet-18 over depth and a
// 2-layer LSTM of 512); the engine is vlfm_b200/policy/pointnav_engine.py.  Activations are NHWC.  Every conv runs as an im2col
// pass plus vlfm_gemm_f16 (fp16 operands, fp32 out); these kernels are the rest:
//   - pointnav_depth_in: area resize of the depth frame to the network's input size, 2x2 average pool, and the conv1 (7x7, stride
//     2, pad 3) im2col rows, in one launch;
//   - pointnav_groupnorm: GroupNorm statistics per (image, group) and out = act(GN_a(x) + r), r = none, an fp32 identity stream
//     or GN_b(y) of the downsample branch, to fp32 and / or fp16;
//   - pointnav_maxpool3s2, pointnav_gather_s2: the stem's max pool and the rows of a stride-2 1x1 conv;
//   - pointnav_gemv: y = act(x W^T + b) in fp32 on CUDA cores, W streamed once for up to 64 environments' inputs;
//   - pointnav_lstm_prep / pointnav_lstm_cell / pointnav_lstm_head: mask, goal and previous-action features, the LSTM cell
//     updates, the action head and the hidden-state write-back.
// Every reduction has a fixed order (no atomics): results are bitwise reproducible, and an environment's result does not depend
// on which other environments share the launch.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace vlfm {

constexpr int PN_HID = 512;      // LSTM hidden size
constexpr int PN_EMB = 32;       // goal and previous-action embedding widths
constexpr int PN_VIS = 512;      // visual_fc output
constexpr int PN_LD0 = PN_VIS + 2 * PN_EMB + PN_HID;   // layer-0 GEMV input row: [visual | goal | prev action | h0]
constexpr int PN_LD1 = 2 * PN_HID;                      // layer-1 GEMV input row: [h0' | h1]
// rows per CTA (one warp each): 16, or 8 for 64 environments, whose 64 accumulators per lane need more than 128 registers
template <int NB> constexpr int gemv_rows() { return NB > 32 ? 8 : 16; }
constexpr int GEMV_KC = 512;     // K chunk staged in shared memory
constexpr int GEMV_MAXB = 64;

#define PN_LAUNCHED(what)  do { VLFM_CHECK_LAUNCH(what); count_launch(); } while (0)

static unsigned pn_grid(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  if (b > 132LL * 32) b = 132LL * 32;
  return (unsigned)(b < 1 ? 1 : b);
}

// Deterministic block sum (fixed shuffle tree, then the warps' partials in warp order); every thread gets the result.
__device__ __forceinline__ float pn_block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < nw; ++i) s += red[i];
  return s;
}

__device__ __forceinline__ float pn_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------------------------------------------------------------ depth in
// torch's "area" interpolation (adaptive average pooling): output index i averages source [floor(i*S/O), ceil((i+1)*S/O)).
__device__ __forceinline__ float pn_area(const float* __restrict__ img, int H, int W, int IH, int IW, int y, int x) {
  const int y0 = (int)(((long long)y * H) / IH), y1 = (int)(((long long)(y + 1) * H + IH - 1) / IH);
  const int x0 = (int)(((long long)x * W) / IW), x1 = (int)(((long long)(x + 1) * W + IW - 1) / IW);
  float s = 0.f;
  for (int yy = y0; yy < y1; ++yy)
    for (int xx = x0; xx < x1; ++xx) s += img[(size_t)yy * W + xx];
  return s / (float)((y1 - y0) * (x1 - x0));
}

// grid (conv1 output rows, B).  The block computes the 7 pooled rows its conv row reads into shared memory, then writes the
// row's im2col columns (tap ky*7 + kx, zero padded to ldk).  With d_resized it also writes resized rows [4y, 4y + 4) (the last
// block: through IH).
__global__ void pointnav_depth_in_kernel(const float* __restrict__ depth, int H, int W, int IH, int IW, int PH, int PW, int OH,
                                         int OW, __half* __restrict__ col, int ldk, float* __restrict__ resized) {
  extern __shared__ float pooled[];   // [7][PW]
  const int y = blockIdx.x, b = blockIdx.y;
  const float* img = depth + (size_t)b * H * W;
  for (int i = threadIdx.x; i < 7 * PW; i += blockDim.x) {
    const int r = i / PW, px = i % PW, py = 2 * y - 3 + r;
    float v = 0.f;
    if (py >= 0 && py < PH) {
      // F.avg_pool2d(2): the four pixels in row-major order, then / 4
      const float a = pn_area(img, H, W, IH, IW, 2 * py, 2 * px), c = pn_area(img, H, W, IH, IW, 2 * py, 2 * px + 1);
      const float d = pn_area(img, H, W, IH, IW, 2 * py + 1, 2 * px), e = pn_area(img, H, W, IH, IW, 2 * py + 1, 2 * px + 1);
      v = (((a + c) + d) + e) / 4.f;
    }
    pooled[i] = v;
  }
  __syncthreads();
  __half* out = col + ((size_t)b * OH + y) * OW * ldk;
  for (int i = threadIdx.x; i < OW * ldk; i += blockDim.x) {
    const int xo = i / ldk, k = i % ldk;
    float v = 0.f;
    if (k < 49) {
      const int ky = k / 7, kx = k % 7, px = 2 * xo - 3 + kx;
      if (px >= 0 && px < PW) v = pooled[ky * PW + px];
    }
    out[i] = __float2half_rn(v);
  }
  if (resized) {
    const int r0 = 4 * y, r1 = (y == OH - 1) ? IH : min(IH, 4 * y + 4);
    float* ro = resized + (size_t)b * IH * IW;
    for (int i = threadIdx.x; i < (r1 - r0) * IW; i += blockDim.x) {
      const int yy = r0 + i / IW, xx = i % IW;
      ro[(size_t)yy * IW + xx] = pn_area(img, H, W, IH, IW, yy, xx);
    }
  }
}

// ----------------------------------------------------------------------------------------------------------- GroupNorm
// One CTA per (group, image).  Two-pass statistics in fp32 (mean, then the mean of squared deviations: torch's biased
// variance), then out = act(GN_a(x) + r).
__device__ __forceinline__ void pn_gn_stats(const float* __restrict__ x, int HW, int C, int c0, int cpg, float* red, float& mean,
                                            float& rstd, float eps) {
  const int n = HW * cpg;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += x[(size_t)(i / cpg) * C + c0 + i % cpg];
  mean = pn_block_sum(s, red) / (float)n;
  float q = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float d = x[(size_t)(i / cpg) * C + c0 + i % cpg] - mean;
    q += d * d;
  }
  rstd = rsqrtf(pn_block_sum(q, red) / (float)n + eps);
}

__global__ void __launch_bounds__(1024) pointnav_groupnorm_kernel(const float* __restrict__ x, const float* __restrict__ ga,
                                                                  const float* __restrict__ ba, const float* r, const float* __restrict__ y,
                                                                  const float* __restrict__ gb, const float* __restrict__ bb, int rmode,
                                                                  float* out32, __half* __restrict__ out16, int HW, int C, int G, float eps,
                                                                  int relu) {
  __shared__ float red[32];
  const int g = blockIdx.x, b = blockIdx.y, cpg = C / G, c0 = g * cpg;
  const size_t base = (size_t)b * HW * C;
  float ma, ra, mb = 0.f, rb = 0.f;
  pn_gn_stats(x + base, HW, C, c0, cpg, red, ma, ra, eps);
  if (rmode == 2) pn_gn_stats(y + base, HW, C, c0, cpg, red, mb, rb, eps);
  const int n = HW * cpg;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = c0 + i % cpg;
    const size_t o = base + (size_t)(i / cpg) * C + c;
    float v = (x[o] - ma) * ra * ga[c] + ba[c];
    if (rmode == 1) v += r[o];
    else if (rmode == 2) v += (y[o] - mb) * rb * gb[c] + bb[c];
    if (relu) v = fmaxf(v, 0.f);
    if (out32) out32[o] = v;
    if (out16) out16[o] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------------ pool and gather
__global__ void pointnav_maxpool3s2_kernel(const float* __restrict__ x, float* __restrict__ out32, __half* __restrict__ out16, int B,
                                           int H, int W, int C, int Ho, int Wo) {
  const long long n = (long long)B * Ho * Wo * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int xo = (int)(r % Wo), yo = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    float m = -INFINITY;
    for (int dy = 0; dy < 3; ++dy)
      for (int dx = 0; dx < 3; ++dx) {
        const int yy = 2 * yo - 1 + dy, xx = 2 * xo - 1 + dx;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) m = fmaxf(m, x[(((size_t)b * H + yy) * W + xx) * C + c]);
      }
    if (out32) out32[i] = m;
    if (out16) out16[i] = __float2half_rn(m);
  }
}

// 8 fp16 (16 bytes) per thread: C % 8 == 0.
__global__ void pointnav_gather_s2_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int C8, int Ho,
                                          int Wo) {
  const long long n = (long long)B * Ho * Wo * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C8);
    const long long r = i / C8;
    const int xo = (int)(r % Wo), yo = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    out[i] = x[(((size_t)b * H + 2 * yo) * W + 2 * xo) * C8 + c];
  }
}

// ---------------------------------------------------------------------------------------------------------------- GEMV
// y[b, n] = act(sum_k x[b, k] W[n, k] + bias[n]) for b < B <= NB.  Warp w of CTA c owns row n = c * gemv_rows<NB>() + w; lane l sums
// k = 4 l + 128 j (+0..3) of every K chunk in k order into one accumulator per environment, then a fixed shuffle tree adds the
// lanes.  So each (b, n) is summed in an order that depends on K only: bitwise the same for any B and NB.
template <int NB>
__global__ void __launch_bounds__(gemv_rows<NB>() * 32) pointnav_gemv_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ Wt,
                                                                       int ldw, const float* __restrict__ bias, float* __restrict__ y,
                                                                       int ldy, int B, int N, int K, int relu) {
  extern __shared__ float4 xs[];   // [NB][GEMV_KC / 4]
  constexpr int KC4 = GEMV_KC / 4;
  const int lane = threadIdx.x & 31, n = blockIdx.x * gemv_rows<NB>() + (threadIdx.x >> 5);
  float acc[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) acc[b] = 0.f;
  const float4* wrow = reinterpret_cast<const float4*>(Wt + (size_t)(n < N ? n : 0) * ldw);
  for (int k0 = 0; k0 < K; k0 += GEMV_KC) {
    float4 w[GEMV_KC / 128];
#pragma unroll
    for (int j = 0; j < GEMV_KC / 128; ++j) {
      const int k = k0 + j * 128 + lane * 4;
      w[j] = (n < N && k < K) ? __ldg(wrow + k / 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NB * KC4; i += blockDim.x) {
      const int b = i / KC4, k = k0 + (i % KC4) * 4;
      xs[i] = (b < B && k < K) ? *reinterpret_cast<const float4*>(x + (size_t)b * ldx + k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < GEMV_KC / 128; ++j) {
      if (k0 + j * 128 + lane * 4 >= K) break;
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 v = xs[b * KC4 + j * 32 + lane];
        float a = acc[b];
        a = __fmaf_rn(w[j].x, v.x, a);
        a = __fmaf_rn(w[j].y, v.y, a);
        a = __fmaf_rn(w[j].z, v.z, a);
        a = __fmaf_rn(w[j].w, v.w, a);
        acc[b] = a;
      }
    }
  }
  if (n >= N) return;
  const float bn = bias ? bias[n] : 0.f;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float s = acc[b];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (b < B && lane == (b & 31)) {
      s += bn;
      y[(size_t)b * ldy + n] = relu ? fmaxf(s, 0.f) : s;
    }
  }
}

template <int NB>
static int pn_gemv_launch(const float* x, int ldx, const float* Wt, int ldw, const float* bias, float* y, int ldy, int B, int N, int K,
                          int relu, cudaStream_t st) {
  const size_t smem = (size_t)NB * GEMV_KC * sizeof(float);
  static bool configured = false;
  if (!configured && smem > 48 * 1024) {
    int rc = check_cuda(cudaFuncSetAttribute(pointnav_gemv_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                        "cudaFuncSetAttribute(pointnav_gemv_kernel)");
    if (rc) return rc;
  }
  configured = true;
  constexpr int rows = gemv_rows<NB>();
  pointnav_gemv_kernel<NB><<<(N + rows - 1) / rows, rows * 32, smem, st>>>(x, ldx, Wt, ldw, bias, y, ldy, B, N, K, relu);
  PN_LAUNCHED("pointnav_gemv_kernel");
  return VLFM_OK;
}

// ---------------------------------------------------------------------------------------------------------------- LSTM
// One CTA of PN_HID threads per environment b (state slot e = env_ids[b]).
__global__ void __launch_bounds__(PN_HID) pointnav_lstm_prep_kernel(const int32_t* __restrict__ env_ids, const float* __restrict__ state,
                                                                   const void* __restrict__ prev, int discrete, const uint8_t* __restrict__ masks,
                                                                   const float* __restrict__ goal, const float* __restrict__ w_goal,
                                                                   const float* __restrict__ b_goal, const float* __restrict__ w_prev,
                                                                   const float* __restrict__ b_prev, float* __restrict__ xin0,
                                                                   float* __restrict__ xin1, float* __restrict__ cbuf) {
  const int b = blockIdx.x, j = threadIdx.x, e = env_ids[b];
  const bool m = masks[b] != 0;
  const float* s = state + (size_t)e * 4 * PN_HID;
  // hidden state [h_l0, h_l1, c_l0, c_l1], zeroed where the mask is False (rnn_state_encoder.py:60)
  xin0[(size_t)b * PN_LD0 + PN_VIS + 2 * PN_EMB + j] = m ? s[j] : 0.f;
  xin1[(size_t)b * PN_LD1 + PN_HID + j] = m ? s[PN_HID + j] : 0.f;
  cbuf[(size_t)b * 2 * PN_HID + j] = m ? s[2 * PN_HID + j] : 0.f;
  cbuf[(size_t)b * 2 * PN_HID + PN_HID + j] = m ? s[3 * PN_HID + j] : 0.f;
  float* row = xin0 + (size_t)b * PN_LD0 + PN_VIS;
  if (j < PN_EMB) {
    // tgt_embeding(rho, cos(-theta), sin(-theta))
    const float rho = goal[2 * b], th = -goal[2 * b + 1];
    const float c = cosf(th), sn = sinf(th);
    const float* w = w_goal + 3 * j;
    row[j] = ((w[0] * rho + w[1] * c) + w[2] * sn) + b_goal[j];
  } else if (j < 2 * PN_EMB) {
    const int t = j - PN_EMB;
    float v;
    if (discrete) {
      // nn.Embedding(5, 32) at where(mask, prev + 1, 0)
      long long a = m ? static_cast<const long long*>(prev)[e] + 1 : 0;
      a = a < 0 ? 0 : (a > 4 ? 4 : a);
      v = w_prev[a * PN_EMB + t];
    } else {
      // Linear(2 -> 32) of mask * prev
      const float* p = static_cast<const float*>(prev) + 2 * e;
      const float p0 = m ? p[0] : 0.f, p1 = m ? p[1] : 0.f;
      v = (w_prev[2 * t] * p0 + w_prev[2 * t + 1] * p1) + b_prev[t];
    }
    row[j] = v;
  }
}

// PyTorch's gate order i, f, g, o: c' = f c + i g, h' = o tanh(c').
__device__ __forceinline__ void pn_cell(const float* g, float c, float& h_out, float& c_out) {
  const int j = threadIdx.x;
  const float i = pn_sigmoid(g[j]), f = pn_sigmoid(g[PN_HID + j]), gg = tanhf(g[2 * PN_HID + j]), o = pn_sigmoid(g[3 * PN_HID + j]);
  c_out = f * c + i * gg;
  h_out = o * tanhf(c_out);
}

// Layer 0: h0' -> xin1[:, 0:512] (the layer-1 GEMV input), c0' -> cbuf[:, 0:512] in place.
__global__ void __launch_bounds__(PN_HID) pointnav_lstm_cell_kernel(const float* __restrict__ gates, float* __restrict__ cbuf,
                                                                   float* __restrict__ xin1) {
  const int b = blockIdx.x, j = threadIdx.x;
  float h, c;
  pn_cell(gates + (size_t)b * 4 * PN_HID, cbuf[(size_t)b * 2 * PN_HID + j], h, c);
  cbuf[(size_t)b * 2 * PN_HID + j] = c;
  xin1[(size_t)b * PN_LD1 + j] = h;
}

// Layer 1, the head and the write-back: features h1' -> d_feat; head outputs (4: logits, or mu | log_std) -> d_head; the action
// (argmax, first index on ties: int64; or tanh(mu): float32 x 2) -> d_action and the previous-action slot; [h0', h1', c0', c1']
// -> the state slot.
__global__ void __launch_bounds__(PN_HID) pointnav_lstm_head_kernel(const float* __restrict__ gates, const float* __restrict__ cbuf,
                                                                   const float* __restrict__ xin1, const float* __restrict__ w_head,
                                                                   const float* __restrict__ b_head, int discrete,
                                                                   const int32_t* __restrict__ env_ids, float* __restrict__ state,
                                                                   void* __restrict__ prev, float* __restrict__ feat,
                                                                   float* __restrict__ head, void* __restrict__ action) {
  __shared__ float h1s[PN_HID];
  __shared__ float outs[4];
  const int b = blockIdx.x, j = threadIdx.x, e = env_ids[b];
  float h, c;
  pn_cell(gates + (size_t)b * 4 * PN_HID, cbuf[(size_t)b * 2 * PN_HID + PN_HID + j], h, c);
  h1s[j] = h;
  if (feat) feat[(size_t)b * PN_HID + j] = h;
  float* s = state + (size_t)e * 4 * PN_HID;
  s[j] = xin1[(size_t)b * PN_LD1 + j];
  s[PN_HID + j] = h;
  s[2 * PN_HID + j] = cbuf[(size_t)b * 2 * PN_HID + j];
  s[3 * PN_HID + j] = c;
  __syncthreads();
  const int w = j >> 5, lane = j & 31;
  if (w < 4) {
    float a = 0.f;
    for (int k = lane; k < PN_HID; k += 32) a = __fmaf_rn(w_head[w * PN_HID + k], h1s[k], a);
#pragma unroll
    for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) outs[w] = a + b_head[w];
  }
  __syncthreads();
  if (j == 0) {
    if (head) for (int k = 0; k < 4; ++k) head[(size_t)b * 4 + k] = outs[k];
    if (discrete) {
      int best = 0;
      for (int k = 1; k < 4; ++k) if (outs[k] > outs[best]) best = k;
      static_cast<long long*>(action)[b] = best;
      static_cast<long long*>(prev)[e] = best;
    } else {
      const float a0 = tanhf(outs[0]), a1 = tanhf(outs[1]);
      static_cast<float*>(action)[2 * b] = a0;
      static_cast<float*>(action)[2 * b + 1] = a1;
      static_cast<float*>(prev)[2 * e] = a0;
      static_cast<float*>(prev)[2 * e + 1] = a1;
    }
  }
}

}  // namespace vlfm

using namespace vlfm;

static bool pn_aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int vlfm_pointnav_depth_in(const float* d_depth, int B, int H, int W, int IH, int IW, void* d_col16, int ldk, float* d_resized,
                                      void* stream) {
  if (!d_depth || !d_col16 || B < 1 || H < 1 || W < 1 || IH < 2 || IW < 2 || ldk < 49 || (ldk & 7)) {
    set_error("vlfm_pointnav_depth_in: bad argument"); return VLFM_E_INVALID; }
  const int PH = IH / 2, PW = IW / 2, OH = (PH - 1) / 2 + 1, OW = (PW - 1) / 2 + 1;
  const size_t smem = (size_t)7 * PW * sizeof(float);
  if (smem > 48 * 1024) { set_error("vlfm_pointnav_depth_in: input width %d too large for the pooled-row staging", IW); return VLFM_E_INVALID; }
  pointnav_depth_in_kernel<<<dim3(OH, B), 256, smem, (cudaStream_t)stream>>>(d_depth, H, W, IH, IW, PH, PW, OH, OW, (__half*)d_col16,
                                                                             ldk, d_resized);
  PN_LAUNCHED("pointnav_depth_in_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_groupnorm(const float* d_x, const float* d_gamma_a, const float* d_beta_a, int rmode, const float* d_r,
                                       const float* d_y, const float* d_gamma_b, const float* d_beta_b, float* d_out32, void* d_out16,
                                       int B, int HW, int C, int G, float eps, int relu, void* stream) {
  if (!d_x || !d_gamma_a || !d_beta_a || B < 1 || HW < 1 || C < 1 || G < 1 || C % G || (!d_out32 && !d_out16) || rmode < 0 || rmode > 2 ||
      (rmode == 1 && !d_r) || (rmode == 2 && (!d_y || !d_gamma_b || !d_beta_b)) || B > 65535 || G > 65535) {
    set_error("vlfm_pointnav_groupnorm: bad argument"); return VLFM_E_INVALID; }
  pointnav_groupnorm_kernel<<<dim3(G, B), 1024, 0, (cudaStream_t)stream>>>(d_x, d_gamma_a, d_beta_a, d_r, d_y, d_gamma_b, d_beta_b,
                                                                           rmode, d_out32, (__half*)d_out16, HW, C, G, eps, relu);
  PN_LAUNCHED("pointnav_groupnorm_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_maxpool3s2(const float* d_x, float* d_out32, void* d_out16, int B, int H, int W, int C, void* stream) {
  if (!d_x || (!d_out32 && !d_out16) || B < 1 || H < 1 || W < 1 || C < 1) {
    set_error("vlfm_pointnav_maxpool3s2: bad argument"); return VLFM_E_INVALID; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  pointnav_maxpool3s2_kernel<<<pn_grid((long long)B * Ho * Wo * C, 256), 256, 0, (cudaStream_t)stream>>>(d_x, d_out32, (__half*)d_out16,
                                                                                                          B, H, W, C, Ho, Wo);
  PN_LAUNCHED("pointnav_maxpool3s2_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_gather_s2(const void* d_x16, void* d_out16, int B, int H, int W, int C, void* stream) {
  if (!d_x16 || !d_out16 || B < 1 || H < 1 || W < 1 || C < 8 || (C & 7) || !pn_aligned16(d_x16) || !pn_aligned16(d_out16)) {
    set_error("vlfm_pointnav_gather_s2: bad argument"); return VLFM_E_INVALID; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  pointnav_gather_s2_kernel<<<pn_grid((long long)B * Ho * Wo * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)d_x16, (uint4*)d_out16, B, H, W, C / 8, Ho, Wo);
  PN_LAUNCHED("pointnav_gather_s2_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_gemv_f32(const float* d_x, int ldx, const float* d_W, int ldw, const float* d_bias, float* d_y, int ldy,
                                      int B, int N, int K, int relu, void* stream) {
  if (!d_x || !d_W || !d_y || B < 1 || B > GEMV_MAXB || N < 1 || K < 4 || (K & 3) || (ldx & 3) || (ldw & 3) || ldx < K || ldw < K ||
      ldy < N || !pn_aligned16(d_x) || !pn_aligned16(d_W)) {
    set_error("vlfm_pointnav_gemv_f32: bad argument (B <= %d; K, ldx, ldw multiples of 4; x, W 16-byte aligned)", GEMV_MAXB);
    return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (B <= 1) return pn_gemv_launch<1>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  if (B <= 2) return pn_gemv_launch<2>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  if (B <= 4) return pn_gemv_launch<4>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  if (B <= 8) return pn_gemv_launch<8>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  if (B <= 16) return pn_gemv_launch<16>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  if (B <= 32) return pn_gemv_launch<32>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
  return pn_gemv_launch<64>(d_x, ldx, d_W, ldw, d_bias, d_y, ldy, B, N, K, relu, st);
}

extern "C" int vlfm_pointnav_lstm_prep(const int32_t* d_env_ids, const float* d_state, const void* d_prev, int discrete,
                                       const uint8_t* d_masks, const float* d_goal, const float* d_w_goal, const float* d_b_goal,
                                       const float* d_w_prev, const float* d_b_prev, float* d_xin0, float* d_xin1, float* d_cbuf, int B,
                                       void* stream) {
  if (!d_env_ids || !d_state || !d_prev || !d_masks || !d_goal || !d_w_goal || !d_b_goal || !d_w_prev || (!discrete && !d_b_prev) ||
      !d_xin0 || !d_xin1 || !d_cbuf || B < 1 || B > 65535) {
    set_error("vlfm_pointnav_lstm_prep: bad argument"); return VLFM_E_INVALID; }
  pointnav_lstm_prep_kernel<<<B, PN_HID, 0, (cudaStream_t)stream>>>(d_env_ids, d_state, d_prev, discrete, d_masks, d_goal, d_w_goal,
                                                                    d_b_goal, d_w_prev, d_b_prev, d_xin0, d_xin1, d_cbuf);
  PN_LAUNCHED("pointnav_lstm_prep_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_lstm_cell(const float* d_gates, float* d_cbuf, float* d_xin1, int B, void* stream) {
  if (!d_gates || !d_cbuf || !d_xin1 || B < 1 || B > 65535) { set_error("vlfm_pointnav_lstm_cell: bad argument"); return VLFM_E_INVALID; }
  pointnav_lstm_cell_kernel<<<B, PN_HID, 0, (cudaStream_t)stream>>>(d_gates, d_cbuf, d_xin1);
  PN_LAUNCHED("pointnav_lstm_cell_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_pointnav_lstm_head(const float* d_gates, const float* d_cbuf, const float* d_xin1, const float* d_w_head,
                                       const float* d_b_head, int discrete, const int32_t* d_env_ids, float* d_state, void* d_prev,
                                       float* d_feat, float* d_head, void* d_action, int B, void* stream) {
  if (!d_gates || !d_cbuf || !d_xin1 || !d_w_head || !d_b_head || !d_env_ids || !d_state || !d_prev || !d_action || B < 1 || B > 65535) {
    set_error("vlfm_pointnav_lstm_head: bad argument"); return VLFM_E_INVALID; }
  pointnav_lstm_head_kernel<<<B, PN_HID, 0, (cudaStream_t)stream>>>(d_gates, d_cbuf, d_xin1, d_w_head, d_b_head, discrete, d_env_ids,
                                                                    d_state, d_prev, d_feat, d_head, d_action);
  PN_LAUNCHED("pointnav_lstm_head_kernel");
  return VLFM_OK;
}
