// GroundingDINO model-level kernels that are not inside an encoder / decoder layer (vlfm_b200/vlm/gdino_forward.py):
// neck GroupNorm on NHWC rows (the fourth level's 3x3 stride-2 conv is vlfm_im2col_f16 plus the GEMM), two-stage proposal
// scoring, language-guided top-k query selection, row gather, box / class heads.
//
// Reference: groundingdino ... `model(image, captions=[caption])` called from vlfm/vlm/grounding_dino.py:61-67; the restated
// module graph is HF `GroundingDinoModel.forward` (input_proj_vision, generate_encoder_output_proposals, encoder_output_class_embed,
// torch.topk, torch.gather) and `GroundingDinoForObjectDetection.forward` (class_embed / bbox_embed of the last decoder layer),
// followed by the `.sigmoid()` of groundingdino.util.inference.predict.
#include <math.h>

#include "common.cuh"

namespace vlfm {

// ------------------------------------------------------------------------------------- GroupNorm ----
// y [B, HW, C] fp32 rows (the 1x1 / 3x3 conv output as a row GEMM), `groups` groups of C/groups consecutive channels; statistics
// over (HW x C/groups) per (image, group) -- torch.nn.GroupNorm on the NCHW tensor -- two-pass in fp32; the result is written
// into the flattened encoder input out[b, row_off + i, :] (row stride C, image stride S*C).  One block per (image, group).
__global__ void __launch_bounds__(256)
groupnorm_rows_kernel(const float* __restrict__ y, int HW, int C, int groups, const float* __restrict__ gamma, const float* __restrict__ beta,
                      float eps, float* __restrict__ out, int row_off, int S) {
  const int b = blockIdx.y, g = blockIdx.x, cpg = C / groups, tid = threadIdx.x;
  const float* base = y + (size_t)b * HW * C + g * cpg;
  const int n = HW * cpg;
  __shared__ float red[8];
  __shared__ float s_mean, s_rstd;
  float s = 0.f;
  for (int i = tid; i < n; i += 256) { const int r = i / cpg, c = i - r * cpg; s += base[(size_t)r * C + c]; }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) { float t = 0.f; for (int i = 0; i < 8; ++i) t += red[i]; s_mean = t / (float)n; }
  __syncthreads();
  const float mean = s_mean;
  float q = 0.f;
  for (int i = tid; i < n; i += 256) { const int r = i / cpg, c = i - r * cpg; const float d = base[(size_t)r * C + c] - mean; q += d * d; }
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  __syncthreads();
  if ((tid & 31) == 0) red[tid >> 5] = q;
  __syncthreads();
  if (tid == 0) { float t = 0.f; for (int i = 0; i < 8; ++i) t += red[i]; s_rstd = rsqrtf(t / (float)n + eps); }
  __syncthreads();
  const float rstd = s_rstd;
  float* ob = out + ((size_t)b * S + row_off) * C + g * cpg;
  for (int i = tid; i < n; i += 256) {
    const int r = i / cpg, c = i - r * cpg;
    ob[(size_t)r * C + c] = (base[(size_t)r * C + c] - mean) * rstd * gamma[g * cpg + c] + beta[g * cpg + c];
  }
}

// fp32 rows -> fp16 GEMM operand with invalid rows zeroed (object_query.masked_fill(~output_proposals_valid, 0))
__global__ void mask_rows_f16_kernel(const float* __restrict__ x, const uint8_t* __restrict__ valid, __half* __restrict__ out, long rows, int D) {
  const long total = rows * (D / 4);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (D / 4);
    float4 v = valid[r] ? *reinterpret_cast<const float4*>(x + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
    __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    *reinterpret_cast<uint2*>(out + 4 * i) = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
  }
}

// ------------------------------------------------------------------------------- proposal scores ----
// score[b, s] = max_t <q[b, s, :], text[b, t, :]>   (encoder_output_class_embed + max(-1); every token valid).  One warp per
// proposal row, the image's text features staged in shared memory; D <= 256, T <= 256.
__global__ void __launch_bounds__(256)
proposal_scores_kernel(const float* __restrict__ q, const float* __restrict__ text, int S, int T, int D, float* __restrict__ scores) {
  extern __shared__ float s_text[];                  // [T, D]
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < T * D; i += blockDim.x) s_text[i] = text[(size_t)b * T * D + i];
  __syncthreads();
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int s = blockIdx.x * wpb + (threadIdx.x >> 5); s < S; s += gridDim.x * wpb) {
    const float* row = q + ((size_t)b * S + s) * D;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = lane + 32 * j < D ? row[lane + 32 * j] : 0.f;
    float best = -INFINITY;
    for (int t = 0; t < T; ++t) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) if (lane + 32 * j < D) acc += v[j] * s_text[t * D + lane + 32 * j];
      for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      best = fmaxf(best, acc);
    }
    if (lane == 0) scores[(size_t)b * S + s] = best;
  }
}

// ------------------------------------------------------------------------------------------ top-k ----
// per image: indices of the k largest scores, descending (ties: lower index first).  One block, bitonic sort of the next power of
// two >= S (<= 16384) (key, index) pairs in shared memory.
__global__ void __launch_bounds__(1024)
topk_rows_kernel(const float* __restrict__ scores, int S, int P, int k, long long* __restrict__ idx_out) {
  extern __shared__ unsigned long long s_keys[];     // P entries: (ordered score bits << 32) | (0xffffffff - index): descending sort
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < P; i += 1024) {
    unsigned long long key = 0ull;
    if (i < S) {
      float f = scores[(size_t)b * S + i];
      if (f != f) f = -INFINITY;                       // NaN sorts last
      unsigned u = __float_as_uint(f);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // monotone map float -> unsigned
      key = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    }
    s_keys[i] = key;
  }
  __syncthreads();
  for (int kk = 2; kk <= P; kk <<= 1)
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += 1024) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = s_keys[i], c = s_keys[ixj];
          const bool desc = (i & kk) == 0;
          if ((a < c) == desc) { s_keys[i] = c; s_keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < k; i += 1024) idx_out[(size_t)b * k + i] = (long long)(0xffffffffu - (unsigned)(s_keys[i] & 0xffffffffull));
}

// S > 16384 (1024 x 1024 frames have 21760 proposals): the keys do not fit one block's shared memory.  Radix-select the k-th largest
// 64-bit key (8 passes of 8 bits over the scores in global memory; the keys are unique, so exactly k of them are >= the k-th),
// collect those k into shared memory and bitonic-sort them.  Same order as topk_rows_kernel: descending score, lower index first.
__device__ __forceinline__ unsigned long long topk_key(const float* __restrict__ row, int i) {
  float f = row[i];
  if (f != f) f = -INFINITY;
  unsigned u = __float_as_uint(f);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
}
__global__ void __launch_bounds__(1024)
topk_select_kernel(const float* __restrict__ scores, int S, int P, int k, long long* __restrict__ idx_out) {
  extern __shared__ unsigned long long s_keys[];     // P >= k entries
  __shared__ unsigned s_hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ unsigned s_need, s_fill;
  const float* row = scores + (size_t)blockIdx.x * S;
  if (threadIdx.x == 0) { s_prefix = 0ull; s_need = (unsigned)k; s_fill = 0u; }
  for (int pass = 0; pass < 8; ++pass) {
    const int shift = 56 - 8 * pass;
    if (threadIdx.x < 256) s_hist[threadIdx.x] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long hi_mask = pass ? (~0ull << (shift + 8)) : 0ull;
    for (int i = threadIdx.x; i < S; i += 1024) {
      const unsigned long long key = topk_key(row, i);
      if ((key & hi_mask) == prefix) atomicAdd(&s_hist[(unsigned)(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned need = s_need, d = 255;
      for (;; --d) { const unsigned c = s_hist[d]; if (c >= need) break; need -= c; }   // some digit holds the need-th largest
      s_need = need;
      s_prefix = prefix | ((unsigned long long)d << shift);
    }
    __syncthreads();
  }
  const unsigned long long kth = s_prefix;
  for (int i = threadIdx.x; i < P; i += 1024) s_keys[i] = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < S; i += 1024) {
    const unsigned long long key = topk_key(row, i);
    if (key >= kth) s_keys[atomicAdd(&s_fill, 1u)] = key;
  }
  __syncthreads();
  for (int kk = 2; kk <= P; kk <<= 1)
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += 1024) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = s_keys[i], c = s_keys[ixj];
          const bool desc = (i & kk) == 0;
          if ((a < c) == desc) { s_keys[i] = c; s_keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < k; i += 1024) idx_out[(size_t)blockIdx.x * k + i] = (long long)(0xffffffffu - (unsigned)(s_keys[i] & 0xffffffffull));
}

// ------------------------------------------------------------------------- decoder query positions ----
// GroundingDinoDecoder.forward, per layer:  reference_points_input = ref[:, :, None] * cat([valid_ratios, valid_ratios], -1)[:, None]
// and get_sine_pos_embed(reference_points_input[:, :, 0, :], num_pos_feats = P): for every coordinate c and j < P
//   v = c * 2*pi / dim_t[j];  e[j] = j even ? sin(v) : cos(v);   output order (y, x, w, h) x P  (exchange_xy).
// One launch instead of ~30 elementwise ones (mul, div, pow, sin, cos, stack, cat per coordinate).  IEEE mul / div in the
// reference's order, sinf / cosf as torch's CUDA kernels use them; dim_t is computed by the caller with the reference's own expression.
__global__ void __launch_bounds__(128)
decoder_query_pos_kernel(const float* __restrict__ ref, const float* __restrict__ vr, const float* __restrict__ dim_t, int nq, int L, int P,
                         float* __restrict__ ref_in, __half* __restrict__ embed) {
  const int row = blockIdx.x, b = row / nq;
  const float4 r = *reinterpret_cast<const float4*>(ref + (size_t)row * 4);
  const float* v = vr + (size_t)b * L * 2;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    const float vx = v[2 * l], vy = v[2 * l + 1];
    *reinterpret_cast<float4*>(ref_in + ((size_t)row * L + l) * 4) = make_float4(__fmul_rn(r.x, vx), __fmul_rn(r.y, vy), __fmul_rn(r.z, vx), __fmul_rn(r.w, vy));
  }
  const float c[4] = {__fmul_rn(r.y, v[1]), __fmul_rn(r.x, v[0]), __fmul_rn(r.z, v[0]), __fmul_rn(r.w, v[1])};   // (y, x, w, h) of level 0
  __half* e = embed + (size_t)row * 4 * P;
  for (int j = threadIdx.x; j < P; j += blockDim.x) {
    const float dt = dim_t[j];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = __fdiv_rn(__fmul_rn(c[k], 6.283185307179586f), dt);
      e[k * P + j] = __float2half_rn((j & 1) ? cosf(a) : sinf(a));
    }
  }
}

// dst[b, i, :] = src[b, idx[b, i], :]
__global__ void gather_rows_kernel(const float* __restrict__ src, const long long* __restrict__ idx, int S, int K, int C, float* __restrict__ dst) {
  const int b = blockIdx.y;
  const long total = (long)K * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int r = (int)(i / C), c = (int)(i - (long)r * C);
    dst[((size_t)b * K + r) * C + c] = src[((size_t)b * S + idx[(size_t)b * K + r]) * C + c];
  }
}

// boxes = sigmoid(delta + logit(ref, eps = 1e-5))   (torch.special.logit clamps ref to [eps, 1 - eps])
__global__ void box_finish_kernel(const float* __restrict__ delta, const float* __restrict__ ref, float* __restrict__ out, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float r = fminf(fmaxf(ref[i], 1e-5f), 1.f - 1e-5f);
    const float z = delta[i] + logf(r / (1.f - r));
    out[i] = 1.f / (1.f + expf(-z));
  }
}

// logits[b, q, t] = sigmoid(<hs[b, q, :], text[b, t, :]>) for t < T, 0 for T <= t < L (sigmoid of the -inf padding)
__global__ void __launch_bounds__(256)
contrastive_sigmoid_kernel(const float* __restrict__ hs, const float* __restrict__ text, int Q, int T, int D, int L, float* __restrict__ out) {
  extern __shared__ float s_text[];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < T * D; i += blockDim.x) s_text[i] = text[(size_t)b * T * D + i];
  __syncthreads();
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int qi = blockIdx.x * wpb + (threadIdx.x >> 5); qi < Q; qi += gridDim.x * wpb) {
    const float* row = hs + ((size_t)b * Q + qi) * D;
    float* o = out + ((size_t)b * Q + qi) * L;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = lane + 32 * j < D ? row[lane + 32 * j] : 0.f;
    for (int t = 0; t < T; ++t) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) if (lane + 32 * j < D) acc += v[j] * s_text[t * D + lane + 32 * j];
      for (int o2 = 16; o2; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
      if (lane == 0) o[t] = 1.f / (1.f + expf(-acc));
    }
    for (int t = T + lane; t < L; t += 32) o[t] = 0.f;
  }
}

}  // namespace vlfm

using namespace vlfm;

static inline int nb(long n, int t = 256, int cap = 4736) { long b = (n + t - 1) / t; return (int)(b < 1 ? 1 : (b > cap ? cap : b)); }

extern "C" int vlfm_groupnorm_rows(const float* d_y, int B, int HW, int C, int groups, const float* d_gamma, const float* d_beta, float eps,
                                   float* d_out, int row_off, int S, void* stream) {
  if (!d_y || !d_gamma || !d_beta || !d_out || B < 1 || HW < 1 || C < 1 || groups < 1 || C % groups || B > 65535 || row_off < 0 || row_off + HW > S) {
    set_error("vlfm_groupnorm_rows: bad argument"); return VLFM_E_INVALID; }
  groupnorm_rows_kernel<<<dim3(groups, B), 256, 0, (cudaStream_t)stream>>>(d_y, HW, C, groups, d_gamma, d_beta, eps, d_out, row_off, S);
  VLFM_CHECK_LAUNCH("groupnorm_rows_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_mask_rows_f16(const float* d_x, const uint8_t* d_valid, void* d_out16, long rows, int D, void* stream) {
  if (!d_x || !d_valid || !d_out16 || rows < 1 || D < 4 || (D & 3)) { set_error("vlfm_mask_rows_f16: bad argument (D %% 4)"); return VLFM_E_INVALID; }
  mask_rows_f16_kernel<<<nb(rows * (D / 4)), 256, 0, (cudaStream_t)stream>>>(d_x, d_valid, (__half*)d_out16, rows, D);
  VLFM_CHECK_LAUNCH("mask_rows_f16_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_proposal_scores(const float* d_q, const float* d_text, int B, int S, int T, int D, float* d_scores, void* stream) {
  if (!d_q || !d_text || !d_scores || B < 1 || S < 1 || T < 1 || D < 1 || D > 256 || B > 65535 || (size_t)T * D * 4 > 200 * 1024) {
    set_error("vlfm_proposal_scores: bad argument (D <= 256, T*D*4 <= 200 KB)"); return VLFM_E_INVALID; }
  const size_t smem = (size_t)T * D * 4;
  static size_t cfg = 0;
  if (smem > 48 * 1024 && smem > cfg) {
    int rc = check_cuda(cudaFuncSetAttribute(proposal_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(proposal_scores)");
    if (rc) return rc; cfg = smem;
  }
  int bx = (S + 7) / 8; if (bx > 264) bx = 264;
  proposal_scores_kernel<<<dim3(bx, B), 256, smem, (cudaStream_t)stream>>>(d_q, d_text, S, T, D, d_scores);
  VLFM_CHECK_LAUNCH("proposal_scores_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_topk_rows(const float* d_scores, int B, int S, int k, long long* d_idx, void* stream) {
  if (!d_scores || !d_idx || B < 1 || S < 1 || k < 1 || k > S || (S > 16384 && k > 16384)) { set_error("vlfm_topk_rows: bad argument (k <= S; k <= 16384 when S > 16384)"); return VLFM_E_INVALID; }
  if (S > 16384) {
    int P = 2; while (P < k) P <<= 1;
    const size_t smem = (size_t)P * 8;
    static size_t cfg2 = 0;
    if (smem > 48 * 1024 && smem > cfg2) {
      int rc = check_cuda(cudaFuncSetAttribute(topk_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(topk_select)");
      if (rc) return rc; cfg2 = smem;
    }
    topk_select_kernel<<<B, 1024, smem, (cudaStream_t)stream>>>(d_scores, S, P, k, d_idx);
    VLFM_CHECK_LAUNCH("topk_select_kernel");
    count_launch();
    return VLFM_OK;
  }
  int P = 2; while (P < S) P <<= 1;
  const size_t smem = (size_t)P * 8;
  static size_t cfg = 0;
  if (smem > 48 * 1024 && smem > cfg) {
    int rc = check_cuda(cudaFuncSetAttribute(topk_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(topk_rows)");
    if (rc) return rc; cfg = smem;
  }
  topk_rows_kernel<<<B, 1024, smem, (cudaStream_t)stream>>>(d_scores, S, P, k, d_idx);
  VLFM_CHECK_LAUNCH("topk_rows_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_decoder_query_pos(const float* d_ref, const float* d_valid_ratios, const float* d_dim_t, int B, int nq, int L, int P,
                                      float* d_ref_in, void* d_embed16, void* stream) {
  if (!d_ref || !d_valid_ratios || !d_dim_t || !d_ref_in || !d_embed16 || B < 1 || nq < 1 || L < 1 || P < 1 || ((uintptr_t)d_ref & 15) || ((uintptr_t)d_ref_in & 15)) {
    set_error("vlfm_decoder_query_pos: bad argument"); return VLFM_E_INVALID; }
  decoder_query_pos_kernel<<<B * nq, 128, 0, (cudaStream_t)stream>>>(d_ref, d_valid_ratios, d_dim_t, nq, L, P, d_ref_in, (__half*)d_embed16);
  VLFM_CHECK_LAUNCH("decoder_query_pos_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_gather_rows(const float* d_src, const long long* d_idx, int B, int S, int K, int C, float* d_dst, void* stream) {
  if (!d_src || !d_idx || !d_dst || B < 1 || S < 1 || K < 1 || C < 1 || B > 65535) { set_error("vlfm_gather_rows: bad argument"); return VLFM_E_INVALID; }
  gather_rows_kernel<<<dim3(nb((long)K * C, 256, 512), B), 256, 0, (cudaStream_t)stream>>>(d_src, d_idx, S, K, C, d_dst);
  VLFM_CHECK_LAUNCH("gather_rows_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_box_finish(const float* d_delta, const float* d_ref, float* d_out, long n, void* stream) {
  if (!d_delta || !d_ref || !d_out || n < 1) { set_error("vlfm_box_finish: bad argument"); return VLFM_E_INVALID; }
  box_finish_kernel<<<nb(n), 256, 0, (cudaStream_t)stream>>>(d_delta, d_ref, d_out, n);
  VLFM_CHECK_LAUNCH("box_finish_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_contrastive_sigmoid(const float* d_hs, const float* d_text, int B, int Q, int T, int D, int L, float* d_out, void* stream) {
  if (!d_hs || !d_text || !d_out || B < 1 || Q < 1 || T < 1 || T > L || D < 1 || D > 256 || B > 65535 || (size_t)T * D * 4 > 200 * 1024) {
    set_error("vlfm_contrastive_sigmoid: bad argument"); return VLFM_E_INVALID; }
  const size_t smem = (size_t)T * D * 4;
  static size_t cfg = 0;
  if (smem > 48 * 1024 && smem > cfg) {
    int rc = check_cuda(cudaFuncSetAttribute(contrastive_sigmoid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(contrastive_sigmoid)");
    if (rc) return rc; cfg = smem;
  }
  int bx = (Q + 7) / 8; if (bx > 132) bx = 132;
  contrastive_sigmoid_kernel<<<dim3(bx, B), 256, smem, (cudaStream_t)stream>>>(d_hs, d_text, Q, T, D, L, d_out);
  VLFM_CHECK_LAUNCH("contrastive_sigmoid_kernel");
  count_launch();
  return VLFM_OK;
}
