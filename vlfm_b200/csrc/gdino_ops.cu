// GroundingDINO feature-enhancer / decoder kernels that are not GEMMs.
//
// Replaces, on the path vlfm/vlm/grounding_dino.py:61-67 -> groundingdino ... MSDeformAttn, the third-party
// `ms_deform_attn_cuda.cu` gather (SURVEY 8f rank 1): multi-scale deformable attention
//   out[b,q,h,:] = sum_{l,p} w[b,q,h,l,p] * bilinear(value_l[b,:,h,:], loc[b,q,h,l,p])      (zeros padding,
// align_corners=False, exactly torch.nn.functional.grid_sample's unnormalisation).
#include "common.cuh"

namespace vlfm {

constexpr int MSDA_MAX_LEVELS = 8;
struct MsdaArgs {
  int B, S, Q, heads, hd, levels, points;
  int H[MSDA_MAX_LEVELS], W[MSDA_MAX_LEVELS], start[MSDA_MAX_LEVELS];
};

// Fused deformable attention for head_dim 32 / fp16 values.  One warp per (b, q, head).  Lanes 0-15 own one (level, point)
// pair each for the softmax and the location arithmetic; the gather runs with lane = (tap = lane >> 3, channel quad =
// lane & 7): all four bilinear taps of a point are ONE 8-byte load per lane, the taps are summed by two shuffles at the end.
template <int REF_DIM, int LEVELS, int POINTS>      // LEVELS == 0: runtime levels / points
__global__ void __launch_bounds__(256)
msda_fused_kernel(const __half* __restrict__ value, const float* __restrict__ offlog, int ld, int logit_col, const float* __restrict__ ref,
                  __half* __restrict__ out, MsdaArgs a) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long total = (long)a.B * a.Q * a.heads;
  if (warp >= total) return;
  const int h = (int)(warp % a.heads);
  const long bq = warp / a.heads;
  const int b = (int)(bq / a.Q);
  const int points = LEVELS ? POINTS : a.points;
  const int LP = LEVELS ? LEVELS * POINTS : a.levels * a.points;
  const float* row = offlog + (size_t)bq * ld;
  // ---- per-point quantities on lanes 0..LP-1: softmax weight, integer tap origin, bilinear fractions, level base
  float logit = -INFINITY, ax = 0.f, ay = 0.f;
  int x0 = -4, y0 = -4, Wl = 1, Hl = 1, lbase = 0;
  if (lane < LP) {
    const float2 off = __ldg(reinterpret_cast<const float2*>(row + (size_t)h * LP * 2) + lane);
    logit = __ldg(row + logit_col + h * LP + lane);
    const int l = lane / points;
    Wl = a.W[0]; Hl = a.H[0]; lbase = a.start[0];
#pragma unroll
    for (int k = 1; k < MSDA_MAX_LEVELS; ++k)          // constant indices only: a dynamic a.W[l] would copy the struct to local memory
      if (l >= k) { Wl = a.W[k]; Hl = a.H[k]; lbase = a.start[k]; }
    const float* rp = ref + ((size_t)bq * (LEVELS ? LEVELS : a.levels) + l) * REF_DIM;
    float lx, ly;
    if (REF_DIM == 2) {
      lx = __fadd_rn(__ldg(rp), __fdiv_rn(off.x, (float)Wl));
      ly = __fadd_rn(__ldg(rp + 1), __fdiv_rn(off.y, (float)Hl));
    } else {
      lx = __fadd_rn(__ldg(rp), __fmul_rn(__fmul_rn(__fdiv_rn(off.x, (float)points), __ldg(rp + 2)), 0.5f));
      ly = __fadd_rn(__ldg(rp + 1), __fmul_rn(__fmul_rn(__fdiv_rn(off.y, (float)points), __ldg(rp + 3)), 0.5f));
    }
    // HF: grid = 2*loc - 1 ; grid_sample: ((grid + 1) / 2) * size - 0.5   (no FMA contraction; /2 is exact)
    const float gx = __fsub_rn(__fmul_rn(2.f, lx), 1.f), gy = __fsub_rn(__fmul_rn(2.f, ly), 1.f);
    const float ix = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)Wl), 0.5f);
    const float iy = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)Hl), 0.5f);
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    ax = ix - fx0; ay = iy - fy0;
    // clamp far-away samples so the int conversion is defined; anything <= -2 or >= size contributes nothing
    x0 = (int)fminf(fmaxf(fx0, -4.f), 16384.f); y0 = (int)fminf(fmaxf(fy0, -4.f), 16384.f);
  }
  float mx = logit;
#pragma unroll
  for (int o = 8; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  mx = __shfl_sync(0xffffffffu, mx, 0);                 // lanes 16-31 hold -inf: take the low half's maximum
  const float e = lane < LP ? expf(logit - mx) : 0.f;
  float sum = e;
#pragma unroll
  for (int o = 8; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  sum = __shfl_sync(0xffffffffu, sum, 0);
  const float wgt = e / sum;
  // ---- gather: lane = (tap, channel quad)
  const int tap = lane >> 3, quad = lane & 7;
  const int tx = tap & 1, ty = tap >> 1;
  const __half* vb = value + (size_t)b * a.S * a.heads * 32 + (size_t)h * 32 + quad * 4;
  const size_t vstride = (size_t)a.heads * 32;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
#pragma unroll
  for (int j = 0; j < (LEVELS ? LEVELS * POINTS : 16); ++j) {
    if (!LEVELS && j >= LP) break;
    const float fx = __shfl_sync(0xffffffffu, ax, j), fy = __shfl_sync(0xffffffffu, ay, j), w = __shfl_sync(0xffffffffu, wgt, j);
    const int px = __shfl_sync(0xffffffffu, x0, j) + tx, py = __shfl_sync(0xffffffffu, y0, j) + ty;
    const int pw = __shfl_sync(0xffffffffu, Wl, j), ph = __shfl_sync(0xffffffffu, Hl, j), pb = __shfl_sync(0xffffffffu, lbase, j);
    const float bw = (tx ? fx : 1.f - fx) * (ty ? fy : 1.f - fy) * w;
    if (px >= 0 && px < pw && py >= 0 && py < ph) {
      const uint2 raw = __ldg(reinterpret_cast<const uint2*>(vb + (size_t)(pb + py * pw + px) * vstride));
      const float2 f01 = __half22float2(*reinterpret_cast<const __half2*>(&raw.x)), f23 = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
      acc0 += bw * f01.x; acc1 += bw * f01.y; acc2 += bw * f23.x; acc3 += bw * f23.y;
    }
  }
#pragma unroll
  for (int o = 8; o <= 16; o <<= 1) {
    acc0 += __shfl_xor_sync(0xffffffffu, acc0, o); acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
    acc2 += __shfl_xor_sync(0xffffffffu, acc2, o); acc3 += __shfl_xor_sync(0xffffffffu, acc3, o);
  }
  if (lane < 8) {
    const __half2 o01 = __floats2half2_rn(acc0, acc1), o23 = __floats2half2_rn(acc2, acc3);
    uint2 pk; pk.x = *reinterpret_cast<const uint32_t*>(&o01); pk.y = *reinterpret_cast<const uint32_t*>(&o23);
    *reinterpret_cast<uint2*>(out + (size_t)warp * 32 + quad * 4) = pk;
  }
}

__global__ void cast_addpos_kernel(const float4* __restrict__ x, const float4* __restrict__ pos, uint2* __restrict__ ox, uint2* __restrict__ oxp, long n4) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    if (ox) {
      const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
      uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b); ox[i] = o;
    }
    if (oxp) {
      const float4 p = pos ? __ldg(pos + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      const __half2 a = __floats2half2_rn(v.x + p.x, v.y + p.y), b = __floats2half2_rn(v.z + p.z, v.w + p.w);
      uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b); oxp[i] = o;
    }
  }
}

__global__ void cast_f32_f16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, long n4, const float* __restrict__ in_tail,
                                    __half* __restrict__ out_tail, int tail) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(in + i);
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b);
    out[i] = o;
  }
  if (blockIdx.x == 0 && threadIdx.x < tail) out_tail[threadIdx.x] = __float2half_rn(in_tail[threadIdx.x]);
}

// ------------------------------------------------------------------------------ bi-directional fusion attention ----
// GroundingDinoBiMultiHeadAttention (groundingdino BiMultiHeadAttention, reached from vlfm/vlm/grounding_dino.py:61-67):
// head_dim 256, 4 heads.  Both directions are plain softmax attentions over the SAME logits S = scale * q_img . k_txt:
//   image <- text : queries = image tokens (thousands), keys/values = text tokens (tens)           -> chunks == 1
//   text <- image : queries = text tokens, keys = the image QUERY projection, values = image values -> keys split into
//                   chunks over CTAs, partial (m, l, O) merged by biattn_merge_kernel.
// Flash-style on mma.sync m16n8k16.  8 warps = 4 row groups of 16 queries x 2 channel halves (128 channels each): the two
// warps of a row group both compute S (tensor cores are idle anyway) so that each keeps only 64 accumulator registers.
struct BiAttnArgs {
  const __half *q, *k, *v;   // rows b*N + i, head h at column h*256
  __half* o16;               // chunks == 1: [B*Nq, ldo]
  float* part;               // chunks > 1: [B, H, chunks, NqP, 258] unnormalised channels, then m, l
  int B, H, Nq, Nk, ldq, ldk, ldv, ldo, KC, chunks, NqP;
  float scale_log2;
};
__device__ __forceinline__ void bi_mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t bi_pack(float a, float b) { __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ void bi_ldm_x2t(uint32_t& r0, uint32_t& r1, const __half* p) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

// HD = head_dim, NS = channel splits per row group: 8 warps = (8 / NS) row groups of 16 queries x NS channel slices of HD / NS
template <int HD, int NS>
__global__ void __launch_bounds__(256)
biattn_kernel(BiAttnArgs a) {
  constexpr int BI_HD = HD, BI_KS = HD + 8, CW = HD / NS, RPB = 16 * (8 / NS);
  extern __shared__ __align__(16) uint8_t bi_smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int rg = warp / NS, half = warp % NS;
  const int qb = blockIdx.x / a.chunks, ch = blockIdx.x - qb * a.chunks, h = blockIdx.y, b = blockIdx.z;
  const int k0 = ch * a.KC, nk = min(a.KC, a.Nk - k0), nkp = (nk + 15) & ~15;
  __half* sK = reinterpret_cast<__half*>(bi_smem);
  __half* sV = sK + (size_t)((a.KC + 15) & ~15) * BI_KS;
  const __half* kbase = a.k + ((size_t)b * a.Nk + k0) * a.ldk + (size_t)h * BI_HD;
  const __half* vbase = a.v + ((size_t)b * a.Nk + k0) * a.ldv + (size_t)h * BI_HD;
  for (int i = tid; i < nkp * (BI_HD / 8); i += 256) {
    const int key = i / (BI_HD / 8), c = (i % (BI_HD / 8)) * 8;
    const bool ok = key < nk;
    const __half* ks = ok ? kbase + (size_t)key * a.ldk + c : kbase;
    const __half* vs = ok ? vbase + (size_t)key * a.ldv + c : vbase;
    const uint32_t kd = (uint32_t)__cvta_generic_to_shared(sK + key * BI_KS + c), vd = (uint32_t)__cvta_generic_to_shared(sV + key * BI_KS + c);
    const int nb = ok ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(kd), "l"(ks), "r"(nb) : "memory");
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(vd), "l"(vs), "r"(nb) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  const int row0 = qb * RPB + rg * 16, r_lo = row0 + g, r_hi = row0 + g + 8;
  const __half* qlo = a.q + ((size_t)b * a.Nq + r_lo) * a.ldq + (size_t)h * BI_HD;
  const __half* qhi = a.q + ((size_t)b * a.Nq + r_hi) * a.ldq + (size_t)h * BI_HD;
  uint32_t qf[BI_HD / 16][4];
#pragma unroll
  for (int kk = 0; kk < BI_HD / 16; ++kk) {
    const int c0 = kk * 16 + 2 * t, c1 = c0 + 8;
    qf[kk][0] = r_lo < a.Nq ? *reinterpret_cast<const uint32_t*>(qlo + c0) : 0u;
    qf[kk][1] = r_hi < a.Nq ? *reinterpret_cast<const uint32_t*>(qhi + c0) : 0u;
    qf[kk][2] = r_lo < a.Nq ? *reinterpret_cast<const uint32_t*>(qlo + c1) : 0u;
    qf[kk][3] = r_hi < a.Nq ? *reinterpret_cast<const uint32_t*>(qhi + c1) : 0u;
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  if (row0 >= a.Nq) return;                        // row group past the last query (no block-wide barrier follows)
  float o[CW / 8][4];
#pragma unroll
  for (int i = 0; i < CW / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  for (int kb = 0; kb < nkp; kb += 64) {
    const int ntiles = min(8, (nkp - kb) >> 3);
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      if (j < ntiles) {
        const __half* kr = sK + (kb + j * 8 + g) * BI_KS + 2 * t;
#pragma unroll
        for (int kk = 0; kk < BI_HD / 16; ++kk)
          bi_mma_16816(s[j], qf[kk], *reinterpret_cast<const uint32_t*>(kr + kk * 16), *reinterpret_cast<const uint32_t*>(kr + kk * 16 + 8));
      }
    }
    float bm_lo = -INFINITY, bm_hi = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = kb + j * 8 + 2 * t;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = (j < ntiles) && (key + (e & 1) < nk);
        s[j][e] = ok ? s[j][e] * a.scale_log2 : -INFINITY;
      }
      bm_lo = fmaxf(bm_lo, fmaxf(s[j][0], s[j][1])); bm_hi = fmaxf(bm_hi, fmaxf(s[j][2], s[j][3]));
    }
    bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 1)); bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 2));
    bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 1)); bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 2));
    const float mn_lo = fmaxf(m_lo, bm_lo), mn_hi = fmaxf(m_hi, bm_hi);
    const float ref_lo = mn_lo == -INFINITY ? 0.f : mn_lo, ref_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
    const float al_lo = exp2f(m_lo - ref_lo), al_hi = exp2f(m_hi - ref_hi);
    m_lo = mn_lo; m_hi = mn_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = exp2f(s[j][0] - ref_lo); s[j][1] = exp2f(s[j][1] - ref_lo);
      s[j][2] = exp2f(s[j][2] - ref_hi); s[j][3] = exp2f(s[j][3] - ref_hi);
      sum_lo += s[j][0] + s[j][1]; sum_hi += s[j][2] + s[j][3];
    }
    l_lo = l_lo * al_lo + sum_lo; l_hi = l_hi * al_hi + sum_hi;
#pragma unroll
    for (int i = 0; i < CW / 8; ++i) { o[i][0] *= al_lo; o[i][1] *= al_lo; o[i][2] *= al_hi; o[i][3] *= al_hi; }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      if (2 * p < ntiles) {
        uint32_t pa[4];
        pa[0] = bi_pack(s[2 * p][0], s[2 * p][1]); pa[1] = bi_pack(s[2 * p][2], s[2 * p][3]);
        pa[2] = bi_pack(s[2 * p + 1][0], s[2 * p + 1][1]); pa[3] = bi_pack(s[2 * p + 1][2], s[2 * p + 1][3]);
        const __half* vr = sV + (kb + p * 16 + (lane & 15)) * BI_KS + half * CW;
#pragma unroll
        for (int i = 0; i < CW / 8; ++i) {
          uint32_t b0, b1;
          bi_ldm_x2t(b0, b1, vr + i * 8);
          bi_mma_16816(o[i], pa, b0, b1);
        }
      }
    }
  }
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  if (a.chunks == 1) {
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
    __half* olo = a.o16 + ((size_t)b * a.Nq + r_lo) * a.ldo + (size_t)h * BI_HD + half * CW;
    __half* ohi = a.o16 + ((size_t)b * a.Nq + r_hi) * a.ldo + (size_t)h * BI_HD + half * CW;
#pragma unroll
    for (int i = 0; i < CW / 8; ++i) {
      const int c = i * 8 + 2 * t;
      if (r_lo < a.Nq) *reinterpret_cast<uint32_t*>(olo + c) = bi_pack(o[i][0] * inv_lo, o[i][1] * inv_lo);
      if (r_hi < a.Nq) *reinterpret_cast<uint32_t*>(ohi + c) = bi_pack(o[i][2] * inv_hi, o[i][3] * inv_hi);
    }
  } else {
    float* plo = a.part + ((((size_t)b * a.H + h) * a.chunks + ch) * a.NqP + r_lo) * (HD + 2);
    float* phi = a.part + ((((size_t)b * a.H + h) * a.chunks + ch) * a.NqP + r_hi) * (HD + 2);
#pragma unroll
    for (int i = 0; i < CW / 8; ++i) {
      const int c = half * CW + i * 8 + 2 * t;
      if (r_lo < a.Nq) *reinterpret_cast<float2*>(plo + c) = make_float2(o[i][0], o[i][1]);
      if (r_hi < a.Nq) *reinterpret_cast<float2*>(phi + c) = make_float2(o[i][2], o[i][3]);
    }
    if (half == 0 && t == 0) {
      if (r_lo < a.Nq) { plo[HD] = m_lo; plo[HD + 1] = l_lo; }
      if (r_hi < a.Nq) { phi[HD] = m_hi; phi[HD + 1] = l_hi; }
    }
  }
}
// log-sum-exp merge of the key chunks: one block per (b, h, query row), thread = channel
__global__ void biattn_merge_kernel(const float* __restrict__ part, __half* __restrict__ o16, int H, int Nq, int NqP, int chunks, int ldo, int HD) {
  const int row = blockIdx.x, h = blockIdx.y, b = blockIdx.z, c = threadIdx.x;
  const int PW = HD + 2;
  const float* p = part + (((size_t)b * H + h) * chunks * NqP + row) * PW;
  const size_t cs = (size_t)NqP * PW;
  float M = -INFINITY;
  for (int k = 0; k < chunks; ++k) M = fmaxf(M, p[k * cs + HD]);
  float L = 0.f, acc = 0.f;
  for (int k = 0; k < chunks; ++k) {
    const float w = exp2f(p[k * cs + HD] - M);
    L += p[k * cs + HD + 1] * w;
    acc += p[k * cs + c] * w;
  }
  o16[((size_t)b * Nq + row) * ldo + (size_t)h * HD + c] = __float2half_rn(acc / L);
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_cast_f32_f16(const float* d_in, void* d_out16, long n, void* stream) {
  if (!d_in || !d_out16 || n < 0) { set_error("vlfm_cast_f32_f16: bad argument"); return VLFM_E_INVALID; }
  if (n == 0) return VLFM_OK;
  if (((uintptr_t)d_in & 15) || ((uintptr_t)d_out16 & 7)) { set_error("vlfm_cast_f32_f16: pointers must be 16 / 8 byte aligned"); return VLFM_E_INVALID; }
  const long n4 = n >> 2; const int tail = (int)(n & 3);
  long blocks = (n4 + 255) / 256; if (blocks < 1) blocks = 1; if (blocks > 132 * 16) blocks = 132 * 16;
  cast_f32_f16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)d_in, (uint2*)d_out16, n4, d_in + 4 * n4,
                                                                          (__half*)d_out16 + 4 * n4, tail);
  VLFM_CHECK_LAUNCH("vlfm_cast_f32_f16");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_msda_fused(const void* d_value16, const float* d_offlog, int ld, int logit_col, const float* d_ref, int ref_dim,
                               void* d_out16, int B, int S, int Q, int heads, int levels, int points, const int32_t* h_shapes_hw,
                               void* stream) {
  if (!d_value16 || !d_offlog || !d_ref || !d_out16 || !h_shapes_hw || B < 1 || S < 1 || Q < 1 || heads < 1 || points < 1 || levels < 1 ||
      levels > MSDA_MAX_LEVELS || levels * points > 16 || (ref_dim != 2 && ref_dim != 4) || (ld & 1) || ((heads * levels * points * 2) & 1)) {
    set_error("vlfm_msda_fused: bad argument"); return VLFM_E_INVALID;
  }
  MsdaArgs a{};
  a.B = B; a.S = S; a.Q = Q; a.heads = heads; a.hd = 32; a.levels = levels; a.points = points;
  int acc = 0;
  for (int l = 0; l < levels; ++l) { a.H[l] = h_shapes_hw[2 * l]; a.W[l] = h_shapes_hw[2 * l + 1]; a.start[l] = acc; acc += a.H[l] * a.W[l]; }
  if (acc != S) { set_error("vlfm_msda_fused: spatial shapes sum to %d, value has %d positions", acc, S); return VLFM_E_INVALID; }
  const long blocks = ((long)B * Q * heads + 7) / 8;
  if (blocks > 0x7fffffffL) { set_error("vlfm_msda_fused: too many queries"); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const __half* v = (const __half*)d_value16; __half* o = (__half*)d_out16;
  const bool std44 = levels == 4 && points == 4;      // GroundingDINO's configuration: fully unrolled gather
  if (ref_dim == 2) {
    if (std44) msda_fused_kernel<2, 4, 4><<<(unsigned)blocks, 256, 0, st>>>(v, d_offlog, ld, logit_col, d_ref, o, a);
    else msda_fused_kernel<2, 0, 0><<<(unsigned)blocks, 256, 0, st>>>(v, d_offlog, ld, logit_col, d_ref, o, a);
  } else {
    if (std44) msda_fused_kernel<4, 4, 4><<<(unsigned)blocks, 256, 0, st>>>(v, d_offlog, ld, logit_col, d_ref, o, a);
    else msda_fused_kernel<4, 0, 0><<<(unsigned)blocks, 256, 0, st>>>(v, d_offlog, ld, logit_col, d_ref, o, a);
  }
  VLFM_CHECK_LAUNCH("vlfm_msda_fused");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_cast_addpos_f16(const float* d_x, const float* d_pos, void* d_out_x16, void* d_out_xp16, long n, void* stream) {
  if (!d_x || (!d_out_x16 && !d_out_xp16) || n < 0 || (n & 3)) { set_error("vlfm_cast_addpos_f16: bad argument"); return VLFM_E_INVALID; }
  if (n == 0) return VLFM_OK;
  const long n4 = n >> 2;
  long blocks = (n4 + 255) / 256; if (blocks > 132 * 16) blocks = 132 * 16;
  cast_addpos_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)d_x, (const float4*)d_pos, (uint2*)d_out_x16, (uint2*)d_out_xp16, n4);
  VLFM_CHECK_LAUNCH("vlfm_cast_addpos_f16");
  count_launch();
  return VLFM_OK;
}

// softmax(scale * q k^T) v per (batch, head) for head_dim 256 (GroundingDINO fusion layers) or 32 (decoder self / text
// cross attention).  q [B*Nq, ldq], k [B*Nk, ldk], v [B*Nk, ldv] fp16 with head h at column h*head_dim; out fp16 [B*Nq, ldo].
// Keys are split into chunks of `key_chunk` (multiple of 16; <= 192 for head_dim 256, <= 1024 for 32) over CTAs when Nk
// exceeds it; d_part then needs B*heads*chunks*ceilR(Nq)*(head_dim+2) floats (R = 64 resp. 128 query rows per CTA).
extern "C" int vlfm_biattn_f16(const void* d_q, const void* d_k, const void* d_v, void* d_out16, float* d_part, size_t part_floats, int B,
                               int heads, int head_dim, int Nq, int Nk, int ldq, int ldk, int ldv, int ldo, int key_chunk, float scale,
                               void* stream) {
  const int kc_max = head_dim == 256 ? 192 : 1024;
  if (!d_q || !d_k || !d_v || !d_out16 || B < 1 || heads < 1 || Nq < 1 || Nk < 1 || (head_dim != 256 && head_dim != 32) || key_chunk < 16 ||
      key_chunk > kc_max || (key_chunk & 15) || (ldq & 7) || (ldk & 7) || (ldv & 7) || (ldo & 1)) {
    set_error("vlfm_biattn_f16: bad argument"); return VLFM_E_INVALID;
  }
  BiAttnArgs a{};
  a.q = (const __half*)d_q; a.k = (const __half*)d_k; a.v = (const __half*)d_v; a.o16 = (__half*)d_out16; a.part = d_part;
  a.B = B; a.H = heads; a.Nq = Nq; a.Nk = Nk; a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo;
  a.KC = Nk <= key_chunk ? ((Nk + 15) & ~15) : key_chunk;
  a.chunks = (Nk + a.KC - 1) / a.KC;
  const int rpb = head_dim == 256 ? 64 : 128;
  const int qblocks = (Nq + rpb - 1) / rpb;
  a.NqP = qblocks * rpb;
  a.scale_log2 = scale * 1.4426950408889634f;
  const size_t need = (size_t)B * heads * a.chunks * a.NqP * (head_dim + 2);
  if (a.chunks > 1 && (!d_part || part_floats < need)) {
    set_error("vlfm_biattn_f16: partial buffer too small (%zu floats needed)", need); return VLFM_E_INVALID;
  }
  const size_t smem = (size_t)2 * a.KC * (head_dim + 8) * 2;
  static bool cfg = false;
  if (!cfg) {
    int rc = check_cuda(cudaFuncSetAttribute(biattn_kernel<256, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 192 * 264 * 2), "attr(biattn256)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(biattn_kernel<32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 1024 * 40 * 2), "attr(biattn32)");
    if (rc) return rc; cfg = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if ((long)qblocks * a.chunks > 0x7fffffffL || heads > 65535 || B > 65535) { set_error("vlfm_biattn_f16: grid too large"); return VLFM_E_INVALID; }
  const dim3 grid((unsigned)(qblocks * a.chunks), heads, B);
  if (head_dim == 256) biattn_kernel<256, 2><<<grid, 256, smem, st>>>(a);
  else biattn_kernel<32, 1><<<grid, 256, smem, st>>>(a);
  VLFM_CHECK_LAUNCH("biattn_kernel");
  count_launch();
  if (a.chunks > 1) {
    biattn_merge_kernel<<<dim3(Nq, heads, B), head_dim, 0, st>>>(d_part, (__half*)d_out16, heads, Nq, a.NqP, a.chunks, ldo, head_dim);
    VLFM_CHECK_LAUNCH("biattn_merge_kernel");
    count_launch();
  }
  return VLFM_OK;
}
