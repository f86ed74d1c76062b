// Non-GEMM operators of the BLIP-2 ITC forward (sm_90a):
//   - image preprocessing: PIL-exact antialiased bicubic resize (uint8, 22-bit fixed
//     point, horizontal then vertical pass) + ToTensor + Normalize, written straight
//     into the im2col layout of the 14x14/14 patch-embedding GEMM
//     (reference: vlfm/vlm/blip2itm.py:48-49 -> lavis BlipImageEvalProcessor);
//   - token assembly (class token + position embedding);
//   - LayerNorm (fp32 in, fp16 and/or fp32 out);
//   - multi-head attention, flash-style online softmax on mma.sync m16n8k16 fp16
//     tensor-core tiles (ViT-g self-attention N=257/hd=88, Q-Former self/cross hd=64);
//   - ITC head: L2-normalise the 32 projected queries, dot with the cached text
//     feature, max over queries (blip2itm.py:52, match_head="itc").
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace vlfm {

// --------------------------------------------------------------- preprocessing ----
// coefficient tables are built on the host exactly like Pillow's precompute_coeffs +
// normalize_coeffs_8bpc (see vlfm_b200/vlm/preprocess.py); layout per output index:
// bounds[2*i] = first input index, bounds[2*i+1] = tap count, kk[i*ksize + t].
__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= 22;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void resize_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ mid, int H, int W, int OW,
                                const int* __restrict__ bounds, const int* __restrict__ kk, int ksize) {
  // in [B,H,W,3] -> mid [B,H,OW,3]
  const int b = blockIdx.z, y = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over OW*3
  if (i >= OW * 3) return;
  const int xo = i / 3, c = i - 3 * xo;
  const int x0 = bounds[2 * xo], n = bounds[2 * xo + 1];
  const uint8_t* row = in + ((size_t)b * H + y) * W * 3;
  int ss = 1 << 21;
  for (int t = 0; t < n; ++t) ss += (int)row[(x0 + t) * 3 + c] * kk[xo * ksize + t];
  mid[(((size_t)b * H + y) * OW + xo) * 3 + c] = clip8(ss);
}

__global__ void resize_v_norm_im2col_kernel(const uint8_t* __restrict__ mid, __half* __restrict__ out, int H, int OW,
                                            int OH, const int* __restrict__ bounds, const int* __restrict__ kk,
                                            int ksize, int patch, int ldk, float m0, float m1, float m2, float s0,
                                            float s1, float s2) {
  // mid [B,H,OW,3] -> out [B*(OH/patch)*(OW/patch), ldk], col = c*patch*patch + ky*patch + kx
  const int b = blockIdx.z, yo = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= OW * 3) return;
  const int xo = i / 3, c = i - 3 * xo;
  const int y0 = bounds[2 * yo], n = bounds[2 * yo + 1];
  int ss = 1 << 21;
  for (int t = 0; t < n; ++t) ss += (int)mid[(((size_t)b * H + y0 + t) * OW + xo) * 3 + c] * kk[yo * ksize + t];
  const float px = (float)clip8(ss);
  const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
  const float v = __fdiv_rn(__fsub_rn(__fdiv_rn(px, 255.f), mean), sd);   // ToTensor, Normalize (float32)
  const int gp = OW / patch;
  const int py = yo / patch, ky = yo - py * patch, pxi = xo / patch, kx = xo - pxi * patch;
  const size_t rowi = (size_t)b * (OH / patch) * gp + (size_t)py * gp + pxi;
  out[rowi * ldk + c * patch * patch + ky * patch + kx] = __float2half_rn(v);
}

// x[b, 0] = cls + pos[0];  x[b, 1+p] = patch[b, p] + pos[1+p]
__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, float* __restrict__ x, int B, int T, int D) {
  const size_t n = (size_t)B * T * D;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const size_t r = i / D;
    const int t = (int)(r % T), b = (int)(r / T);
    float v = t == 0 ? cls[d] : patch[((size_t)b * (T - 1) + (t - 1)) * D + d];
    x[i] = v + pos[(size_t)t * D + d];
  }
}

// ------------------------------------------------------------------- LayerNorm ----
// one warp per row, float4 lanes; x, gamma and beta are all fetched up front (every load of the
// kernel is in flight before the first reduction), two-pass statistics in registers.
template <int MAXV4>
__global__ void __launch_bounds__(128)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 __half* __restrict__ out16, float* __restrict__ out32, int rows, int D, int ldx, int ldo16, int ldo32,
                 float eps, __half* __restrict__ out16_lo) {   // out16_lo: the x2 residual of out16 (same stride), or null
  pdl_trigger();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int D4 = D >> 2;
  float4 g[MAXV4], bt[MAXV4], v[MAXV4];
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {   // parameters do not depend on the predecessor kernel
    const int j = lane + 32 * i;
    g[i] = j < D4 ? __ldg(reinterpret_cast<const float4*>(gamma) + j) : make_float4(0, 0, 0, 0);
    bt[i] = j < D4 ? __ldg(reinterpret_cast<const float4*>(beta) + j) : make_float4(0, 0, 0, 0);
  }
  pdl_wait();
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * ldx);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < D4 ? xr[j] : make_float4(0, 0, 0, 0);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    if (lane + 32 * i < D4) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)D + eps);
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    const int j = lane + 32 * i;
    if (j < D4) {
      float4 y;
      y.x = (v[i].x - mean) * rstd * g[i].x + bt[i].x;
      y.y = (v[i].y - mean) * rstd * g[i].y + bt[i].y;
      y.z = (v[i].z - mean) * rstd * g[i].z + bt[i].z;
      y.w = (v[i].w - mean) * rstd * g[i].w + bt[i].w;
      if (out16) {
        __half2 h0 = __floats2half2_rn(y.x, y.y), h1 = __floats2half2_rn(y.z, y.w);
        uint2 pk = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
        *reinterpret_cast<uint2*>(out16 + (size_t)row * ldo16 + 4 * j) = pk;
        if (out16_lo) {
          const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
          __half2 l0 = __floats2half2_rn((y.x - f0.x) * X2_SCALE, (y.y - f0.y) * X2_SCALE), l1 = __floats2half2_rn((y.z - f1.x) * X2_SCALE, (y.w - f1.y) * X2_SCALE);
          uint2 pl = make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
          *reinterpret_cast<uint2*>(out16_lo + (size_t)row * ldo16 + 4 * j) = pl;
        }
      }
      if (out32) *reinterpret_cast<float4*>(out32 + (size_t)row * ldo32 + 4 * j) = y;
    }
  }
}

// x_row += the partial sums of a split residual GEMM (layout: SplitK in common.cuh), added in K order and written back; then
// LayerNorm of the updated row.  The deterministic reduction of vlfm_gemm_f16_resid_ln / vlfm_gemm_f16x2_resid_ln: the adds
// always run in the same order -> bitwise reproducible.  Each thread owns one float4 of the row, so it reads the slabs of one
// output tile (stream-K: the segments of that tile, their number differs between column blocks); the loads of up to four slabs
// are issued before the first add: with a warp per row and a runtime loop over the splits (first version) the kernel paid one
// L2 round trip per split (9.5 us for 8 splits at 257 x 1408; the deterministic forward was 12 % slower than the red.add one).
// One float4 per thread, D/4 threads per row (<= 384): 11 warps per 1408-wide row keep ~20 warps per SM in flight (the 128-thread
// version ran at 10 % occupancy, 6.5-8.5 us per launch, 78 launches per ViT forward).
__global__ void __launch_bounds__(384)
layernorm_reduce_kernel(float* x, const float* __restrict__ partials, SplitK sk,
                        const float* __restrict__ gamma, const float* __restrict__ beta, __half* __restrict__ out16,
                        float* out32, int rows, int D, int ldx, int ldo16, int ldo32, float eps, __half* __restrict__ out16_lo) {   // out32 may alias x (post-LN blocks)
  pdl_trigger();
  __shared__ float red[2][12];
  const int row = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
  const int D4 = D >> 2;
  const bool on = t < D4;
  const float4 g = on ? __ldg(reinterpret_cast<const float4*>(gamma) + t) : make_float4(0, 0, 0, 0);   // parameters do not depend on
  const float4 bt = on ? __ldg(reinterpret_cast<const float4*>(beta) + t) : make_float4(0, 0, 0, 0);   // the predecessor kernel
  // slabs [s0, s1) hold this thread's four columns, at partials + s * stride + off
  int s0 = 0, s1 = sk.splits;
  long long stride = sk.stride, off = (long long)row * D + 4 * t;
  if (sk.splits == 0) {
    const int m = min(row / SK_TILE, sk.row_tiles - 1), nb = (4 * t) / SK_TILE, tile = nb * sk.row_tiles + m;
    s0 = sk.sk_owner(tile * sk.num_k) + tile;
    s1 = sk.sk_owner((tile + 1) * sk.num_k - 1) + tile + 1;
    stride = SK_SLAB;
    off = (long long)(row - m * SK_TILE) * SK_TILE + (4 * t - nb * SK_TILE);
  }
  pdl_wait();
  float4* xr = reinterpret_cast<float4*>(x + (size_t)row * ldx);
  float4 v = on ? xr[t] : make_float4(0, 0, 0, 0);
  for (int sp0 = s0; sp0 < s1; sp0 += 4) {
    float4 pv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4* pr = reinterpret_cast<const float4*>(partials + (size_t)(sp0 + u) * (size_t)stride + (size_t)off);
      pv[u] = (sp0 + u < s1 && on) ? __ldcg(pr) : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)          // fixed order: bitwise reproducible
      if (sp0 + u < s1) { v.x += pv[u].x; v.y += pv[u].y; v.z += pv[u].z; v.w += pv[u].w; }
  }
  float s = 0.f;
  if (on) { xr[t] = v; s = (v.x + v.y) + (v.z + v.w); }
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) red[0][w] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < nw; ++i) tot += red[0][i];          // same order in every thread
  const float mean = tot / (float)D;
  float q = 0.f;
  if (on) { const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean; q = (a * a + b * b) + (c * c + d * d); }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if (lane == 0) red[1][w] = q;
  __syncthreads();
  float qt = 0.f;
  for (int i = 0; i < nw; ++i) qt += red[1][i];
  const float rstd = rsqrtf(qt / (float)D + eps);
  if (on) {
    float4 y;
    y.x = (v.x - mean) * rstd * g.x + bt.x;
    y.y = (v.y - mean) * rstd * g.y + bt.y;
    y.z = (v.z - mean) * rstd * g.z + bt.z;
    y.w = (v.w - mean) * rstd * g.w + bt.w;
    if (out16) {
      __half2 h0 = __floats2half2_rn(y.x, y.y), h1 = __floats2half2_rn(y.z, y.w);
      uint2 pk = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
      *reinterpret_cast<uint2*>(out16 + (size_t)row * ldo16 + 4 * t) = pk;
      if (out16_lo) {
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        __half2 l0 = __floats2half2_rn((y.x - f0.x) * X2_SCALE, (y.y - f0.y) * X2_SCALE), l1 = __floats2half2_rn((y.z - f1.x) * X2_SCALE, (y.w - f1.y) * X2_SCALE);
        uint2 pl = make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
        *reinterpret_cast<uint2*>(out16_lo + (size_t)row * ldo16 + 4 * t) = pl;
      }
    }
    if (out32) *reinterpret_cast<float4*>(out32 + (size_t)row * ldo32 + 4 * t) = y;
  }
}

// ------------------------------------------------------------------- attention ----
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

struct AttnArgs {
  const __half* q; const __half* k; const __half* v; __half* o;
  int ldq, ldk, ldv, ldo;   // row strides (elements)
  int Nq, Nk, hd, heads;
  float scale_log2;         // softmax scale * log2(e)
};

constexpr int ATT_WARPS = 4;
constexpr int ATT_NKMAX = 272;             // keys padded to a multiple of 16

__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const __half* p) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

// Batch-1 staging (attention_kernel<HDP, 4, true>): 64 query rows per CTA, so each head's K / V is read by ceil(Nq/64) CTAs instead
// of ceil(Nq/32) (the ViT-g at batch 1: 80 CTAs, one wave), and nothing waits for all of it.  Shared memory: sK, sV [NKP][HDP + 8],
// sQ [64][HDP + 8] (the merge buffer overlays them), then ATT_B1_BARS mbarriers.  Every thread issues its 16-byte cp.async copies
// for Q, then K and V of each of the four key parts in turn, and after each piece a cp.async.mbarrier.arrive on the piece's
// barrier (count: every thread): a barrier completes when every copy issued up to it has landed, so part 0 starts computing on
// its keys while the other parts' are in flight.  The parts and their 64-key blocks are those of attention_kernel<HDP, 4>, so a
// row's arithmetic, and its result, are the same.
constexpr int ATT_B1_ROWS = 64;
constexpr int ATT_B1_THREADS = 512;
constexpr int ATT_B1_BARS = 5;             // Q, then K and V of each key part

__host__ __device__ constexpr int attn_b1_bar_offset(int nkp, int hdp) {   // bytes; the merge of 12 warps may need more than the staging
  return (2 * nkp + ATT_B1_ROWS) * (hdp + 8) * 2 > 12 * (hdp / 2 + 4) * 32 * 4 ? (2 * nkp + ATT_B1_ROWS) * (hdp + 8) * 2
                                                                              : 12 * (hdp / 2 + 4) * 32 * 4;
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const __half* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

template <int HDP>
__device__ __forceinline__ void attn_b1_stage(const AttnArgs& a, uint8_t* smem, __half* sK, __half* sV, const __half* kbase,
                                              const __half* vbase, int NKP, int qb, int tid) {
  constexpr int KS = HDP + 8, CH = HDP / 8;
  const uint32_t bars = smem_u32(smem + attn_b1_bar_offset(NKP, HDP));
  if (tid == 0) {
    for (int i = 0; i < ATT_B1_BARS; ++i) mbar_init(bars + 8 * i, ATT_B1_THREADS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // rows [r0, r1) of a [rows][KS] tile; src-size 0 zero-fills rows >= rlim and columns >= hd
  auto copy_rows = [&](__half* dst, const __half* src, int ld, int r0, int r1, int rlim) {
    for (int i = r0 * CH + tid; i < r1 * CH; i += ATT_B1_THREADS) {
      const int r = i / CH, c = (i - r * CH) * 8;
      const bool ok = r < rlim && c < a.hd;
      const __half* p = ok ? src + (size_t)r * ld + c : src;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst + r * KS + c)), "l"(p), "r"(ok ? 16 : 0) : "memory");
    }
  };
  const __half* qbase = a.q + ((size_t)blockIdx.z * a.Nq + (size_t)qb * ATT_B1_ROWS) * a.ldq + (size_t)blockIdx.y * a.hd;
  copy_rows(sV + NKP * KS, qbase, a.ldq, 0, ATT_B1_ROWS, min(ATT_B1_ROWS, a.Nq - qb * ATT_B1_ROWS));
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bars) : "memory");
  const int tiles = NKP >> 4, tbase = tiles / 4, trem = tiles % 4;
  for (int p = 0; p < 4; ++p) {
    const int k0 = 16 * (p * tbase + min(p, trem)), k1 = k0 + 16 * (tbase + (p < trem ? 1 : 0));
    copy_rows(sK, kbase, a.ldk, k0, k1, a.Nk);
    copy_rows(sV, vbase, a.ldv, k0, k1, a.Nk);
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bars + 8 * (1 + p)) : "memory");
  }
}

// grid (ceil(Nq/32), heads, B), 4 warps.  K and V of one (batch, head) are staged row-major
// [key][hd] in padded (conflict-free) shared memory with 16-byte copies.  Warp w owns query rows
// 16*(w&1).. and the key half (w>>1); the two halves are merged flash-style through shared memory.
// S = Q K^T and O = P V run on mma.sync m16n8k16 (fp16 in, fp32 accumulate); V fragments come from
// ldmatrix.trans.
// KH = 2: 32 query rows per CTA, each row group's keys split over two warps (small batches: more CTAs,
// shorter critical path).  KH = 1: 64 query rows per CTA, every warp sees all keys (large batches: the K/V
// staging is amortised over twice the queries, no merge).
template <int HDP, int KH, bool B1 = false>
__global__ void __launch_bounds__(32 * (B1 ? 16 : (KH == 4 ? 8 : ATT_WARPS)))
attention_kernel(AttnArgs a) {
  static_assert(!B1 || KH == 4, "the batch-1 variant splits the keys in four");
  // KH = 4: eight warps = 2 row groups x 4 key quarters (small batches: shortest critical path); B1: sixteen = 4 x 4
  constexpr int NW = B1 ? 16 : (KH == 4 ? 8 : ATT_WARPS);
  constexpr int RG = NW / KH;            // row groups of 16 queries
  constexpr int ATT_QBLK = 16 * RG;
  constexpr int KS = HDP + 8;            // row stride (halves) of sK / sV
  extern __shared__ __align__(16) uint8_t att_smem[];
  __half* sK = reinterpret_cast<__half*>(att_smem);            // [NKP][KS]
  const int b = blockIdx.z, h = blockIdx.y, qb = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int NKP = (a.Nk + 15) & ~15;
  __half* sV = sK + NKP * KS;                                  // [NKP][KS]
  pdl_trigger();
  pdl_wait();
  const __half* kbase = a.k + (size_t)b * a.Nk * a.ldk + (size_t)h * a.hd;
  const __half* vbase = a.v + (size_t)b * a.Nk * a.ldv + (size_t)h * a.hd;

  constexpr int CH = HDP / 8;
  if constexpr (B1) {
    attn_b1_stage<HDP>(a, att_smem, sK, sV, kbase, vbase, NKP, qb, tid);
  } else {
  // ---- stage K and V with cp.async (16-byte LDGSTS, all copies in flight at once; src-size 0 zero-fills the
  // padding rows >= Nk and columns >= hd)
  for (int i = tid; i < NKP * CH; i += 32 * NW) {
    const int key = i / CH, c = (i - key * CH) * 8;
    const bool ok = key < a.Nk && c < a.hd;
    const __half* ksrc = ok ? kbase + (size_t)key * a.ldk + c : kbase;
    const __half* vsrc = ok ? vbase + (size_t)key * a.ldv + c : vbase;
    const uint32_t kd = (uint32_t)__cvta_generic_to_shared(sK + key * KS + c), vd = (uint32_t)__cvta_generic_to_shared(sV + key * KS + c);
    const int nbytes = ok ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(kd), "l"(ksrc), "r"(nbytes) : "memory");
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(vd), "l"(vsrc), "r"(nbytes) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  }

  // ---- Q fragments: rows 16*(warp&1) + {g, g+8} of this CTA's 32-row block
  const int row0 = qb * ATT_QBLK + (warp % RG) * 16;
  const int r_lo = row0 + g, r_hi = row0 + g + 8;
  uint32_t qf[HDP / 16][4];
  if constexpr (B1) {   // Q fragments: read from sQ in each key block (fewer registers live across P.V: 16 warps of 128)
    mbar_wait(smem_u32(att_smem + attn_b1_bar_offset(NKP, HDP)), 0);
  } else {
  const __half* qlo = a.q + ((size_t)b * a.Nq + r_lo) * a.ldq + (size_t)h * a.hd;
  const __half* qhi = a.q + ((size_t)b * a.Nq + r_hi) * a.ldq + (size_t)h * a.hd;
#pragma unroll
  for (int kk = 0; kk < HDP / 16; ++kk) {
    const int c0 = kk * 16 + 2 * t, c1 = c0 + 8;
    qf[kk][0] = (r_lo < a.Nq && c0 < a.hd) ? *reinterpret_cast<const uint32_t*>(qlo + c0) : 0u;
    qf[kk][1] = (r_hi < a.Nq && c0 < a.hd) ? *reinterpret_cast<const uint32_t*>(qhi + c0) : 0u;
    qf[kk][2] = (r_lo < a.Nq && c1 < a.hd) ? *reinterpret_cast<const uint32_t*>(qlo + c1) : 0u;
    qf[kk][3] = (r_hi < a.Nq && c1 < a.hd) ? *reinterpret_cast<const uint32_t*>(qhi + c1) : 0u;
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  }

  float o[HDP / 8][4];
#pragma unroll
  for (int i = 0; i < HDP / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;

  // key range of this warp: the 16-key tiles are dealt to the KH parts, the first parts take the remainder
  const int part = warp / RG, tiles = NKP >> 4, tbase = tiles / KH, trem = tiles % KH;
  const int k_begin = 16 * (part * tbase + min(part, trem)), k_end = k_begin + 16 * (tbase + (part < trem ? 1 : 0));
  if constexpr (B1) mbar_wait(smem_u32(att_smem + attn_b1_bar_offset(NKP, HDP)) + 8 * (1 + part), 0);   // K and V of this part
  for (int kb = k_begin; kb < k_end; kb += 64) {
    const int ntiles = min(8, (k_end - kb) >> 3);   // warp-uniform, even
    if constexpr (B1) {   // ldmatrix.x4: lanes 0-15 address rows +0..15 at column 16 kk, lanes 16-31 at 16 kk + 8
      const __half* qr = sV + NKP * KS + ((warp % RG) * 16 + (lane & 15)) * KS + (lane >> 4) * 8;
#pragma unroll
      for (int kk = 0; kk < HDP / 16; ++kk) ldmatrix_x4(qf[kk], qr + kk * 16);
    }
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      if (j < ntiles) {
        const __half* kr = sK + (kb + j * 8 + g) * KS + 2 * t;
#pragma unroll
        for (int kk = 0; kk < HDP / 16; ++kk) {
          uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr + kk * 16);
          uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + kk * 16 + 8);
          mma_16816(s[j], qf[kk], b0, b1);
        }
      }
    }
    float bm_lo = -INFINITY, bm_hi = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int key = kb + j * 8 + 2 * t;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = (j < ntiles) && (key + (e & 1) < a.Nk);
        s[j][e] = ok ? s[j][e] * a.scale_log2 : -INFINITY;
      }
      bm_lo = fmaxf(bm_lo, fmaxf(s[j][0], s[j][1]));
      bm_hi = fmaxf(bm_hi, fmaxf(s[j][2], s[j][3]));
    }
    bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 1));
    bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 2));
    bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 1));
    bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 2));
    // a block may be fully masked (keys >= Nk in the second half): keep the running max finite-safe
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
    for (int i = 0; i < HDP / 8; ++i) { o[i][0] *= al_lo; o[i][1] *= al_lo; o[i][2] *= al_hi; o[i][3] *= al_hi; }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      if (2 * p < ntiles) {
        uint32_t pa[4];
        pa[0] = pack_half2(s[2 * p][0], s[2 * p][1]);
        pa[1] = pack_half2(s[2 * p][2], s[2 * p][3]);
        pa[2] = pack_half2(s[2 * p + 1][0], s[2 * p + 1][1]);
        pa[3] = pack_half2(s[2 * p + 1][2], s[2 * p + 1][3]);
        // lanes 0-7 address keys +0..7, lanes 8-15 keys +8..15 (lanes >= 16 ignored by .x2)
        const __half* vr = sV + (kb + p * 16 + (lane & 15)) * KS;
#pragma unroll
        for (int i = 0; i < HDP / 8; ++i) {
          uint32_t b0, b1;
          ldmatrix_x2_trans(b0, b1, vr + i * 8);
          mma_16816(o[i], pa, b0, b1);
        }
      }
    }
  }
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);

  if (KH == 1) {   // every warp already holds complete rows
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
    __half* olo = a.o + ((size_t)b * a.Nq + r_lo) * a.ldo + (size_t)h * a.hd;
    __half* ohi = a.o + ((size_t)b * a.Nq + r_hi) * a.ldo + (size_t)h * a.hd;
#pragma unroll
    for (int i = 0; i < HDP / 8; ++i) {
      const int c = i * 8 + 2 * t;
      if (c < a.hd) {
        if (r_lo < a.Nq) *reinterpret_cast<uint32_t*>(olo + c) = pack_half2(o[i][0] * inv_lo, o[i][1] * inv_lo);
        if (r_hi < a.Nq) *reinterpret_cast<uint32_t*>(ohi + c) = pack_half2(o[i][2] * inv_hi, o[i][3] * inv_hi);
      }
    }
    return;
  }
  // ---- merge the key parts (warps >= RG -> warps < RG) through shared memory, flash-style
  __syncthreads();                                   // everyone is done with sK / sV
  float* mrg = reinterpret_cast<float*>(att_smem);   // [(KH-1)*RG warps][HDP/8*4 + 4][32 lanes]
  constexpr int MW = HDP / 8 * 4 + 4;
  if (warp >= RG) {
    float* dst = mrg + (size_t)(warp - RG) * MW * 32 + lane;
#pragma unroll
    for (int i = 0; i < HDP / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) dst[(i * 4 + e) * 32] = o[i][e];
    }
    dst[(MW - 4) * 32] = m_lo; dst[(MW - 3) * 32] = m_hi; dst[(MW - 2) * 32] = l_lo; dst[(MW - 1) * 32] = l_hi;
  }
  __syncthreads();
  if (warp >= RG) return;
#pragma unroll
  for (int p = 1; p < KH; ++p) {
    const float* src = mrg + (size_t)((p - 1) * RG + warp) * MW * 32 + lane;
    const float m2_lo = src[(MW - 4) * 32], m2_hi = src[(MW - 3) * 32], l2_lo = src[(MW - 2) * 32], l2_hi = src[(MW - 1) * 32];
    const float mm_lo = fmaxf(m_lo, m2_lo), mm_hi = fmaxf(m_hi, m2_hi);
    const float r_lo_ = mm_lo == -INFINITY ? 0.f : mm_lo, r_hi_ = mm_hi == -INFINITY ? 0.f : mm_hi;
    const float a1_lo = exp2f(m_lo - r_lo_), a2_lo = exp2f(m2_lo - r_lo_);
    const float a1_hi = exp2f(m_hi - r_hi_), a2_hi = exp2f(m2_hi - r_hi_);
    l_lo = l_lo * a1_lo + l2_lo * a2_lo; l_hi = l_hi * a1_hi + l2_hi * a2_hi;
    m_lo = mm_lo; m_hi = mm_hi;
#pragma unroll
    for (int i = 0; i < HDP / 8; ++i) {
      o[i][0] = o[i][0] * a1_lo + src[(i * 4 + 0) * 32] * a2_lo;
      o[i][1] = o[i][1] * a1_lo + src[(i * 4 + 1) * 32] * a2_lo;
      o[i][2] = o[i][2] * a1_hi + src[(i * 4 + 2) * 32] * a2_hi;
      o[i][3] = o[i][3] * a1_hi + src[(i * 4 + 3) * 32] * a2_hi;
    }
  }
  {
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
    __half* olo = a.o + ((size_t)b * a.Nq + r_lo) * a.ldo + (size_t)h * a.hd;
    __half* ohi = a.o + ((size_t)b * a.Nq + r_hi) * a.ldo + (size_t)h * a.hd;
#pragma unroll
    for (int i = 0; i < HDP / 8; ++i) {
      const int c = i * 8 + 2 * t;
      if (c < a.hd) {
        if (r_lo < a.Nq) *reinterpret_cast<uint32_t*>(olo + c) = pack_half2(o[i][0] * inv_lo, o[i][1] * inv_lo);
        if (r_hi < a.Nq) *reinterpret_cast<uint32_t*>(ohi + c) = pack_half2(o[i][2] * inv_hi, o[i][3] * inv_hi);
      }
    }
  }
}

// -------------------------------------------------------------------- ITC head ----
// proj [B, Q, D] fp32 (vision_proj output), text [P, D] fp32 rows L2-normalised -> out[b * ldo + p] = max_q cos(proj[b,q], text[p]).
// One CTA per image.  Warp w owns queries w, w + nw, ...; the prompts go in chunks of ITC_PT, each chunk reading a query row once.
// The query norm is reduced in the first chunk and kept in shared memory (den[Q], dynamic) for the others.  Every (q, p) dot
// product is the same lane-strided fp32 sum and xor-shuffle tree whatever P is, so column p equals a P = 1 launch on text[p].
constexpr int ITC_PT = 8;

__global__ void __launch_bounds__(256) itc_head_kernel(const float* __restrict__ proj, const float* __restrict__ text,
                                                       float* __restrict__ out, int P, int Q, int D, int ldo) {
  extern __shared__ float den[];
  __shared__ float best[ITC_PT][32];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int p0 = 0; p0 < P; p0 += ITC_PT) {
    const int np = min(ITC_PT, P - p0);
    const float* tx = text + (size_t)p0 * D;
    float mx[ITC_PT];
#pragma unroll
    for (int j = 0; j < ITC_PT; ++j) mx[j] = -INFINITY;
    for (int q = warp; q < Q; q += nw) {
      const float* pr = proj + ((size_t)b * Q + q) * D;
      float nn = 0.f, dt[ITC_PT];
#pragma unroll
      for (int j = 0; j < ITC_PT; ++j) dt[j] = 0.f;
      for (int d = lane; d < D; d += 32) {
        const float v = pr[d];
        if (p0 == 0) nn += v * v;
#pragma unroll
        for (int j = 0; j < ITC_PT; ++j)
          if (j < np) dt[j] += v * tx[(size_t)j * D + d];
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        if (p0 == 0) nn += __shfl_xor_sync(0xffffffffu, nn, o);
#pragma unroll
        for (int j = 0; j < ITC_PT; ++j)
          if (j < np) dt[j] += __shfl_xor_sync(0xffffffffu, dt[j], o);
      }
      const float dq = p0 == 0 ? fmaxf(sqrtf(nn), 1e-12f) : den[q];   // F.normalize eps
      // the owning warp writes den[q] here and reads it in later chunks; the CTA barrier closing each chunk orders the two
      if (p0 == 0 && lane == 0) den[q] = dq;
#pragma unroll
      for (int j = 0; j < ITC_PT; ++j) mx[j] = fmaxf(mx[j], dt[j] / dq);
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < ITC_PT; ++j) best[j][warp] = mx[j];
    }
    __syncthreads();
    if (threadIdx.x < np) {
      float m = best[threadIdx.x][0];
      for (int i = 1; i < nw; ++i) m = fmaxf(m, best[threadIdx.x][i]);
      out[(size_t)b * ldo + p0 + threadIdx.x] = m;
    }
    __syncthreads();
  }
}


// x2 operands of an fp32 array: hi = fp16(v) (optional output), lo = fp16((v - hi) * 2048)
__global__ void split_x2_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long n4) {
  pdl_trigger();
  pdl_wait();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    __half h[4], l[4];
    split_x2(v.x, h[0], l[0]); split_x2(v.y, h[1], l[1]); split_x2(v.z, h[2], l[2]); split_x2(v.w, h[3], l[3]);
    if (hi) reinterpret_cast<uint2*>(hi)[i] = *reinterpret_cast<uint2*>(h);
    reinterpret_cast<uint2*>(lo)[i] = *reinterpret_cast<uint2*>(l);
  }
}

// ----------------------------------------------------------- fp32 attention (Q-Former) ----
// The reference runs the Q-Former in float32 (lavis keeps only the ViT in half precision), and the ITC cosine is sensitive to
// it: fp16 operands in the Q-Former alone move the cosine by 3e-5 on average, the ViT's by 1e-6 (measured on the fp32 oracle).
// 32 queries x <= 272 keys x 12 heads per image is ~25 MFLOP: plain fp32 on CUDA cores.  One CTA per (head, image): K (padded
// rows: lanes read different keys at the same channel) and V staged in shared memory as fp32; a warp owns a query row at a time:
// lane = key for the scores, lane = channel for P.V.  Output = x2 operands (hi, lo) of the output projection GEMM.
constexpr int ATT32_NKMAX = 272;
constexpr int ATT32_KT = (ATT32_NKMAX + 31) / 32;
// grid (heads, images, row groups): a CTA stages K / V of its (image, head) once and its eight warps take one query row each per
// pass.  All the keys of a lane advance together through the channel loop (KT independent FMA chains per lane) and P.V keeps four
// partial sums per output channel: the first version (one chain per lane) was bound by the FMA / shared-memory latency, 86 us for
// 32 x 257 x 12 heads.
template <int HD>
__global__ void __launch_bounds__(256)
attention_f32_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, __half* __restrict__ o_hi,
                     __half* __restrict__ o_lo, int ldq, int ldk, int ldv, int ldo, int Nq, int Nk, float scale) {
  extern __shared__ float sm32[];
  pdl_trigger();
  const int h = blockIdx.x, b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int KP = HD + 1, HD4 = HD / 4, NC = HD / 32;
  float* sK = sm32;                                           // [Nk][HD + 1]
  float* sV = sK + (((size_t)Nk * KP + 3) & ~(size_t)3);      // [Nk][HD], 16-byte aligned
  float* sQ = sV + (size_t)Nk * HD;                           // [8][HD]
  float* sP = sQ + 8 * HD;                                    // [8][Nk]
  pdl_wait();
  const int total = Nk * HD4;
#pragma unroll 4
  for (int i = threadIdx.x; i < total; i += 256) {
    const int j = i / HD4, c = (i - j * HD4) << 2;
    const float4 kv = __ldg(reinterpret_cast<const float4*>(k + (size_t)(b * Nk + j) * ldk + h * HD + c));
    const float4 vv = __ldg(reinterpret_cast<const float4*>(v + (size_t)(b * Nk + j) * ldv + h * HD + c));
    float* kd = sK + (size_t)j * KP + c;
    kd[0] = kv.x; kd[1] = kv.y; kd[2] = kv.z; kd[3] = kv.w;
    *reinterpret_cast<float4*>(sV + (size_t)j * HD + c) = vv;
  }
  __syncthreads();
  float* myq = sQ + warp * HD;
  float* myp = sP + (size_t)warp * Nk;
  const int kt = (Nk + 31) >> 5;
  for (int r = blockIdx.z * 8 + warp; r < Nq; r += gridDim.z * 8) {
    const float* qr = q + (size_t)(b * Nq + r) * ldq + h * HD;
#pragma unroll
    for (int c = 0; c < NC; ++c) myq[lane + 32 * c] = qr[lane + 32 * c];
    __syncwarp();
    float sc[ATT32_KT];
    const float* kr[ATT32_KT];
#pragma unroll
    for (int t = 0; t < ATT32_KT; ++t) { sc[t] = 0.f; kr[t] = sK + (size_t)min(lane + 32 * t, Nk - 1) * KP; }
#pragma unroll 4
    for (int d = 0; d < HD; ++d) {
      const float qd = myq[d];
#pragma unroll
      for (int t = 0; t < ATT32_KT; ++t) if (t < kt) sc[t] = fmaf(qd, kr[t][d], sc[t]);
    }
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < ATT32_KT; ++t) {
      sc[t] = (lane + 32 * t < Nk) ? sc[t] * scale : -INFINITY;
      mx = fmaxf(mx, sc[t]);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < ATT32_KT; ++t) {
      const float e = (lane + 32 * t < Nk) ? expf(sc[t] - mx) : 0.f;
      sc[t] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
#pragma unroll
    for (int t = 0; t < ATT32_KT; ++t) if (lane + 32 * t < Nk) myp[lane + 32 * t] = sc[t] * inv;
    __syncwarp();
    float acc[4][NC];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int c = 0; c < NC; ++c) acc[u][c] = 0.f;
    int j = 0;
    for (; j + 4 <= Nk; j += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float p = myp[j + u];
#pragma unroll
        for (int c = 0; c < NC; ++c) acc[u][c] = fmaf(p, sV[(size_t)(j + u) * HD + lane + 32 * c], acc[u][c]);
      }
    }
    for (; j < Nk; ++j) {
      const float p = myp[j];
#pragma unroll
      for (int c = 0; c < NC; ++c) acc[0][c] = fmaf(p, sV[(size_t)j * HD + lane + 32 * c], acc[0][c]);
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const float a = (acc[0][c] + acc[1][c]) + (acc[2][c] + acc[3][c]);
      __half hi, lo;
      split_x2(a, hi, lo);
      const size_t o = (size_t)(b * Nq + r) * ldo + h * HD + lane + 32 * c;
      o_hi[o] = hi; o_lo[o] = lo;
    }
    __syncwarp();
  }
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_preprocess_im2col(const uint8_t* d_img, uint8_t* d_mid, void* d_out, int B, int H, int W, int OH,
                                      int OW, int patch, int ldk, const int32_t* d_hbounds, const int32_t* d_hkk,
                                      int hksize, const int32_t* d_vbounds, const int32_t* d_vkk, int vksize,
                                      const float* h_mean3, const float* h_std3, void* stream) {
  if (!d_img || !d_mid || !d_out || !d_hbounds || !d_hkk || !d_vbounds || !d_vkk || !h_mean3 || !h_std3 ||
      OH % patch || OW % patch || B < 1 || B > 65535) { set_error("vlfm_preprocess_im2col: bad argument"); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 g1((OW * 3 + 127) / 128, H, B);
  resize_h_kernel<<<g1, 128, 0, st>>>(d_img, d_mid, H, W, OW, d_hbounds, d_hkk, hksize);
  VLFM_CHECK_LAUNCH("resize_h_kernel");
  dim3 g2((OW * 3 + 127) / 128, OH, B);
  resize_v_norm_im2col_kernel<<<g2, 128, 0, st>>>(d_mid, (__half*)d_out, H, OW, OH, d_vbounds, d_vkk, vksize, patch, ldk,
                                                  h_mean3[0], h_mean3[1], h_mean3[2], h_std3[0], h_std3[1], h_std3[2]);
  VLFM_CHECK_LAUNCH("resize_v_norm_im2col_kernel");
  count_launch(2);
  return VLFM_OK;
}

extern "C" int vlfm_assemble_tokens(const float* d_patch, const float* d_cls, const float* d_pos, float* d_x, int B,
                                    int T, int D, void* stream) {
  if (!d_patch || !d_cls || !d_pos || !d_x) { set_error("vlfm_assemble_tokens: null argument"); return VLFM_E_INVALID; }
  size_t n = (size_t)B * T * D;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  assemble_tokens_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_patch, d_cls, d_pos, d_x, B, T, D);
  VLFM_CHECK_LAUNCH("assemble_tokens_kernel");
  count_launch();
  return VLFM_OK;
}

namespace vlfm {
// The shape and alignment both LayerNorm kernels need, checked before anything launches (the resid-LN GEMMs run it before their
// GEMM, so a refused call leaves x and the workspace as they were).  D <= 1536; D and the strides multiples of 4; x, gamma, beta
// and out32 read / written as float4 (16-byte aligned), out16 and out_lo as 4 halves (8-byte aligned).  Null outputs are skipped.
int layernorm_check(const char* who, const float* d_x, const float* d_gamma, const float* d_beta, const void* d_out16, const void* d_out16_lo,
                    const float* d_out32, int D, int ldx, int ldo16, int ldo32) {
  if (D > LN_DMAX) { set_error("%s: D=%d too large (max %d)", who, D, LN_DMAX); return VLFM_E_UNSUPPORTED; }
  if ((D & 3) || (ldx & 3) || (ldo16 & 3) || (ldo32 & 3)) { set_error("%s: D and strides must be multiples of 4", who); return VLFM_E_UNSUPPORTED; }
  if (((uintptr_t)d_x & 15) || ((uintptr_t)d_gamma & 15) || ((uintptr_t)d_beta & 15) || ((uintptr_t)d_out32 & 15) ||
      ((uintptr_t)d_out16 & 7) || ((uintptr_t)d_out16_lo & 7)) {
    set_error("%s: x, gamma, beta, out32 must be 16-byte aligned, the fp16 outputs 8-byte aligned", who); return VLFM_E_INVALID; }
  return VLFM_OK;
}
}  // namespace vlfm

static int layernorm_impl(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out16, void* d_out16_lo, float* d_out32,
                          int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream) {
  __half* lo16 = (__half*)d_out16_lo;
  if (!d_x || !d_gamma || !d_beta || (!d_out16 && !d_out32) || rows < 1 || D < 1) { set_error("vlfm_layernorm: bad argument"); return VLFM_E_INVALID; }
  if (int rc = layernorm_check("vlfm_layernorm", d_x, d_gamma, d_beta, d_out16, d_out16_lo, d_out32, D, ldx, ldo16, ldo32)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((rows + 3) / 4);
  cudaError_t e;
  __half* o16 = (__half*)d_out16;
  if (D <= 128 * 2) e = launch_pdl(layernorm_kernel<2>, grid, dim3(128), 0, st, d_x, d_gamma, d_beta, o16, d_out32, rows, D, ldx, ldo16, ldo32, eps, lo16);
  else if (D <= 128 * 6) e = launch_pdl(layernorm_kernel<6>, grid, dim3(128), 0, st, d_x, d_gamma, d_beta, o16, d_out32, rows, D, ldx, ldo16, ldo32, eps, lo16);
  else e = launch_pdl(layernorm_kernel<12>, grid, dim3(128), 0, st, d_x, d_gamma, d_beta, o16, d_out32, rows, D, ldx, ldo16, ldo32, eps, lo16);
  { int rc = check_cuda(e, "layernorm_kernel"); if (rc) return rc; }
  count_launch();
  return VLFM_OK;
}
extern "C" int vlfm_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out16, float* d_out32,
                              int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream) {
  return layernorm_impl(d_x, d_gamma, d_beta, d_out16, nullptr, d_out32, rows, D, ldx, ldo16, ldo32, eps, stream);
}
// LayerNorm with the fp16 output split into x2 operands (hi, lo); d_out32 optional
extern "C" int vlfm_layernorm_x2(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32,
                                 int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream) {
  if (!d_out_hi || !d_out_lo) { set_error("vlfm_layernorm_x2: null output"); return VLFM_E_INVALID; }
  return layernorm_impl(d_x, d_gamma, d_beta, d_out_hi, d_out_lo, d_out32, rows, D, ldx, ldo16, ldo32, eps, stream);
}

namespace vlfm {
int layernorm_reduce_impl(float* d_x, const float* d_partials, const SplitK& sk, const float* d_gamma,
                          const float* d_beta, void* d_out16, void* d_out16_lo, float* d_out32, int rows, int D, int ldx, int ldo16, int ldo32,
                          float eps, void* stream) {
  __half* lo16 = (__half*)d_out16_lo;
  if (!d_x || !d_partials || !d_gamma || !d_beta || (!d_out16 && !d_out32) || rows < 1 || D < 1 || sk.splits < 0 || sk.splits > 16 ||
      (sk.splits == 0 && (sk.ctas < 1 || sk.row_tiles < 1 || sk.tiles != sk.row_tiles * ((D + SK_TILE - 1) / SK_TILE) || sk.num_k < 1))) {
    set_error("vlfm_layernorm_reduce: bad argument"); return VLFM_E_INVALID; }
  if (int rc = layernorm_check("vlfm_layernorm_reduce", d_x, d_gamma, d_beta, d_out16, d_out16_lo, d_out32, D, ldx, ldo16, ldo32)) return rc;
  if (sk.stride & 3) { set_error("vlfm_layernorm_reduce: D and strides must be multiples of 4"); return VLFM_E_UNSUPPORTED; }
  if ((uintptr_t)d_partials & 15) { set_error("vlfm_layernorm_reduce: partials must be 16-byte aligned"); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(rows);
  __half* o16 = (__half*)d_out16;
  cudaError_t e;
  const int threads = (((D >> 2) + 31) / 32) * 32;
  e = launch_pdl(layernorm_reduce_kernel, grid, dim3(threads), 0, st, d_x, d_partials, sk, d_gamma, d_beta, o16, d_out32, rows, D, ldx, ldo16, ldo32, eps, lo16);
  { int rc = check_cuda(e, "layernorm_reduce_kernel"); if (rc) return rc; }
  count_launch();
  return VLFM_OK;
}
}  // namespace vlfm
extern "C" int vlfm_layernorm_reduce(float* d_x, const float* d_partials, int splits, long long split_stride, const float* d_gamma,
                                     const float* d_beta, void* d_out16, float* d_out32, int rows, int D, int ldx, int ldo16, int ldo32,
                                     float eps, void* stream) {
  if (splits < 1) { set_error("vlfm_layernorm_reduce: bad argument"); return VLFM_E_INVALID; }
  return layernorm_reduce_impl(d_x, d_partials, SplitK{splits, split_stride}, d_gamma, d_beta, d_out16, nullptr, d_out32, rows, D, ldx, ldo16, ldo32, eps, stream);
}
extern "C" int vlfm_layernorm_reduce_x2(float* d_x, const float* d_partials, int splits, long long split_stride, const float* d_gamma,
                                        const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32, int rows, int D, int ldx, int ldo16,
                                        int ldo32, float eps, void* stream) {
  if (!d_out_hi || !d_out_lo) { set_error("vlfm_layernorm_reduce_x2: null output"); return VLFM_E_INVALID; }
  if (splits < 1) { set_error("vlfm_layernorm_reduce_x2: bad argument"); return VLFM_E_INVALID; }
  return layernorm_reduce_impl(d_x, d_partials, SplitK{splits, split_stride}, d_gamma, d_beta, d_out_hi, d_out_lo, d_out32, rows, D, ldx, ldo16, ldo32, eps, stream);
}

extern "C" int vlfm_attention_f16(const void* d_q, const void* d_k, const void* d_v, void* d_o, int B, int heads, int Nq,
                                  int Nk, int hd, int ldq, int ldk, int ldv, int ldo, float scale, void* stream) {
  if (!d_q || !d_k || !d_v || !d_o || B < 1 || heads < 1 || Nq < 1 || Nk < 1) { set_error("vlfm_attention_f16: bad argument"); return VLFM_E_INVALID; }
  if (Nk > ATT_NKMAX || hd > 96 || (hd & 7) || (ldq & 7) || (ldk & 7) || (ldv & 7) || (ldo & 1) || B > 65535) {
    set_error("vlfm_attention_f16: unsupported shape (Nk<=%d, hd<=96 and %%8==0, strides %%8==0)", ATT_NKMAX); return VLFM_E_UNSUPPORTED; }
  AttnArgs a{(const __half*)d_q, (const __half*)d_k, (const __half*)d_v, (__half*)d_o, ldq, ldk, ldv, ldo, Nq, Nk, hd, heads,
             scale * 1.4426950408889634f};
  cudaStream_t st = (cudaStream_t)stream;
  // VLFM_ATT_IMPL: unset = by shape; "legacy" = never the batch-1 kernel; "b1" = the batch-1 kernel for every shape (tests)
  const char* impl = getenv("VLFM_ATT_IMPL");
  const bool force_legacy = impl && !strcmp(impl, "legacy"), force_b1 = impl && !strcmp(impl, "b1");
  if (impl && impl[0] && !force_legacy && !force_b1) { set_error("vlfm_attention_f16: VLFM_ATT_IMPL=%s (legacy or b1)", impl); return VLFM_E_INVALID; }
  const size_t nkp = ((size_t)Nk + 15) & ~(size_t)15;
  const int hdp = hd <= 64 ? 64 : 96;
  // the batch-1 kernel when its 64-row blocks fit one wave of one CTA per SM and the keys fill at least one 64-key chunk (the
  // ViT-g at batch 1); the short attentions of MobileSAM and every larger batch keep the variants below
  const long items64 = (long)B * heads * ((Nq + ATT_B1_ROWS - 1) / ATT_B1_ROWS);
  if (force_b1 || (!force_legacy && items64 <= 132 && Nk >= 64)) {
    static bool cfg_b1 = false;
    if (!cfg_b1) {
      const int mx = attn_b1_bar_offset(ATT_NKMAX, 96) + 8 * ATT_B1_BARS;
      int rc = check_cuda(cudaFuncSetAttribute(attention_kernel<64, 4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx), "attr(attention b1)");
      if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<96, 4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx), "attr(attention b1)");
      if (rc) return rc;
      cfg_b1 = true;
    }
    const size_t sm = attn_b1_bar_offset((int)nkp, hdp) + 8 * ATT_B1_BARS;
    const dim3 grid((Nq + ATT_B1_ROWS - 1) / ATT_B1_ROWS, heads, B);
    cudaError_t e = hdp == 64 ? launch_pdl(attention_kernel<64, 4, true>, grid, dim3(ATT_B1_THREADS), sm, st, a)
                              : launch_pdl(attention_kernel<96, 4, true>, grid, dim3(ATT_B1_THREADS), sm, st, a);
    { int rc = check_cuda(e, "attention_kernel (batch 1)"); if (rc) return rc; }
    count_launch();
    return VLFM_OK;
  }
  // few (batch, head, block) work items -> 32-row blocks with split keys (4-way when they fit one wave of 8-warp CTAs,
  // else 2-way); many -> 64-row blocks
  const long items = (long)B * heads * ((Nq + 31) / 32);
  const bool big = items > 2 * 264;
  static int kh4 = -1;
  if (kh4 < 0) { const char* e = getenv("VLFM_ATT_KH4"); kh4 = e ? atoi(e) : 1; }
  const bool quad = !big && kh4 && items <= 264 && Nk >= 64;
  const int qblk = big ? 64 : 32;
  dim3 grid((Nq + qblk - 1) / qblk, heads, B);
  static bool cfg = false;
  if (!cfg) {
    int rc = check_cuda(cudaFuncSetAttribute(attention_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (64 + 8) * 2), "attr(attention)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (64 + 8) * 2), "attr(attention)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<96, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (96 + 8) * 2), "attr(attention)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<96, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (96 + 8) * 2), "attr(attention)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<64, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (64 + 8) * 2), "attr(attention)");
    if (!rc) rc = check_cuda(cudaFuncSetAttribute(attention_kernel<96, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * ATT_NKMAX * (96 + 8) * 2), "attr(attention)");
    if (rc) return rc;
    cfg = true;
  }
  size_t sm = 2 * nkp * (hdp + 8) * 2;
  if (sm < 6 * 52 * 32 * 4) sm = 6 * 52 * 32 * 4;   // merge buffer of the split-key variants
  cudaError_t e;
  if (quad) e = hdp == 64 ? launch_pdl(attention_kernel<64, 4>, grid, dim3(256), sm, st, a) : launch_pdl(attention_kernel<96, 4>, grid, dim3(256), sm, st, a);
  else if (hdp == 64) e = big ? launch_pdl(attention_kernel<64, 1>, grid, dim3(32 * ATT_WARPS), sm, st, a) : launch_pdl(attention_kernel<64, 2>, grid, dim3(32 * ATT_WARPS), sm, st, a);
  else e = big ? launch_pdl(attention_kernel<96, 1>, grid, dim3(32 * ATT_WARPS), sm, st, a) : launch_pdl(attention_kernel<96, 2>, grid, dim3(32 * ATT_WARPS), sm, st, a);
  { int rc = check_cuda(e, "attention_kernel"); if (rc) return rc; }
  count_launch();
  return VLFM_OK;
}

// softmax(q k^T * scale) v in float32 for small problems (Q-Former); q, k, v fp32 rows (b * N + i), head h at columns [h*hd, (h+1)*hd);
// output as x2 operands (hi, lo fp16, same stride).  hd in {32, 64}, Nk <= 272.
extern "C" int vlfm_attention_f32(const float* d_q, const float* d_k, const float* d_v, void* d_o_hi, void* d_o_lo, int B, int heads, int Nq,
                                  int Nk, int hd, int ldq, int ldk, int ldv, int ldo, float scale, void* stream) {
  if (!d_q || !d_k || !d_v || !d_o_hi || !d_o_lo || B < 1 || heads < 1 || Nq < 1 || Nk < 1) { set_error("vlfm_attention_f32: bad argument"); return VLFM_E_INVALID; }
  if (Nk > ATT32_NKMAX || (hd != 32 && hd != 64) || (ldk & 3) || (ldv & 3) || B > 65535) {
    set_error("vlfm_attention_f32: unsupported shape (Nk<=%d, hd in {32,64}, strides %%4==0)", ATT32_NKMAX); return VLFM_E_UNSUPPORTED; }
  const size_t smem = ((((size_t)Nk * (hd + 1) + 3) & ~(size_t)3) + (size_t)Nk * hd + 8 * hd + 8 * (size_t)Nk) * 4;
  static size_t cfg32 = 0, cfg64 = 0;
  size_t& cfg = hd == 32 ? cfg32 : cfg64;
  if (smem > 48 * 1024 && smem > cfg) {
    int rc = hd == 32 ? check_cuda(cudaFuncSetAttribute(attention_f32_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(attention_f32)")
                      : check_cuda(cudaFuncSetAttribute(attention_f32_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "attr(attention_f32)");
    if (rc) return rc; cfg = smem;
  }
  // row groups: enough CTAs to cover the machine when few (image, head) pairs exist; every CTA stages K / V once
  int z = (Nq + 7) / 8;
  while (z > 1 && (long)heads * B * z > 2 * 132) --z;
  const dim3 grid(heads, B, z);
  cudaError_t e = hd == 32 ? launch_pdl(attention_f32_kernel<32>, grid, dim3(256), smem, (cudaStream_t)stream, d_q, d_k, d_v, (__half*)d_o_hi, (__half*)d_o_lo,
                                        ldq, ldk, ldv, ldo, Nq, Nk, scale)
                           : launch_pdl(attention_f32_kernel<64>, grid, dim3(256), smem, (cudaStream_t)stream, d_q, d_k, d_v, (__half*)d_o_hi, (__half*)d_o_lo,
                                        ldq, ldk, ldv, ldo, Nq, Nk, scale);
  { int rc = check_cuda(e, "attention_f32_kernel"); if (rc) return rc; }
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_split_x2(const float* d_src, void* d_hi, void* d_lo, long long n, void* stream) {
  if (!d_src || !d_lo || n < 4 || (n & 3) || ((uintptr_t)d_src & 15) || ((uintptr_t)d_lo & 7) || ((uintptr_t)d_hi & 7)) {
    set_error("vlfm_split_x2: bad argument (n %% 4 == 0, aligned pointers)"); return VLFM_E_INVALID; }
  long blocks = (n / 4 + 255) / 256; if (blocks > 132 * 8) blocks = 132 * 8;
  cudaError_t e = launch_pdl(split_x2_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, d_src, (__half*)d_hi, (__half*)d_lo, (long)(n / 4));
  { int rc = check_cuda(e, "split_x2_kernel"); if (rc) return rc; }
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_itc_head_multi(const float* d_proj, const float* d_text, float* d_out, int B, int P, int Q, int D, int ldo,
                                   void* stream) {
  if (!d_proj || !d_text || !d_out || B < 1 || P < 1 || Q < 1 || D < 1 || ldo < P || (size_t)Q * sizeof(float) > 48 * 1024) {
    set_error("vlfm_itc_head_multi: bad argument (B, P, Q, D >= 1, ldo >= P, Q <= 12288)"); return VLFM_E_INVALID; }
  itc_head_kernel<<<B, 256, Q * sizeof(float), (cudaStream_t)stream>>>(d_proj, d_text, d_out, P, Q, D, ldo);
  VLFM_CHECK_LAUNCH("itc_head_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_itc_head(const float* d_proj, const float* d_text, float* d_out, int B, int Q, int D, void* stream) {
  if (!d_proj || !d_text || !d_out || B < 1) { set_error("vlfm_itc_head: bad argument"); return VLFM_E_INVALID; }
  return vlfm_itc_head_multi(d_proj, d_text, d_out, B, 1, Q, D, 1, stream);
}
