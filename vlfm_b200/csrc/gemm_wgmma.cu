// fp16 x fp16 -> fp32 GEMM on Hopper tensor cores (wgmma + TMA + mbarrier).
//
//   out[M,N] = epilogue(A[M,K] @ W[N,K]^T + bias[N])      A, W row-major (K-major)
//
// Replaces the nn.Linear layers of the BLIP-2 ViT-g / Q-Former forward that
// vlfm/vlm/blip2itm.py:52 runs through lavis (fp16 autocast in the reference).
//
// Structure (one 128 x BN output tile per CTA, 384 threads = three warpgroups):
//   warpgroup 0   warp 0, one thread: TMA producer.  cp.async.bulk.tensor 2D loads of the A (128x64)
//                 and W (BNx64) K-slices into a STAGES-deep 128B-swizzled smem ring, mbarrier
//                 complete_tx signalling.  The other three warps have nothing to do and exit.
//   warpgroups 1-2  consumers: each owns 64 rows of the tile.  wgmma.mma_async m64nBNk16 (both operands
//                 read from shared memory through matrix descriptors, fp32 accumulators in registers),
//                 one wgmma group in flight while the next stage is awaited; a stage goes back to the
//                 producer when the group that read it has retired.  Then the epilogue from the
//                 accumulator fragments: fused bias / GELU(erf) / fp32-residual-add, paired stores.
// M / N / K tails are handled by TMA out-of-bounds zero fill + store guards.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"

namespace vlfm {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 fp16 = 128 bytes = one swizzle atom row
constexpr int GEMM_THREADS = 384;     // warpgroup 0 TMA producer, warpgroups 1-2 wgmma consumers + epilogue
constexpr int GEMM_CONSUMERS = 256;   // threads of the two consumer warpgroups

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (cute::GmmaDescriptor):
// start>>4 | LBO(1, unused for swizzled K-major)<<16 | SBO(1024B>>4)<<32 | layout SWIZZLE_128B(1)<<62
__device__ __forceinline__ uint64_t wgmma_desc_k128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// D[64, BN] (+)= A[64, 16] . B[BN, 16]^T, operands from shared memory, D = BN/2 fp32 registers per thread.
// Fragment of thread t of the warpgroup: rows 16*(t/32) + (t%32)/4 (+8), columns 8*j + 2*(t%4) (+1);
// d[4*j + 0,1] is the upper row's column pair, d[4*j + 2,3] the lower row's.
#define VLFM_D4(d, i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define VLFM_D16(d, i) VLFM_D4(d, i), VLFM_D4(d, i + 4), VLFM_D4(d, i + 8), VLFM_D4(d, i + 12)
template <int BN> struct Wgmma;
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : VLFM_D16(d, 0) : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : VLFM_D16(d, 0), VLFM_D16(d, 16) : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wgmma<96> {
  static __device__ __forceinline__ void mma(float (&d)[48], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : VLFM_D16(d, 0), VLFM_D16(d, 16), VLFM_D16(d, 32) : "l"(a), "l"(b), "r"(acc));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : VLFM_D16(d, 0), VLFM_D16(d, 16), VLFM_D16(d, 32), VLFM_D16(d, 48) : "l"(a), "l"(b), "r"(acc));
  }
};
#undef VLFM_D16
#undef VLFM_D4

struct GemmArgs {
  const float* bias;
  void* out;
  int M, N, K, ldo, epi;
  int kb_per_split;   // K-blocks per grid.z slice (split-K, residual epilogue only)
  // VLFM_EPI_PARTIAL_F32 (deterministic split-K): split z stores its tile at out + z * split_stride (plain stores, no atomics);
  // the consumer (layernorm_reduce_kernel) adds the partial sums to the residual stream in a fixed order
  long long split_stride;
  // "tail rows": when M = 128*q + r with 1 <= r <= GEMM_TAIL_MAX (ViT: 257 tokens), only q row tiles are launched and the CTAs
  // of the last one also compute the r extra rows on CUDA cores from the W tiles already staged for the tensor core
  const __half* a_tail; int lda, tail_rows, tail_row0;
  void* out_lo;       // VLFM_EPI_BIAS_GELU_F16X2: the x2 residual of the fp16 output (same ldo)
  // rows of the A tile the TMA box carries (32 / 64 / 128): with M <= 32 (Q-Former queries, text tokens) a 128-row box spends 3/4 of
  // every stage's TMA time on out-of-bounds zero fill.  Rows of the smem tile beyond the box keep whatever they held: row i of the
  // accumulator depends on row i of A only, and rows >= M are never stored.
  int a_box_rows;
  SplitK sk;          // sk.ctas > 0: stream-K launch (1-D grid of sk.ctas CTAs, BN = SK_TILE); `out` is the slab workspace
};
constexpr int GEMM_TAIL_MAX = 2;
static_assert(SK_SLAB_ROWS == BM + GEMM_TAIL_MAX && SK_TILE == BM, "stream-K slab = one 128 x 128 tile + its tail rows");
constexpr int GEMM_TAIL_KMAX = 6144;   // K elements of one CTA's slice that fit the tail-row staging buffer

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// torch's SiLU in fp32 (the opmath of its fp16 kernel)
__device__ __forceinline__ float silu(float x) { return x / (1.f + expf(-x)); }

// One column pair (n, n + 1) of one output row: activation, conversion and the store the epilogue kind asks for.
// v0 / v1 already carry the bias.  `pair` = column n + 1 exists.
__device__ __forceinline__ void epilogue_store2(const GemmArgs& g, int row, int n, float v0, float v1, bool pair, bool split) {
  const size_t idx = (size_t)row * g.ldo + n;
  if (g.epi == VLFM_EPI_BIAS_F16 || g.epi == VLFM_EPI_BIAS_GELU_F16 || g.epi == VLFM_EPI_BIAS_RELU_F16 || g.epi == VLFM_EPI_BIAS_GELU_F16X2) {
    if (g.epi == VLFM_EPI_BIAS_GELU_F16 || g.epi == VLFM_EPI_BIAS_GELU_F16X2) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
    else if (g.epi == VLFM_EPI_BIAS_RELU_F16) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    __half* o = reinterpret_cast<__half*>(g.out) + idx;
    const __half2 h = __floats2half2_rn(v0, v1);
    if (pair) *reinterpret_cast<__half2*>(o) = h; else o[0] = __low2half(h);
    if (g.epi == VLFM_EPI_BIAS_GELU_F16X2) {
      const float2 f = __half22float2(h);
      const __half2 l = __floats2half2_rn((v0 - f.x) * X2_SCALE, (v1 - f.y) * X2_SCALE);
      __half* ol = reinterpret_cast<__half*>(g.out_lo) + idx;
      if (pair) *reinterpret_cast<__half2*>(ol) = l; else ol[0] = __low2half(l);
    }
  } else {
    const bool partial = (g.epi == VLFM_EPI_PARTIAL_F32);
    float* o = reinterpret_cast<float*>(g.out) + (partial ? (size_t)blockIdx.z * (size_t)g.split_stride : 0) + idx;
    if (split && !partial) {
      atomicAdd(o, v0);
      if (pair) atomicAdd(o + 1, v1);
    } else if (pair) {
      float2 t = make_float2(v0, v1);
      if (g.epi == VLFM_EPI_BIAS_RESID_F32) { const float2 old = *reinterpret_cast<const float2*>(o); t.x += old.x; t.y += old.y; }
      *reinterpret_cast<float2*>(o) = t;
    } else {
      o[0] = (g.epi == VLFM_EPI_BIAS_RESID_F32) ? o[0] + v0 : v0;
    }
  }
}

// VLFM_EPI_BIAS_SILU_F16: SiLU -> fp16.  Its own kernel instantiation (SILU = true below), so that the other epilogues' code is
// exactly what it was without it.
__device__ __forceinline__ void epilogue_store2_silu(const GemmArgs& g, int row, int n, float v0, float v1, bool pair) {
  __half* o = reinterpret_cast<__half*>(g.out) + (size_t)row * g.ldo + n;
  const __half2 h = __floats2half2_rn(silu(v0), silu(v1));
  if (pair) *reinterpret_cast<__half2*>(o) = h; else o[0] = __low2half(h);
}

// Epilogue of one warp's 16 x BN accumulator slab, straight from the wgmma fragment.  `row0` = first row of the slab;
// `sbias` = this tile's bias slice in shared memory (zero-filled past N / without bias), added when `addb` (the first K split).
template <int BN, bool SILU = false>
__device__ __forceinline__ void epilogue_frag(const float (&acc)[BN / 2], int row0, int n_blk, const GemmArgs& g, bool split, bool addb, const float* sbias) {
  const int lane = threadIdx.x & 31;
  const int r_up = row0 + (lane >> 2), cq = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int cl = j * 8 + cq, n = n_blk * BN + cl;
    if (n >= g.N) continue;
    const bool pair = n + 1 < g.N;
    const float b0 = addb ? sbias[cl] : 0.f, b1 = addb ? sbias[cl + 1] : 0.f;
    if constexpr (SILU) {
      if (r_up < g.M) epilogue_store2_silu(g, r_up, n, acc[4 * j] + b0, acc[4 * j + 1] + b1, pair);
      if (r_up + 8 < g.M) epilogue_store2_silu(g, r_up + 8, n, acc[4 * j + 2] + b0, acc[4 * j + 3] + b1, pair);
    } else {
      if (r_up < g.M) epilogue_store2(g, r_up, n, acc[4 * j] + b0, acc[4 * j + 1] + b1, pair, split);
      if (r_up + 8 < g.M) epilogue_store2(g, r_up + 8, n, acc[4 * j + 2] + b0, acc[4 * j + 3] + b1, pair, split);
    }
  }
}

// Shared-memory carve-up common to both kernels: the tile ring (1024-byte aligned for the 128B swizzle), then the
// full / empty barriers of the ring, then the bias slice.
__device__ __forceinline__ uint8_t* smem_align_1024(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
}

// Stream-K segment store: this warp's 16 x BN slab of the accumulator (+ bias when the segment starts at K-block 0) into the
// tile's slab of the workspace (SplitK in common.cuh).  Every column and row of the slab is written; the reduction reads those < N, < M.
template <int BN>
__device__ __forceinline__ void segment_store_frag(const float (&acc)[BN / 2], int row0, int n_blk, const GemmArgs& g, bool addb, float* slab) {
  const int lane = threadIdx.x & 31;
  const int r_up = row0 + (lane >> 2), cq = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int cl = j * 8 + cq, n = n_blk * BN + cl;
    const float b0 = (addb && g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f, b1 = (addb && g.bias && n + 1 < g.N) ? __ldg(g.bias + n + 1) : 0.f;
    *reinterpret_cast<float2*>(slab + (size_t)r_up * BN + cl) = make_float2(acc[4 * j] + b0, acc[4 * j + 1] + b1);
    *reinterpret_cast<float2*>(slab + (size_t)(r_up + 8) * BN + cl) = make_float2(acc[4 * j + 2] + b0, acc[4 * j + 3] + b1);
  }
}

// A CTA works through iterations [it0, it1) of a sequence of (output tile, K-block) pairs.  A grid launch gives it one tile
// (blockIdx.x, blockIdx.y) and the K-blocks of split blockIdx.z.  A stream-K launch (g.sk.ctas > 0, 1-D grid) gives it a range
// of the sequence of all tiles' K-blocks (SplitK in common.cuh), which may cover parts of two tiles: the producer streams straight
// across the tile boundary, and the consumers finish a segment there (store it to the workspace, zero the accumulators) and go on.
template <int BN, int STAGES, bool SILU = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmArgs g) {
  constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* sA = smem_align_1024(smem_raw);
  uint8_t* sB = sA + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);
  float* sbias = reinterpret_cast<float*>(bars + 2 * STAGES);   // [BN], 16-byte aligned (tiles are 1024-byte multiples)

  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = (g.K + BK - 1) / BK;
  const bool sk = g.sk.ctas > 0;
  const int it0 = sk ? g.sk.sk_begin(blockIdx.x) : blockIdx.z * g.kb_per_split;
  const int it1 = sk ? g.sk.sk_begin(blockIdx.x + 1) : min(nk, it0 + g.kb_per_split);
  const int last_m = sk ? g.sk.row_tiles - 1 : (int)gridDim.y - 1;
  auto coords = [&](int it, int& m_blk, int& n_blk, int& kb) {
    if (sk) { const int t = it / nk; kb = it - t * nk; m_blk = t % g.sk.row_tiles; n_blk = t / g.sk.row_tiles; }
    else { kb = it; m_blk = blockIdx.y; n_blk = blockIdx.x; }
  };
  const bool split = !sk && gridDim.z > 1;
  // tail rows (see GemmArgs): a grid CTA of the last row tile stages its K slice of them; a stream-K CTA whose range touches a
  // tile of the last row stages the whole K (at most GEMM_TAIL_KMAX, checked by the host plan)
  int m_first, n_first, kb_first;
  coords(it0, m_first, n_first, kb_first);
  // (tiles t of the last row: t % row_tiles == row_tiles - 1; floor((t + 1) / row_tiles) of them lie in [0, t])
  const bool tail_cta = g.tail_rows > 0 &&
      (sk ? ((it1 - 1) / nk + 1) / g.sk.row_tiles > (it0 / nk) / g.sk.row_tiles : m_first == last_m);
  const int kb_lo = sk ? 0 : it0, kb_hi = sk ? nk : it1;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    // a stage is full when its TMA bytes have landed and empty again when each of the eight consumer warps has let go of it
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, GEMM_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // Weights do not depend on the predecessor kernel: start streaming the first STAGES W tiles BEFORE the
      // programmatic-dependency wait (hides the HBM/L2 latency of the first loads behind the predecessor's tail);
      // the matching A tiles (activations) are issued right after the wait and complete the same barriers.
      const int pre = min(it1 - it0, STAGES);
      const uint32_t a_tx = (uint32_t)g.a_box_rows * BK * 2;
      int m_blk, n_blk, kb;
      for (int i = 0; i < pre; ++i) {
        coords(it0 + i, m_blk, n_blk, kb);
        mbar_expect_tx(full0 + 8 * i, a_tx + B_BYTES);
        tma_load_2d(smem_u32(sB + i * B_BYTES), &tmB, kb * BK, n_blk * BN, full0 + 8 * i);
      }
      pdl_wait();
      for (int i = 0; i < pre; ++i) {
        coords(it0 + i, m_blk, n_blk, kb);
        tma_load_2d(smem_u32(sA + i * A_BYTES), &tmA, kb * BK, m_blk * BM, full0 + 8 * i);
      }
      int s = pre == STAGES ? 0 : pre; uint32_t ph = pre == STAGES ? 1 : 0;
      for (int it = it0 + pre; it < it1; ++it) {
        coords(it, m_blk, n_blk, kb);
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        mbar_expect_tx(full0 + 8 * s, a_tx + B_BYTES);
        tma_load_2d(smem_u32(sA + s * A_BYTES), &tmA, kb * BK, m_blk * BM, full0 + 8 * s);
        tma_load_2d(smem_u32(sB + s * B_BYTES), &tmB, kb * BK, n_blk * BN, full0 + 8 * s);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ---- consumers: warpgroup wg owns rows [64 * wg, +64) of the tile, warp wq of it rows [16 * wq, +16) of those.
    // wg is broadcast from lane 0 so that ptxas can treat it as warp-uniform.  Computed from threadIdx alone, it makes the
    // `!active` branch below look divergent, and ptxas then serialises every wgmma of the loop (warning C7518): a wait after
    // each one, so no group stays in flight across K-blocks (DESIGN §3.3).
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0), wq = warp & 3;
    const int et = threadIdx.x - (GEMM_THREADS - GEMM_CONSUMERS);
    // a warpgroup whose rows are all past M issues no MMA (a stream-K range may span row tiles: there both always compute)
    const bool active = sk || m_first * BM + wg * 64 < g.M;
    // bias is a weight (no dependency on the predecessor): stage this tile's slice while the first loads are in flight.
    // (Stream-K segments read it from global memory: their tiles change along the range.)
    if (!sk && et < BN) { const int n = n_first * BN + et; sbias[et] = (g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f; }
    asm volatile("bar.sync 1, 256;" ::: "memory");   // the eight consumer warps only
    pdl_wait();          // residual stream / output buffers of the predecessor are visible
    // ---- tail rows on CUDA cores: thread = (feature f of this tile, K half hk); W from the 128B-swizzled stage
    const int f = et >> 1, hk = et & 1;
    float tacc[GEMM_TAIL_MAX];
    __half* sx = reinterpret_cast<__half*>(sbias + BN);
    const int kslice = (kb_hi - kb_lo) * BK, kbase = kb_lo * BK;
    if (tail_cta) {
      // stage the K slice of the tail rows once (global latency must not sit between "stage full" and "stage released")
      for (int i = et; i < g.tail_rows * (kslice >> 3); i += GEMM_CONSUMERS) {
        const int r = i / (kslice >> 3), c8 = (i - r * (kslice >> 3)) << 3;
        uint4 xv = make_uint4(0u, 0u, 0u, 0u);
        if (kbase + c8 < g.K) xv = __ldg(reinterpret_cast<const uint4*>(g.a_tail + (size_t)r * g.lda + kbase + c8));
        *reinterpret_cast<uint4*>(sx + (size_t)r * kslice + c8) = xv;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    if (!active) {     // keep the ring turning for the other warpgroup: take every stage and hand it straight back
      int s = 0; uint32_t ph = 0;
      for (int it = it0; it < it1; ++it) {
        mbar_wait(full0 + 8 * s, ph);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * s);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      return;
    }
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    bool held = false;       // the stage before s is still held (its wgmma group may be in flight)
    bool addb = false;       // the current segment starts at K-block 0: it carries the bias
    for (int it = it0; it < it1; ++it) {
      int m_blk, n_blk, kb;
      coords(it, m_blk, n_blk, kb);
      const bool seg_first = it == it0 || kb == 0, seg_last = it + 1 == it1 || kb + 1 == nk;
      const bool tail_seg = tail_cta && m_blk == last_m;
      if (seg_first) {
        addb = kb == 0;
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r) tacc[r] = 0.f;
      }
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t a0 = smem_u32(sA + s * A_BYTES) + (uint32_t)wg * (64 * BK * 2), b0 = smem_u32(sB + s * B_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        Wgmma<BN>::mma(acc, wgmma_desc_k128(a0 + k * 32), wgmma_desc_k128(b0 + k * 32), (!seg_first || k > 0) ? 1u : 0u);
      wg_commit();
      if (tail_seg && f < BN) {     // overlaps the MMAs just issued
        const uint8_t* wrow = sB + (size_t)s * B_BYTES + (size_t)f * 128;
        const int k0 = (kb - kb_lo) * BK + hk * 32;          // offset inside the staged slice
        uint4 wv[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) wv[c] = *reinterpret_cast<const uint4*>(wrow + (((hk * 4 + c) ^ (f & 7)) << 4));
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r) {
          if (r < g.tail_rows) {
            const __half* xr = sx + (size_t)r * kslice + k0;
            float a = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {                    // chunks past K were staged as zeros (and W is zero-filled by TMA)
              const uint4 xv = *reinterpret_cast<const uint4*>(xr + c * 8);
              const __half2* xh = reinterpret_cast<const __half2*>(&xv);
              const __half2* wh = reinterpret_cast<const __half2*>(&wv[c]);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 xf = __half22float2(xh[e]), wf = __half22float2(wh[e]);
                a = fmaf(xf.x, wf.x, a); a = fmaf(xf.y, wf.y, a);
              }
            }
            tacc[r] += a;
          }
        }
      }
      // the group issued one K-block ago has retired once at most one is pending: its stage goes back to the producer
      wg_wait<1>();
      if (held) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * (s == 0 ? STAGES - 1 : s - 1));
      }
      held = true;
      if (seg_last) {
        wg_wait<0>();
        if (sk) {            // this stage is done with: hand it back before the segment's stores
          __syncwarp();
          if (lane == 0) mbar_arrive(empty0 + 8 * s);
          held = false;
        }
        float* slab = sk ? reinterpret_cast<float*>(g.out) + (size_t)(blockIdx.x + n_blk * g.sk.row_tiles + m_blk) * SK_SLAB : nullptr;
        if (tail_seg) {
#pragma unroll
          for (int r = 0; r < GEMM_TAIL_MAX; ++r) tacc[r] += __shfl_xor_sync(0xffffffffu, tacc[r], 1);
          const int n = n_blk * BN + f;
          if (hk == 0 && f < BN && (sk || n < g.N)) {
#pragma unroll
            for (int r = 0; r < GEMM_TAIL_MAX; ++r) {
              if (r < g.tail_rows) {
                if (sk) {
                  slab[(size_t)(BM + r) * BN + f] = tacc[r] + ((addb && g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f);
                  continue;
                }
                float v = tacc[r] + (addb ? sbias[f] : 0.f);
                const size_t o = (size_t)(g.tail_row0 + r) * g.ldo + n;
                if (SILU || g.epi == VLFM_EPI_BIAS_F16 || g.epi == VLFM_EPI_BIAS_GELU_F16 || g.epi == VLFM_EPI_BIAS_RELU_F16) {
                  if constexpr (SILU) v = silu(v);
                  else if (g.epi == VLFM_EPI_BIAS_GELU_F16) v = gelu_erf(v);
                  else if (g.epi == VLFM_EPI_BIAS_RELU_F16) v = fmaxf(v, 0.f);
                  reinterpret_cast<__half*>(g.out)[o] = __float2half_rn(v);
                } else {
                  const bool partial = (g.epi == VLFM_EPI_PARTIAL_F32);
                  float* po = reinterpret_cast<float*>(g.out) + (partial ? (size_t)blockIdx.z * (size_t)g.split_stride : 0) + o;
                  if (split && !partial) atomicAdd(po, v);
                  else *po = (g.epi == VLFM_EPI_BIAS_RESID_F32) ? *po + v : v;
                }
              }
            }
          }
        }
        if (sk) {
          segment_store_frag<BN>(acc, wg * 64 + wq * 16, n_blk, g, addb, slab);
        } else {
          epilogue_frag<BN, SILU>(acc, m_blk * BM + wg * 64 + wq * 16, n_blk, g, split, addb, sbias);
        }
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  }
}

// ================================================================================================
// Batch-1 ViT GEMMs (256 < M <= 256 + GEMM_TAIL_MAX, the caller allows a cluster split): one 256 x BN tile covers all rows, so
// every weight byte is delivered to one CTA only, and K is split over the s CTAs of a thread-block cluster.
//   warpgroup 0     warp 0, one thread: TMA producer (A 256 x 64 and W BN x 64 per stage), as in gemm_f16_wgmma_kernel.
//   warpgroups 1-4  consumers, 64 rows each (m64nBNk16); the consumer threads of warpgroups 1-2 also compute the tail rows
//                   (rows 256, 257) on CUDA cores from the swizzled W stages.
// CTA r of the cluster runs K-blocks [r nk / s, (r + 1) nk / s).  After its slice it stores the fp32 accumulators and tail-row
// sums into its own shared memory (over the ring), one cluster barrier publishes them, and CTA r reduces rows
// [r R / s, (r + 1) R / s) of the R = M rows by reading every peer's tile (ld.shared::cluster) in rank order 0..s-1, adds the
// bias once and runs the epilogue: one writer per element, nothing through global memory, the same bits on every run.
// A second cluster barrier keeps each CTA's shared memory alive until its peers have read it.  The cluster is touched only
// after the main loop: the K loop has no cluster-scope barrier.
// ================================================================================================
constexpr int CS_BM = 256;
constexpr int CS_THREADS = 640;      // warpgroup 0 TMA producer, warpgroups 1-4 consumers
constexpr int CS_CONSUMERS = 512;

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  __syncwarp();
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float2 ld_peer_f2(uint32_t saddr, uint32_t rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(saddr), "r"(rank));
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(CS_THREADS, 1)
gemm_f16_csplit_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmArgs g) {
  constexpr uint32_t A_BYTES = CS_BM * BK * 2, B_BYTES = BN * BK * 2;
  constexpr int LDP = BN + 8;   // row stride (floats) of the fp32 partial tile: rows 32 bytes apart, conflict-free fragment stores
  static_assert((size_t)(CS_BM + GEMM_TAIL_MAX) * LDP * 4 <= (size_t)STAGES * (A_BYTES + B_BYTES), "partial tile must fit the ring");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* sA = smem_align_1024(smem_raw);
  uint8_t* sB = sA + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);
  float* sbias = reinterpret_cast<float*>(bars + 2 * STAGES);   // [BN]
  __half* sx = reinterpret_cast<__half*>(sbias + BN);           // the tail rows' K slice
  float* part = reinterpret_cast<float*>(sA);                    // after the K loop: [CS_BM + tail_rows][LDP] fp32, over the ring

  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = (g.K + BK - 1) / BK;
  const int s_cl = (int)cluster_nctarank(), rank = (int)cluster_ctarank();
  const int n_blk = blockIdx.x / s_cl;
  const int kb_lo = rank * nk / s_cl, kb_hi = (rank + 1) * nk / s_cl;    // the host plan keeps s <= nk: no slice is empty

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, CS_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      // weight tiles before the programmatic-dependency wait, activations after it (as in gemm_f16_wgmma_kernel)
      const int pre = min(kb_hi - kb_lo, STAGES);
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(full0 + 8 * i, A_BYTES + B_BYTES);
        tma_load_2d(smem_u32(sB + i * B_BYTES), &tmB, (kb_lo + i) * BK, n_blk * BN, full0 + 8 * i);
      }
      pdl_wait();
      for (int i = 0; i < pre; ++i) tma_load_2d(smem_u32(sA + i * A_BYTES), &tmA, (kb_lo + i) * BK, 0, full0 + 8 * i);
      int s = pre == STAGES ? 0 : pre; uint32_t ph = pre == STAGES ? 1 : 0;
      for (int kb = kb_lo + pre; kb < kb_hi; ++kb) {
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        mbar_expect_tx(full0 + 8 * s, A_BYTES + B_BYTES);
        tma_load_2d(smem_u32(sA + s * A_BYTES), &tmA, kb * BK, 0, full0 + 8 * s);
        tma_load_2d(smem_u32(sB + s * B_BYTES), &tmB, kb * BK, n_blk * BN, full0 + 8 * s);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
    __syncwarp();
  } else {
    // wg broadcast from lane 0 so that ptxas treats it as warp-uniform (see gemm_f16_wgmma_kernel)
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0), wq = warp & 3;
    const int et = threadIdx.x - (CS_THREADS - CS_CONSUMERS);
    if (et < BN) { const int n = n_blk * BN + et; sbias[et] = (g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f; }
    asm volatile("bar.sync 1, 512;" ::: "memory");
    pdl_wait();
    // tail rows on CUDA cores: thread = (feature f, K half hk) over the first 2 BN consumer threads
    const int f = et >> 1, hk = et & 1;
    float tacc[GEMM_TAIL_MAX];
#pragma unroll
    for (int r = 0; r < GEMM_TAIL_MAX; ++r) tacc[r] = 0.f;
    const int kslice = (kb_hi - kb_lo) * BK, kbase = kb_lo * BK;
    for (int i = et; i < g.tail_rows * (kslice >> 3); i += CS_CONSUMERS) {
      const int r = i / (kslice >> 3), c8 = (i - r * (kslice >> 3)) << 3;
      uint4 xv = make_uint4(0u, 0u, 0u, 0u);
      if (kbase + c8 < g.K) xv = __ldg(reinterpret_cast<const uint4*>(g.a_tail + (size_t)r * g.lda + kbase + c8));
      *reinterpret_cast<uint4*>(sx + (size_t)r * kslice + c8) = xv;
    }
    asm volatile("bar.sync 1, 512;" ::: "memory");
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t a0 = smem_u32(sA + s * A_BYTES) + (uint32_t)wg * (64 * BK * 2), b0 = smem_u32(sB + s * B_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        Wgmma<BN>::mma(acc, wgmma_desc_k128(a0 + k * 32), wgmma_desc_k128(b0 + k * 32), (kb > kb_lo || k > 0) ? 1u : 0u);
      wg_commit();
      if (f < BN) {     // overlaps the MMAs just issued
        const uint8_t* wrow = sB + (size_t)s * B_BYTES + (size_t)f * 128;
        const int k0 = (kb - kb_lo) * BK + hk * 32;
        // one 16-byte W chunk at a time (registers: the 64 accumulators of BN 128 share 96 per thread); per row the FMA chain
        // runs over c, e in the same order as in gemm_f16_wgmma_kernel
        float a[GEMM_TAIL_MAX];
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r) a[r] = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint4 wv = *reinterpret_cast<const uint4*>(wrow + (((hk * 4 + c) ^ (f & 7)) << 4));
          const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
          for (int r = 0; r < GEMM_TAIL_MAX; ++r) {
            if (r < g.tail_rows) {
              const uint4 xv = *reinterpret_cast<const uint4*>(sx + (size_t)r * kslice + k0 + c * 8);
              const __half2* xh = reinterpret_cast<const __half2*>(&xv);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 xf = __half22float2(xh[e]), wf = __half22float2(wh[e]);
                a[r] = fmaf(xf.x, wf.x, a[r]); a[r] = fmaf(xf.y, wf.y, a[r]);
              }
            }
          }
        }
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r) tacc[r] += a[r];
      }
      wg_wait<1>();
      if (kb > kb_lo) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * (s == 0 ? STAGES - 1 : s - 1));
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
#pragma unroll
    for (int r = 0; r < GEMM_TAIL_MAX; ++r) tacc[r] += __shfl_xor_sync(0xffffffffu, tacc[r], 1);
    if (s_cl == 1) {
      // unsplit: the epilogue straight from the fragments
      if (hk == 0 && f < BN && n_blk * BN + f < g.N) {
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r)
          if (r < g.tail_rows) epilogue_store2(g, CS_BM + r, n_blk * BN + f, tacc[r] + sbias[f], 0.f, false, false);
      }
      epilogue_frag<BN>(acc, wg * 64 + wq * 16, n_blk, g, false, true, sbias);
    } else {
      asm volatile("bar.sync 1, 512;" ::: "memory");     // every warpgroup has finished reading the ring
      const int r_up = wg * 64 + wq * 16 + (lane >> 2), cq = (lane & 3) * 2;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(part + r_up * LDP + j * 8 + cq) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(part + (r_up + 8) * LDP + j * 8 + cq) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      if (hk == 0 && f < BN) {
#pragma unroll
        for (int r = 0; r < GEMM_TAIL_MAX; ++r)
          if (r < g.tail_rows) part[(CS_BM + r) * LDP + f] = tacc[r];
      }
    }
  }
  if (s_cl > 1) {
    cluster_sync_all();           // every CTA's partial tile is visible to the cluster
    if (warp >= 4) {
      const int et = threadIdx.x - (CS_THREADS - CS_CONSUMERS);
      const int rows = CS_BM + g.tail_rows, r0 = rank * rows / s_cl, r1 = (rank + 1) * rows / s_cl;
      const uint32_t base = smem_u32(part);
      for (int i = et; i < (r1 - r0) * (BN / 2); i += CS_CONSUMERS) {
        const int row = r0 + i / (BN / 2), c = (i % (BN / 2)) * 2, n = n_blk * BN + c;
        if (n >= g.N) continue;
        const uint32_t off = base + (uint32_t)(row * LDP + c) * 4;
        float2 sum = ld_peer_f2(off, 0);
        for (int p = 1; p < s_cl; ++p) { const float2 v = ld_peer_f2(off, p); sum.x += v.x; sum.y += v.y; }
        epilogue_store2(g, row, n, sum.x + sbias[c], sum.y + sbias[c + 1], n + 1 < g.N, false);
      }
    }
    cluster_sync_all();           // no CTA exits while a peer may still read its shared memory
  }
}

// ================================================================================================
// "x2" GEMM: fp32-grade product on the fp16 tensor path (the Q-Former, which the reference runs in float32).
//   A = A_hi + A_lo / 2048,  W = W_hi + W_lo / 2048   (fp16 pairs, see split_x2 in common.cuh)
//   out = A_hi.W_hi  +  (A_lo.W_hi + A_hi.W_lo) / 2048          (the lo.lo term is ~2^-22 relative: dropped)
// Same structure as gemm_f16_wgmma_kernel; a stage holds FOUR tiles, each consumer warpgroup issues three wgmma per K step into
// TWO register accumulators (main, correction) and merges them before the epilogue.  At 32 query rows the tensor pipe is idle
// anyway: the cost is the second weight tile per stage (fp32-sized weight traffic).
// ================================================================================================
template <int BN, int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16x2_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmAl,
                        const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmBl, GemmArgs g) {
  constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* sA = smem_align_1024(smem_raw);
  uint8_t* sAl = sA + STAGES * A_BYTES;
  uint8_t* sB = sAl + STAGES * A_BYTES;
  uint8_t* sBl = sB + STAGES * B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBl + STAGES * B_BYTES);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + STAGES);
  float* sbias = reinterpret_cast<float*>(bars + 2 * STAGES);   // [BN]

  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_blk = blockIdx.x, m_blk = blockIdx.y;
  const int kb_begin = blockIdx.z * g.kb_per_split;
  const int num_k = min((g.K + BK - 1) / BK - kb_begin, g.kb_per_split);
  const bool split = gridDim.z > 1;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmAl) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBl) : "memory");
    for (int i = 0; i < STAGES; ++i) { mbar_init(full0 + 8 * i, 1); mbar_init(empty0 + 8 * i, GEMM_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // weights first (independent of the predecessor kernel), activations after the dependency wait
      const int pre = num_k < STAGES ? num_k : STAGES;
      const uint32_t a_tx = (uint32_t)g.a_box_rows * BK * 2;
      for (int kb = 0; kb < pre; ++kb) {
        mbar_expect_tx(full0 + 8 * kb, 2 * (a_tx + B_BYTES));
        tma_load_2d(smem_u32(sB + kb * B_BYTES), &tmB, (kb_begin + kb) * BK, n_blk * BN, full0 + 8 * kb);
        tma_load_2d(smem_u32(sBl + kb * B_BYTES), &tmBl, (kb_begin + kb) * BK, n_blk * BN, full0 + 8 * kb);
      }
      pdl_wait();
      for (int kb = 0; kb < pre; ++kb) {
        tma_load_2d(smem_u32(sA + kb * A_BYTES), &tmA, (kb_begin + kb) * BK, m_blk * BM, full0 + 8 * kb);
        tma_load_2d(smem_u32(sAl + kb * A_BYTES), &tmAl, (kb_begin + kb) * BK, m_blk * BM, full0 + 8 * kb);
      }
      int s = pre == STAGES ? 0 : pre; uint32_t ph = pre == STAGES ? 1 : 0;
      for (int kb = pre; kb < num_k; ++kb) {
        mbar_wait(empty0 + 8 * s, ph ^ 1);
        mbar_expect_tx(full0 + 8 * s, 2 * (a_tx + B_BYTES));
        tma_load_2d(smem_u32(sA + s * A_BYTES), &tmA, (kb_begin + kb) * BK, m_blk * BM, full0 + 8 * s);
        tma_load_2d(smem_u32(sAl + s * A_BYTES), &tmAl, (kb_begin + kb) * BK, m_blk * BM, full0 + 8 * s);
        tma_load_2d(smem_u32(sB + s * B_BYTES), &tmB, (kb_begin + kb) * BK, n_blk * BN, full0 + 8 * s);
        tma_load_2d(smem_u32(sBl + s * B_BYTES), &tmBl, (kb_begin + kb) * BK, n_blk * BN, full0 + 8 * s);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp >> 2) - 1, wq = warp & 3;
    const int et = threadIdx.x - (GEMM_THREADS - GEMM_CONSUMERS);
    const int wg_row0 = m_blk * BM + wg * 64;
    const bool active = wg_row0 < g.M;
    if (et < BN) { const int n = n_blk * BN + et; sbias[et] = (g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f; }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    pdl_wait();
    if (!active) {     // keep the ring turning for the other warpgroup: take every stage and hand it straight back
      int s = 0; uint32_t ph = 0;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(full0 + 8 * s, ph);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * s);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      return;
    }
    float acc[BN / 2], corr[BN / 2];   // main (hi.hi) and correction (lo.hi + hi.lo, scaled by 2048) accumulators
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[i] = 0.f; corr[i] = 0.f; }
    int s = 0; uint32_t ph = 0;
    for (int kb = 0; kb < num_k; ++kb) {
      mbar_wait(full0 + 8 * s, ph);
      const uint32_t wg_off = (uint32_t)wg * (64 * BK * 2);
      const uint32_t a0 = smem_u32(sA + s * A_BYTES) + wg_off, al0 = smem_u32(sAl + s * A_BYTES) + wg_off;
      const uint32_t b0 = smem_u32(sB + s * B_BYTES), bl0 = smem_u32(sBl + s * B_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t da = wgmma_desc_k128(a0 + k * 32), dal = wgmma_desc_k128(al0 + k * 32);
        const uint64_t db = wgmma_desc_k128(b0 + k * 32), dbl = wgmma_desc_k128(bl0 + k * 32);
        const uint32_t first = (kb > 0 || k > 0) ? 1u : 0u;
        Wgmma<BN>::mma(acc, da, db, first);
        Wgmma<BN>::mma(corr, dal, db, first);
        Wgmma<BN>::mma(corr, da, dbl, 1u);
      }
      wg_commit();
      wg_wait<1>();
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * (s == 0 ? STAGES - 1 : s - 1));
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wg_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = fmaf(corr[i], 1.f / X2_SCALE, acc[i]);
    epilogue_frag<BN>(acc, wg_row0 + wq * 16, n_blk, g, split, blockIdx.z == 0, sbias);
  }
}

// ---------------------------------------------------------------- host side ------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2D fp16 row-major [rows, cols] (cols contiguous, leading dimension ld elements), box {64, boxRows}
static int make_map(CUtensorMap* m, const void* base, int rows, int cols, int ld, int boxRows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return VLFM_E_DRIVER; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)boxRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d", (int)r, rows, cols, ld); return VLFM_E_DRIVER; }
  return VLFM_OK;
}

template <int BN, int STAGES, bool SILU = false>
static int launch_gemm(const CUtensorMap& ta, const void* W, int ldw, const GemmArgs& g, cudaStream_t st) {
  if constexpr (!SILU) {
    if (g.epi == VLFM_EPI_BIAS_SILU_F16) return launch_gemm<BN, STAGES, true>(ta, W, ldw, g, st);
  }
  CUtensorMap tb;
  int rc = make_map(&tb, W, g.N, g.K, ldw, BN);
  if (rc) return rc;
  constexpr size_t smem = (size_t)STAGES * (BM * BK * 2 + BN * BK * 2) + 2 * STAGES * 8 + 1024 + BN * 4 +
                          (size_t)GEMM_TAIL_MAX * GEMM_TAIL_KMAX * 2;
  static_assert(smem <= 227 * 1024, "GEMM stage ring exceeds the 227 KB a block may use");
  static bool configured = false;
  if (!configured) {
    rc = check_cuda(cudaFuncSetAttribute(gemm_f16_wgmma_kernel<BN, STAGES, SILU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(gemm)");
    if (rc) return rc;
    configured = true;
  }
  const int num_k = (g.K + BK - 1) / BK;
  dim3 grid((g.N + BN - 1) / BN, g.tail_rows > 0 ? g.M / BM : (g.M + BM - 1) / BM, (num_k + g.kb_per_split - 1) / g.kb_per_split);
  if (g.sk.ctas > 0) grid = dim3(g.sk.ctas);
  rc = check_cuda(launch_pdl(gemm_f16_wgmma_kernel<BN, STAGES, SILU>, grid, dim3(GEMM_THREADS), smem, st, ta, tb, g), "gemm_f16_wgmma_kernel");
  if (rc) return rc;
  count_launch();
  return VLFM_OK;
}


template <int BN, int STAGES>
static int launch_gemm_x2(const CUtensorMap& ta, const CUtensorMap& tal, const void* W, const void* Wl, int ldw, const GemmArgs& g, cudaStream_t st) {
  CUtensorMap tb, tbl;
  int rc = make_map(&tb, W, g.N, g.K, ldw, BN);
  if (!rc) rc = make_map(&tbl, Wl, g.N, g.K, ldw, BN);
  if (rc) return rc;
  constexpr size_t smem = (size_t)STAGES * 2 * (BM * BK * 2 + BN * BK * 2) + 2 * STAGES * 8 + 1024 + BN * 4;
  static_assert(smem <= 227 * 1024, "x2 GEMM stage ring exceeds the 227 KB a block may use");
  static bool configured = false;
  if (!configured) {
    rc = check_cuda(cudaFuncSetAttribute(gemm_f16x2_wgmma_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute(gemm x2)");
    if (rc) return rc;
    configured = true;
  }
  const int num_k = (g.K + BK - 1) / BK;
  dim3 grid((g.N + BN - 1) / BN, (g.M + BM - 1) / BM, (num_k + g.kb_per_split - 1) / g.kb_per_split);
  rc = check_cuda(launch_pdl(gemm_f16x2_wgmma_kernel<BN, STAGES>, grid, dim3(GEMM_THREADS), smem, st, ta, tal, tb, tbl, g), "gemm_f16x2_wgmma_kernel");
  if (rc) return rc;
  count_launch();
  return VLFM_OK;
}

// gemm_f16_csplit_wgmma_kernel<BN, STAGES>: its shared memory, how many s-CTA clusters of it the device runs at once, and the
// launch (grid of column tiles x s, cluster (s, 1, 1), programmatic dependent launch as for the other kernels)
template <int BN, int STAGES>
struct Csplit {
  static constexpr size_t smem = (size_t)STAGES * (CS_BM * BK * 2 + BN * BK * 2) + 2 * STAGES * 8 + 1024 + BN * 4 +
                                 (size_t)GEMM_TAIL_MAX * GEMM_TAIL_KMAX * 2;
  static_assert(smem <= 227 * 1024, "cluster-split GEMM stage ring exceeds the 227 KB a block may use");
  static int configure() {
    static int rc = -1;
    if (rc < 0) rc = check_cuda(cudaFuncSetAttribute(gemm_f16_csplit_wgmma_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                                "cudaFuncSetAttribute(gemm csplit)");
    return rc;
  }
  static int max_clusters(int s) {
    static int fit[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};
    if (fit[s] < 0) {
      fit[s] = 0;
      if (configure()) return 0;
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3(s); cfg.blockDim = dim3(CS_THREADS); cfg.dynamicSmemBytes = smem;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = s; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.attrs = attr; cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, gemm_f16_csplit_wgmma_kernel<BN, STAGES>, &cfg) == cudaSuccess) fit[s] = n;
      else cudaGetLastError();
    }
    return fit[s];
  }
  static int launch(const CUtensorMap& ta, const void* W, int ldw, const GemmArgs& g, int s, cudaStream_t st) {
    CUtensorMap tb;
    int rc = make_map(&tb, W, g.N, g.K, ldw, BN);
    if (!rc) rc = configure();
    if (rc) return rc;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(((g.N + BN - 1) / BN) * s); cfg.blockDim = dim3(CS_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = s; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 2 : 1;
    rc = check_cuda(cudaLaunchKernelEx(&cfg, gemm_f16_csplit_wgmma_kernel<BN, STAGES>, ta, tb, g), "gemm_f16_csplit_wgmma_kernel");
    if (rc) return rc;
    count_launch();
    return VLFM_OK;
  }
};

}  // namespace vlfm

using namespace vlfm;

static int gemm_dispatch(const void* d_A, const void* d_W, int M, int N, int K, int lda, int ldw, GemmArgs g, void* stream, float* d_partials,
                         size_t partial_bytes, SplitK* layout, bool csplit);

// SMs of the current device (one GEMM CTA per SM): the launch plans size a wave by it.  132 on an H100 SXM.
static int sm_count() {
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) sms = 132; }
  return sms;
}

extern "C" int vlfm_gemm_f16(const void* d_A, const void* d_W, const float* d_bias, void* d_out, int M, int N,
                             int K, int lda, int ldw, int ldo, int epilogue, void* stream) {
  if (!d_A || !d_W || !d_out || M < 1 || N < 1 || K < 1) { set_error("vlfm_gemm_f16: bad argument"); return VLFM_E_INVALID; }
  if ((K & 7) || (lda & 7) || (ldw & 7) || (ldo & 7) || ((uintptr_t)d_A & 15) || ((uintptr_t)d_W & 15) || ((uintptr_t)d_out & 15)) {
    set_error("vlfm_gemm_f16: K, lda, ldw, ldo must be multiples of 8 and pointers 16-byte aligned"); return VLFM_E_INVALID; }
  // the cluster-split kernel has no SiLU instantiation: that epilogue ignores the flag
  const bool csplit = (epilogue & VLFM_EPI_CLUSTER_SPLIT) != 0 && (epilogue & ~VLFM_EPI_CLUSTER_SPLIT) != VLFM_EPI_BIAS_SILU_F16;
  epilogue &= ~VLFM_EPI_CLUSTER_SPLIT;
  if (epilogue < 0 || (epilogue > 4 && epilogue != VLFM_EPI_BIAS_SILU_F16)) { set_error("vlfm_gemm_f16: unknown epilogue %d", epilogue); return VLFM_E_INVALID; }
  GemmArgs g{d_bias, d_out, M, N, K, ldo, epilogue, (K + BK - 1) / BK, 0, nullptr, 0, 0, 0, nullptr, BM};
  return gemm_dispatch(d_A, d_W, M, N, K, lda, ldw, g, stream, nullptr, 0, nullptr, csplit);
}

// Cluster-split plan (gemm_f16_csplit_wgmma_kernel) for 256 < M <= 256 + GEMM_TAIL_MAX.  Over the tile widths BN and cluster
// sizes s whose clusters all run at once (cudaOccupancyMaxActiveClusters: the GPCs do not split evenly into clusters), the one
// that minimises what the busiest CTA takes in: its K-blocks x (256 + BN) x 64 fp16, plus, when split, the peers' fp32 partials
// its reduction reads ((s - 1) / s of an M x BN tile) and a fixed cost per cluster reduction.  A byte model, not a fitted one.
constexpr double CS_RED_FIXED_BYTES = 16384;   // the two cluster barriers and the reduction's latency, counted as K-loop bytes
// Which shapes take it.  On an H100 (DESIGN §3.3) the plan below is faster than the 128-row plan for the ViT's fc1 and fc2
// (8.7 M weights each) and slower for qkv (5.9 M) and proj (2.0 M), whose shorter K loops do not pay back the cluster launch
// and the reduction.  So by default it runs for weights of at least CS_MIN_WEIGHTS elements.  VLFM_GEMM_CSPLIT=0 turns it off,
// =2 runs it for every shape it can take (tests, sweeps).
constexpr long long CS_MIN_WEIGHTS = 8ll << 20;
static bool csplit_eligible(int M, int N, int K) {
  const char* e = getenv("VLFM_GEMM_CSPLIT");
  const int mode = (e && e[0]) ? atoi(e) : 1;
  return mode > 0 && M > CS_BM && M - CS_BM <= GEMM_TAIL_MAX && K <= GEMM_TAIL_KMAX && (mode >= 2 || (long long)N * K >= CS_MIN_WEIGHTS);
}
struct CsplitPlan { int bn, s; double cta_bytes; };
static int csplit_fit(int bn, int s) {
  if (bn == 128) return Csplit<128, 4>::max_clusters(s);
  if (bn == 96) return Csplit<96, 4>::max_clusters(s);
  return Csplit<64, 5>::max_clusters(s);
}
static CsplitPlan csplit_plan(int M, int N, int K) {
  const int nk = (K + BK - 1) / BK;
  CsplitPlan best{0, 0, 0.0};
  const int bns[3] = {128, 96, 64};
  for (int bn : bns) {
    const int nt = (N + bn - 1) / bn;
    for (int s = 1; s <= 8 && s <= nk; ++s) {
      if (nt > csplit_fit(bn, s)) continue;
      double bytes = (double)((nk + s - 1) / s) * (CS_BM + bn) * BK * 2;
      if (s > 1) bytes += (double)(s - 1) / s * M * bn * 4 + CS_RED_FIXED_BYTES;
      if (!best.bn || bytes < best.cta_bytes) best = CsplitPlan{bn, s, bytes};
    }
  }
  return best;
}

// The plan vlfm_gemm_f16 / vlfm_gemm_f16_resid_ln would run for an allowed cluster split of this shape: {BN, s, bytes the busiest
// CTA loads}, or {0, 0, 0} when the shape does not take that path.  For scripts/gemm_graph_bench.py.
extern "C" int vlfm_gemm_csplit_plan(int M, int N, int K, int* bn, int* splits, double* cta_bytes) {
  CsplitPlan p{0, 0, 0.0};
  if (csplit_eligible(M, N, K)) p = csplit_plan(M, N, K);
  if (bn) *bn = p.bn;
  if (splits) *splits = p.s;
  if (cta_bytes) *cta_bytes = p.cta_bytes;
  return VLFM_OK;
}

// Stream-K: the least number of K-blocks a CTA works through.  Below it the fixed cost of a CTA (barrier set-up, the first
// loads, one or two segment stores of 66 KB) outweighs the K-blocks it takes off the other CTAs.
constexpr int SK_MIN_ITERS = 3;

static int gemm_dispatch(const void* d_A, const void* d_W, int M, int N, int K, int lda, int ldw, GemmArgs g, void* stream, float* d_partials,
                         size_t partial_bytes, SplitK* layout, bool csplit) {
  if (layout) *layout = SplitK{1, 0};
  const int epilogue = g.epi;
  CUtensorMap ta;
  // Batch-1 ViT rows (256 < M <= 256 + GEMM_TAIL_MAX) when the caller allows a split whose bits depend on the plan: one 256-row
  // tile per column block, K split over a thread-block cluster and reduced in shared memory (csplit_eligible: which shapes).
  if (csplit && !getenv("VLFM_GEMM_FORCE") && csplit_eligible(M, N, K)) {
    const CsplitPlan p = csplit_plan(M, N, K);
    if (p.bn) {
      int rc = make_map(&ta, d_A, M, K, lda, CS_BM);
      if (rc) return rc;
      g.a_tail = (const __half*)d_A + (size_t)CS_BM * lda; g.lda = lda; g.tail_rows = M - CS_BM; g.tail_row0 = CS_BM;
      cudaStream_t cst = (cudaStream_t)stream;
      if (p.bn == 128) return Csplit<128, 4>::launch(ta, d_W, ldw, g, p.s, cst);
      if (p.bn == 96) return Csplit<96, 4>::launch(ta, d_W, ldw, g, p.s, cst);
      return Csplit<64, 5>::launch(ta, d_W, ldw, g, p.s, cst);
    }
  }
  g.a_box_rows = M <= 32 ? 32 : (M <= 64 ? 64 : BM);
  int rc = make_map(&ta, d_A, M, K, lda, g.a_box_rows);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int mt = (M + BM - 1) / BM, num_k = (K + BK - 1) / BK;
  const int sms = sm_count();
  // M = 128*q + r with a tiny remainder (ViT: 257 tokens = 2*128 + 1): launch q row tiles only; the last tile's CTAs compute
  // the r tail rows on CUDA cores from the W tiles they stage anyway.  A third of the CTAs (and of the W traffic) disappears,
  // which buys narrower tiles / deeper split-K inside one wave.
  static int tail_on = -1;
  if (tail_on < 0) { const char* e = getenv("VLFM_GEMM_TAIL"); tail_on = (e && e[0] == '0') ? 0 : 1; }
  const int rem = M % BM;
  const bool tail = tail_on && M > BM && rem >= 1 && rem <= GEMM_TAIL_MAX && num_k * BK <= GEMM_TAIL_KMAX;
  const int rt = tail ? M / BM : mt;     // row tiles launched
  const char* force = getenv("VLFM_GEMM_FORCE");   // development sweep: "bn:splits" (grid launches only)
  const bool resid = epilogue == VLFM_EPI_BIAS_RESID_F32;
  const int tiles128 = rt * ((N + BM - 1) / BM);
  // A resid-LN call (layout != null) never reduces with red.global.add: its splits must fit the workspace as partial sums, so a
  // split that does not fit runs unsplit.  Only vlfm_gemm_f16 with the residual epilogue (no workspace) splits into x atomically.
  long long split_cap = num_k;
  if (layout) {
    split_cap = (long long)(partial_bytes / ((size_t)M * (size_t)N * 4));
    if (split_cap < 1) split_cap = 1;
  }
  int best_bn = 128, best_s = 1;
  bool best_tail = tail;
  if (tiles128 < sms && resid && d_partials && !force) {
    // Less than one wave of 128 x 128 tiles, and a workspace: stream-K.  Every SM gets the same number of K-blocks (+-1) of the
    // tiles' K-block sequence (SplitK in common.cuh); the LayerNorm launch adds the segments of each tile in K order.
    const long long iters = (long long)tiles128 * num_k;
    long long P = iters / SK_MIN_ITERS;
    if (P > sms) P = sms;
    const long long fit = (long long)(partial_bytes / (SK_SLAB * 4)) - (tiles128 - 1);
    if (P > fit) P = fit;
    if (P > tiles128) {
      g.sk = SplitK{0, 0, (int)P, rt, tiles128, num_k};
      g.out = d_partials;
      if (tail) { g.a_tail = (const __half*)d_A + (size_t)rt * BM * lda; g.lda = lda; g.tail_rows = rem; g.tail_row0 = rt * BM; }
      if (layout) *layout = g.sk;
      return launch_gemm<128, 6>(ta, d_W, ldw, g, st);
    }
  }
  if (tiles128 <= sms && !resid) {
    // Less than one wave, no split: the tile width that leaves the busiest SM the fewest columns, ceil(tiles / SMs) * BN
    // (the wider tile on a tie: fewer A re-reads).  ViT-g at batch 1: qkv BN 64 (132 CTAs), fc1 BN 96 (128 CTAs).
    const int bns[4] = {128, 96, 64, 32};
    long long best = -1;
    for (int bn : bns) {
      const long long tl = (long long)rt * ((N + bn - 1) / bn), cols = (tl + sms - 1) / sms * bn;
      if (best < 0 || cols < best) { best = cols; best_bn = bn; }
    }
  } else {
    // Tile / split-K plan from a small cost model (us): waves x (fixed + bytes a CTA must pull / its share of the L2->SM
    // bandwidth).  Never spill into a second wave for a handful of CTAs; split K only for the fp32 residual epilogue (partial
    // sums the LayerNorm launch reduces, at most split_cap of them; red.add only for vlfm_gemm_f16 without a workspace), and not
    // at all for residual calls with a workspace below a wave (those are stream-K, or unsplit when the workspace is too small).
    double best_t = 1e30;
    // Cost model:  t = waves * (c0 + K-blocks per CTA * per_kb),  per_kb = max(pipeline floor, CTAs * KB per K-block / chip L2->SM rate),
    //   c0 = prologue + epilogue per tile width, + split-K stores, + the tail-row work.  One CTA per SM (H100: 132).  The rate
    //   (5.5 TB/s) and the floor / c0 terms are estimates for H100, not fitted to measurements on it.
    const int bns[3] = {128, 64, 32};
    for (int tm = 0; tm < (tail ? 2 : 1); ++tm) {
      const bool use_tail = tail && tm == 0;
      const int mte = use_tail ? M / BM : mt;
      for (int bi = 0; bi < 3; ++bi) {
        const int bn = bns[bi], nt = (N + bn - 1) / bn;
        int smax = resid && !(d_partials && tiles128 < sms) ? num_k / 4 : 1;
        if (smax < 1) smax = 1;
        if (smax > 8) smax = 8;
        if (smax > split_cap) smax = (int)split_cap;
        for (int sp = 1; sp <= smax; ++sp) {
          const double ctas = (double)mte * nt * sp;
          const int kb = (num_k + sp - 1) / sp;
          const double waves = (double)(long)((ctas + sms - 1) / sms);
          const double active = ctas < sms ? ctas : sms;
          const double kb_kbytes = (double)(128 + bn) * 128 / 1024.0;
          double per_kb = active * kb_kbytes / 5500.0;
          if (per_kb < 0.33) per_kb = 0.33;
          double c0 = bn == 128 ? 3.8 + 0.22 * sp : (bn == 64 ? 3.0 : 2.6) + (sp > 1 ? 0.1 * sp : 0.0);
          if (use_tail) c0 += bn == 128 ? 0.9 : 0.3;
          const double t = waves * (c0 + kb * per_kb);
          if (t < best_t) { best_t = t; best_bn = bn; best_s = sp; best_tail = use_tail; }
        }
      }
    }
  }
  if (force) {
    int fb = 0, fs = 0;
    if (sscanf(force, "%d:%d", &fb, &fs) == 2 && (fb == 128 || fb == 96 || fb == 64 || fb == 32) && fs >= 1) {
      best_bn = fb;
      best_s = resid ? (fs > num_k ? num_k : fs) : 1;
      if (best_s > split_cap) best_s = (int)split_cap;
    }
  }
  g.kb_per_split = (num_k + best_s - 1) / best_s;
  if (best_tail) { g.a_tail = (const __half*)d_A + (size_t)(M / BM) * BM * lda; g.lda = lda; g.tail_rows = rem; g.tail_row0 = (M / BM) * BM; }
  // deterministic split-K: the splits store their partial sums side by side and the caller reduces them in a fixed order
  const int launched_splits = (num_k + g.kb_per_split - 1) / g.kb_per_split;      // grid.z (can be below best_s when num_k is small)
  if (d_partials && launched_splits > 1 && resid && (size_t)launched_splits * (size_t)M * (size_t)N * 4 <= partial_bytes) {
    g.epi = VLFM_EPI_PARTIAL_F32; g.out = d_partials; g.ldo = N; g.split_stride = (long long)M * N;
    if (layout) *layout = SplitK{launched_splits, (long long)M * N};
  }
  if (best_bn == 128) return launch_gemm<128, 6>(ta, d_W, ldw, g, st);
  if (best_bn == 96) return launch_gemm<96, 7>(ta, d_W, ldw, g, st);
  if (best_bn == 64) return launch_gemm<64, 8>(ta, d_W, ldw, g, st);
  return launch_gemm<32, 8>(ta, d_W, ldw, g, st);
}

extern "C" int vlfm_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out16, float* d_out32,
                   int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream);
namespace vlfm {
int layernorm_reduce_impl(float* d_x, const float* d_partials, const SplitK& sk, const float* d_gamma, const float* d_beta, void* d_out16,
                          void* d_out16_lo, float* d_out32, int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream);
}

// x += A @ W^T + bias ; out = LayerNorm(x) -- bitwise reproducible: when the plan splits K (stream-K below a wave of tiles, uniform
// splits above), the splits store their partial sums in d_partials (no atomics) and the LayerNorm kernel adds them to x in K order
// before normalising; an unsplit GEMM adds
// into x directly (one writer per element).  (Round 1 reduced the splits with red.global.add: the order of arrival varied from run
// to run and the 39-layer residual stream amplified the last-bit differences to ~6e-5 on the cosine.)
extern "C" int vlfm_gemm_f16_resid_ln(const void* d_A, const void* d_W, const float* d_bias, float* d_x, int M, int N, int K,
                                      int lda, int ldw, int ldx, const float* d_gamma, const float* d_beta, void* d_out16,
                                      int ld16, float* d_out32, int ld32, float eps, float* d_partials, size_t partial_bytes, void* stream) {
  if (!d_A || !d_W || !d_x || !d_gamma || !d_beta || (!d_out16 && !d_out32) || M < 1 || N < 1 || K < 1) {
    set_error("vlfm_gemm_f16_resid_ln: bad argument"); return VLFM_E_INVALID; }
  if ((K & 7) || (lda & 7) || (ldw & 7) || (ldx & 7) || (N & 3) || (ld16 & 3) || (ld32 & 3) || ((uintptr_t)d_A & 15) || ((uintptr_t)d_W & 15) ||
      ((uintptr_t)d_x & 15) || ((uintptr_t)d_partials & 15)) { set_error("vlfm_gemm_f16_resid_ln: alignment (K, strides %% 8; N %% 4; 16-byte pointers)"); return VLFM_E_INVALID; }
  // the LayerNorm's own limits, before the GEMM changes x or the workspace
  int rc = layernorm_check("vlfm_gemm_f16_resid_ln", d_x, d_gamma, d_beta, d_out16, nullptr, d_out32, N, ldx, ld16, ld32);
  if (rc) return rc;
  GemmArgs g{d_bias, d_x, M, N, K, ldx, VLFM_EPI_BIAS_RESID_F32, (K + BK - 1) / BK, 0, nullptr, 0, 0, 0, nullptr, BM};
  SplitK layout;
  // a workspace means the caller allows a split K, which includes the cluster split (MobileSAM passes none: its rows' bits must
  // not depend on M)
  rc = gemm_dispatch(d_A, d_W, M, N, K, lda, ldw, g, stream, d_partials, partial_bytes, &layout, d_partials != nullptr);
  if (rc) return rc;
  if (layout.splits != 1) return layernorm_reduce_impl(d_x, d_partials, layout, d_gamma, d_beta, d_out16, nullptr, d_out32, M, N, ldx, ld16, ld32, eps, stream);
  return vlfm_layernorm(d_x, d_gamma, d_beta, d_out16, d_out32, M, N, ldx, ld16, ld32, eps, stream);
}

// ---- x2 GEMMs (fp32-grade, see gemm_f16x2_wgmma_kernel) ----
static int gemm_x2_dispatch(const void* d_A_hi, const void* d_A_lo, const void* d_W_hi, const void* d_W_lo, int M, int N, int K, int lda, int ldw,
                            GemmArgs g, void* stream, float* d_partials, size_t partial_bytes, int* splits_out) {
  if (splits_out) *splits_out = 1;
  // M = 128 q + r with a small remainder (257 image tokens): the r rows would cost a whole extra row of tiles -- run them as their
  // own skinny launch (32-row A box) after the q full row tiles
  const int rem = M % BM;
  if (M > BM && rem >= 1 && rem <= 32 && (g.epi == VLFM_EPI_BIAS_F32 || g.epi == VLFM_EPI_BIAS_GELU_F16X2)) {
    const int m0 = M - rem;
    GemmArgs g0 = g; g0.M = m0;
    int rc0 = gemm_x2_dispatch(d_A_hi, d_A_lo, d_W_hi, d_W_lo, m0, N, K, lda, ldw, g0, stream, nullptr, 0, nullptr);
    if (rc0) return rc0;
    GemmArgs g1 = g; g1.M = rem;
    const size_t esz = g.epi == VLFM_EPI_BIAS_F32 ? 4 : 2;
    g1.out = (uint8_t*)g.out + (size_t)m0 * g.ldo * esz;
    if (g.out_lo) g1.out_lo = (uint8_t*)g.out_lo + (size_t)m0 * g.ldo * 2;
    return gemm_x2_dispatch((const __half*)d_A_hi + (size_t)m0 * lda, (const __half*)d_A_lo + (size_t)m0 * lda, d_W_hi, d_W_lo, rem, N, K, lda, ldw, g1,
                            stream, nullptr, 0, nullptr);
  }
  CUtensorMap ta, tal;
  g.a_box_rows = M <= 32 ? 32 : (M <= 64 ? 64 : BM);
  int rc = make_map(&ta, d_A_hi, M, K, lda, g.a_box_rows);
  if (!rc) rc = make_map(&tal, d_A_lo, M, K, lda, g.a_box_rows);
  if (rc) return rc;
  const int mt = (M + BM - 1) / BM, num_k = (K + BK - 1) / BK;
  // tile width: wide tiles for the one big problem (cross-attention K/V of all layers: 257 x 9216 x 1408), else enough CTAs to
  // cover the machine; split K (deterministic partial sums) only for the residual epilogue -- at 32 rows a partial slab is 100 KB
  int bn = 32;
  if (mt >= 2 && N >= 4096) bn = 128;
  else if ((long)mt * ((N + 63) / 64) >= 96) bn = 64;
  const int tiles = mt * ((N + bn - 1) / bn);
  int sp = 1;
  if (g.epi == VLFM_EPI_BIAS_RESID_F32 && d_partials) {
    sp = sm_count() / tiles; if (sp > num_k / 3) sp = num_k / 3; if (sp > 8) sp = 8; if (sp < 1) sp = 1;
  }
  g.kb_per_split = (num_k + sp - 1) / sp;
  const int launched = (num_k + g.kb_per_split - 1) / g.kb_per_split;
  if (launched > 1) {
    if ((size_t)launched * (size_t)M * (size_t)N * 4 > partial_bytes) { g.kb_per_split = num_k; }
    else { g.epi = VLFM_EPI_PARTIAL_F32; g.out = d_partials; g.ldo = N; g.split_stride = (long long)M * N; if (splits_out) *splits_out = launched; }
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (bn == 128) return launch_gemm_x2<128, 3>(ta, tal, d_W_hi, d_W_lo, ldw, g, st);
  if (bn == 64) return launch_gemm_x2<64, 4>(ta, tal, d_W_hi, d_W_lo, ldw, g, st);
  return launch_gemm_x2<32, 5>(ta, tal, d_W_hi, d_W_lo, ldw, g, st);
}

static int x2_args_ok(const char* who, const void* a, const void* al, const void* w, const void* wl, const void* out, int M, int N, int K, int lda, int ldw, int ldo) {
  if (!a || !al || !w || !wl || !out || M < 1 || N < 1 || K < 1) { set_error("%s: bad argument", who); return VLFM_E_INVALID; }
  if ((K & 7) || (lda & 7) || (ldw & 7) || (ldo & 7) || ((uintptr_t)a & 15) || ((uintptr_t)al & 15) || ((uintptr_t)w & 15) || ((uintptr_t)wl & 15) || ((uintptr_t)out & 15)) {
    set_error("%s: K, lda, ldw, ldo must be multiples of 8 and pointers 16-byte aligned", who); return VLFM_E_INVALID; }
  return VLFM_OK;
}

// out = epilogue((A_hi + A_lo/2048) @ (W_hi + W_lo/2048)^T + bias).  epilogue: VLFM_EPI_BIAS_F32 (fp32 out), VLFM_EPI_BIAS_RESID_F32
// (fp32 out += ...), VLFM_EPI_BIAS_GELU_F16X2 (GELU, then fp16 x2 operands into d_out / d_out_lo).
extern "C" int vlfm_gemm_f16x2(const void* d_A_hi, const void* d_A_lo, const void* d_W_hi, const void* d_W_lo, const float* d_bias, void* d_out,
                               void* d_out_lo, int M, int N, int K, int lda, int ldw, int ldo, int epilogue, void* stream) {
  int rc = x2_args_ok("vlfm_gemm_f16x2", d_A_hi, d_A_lo, d_W_hi, d_W_lo, d_out, M, N, K, lda, ldw, ldo);
  if (rc) return rc;
  if (epilogue != VLFM_EPI_BIAS_F32 && epilogue != VLFM_EPI_BIAS_RESID_F32 && epilogue != VLFM_EPI_BIAS_GELU_F16X2) {
    set_error("vlfm_gemm_f16x2: epilogue %d unsupported (fp32, fp32 residual, GELU x2)", epilogue); return VLFM_E_INVALID; }
  if (epilogue == VLFM_EPI_BIAS_GELU_F16X2 && (!d_out_lo || ((uintptr_t)d_out_lo & 15))) { set_error("vlfm_gemm_f16x2: d_out_lo missing / unaligned"); return VLFM_E_INVALID; }
  GemmArgs g{d_bias, d_out, M, N, K, ldo, epilogue, (K + BK - 1) / BK, 0, nullptr, 0, 0, 0, d_out_lo, BM};
  return gemm_x2_dispatch(d_A_hi, d_A_lo, d_W_hi, d_W_lo, M, N, K, lda, ldw, g, stream, nullptr, 0, nullptr);
}

extern "C" int vlfm_layernorm_x2(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32,
                                 int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream);
extern "C" int vlfm_layernorm_reduce_x2(float* d_x, const float* d_partials, int splits, long long split_stride, const float* d_gamma,
                                        const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32, int rows, int D, int ldx, int ldo16,
                                        int ldo32, float eps, void* stream);

// x += (x2 product) + bias ; LayerNorm(x) -> x2 operands (hi, lo) and/or fp32.  Bitwise reproducible like vlfm_gemm_f16_resid_ln.
extern "C" int vlfm_gemm_f16x2_resid_ln(const void* d_A_hi, const void* d_A_lo, const void* d_W_hi, const void* d_W_lo, const float* d_bias,
                                        float* d_x, int M, int N, int K, int lda, int ldw, int ldx, const float* d_gamma, const float* d_beta,
                                        void* d_out_hi, void* d_out_lo, int ld16, float* d_out32, int ld32, float eps, float* d_partials,
                                        size_t partial_bytes, void* stream) {
  int rc = x2_args_ok("vlfm_gemm_f16x2_resid_ln", d_A_hi, d_A_lo, d_W_hi, d_W_lo, d_x, M, N, K, lda, ldw, ldx);
  if (rc) return rc;
  if (!d_gamma || !d_beta || !d_out_hi || !d_out_lo || (N & 3) || (ld16 & 3) || (ld32 & 3) || ((uintptr_t)d_partials & 15)) {
    set_error("vlfm_gemm_f16x2_resid_ln: bad argument / alignment"); return VLFM_E_INVALID; }
  rc = layernorm_check("vlfm_gemm_f16x2_resid_ln", d_x, d_gamma, d_beta, d_out_hi, d_out_lo, d_out32, N, ldx, ld16, ld32);
  if (rc) return rc;
  GemmArgs g{d_bias, d_x, M, N, K, ldx, VLFM_EPI_BIAS_RESID_F32, (K + BK - 1) / BK, 0, nullptr, 0, 0, 0, nullptr, BM};
  int splits = 1;
  rc = gemm_x2_dispatch(d_A_hi, d_A_lo, d_W_hi, d_W_lo, M, N, K, lda, ldw, g, stream, d_partials, partial_bytes, &splits);
  if (rc) return rc;
  if (splits > 1) return vlfm_layernorm_reduce_x2(d_x, d_partials, splits, (long long)M * N, d_gamma, d_beta, d_out_hi, d_out_lo, d_out32, M, N, ldx, ld16, ld32, eps, stream);
  return vlfm_layernorm_x2(d_x, d_gamma, d_beta, d_out_hi, d_out_lo, d_out32, M, N, ldx, ld16, ld32, eps, stream);
}
