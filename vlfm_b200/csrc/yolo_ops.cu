// YOLOv7-E6E kernels (vlfm/vlm/yolov7.py YOLOv7.predict); the engine is vlfm_b200/vlm/yolov7_engine.py.  Activations are fp16
// NHWC rows with a row stride (`ld*`, in elements), so a layer can read or write one channel slice of a concat buffer.  Every
// conv is vlfm_im2col_f16 (3x3) or nothing (1x1) plus vlfm_gemm_f16 with VLFM_EPI_BIAS_SILU_F16; these kernels are the rest:
//   - yolo_preprocess: cv2 INTER_AREA resize of uint8 frames, /255 to fp16 and ReOrg (space-to-depth), one launch;
//   - yolo_maxpool2, yolo_spp_pools, yolo_upsample2, yolo_add: strided layer primitives;
//   - yolo_decode, yolo_sort, yolo_nms, yolo_boxes: the IDetect decode with the confidence filter, the score order, greedy NMS
//     and scale_coords, into fixed-size per-frame buffers so that the whole predict is one CUDA graph.
// Nothing here uses atomics in a way that changes results: candidate compaction order is undone by the sort, whose key
// (score, row) is unique.  Results are bitwise reproducible.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace vlfm {

#define YOLO_LAUNCHED(what)  do { VLFM_CHECK_LAUNCH(what); count_launch(); } while (0)

static unsigned yolo_grid(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  if (b > 132LL * 64) b = 132LL * 64;
  return (unsigned)(b < 1 ? 1 : b);
}

// ------------------------------------------------------------------------------------------------------------ preprocess
// cv2.resize(INTER_AREA) for a downscale, ResizeArea_Invoker: per source row sy of a destination row, buf = sum over the x-table
// entries (S * alpha, table order, fp32), then sum = beta_0 * buf_0, sum += beta_j * buf_j; saturate_cast<uchar> rounds half to
// even.  No FMA contraction (cv2's generic code is built without it).  The tables are built on the host in double, as cv2 does.
// Then fp16(v / 255) and ReOrg: out[b, y, x, g*3 + c] with g = (row parity) + 2 * (column parity); channels 12..15 are zero.
__global__ void __launch_bounds__(256)
yolo_preprocess_kernel(const uint8_t* __restrict__ img, __half* __restrict__ out, int B, int H, int W, int OH, int OW,
                       const int32_t* __restrict__ yofs, const int32_t* __restrict__ ysi, const float* __restrict__ ybeta,
                       const int32_t* __restrict__ xofs, const int32_t* __restrict__ xsi, const float* __restrict__ xalpha) {
  const long long total = (long long)B * OH * OW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % OW);
    const int dy = (int)((i / OW) % OH);
    const int b = (int)(i / ((long long)OW * OH));
    const uint8_t* src = img + (size_t)b * H * W * 3;
    float sum[3] = {0.f, 0.f, 0.f};
    const int k0 = xofs[dx], k1 = xofs[dx + 1];
    for (int j = yofs[dy]; j < yofs[dy + 1]; ++j) {
      const uint8_t* row = src + (size_t)ysi[j] * W * 3;
      float buf[3] = {0.f, 0.f, 0.f};
      for (int k = k0; k < k1; ++k) {
        const float a = xalpha[k];
        const uint8_t* p = row + xsi[k] * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)p[c], a));
      }
      const float beta = ybeta[j];
#pragma unroll
      for (int c = 0; c < 3; ++c) sum[c] = (j == yofs[dy]) ? __fmul_rn(beta, buf[c]) : __fadd_rn(sum[c], __fmul_rn(beta, buf[c]));
    }
    const int g = (dy & 1) + 2 * (dx & 1);
    __half* o = out + (((size_t)b * (OH / 2) + (dy >> 1)) * (OW / 2) + (dx >> 1)) * 16;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int v = __float2int_rn(sum[c]);
      v = v < 0 ? 0 : (v > 255 ? 255 : v);
      o[g * 3 + c] = __float2half_rn(__fdiv_rn((float)v, 255.f));
    }
    if (g == 0) {
#pragma unroll
      for (int c = 12; c < 16; ++c) o[c] = __float2half_rn(0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ layer ops
// MaxPool2d(2, 2): x [B,H,W,C] (ldx) -> out [B,H/2,W/2,C] (ldo)
__global__ void yolo_maxpool2_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ out, int ldo, int B, int H, int W,
                                     int C, int Ho, int Wo) {
  const long long total = (long long)B * Ho * Wo * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int ox = (int)(r % Wo), oy = (int)((r / Wo) % Ho), b = (int)(r / ((long long)Wo * Ho));
    const __half* p = x + (((size_t)b * H + 2 * oy) * W + 2 * ox) * ldx + c;
    const __half m = __hmax(__hmax(p[0], p[ldx]), __hmax(p[(size_t)W * ldx], p[(size_t)W * ldx + ldx]));
    out[r * ldo + c] = m;
  }
}

// SPPCSPC's MaxPool2d(k, 1, k // 2) for k = 5, 9, 13 (padding -inf): out + j*C (ldo) for the j-th pool.  A direct window max,
// which is exact for any order.
__global__ void yolo_spp_pools_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ out, int ldo, int B, int H, int W,
                                      int C) {
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int ox = (int)(r % W), oy = (int)((r / W) % H), b = (int)(r / ((long long)W * H));
    float m[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int dy = -6; dy <= 6; ++dy) {
      const int y = oy + dy;
      if ((unsigned)y >= (unsigned)H) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int xx = ox + dx;
        if ((unsigned)xx >= (unsigned)W) continue;
        const float v = __half2float(x[(((size_t)b * H + y) * W + xx) * ldx + c]);
        const int d = max(abs(dy), abs(dx));
        if (d <= 2) m[0] = fmaxf(m[0], v);
        if (d <= 4) m[1] = fmaxf(m[1], v);
        m[2] = fmaxf(m[2], v);
      }
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) out[r * ldo + j * C + c] = __float2half_rn(m[j]);
  }
}

// nn.Upsample(scale_factor=2, mode="nearest"): x [B,H,W,C] (ldx) -> out [B,2H,2W,C] (ldo)
__global__ void yolo_upsample2_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ out, int ldo, int B, int H, int W, int C) {
  const int C8 = C / 8;
  const long long total = (long long)B * 2 * H * 2 * W * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % C8);
    const long long r = i / C8;
    const int ox = (int)(r % (2 * W)), oy = (int)((r / (2 * W)) % (2 * H)), b = (int)(r / (4LL * W * H));
    *reinterpret_cast<uint4*>(out + r * ldo + 8 * q) =
        *reinterpret_cast<const uint4*>(x + (((size_t)b * H + oy / 2) * W + ox / 2) * ldx + 8 * q);
  }
}

// Shortcut: out = fp16(a + b) over [rows, C] (strides lda, ldb, ldo)
__global__ void yolo_add_kernel(const __half* __restrict__ a, int lda, const __half* __restrict__ b, int ldb, __half* __restrict__ out,
                                int ldo, long long rows, int C) {
  const int C2 = C / 2;
  const long long total = rows * C2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % C2);
    const long long r = i / C2;
    const float2 u = __half22float2(*reinterpret_cast<const __half2*>(a + r * lda + 2 * q));
    const float2 v = __half22float2(*reinterpret_cast<const __half2*>(b + r * ldb + 2 * q));
    *reinterpret_cast<__half2*>(out + r * ldo + 2 * q) = __floats2half2_rn(u.x + v.x, u.y + v.y);
  }
}

// ---------------------------------------------------------------------------------------------------------------- decode
// One detection level: head [B, ny, nx, ldh] fp16 (channel a*no + k; the 1x1 conv of IDetect.m[i]) -> candidate rows
// (level, anchor, y, x) from `row0`.  y = sigmoid(head); xy = (2y - 0.5 + grid) * stride, wh = (2y)^2 * anchor (pixels);
// kept when obj > conf_thres and conf = max_j(cls_j * obj) > conf_thres (first j on ties) and class j is allowed.
// A kept row is appended to its frame's candidates: [x1, y1, x2, y2, conf, class, row, 0].
__global__ void __launch_bounds__(128)
yolo_decode_kernel(const __half* __restrict__ head, int ldh, int B, int ny, int nx, int na, int nc, const float* __restrict__ anchors, float stride,
                   int row0, int R, const VlfmYoloParams* __restrict__ prm, float* __restrict__ cand, int* __restrict__ count) {
  const int no = nc + 5;
  const long long total = (long long)B * na * ny * nx;
  const float thr = prm->conf_thres;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % nx), y = (int)((i / nx) % ny), a = (int)((i / ((long long)nx * ny)) % na);
    const int b = (int)(i / ((long long)nx * ny * na));
    const __half* h = head + (((size_t)b * ny + y) * nx + x) * (size_t)ldh + a * no;
    const float obj = 1.f / (1.f + expf(-__half2float(h[4])));
    if (!(obj > thr)) continue;
    float best = -1.f;
    int bj = 0;
    for (int j = 0; j < nc; ++j) {
      const float s = (1.f / (1.f + expf(-__half2float(h[5 + j])))) * obj;
      if (s > best) { best = s; bj = j; }
    }
    if (!(best > thr) || !((prm->class_mask[bj >> 5] >> (bj & 31)) & 1u)) continue;
    float s[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] = 1.f / (1.f + expf(-__half2float(h[k])));
    const float cx = (s[0] * 2.f - 0.5f + (float)x) * stride, cy = (s[1] * 2.f - 0.5f + (float)y) * stride;
    const float w = (s[2] * 2.f) * (s[2] * 2.f) * anchors[2 * a], hh = (s[3] * 2.f) * (s[3] * 2.f) * anchors[2 * a + 1];
    const int slot = atomicAdd(count + b, 1);
    const int row = row0 + (int)((((long long)a * ny + y) * nx) + x);
    float4* c = reinterpret_cast<float4*>(cand + ((size_t)b * R + slot) * 8);
    c[0] = make_float4(cx - w / 2.f, cy - hh / 2.f, cx + w / 2.f, cy + hh / 2.f);
    c[1] = make_float4(best, (float)bj, (float)row, 0.f);
  }
}

// ------------------------------------------------------------------------------------------------------------------ sort
// order[b, rank] = candidate slot, rank = descending conf, then ascending row (the stable order of the reference's candidate
// rows).  The key (conf, row) is unique, so rank = #{keys greater}.  Grid (ceil(R / 256), B); candidates staged 256 at a time.
__device__ __forceinline__ unsigned long long yolo_key(const float* c) {
  unsigned u = __float_as_uint(c[4]);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)c[6]);
}
__global__ void __launch_bounds__(256)
yolo_sort_kernel(const float* __restrict__ cand, const int* __restrict__ count, int R, int32_t* __restrict__ order) {
  __shared__ unsigned long long s_key[256];
  const int b = blockIdx.y, n = min(count[b], R);
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (blockIdx.x * 256 >= n) return;
  const float* cb = cand + (size_t)b * R * 8;
  const unsigned long long mine = i < n ? yolo_key(cb + (size_t)i * 8) : 0ull;
  int rank = 0;
  for (int t = 0; t < n; t += 256) {
    __syncthreads();
    if (t + threadIdx.x < n) s_key[threadIdx.x] = yolo_key(cb + (size_t)(t + threadIdx.x) * 8);
    __syncthreads();
    const int m = min(256, n - t);
    for (int j = 0; j < m; ++j) rank += s_key[j] > mine;
  }
  if (i < n) order[(size_t)b * R + rank] = i;
}

// ------------------------------------------------------------------------------------------------------------------- NMS
// torchvision.ops.nms on the boxes offset by class * 4096 (0 when agnostic): in score order, keep a box unless an earlier kept
// box overlaps it with IoU > iou_thres; IoU as torchvision computes it in fp32.  One block per frame; `removed` is a bitmask
// over the sorted candidates in shared memory.  Stops at max_det keeps (the reference truncates the keep list there).
constexpr int YOLO_NMS_THREADS = 1024;
__device__ __forceinline__ void yolo_obox(const float* c, float off, float* o) {
  const float d = c[5] * off;
  o[0] = __fadd_rn(c[0], d); o[1] = __fadd_rn(c[1], d); o[2] = __fadd_rn(c[2], d); o[3] = __fadd_rn(c[3], d);
}
__global__ void __launch_bounds__(YOLO_NMS_THREADS)
yolo_nms_kernel(const float* __restrict__ cand, const int32_t* __restrict__ order, const int* __restrict__ count, int R,
                const VlfmYoloParams* __restrict__ prm, int max_det, int32_t* __restrict__ keep, int* __restrict__ nkeep) {
  extern __shared__ uint32_t s_removed[];
  __shared__ int s_cur, s_kept;
  const int b = blockIdx.x, n = min(count[b], R), words = (n + 31) / 32;
  const float* cb = cand + (size_t)b * R * 8;
  const int32_t* ob = order + (size_t)b * R;
  const float off = prm->agnostic ? 0.f : 4096.f, thr = prm->iou_thres;
  for (int w = threadIdx.x; w < words; w += blockDim.x) s_removed[w] = 0u;
  if (threadIdx.x == 0) { s_cur = 0; s_kept = 0; }
  __syncthreads();
  while (true) {
    const int cur = s_cur, kept = s_kept;
    if (cur >= n || kept >= max_det) break;
    float a[4];
    yolo_obox(cb + (size_t)ob[cur] * 8, off, a);
    const float sa = __fmul_rn(__fsub_rn(a[2], a[0]), __fsub_rn(a[3], a[1]));
    for (int j = cur + 1 + threadIdx.x; j < n; j += blockDim.x) {
      if ((s_removed[j >> 5] >> (j & 31)) & 1u) continue;
      float o[4];
      yolo_obox(cb + (size_t)ob[j] * 8, off, o);
      const float w = fmaxf(__fsub_rn(fminf(a[2], o[2]), fmaxf(a[0], o[0])), 0.f);
      const float h = fmaxf(__fsub_rn(fminf(a[3], o[3]), fmaxf(a[1], o[1])), 0.f);
      const float inter = __fmul_rn(w, h);
      const float sb = __fmul_rn(__fsub_rn(o[2], o[0]), __fsub_rn(o[3], o[1]));
      if (__fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > thr) atomicOr(&s_removed[j >> 5], 1u << (j & 31));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      keep[(size_t)b * max_det + kept] = ob[cur];
      s_kept = kept + 1;
      int nxt = n;
      for (int j = cur + 1; j < n; ) {            // next candidate not removed, a word at a time
        const uint32_t free_bits = ~s_removed[j >> 5] & (0xffffffffu << (j & 31));
        if (free_bits) { nxt = min(n, (j & ~31) + __ffs(free_bits) - 1); break; }
        j = (j & ~31) + 32;
      }
      s_cur = nxt;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) nkeep[b] = s_kept;
}

// -------------------------------------------------------------------------------------------------------------- boxes
// scale_coords(img1_shape, boxes, img0_shape) + clip + round + normalise: x = clamp((x - padx) / gain, 0, W), y likewise with
// pady and H; round half to even; x / W, y / H.  Rows past the frame's keep count are zero with class -1.
__global__ void yolo_boxes_kernel(const float* __restrict__ cand, const int32_t* __restrict__ keep, const int* __restrict__ nkeep, int R,
                                  int B, int max_det, float gain, float padx, float pady, int H, int W, float* __restrict__ boxes,
                                  float* __restrict__ scores, int32_t* __restrict__ classes, int* __restrict__ counts) {
  const int total = B * max_det;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i / max_det, r = i - b * max_det;
    const int n = nkeep[b];
    if (r == 0) counts[b] = n;
    if (r >= n) {
      reinterpret_cast<float4*>(boxes)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      scores[i] = 0.f;
      classes[i] = -1;
      continue;
    }
    const float* c = cand + ((size_t)b * R + keep[i]) * 8;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool isx = (k & 1) == 0;
      float t = __fdiv_rn(__fsub_rn(c[k], isx ? padx : pady), gain);
      t = fminf(fmaxf(t, 0.f), (float)(isx ? W : H));
      v[k] = __fdiv_rn(rintf(t), (float)(isx ? W : H));
    }
    reinterpret_cast<float4*>(boxes)[i] = make_float4(v[0], v[1], v[2], v[3]);
    scores[i] = c[4];
    classes[i] = (int32_t)c[5];
  }
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_yolo_preprocess(const uint8_t* d_img, void* d_out16, int B, int H, int W, int OH, int OW, const int32_t* d_yofs,
                                    const int32_t* d_ysi, const float* d_ybeta, const int32_t* d_xofs, const int32_t* d_xsi,
                                    const float* d_xalpha, void* stream) {
  if (!d_img || !d_out16 || !d_yofs || !d_ysi || !d_ybeta || !d_xofs || !d_xsi || !d_xalpha || B < 1 || OH < 2 || OW < 2 || (OH & 1) ||
      (OW & 1) || H < OH || W < OW || ((uintptr_t)d_out16 & 15)) {
    set_error("vlfm_yolo_preprocess: bad argument"); return VLFM_E_INVALID; }
  yolo_preprocess_kernel<<<yolo_grid((long long)B * OH * OW, 256), 256, 0, (cudaStream_t)stream>>>(
      d_img, (__half*)d_out16, B, H, W, OH, OW, d_yofs, d_ysi, d_ybeta, d_xofs, d_xsi, d_xalpha);
  YOLO_LAUNCHED("yolo_preprocess_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_maxpool2(const void* d_x16, int ldx, void* d_out16, int ldo, int B, int H, int W, int C, void* stream) {
  if (!d_x16 || !d_out16 || B < 1 || H < 2 || W < 2 || C < 1 || ldx < C || ldo < C) { set_error("vlfm_yolo_maxpool2: bad argument"); return VLFM_E_INVALID; }
  const int Ho = H / 2, Wo = W / 2;
  yolo_maxpool2_kernel<<<yolo_grid((long long)B * Ho * Wo * C, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_x16, ldx, (__half*)d_out16, ldo, B, H, W, C, Ho, Wo);
  YOLO_LAUNCHED("yolo_maxpool2_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_spp_pools(const void* d_x16, int ldx, void* d_out16, int ldo, int B, int H, int W, int C, void* stream) {
  if (!d_x16 || !d_out16 || B < 1 || H < 1 || W < 1 || C < 1 || ldx < C || ldo < 3 * C) { set_error("vlfm_yolo_spp_pools: bad argument"); return VLFM_E_INVALID; }
  yolo_spp_pools_kernel<<<yolo_grid((long long)B * H * W * C, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_x16, ldx, (__half*)d_out16, ldo, B, H, W, C);
  YOLO_LAUNCHED("yolo_spp_pools_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_upsample2(const void* d_x16, int ldx, void* d_out16, int ldo, int B, int H, int W, int C, void* stream) {
  if (!d_x16 || !d_out16 || B < 1 || H < 1 || W < 1 || C < 8 || (C & 7) || ldx < C || ldo < C || (ldx & 7) || (ldo & 7) ||
      ((uintptr_t)d_x16 & 15) || ((uintptr_t)d_out16 & 15)) { set_error("vlfm_yolo_upsample2: bad argument"); return VLFM_E_INVALID; }
  yolo_upsample2_kernel<<<yolo_grid((long long)B * 4 * H * W * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_x16, ldx, (__half*)d_out16, ldo, B, H, W, C);
  YOLO_LAUNCHED("yolo_upsample2_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_add(const void* d_a16, int lda, const void* d_b16, int ldb, void* d_out16, int ldo, long long rows, int C, void* stream) {
  if (!d_a16 || !d_b16 || !d_out16 || rows < 1 || C < 2 || (C & 1) || (lda & 1) || (ldb & 1) || (ldo & 1) || lda < C || ldb < C || ldo < C ||
      ((uintptr_t)d_a16 & 3) || ((uintptr_t)d_b16 & 3) || ((uintptr_t)d_out16 & 3)) { set_error("vlfm_yolo_add: bad argument"); return VLFM_E_INVALID; }
  yolo_add_kernel<<<yolo_grid(rows * (C / 2), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)d_a16, lda, (const __half*)d_b16, ldb, (__half*)d_out16, ldo, rows, C);
  YOLO_LAUNCHED("yolo_add_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_decode(const void* d_head16, int ldh, int B, int ny, int nx, int na, int nc, const float* d_anchors, float stride, int row0,
                                int R, const VlfmYoloParams* d_params, float* d_cand, int* d_count, void* stream) {
  if (!d_head16 || !d_anchors || !d_params || !d_cand || !d_count || B < 1 || ny < 1 || nx < 1 || na < 1 || nc < 1 || nc > 128 ||
      ldh < na * (nc + 5) || row0 < 0 || (long long)row0 + (long long)na * ny * nx > R || !(stride > 0.f)) {
    set_error("vlfm_yolo_decode: bad argument"); return VLFM_E_INVALID; }
  yolo_decode_kernel<<<yolo_grid((long long)B * na * ny * nx, 128), 128, 0, (cudaStream_t)stream>>>(
      (const __half*)d_head16, ldh, B, ny, nx, na, nc, d_anchors, stride, row0, R, d_params, d_cand, d_count);
  YOLO_LAUNCHED("yolo_decode_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_sort(const float* d_cand, const int* d_count, int R, int B, int32_t* d_order, void* stream) {
  if (!d_cand || !d_count || !d_order || R < 1 || B < 1 || B > 65535) { set_error("vlfm_yolo_sort: bad argument"); return VLFM_E_INVALID; }
  yolo_sort_kernel<<<dim3((R + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(d_cand, d_count, R, d_order);
  YOLO_LAUNCHED("yolo_sort_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_nms(const float* d_cand, const int32_t* d_order, const int* d_count, int R, int B, const VlfmYoloParams* d_params,
                             int max_det, int32_t* d_keep, int* d_nkeep, void* stream) {
  if (!d_cand || !d_order || !d_count || !d_params || !d_keep || !d_nkeep || R < 1 || R > 65536 || B < 1 || max_det < 1) {
    set_error("vlfm_yolo_nms: bad argument"); return VLFM_E_INVALID; }
  const size_t smem = (size_t)((R + 31) / 32) * 4;
  yolo_nms_kernel<<<B, YOLO_NMS_THREADS, smem, (cudaStream_t)stream>>>(d_cand, d_order, d_count, R, d_params, max_det, d_keep, d_nkeep);
  YOLO_LAUNCHED("yolo_nms_kernel");
  return VLFM_OK;
}

extern "C" int vlfm_yolo_boxes(const float* d_cand, const int32_t* d_keep, const int* d_nkeep, int R, int B, int max_det, float gain, float padx,
                               float pady, int H, int W, float* d_boxes, float* d_scores, int32_t* d_classes, int* d_counts, void* stream) {
  if (!d_cand || !d_keep || !d_nkeep || !d_boxes || !d_scores || !d_classes || !d_counts || R < 1 || B < 1 || max_det < 1 || H < 1 ||
      W < 1 || !(gain > 0.f) || ((uintptr_t)d_boxes & 15)) { set_error("vlfm_yolo_boxes: bad argument"); return VLFM_E_INVALID; }
  yolo_boxes_kernel<<<yolo_grid((long long)B * max_det, 256), 256, 0, (cudaStream_t)stream>>>(
      d_cand, d_keep, d_nkeep, R, B, max_det, gain, padx, pady, H, W, d_boxes, d_scores, d_classes, d_counts);
  YOLO_LAUNCHED("yolo_boxes_kernel");
  return VLFM_OK;
}
