// Map frames for video (sm_90a): ValueMap.visualize / ObstacleMap.visualize and the trajectory + marker overlay, for a BATCH
// of environments per call.
//
// Reference: vlfm/mapping/value_map.py:189-219 (inferno rendering of the reduced map, vlfm/utils/img_utils.py:64-85),
// vlfm/mapping/obstacle_map.py:171-193 and vlfm/mapping/traj_visualizer.py (path, agent disc, heading line, markers).
// Output frames are [n, G, G, 3] uint8 BGR, C-contiguous: the array visualize() returns.
//
//   value_minmax / value_frame   masked (explored == 0 -> 0), flipped, zero cells -> max, min/max (exact, order-free),
//                                idx = uint8(((v - lo) / (hi - lo)) * 255) with one rounding per operation in the map's dtype
//                                (float32 or float64, no FMA contraction), inferno LUT, zero cells white.
//   obstacle_base / frontiers    white, explored, padding colour where nav == 0, obstacles black; frontier circles
//                                (radius 5, thickness 2) rasterised in UNFLIPPED grid coordinates and stored at row G-1-y,
//                                as the reference draws them before cv2.flip.  cv2's thickness-2 circle is not mirror-
//                                symmetric at every radius (3, 7, 9, 10 are not); at radius 5 it is, so drawing the mirrored
//                                circle after the flip would give the same pixels -- the order is kept for any radius.
//   draw_list                    per environment an ordered list of cv2.line / cv2.circle calls (LINE_8, shift 0), drawn in
//                                painter's order by one block: runs of same-colour records (the path) spread over its warps,
//                                within a primitive the lanes split rows / spans / steps.
//
// Rasterisation (csrc/cv_raster.cuh, shared with the explore half's occlusion rays) follows OpenCV 4.13's drawing.cpp, pinned
// against cv2 by tests/test_visualize_gpu.py:
//   thickness 1 line     LineIterator (8-connected) of the segment clipped to the image.
//   thickness t >= 2     ThickLine: the integer centre line is clipped to the image grown by t on every side, then
//                        FillConvexPoly of the 16.16 quad (half width (t + (t & 1)) / 2 along the fixed-point normal) +
//                        filled Circle caps of radius (t + 1) / 2 at both ends.
//   circle, t = 1 / -1   Circle (midpoint walk; outline points or horizontal spans), clipped per pixel.
//   circle, t >= 2       EllipseEx: ellipse2Poly (integer degrees, OpenCV's seven-decimal sine table) -> open PolyLine of
//                        16.16 points: ThickLine per segment WITHOUT the centre-line clip (shift 16), caps at the first
//                        segment's start and every segment's end.
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "cv_raster.cuh"

namespace vlfm {
namespace {

constexpr int MINMAX_PARTS = 64;            // partial reductions per environment (value frame)
constexpr int DRAW_MAX_THICKNESS = 16;
constexpr int DRAW_MAX_RADIUS = 255;
constexpr long long DRAW_MAX_COORD = 1ll << 24;

// ------------------------------------------------------------------------------------------------ canvas ----
// One frame [G, G, 3] as a cv_raster.cuh sink; `flip` stores grid row y at row G-1-y (the obstacle map draws its frontiers
// before cv2.flip).  Pixels outside the grid are dropped: cv2's per-pixel clipping.
struct Canvas {
  uint8_t* img;
  int G, flip;
  uint8_t b, g, r;
  __device__ __forceinline__ void put(long long x, long long y) const {
    if (x < 0 || y < 0 || x >= G || y >= G) return;
    const long long row = flip ? G - 1 - y : y;
    uint8_t* p = img + (row * G + x) * 3;
    p[0] = b; p[1] = g; p[2] = r;
  }
  __device__ __forceinline__ void span(long long y, long long x1, long long x2, int first, int step) const {
    if (y < 0 || y >= G) return;
    if (x1 < 0) x1 = 0;
    if (x2 > G - 1) x2 = G - 1;
    for (long long x = x1 + first; x <= x2; x += step) put(x, y);
  }
};

// ---------------------------------------------------------------------------------------------- kernels ----
template <typename T> struct Lim;
template <> struct Lim<float> { static __device__ float inf() { return __int_as_float(0x7f800000); } };
template <> struct Lim<double> { static __device__ double inf() { return __longlong_as_double(0x7ff0000000000000ll); } };

__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

__device__ __forceinline__ const uint8_t* explored_of(const uint8_t* ex, const int32_t* slots, int i, int G) {
  return ex ? ex + (size_t)(slots ? slots[i] : i) * G * G : nullptr;
}

// per part p of environment i: max over all cells (masked), min over the non-zero cells, whether a zero cell exists
template <typename T>
__global__ void __launch_bounds__(256) value_minmax_kernel(const T* __restrict__ red, const uint8_t* __restrict__ ex, const int32_t* __restrict__ slots,
                                                           int G, double* __restrict__ parts) {
  const int i = blockIdx.y, p = blockIdx.x;
  const T* v = red + (size_t)i * G * G;
  const uint8_t* e = explored_of(ex, slots, i, G);
  const long long n = (long long)G * G, lo = n * p / MINMAX_PARTS, hi_ = n * (p + 1) / MINMAX_PARTS;
  T mx = -Lim<T>::inf(), mn = Lim<T>::inf();
  int anyz = 0;
  for (long long k = lo + threadIdx.x; k < hi_; k += blockDim.x) {
    T x = v[k];
    if (e && e[k] == 0) x = T(0);
    mx = x > mx ? x : mx;
    if (x == T(0)) anyz = 1; else mn = x < mn ? x : mn;
  }
  __shared__ T s_mx[8], s_mn[8];
  __shared__ int s_z[8];
  for (int o = 16; o > 0; o >>= 1) {
    const T a = __shfl_xor_sync(0xffffffffu, mx, o), b = __shfl_xor_sync(0xffffffffu, mn, o);
    mx = a > mx ? a : mx; mn = b < mn ? b : mn;
    anyz |= __shfl_xor_sync(0xffffffffu, anyz, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s_mx[w] = mx; s_mn[w] = mn; s_z[w] = anyz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) { mx = s_mx[k] > mx ? s_mx[k] : mx; mn = s_mn[k] < mn ? s_mn[k] : mn; anyz |= s_z[k]; }
    double* o = parts + ((size_t)i * MINMAX_PARTS + p) * 3;
    o[0] = (double)mx; o[1] = (double)mn; o[2] = anyz;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) value_frame_kernel(const T* __restrict__ red, const uint8_t* __restrict__ ex, const int32_t* __restrict__ slots,
                                                          int G, const double* __restrict__ parts, const uint8_t* __restrict__ lut,
                                                          uint8_t* __restrict__ out) {
  const int i = blockIdx.y;
  __shared__ T s_lo, s_hi;
  if (threadIdx.x == 0) {
    T mx = -Lim<T>::inf(), mn = Lim<T>::inf();
    int anyz = 0;
    const double* q = parts + (size_t)i * MINMAX_PARTS * 3;
    for (int p = 0; p < MINMAX_PARTS; ++p) {
      const T a = (T)q[3 * p], b = (T)q[3 * p + 1];
      mx = a > mx ? a : mx; mn = b < mn ? b : mn; anyz |= q[3 * p + 2] != 0.0;
    }
    // zero cells take the map's max, which is >= every non-zero cell: it only becomes the min when nothing else is left
    s_hi = mx;
    s_lo = anyz ? (mn < mx ? mn : mx) : mn;
  }
  __syncthreads();
  const T lo = s_lo, hi = s_hi, ptp = sub_rn(hi, lo);
  const T* v = red + (size_t)i * G * G;
  const uint8_t* e = explored_of(ex, slots, i, G);
  uint8_t* o = out + (size_t)i * G * G * 3;
  const long long n = (long long)G * G;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const long long r = k / G, col = k - r * G;
    const long long src = (G - 1 - r) * G + col;                   // np.flipud
    T x = v[src];
    if (e && e[src] == 0) x = T(0);
    uint8_t* px = o + k * 3;
    if (x == T(0)) { px[0] = 255; px[1] = 255; px[2] = 255; continue; }
    const int idx = ptp == T(0) ? 0 : (int)mul_rn(div_rn(sub_rn(x, lo), ptp), T(255));
    px[0] = __ldg(lut + idx * 3); px[1] = __ldg(lut + idx * 3 + 1); px[2] = __ldg(lut + idx * 3 + 2);
  }
}

__global__ void __launch_bounds__(256) obstacle_base_kernel(const uint8_t* __restrict__ obst, const uint8_t* __restrict__ nav, const uint8_t* __restrict__ ex,
                                                            const int32_t* __restrict__ slots, int G, uchar3 pad, uint8_t* __restrict__ out) {
  const int i = blockIdx.y;
  const size_t base = (size_t)(slots ? slots[i] : i) * G * G;
  uint8_t* o = out + (size_t)i * G * G * 3;
  const long long n = (long long)G * G;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const long long r = k / G, col = k - r * G;
    const size_t src = base + (G - 1 - r) * G + col;                // cv2.flip(vis, 0)
    uchar3 c = make_uchar3(255, 255, 255);
    if (ex[src]) c = make_uchar3(200, 255, 200);
    if (nav[src] == 0) c = pad;
    if (obst[src]) c = make_uchar3(0, 0, 0);
    uint8_t* px = o + k * 3;
    px[0] = c.x; px[1] = c.y; px[2] = c.z;
  }
}

// cv2.circle(vis, (int(x), int(y)), 5, (200, 0, 0), 2) for every frontier midpoint, before the flip; one warp per frontier
// (every circle has the same colour, so their order does not matter)
__global__ void obstacle_frontiers_kernel(const double* __restrict__ fr, const int32_t* __restrict__ count, const int32_t* __restrict__ slots,
                                          int G, int max_frontiers, uint8_t* __restrict__ out) {
  const int i = blockIdx.y, s = slots ? slots[i] : i;
  int nf = count[s];
  nf = nf < max_frontiers ? nf : max_frontiers;
  const Canvas c{out + (size_t)i * G * G * 3, G, 1, 200, 0, 0};
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; f < nf; f += nw) {
    const double* p = fr + ((size_t)s * max_frontiers + f) * 2;
    cvr::circle_cv(c, G, (long long)p[0], (long long)p[1], 5, 2, lane);
  }
}

// one block per environment.  Painter's order only matters between primitives of different colours: a run of consecutive
// records with the same colour is drawn by the block's warps in parallel (one primitive per warp), runs one after another.
constexpr int DRAW_WARPS = 8;
__global__ void __launch_bounds__(DRAW_WARPS * 32) draw_list_kernel(uint8_t* __restrict__ frames, int G, const int32_t* __restrict__ lists, int batch) {
  const int i = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int32_t* off = lists;
  const int32_t* rec = lists + batch + 1;
  const int end = off[i + 1];
  for (int k = off[i]; k < end;) {
    const int32_t bgr = rec[(size_t)k * VLFM_DRAW_RECORD_INTS + 7];
    int run = k + 1;
    while (run < end && rec[(size_t)run * VLFM_DRAW_RECORD_INTS + 7] == bgr) ++run;
    const Canvas c{frames + (size_t)i * G * G * 3, G, 0, (uint8_t)(bgr & 0xff), (uint8_t)((bgr >> 8) & 0xff), (uint8_t)((bgr >> 16) & 0xff)};
    for (int j = k + warp; j < run; j += DRAW_WARPS) {
      const int32_t* r = rec + (size_t)j * VLFM_DRAW_RECORD_INTS;
      if (r[0] == VLFM_DRAW_LINE) cvr::line(c, G, r[1], r[2], r[3], r[4], r[6], lane);
      else cvr::circle_cv(c, G, r[1], r[2], r[5], r[6], lane);
    }
    __syncthreads();
    k = run;
  }
}

int blocks_for(long long n, int batch) {
  long long b = (n + 255) / 256;
  const long long cap = 1024 / (batch < 1 ? 1 : batch) + 8;
  return (int)(b < cap ? b : cap);
}

}  // namespace
}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_render_workspace_bytes(int batch, size_t* bytes) {
  if (batch < 1 || !bytes) { set_error("vlfm_render_workspace_bytes: bad argument"); return VLFM_E_INVALID; }
  *bytes = (size_t)batch * MINMAX_PARTS * 3 * sizeof(double);
  return VLFM_OK;
}

extern "C" int vlfm_render_value(int G, int batch, const int32_t* d_slots, const void* d_reduced, int reduced_f64, const uint8_t* d_explored,
                                 const uint8_t* d_lut, uint8_t* d_out, void* d_workspace, size_t workspace_bytes, void* stream) {
  size_t need = 0;
  if (G < 1 || batch < 1 || !d_reduced || !d_lut || !d_out || !d_workspace || (reduced_f64 != 0 && reduced_f64 != 1) ||
      vlfm_render_workspace_bytes(batch, &need) != VLFM_OK || workspace_bytes < need) {
    set_error("vlfm_render_value: bad argument (G %d, batch %d, workspace %zu < %zu)", G, batch, workspace_bytes, need);
    return VLFM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  double* parts = (double*)d_workspace;
  const dim3 g1(MINMAX_PARTS, batch), g2(blocks_for((long long)G * G, batch), batch);
  if (reduced_f64) {
    value_minmax_kernel<double><<<g1, 256, 0, st>>>((const double*)d_reduced, d_explored, d_slots, G, parts);
    value_frame_kernel<double><<<g2, 256, 0, st>>>((const double*)d_reduced, d_explored, d_slots, G, parts, d_lut, d_out);
  } else {
    value_minmax_kernel<float><<<g1, 256, 0, st>>>((const float*)d_reduced, d_explored, d_slots, G, parts);
    value_frame_kernel<float><<<g2, 256, 0, st>>>((const float*)d_reduced, d_explored, d_slots, G, parts, d_lut, d_out);
  }
  VLFM_CHECK_LAUNCH("vlfm_render_value");
  count_launch(2);
  return VLFM_OK;
}

extern "C" int vlfm_render_obstacle(int G, int batch, const int32_t* d_slots, const uint8_t* d_obst, const uint8_t* d_nav, const uint8_t* d_explored,
                                    const double* d_frontiers, const int32_t* d_count, int max_frontiers, int pad_b, int pad_g, int pad_r,
                                    uint8_t* d_out, void* stream) {
  const bool bad_pad = pad_b < 0 || pad_b > 255 || pad_g < 0 || pad_g > 255 || pad_r < 0 || pad_r > 255;
  if (G < 1 || batch < 1 || !d_obst || !d_nav || !d_explored || !d_frontiers || !d_count || max_frontiers < 1 || bad_pad || !d_out) {
    set_error("vlfm_render_obstacle: bad argument (G %d, batch %d, max_frontiers %d, padding colour %d %d %d)", G, batch, max_frontiers,
              pad_b, pad_g, pad_r);
    return VLFM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  obstacle_base_kernel<<<dim3(blocks_for((long long)G * G, batch), batch), 256, 0, st>>>(
      d_obst, d_nav, d_explored, d_slots, G, make_uchar3((uint8_t)pad_b, (uint8_t)pad_g, (uint8_t)pad_r), d_out);
  obstacle_frontiers_kernel<<<dim3(4, batch), 256, 0, st>>>(d_frontiers, d_count, d_slots, G, max_frontiers, d_out);
  VLFM_CHECK_LAUNCH("vlfm_render_obstacle");
  count_launch(2);
  return VLFM_OK;
}

extern "C" int vlfm_render_draw(int G, int batch, uint8_t* d_frames, const int32_t* h_lists, size_t list_ints, int32_t* d_lists,
                                size_t d_list_ints, void* stream) {
  if (G < 1 || batch < 1 || !d_frames || !h_lists || !d_lists || list_ints < (size_t)batch + 1 || d_list_ints < list_ints) {
    set_error("vlfm_render_draw: bad argument (G %d, batch %d, %zu list ints, device buffer %zu)", G, batch, list_ints, d_list_ints);
    return VLFM_E_INVALID;
  }
  const int32_t* off = h_lists;
  if (off[0] != 0) { set_error("vlfm_render_draw: offsets[0] = %d, expected 0", off[0]); return VLFM_E_INVALID; }
  for (int i = 0; i < batch; ++i)
    if (off[i + 1] < off[i]) { set_error("vlfm_render_draw: offsets decrease at environment %d", i); return VLFM_E_INVALID; }
  const size_t total = (size_t)off[batch];
  if ((size_t)batch + 1 + total * VLFM_DRAW_RECORD_INTS != list_ints) {
    set_error("vlfm_render_draw: %zu list ints, the offsets describe %zu", list_ints, (size_t)batch + 1 + total * VLFM_DRAW_RECORD_INTS);
    return VLFM_E_INVALID;
  }
  const int32_t* rec = h_lists + batch + 1;
  for (size_t k = 0; k < total; ++k) {
    const int32_t* r = rec + k * VLFM_DRAW_RECORD_INTS;
    bool ok = r[0] == VLFM_DRAW_LINE || r[0] == VLFM_DRAW_CIRCLE;
    for (int j = 1; j <= 4; ++j) ok = ok && r[j] > -DRAW_MAX_COORD && r[j] < DRAW_MAX_COORD;
    if (r[0] == VLFM_DRAW_LINE) ok = ok && r[6] >= 1 && r[6] <= DRAW_MAX_THICKNESS;
    else ok = ok && r[5] >= 0 && r[5] <= DRAW_MAX_RADIUS && (r[6] == -1 || (r[6] >= 1 && r[6] <= DRAW_MAX_THICKNESS));
    ok = ok && ((uint32_t)r[7] >> 24) == 0;
    if (!ok) {
      set_error("vlfm_render_draw: record %zu is invalid (op %d, (%d, %d) (%d, %d), radius %d, thickness %d, colour %#x)", k, r[0], r[1], r[2],
                r[3], r[4], r[5], r[6], (unsigned)r[7]);
      return VLFM_E_INVALID;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = check_cuda(cudaMemcpyAsync(d_lists, h_lists, list_ints * sizeof(int32_t), cudaMemcpyHostToDevice, st), "vlfm_render_draw: upload");
  if (rc) return rc;
  if (total == 0) return VLFM_OK;
  draw_list_kernel<<<batch, DRAW_WARPS * 32, 0, st>>>(d_frames, G, d_lists, batch);
  VLFM_CHECK_LAUNCH("vlfm_render_draw");
  count_launch(1);
  return VLFM_OK;
}
