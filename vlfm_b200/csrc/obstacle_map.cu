// Obstacle map: depth -> occupancy scatter and agent-radius dilation (sm_90a).
//
// Reference path: vlfm/mapping/obstacle_map.py:86-109
//   hole fill (:87-89, the hole_area_thresh == -1 form) -> metres (:92) -> mask (:93)
//   -> get_point_cloud (vlfm/utils/geometry_utils.py:216-236)
//   -> transform_points (:205-213) -> filter_points_by_height (obstacle_map.py:196-197)
//   -> _xy_to_px (vlfm/mapping/base_map.py:35-46, np.rint) -> boolean scatter (:101)
//   -> navigable = 1 - dilate(obstacles, ones(k,k)) (:105-109).
//
//  O1 obstacle_scatter_kernel  one thread per 4 depth pixels (float4), float64 geometry
//     exactly as numpy evaluates it, idempotent byte stores of 1 (no atomics).
//  O2 obstacle_dilate_kernel   k x k box dilation of the obstacle bytes into the
//     navigable bytes over a window around the camera (obstacles only ever appear
//     within max_depth/cos(hfov/2) of the camera and dilation is monotone, so the
//     windowed update equals the reference's full-grid cv2.dilate -- SURVEY A6), or
//     over the whole grid on the first update after reset.  Shared-memory tile with
//     halo, separable row/column max.
//
// Algorithmic bytes per environment step: 4*H*W depth read (+ <= H*W byte stores),
// window: 2*(2*half+1)^2 bytes.
#include <math.h>

#include "common.cuh"

namespace vlfm {

struct ObstDev {
  int H, W, G, ppm;
  float dscale, doff, maxd;
  double fx, fy, minh, maxh;
  int k, full, half;
};

// One depth pixel.  The evaluation order of every output is numpy's (see the header); what is reorganised is only WHICH outputs are
// evaluated: the height test (:196-197) needs ez alone, so ex / ey (and the lateral division feeding them) are computed for the
// few pixels that pass it.  `lazy_y`: T[9] == 0, so ez does not depend on the lateral coordinate (fma(0, py, acc) == acc);
// `affine`: the last row of T is (0, 0, 0, 1), so the homogeneous divisor is exactly 1.0 and x / 1.0 == x.  Both hold for every
// camera->episodic transform the policies build (xyz_yaw_to_tf_matrix); otherwise the general path runs.  FP64 divisions per pixel:
// 5 -> ~1.05 (an FP64 division costs about twenty FP64 FMAs -- the kernel was division-bound).
// Float32 pre-screen of the height test (affine transforms only): the episodic height of the point evaluated in float32 is within
// ~1e-5 m of the float64 value (|coordinates| < 100 m, four products); points farther than 5 mm outside the height band are
// dropped before any float64 work -- the exact float64 test below still decides everything that is kept.  Nine pixels in ten stop here.
struct ObstScreen { float t8, t9, t10, t11, inv_fx, inv_fy, lo, hi; bool on; };
__device__ __forceinline__ void obst_point(const ObstDev& p, const double* T, bool lazy_y, bool affine, uint8_t* obst, int* status,
                                           int b, int u, int v, float d, const uint8_t* fill, const ObstScreen& sc) {
  if (fill) { if (fill[v * p.W + u]) d = 1.f; }                  // fill_small_holes mask (:91, img_utils.py:388)
  else if (d == 0.f) d = 1.f;                                    // hole_area_thresh == -1 (:88-89)
  float z32 = __fadd_rn(__fmul_rn(d, p.dscale), p.doff);         // :92 float32
  if (!(z32 < p.maxd)) return;                                   // :93
  if (sc.on) {
    const float pzf = -(float)(v - p.H / 2) * z32 * sc.inv_fy, pyf = -(float)(u - p.W / 2) * z32 * sc.inv_fx;
    const float ezf = sc.t11 + sc.t10 * pzf + sc.t9 * pyf + sc.t8 * z32;
    if (ezf < sc.lo || ezf > sc.hi) return;
  }
  // get_point_cloud: int64 * float32 -> float64, then / fx  (geometry_utils.py:230-234)
  const double z = (double)z32;
  const double yc = __ddiv_rn(__dmul_rn((double)(v - p.H / 2), z), p.fy);
  const double px = z, pz = -yc;                                 // cloud = (z, -x, -y)
  double py = 0.0;
  if (!lazy_y) py = -__ddiv_rn(__dmul_rn((double)(u - p.W / 2), z), p.fx);
  // transform_points: np.dot(T, [p,1]) -- BLAS dgemm accumulates k=0..3 with FMA
  double ew = 1.0;
  if (!affine) ew = fma(T[15], 1.0, fma(T[14], pz, fma(T[13], py, __dmul_rn(T[12], px))));
  double ez = fma(T[11], 1.0, fma(T[10], pz, fma(T[9], py, __dmul_rn(T[8], px))));
  if (!affine) ez = __ddiv_rn(ez, ew);
  if (!(ez >= p.minh && ez <= p.maxh)) return;                   // obstacle_map.py:196-197
  if (lazy_y) py = -__ddiv_rn(__dmul_rn((double)(u - p.W / 2), z), p.fx);
  double ex = fma(T[3], 1.0, fma(T[2], pz, fma(T[1], py, __dmul_rn(T[0], px))));
  double ey = fma(T[7], 1.0, fma(T[6], pz, fma(T[5], py, __dmul_rn(T[4], px))));
  if (!affine) { ex = __ddiv_rn(ex, ew); ey = __ddiv_rn(ey, ew); }
  // _xy_to_px (base_map.py:44-46): px = rint(xy[::-1]*ppm) + origin; px[:,0] = G - px[:,0]
  long long c0 = (long long)rint(__dmul_rn(ey, (double)p.ppm)) + p.G / 2;
  long long r0 = (long long)rint(__dmul_rn(ex, (double)p.ppm)) + p.G / 2;
  long long col = (long long)p.G - c0;
  long long row = r0;
  // numpy fancy-index semantics: negative indices wrap once, otherwise IndexError
  if (row < 0) row += p.G;
  if (col < 0) col += p.G;
  if (row < 0 || row >= p.G || col < 0 || col >= p.G) { atomicOr(&status[b], VLFM_ST_SCATTER_OOB); return; }
  obst[(size_t)row * p.G + (size_t)col] = 1;                     // :101
}

__global__ void __launch_bounds__(256)
obstacle_scatter_kernel(ObstDev p, const int* __restrict__ slot, uint8_t* __restrict__ obstAll,
                        const float* __restrict__ depth, const double* __restrict__ tf,
                        int* __restrict__ status, const uint8_t* __restrict__ fillAll) {
  const int b = blockIdx.y;
  const uint8_t* fill = fillAll ? fillAll + (size_t)b * p.H * p.W : nullptr;
  __shared__ double T[16];
  if (threadIdx.x < 16) T[threadIdx.x] = tf[(size_t)b * 16 + threadIdx.x];
  __syncthreads();
  const bool lazy_y = T[9] == 0.0;
  const bool affine = T[12] == 0.0 && T[13] == 0.0 && T[14] == 0.0 && T[15] == 1.0;
  const ObstScreen sc{(float)T[8], (float)T[9], (float)T[10], (float)T[11], (float)(1.0 / p.fx), (float)(1.0 / p.fy),
                      (float)p.minh - 5e-3f, (float)p.maxh + 5e-3f,
                      // the error bound assumes metre-scale numbers (|R| <= 1, |t_z| and depth below 64 m, image offsets below 2^15 px)
                      affine && fabs(T[11]) < 64.0 && p.maxd < 64.f && fabs(T[8]) <= 1.0001 && fabs(T[9]) <= 1.0001 && fabs(T[10]) <= 1.0001 && p.H < 32768 && p.W < 32768};
  const int s = slot ? slot[b] : b;
  uint8_t* obst = obstAll + (size_t)s * p.G * p.G;
  const float* img = depth + (size_t)b * p.H * p.W;
  const int n = p.H * p.W;
  if ((p.W & 3) == 0) {
    const int n4 = n >> 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
      float4 d = __ldg(reinterpret_cast<const float4*>(img) + i);
      int pix = i << 2, v = pix / p.W, u = pix - v * p.W;
      obst_point(p, T, lazy_y, affine, obst, status, b, u + 0, v, d.x, fill, sc);
      obst_point(p, T, lazy_y, affine, obst, status, b, u + 1, v, d.y, fill, sc);
      obst_point(p, T, lazy_y, affine, obst, status, b, u + 2, v, d.z, fill, sc);
      obst_point(p, T, lazy_y, affine, obst, status, b, u + 3, v, d.w, fill, sc);
    }
  } else {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      int v = i / p.W, u = i - v * p.W;
      obst_point(p, T, lazy_y, affine, obst, status, b, u, v, __ldg(img + i), fill, sc);
    }
  }
}

// window (or whole grid) box dilation; tile 32 rows x 128 cols per block.
constexpr int DT_ROWS = 32, DT_COLS = 128, DT_MAXK = 31;

__global__ void __launch_bounds__(256)
obstacle_dilate_kernel(ObstDev p, const int* __restrict__ slot, const uint8_t* __restrict__ obstAll,
                       uint8_t* __restrict__ navAll, const double* __restrict__ tf, int tilesX) {
  __shared__ uint8_t tile[(DT_ROWS + DT_MAXK - 1)][DT_COLS + DT_MAXK - 1 + 1];
  __shared__ uint8_t rowmax[(DT_ROWS + DT_MAXK - 1)][DT_COLS];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int s = slot ? slot[b] : b;
  const int G = p.G, k = p.k, r = k / 2;
  const uint8_t* obst = obstAll + (size_t)s * G * G;
  uint8_t* nav = navAll + (size_t)s * G * G;
  int wr0 = 0, wc0 = 0, wr1 = G, wc1 = G;
  if (!p.full) {
    // agent cell as in obstacle_map.py:115-116 / base_map.py:44-46
    const double* T = tf + (size_t)b * 16;
    long long ar = (long long)rint(__dmul_rn(T[3], (double)p.ppm)) + G / 2;
    long long ac = (long long)G - ((long long)rint(__dmul_rn(T[7], (double)p.ppm)) + G / 2);
    long long a0 = ar - p.half, a1 = ar + p.half + 1, b0 = ac - p.half, b1 = ac + p.half + 1;
    if (a0 < 0 || b0 < 0 || a1 > G || b1 > G) { wr0 = 0; wc0 = 0; wr1 = G; wc1 = G; }  // near the edge: whole grid
    else { wr0 = (int)a0; wr1 = (int)a1; wc0 = (int)b0 & ~15; wc1 = (int)b1; }
  }
  const int wW = wc1 - wc0, wH = wr1 - wr0;
  const int tX = (wW + DT_COLS - 1) / DT_COLS, tY = (wH + DT_ROWS - 1) / DT_ROWS;
  for (int t = blockIdx.x; t < tX * tY; t += gridDim.x) {
    const int tr = wr0 + (t / tX) * DT_ROWS, tc = wc0 + (t % tX) * DT_COLS;
    const int inH = DT_ROWS + k - 1, inW = DT_COLS + k - 1;
    __syncthreads();
    for (int i = tid; i < inH * inW; i += 256) {
      int rr = i / inW, cc = i - rr * inW;
      int gr = tr - r + rr, gc = tc - r + cc;
      tile[rr][cc] = ((unsigned)gr < (unsigned)G && (unsigned)gc < (unsigned)G) ? obst[(size_t)gr * G + gc] : 0;
    }
    __syncthreads();
    for (int i = tid; i < inH * DT_COLS; i += 256) {
      int rr = i / DT_COLS, cc = i - rr * DT_COLS;
      uint8_t m = 0;
      for (int d = 0; d < k; ++d) m |= tile[rr][cc + d];
      rowmax[rr][cc] = m;
    }
    __syncthreads();
    // 4 output bytes per thread, one 32-bit store
    for (int i = tid; i < DT_ROWS * (DT_COLS / 4); i += 256) {
      int rr = i / (DT_COLS / 4), c4 = (i - rr * (DT_COLS / 4)) * 4;
      int gr = tr + rr, gc = tc + c4;
      if (gr >= wr1 || gc >= wc1) continue;
      uint8_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint8_t m = 0;
        for (int d = 0; d < k; ++d) m |= rowmax[rr + d][c4 + j];
        o[j] = m ? 0 : 1;                                         // 1 - dilate(...)
      }
      if (gc + 3 < G && ((G & 3) == 0)) {
        *reinterpret_cast<uchar4*>(nav + (size_t)gr * G + gc) = make_uchar4(o[0], o[1], o[2], o[3]);
      } else {
        for (int j = 0; j < 4 && gc + j < G; ++j) nav[(size_t)gr * G + gc + j] = o[j];
      }
    }
  }
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_obstacle_update(const VlfmObstacleParams* p, int batch, const int32_t* d_slot,
                                    uint8_t* d_obst, uint8_t* d_nav, const float* d_depth,
                                    const double* d_tf, const uint8_t* d_hole_fill, int32_t* d_status, void* stream) {
  if (!p || !d_obst || !d_nav || !d_depth || !d_tf || !d_status) { set_error("vlfm_obstacle_update: null argument"); return VLFM_E_INVALID; }
  if (batch <= 0) return VLFM_OK;
  if (p->kernel < 1 || p->kernel > DT_MAXK || (p->kernel & 1) == 0 || batch > 65535) {
    set_error("vlfm_obstacle_update: dilation kernel must be odd and <= %d", DT_MAXK); return VLFM_E_UNSUPPORTED; }
  ObstDev d;
  d.H = p->H; d.W = p->W; d.G = p->G; d.ppm = p->ppm;
  d.dscale = p->depth_scale; d.doff = p->depth_offset; d.maxd = p->max_depth_f32;
  d.fx = p->fx; d.fy = p->fy; d.minh = p->min_height; d.maxh = p->max_height;
  d.k = p->kernel; d.full = p->full_grid; d.half = p->roi_half;
  cudaStream_t st = (cudaStream_t)stream;
  int n4 = (p->H * p->W + 3) / 4;
  int bx = (n4 + 255) / 256;
  if (bx > 1184) bx = 1184;
  obstacle_scatter_kernel<<<dim3(bx, batch), 256, 0, st>>>(d, d_slot, d_obst, d_depth, d_tf, d_status, d_hole_fill);
  VLFM_CHECK_LAUNCH("obstacle_scatter_kernel");
  int side = d.full ? d.G : (2 * d.half + 1 + 16);
  int tiles = ((side + DT_COLS - 1) / DT_COLS) * ((side + DT_ROWS - 1) / DT_ROWS);
  if (!d.full) {
    // a window that would cross the grid border falls back to the whole grid inside the kernel
    int fullTiles = ((d.G + DT_COLS - 1) / DT_COLS) * ((d.G + DT_ROWS - 1) / DT_ROWS);
    if (fullTiles < tiles) tiles = fullTiles;
  }
  if (tiles > 2048) tiles = 2048;
  obstacle_dilate_kernel<<<dim3(tiles, batch), 256, 0, st>>>(d, d_slot, d_obst, d_nav, d_tf, 0);
  VLFM_CHECK_LAUNCH("obstacle_dilate_kernel");
  count_launch(2);
  return VLFM_OK;
}
