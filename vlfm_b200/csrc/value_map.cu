// Value-map FOV-cone projection + confidence-weighted fusion (sm_90a).
//
// Reference path: vlfm/mapping/value_map.py:100-128 (update_map) =
//   _process_local_data :221-286, _localize_new_data :288-319,
//   rotate_image (vlfm/utils/img_utils.py:9-28), place_img_in_img (:31-61),
//   _fuse_new_data :357-429.
//
// Two launches per batch of environments:
//
//  K1 value_depth_geom_kernel   grid (W/128, H/32, B)
//     streaming pass over depth: per-column max (np.max(depth, axis=0), :234) into
//     per-chunk partials; the LAST block of each environment (ticket counter) then
//       - reduces the partials, turns them into the (W+2)-vertex occlusion polygon
//         (:234-257; float32 row arithmetic, float64 column arithmetic),
//       - rasterises cv2.drawContours(cone,[poly],-1,0,-1) (:260) into a kill
//         bitmap in shared memory: 8-connected outline (closed-form OpenCV
//         LineIterator) + even-odd 16.16 scanline interior (XOR toggles + per-row
//         prefix XOR),
//     and publishes the kill bitmap; block (0,0) of each environment, concurrently with the
//     streaming pass, derives cv2.warpAffine's fixed-point coordinate tables for the rotation
//     by -yaw (img_utils.py:23-26; AB_BITS=10, INTER_BITS=5) and the camera cell (:309-313).
//     {camera cell, tables, kill bitmap} = the "geometry blob" K2 consumes.
//  K2 value_cone_fuse_kernel    grid (tiles, B)
//     for every cell of the R x R window around the camera cell: inverse-map through
//     the fixed-point rotation, 4-tap bilinear sample of (template AND NOT kill),
//     cast to float32 (curr_map, :316-317) and fuse into conf/value in place
//     (:398-429).  Only cells with a positive new confidence touch HBM; aligned
//     16-byte accesses on the C==1 path.
//
// Algorithmic bytes per environment step: 4*H*W (depth) + 4*R^2 (template)
// + (4+4C)*R^2 read + (4+4C)*R^2 write  (SURVEY.md section 8d).
#include <math.h>

#include "common.cuh"

namespace vlfm {

constexpr int K1_THREADS = 256;
constexpr int GEOM_THREADS = 1024;
constexpr int K1_ROWS = 32;   // rows per chunk: 8 warps x 4 rows
constexpr int K1_COLS = 128;  // 32 lanes x float4
constexpr int K2_THREADS = 256;
constexpr int LONG_EDGE = 24;

struct ValueDev {
  int H, W, G, C, R, ppm;
  float dscale, doff, thr;
  int fusion;
  int nChunks, nColTiles, WPR;
  int wsWords;      // 32-bit words of workspace per environment
  int offCounter;   // word offsets inside an environment's workspace
  int offHeader;
  int offTables;
  int offKill;
};

static ValueDev make_dev(const VlfmValueParams& p) {
  ValueDev d;
  d.H = p.H; d.W = p.W; d.G = p.G; d.C = p.C; d.R = p.R; d.ppm = p.ppm;
  d.dscale = p.depth_scale; d.doff = p.depth_offset; d.thr = p.decision_threshold;
  d.fusion = p.fusion;
  d.nChunks = (p.H + K1_ROWS - 1) / K1_ROWS;
  d.nColTiles = (p.W + K1_COLS - 1) / K1_COLS;
  d.WPR = (p.R + 31) / 32;
  int o = d.nChunks * p.W;
  o = (o + 3) & ~3;
  d.offCounter = o; o += 4;
  d.offHeader = o;  o += 4;
  d.offTables = o;  o += 4 * p.R;
  o = (o + 3) & ~3;
  d.offKill = o;    o += p.R * d.WPR;
  d.wsWords = (o + 3) & ~3;
  return d;
}

// ---------------------------------------------------------------------------------
// OpenCV LineIterator (8-connected), pixel k in closed form.  (oracle/cv_prims.py)
// ---------------------------------------------------------------------------------
struct LineWalk {
  int x0, y0, sy, major, minor;
  bool ymajor;
  __device__ LineWalk(int ax, int ay, int bx, int by) {
    if (bx < ax) { int t = ax; ax = bx; bx = t; t = ay; ay = by; by = t; }
    int dx = bx - ax, dy = by - ay;
    sy = dy >= 0 ? 1 : -1;
    int ady = dy >= 0 ? dy : -dy;
    ymajor = ady > dx;
    major = ymajor ? ady : dx;
    minor = ymajor ? dx : ady;
    x0 = ax; y0 = ay;
  }
  __device__ void pixel(int k, int& x, int& y) const {
    int s = major ? (2 * minor * k + major - 1) / (2 * major) : 0;
    if (ymajor) { x = x0 + s; y = y0 + sy * k; }
    else        { x = x0 + k; y = y0 + sy * s; }
  }
};

__device__ __forceinline__ void plot_or(uint32_t* plane, int WPR, int R, int x, int y) {
  if ((unsigned)x < (unsigned)R && (unsigned)y < (unsigned)R)
    atomicOr(&plane[y * WPR + (x >> 5)], 1u << (x & 31));
}

// one scanline of one polygon edge: even-odd toggle + exact-hit bit
__device__ __forceinline__ void edge_row(uint32_t* tog, uint32_t* orb, int WPR, int R,
                                         long long x16, long long dxe, int ya, int r) {
  long long X = x16 + dxe * (long long)(r - ya);
  long long t = (X >> 16) + 1;  // first column c with (c << 16) > X
  if (t < 0) t = 0;
  if (t < R) atomicXor(&tog[r * WPR + (int)(t >> 5)], 1u << ((int)t & 31));
  if ((X & 0xFFFF) == 0) {
    long long c = X >> 16;
    if (c >= 0 && c < R) atomicOr(&orb[r * WPR + (int)(c >> 5)], 1u << ((int)c & 31));
  }
}

// ---------------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(K1_THREADS)
value_depth_geom_kernel(ValueDev p, const float* __restrict__ depth, const double* __restrict__ tf,
                        const double* __restrict__ tanv, uint32_t* __restrict__ ws,
                        const int* __restrict__ slot, int* __restrict__ status) {
  extern __shared__ __align__(16) uint32_t smem[];
  const int b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint32_t* wsb = ws + (size_t)b * p.wsWords;
  float* partial = reinterpret_cast<float*>(wsb);
  const float* img = depth + (size_t)b * p.H * p.W;
  pdl_trigger();

  // ---- phase 1: column max over this block's 32 x 128 tile
  {
    float* sm = reinterpret_cast<float*>(smem);  // [8][128]
    const int col0 = blockIdx.x * K1_COLS + lane * 4;
    const int row0 = blockIdx.y * K1_ROWS + warp * 4;
    float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;
    if ((p.W & 3) == 0 && col0 + 3 < p.W) {
      float4 v[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        int row = row0 + r;
        v[r] = row < p.H ? __ldg(reinterpret_cast<const float4*>(img + (size_t)row * p.W + col0))
                         : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        m0 = fmaxf(m0, v[r].x); m1 = fmaxf(m1, v[r].y);
        m2 = fmaxf(m2, v[r].z); m3 = fmaxf(m3, v[r].w);
      }
    } else {
      for (int r = 0; r < 4; ++r) {
        int row = row0 + r;
        if (row >= p.H) break;
        const float* q = img + (size_t)row * p.W;
        if (col0 + 0 < p.W) m0 = fmaxf(m0, __ldg(q + col0 + 0));
        if (col0 + 1 < p.W) m1 = fmaxf(m1, __ldg(q + col0 + 1));
        if (col0 + 2 < p.W) m2 = fmaxf(m2, __ldg(q + col0 + 2));
        if (col0 + 3 < p.W) m3 = fmaxf(m3, __ldg(q + col0 + 3));
      }
    }
    *reinterpret_cast<float4*>(&sm[warp * K1_COLS + lane * 4]) = make_float4(m0, m1, m2, m3);
    __syncthreads();
    if (tid < K1_COLS) {
      int col = blockIdx.x * K1_COLS + tid;
      if (col < p.W) {
        float m = sm[tid];
#pragma unroll
        for (int w = 1; w < 8; ++w) m = fmaxf(m, sm[w * K1_COLS + tid]);
        __stcg(&partial[blockIdx.y * p.W + col], m);
      }
    }
  }

  // ---- block (0,0) of each environment: pose-only geometry (independent of the depth image), overlapped
  // with the other blocks' streaming pass: camera cell (:309-313) and cv2.warpAffine's fixed-point tables
  // for the rotation by -yaw (img_utils.py:23-26).
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    __shared__ double s_mi[6];
    const int R = p.R;
    if (tid == 0) {
      const double* T = tf + (size_t)b * 16;
      // extract_yaw (geometry_utils.py:145-159), rotate_image(curr, -yaw) (value_map.py:306)
      double yaw = atan2(T[4], T[0]);
      double deg = (-yaw) * 57.295779513082323;           // np.degrees
      double ang = deg * 0.017453292519943295;            // cv: angle *= CV_PI/180
      double a = cos(ang), bb = sin(ang);
      double c = (double)(R / 2);
      // cv2.getRotationMatrix2D, then cv2.warpAffine's in-place inversion (no FMA)
      double m00 = a, m01 = bb, m02 = __dsub_rn(__dmul_rn(__dsub_rn(1.0, a), c), __dmul_rn(bb, c));
      double m10 = -bb, m11 = a, m12 = __dadd_rn(__dmul_rn(bb, c), __dmul_rn(__dsub_rn(1.0, a), c));
      double det = __dsub_rn(__dmul_rn(m00, m11), __dmul_rn(m01, m10));
      det = det != 0.0 ? __ddiv_rn(1.0, det) : 0.0;
      double i00 = __dmul_rn(m11, det), i11 = __dmul_rn(m00, det);
      double i01 = __dmul_rn(m01, -det), i10 = __dmul_rn(m10, -det);
      double b1 = __dsub_rn(__dmul_rn(-i00, m02), __dmul_rn(i01, m12));
      double b2 = __dsub_rn(__dmul_rn(-i10, m02), __dmul_rn(i11, m12));
      s_mi[0] = i00; s_mi[1] = i01; s_mi[2] = b1; s_mi[3] = i10; s_mi[4] = i11; s_mi[5] = b2;
      // camera cell (value_map.py:309-313): int() truncation, not rint
      double cx = __ddiv_rn(T[3], T[15]), cy = __ddiv_rn(T[7], T[15]);
      int px = (int)__dmul_rn(cx, (double)p.ppm) + p.G / 2;
      int py = (int)__dmul_rn(-cy, (double)p.ppm) + p.G / 2;
      int valid = (px >= 0 && px < p.G && py >= 0 && py < p.G);
      if (!valid) atomicOr(&status[slot ? slot[b] : b], VLFM_ST_CAMERA_OFF_GRID);   // flags belong to the grid slot
      wsb[p.offHeader + 0] = (uint32_t)px;
      wsb[p.offHeader + 1] = (uint32_t)py;
      wsb[p.offHeader + 2] = (uint32_t)valid;
    }
    __syncthreads();
    int* tab = reinterpret_cast<int*>(wsb + p.offTables);
    for (int i = tid; i < R; i += K1_THREADS) {
      double di = (double)i;
      // X0 = saturate_cast<int>((M[1]*y + M[2])*AB_SCALE) + round_delta; adelta = saturate_cast<int>(M[0]*x*AB_SCALE)
      tab[0 * R + i] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(s_mi[1], di), s_mi[2]), 1024.0)) + 16;
      tab[1 * R + i] = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(s_mi[4], di), s_mi[5]), 1024.0)) + 16;
      tab[2 * R + i] = __double2int_rn(__dmul_rn(__dmul_rn(s_mi[0], di), 1024.0));
      tab[3 * R + i] = __double2int_rn(__dmul_rn(__dmul_rn(s_mi[3], di), 1024.0));
    }
  }

}

// K1b: one 1024-thread block per environment turns the column maxima into the occlusion polygon and rasterises it into the kill
// bitmap.  Launched with programmatic dependent launch: the shared-memory planes are cleared while K1a drains.
__global__ void __launch_bounds__(GEOM_THREADS)
value_geom_kernel(ValueDev p, const double* __restrict__ tanv, uint32_t* __restrict__ ws) {
  extern __shared__ __align__(16) uint32_t smem[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint32_t* wsb = ws + (size_t)b * p.wsWords;
  const float* partial = reinterpret_cast<const float*>(wsb);
  pdl_trigger();

  // ---- phase 2: geometry blob (one block per environment)
  const int R = p.R, W = p.W, WPR = p.WPR, E = W + 2;
  int2* verts = reinterpret_cast<int2*>(smem);                 // [E]
  uint32_t* tog = smem + 2 * ((E + 1) & ~1);                   // [R*WPR]
  uint32_t* orb = tog + R * WPR;                               // [R*WPR]
  int* longList = reinterpret_cast<int*>(orb + R * WPR);       // [E]
  __shared__ int s_nlong;

  for (int i = tid; i < R * WPR; i += GEOM_THREADS) { tog[i] = 0; orb[i] = 0; }
  pdl_wait();                                                  // the column maxima of K1a are visible from here on
  if (tid == 0) {
    s_nlong = 0;
    verts[0] = make_int2(0, R - 1);          // start = [[0, last_col]]  (value_map.py:255)
    verts[E - 1] = make_int2(R - 1, R - 1);  // end   = [[last_row, last_col]]
  }
  const float half_f = (float)((double)R * 0.5);
  const double half_d = (double)R * 0.5;
  for (int i = tid; i < W; i += GEOM_THREADS) {
    float m = ld_cg_f32(&partial[i]);
    for (int ch = 1; ch < p.nChunks; ++ch) m = fmaxf(m, ld_cg_f32(&partial[ch * W + i]));
    float far = __fadd_rn(__fmul_rn(m, p.dscale), p.doff);                   // :234 float32
    int row = (int)__fadd_rn(__fmul_rn(far, (float)p.ppm), half_f);          // :248 float32
    double lat = __dmul_rn((double)far, tanv[i]);                            // :242 float64
    int col = (int)__dadd_rn(__dmul_rn(lat, (double)p.ppm), half_d);         // :249 float64
    verts[i + 1] = make_int2(col, row);                                      // cv2 point (x=col, y=row)
  }
  __syncthreads();

  // edges: thread-per-edge for short ones, warp-cooperative for long ones
  for (int e = tid; e < E; e += GEOM_THREADS) {
    int2 A = verts[e], B = verts[e + 1 == E ? 0 : e + 1];
    LineWalk lw(A.x, A.y, B.x, B.y);
    int dyabs = A.y > B.y ? A.y - B.y : B.y - A.y;
    if (lw.major > LONG_EDGE || dyabs > LONG_EDGE) {
      longList[atomicAdd(&s_nlong, 1)] = e;
      continue;
    }
    {  // OpenCV LineIterator, incremental form (no divisions): err<0 steps the minor axis
      int x = lw.x0, y = lw.y0, err = lw.major - 2 * lw.minor;
      for (int k = 0; k <= lw.major; ++k) {
        plot_or(orb, WPR, R, x, y);
        const bool m = err < 0;
        err += -2 * lw.minor + (m ? 2 * lw.major : 0);
        if (lw.ymajor) { y += lw.sy; x += m ? 1 : 0; } else { x += 1; y += m ? lw.sy : 0; }
      }
    }
    if (A.y != B.y) {
      int xa = A.x, ya = A.y, xb = B.x, yb = B.y;
      if (ya > yb) { int t = xa; xa = xb; xb = t; t = ya; ya = yb; yb = t; }
      long long dxe = ((long long)(xb - xa) << 16) / (long long)(yb - ya);
      long long x16 = (long long)xa << 16;
      int r0 = ya < 0 ? 0 : ya, r1 = yb < R ? yb : R;
      for (int r = r0; r < r1; ++r) edge_row(tog, orb, WPR, R, x16, dxe, ya, r);
    }
  }
  __syncthreads();
  for (int li = warp; li < s_nlong; li += GEOM_THREADS / 32) {
    int e = longList[li];
    int2 A = verts[e], B = verts[e + 1 == E ? 0 : e + 1];
    LineWalk lw(A.x, A.y, B.x, B.y);
    for (int k = lane; k <= lw.major; k += 32) { int x, y; lw.pixel(k, x, y); plot_or(orb, WPR, R, x, y); }
    if (A.y != B.y) {
      int xa = A.x, ya = A.y, xb = B.x, yb = B.y;
      if (ya > yb) { int t = xa; xa = xb; xb = t; t = ya; ya = yb; yb = t; }
      long long dxe = ((long long)(xb - xa) << 16) / (long long)(yb - ya);
      long long x16 = (long long)xa << 16;
      int r0 = ya < 0 ? 0 : ya, r1 = yb < R ? yb : R;
      for (int r = r0 + lane; r < r1; r += 32) edge_row(tog, orb, WPR, R, x16, dxe, ya, r);
    }
  }
  __syncthreads();

  // publish the kill bitmap
  uint32_t* kill = wsb + p.offKill;
  for (int r = tid; r < R; r += GEOM_THREADS) {
    uint32_t carry = 0;
    for (int w = 0; w < WPR; ++w) {
      uint32_t t = tog[r * WPR + w];
      uint32_t x = t;
      x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
      x ^= carry;
      if (__popc(t) & 1) carry = ~carry;
      kill[r * WPR + w] = x | orb[r * WPR + w];
    }
  }
}

// ---------------------------------------------------------------------------------
// K2
// ---------------------------------------------------------------------------------
struct FuseCtx {
  const int* X0; const int* Y0; const int* AD; const int* BD;
  const uint32_t* kill;
  const float* tmpl;
  int R, WPR;
};

// warpAffine INTER_LINEAR sample of the occlusion-cut template at output (y, x), then
// the float64 -> float32 cast of the paste into curr_map (value_map.py:316-317).
// The four template loads are issued unconditionally (clamped addresses) BEFORE the range / kill-bit tests, so they are
// independent and overlap; round 1 tested each tap's kill bit first, which serialised 16 L2 round trips per 4-cell item
// (value_cone_fuse_kernel: 33 us for 32 environments at 21 % occupancy).
__device__ __forceinline__ float cone_sample(const FuseCtx& c, int y, int x) {
  const int X = (c.X0[y] + c.AD[x]) >> 5, Y = (c.Y0[y] + c.BD[x]) >> 5;
  const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
  if (sx < -1 || sx >= c.R || sy < -1 || sy >= c.R) return 0.f;
  const int R = c.R;
  const int x0 = max(sx, 0), x1 = min(sx + 1, R - 1), y0 = max(sy, 0), y1 = min(sy + 1, R - 1);
  const float t00 = __ldg(c.tmpl + y0 * R + x0), t01 = __ldg(c.tmpl + y0 * R + x1);
  const float t10 = __ldg(c.tmpl + y1 * R + x0), t11 = __ldg(c.tmpl + y1 * R + x1);
  const bool cx0 = sx >= 0, cx1 = sx + 1 < R, cy0 = sy >= 0, cy1 = sy + 1 < R;
  auto alive = [&](int yy, int xx) { return !((c.kill[yy * c.WPR + (xx >> 5)] >> (xx & 31)) & 1u); };
  const double v00 = (cx0 && cy0 && alive(y0, x0)) ? (double)t00 : 0.0, v01 = (cx1 && cy0 && alive(y0, x1)) ? (double)t01 : 0.0;
  const double v10 = (cx0 && cy1 && alive(y1, x0)) ? (double)t10 : 0.0, v11 = (cx1 && cy1 && alive(y1, x1)) ? (double)t11 : 0.0;
  const double s = 1.0 / 1024.0;
  double acc = v00 * ((32 - fx) * (32 - fy) * s) + v01 * (fx * (32 - fy) * s) +
               v10 * ((32 - fx) * fy * s) + v11 * (fx * fy * s);  // exact in float64
  return (float)acc;
}

// _fuse_new_data for one cell with nw > 0.  Returns false when the cell is unchanged.
__device__ __forceinline__ bool fuse_cell(const ValueDev& p, float nw, float& conf, float* val,
                                          const double* vals) {
  const int mode = p.fusion & 3;
  if (mode == VLFM_FUSE_REPLACE) {
    conf = nw;
    for (int ch = 0; ch < p.C; ++ch) val[ch] = (float)vals[ch];
    return true;
  }
  float c = conf;
  if (p.fusion & VLFM_FUSE_EQUAL) { if (c > 0.f) c = 1.f; nw = 1.f; }
  if (nw < p.thr && nw < c) return false;            // :398-399 silenced -> no-op
  if (mode == VLFM_FUSE_MAX_CONFIDENCE) {
    if (!(nw > c)) return false;                     // :401-408
    conf = nw;
    for (int ch = 0; ch < p.C; ++ch) val[ch] = (float)vals[ch];
    return true;
  }
  float den = __fadd_rn(c, nw);                      // :413-417 float32
  float w1 = __fdiv_rn(c, den), w2 = __fdiv_rn(nw, den);
  conf = __fadd_rn(__fmul_rn(c, w1), __fmul_rn(nw, w2));
  for (int ch = 0; ch < p.C; ++ch)                   // :422 float64 (value grid stored as float32)
    val[ch] = (float)__dadd_rn(__dmul_rn((double)val[ch], (double)w1), __dmul_rn(vals[ch], (double)w2));
  return true;
}

__global__ void __launch_bounds__(K2_THREADS)
value_cone_fuse_kernel(ValueDev p, const int* __restrict__ slot, float* __restrict__ conf,
                       float* __restrict__ value, const double* __restrict__ values,
                       const float* __restrict__ tmpl, const uint8_t* __restrict__ explored,
                       const uint32_t* __restrict__ ws, int rowsPerTile) {
  extern __shared__ __align__(16) uint32_t smem[];
  const int b = blockIdx.y, tid = threadIdx.x;
  const uint32_t* wsb = ws + (size_t)b * p.wsWords;
  pdl_wait();                                                  // geometry blob of K1a / K1b
  const int px = (int)wsb[p.offHeader + 0], py = (int)wsb[p.offHeader + 1];
  if (!wsb[p.offHeader + 2]) return;
  const int R = p.R, G = p.G, C = p.C, WPR = p.WPR;
  int* tab = reinterpret_cast<int*>(smem);
  uint32_t* kill = smem + 4 * R;
  for (int i = tid; i < 4 * R; i += K2_THREADS) tab[i] = (int)wsb[p.offTables + i];
  for (int i = tid; i < R * WPR; i += K2_THREADS) kill[i] = wsb[p.offKill + i];
  __syncthreads();
  FuseCtx c{tab, tab + R, tab + 2 * R, tab + 3 * R, kill, tmpl, R, WPR};

  const int s = slot ? slot[b] : b;
  float* confS = conf + (size_t)s * G * G;
  float* valS = value + (size_t)s * G * G * C;
  const uint8_t* expS = explored ? explored + (size_t)s * G * G : nullptr;
  const double* vals = values + (size_t)b * C;

  const int top = px - R / 2, left = py - R / 2;   // place_img_in_img (img_utils.py:44-45)
  const int y0 = blockIdx.x * rowsPerTile;
  const int y1 = min(R, y0 + rowsPerTile);
  const int gcLo = max(left, 0), gcHi = min(left + R, G);
  if (gcHi <= gcLo) return;
  const int gcStart = gcLo & ~3;
  const int nGroups = (gcHi - gcStart + 3) >> 2;
  const bool vec = (C == 1) && ((G & 3) == 0);
  const int items = (y1 - y0) * nGroups;
  for (int it = tid; it < items; it += K2_THREADS) {
    const int yy = y0 + it / nGroups;
    const int gr = top + yy;
    if ((unsigned)gr >= (unsigned)G) continue;
    const int gc0 = gcStart + 4 * (it % nGroups);
    float nw[4];
    bool any = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int gc = gc0 + j, x = gc - left;
      float v = 0.f;
      if (x >= 0 && x < R && gc < G) {
        v = cone_sample(c, yy, x);
        if (expS && v > 0.f && expS[(size_t)gr * G + gc] == 0) v = 0.f;   // :372
      }
      nw[j] = v;
      any |= v > 0.f;
    }
    if (!any) continue;
    const size_t cell0 = (size_t)gr * G + gc0;
    if (vec) {
      float4 cf = *reinterpret_cast<const float4*>(confS + cell0);
      float4 vl = *reinterpret_cast<const float4*>(valS + cell0);
      float cfa[4] = {cf.x, cf.y, cf.z, cf.w}, vla[4] = {vl.x, vl.y, vl.z, vl.w};
      bool ch = false;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (nw[j] > 0.f) ch |= fuse_cell(p, nw[j], cfa[j], &vla[j], vals);
      if (ch) {
        *reinterpret_cast<float4*>(confS + cell0) = make_float4(cfa[0], cfa[1], cfa[2], cfa[3]);
        *reinterpret_cast<float4*>(valS + cell0) = make_float4(vla[0], vla[1], vla[2], vla[3]);
      }
    } else {
      for (int j = 0; j < 4; ++j) {
        if (!(nw[j] > 0.f)) continue;
        size_t cell = cell0 + j;
        float cfv = confS[cell];
        float vbuf[8];
        for (int q = 0; q < C; ++q) vbuf[q] = valS[cell * C + q];
        if (fuse_cell(p, nw[j], cfv, vbuf, vals)) {
          confS[cell] = cfv;
          for (int q = 0; q < C; ++q) valS[cell * C + q] = vbuf[q];
        }
      }
    }
  }
}

// value_map.py:369-375, whole-grid part
__global__ void value_mask_unexplored_kernel(int G, int C, const int* __restrict__ slot,
                                             float* __restrict__ conf, float* __restrict__ value,
                                             const uint8_t* __restrict__ explored) {
  const int b = blockIdx.y;
  const int s = slot ? slot[b] : b;
  const size_t n = (size_t)G * G;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (explored[(size_t)s * n + i] == 0) {
      if (conf[(size_t)s * n + i] != 0.f) conf[(size_t)s * n + i] = 0.f;
      for (int q = 0; q < C; ++q)
        if (value[((size_t)s * n + i) * C + q] != 0.f) value[((size_t)s * n + i) * C + q] = 0.f;
    }
  }
}

// pixel_value_within_radius (img_utils.py:213-266), reduction="median".
// one block per (point, channel); bitonic sort of the <= CAP candidate values (CAP = 1024: radius <= 15 cells, 4096: <= 31).
// np.median averages the two middle values of an even count in the grid's dtype: float64 for the reference's weighted maps
// (grid_f64 = 1), float32 for max-confidence and replace maps, whose value grid stays float32 (grid_f64 = 0).
template <int CAP>
__global__ void __launch_bounds__(256)
value_disc_median_kernel(int G, int C, const float* __restrict__ valueAll, const int* __restrict__ pts, int with_slot,
                         int radius, int grid_f64, const uint8_t* __restrict__ disc, double* __restrict__ out) {
  __shared__ float vals[CAP];
  __shared__ int s_n;
  const int pi = blockIdx.x, ch = blockIdx.y, tid = threadIdx.x;
  // points are (row, col) or, for the batched entry, (slot, row, col): one launch scores the frontiers of every environment
  const int row = with_slot ? pts[3 * pi + 1] : pts[2 * pi], col = with_slot ? pts[3 * pi + 2] : pts[2 * pi + 1];
  const float* valueS = valueAll + (with_slot ? (size_t)pts[3 * pi] * G * G * C : 0);
  if (tid == 0) s_n = 0;
  for (int i = tid; i < CAP; i += 256) vals[i] = INFINITY;
  __syncthreads();
  const int D = 2 * radius + 1;
  const int r0 = max(0, row - radius), c0 = max(0, col - radius);
  const int r1 = min(G, row + radius + 1), c1 = min(G, col + radius + 1);
  const int h = r1 - r0, w = c1 - c0;
  if ((unsigned)row < (unsigned)G && (unsigned)col < (unsigned)G) {
    for (int i = tid; i < h * w; i += 256) {
      int rr = i / w, cc = i % w;
      if (disc[rr * D + cc]) {  // disc centred at (radius, radius) of the clipped crop
        float v = valueS[((size_t)(r0 + rr) * G + (c0 + cc)) * C + ch];
        if (v > 0.f) { int k = atomicAdd(&s_n, 1); if (k < CAP) vals[k] = v; }
      }
    }
  }
  __syncthreads();
  const int n = min(s_n, CAP);
  int P = 2;
  while (P < n) P <<= 1;                      // the unused tail is +inf: sorting the next power of two suffices
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += 256) {
        int ixj = i ^ j;
        if (ixj > i) {
          float a = vals[i], bq = vals[ixj];
          bool up = (i & k) == 0;
          if ((a > bq) == up) { vals[i] = bq; vals[ixj] = a; }
        }
      }
      __syncthreads();
    }
  if (tid == 0) {
    double r;
    if (n == 0) r = -1.0;
    else if (n & 1) r = (double)vals[n / 2];
    else if (grid_f64) r = ((double)vals[n / 2 - 1] + (double)vals[n / 2]) * 0.5;
    else r = (double)__fmul_rn(__fadd_rn(vals[n / 2 - 1], vals[n / 2]), 0.5f);
    out[(size_t)pi * C + ch] = r;
  }
}

}  // namespace vlfm

using namespace vlfm;

extern "C" int vlfm_value_workspace_bytes(const VlfmValueParams* p, int batch, size_t* bytes) {
  if (!p || !bytes || batch < 0) { set_error("vlfm_value_workspace_bytes: bad argument"); return VLFM_E_INVALID; }
  ValueDev d = make_dev(*p);
  *bytes = (size_t)d.wsWords * 4 * (size_t)batch;
  return VLFM_OK;
}

static size_t k1_smem(const ValueDev& d) {
  size_t E = d.W + 2;
  size_t words = 2 * ((E + 1) & ~(size_t)1) + 2 * (size_t)d.R * d.WPR + E;
  size_t b = words * 4;
  return b < 8 * K1_COLS * 4 ? 8 * K1_COLS * 4 : b;
}

extern "C" int vlfm_value_update(const VlfmValueParams* p, int batch, const int32_t* d_slot,
                                 float* d_conf, float* d_value, const float* d_depth,
                                 const double* d_tf, const double* d_values, const float* d_template,
                                 const double* d_tan, const uint8_t* d_explored, void* d_workspace,
                                 int32_t* d_status, void* stream) {
  if (!p || !d_conf || !d_value || !d_depth || !d_tf || !d_values || !d_template || !d_tan ||
      !d_workspace || !d_status) { set_error("vlfm_value_update: null argument"); return VLFM_E_INVALID; }
  if (batch <= 0) return VLFM_OK;
  if (p->C < 1 || p->C > 8 || p->R < 3 || (p->R & 1) == 0 || p->H < 1 || p->W < 1 || p->G < 1 ||
      batch > 65535) { set_error("vlfm_value_update: unsupported shape (C in 1..8, odd R, batch<=65535)"); return VLFM_E_INVALID; }
  ValueDev d = make_dev(*p);
  cudaStream_t st = (cudaStream_t)stream;
  size_t sm1 = k1_smem(d);
  size_t sm2 = (size_t)(4 * d.R + d.R * d.WPR) * 4;
  if (sm1 > 200 * 1024 || sm2 > 200 * 1024) { set_error("vlfm_value_update: template too large for shared memory"); return VLFM_E_UNSUPPORTED; }
  static size_t cfg1 = 0, cfg2 = 0;
  if (sm1 > 48 * 1024 && sm1 > cfg1) {
    int rc = check_cuda(cudaFuncSetAttribute(value_geom_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm1), "cudaFuncSetAttribute(K1b)");
    if (rc) return rc; cfg1 = sm1;
  }
  if (sm2 > 48 * 1024 && sm2 > cfg2) {
    int rc = check_cuda(cudaFuncSetAttribute(value_cone_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2), "cudaFuncSetAttribute(K2)");
    if (rc) return rc; cfg2 = sm2;
  }
  dim3 g1(d.nColTiles, d.nChunks, batch);
  value_depth_geom_kernel<<<g1, K1_THREADS, 8 * K1_COLS * 4, st>>>(d, d_depth, d_tf, d_tan, (uint32_t*)d_workspace, d_slot, d_status);
  VLFM_CHECK_LAUNCH("value_depth_geom_kernel");
  {
    int rc = check_cuda(launch_pdl(value_geom_kernel, dim3(batch), dim3(GEOM_THREADS), sm1, st, d, d_tan, (uint32_t*)d_workspace), "value_geom_kernel");
    if (rc) return rc;
  }
  int rpt = p->rows_per_tile;
  if (rpt <= 0) {
    // aim for >= ~2 waves of 132 SMs while keeping the per-block blob load amortised
    int tiles = (264 + batch - 1) / batch;
    if (tiles < 1) tiles = 1;
    if (tiles > d.R) tiles = d.R;
    rpt = (d.R + tiles - 1) / tiles;
    if (rpt < 4) rpt = 4;
  }
  dim3 g2((d.R + rpt - 1) / rpt, batch);
  {
    int rc = check_cuda(launch_pdl(value_cone_fuse_kernel, g2, dim3(K2_THREADS), sm2, st, d, d_slot, d_conf, d_value, d_values, d_template,
                                   d_explored, (const uint32_t*)d_workspace, rpt), "value_cone_fuse_kernel");
    if (rc) return rc;
  }
  count_launch(3);
  return VLFM_OK;
}

extern "C" int vlfm_value_mask_unexplored(int G, int C, int batch, const int32_t* d_slot, float* d_conf,
                                          float* d_value, const uint8_t* d_explored, void* stream) {
  if (!d_conf || !d_value || !d_explored || G < 1 || C < 1) { set_error("vlfm_value_mask_unexplored: bad argument"); return VLFM_E_INVALID; }
  if (batch <= 0) return VLFM_OK;
  dim3 g(264, batch);
  value_mask_unexplored_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(G, C, d_slot, d_conf, d_value, d_explored);
  VLFM_CHECK_LAUNCH("value_mask_unexplored_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_value_disc_median(int G, int C, int slot, const float* d_value, const int32_t* d_points,
                                      int npoints, int radius, int grid_f64, const uint8_t* d_disc, double* d_out,
                                      void* stream) {
  if (!d_value || !d_points || !d_disc || !d_out || radius < 0 || radius > 31 || C < 1) {
    set_error("vlfm_value_disc_median: bad argument (radius must be <= 31 cells)"); return VLFM_E_INVALID; }
  if (npoints <= 0) return VLFM_OK;
  dim3 g(npoints, C);
  if (radius <= 15)
    value_disc_median_kernel<1024><<<g, 256, 0, (cudaStream_t)stream>>>(G, C, d_value + (size_t)slot * G * G * C,
                                                                       d_points, 0, radius, grid_f64, d_disc, d_out);
  else
    value_disc_median_kernel<4096><<<g, 256, 0, (cudaStream_t)stream>>>(G, C, d_value + (size_t)slot * G * G * C,
                                                                       d_points, 0, radius, grid_f64, d_disc, d_out);
  VLFM_CHECK_LAUNCH("value_disc_median_kernel");
  count_launch();
  return VLFM_OK;
}

extern "C" int vlfm_value_disc_median_batch(int G, int C, const float* d_value, const int32_t* d_points_srl, int npoints, int radius,
                                            int grid_f64, const uint8_t* d_disc, double* d_out, void* stream) {
  if (!d_value || !d_points_srl || !d_disc || !d_out || radius < 0 || radius > 31 || C < 1) {
    set_error("vlfm_value_disc_median_batch: bad argument (radius must be <= 31 cells)"); return VLFM_E_INVALID; }
  if (npoints <= 0) return VLFM_OK;
  dim3 g(npoints, C);
  if (radius <= 15) value_disc_median_kernel<1024><<<g, 256, 0, (cudaStream_t)stream>>>(G, C, d_value, d_points_srl, 1, radius, grid_f64, d_disc, d_out);
  else value_disc_median_kernel<4096><<<g, 256, 0, (cudaStream_t)stream>>>(G, C, d_value, d_points_srl, 1, radius, grid_f64, d_disc, d_out);
  VLFM_CHECK_LAUNCH("value_disc_median_kernel");
  count_launch();
  return VLFM_OK;
}
