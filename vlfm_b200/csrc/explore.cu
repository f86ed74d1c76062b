// Explore half of the obstacle map on the GPU (sm_90a): fog-of-war, explored-area component selection,
// frontier waypoints -- for a BATCH of environments per call.
//
// Reference: vlfm/mapping/obstacle_map.py:114-169 and the two `frontier_exploration` functions it calls
// (reveal_fog_of_war, detect_frontier_waypoints; third-party, absent from the reference tree).  The SPEC these
// kernels follow step by step is oracle/explore_oracle.py (numpy backend) with oracle/contours.py,
// oracle/cv_draw.py and oracle/cv_prims.py -- restatements of the OpenCV primitives pinned against cv2.
//
// Batching: every kernel runs with gridDim.y = environments of the call and reads its environment's record (ExEnv: image
// pointers, frame geometry, pose scalars) from device memory; one call = one launch SEQUENCE for all environments.
//
// Frames.  The fog-of-war runs in a (2L+9)^2 WINDOW around the agent (L = max_depth*ppm), which may hang over the grid edge
// (cv2's clipping rules are reproduced; cells outside the grid are masked).  Component selection and the frontier search --
// full-grid operations in the reference -- run in the S-FRAME: a grid rectangle that contains every cell the explore / obstacle
// updates of this episode have touched plus a margin; outside it explored == 0 and navigable == 1, which makes the restriction
// exact (DESIGN.md section 3.2b): label arrays and masks cover the S-frame, not G^2 cells.
//
// Building blocks
//   ccl_*            label-equivalence connected components (union-find, atomicMin): 8-connected foreground
//                    and 4-connected background; root = raster-first pixel of the component.
//   collect_roots    cv2.findContours(RETR_EXTERNAL): outer borders of the components whose west background
//                    region is the outer background, in REVERSE raster order of their first pixels.
//   trace_kernel     Suzuki-Abe border following (one thread per contour), CHAIN_APPROX_NONE
//                    chain + bounding box; CHAIN_APPROX_SIMPLE vertices = direction changes of the chain.
//   chain_edges      cv2.drawContours(..., -1) of a traced chain: outline + even-odd scan conversion as XOR toggles
//                    + per-row prefix XOR (every chain edge is a unit step, so intercepts are exact).
//   sector_edges     cv2.ellipse filled sector: 16.16 polygon from the host (integer-degree ellipse2Poly), same
//                    scan conversion with fractional columns, PolyEdges from clipped end points at the grid edge.
//   rays / thick     occlusion rays: cv2.polylines thickness 2 = FillConvexPoly rectangle (Line2 outline + two-edge
//                    scan) + radius-1 discs, clipped like cv2 (grid + 2 px for the centre line, grid for Line2);
//                    the rasteriser is csrc/cv_raster.cuh, shared with the map frames (csrc/render.cu).
//   frontier_kernel  contour split at cells whose 3x3 blurred unexplored mask is 0, arc-length midpoints.
#include <math.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "cv_raster.cuh"

namespace vlfm {

constexpr int EX_MAXC = 8192;      // contours per image (explore); fill_small_holes uses HOLES_MAXC
constexpr int XYS = 16;
constexpr long long XYONE = 1ll << XYS;
constexpr int MAXV = 64;           // sector polygon vertices

struct Contour { int start, off, len, x0, y0, x1, y1, ed; };   // start pixel, chain offset/length, bbox, entry direction (0 = west: outer border, 4 = east: hole border)

// device-side bookkeeping of one explore step
struct ExState {
  int n_cont;          // contours of the image being processed
  int cursor;          // chain buffer cursor
  int n_rays;
  int skip_fog;        // reveal_fog_of_war returned the (empty) input mask
  int chosen;          // selected contour index
  int n_front;
  int overflow;
  int pad;
};

enum { IMG_BLOCKED = 0, IMG_VISIBLE = 1, IMG_EXS = 2, IMG_UNEXP = 3, IMG_EX2 = 4 };
enum { FRAME_WIN = 0, FRAME_S = 1 };

// one environment of a call (device memory)
struct ExEnv {
  uint8_t *cone, *blocked, *visible, *cut, *newexp;     // window frame [W0 * W0]
  uint8_t *exS, *navS, *grown, *unexp, *ex2;            // S frame [Sw * Sh]
  uint8_t *outer, *hashole, *nbm, *flags;               // per-label flags / 8-neighbour masks of the image being processed; bad flags per chain point
  int *Lfg, *Lbg, *which, *nsv;
  Contour* cont; int2 *chain, *sv; int4* rays; double* dist; uint32_t *tog, *orb; ExState* st;
  uint8_t* explored; const uint8_t* nav;                // this environment's [G, G] grids
  double* frontiers; int* out_count; int* out_status;
  const float* depth; uint8_t* filled;                  // fill_small_holes: depth image in, byte mask out
  int G, maxc, chain_cap, rays_cap, maxf;
  int ox, oy, W0, sx, sy;                               // window origin (grid coordinates), side, agent in window coordinates
  int fx0, fy0, Sw, Sh;                                 // S frame origin (grid coordinates) and size
  int ax, ay;                                           // agent cell (col, row), grid coordinates
  int ext_l, ext_t, ext_r, ext_b;                       // that edge of the S frame is NOT a grid edge: the exterior continues beyond it
  int nv, pad0;
  double heading_deg, ray_len, area_thresh;
  long long verts[2 * MAXV];
};

struct View { uint8_t* p; int W, H; };
__device__ __forceinline__ View view(const ExEnv& E, int id) {
  View v;
  switch (id) {
    case IMG_BLOCKED: v.p = E.blocked; v.W = E.W0; v.H = E.W0; break;
    case IMG_VISIBLE: v.p = E.visible; v.W = E.W0; v.H = E.W0; break;
    case IMG_EXS: v.p = E.exS; v.W = E.Sw; v.H = E.Sh; break;
    case IMG_UNEXP: v.p = E.unexp; v.W = E.Sw; v.H = E.Sh; break;
    default: v.p = E.ex2; v.W = E.Sw; v.H = E.Sh; break;
  }
  return v;
}

// ------------------------------------------------------------------------------------------- CCL ----
__device__ __forceinline__ int uf_find(int* L, int i) {
  while (true) {
    int p = *reinterpret_cast<volatile int*>(&L[i]);
    if (p == i) return i;
    i = p;
  }
}
__device__ __forceinline__ void uf_union(int* L, int a, int b) {
  while (true) {
    a = uf_find(L, a); b = uf_find(L, b);
    if (a == b) return;
    if (a < b) { int t = a; a = b; b = t; }
    int old = atomicMin(&L[a], b);
    if (old == a) return;
    a = old;
  }
}


// init: every pixel points at the first pixel of its horizontal run, for the foreground (8-connected) and the background
// (4-connected) label arrays at once, so that the union phase only has to stitch runs of adjacent rows.  One warp per
// row, 32 cells per ballot.  Block 0 also resets the per-image bookkeeping.
__global__ void __launch_bounds__(256)
ccl_init2_kernel(const ExEnv* __restrict__ envs, int img, int keep_fog) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, img);
  ExState* st = E.st;
  int* Lfg = E.Lfg; int* Lbg = E.Lbg;
  const int W = v.W, H = v.H;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->n_cont = 0; st->cursor = 0; st->n_rays = 0; st->chosen = -1;
    if (!keep_fog) { st->skip_fog = 0; st->overflow = 0; st->n_front = 0; }
  }
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int y = blockIdx.x * wpb + (threadIdx.x >> 5); y < H; y += gridDim.x * wpb) {
    const uint8_t* row = v.p + (size_t)y * W;
    const int base = y * W;
    int carry_fg = -1, carry_bg = -1;                 // column where a run that reaches the chunk boundary started
    const unsigned below = (1u << lane) - 1;
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane;
      const bool valid = x < W;
      const bool fg = valid && row[x] != 0;
      const unsigned m = __ballot_sync(0xffffffffu, fg);
      const unsigned zf = ~m & below, zb = m & below;  // cells below this lane that end a fg / bg run
      const int sf = zf ? x0 + 32 - __clz(zf) : (carry_fg >= 0 ? carry_fg : x0);
      const int sb = zb ? x0 + 32 - __clz(zb) : (carry_bg >= 0 ? carry_bg : x0);
      if (valid) { Lfg[base + x] = fg ? base + sf : -1; Lbg[base + x] = fg ? -1 : base + sb; }
      const int sf31 = __shfl_sync(0xffffffffu, sf, 31), sb31 = __shfl_sync(0xffffffffu, sb, 31);
      carry_fg = (m >> 31) ? sf31 : -1;
      carry_bg = (m >> 31) ? -1 : sb31;
    }
  }
}
// stitch: a pixel unions with the row above only where a NEW overlap between runs begins; also clears the per-label flags
__global__ void ccl_merge2_kernel(const ExEnv* __restrict__ envs, int id, int want_hashole) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  const uint8_t* __restrict__ img = v.p;
  int* Lfg = E.Lfg; int* Lbg = E.Lbg;
  uint8_t* outer = E.outer; uint8_t* hashole = want_hashole ? E.hashole : nullptr; uint8_t* nbm = E.nbm;
  const int W = v.W, H = v.H, n = W * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    outer[i] = 0;
    if (hashole) hashole[i] = 0;
    const int y = i / W, x = i - y * W;
    const bool c = img[i] != 0;
    if (c) {   // 8-neighbourhood mask for the border tracer, bit d = neighbour in direction d (clockwise from west)
      const bool l = x > 0, r = x + 1 < W, u = y > 0, d = y + 1 < H;
      unsigned m = 0;
      if (l && img[i - 1]) m |= 1u;
      if (l && u && img[i - W - 1]) m |= 2u;
      if (u && img[i - W]) m |= 4u;
      if (r && u && img[i - W + 1]) m |= 8u;
      if (r && img[i + 1]) m |= 16u;
      if (r && d && img[i + W + 1]) m |= 32u;
      if (d && img[i + W]) m |= 64u;
      if (l && d && img[i + W - 1]) m |= 128u;
      nbm[i] = (uint8_t)m;
    }
    if (y == 0) continue;
    const bool west = x > 0 && ((img[i - 1] != 0) == c);
    const bool north = (img[i - W] != 0) == c;
    const bool nwest = x > 0 && ((img[i - W - 1] != 0) == c);
    int* L = c ? Lfg : Lbg;
    if (north && (!west || !nwest)) uf_union(L, i, i - W);
    if (c) {   // foreground is 8-connected: diagonal contacts not already implied by a north contact
      const bool neast = x + 1 < W && img[i - W + 1] != 0;
      if (nwest && !north && !west) uf_union(L, i, i - W - 1);
      if (neast && !north) uf_union(L, i, i - W + 1);
    }
  }
}
// Every cell of a horizontal run still points at the run's first cell (only roots are ever re-linked), so the cells of a run
// would all walk the same parent chain: the lanes of a warp that share a parent elect one walker (__match_any_sync) and take its
// answer.  32 consecutive cells are usually one or two runs -- the walks drop by an order of magnitude.
__global__ void ccl_flatten2_kernel(const ExEnv* __restrict__ envs, int id) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  int* Lfg = E.Lfg; int* Lbg = E.Lbg;
  const int n = v.W * v.H;
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.x * blockDim.x;
  for (int i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31); i0 < n; i0 += stride) {      // warp-uniform trip count
    const int i = i0 + lane;
    const bool in = i < n;
    int lf = -1, parent = -1;
    if (in) { lf = Lfg[i]; parent = lf >= 0 ? lf : Lbg[i]; }
    const bool fg = lf >= 0;
    // key: parent cell, foreground / background arrays apart; lanes past the end get private keys
    const int key = in ? (fg ? parent : parent + n) : -1 - lane;
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int leader = __ffs(peers) - 1;
    int root = 0;
    if (in && lane == leader) root = uf_find(fg ? Lfg : Lbg, parent);
    root = __shfl_sync(0xffffffffu, root, leader);
    if (in) { if (fg) Lfg[i] = root; else Lbg[i] = root; }
  }
}
// background components touching the image frame are the "outer" background (the frame is background for Suzuki).
// mark_exterior: foreground components touching an S-frame edge that is not a grid edge continue outside the frame -- they are
// (part of) the unexplored exterior, whose contourArea is far above any absorb threshold: flagged like hole-enclosing components.
__global__ void bg_outer_kernel(const ExEnv* __restrict__ envs, int id, int mark_exterior) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  const int W = v.W, H = v.H;
  const int per = 2 * (W + H);
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < per; t += gridDim.x * blockDim.x) {
    int x, y, ext;
    if (t < W) { x = t; y = 0; ext = E.ext_t; } else if (t < 2 * W) { x = t - W; y = H - 1; ext = E.ext_b; }
    else if (t < 2 * W + H) { x = 0; y = t - 2 * W; ext = E.ext_l; } else { x = W - 1; y = t - 2 * W - H; ext = E.ext_r; }
    const int l = E.Lbg[y * W + x];
    if (l >= 0) E.outer[l] = 1;
    else if (mark_exterior && ext) E.hashole[E.Lfg[y * W + x]] = 1;
  }
}
__global__ void collect_roots_kernel(const ExEnv* __restrict__ envs, int id) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  const int* __restrict__ Lfg = E.Lfg; const int* __restrict__ Lbg = E.Lbg; const uint8_t* __restrict__ outer = E.outer;
  const int W = v.W, n = v.W * v.H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (Lfg[i] != i) continue;                      // roots only (= raster-first pixel of the component)
    const int y = i / W, x = i - y * W;
    bool top = true;
    if (x > 0) { const int lb = Lbg[i - 1]; top = lb >= 0 && outer[lb]; }
    if (!top) continue;                             // nested inside a hole of another component: not external
    const int k = atomicAdd(&E.st->n_cont, 1);
    if (k < EX_MAXC) { E.cont[k].start = i; E.cont[k].ed = 0; } else E.st->overflow = 1;
  }
}
// a foreground component that directly encloses a background region (a hole): flag its root
__global__ void mark_holes_kernel(const ExEnv* __restrict__ envs, int id) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  const int W = v.W, n = v.W * v.H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (E.Lbg[i] != i || E.outer[i]) continue;        // raster-first pixel of an enclosed background region
    const int x = i % W;
    if (x > 0 && E.Lfg[i - 1] >= 0) E.hashole[E.Lfg[i - 1]] = 1;
  }
}
// reverse raster order (cv2 returns the last-found contour first); one block per environment, bitonic sort in shared memory
__global__ void __launch_bounds__(1024) sort_roots_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  Contour* cont = E.cont; ExState* st = E.st;
  __shared__ int keys[EX_MAXC];
  int n = st->n_cont;
  if (n > EX_MAXC) n = EX_MAXC;
  __syncthreads();
  if (threadIdx.x == 0) st->n_cont = n;
  int P = 2;
  while (P < n) P <<= 1;                              // bitonic network over the next power of two only
  for (int i = threadIdx.x; i < P; i += 1024) keys[i] = i < n ? cont[i].start : -1;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += 1024) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const int a = keys[i], b = keys[ixj];
          const bool desc = (i & k) == 0;           // descending overall
          if ((a < b) == desc) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < n; i += 1024) { cont[i].start = keys[i]; cont[i].ed = 0; }
}

// ----------------------------------------------------------------------------------------- tracing ----
// directions 0..7: clockwise from west (image coordinates, y down): dx = {-1,-1,0,1,1,1,0,-1}, dy = {0,-1,-1,-1,0,1,1,1}

// direction tables packed into registers (a dynamically indexed __constant__ array costs a dependent LDC per probe)
__device__ __forceinline__ int dir_dx(int d) { return (int)((0x01222100u >> (d * 4)) & 0xFu) - 1; }
__device__ __forceinline__ int dir_dy(int d) { return (int)((0x22210001u >> (d * 4)) & 0xFu) - 1; }
__device__ __forceinline__ unsigned rotr8(unsigned v, int r) { return ((v >> r) | (v << (8 - r))) & 0xFFu; }
// Suzuki-Abe steps 3.1-3.5 (oracle/contours.py::_trace) on the per-pixel neighbour masks written by ccl_merge2_kernel: one
// byte load per step; the clockwise / counter-clockwise probe loops are a byte rotation + ffs / clz.  WRITE=false only counts.
// Writes the first `cap` points to out (when non-null) and always returns the full length and the bounding box.
__device__ int trace_border(const uint8_t* __restrict__ nbm, int W, int x0, int y0, int2* out, int cap, Contour* c, int ed = 0) {
  int n = 0, minx = x0, maxx = x0, miny = y0, maxy = y0;
  // 3.1 clockwise from the (zero) entry pixel (west for outer, east for hole borders): first set bit among ed+1 .. ed+7
  const unsigned r0 = rotr8(nbm[y0 * W + x0], ed) & 0xFEu;
  if (!r0) {
    if (out && cap > 0) out[0] = make_int2(x0, y0);
    n = 1;
  } else {
    const int df = (ed + __ffs(r0) - 1) & 7;
    const int fx = x0 + dir_dx(df), fy = y0 + dir_dy(df);
    int x3 = x0, y3 = y0, d0 = df;                   // d0: direction from (x3,y3) to the previously examined pixel (x2,y2)
    while (true) {
      // 3.3 counter-clockwise, starting after (x2,y2): probes d0-1, ..., d0-8 are bits 7..0 after rotating right by d0, so the
      // first hit is the highest set bit (bit 0 = (x2,y2) itself is always set)
      const unsigned r = rotr8(nbm[y3 * W + x3], d0);
      const int di = (d0 + (31 - __clz(r))) & 7;
      const int x4 = x3 + dir_dx(di), y4 = y3 + dir_dy(di);
      if (out && n < cap) out[n] = make_int2(x3, y3);
      minx = min(minx, x3); maxx = max(maxx, x3); miny = min(miny, y3); maxy = max(maxy, y3);
      ++n;
      if (x4 == x0 && y4 == y0 && x3 == fx && y3 == fy) break;   // 3.5
      x3 = x4; y3 = y4; d0 = (di + 4) & 7;          // seen from the new pixel, the old one lies in the opposite direction
      if (n > (1 << 22)) break;                      // safety
    }
  }
  c->x0 = minx; c->x1 = maxx; c->y0 = miny; c->y1 = maxy;
  return n;
}

// mode 0: trace every contour; 1: only when more than one contour exists (component selection); 2: skip components
// flagged in hashole (they enclose a hole -- their filled polygon contains a zero cell -- or reach the exterior: F1 can never
// absorb them).
// Chain storage: the first half of the chain buffer is cut into one equal slot per contour, which the walk fills directly -- ONE
// pass in the common case; a border longer than its slot (many contours and a long one among them) is walked a second time into
// space taken from the second half with the cursor.  (Round 1 always walked twice: count, allocate, write.)
__global__ void trace_kernel(const ExEnv* __restrict__ envs, int id, int mode) {
  const ExEnv& E = envs[blockIdx.y];
  const View v = view(E, id);
  ExState* st = E.st;
  const int W = v.W;
  const int nc = min(st->n_cont, E.maxc);
  const int half = E.chain_cap >> 1;
  const int slot = nc > 0 ? half / nc : 0;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += gridDim.x * blockDim.x) {
    const int s = E.cont[c].start, y0 = s / W, x0 = s - y0 * W;
    if ((mode == 1 && st->n_cont <= 1) || (mode == 2 && E.hashole[s])) { E.cont[c].off = 0; E.cont[c].len = 0; continue; }
    const int n = trace_border(E.nbm, W, x0, y0, E.chain + (size_t)c * slot, slot, &E.cont[c], E.cont[c].ed);
    if (n <= slot) { E.cont[c].off = c * slot; E.cont[c].len = n; continue; }
    const int off = half + atomicAdd(&st->cursor, n);
    if (off + n > E.chain_cap) { st->overflow = 1; E.cont[c].off = 0; E.cont[c].len = 0; continue; }
    E.cont[c].off = off; E.cont[c].len = n;
    trace_border(E.nbm, W, x0, y0, E.chain + off, n, &E.cont[c], E.cont[c].ed);
  }
}

// CHAIN_APPROX_SIMPLE: point i of a chain is kept iff the step into it differs from the step out of it
__device__ __forceinline__ bool simple_vertex(const int2* p, int n, int i) {
  if (n <= 2) return true;
  const int2 a = p[i == 0 ? n - 1 : i - 1], b = p[i], c = p[i + 1 == n ? 0 : i + 1];
  return (b.x - a.x != c.x - b.x) || (b.y - a.y != c.y - b.y);
}

// cv2.pointPolygonTest(cnt, pt, True) on the SIMPLE vertices (oracle/contours.py::point_polygon_distance): float32 vertices, double
// arithmetic, first strictly smaller squared distance wins, crossing parity gives the sign.  One WARP per contour: lane L scans the L-th contiguous chunk of the chain with the sequential rule (first
// strictly smaller squared distance wins), the 32 chunk results are then combined in chunk order with the same comparison, the
// crossing counts add up.  A vertex ON the point (distance 0) ends the sequential scan with +-0: any lane finding one decides.
__device__ double ppt_distance_warp(const int2* p, int n, int ptx, int pty, int lane) {
  if (n == 0) return -1.7976931348623157e308;
  const float px = (float)ptx, py = (float)pty;
  const int chunk = (n + 31) >> 5;
  const int c0 = min(n, lane * chunk), c1 = min(n, c0 + chunk);
  double min_num = 3.4028234663852886e38, min_den = 1.0;
  int counter = 0, zero = 0;
  if (c0 < c1) {
    int last = -1;                                     // the simple vertex preceding this chunk (cyclically)
    for (int k = 1; k <= n; ++k) { const int i = c0 - k < 0 ? c0 - k + n : c0 - k; if (simple_vertex(p, n, i)) { last = i; break; } }
    if (last < 0) last = n - 1;
    float vx = (float)p[last].x, vy = (float)p[last].y;
    for (int i = c0; i < c1; ++i) {
      if (!simple_vertex(p, n, i)) continue;
      const float v0x = vx, v0y = vy;
      vx = (float)p[i].x; vy = (float)p[i].y;
      const double dx = vx - v0x, dy = vy - v0y, dx1 = px - v0x, dy1 = py - v0y, dx2 = px - vx, dy2 = py - vy;
      double num, den = 1.0;
      if (dx1 * dx + dy1 * dy <= 0) num = dx1 * dx1 + dy1 * dy1;
      else if (dx2 * dx + dy2 * dy >= 0) num = dx2 * dx2 + dy2 * dy2;
      else { num = dy1 * dx - dx1 * dy; num *= num; den = dx * dx + dy * dy; }
      if (num * min_den < min_num * den) { min_num = num; min_den = den; if (min_num == 0) { zero = 1; break; } }
      if ((v0y <= py && vy <= py) || (v0y > py && vy > py)) continue;
      double cr = dy1 * dx - dx1 * dy;
      if (dy < 0) cr = -cr;
      counter += cr > 0;
    }
  }
  if (__any_sync(0xffffffffu, zero)) return 0.0;
#pragma unroll
  for (int o = 16; o; o >>= 1) counter += __shfl_xor_sync(0xffffffffu, counter, o);
  double bn = __shfl_sync(0xffffffffu, min_num, 0), bd = __shfl_sync(0xffffffffu, min_den, 0);
  for (int l = 1; l < 32; ++l) {                        // chunk order, the sequential comparison
    const double num = __shfl_sync(0xffffffffu, min_num, l), den = __shfl_sync(0xffffffffu, min_den, l);
    if (num * bd < bn * den) { bn = num; bd = den; }
  }
  const double r = sqrt(bn / bd);
  return (counter & 1) ? r : -r;
}


// ------------------------------------------------------------------------------ scan conversion ----
// planes: tog / orb, `pw` 32-bit words per row of the frame
__device__ __forceinline__ void frame_dims(const ExEnv& E, int frame, int& W, int& H) {
  if (frame == FRAME_WIN) { W = E.W0; H = E.W0; } else { W = E.Sw; H = E.Sh; }
}
__global__ void zero_planes_kernel(const ExEnv* __restrict__ envs, int frame) {
  const ExEnv& E = envs[blockIdx.y];
  int W, H; frame_dims(E, frame, W, H);
  const int words = ((W + 31) / 32) * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) { E.tog[i] = 0; E.orb[i] = 0; }
}
// chain polygon: every edge is a unit step; outline = the chain points.  Contour index = *E.which.
__global__ void chain_edges_kernel(const ExEnv* __restrict__ envs, int frame) {
  const ExEnv& E = envs[blockIdx.y];
  int W, H; frame_dims(E, frame, W, H);
  const int pw = (W + 31) / 32;
  const int ci = *E.which;
  if (ci < 0 || ci >= E.st->n_cont) return;
  const Contour c = E.cont[ci];
  const int2* p = E.chain + c.off;
  uint32_t* tog = E.tog; uint32_t* orb = E.orb;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < c.len; i += gridDim.x * blockDim.x) {
    const int2 a = p[i], b = p[i + 1 == c.len ? 0 : i + 1];
    atomicOr(&orb[a.y * pw + (a.x >> 5)], 1u << (a.x & 31));
    if (a.y != b.y) {
      const int xa = a.y < b.y ? a.x : b.x, ya = min(a.y, b.y);     // active on row ya only; intercept exactly xa
      const int t = xa + 1;
      if (t < W) atomicXor(&tog[ya * pw + (t >> 5)], 1u << (t & 31));
      atomicOr(&orb[ya * pw + (xa >> 5)], 1u << (xa & 31));
    }
  }
}
// rows -> image: img[cell] = value where filled; optionally everything else := 0 (clear_rest).  One WARP per row: lane = 32-bit
// word of the toggle plane (rows wider than 1024 cells take several passes); the even-odd state entering a word is the XOR of
// the parities of the words before it (warp scan), the 32 cells of a word are written by its lane.
__device__ __forceinline__ void planes_row_to_image(const uint32_t* __restrict__ tog, const uint32_t* __restrict__ orb, uint8_t* __restrict__ img,
                                                    int W, int pw, int r, int value, int clear_rest, int lane) {
  uint32_t carry = 0;                                   // 0 or ~0: fill state entering this pass
  for (int w0 = 0; w0 < pw; w0 += 32) {
    const int w = w0 + lane;
    const uint32_t t = w < pw ? tog[r * pw + w] : 0u;
    uint32_t x = t;
    x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
    uint32_t par = __popc(t) & 1u;                      // parity of this word, then exclusive XOR-scan over the lanes
    uint32_t inc = par;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc ^= u; }
    const uint32_t before = inc ^ par;                  // XOR of the parities of the lower lanes
    x ^= (before ? ~0u : 0u) ^ carry;
    const uint32_t tot = __shfl_sync(0xffffffffu, inc, 31);
    if (w < pw) {
      const uint32_t f = x | orb[r * pw + w];
      uint8_t* o = img + (size_t)r * W + w * 32;
      const int nb = min(32, W - w * 32);
      for (int bq = 0; bq < nb; ++bq) {
        if ((f >> bq) & 1u) o[bq] = (uint8_t)value;
        else if (clear_rest) o[bq] = 0;
      }
    }
    if (tot) carry = ~carry;
  }
}
// dst: 0 = cone (window), 1 = newexp (window), 2 = exS (S frame); gated by *E.which >= 0 when `gated`
__global__ void planes_to_image_kernel(const ExEnv* __restrict__ envs, int dst, int clear_rest, int gated) {
  const ExEnv& E = envs[blockIdx.y];
  if (gated && *E.which < 0) return;
  int W, H; frame_dims(E, dst == 2 ? FRAME_S : FRAME_WIN, W, H);
  uint8_t* img = dst == 0 ? E.cone : (dst == 1 ? E.newexp : E.exS);
  const int pw = (W + 31) / 32;
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < H; r += nw) planes_row_to_image(E.tog, E.orb, img, W, pw, r, 1, clear_rest, lane);
}
__global__ void planes_to_image_plain_kernel(const uint32_t* __restrict__ tog, const uint32_t* __restrict__ orb, uint8_t* __restrict__ img, int W, int H, int pw) {
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < H; r += nw) planes_row_to_image(tog, orb, img, W, pw, r, 1, 1, lane);
}
__global__ void zero_planes_plain_kernel(uint32_t* tog, uint32_t* orb, int words) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) { tog[i] = 0; orb[i] = 0; }
}

using cvr::clip_line;   // cv::clipLine (csrc/cv_raster.cuh)

// cv2.ellipse filled sector: polygon (x, y in 16.16, last vertex = centre) from the host; CollectPolyEdges +
// FillEdgeCollection (oracle/cv_draw.py::fill_poly_fixed / poly_edge).  One block; the image is the GW x GH grid, of which the
// W x H window at (ox, oy) is rasterised (the window may hang over the grid edge: those cells are masked by the caller).
// 8-connected line between two pixels of the grid (already clipped), plotted into the window's outline plane
__device__ __forceinline__ void plot_line8(uint32_t* orb, int pw, int W, int H, int ox, int oy, int ax, int ay, int bx, int by) {
  if (bx < ax) { int t = ax; ax = bx; bx = t; t = ay; ay = by; by = t; }
  const int dx = bx - ax, dy = by - ay, sy = dy >= 0 ? 1 : -1, ady = dy >= 0 ? dy : -dy;
  const bool ymaj = ady > dx;
  const int major = ymaj ? ady : dx, minor = ymaj ? dx : ady;
  int x = ax - ox, y = ay - oy, err = major - 2 * minor;
  for (int k = 0; k <= major; ++k) {
    if ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) atomicOr(&orb[y * pw + (x >> 5)], 1u << (x & 31));
    const bool m = err < 0;
    err += -2 * minor + (m ? 2 * major : 0);
    if (ymaj) { y += sy; x += m ? 1 : 0; } else { x += 1; y += m ? sy : 0; }
  }
}

__device__ void sector_edges(const long long* __restrict__ v, int nv, int ox, int oy, int GW, int GH, uint32_t* tog, uint32_t* orb,
                             int W, int H, int pw) {
  for (int e = threadIdx.x; e < nv; e += blockDim.x) {
    const int e0 = e == 0 ? nv - 1 : e - 1;
    const long long x0 = v[2 * e0], x1 = v[2 * e];                                                 // 16.16 columns
    const long long y0 = (v[2 * e0 + 1] + (XYONE >> 1)) >> XYS, y1 = (v[2 * e + 1] + (XYONE >> 1)) >> XYS;   // rounded rows
    long long ax = (x0 + (XYONE >> 1)) >> XYS, ay = y0, bx = (x1 + (XYONE >> 1)) >> XYS, by = y1;        // pixel end points
    const bool outside = (unsigned long long)ax >= (unsigned long long)GW || (unsigned long long)bx >= (unsigned long long)GW ||
                         (unsigned long long)ay >= (unsigned long long)GH || (unsigned long long)by >= (unsigned long long)GH;
    long long cx0 = x0, cy0 = y0, cx1 = x1, cy1 = y1;
    bool vis = true;
    if (outside) {
      vis = clip_line(GW, GH, ax, ay, bx, by);
      // PolyEdge from the clipped columns (always) and the clipped rows (when they differ)
      cx0 = ax << XYS; cx1 = bx << XYS;
      if (ay != by) { cy0 = ay; cy1 = by; }
    }
    if (vis) plot_line8(orb, pw, W, H, ox, oy, (int)ax, (int)ay, (int)bx, (int)by);
    if (y0 == y1) continue;
    const long long dxe = (cx1 - cx0) / (cy1 - cy0);          // C truncating division
    long long ya, yb, xs;
    if (y0 < y1) { ya = y0; yb = y1; xs = cx0 + (y0 - cy0) * dxe; } else { ya = y1; yb = y0; xs = cx1 + (y1 - cy1) * dxe; }
    long long r0 = ya > 0 ? ya : 0, r1 = yb < GH ? yb : GH;
    if (r0 < oy) r0 = oy;
    if (r1 > oy + H) r1 = oy + H;
    for (long long r = r0; r < r1; ++r) {
      const long long X = xs + dxe * (r - ya);
      const int wr = (int)(r - oy);
      long long t = (X >> XYS) + 1 - ox;
      if (t < 0) t = 0;
      if (t < W) atomicXor(&tog[wr * pw + (int)(t >> 5)], 1u << ((int)t & 31));
      if ((X & (XYONE - 1)) == 0) { const long long c = (X >> XYS) - ox; if (c >= 0 && c < W) atomicOr(&orb[wr * pw + (int)(c >> 5)], 1u << ((int)c & 31)); }
    }
  }
}
__global__ void sector_edges_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  sector_edges(E.verts, E.nv, E.ox, E.oy, E.G, E.G, E.tog, E.orb, E.W0, E.W0, (E.W0 + 31) / 32);
}
__global__ void sector_edges_plain_kernel(const long long* __restrict__ v, int nv, int R, uint32_t* tog, uint32_t* orb, int pw) {
  sector_edges(v, nv, 0, 0, R, R, tog, orb, R, R, pw);
}

// ValueMap confidence cone (value_map.py:321-355): sector(0/1 byte image) x remap(cos^2(remap(atan2(|dc|,|dr|), 0, fov/2, 0, pi/2)),
// 0, 1, min_conf, 1) in float64 with numpy's operation order, cast to float32.
__global__ void cone_template_kernel(const uint8_t* __restrict__ sector, float* __restrict__ out, int R, double fov, double min_conf) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < R * R; i += gridDim.x * blockDim.x) {
    const int r = i / R, c = i - r * R;
    const double dr = fabs((double)(r - R / 2)), dc = fabs((double)(c - R / 2));
    const double ang = __ddiv_rn(__dmul_rn(atan2(dc, dr), 3.14159265358979323846 / 2), fov / 2);
    const double cs = cos(ang);
    const double conf = __dadd_rn(__dmul_rn(__dmul_rn(cs, cs), 1.0 - min_conf), min_conf);
    out[i] = sector[i] ? (float)conf : 0.f;
  }
}

// --------------------------------------------------------------------------------- window images ----
// blocked = cone & !nav ; visible = cone & nav   (window W0 x W0 at grid origin (ox, oy)); also clears cut and newexp
__global__ void fog_masks_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int W0 = E.W0, G = E.G;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W0 * W0; i += gridDim.x * blockDim.x) {
    const int y = i / W0, x = i - y * W0;
    const int gx = E.ox + x, gy = E.oy + y;
    E.cut[i] = 0; E.newexp[i] = 0;
    if ((unsigned)gx >= (unsigned)G || (unsigned)gy >= (unsigned)G) { E.blocked[i] = 0; E.visible[i] = 0; continue; }   // cv2 clips at the grid edge
    const uint8_t c = E.cone[i], nv = E.nav[(size_t)gy * G + gx];
    E.blocked[i] = c && !nv; E.visible[i] = c && nv;
  }
}

// CHAIN_APPROX_SIMPLE vertex list of every contour, compacted in order (one warp per contour)
__global__ void simple_vertices_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  const int nc = E.st->n_cont;
  for (int ci = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ci < nc; ci += nw) {
    const Contour c = E.cont[ci];
    const int2* p = E.chain + c.off;
    int2* o = E.sv + c.off;
    int cnt = 0;
    for (int b = 0; b < c.len; b += 32) {
      const int i = b + lane;
      const bool keep = i < c.len && simple_vertex(p, c.len, i);
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) o[cnt + __popc(m & ((1u << lane) - 1))] = p[i];
      cnt += __popc(m);
    }
    if (lane == 0) E.nsv[ci] = cnt;
  }
}
// R3/R4: obstacle contours -> ray list (x0,y0,x1,y1 in window coordinates); one warp per contour
__global__ void rays_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  ExState* st = E.st;
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  const int nc = st->n_cont, sx = E.sx, sy = E.sy, ox = E.ox, oy = E.oy, cap = E.rays_cap;
  const double heading_deg = E.heading_deg, ray_len = E.ray_len;
  int4* rays = E.rays;
  for (int ci = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ci < nc; ci += nw) {
    const int2* v = E.sv + E.cont[ci].off;
    const int nv = E.nsv[ci];
    // cv2.isContourConvex on the SIMPLE vertices (oracle/contours.py::is_convex): every turn has the same strict sign
    int orient = 0;
    for (int j = lane; j < nv; j += 32) {
      const int2 a = v[(j + 2 * nv - 2) % nv], b = v[(j + nv - 1) % nv], c = v[j];
      const long long dx0 = b.x - a.x, dy0 = b.y - a.y, dx = c.x - b.x, dy = c.y - b.y;
      const long long dxdy0 = dx * dy0, dydx0 = dy * dx0;
      orient |= dydx0 > dxdy0 ? 1 : (dydx0 < dxdy0 ? 2 : 3);
    }
    orient = __reduce_or_sync(0xffffffffu, orient);
    const bool convex = nv > 0 && orient != 3;
    auto emit = [&](int qx, int qy) {
      const double ang = atan2((double)(qy - sy), (double)(qx - sx));
      // astype(np.int32) truncates toward zero in GRID coordinates (the window origin is subtracted afterwards)
      // numpy evaluates pts + length * cos(ang) as a rounded product and a rounded sum: no fused multiply-add
      const int ex = (int)__dadd_rn((double)(qx + ox), __dmul_rn(ray_len, cos(ang))) - ox, ey = (int)__dadd_rn((double)(qy + oy), __dmul_rn(ray_len, sin(ang))) - oy;
      const int k = atomicAdd(&st->n_rays, 1);
      if (k < cap) rays[k] = make_int4(qx, qy, ex, ey); else st->overflow = 1;
    };
    if (convex) {
      // _extreme_bearing_points: the heading in DEGREES is used as radians, as in the restated package; np.argmin /
      // np.argmax return the FIRST extreme vertex
      const double cs = cos(-heading_deg), sn = sin(-heading_deg);
      double amin = 1e300, amax = -1e300; int imin = 0x7fffffff, imax = 0x7fffffff;
      for (int j = lane; j < nv; j += 32) {
        const double qx = (double)(v[j].x - sx), qy = (double)(v[j].y - sy);
        const double rx = qx * cs + qy * sn, ry = qx * (-sn) + qy * cs;
        const double a = atan2(ry, rx);
        if (a < amin) { amin = a; imin = j; }
        if (a > amax) { amax = a; imax = j; }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double a1 = __shfl_xor_sync(0xffffffffu, amin, o), a2 = __shfl_xor_sync(0xffffffffu, amax, o);
        const int i1 = __shfl_xor_sync(0xffffffffu, imin, o), i2 = __shfl_xor_sync(0xffffffffu, imax, o);
        if (a1 < amin || (a1 == amin && i1 < imin)) { amin = a1; imin = i1; }
        if (a2 > amax || (a2 == amax && i2 < imax)) { amax = a2; imax = i2; }
      }
      if (lane == 0) { emit(v[imin].x, v[imin].y); emit(v[imax].x, v[imax].y); }
    } else {
      for (int j = lane; j < nv; j += 32) emit(v[j].x, v[j].y);
    }
  }
}

// cv2 thickness-2 line into the byte image `cut` (oracle/cv_draw.py::thick_line2) with the shared rasteriser (csrc/cv_raster.cuh).
// All geometry is in GRID coordinates (the clipping rules refer to the grid); `cut` is the window at (ox, oy), pixels outside
// it are skipped.
struct CutWin {
  uint8_t* img; int W, H, ox, oy;
  __device__ __forceinline__ void put(long long x, long long y) const {
    x -= ox; y -= oy;
    if (x >= 0 && x < W && y >= 0 && y < H) img[y * W + x] = 1;
  }
  __device__ __forceinline__ void span(long long y, long long x1, long long x2, int first, int step) const {
    const long long wy = y - oy;
    if (wy < 0 || wy >= H) return;
    x1 -= ox; x2 -= ox;
    for (long long x = (x1 < 0 ? 0 : x1) + first; x <= x2 && x < W; x += step) img[wy * W + x] = 1;
  }
};
// One warp per ray (r: end points in window coordinates)
__device__ void thick_ray(const int4 r, uint8_t* __restrict__ cut, int W, int H, int ox, int oy, int G, int lane) {
  cvr::line(CutWin{cut, W, H, ox, oy}, G, r.x + ox, r.y + oy, r.z + ox, r.w + oy, 2, lane);
}

__global__ void thick_rays_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int nr = min(E.st->n_rays, E.rays_cap);
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int ri = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ri < nr; ri += nw)
    thick_ray(E.rays[ri], E.cut, E.W0, E.W0, E.ox, E.oy, E.G, lane);
}
// visible &= !cut; no obstacle contour in the cone -> reveal_fog_of_war returns the (all-zero) input mask
__global__ void apply_cut_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int n = E.W0 * E.W0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) if (E.cut[i]) E.visible[i] = 0;
}
__global__ void fog_gate_kernel(const ExEnv* __restrict__ envs) { ExState* st = envs[blockIdx.y].st; if (threadIdx.x == 0 && st->n_cont == 0) st->skip_fog = 1; }

// R5: pick the contour with the smallest |pointPolygonTest| to the agent; > 3 px -> nothing revealed
// obstacle_map.py:133-146: more than one external contour -> keep the first (cv2 order) that contains the agent (dist >= 0),
// else the nearest; the kept one is redrawn FILLED.   what: 0 = fog (R5), 1 = component selection
__global__ void contour_dist_kernel(const ExEnv* __restrict__ envs, int what) {
  const ExEnv& E = envs[blockIdx.y];
  const int nc = E.st->n_cont;
  if (what == 1 && nc <= 1) return;
  const int px = what == 0 ? E.sx : E.ax - E.fx0, py = what == 0 ? E.sy : E.ay - E.fy0;
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int ci = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ci < nc; ci += nw) {
    const double d = ppt_distance_warp(E.chain + E.cont[ci].off, E.cont[ci].len, px, py, lane);
    if (lane == 0) E.dist[ci] = d;
  }
}
__global__ void contour_pick_kernel(const ExEnv* __restrict__ envs, int what) {
  const ExEnv& E = envs[blockIdx.y];
  if (threadIdx.x != 0) return;
  ExState* st = E.st;
  if (what == 0) {
    int best = -1; double bd = INFINITY;
    for (int i = 0; i < st->n_cont; ++i) { const double d = fabs(E.dist[i]); if (d < bd) { bd = d; best = i; } }
    st->chosen = (st->skip_fog || bd > 3.0) ? -1 : best;
    if (st->chosen < 0) st->skip_fog = 1;
    *E.which = st->skip_fog ? -1 : st->chosen;
  } else {
    int best = -1;
    if (st->n_cont > 1) {
      double md = INFINITY; best = 0;
      for (int i = 0; i < st->n_cont; ++i) {
        const double d = E.dist[i];
        if (d >= 0) { best = i; break; }
        if (fabs(d) < md) { md = fabs(d); best = i; }
      }
    }
    *E.which = best;      // -1: a single contour, explored area stays as it is
  }
}

// S frame images of this step:  exS = ((explored | dilate3(newexp)) & nav) , navS = nav   (obstacle_map.py:125-127; outside the
// S frame explored is 0, so masking the S frame is masking the whole grid)
__global__ void explored_update_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int Sw = E.Sw, n = E.Sw * E.Sh, G = E.G, W0 = E.W0;
  const bool fog = !E.st->skip_fog;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int gy = E.fy0 + i / Sw, gx = E.fx0 + i % Sw;
    uint8_t e = E.explored[(size_t)gy * G + gx];
    if (fog && !e) {
      const int wx = gx - E.ox, wy = gy - E.oy;
      bool hit = false;
      for (int dy = -1; dy <= 1 && !hit; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int x = wx + dx, y = wy + dy;
          if ((unsigned)x < (unsigned)W0 && (unsigned)y < (unsigned)W0 && E.newexp[y * W0 + x]) { hit = true; break; }
        }
      if (hit) e = 1;
    }
    const uint8_t nv = E.nav[(size_t)gy * G + gx];
    if (nv == 0) e = 0;
    E.exS[i] = e; E.navS[i] = nv;
  }
}
// explored[S frame] = exS ; grown = dilate5(exS) ; unexp = nav & !grown ; ex2 = grown   (obstacle_map.py:159-163 + F1's input)
__global__ void paste_grow_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int W = E.Sw, H = E.Sh, n = W * H, G = E.G;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int y = i / W, x = i - y * W;
    E.explored[(size_t)(E.fy0 + y) * G + E.fx0 + x] = E.exS[i];
    uint8_t m = 0;
    for (int dy = -2; dy <= 2 && !m; ++dy) {
      const int yy = y + dy;
      if ((unsigned)yy >= (unsigned)H) continue;
      for (int dx = -2; dx <= 2; ++dx) { const int xx = x + dx; if ((unsigned)xx < (unsigned)W && E.exS[yy * W + xx]) { m = 1; break; } }
    }
    E.grown[i] = m; E.ex2[i] = m;
    E.unexp[i] = (E.navS[i] && !m) ? 1 : 0;
  }
}

// F1: small unexplored pockets (contourArea < thresh, filled mask only covers unexplored cells) are absorbed
// into the explored mask as 255.  One block per contour; cells of the bounding box are tested against the chain polygon.
__global__ void absorb_small_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int W = E.Sw;
  const int nc = E.st->n_cont;
  __shared__ long long s_a2;
  __shared__ int s_bad;
  for (int ci = blockIdx.x; ci < nc; ci += gridDim.x) {
    const Contour c = E.cont[ci];
    if (c.len == 0) continue;                     // not traced: the component encloses a hole or reaches the exterior
    const int2* p = E.chain + c.off;
    __syncthreads();
    if (threadIdx.x == 0) { s_a2 = 0; s_bad = 0; }
    __syncthreads();
    long long acc = 0;                                             // shoelace (twice the signed area), exact in integers
    for (int i = threadIdx.x; i < c.len; i += blockDim.x) {
      const int2 q = p[i == 0 ? c.len - 1 : i - 1], b = p[i];
      acc += (long long)q.x * b.y - (long long)b.x * q.y;
    }
    atomicAdd(reinterpret_cast<unsigned long long*>(&s_a2), (unsigned long long)acc);
    __syncthreads();
    const double area = fabs((double)s_a2 * 0.5);
    if (!(area < E.area_thresh)) continue;
    const int bw = c.x1 - c.x0 + 1, bh = c.y1 - c.y0 + 1;
    // pass 0: every cell drawContours would fill must be an unexplored (== 1) cell; pass 1: write
    for (int pass = 0; pass < 2; ++pass) {
      for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
        const int x = c.x0 + i % bw, y = c.y0 + i / bw;
        // even-odd with the exact-hit rule (unit edges: intercept is the lower endpoint's column) + outline
        int less = 0; bool exact = false;
        for (int e = 0; e < c.len; ++e) {
          const int2 a = p[e], b = p[e + 1 == c.len ? 0 : e + 1];
          if (a.x == x && a.y == y) exact = true;
          if (a.y == b.y) continue;
          const int ya = min(a.y, b.y), xa = a.y < b.y ? a.x : b.x;
          if (ya != y) continue;
          if (xa < x) ++less; else if (xa == x) exact = true;
        }
        if (exact || (less & 1)) {
          if (pass == 0) { if (E.unexp[y * W + x] != 1) s_bad = 1; }
          else E.ex2[y * W + x] = 255;
        }
      }
      __syncthreads();
      if (s_bad) break;
    }
  }
}

// F2-F4 (oracle/explore_oracle.py::_interpolate/_split/_midpoint)
__device__ __forceinline__ bool blur_zero(const uint8_t* nav, const uint8_t* ex2, int W, int H, int x, int y) {
  // cv2.blur 3x3 of 255*(nav & !explored2) is 0 iff all nine (BORDER_REFLECT_101) cells are 0
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      int xx = x + dx, yy = y + dy;
      if (xx < 0) xx = -xx; if (xx >= W) xx = 2 * W - 2 - xx;
      if (yy < 0) yy = -yy; if (yy >= H) yy = 2 * H - 2 - yy;
      if (nav[yy * W + xx] && !ex2[yy * W + xx]) return false;
    }
  return true;
}

// arc-length midpoint of the frontier q[a..b) followed by q[a2..b2) (second range empty unless merged); q[k] = p[(k+1)/2 mod n];
// written in GRID coordinates ((fx0, fy0) = S-frame origin) at out[0..1]
// length of one step of the interpolated chain: consecutive entries coincide or are 8-neighbours, so sqrt(d2) is 0, 1 or sqrt(2)
// (the correctly rounded double, exactly what np.sqrt returns); only the junction of a merged piece can be longer
__device__ __forceinline__ double seg_len(int2 u, int2 v) {
  const int d2 = (u.x - v.x) * (u.x - v.x) + (u.y - v.y) * (u.y - v.y);
  return d2 == 0 ? 0.0 : (d2 == 1 ? 1.0 : (d2 == 2 ? 1.4142135623730951 : sqrt((double)d2)));
}
// Entry i of the piece is q[k_i]; k advances by one (same point when k is odd -> a zero-length step that neither changes a sum nor
// can satisfy cum + 0 > half) except at the junction of a merged piece.  The walk keeps (k, index into p, point) incrementally: one
// load per chain point, no modulo in the loop.
struct QWalk {
  const int2* p; int n, a, len1, a2;
  int i, k, idx; int2 pt;
  __device__ void start(const int2* p_, int n_, int a_, int len1_, int a2_) {
    p = p_; n = n_; a = a_; len1 = len1_; a2 = a2_; i = 0;
    k = len1 > 0 ? a : a2; idx = ((k + 1) >> 1) % n; pt = p[idx];
  }
  // advance to entry i + 1; returns the length of the step
  __device__ double step() {
    ++i;
    int nidx;
    if (i == len1) { k = a2; nidx = ((k + 1) >> 1) % n; }
    else { nidx = (k & 1) ? idx : (idx + 1 == n ? 0 : idx + 1); ++k; }
    if (nidx == idx) return 0.0;
    const int2 q = p[nidx];
    const double l = seg_len(pt, q);
    idx = nidx; pt = q;
    return l;
  }
};
__device__ void midpoint(const int2* p, int n, int a, int b, int a2, int b2, int fx0, int fy0, double* out) {
  const int len1 = b - a, len2 = b2 - a2, len = len1 + len2;
  QWalk w;
  double total = 0.0;
  w.start(p, n, a, len1, a2);
  for (int i = 0; i + 1 < len; ++i) total += w.step();
  const double half = total / 2;
  double cum = 0.0, before = 0.0, l = 0.0;
  int2 u = make_int2(0, 0), v = make_int2(0, 0);
  bool found = false;
  w.start(p, n, a, len1, a2);
  const int2 first = w.pt;
  int2 second = first; bool have_second = false;
  for (int i = 0; i + 1 < len; ++i) {
    const int2 prev = w.pt;
    const double li = w.step();
    if (i == 0) { second = w.pt; have_second = true; }
    if (cum + li > half) { u = prev; v = w.pt; l = li; before = cum; found = true; break; }
    cum += li;
  }
  if (!found) {          // np.argmax of an all-False array is 0: segment 0
    u = first; v = have_second ? second : first; l = seg_len(u, v); before = 0.0;
  }
  const double t = (half - before) / l;
  out[0] = (double)(u.x + fx0) + t * (double)(v.x - u.x); out[1] = (double)(u.y + fy0) + t * (double)(v.y - u.y);
}

// F3 "bad" test of every traced border point at once (the walk below only reads the flags)
__global__ void bad_flags_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int nc = min(E.st->n_cont, E.maxc);
  for (int c = blockIdx.x; c < nc; c += gridDim.x) {        // chains live in per-contour slots: block per contour, threads over its points
    const int off = E.cont[c].off, n = E.cont[c].len;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      E.flags[off + i] = blur_zero(E.navS, E.ex2, E.Sw, E.Sh, E.chain[off + i].x, E.chain[off + i].y) ? 1 : 0;
  }
}
constexpr int FRONTIER_THREADS = 256;
// ordered compaction step: every thread of the block calls it; returns this thread's slot (or -1); `running` (identical in all
// threads) advances by the number of flagged threads
__device__ __forceinline__ int block_rank(bool flag, int* s_warp, int& running) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) s_warp[w] = __popc(m);
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int i = 0; i < FRONTIER_THREADS / 32; ++i) { const int c = s_warp[i]; if (i < w) before += c; total += c; }
  const int slot = flag ? running + before + __popc(m & ((1u << lane) - 1)) : -1;
  running += total;
  __syncthreads();
  return slot;
}
// One block per environment walks the external contours of the grown + absorbed explored mask in cv2 order: bad points split the
// (twice-interpolated) contour into pieces; pieces with <= 2 points are dropped, first and last merge when the contour start is
// not a bad point; every kept piece yields its arc-length midpoint.  The piece list is built by ordered block compactions and the
// midpoints are computed one thread per piece (each walk is a few hundred points).
__global__ void __launch_bounds__(FRONTIER_THREADS) frontier_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  ExState* st = E.st;
  __shared__ int s_warp[FRONTIER_THREADS / 32];
  int* blist = reinterpret_cast<int*>(E.sv);            // scratch: the SIMPLE-vertex buffer is free by now
  const int cap_ints = 2 * E.chain_cap;
  int n_front = 0;                                     // identical in all threads
  const int nc = st->n_cont;
  for (int ci = 0; ci < nc; ++ci) {
    const int2* p = E.chain + E.cont[ci].off;
    const uint8_t* fl = E.flags + E.cont[ci].off;
    const int n = E.cont[ci].len, m = 2 * n;            // the interpolated sequence q has 2n entries
    if (n == 0) continue;
    __syncthreads();                                   // the previous contour's lists are no longer read
    int nbad = 0;
    for (int base = 0; base < m; base += FRONTIER_THREADS) {
      const int k = base + threadIdx.x;
      const bool bd = k < m && fl[((k + 1) >> 1) % n] != 0;
      const int slot = block_rank(bd, s_warp, nbad);
      if (slot >= 0 && slot < cap_ints) blist[slot] = k;
    }
    if (nbad == 0) {                                   // a single piece, kept iff len > 2
      if (m > 2) {
        if (threadIdx.x == 0) { if (n_front < E.maxf) midpoint(p, n, 0, m, 0, 0, E.fx0, E.fy0, E.frontiers + 2 * n_front); else st->overflow = 1; }
        ++n_front;
      }
      continue;
    }
    if (3 * (long)nbad + 4 > cap_ints) { if (threadIdx.x == 0) st->overflow = 1; continue; }
    __syncthreads();
    // bad indices split q: piece 0 = [0, b0), piece j = [b_{j-1}, b_j) minus its first element, last = [b_last, m)
    const int first_bad = blist[0], last_bad = blist[nbad - 1];
    const bool wrap = first_bad != 0 && last_bad < m - 2;
    int* klist = blist + nbad;                          // kept pieces (ka, b), in order
    int nkept = 0;
    for (int base = 0; base <= nbad; base += FRONTIER_THREADS) {
      const int j = base + threadIdx.x;
      bool keep = false; int ka = 0, b = 0;
      if (j <= nbad) {
        const int a = j == 0 ? 0 : blist[j - 1];
        b = j == nbad ? m : blist[j];
        keep = (b - a > 2) || (j == 0 && wrap);
        ka = j == 0 ? a : a + 1;
      }
      const int slot = block_rank(keep, s_warp, nkept);
      if (slot >= 0) { klist[2 * slot] = ka; klist[2 * slot + 1] = b; }
    }
    if (nkept == 0) continue;
    __syncthreads();
    // with wrap the LAST kept piece is prepended to the FIRST kept piece (and comes first in the output)
    const bool merge = nkept > 1 && wrap;
    const int nslots = merge ? nkept - 1 : nkept;
    int nout = 0;
    for (int base = 0; base < nslots; base += FRONTIER_THREADS) {
      const int s = base + threadIdx.x;
      bool em = false; int a = 0, b = 0, a2 = 0, b2 = 0;
      if (s < nslots) {
        if (merge && s == 0) { a = klist[2 * (nkept - 1)]; b = klist[2 * (nkept - 1) + 1]; a2 = klist[0]; b2 = klist[1]; em = (b - a) + (b2 - a2) >= 2; }
        else { a = klist[2 * s]; b = klist[2 * s + 1]; em = b - a >= 2; }
      }
      const int slot = block_rank(em, s_warp, nout);
      if (slot >= 0) {
        const int k = n_front + slot;
        if (k < E.maxf) midpoint(p, n, a, b, a2, b2, E.fx0, E.fy0, E.frontiers + 2 * k); else st->overflow = 1;
      }
    }
    n_front += nout;
  }
  if (threadIdx.x == 0) st->n_front = n_front < E.maxf ? n_front : E.maxf;
}


// ---------------------------------------------------------------- fill_small_holes (img_utils.py:361-390) ----
// mask = (depth == 0) into the S-frame `unexp` plane (frame = the depth image), filled := 0
__global__ void zero_mask_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int n = E.Sw * E.Sh;
  if ((n & 3) == 0) {          // images are contiguous and 16-byte aligned per environment when H*W % 4 == 0
    const float4* d4 = reinterpret_cast<const float4*>(E.depth);
    uchar4* m4 = reinterpret_cast<uchar4*>(E.unexp); uchar4* f4 = reinterpret_cast<uchar4*>(E.filled);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n >> 2); i += gridDim.x * blockDim.x) {
      const float4 v = d4[i];
      m4[i] = make_uchar4(v.x == 0.f, v.y == 0.f, v.z == 0.f, v.w == 0.f);
      f4[i] = make_uchar4(0, 0, 0, 0);
    }
    return;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { E.unexp[i] = E.depth[i] == 0.f ? 1 : 0; E.filled[i] = 0; }
}
// RETR_TREE: the outer border of EVERY component and the border of every hole
__global__ void collect_all_kernel(const ExEnv* __restrict__ envs) {
  const ExEnv& E = envs[blockIdx.y];
  const int n = E.Sw * E.Sh;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int start = -1, ed = 0;
    if (E.Lfg[i] == i) { start = i; ed = 0; }
    else if (E.Lbg[i] == i && !E.outer[i]) { start = i - 1; ed = 4; }     // hole: the pixel west of its raster-first cell, entered from the east
    if (start < 0) continue;
    const int k = atomicAdd(&E.st->n_cont, 1);
    if (k < E.maxc) { E.cont[k].start = start; E.cont[k].ed = ed; } else E.st->overflow = 1;
  }
}
// one block per contour: contourArea < thresh -> drawContours(filled, [cnt], 0, 1, -1); bounding-box scan conversion in
// shared memory, processed in row bands when the box is tall
__global__ void __launch_bounds__(256)
fill_small_contours_kernel(const ExEnv* __restrict__ envs, int smem_words) {
  const ExEnv& E = envs[blockIdx.y];
  extern __shared__ uint32_t fs_smem[];
  __shared__ long long s_a2;
  const int W = E.Sw;
  const int nc = min(E.st->n_cont, E.maxc);
  const double area_thresh = E.area_thresh;
  uint8_t* filled = E.filled;
  for (int ci = blockIdx.x; ci < nc; ci += gridDim.x) {
    const Contour c = E.cont[ci];
    if (c.len == 0) continue;
    const int2* p = E.chain + c.off;
    __syncthreads();
    if (threadIdx.x == 0) s_a2 = 0;
    __syncthreads();
    long long acc = 0;
    for (int i = threadIdx.x; i < c.len; i += blockDim.x) {
      const int2 q = p[i == 0 ? c.len - 1 : i - 1], b = p[i];
      acc += (long long)q.x * b.y - (long long)b.x * q.y;
    }
    atomicAdd(reinterpret_cast<unsigned long long*>(&s_a2), (unsigned long long)acc);
    __syncthreads();
    if (!(fabs((double)s_a2 * 0.5) < area_thresh)) continue;
    if (c.len == 1) { if (threadIdx.x == 0) filled[(size_t)c.y0 * W + c.x0] = 1; continue; }   // speckle: the common case
    const int bw = c.x1 - c.x0 + 2, pw = (bw + 31) / 32;           // +1 column for the toggle right of the last cell
    const int band = smem_words / (2 * pw);
    for (int r0 = c.y0; r0 <= c.y1; r0 += band) {
      const int rows = min(band, c.y1 - r0 + 1);
      uint32_t* tog = fs_smem; uint32_t* orb = fs_smem + rows * pw;
      for (int i = threadIdx.x; i < 2 * rows * pw; i += blockDim.x) fs_smem[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < c.len; i += blockDim.x) {
        const int2 a = p[i], b = p[i + 1 == c.len ? 0 : i + 1];
        if (a.y >= r0 && a.y < r0 + rows) atomicOr(&orb[(a.y - r0) * pw + ((a.x - c.x0) >> 5)], 1u << ((a.x - c.x0) & 31));
        if (a.y != b.y) {
          const int xa = (a.y < b.y ? a.x : b.x) - c.x0, ya = min(a.y, b.y);
          if (ya >= r0 && ya < r0 + rows) {
            atomicXor(&tog[(ya - r0) * pw + ((xa + 1) >> 5)], 1u << ((xa + 1) & 31));
            atomicOr(&orb[(ya - r0) * pw + (xa >> 5)], 1u << (xa & 31));
          }
        }
      }
      __syncthreads();
      for (int r = threadIdx.x; r < rows; r += blockDim.x) {
        uint32_t carry = 0;
        for (int w = 0; w < pw; ++w) {
          const uint32_t t = tog[r * pw + w];
          uint32_t x = t;
          x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
          x ^= carry;
          if (__popc(t) & 1) carry = ~carry;
          uint32_t f = x | orb[r * pw + w];
          while (f) {
            const int bq = __ffs(f) - 1; f &= f - 1;
            const int col = c.x0 + w * 32 + bq;
            if (col <= c.x1) filled[(size_t)(r0 + r) * W + col] = 1;
          }
        }
      }
      __syncthreads();
    }
  }
}
// publish counters: frontier count / overflow flag (explore), sticky overflow status (holes)
__global__ void publish_kernel(const ExEnv* __restrict__ envs, int sticky) {
  const ExEnv& E = envs[blockIdx.x];
  if (threadIdx.x != 0) return;
  if (sticky) { if (E.st->overflow) *E.out_status |= 1; }
  else { *E.out_count = E.st->n_front; *E.out_status = E.st->overflow; }
}

}  // namespace vlfm

using namespace vlfm;

// -------------------------------------------------------------------------------------- host side ----
namespace {

constexpr int WIN_MAX = 512;
constexpr int CHAIN_CAP = 1 << 20, RAYS_CAP = 1 << 16, MAXF = 4096;
constexpr int HOLES_MAXC = 1 << 16;   // fill_small_holes sees sensor speckle: many more (tiny) contours than a map does

// carve one environment's arrays out of its workspace slice; `frame_cells` = cells of the largest frame (G*G or H*W)
size_t carve(ExEnv* e, uint8_t* base, size_t frame_cells, int frame_side, int maxc, bool explore) {
  size_t o = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + o : nullptr; o += (bytes + 255) & ~(size_t)255; return p; };
  const size_t wn = explore ? (size_t)WIN_MAX * WIN_MAX : 0;
  const size_t n = frame_cells > wn ? frame_cells : wn;                // label / flag arrays serve the window images too
  uint8_t* p;
  p = take(wn); if (e) e->cone = p;
  p = take(wn); if (e) e->blocked = p;
  p = take(wn); if (e) e->visible = p;
  p = take(wn); if (e) e->cut = p;
  p = take(wn); if (e) e->newexp = p;
  p = take(explore ? frame_cells : 0); if (e) e->exS = p;
  p = take(explore ? frame_cells : 0); if (e) e->navS = p;
  p = take(explore ? frame_cells : 0); if (e) e->grown = p;
  p = take(frame_cells); if (e) e->unexp = p;
  p = take(explore ? frame_cells : 0); if (e) e->ex2 = p;
  p = take(n); if (e) e->outer = p;
  p = take(n); if (e) e->hashole = p;
  p = take(n); if (e) e->nbm = p;
  p = take(n * 4); if (e) e->Lfg = (int*)p;
  p = take(n * 4); if (e) e->Lbg = (int*)p;
  p = take(sizeof(Contour) * (size_t)maxc); if (e) e->cont = (Contour*)p;
  p = take(sizeof(int2) * (size_t)CHAIN_CAP); if (e) e->chain = (int2*)p;
  p = take(explore ? sizeof(int2) * (size_t)CHAIN_CAP : 0); if (e) e->sv = (int2*)p;
  p = take(explore ? (size_t)CHAIN_CAP : 0); if (e) e->flags = p;
  p = take(explore ? sizeof(int) * (size_t)maxc : 0); if (e) e->nsv = (int*)p;
  p = take(explore ? sizeof(int4) * (size_t)RAYS_CAP : 0); if (e) e->rays = (int4*)p;
  p = take(explore ? sizeof(double) * EX_MAXC : 0); if (e) e->dist = (double*)p;
  const int side = frame_side > WIN_MAX || !explore ? frame_side : WIN_MAX;
  const size_t pw = ((size_t)side + 31) / 32;
  p = take(explore ? pw * side * 4 : 0); if (e) e->tog = (uint32_t*)p;
  p = take(explore ? pw * side * 4 : 0); if (e) e->orb = (uint32_t*)p;
  p = take(sizeof(ExState)); if (e) e->st = (ExState*)p;
  p = take(64); if (e) e->which = (int*)p;
  if (e) { e->chain_cap = CHAIN_CAP; e->rays_cap = RAYS_CAP; e->maxc = maxc; e->maxf = MAXF; }
  return o;
}

inline int nblk(long n, int t = 256, int cap = 2112) { long b = (n + t - 1) / t; return (int)(b < 1 ? 1 : (b > cap ? cap : b)); }
// Launch geometry of the batched sequences is FIXED (every kernel is grid-stride over its frame): the sequence of a call depends
// on the batch size only, so a caller can capture it in a CUDA graph and replay it with new per-environment records.
inline int gx_cells(int B) { return B >= 16 ? 132 : (B >= 4 ? 264 : 528); }     // blocks.x of the per-cell kernels
constexpr int GX_ROWS = 66;                                                     // blocks.x of the per-row kernels (8 warps each)

// external contours of image `id` of every environment: CCL fg/bg, top-level roots in cv2 order, traced chains.
// n_max / h_max / per_max: the largest image over the environments of the call.
void contours(const ExEnv* d_envs, int B, int id, cudaStream_t st, int keep_fog, int mode, int mark_exterior) {
  const int bx = gx_cells(B);
  ccl_init2_kernel<<<dim3(GX_ROWS, B), 256, 0, st>>>(d_envs, id, keep_fog);
  ccl_merge2_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, id, mode == 2);
  ccl_flatten2_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, id);
  bg_outer_kernel<<<dim3(16, B), 256, 0, st>>>(d_envs, id, mark_exterior);
  collect_roots_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, id);
  sort_roots_kernel<<<dim3(1, B), 1024, 0, st>>>(d_envs);
  if (mode == 2) mark_holes_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, id);
  trace_kernel<<<dim3(EX_MAXC / 64, B), 64, 0, st>>>(d_envs, id, mode);
  count_launch(mode == 2 ? 8 : 7);
}

// cv2.ellipse sector polygon (oracle/cv_draw.py::ellipse_sector), vertices in grid coordinates, 16.16
int sector_polygon(int cx, int cy, int radius, double start_deg, double end_deg, long long* v) {
  static float sintab[451];
  static bool init = false;
  if (!init) {
    for (int a = 0; a <= 450; ++a) { double s = sin(a * 3.14159265358979323846 / 180.0); sintab[a] = (float)(nearbyint(s * 1e7) / 1e7); }
    init = true;
  }
  auto cvr = [](double x) { return (long long)nearbyint(x); };
  int a0 = (int)cvr(start_deg), a1 = (int)cvr(end_deg);
  const long long CX = (long long)cx << XYS, CY = (long long)cy << XYS, AX = (long long)abs(radius) << XYS;
  long long d = (AX + (XYONE >> 1)) >> XYS;
  const int delta = d < 3 ? 90 : d < 10 ? 30 : d < 15 ? 18 : 5;
  if (a0 > a1) { int t = a0; a0 = a1; a1 = t; }
  while (a0 < 0) { a0 += 360; a1 += 360; }
  while (a1 > 360) { a1 -= 360; a0 -= 360; }
  if (a1 - a0 > 360) { a0 = 0; a1 = 360; }
  int nv = 0;
  long long px = 0, py = 0; bool have = false;
  for (int i = a0; i < a1 + delta; i += delta) {
    int ang = i > a1 ? a1 : i;
    if (ang < 0) ang += 360;
    const double x = (double)AX * (double)sintab[450 - ang], y = (double)AX * (double)sintab[ang];
    const double fx = (double)CX + x, fy = (double)CY + y;
    long long qx = cvr(fx / 65536.0) << XYS, qy = cvr(fy / 65536.0) << XYS;
    qx += cvr(fx - (double)qx); qy += cvr(fy - (double)qy);
    if (!have || qx != px || qy != py) { if (nv < 62) { v[2 * nv] = qx; v[2 * nv + 1] = qy; ++nv; } px = qx; py = qy; have = true; }
  }
  if (nv <= 1) { v[0] = CX; v[1] = CY; v[2] = CX; v[3] = CY; nv = 2; }
  v[2 * nv] = CX; v[2 * nv + 1] = CY; ++nv;
  return nv;
}


}  // namespace

extern "C" size_t vlfm_explore_env_record_bytes(void) { return sizeof(ExEnv); }

extern "C" int vlfm_explore_batch_workspace_bytes(int G, int batch, size_t* bytes) {
  if (!bytes || G < 8 || batch < 1) { set_error("vlfm_explore_batch_workspace_bytes: bad argument"); return VLFM_E_INVALID; }
  const size_t per = carve(nullptr, nullptr, (size_t)G * G, G, EX_MAXC, true);
  *bytes = per * (size_t)batch + (((size_t)batch * sizeof(ExEnv) + 255) & ~(size_t)255);
  return VLFM_OK;
}

// Batched explore step = vlfm_explore_prepare_batch (host: per-environment records into page-locked staging) +
// vlfm_explore_launch_batch (device: record upload + the launch sequence; CUDA-graph capturable, its launch geometry depends on
// `batch` only).  h_envs: `batch` VlfmExploreEnv records (host memory).  d_explored / d_nav: [nslots, G, G] uint8.
// d_frontiers [batch, 4096, 2] float64 (x = col, y = row), d_count / d_status [batch] int32 (in call order).
extern "C" int vlfm_explore_prepare_batch(int G, int batch, const VlfmExploreEnv* h_envs, uint8_t* d_explored, const uint8_t* d_nav,
                                          double* d_frontiers, int32_t* d_count, int32_t* d_status, void* d_workspace, size_t workspace_bytes,
                                          void* h_records, size_t h_records_bytes) {
  if (!h_envs || !d_explored || !d_nav || !d_frontiers || !d_count || !d_status || !d_workspace || !h_records || G < 8 || batch < 1 || batch > 65535) {
    set_error("vlfm_explore_prepare_batch: bad argument"); return VLFM_E_INVALID; }
  size_t need = 0;
  vlfm_explore_batch_workspace_bytes(G, batch, &need);
  if (workspace_bytes < need || h_records_bytes < sizeof(ExEnv) * (size_t)batch) {
    set_error("vlfm_explore_prepare_batch: workspace %zu < %zu bytes or staging %zu < %zu", workspace_bytes, need, h_records_bytes, sizeof(ExEnv) * (size_t)batch);
    return VLFM_E_INVALID; }
  const size_t per = carve(nullptr, nullptr, (size_t)G * G, G, EX_MAXC, true);
  uint8_t* wsb = (uint8_t*)d_workspace;
  ExEnv* envs = (ExEnv*)h_records;
  for (int b = 0; b < batch; ++b) {
    const VlfmExploreEnv& in = h_envs[b];
    ExEnv& e = envs[b];
    memset(&e, 0, sizeof(ExEnv));
    carve(&e, wsb + per * (size_t)b, (size_t)G * G, G, EX_MAXC, true);
    const int L = (int)in.max_line_len, W0 = 2 * L + 9;
    if (W0 > WIN_MAX || L < 1) { set_error("vlfm_explore_prepare_batch: max_line_len %d unsupported (window %d > %d)", L, W0, WIN_MAX); return VLFM_E_UNSUPPORTED; }
    int x0 = in.frame[0], y0 = in.frame[1], x1 = in.frame[2], y1 = in.frame[3];
    if (x0 < 0 || y0 < 0 || x1 > G || y1 > G || x1 - x0 < 1 || y1 - y0 < 1 || in.slot < 0) { set_error("vlfm_explore_prepare_batch: bad frame / slot (env %d)", b); return VLFM_E_INVALID; }
    e.G = G;
    e.explored = d_explored + (size_t)in.slot * G * G; e.nav = d_nav + (size_t)in.slot * G * G;
    e.frontiers = d_frontiers + (size_t)b * MAXF * 2; e.out_count = d_count + b; e.out_status = d_status + b;
    // the window is centred on the agent and may hang over the grid edge: cv2 clips the cone and the rays there
    e.ox = in.agent_col - L - 4; e.oy = in.agent_row - L - 4; e.W0 = W0; e.sx = in.agent_col - e.ox; e.sy = in.agent_row - e.oy;
    e.ax = in.agent_col; e.ay = in.agent_row;
    e.fx0 = x0; e.fy0 = y0; e.Sw = x1 - x0; e.Sh = y1 - y0;
    e.ext_l = x0 > 0; e.ext_t = y0 > 0; e.ext_r = x1 < G; e.ext_b = y1 < G;
    e.heading_deg = in.heading_deg; e.ray_len = in.max_line_len * 1.05; e.area_thresh = in.area_thresh_px;
    e.nv = sector_polygon(in.agent_col, in.agent_row, L, in.heading_deg - in.fov_deg / 2, in.heading_deg + in.fov_deg / 2, e.verts);   // R1
  }
  return VLFM_OK;
}

extern "C" int vlfm_explore_launch_batch(int G, int batch, void* d_workspace, const void* h_records, void* stream) {
  if (!d_workspace || !h_records || G < 8 || batch < 1 || batch > 65535) { set_error("vlfm_explore_launch_batch: bad argument"); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t per = carve(nullptr, nullptr, (size_t)G * G, G, EX_MAXC, true);
  ExEnv* d_envs = (ExEnv*)((uint8_t*)d_workspace + per * (size_t)batch);
  int rc = check_cuda(cudaMemcpyAsync(d_envs, h_records, sizeof(ExEnv) * (size_t)batch, cudaMemcpyHostToDevice, st), "explore: environment records");
  if (rc) return rc;
  const int B = batch;
  const int bc = gx_cells(B);
  // ---- R1: cone sector (window)
  zero_planes_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs, FRAME_WIN);
  sector_edges_kernel<<<dim3(1, B), 64, 0, st>>>(d_envs);
  planes_to_image_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs, 0, 1, 0);
  fog_masks_kernel<<<dim3(bc, B), 256, 0, st>>>(d_envs);
  // ---- R2/R3/R4: obstacle contours -> rays -> cut
  contours(d_envs, B, IMG_BLOCKED, st, 0, 0, 0);
  fog_gate_kernel<<<dim3(1, B), 32, 0, st>>>(d_envs);
  simple_vertices_kernel<<<dim3(64, B), 256, 0, st>>>(d_envs);
  rays_kernel<<<dim3(64, B), 256, 0, st>>>(d_envs);
  thick_rays_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs);
  apply_cut_kernel<<<dim3(bc, B), 256, 0, st>>>(d_envs);
  // ---- R5: contours of the visible area, nearest to the agent, filled
  contours(d_envs, B, IMG_VISIBLE, st, 1, 0, 0);
  contour_dist_kernel<<<dim3(EX_MAXC / 64, B), 64, 0, st>>>(d_envs, 0);
  contour_pick_kernel<<<dim3(1, B), 32, 0, st>>>(d_envs, 0);
  zero_planes_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs, FRAME_WIN);
  chain_edges_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs, FRAME_WIN);
  planes_to_image_kernel<<<dim3(32, B), 256, 0, st>>>(d_envs, 1, 0, 1);
  // ---- explored |= dilate3(new); explored[nav == 0] = 0  -> S frame images
  explored_update_kernel<<<dim3(bc, B), 256, 0, st>>>(d_envs);
  // ---- component selection (obstacle_map.py:128-146)
  contours(d_envs, B, IMG_EXS, st, 1, 1, 0);
  contour_dist_kernel<<<dim3(EX_MAXC / 64, B), 64, 0, st>>>(d_envs, 1);
  contour_pick_kernel<<<dim3(1, B), 32, 0, st>>>(d_envs, 1);
  zero_planes_kernel<<<dim3(bc, B), 256, 0, st>>>(d_envs, FRAME_S);
  chain_edges_kernel<<<dim3(64, B), 256, 0, st>>>(d_envs, FRAME_S);
  planes_to_image_kernel<<<dim3(64, B), 256, 0, st>>>(d_envs, 2, 1, 1);   // no-op when a single contour exists (which == -1)
  // ---- frontiers (obstacle_map.py:155-169 -> detect_frontier_waypoints)
  paste_grow_kernel<<<dim3(bc, B), 256, 0, st>>>(d_envs);
  contours(d_envs, B, IMG_UNEXP, st, 1, 2, 1);
  absorb_small_kernel<<<dim3(128, B), 128, 0, st>>>(d_envs);
  contours(d_envs, B, IMG_EX2, st, 1, 0, 0);     // every external contour is walked (mode 0)
  bad_flags_kernel<<<dim3(64, B), 256, 0, st>>>(d_envs);
  frontier_kernel<<<dim3(1, B), FRONTIER_THREADS, 0, st>>>(d_envs);
  publish_kernel<<<B, 32, 0, st>>>(d_envs, 0);
  VLFM_CHECK_LAUNCH("vlfm_explore_launch_batch");
  count_launch(26);
  return VLFM_OK;
}

extern "C" int vlfm_explore_update_batch(int G, int batch, const VlfmExploreEnv* h_envs, uint8_t* d_explored, const uint8_t* d_nav,
                                         double* d_frontiers, int32_t* d_count, int32_t* d_status, void* d_workspace, size_t workspace_bytes,
                                         void* h_pinned, size_t h_pinned_bytes, void* stream) {
  // without page-locked staging the records are built in a pageable buffer (cudaMemcpyAsync then waits for the stream first)
  std::vector<ExEnv> pageable;
  void* rec = h_pinned;
  size_t rec_bytes = h_pinned_bytes;
  if (!rec || rec_bytes < sizeof(ExEnv) * (size_t)batch) { if (batch < 1) { set_error("vlfm_explore_update_batch: bad argument"); return VLFM_E_INVALID; }
    pageable.resize((size_t)batch); rec = pageable.data(); rec_bytes = sizeof(ExEnv) * (size_t)batch; }
  int rc = vlfm_explore_prepare_batch(G, batch, h_envs, d_explored, d_nav, d_frontiers, d_count, d_status, d_workspace, workspace_bytes, rec, rec_bytes);
  if (rc) return rc;
  return vlfm_explore_launch_batch(G, batch, d_workspace, rec, stream);
}

extern "C" int vlfm_explore_workspace_bytes(int G, size_t* bytes) { return vlfm_explore_batch_workspace_bytes(G, 1, bytes); }

// one environment, whole-grid S frame (kept for callers that hold a single [G,G] pair)
extern "C" int vlfm_explore_update(int G, uint8_t* d_explored, const uint8_t* d_nav, int agent_col, int agent_row, double heading_deg,
                                   double fov_deg, double max_line_len, double area_thresh_px, int nav_half, double* d_frontiers,
                                   int32_t* d_count, void* d_workspace, int32_t* d_status, void* stream) {
  (void)nav_half;
  VlfmExploreEnv e;
  e.slot = 0; e.agent_col = agent_col; e.agent_row = agent_row; e.frame[0] = 0; e.frame[1] = 0; e.frame[2] = G; e.frame[3] = G; e.pad = 0;
  e.heading_deg = heading_deg; e.fov_deg = fov_deg; e.max_line_len = max_line_len; e.area_thresh_px = area_thresh_px;
  size_t ws = 0;
  int rc = vlfm_explore_batch_workspace_bytes(G, 1, &ws);
  if (rc) return rc;
  return vlfm_explore_update_batch(G, 1, &e, d_explored, d_nav, d_frontiers, d_count, d_status, d_workspace, ws, nullptr, 0, stream);
}

extern "C" int vlfm_holes_batch_workspace_bytes(int H, int W, int batch, size_t* bytes) {
  if (!bytes || H < 1 || W < 1 || batch < 1) { set_error("vlfm_holes_batch_workspace_bytes: bad argument"); return VLFM_E_INVALID; }
  const size_t per = carve(nullptr, nullptr, (size_t)H * W, H > W ? H : W, HOLES_MAXC, false);
  *bytes = per * (size_t)batch + (((size_t)batch * sizeof(ExEnv) + 255) & ~(size_t)255);
  return VLFM_OK;
}
extern "C" int vlfm_holes_workspace_bytes(int H, int W, size_t* bytes) { return vlfm_holes_batch_workspace_bytes(H, W, 1, bytes); }

// fill_small_holes (vlfm/utils/img_utils.py:361-390) for a batch of depth images: d_filled[b,H,W] := 1 where the reference
// would write depth 1.0.  d_status [batch]: sticky overflow flags.
extern "C" int vlfm_fill_small_holes_batch(const float* d_depth, int H, int W, int batch, double area_thresh, uint8_t* d_filled, void* d_workspace,
                                           size_t workspace_bytes, int32_t* d_status, void* h_pinned, size_t h_pinned_bytes, void* stream) {
  if (!d_depth || !d_filled || !d_workspace || !d_status || H < 1 || W < 1 || batch < 1 || batch > 65535) { set_error("vlfm_fill_small_holes_batch: bad argument"); return VLFM_E_INVALID; }
  size_t need = 0;
  vlfm_holes_batch_workspace_bytes(H, W, batch, &need);
  if (workspace_bytes < need) { set_error("vlfm_fill_small_holes_batch: workspace %zu < %zu bytes", workspace_bytes, need); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t per = carve(nullptr, nullptr, (size_t)H * W, H > W ? H : W, HOLES_MAXC, false);
  uint8_t* wsb = (uint8_t*)d_workspace;
  ExEnv* d_envs = (ExEnv*)(wsb + per * (size_t)batch);
  std::vector<ExEnv> pageable;
  ExEnv* envs;
  if (h_pinned && h_pinned_bytes >= sizeof(ExEnv) * (size_t)batch) envs = (ExEnv*)h_pinned;
  else { pageable.resize((size_t)batch); envs = pageable.data(); }
  for (int b = 0; b < batch; ++b) {
    ExEnv& e = envs[b];
    memset(&e, 0, sizeof(ExEnv));
    carve(&e, wsb + per * (size_t)b, (size_t)H * W, H > W ? H : W, HOLES_MAXC, false);
    e.G = W; e.Sw = W; e.Sh = H; e.W0 = 1;
    e.depth = d_depth + (size_t)b * H * W; e.filled = d_filled + (size_t)b * H * W; e.out_status = d_status + b; e.out_count = d_status + b;
    e.area_thresh = area_thresh;
  }
  int rc = check_cuda(cudaMemcpyAsync(d_envs, envs, sizeof(ExEnv) * (size_t)batch, cudaMemcpyHostToDevice, st), "holes: environment records");
  if (rc) return rc;
  const int B = batch;
  const int bx = gx_cells(B);
  zero_mask_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs);
  ccl_init2_kernel<<<dim3(GX_ROWS, B), 256, 0, st>>>(d_envs, IMG_UNEXP, 0);
  ccl_merge2_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, IMG_UNEXP, 0);
  ccl_flatten2_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs, IMG_UNEXP);
  bg_outer_kernel<<<dim3(16, B), 256, 0, st>>>(d_envs, IMG_UNEXP, 0);
  collect_all_kernel<<<dim3(bx, B), 256, 0, st>>>(d_envs);
  trace_kernel<<<dim3(128, B), 64, 0, st>>>(d_envs, IMG_UNEXP, 0);
  static bool cfg = false;
  const int smem_words = 24 * 1024;             // 96 KB of toggle / outline bit planes per block
  if (!cfg) {
    rc = check_cuda(cudaFuncSetAttribute(fill_small_contours_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_words * 4), "attr(fill_small_contours)");
    if (rc) return rc; cfg = true;
  }
  const int fb = B >= 8 ? 33 : (B >= 2 ? 132 : 264);
  fill_small_contours_kernel<<<dim3(fb, B), 256, smem_words * 4, st>>>(d_envs, smem_words);
  publish_kernel<<<B, 32, 0, st>>>(d_envs, 1);      // sticky: the host may poll it many steps later
  VLFM_CHECK_LAUNCH("vlfm_fill_small_holes_batch");
  count_launch(10);
  return VLFM_OK;
}
extern "C" int vlfm_fill_small_holes(const float* d_depth, int H, int W, double area_thresh, uint8_t* d_filled, void* d_workspace,
                                     int32_t* d_status, void* stream) {
  size_t ws = 0;
  int rc = vlfm_holes_batch_workspace_bytes(H, W, 1, &ws);
  if (rc) return rc;
  return vlfm_fill_small_holes_batch(d_depth, H, W, 1, area_thresh, d_filled, d_workspace, ws, d_status, nullptr, 0, stream);
}

// Confidence-cone template of ValueMap (vlfm/mapping/value_map.py:321-355 `_get_confidence_mask` / `_get_blank_cone_mask`):
// cv2.ellipse filled sector (+-fov/2 about +row) x cos^2 falloff.  d_out [R,R] float32, R = 2*int(max_depth*ppm)+1;
// d_scratch: R*R bytes + 2*R*ceil(R/32) uint32 + 2 KB.
extern "C" int vlfm_value_cone_template(double fov, double max_depth, int ppm, double min_conf, float* d_out, void* d_scratch,
                                        size_t scratch_bytes, void* stream) {
  const int half = (int)(max_depth * ppm), R = 2 * half + 1, pw = (R + 31) / 32;
  const size_t need = (((size_t)R * R + 255) & ~(size_t)255) + (size_t)2 * R * pw * 4 + 2048;
  if (!d_out || !d_scratch || half < 1 || scratch_bytes < need) { set_error("vlfm_value_cone_template: bad argument (scratch %zu < %zu)", scratch_bytes, need); return VLFM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sector = (uint8_t*)d_scratch;
  uint32_t* tog = (uint32_t*)(sector + (((size_t)R * R + 255) & ~(size_t)255));
  uint32_t* orb = tog + (size_t)R * pw;
  long long* verts = (long long*)(orb + (size_t)R * pw);
  const double deg = fov * 180.0 / 3.14159265358979323846;       // np.rad2deg
  long long hv[2 * MAXV];
  const int nv = sector_polygon(half, half, half, -deg / 2 + 90, deg / 2 + 90, hv);
  int rc = check_cuda(cudaMemcpyAsync(verts, hv, sizeof(long long) * 2 * nv, cudaMemcpyHostToDevice, st), "cone template: vertex upload");
  if (rc) return rc;
  zero_planes_plain_kernel<<<nblk((long)pw * R), 256, 0, st>>>(tog, orb, pw * R);
  sector_edges_plain_kernel<<<1, 64, 0, st>>>(verts, nv, R, tog, orb, pw);
  planes_to_image_plain_kernel<<<nblk((long)R * 32, 256), 256, 0, st>>>(tog, orb, sector, R, R, pw);
  cone_template_kernel<<<nblk((long)R * R), 256, 0, st>>>(sector, d_out, R, fov, min_conf);
  rc = check_cuda(cudaStreamSynchronize(st), "cone template");   // hv is a stack buffer: the upload must finish before returning
  if (rc) return rc;
  VLFM_CHECK_LAUNCH("vlfm_value_cone_template");
  count_launch(4);
  return VLFM_OK;
}
