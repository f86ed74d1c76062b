// OpenCV 4.13 drawing.cpp rasterisation rules on the device (LINE_8, integer / 16.16 fixed point), shared by the explore
// half's occlusion rays (csrc/explore.cu, thickness 2 into a window mask) and the map frames (csrc/render.cu, any thickness
// into a BGR frame).  Restated in Python by oracle/cv_prims.py / oracle/cv_draw.py and pinned against cv2 by the tests.
//
// Every function is called by all 32 lanes of a warp with the same arguments: the control flow is replayed by every lane and
// the pixel writes are split among them.  Pixels go to a Sink, which clips to what it can hold:
//   s.put(x, y)                      one pixel (grid coordinates, may lie outside the grid)
//   s.span(y, x1, x2, first, step)   pixels x1 + first, x1 + first + step, ... <= x2 of row y (unclipped range)
// G is the side of the grid the clipping rules refer to (cv2's image).
#pragma once
#include <math.h>
#include <stdint.h>

namespace vlfm {
namespace cvr {

constexpr int SHIFT = 16;                   // XY_SHIFT
constexpr long long ONE = 1ll << SHIFT;

// cv::clipLine(Size2l(W, H), pt1, pt2) (oracle/cv_prims.py::clip_line): Cohen-Sutherland, intersections in double, truncated
// toward zero.  cv2 clips every line to the image before walking it, so a line that leaves the grid is the walk of the CLIPPED
// segment.  The end points are modified even when the function returns false (as in OpenCV).
__device__ __forceinline__ long long clip_isect(long long a, long long b, long long c) {   // (int64)((double)a * b / c)
  return (long long)__ddiv_rn(__dmul_rn((double)a, (double)b), (double)c);
}
__device__ inline bool clip_line(long long W, long long H, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = W - 1, bottom = H - 1;
  if (W <= 0 || H <= 0) return false;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) { a = c1 < 8 ? 0 : bottom; x1 += clip_isect(a - y1, x2 - x1, y2 - y1); y1 = a; c1 = (x1 < 0) + (x1 > right) * 2; }
    if (c2 & 12) { a = c2 < 8 ? 0 : bottom; x2 += clip_isect(a - y2, x2 - x1, y2 - y1); y2 = a; c2 = (x2 < 0) + (x2 > right) * 2; }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) { a = c1 == 1 ? 0 : right; y1 += clip_isect(a - x1, y2 - y1, x2 - x1); x1 = a; c1 = 0; }
      if (c2) { a = c2 == 1 ? 0 : right; y2 += clip_isect(a - x2, y2 - y1, x2 - x1); x2 = a; c2 = 0; }
    }
  }
  return (c1 | c2) == 0;
}

// cv2.line thickness 1: LineIterator walks the clipped segment towards +x; pixel k of the walk is closed-form
// (oracle/cv_prims.py::line_minor_steps), so the lanes stride over k
template <class Sink>
__device__ void line8(const Sink& s, int G, long long x0, long long y0, long long x1, long long y1, int lane) {
  if (!clip_line(G, G, x0, y0, x1, y1)) return;
  if (x1 < x0) { long long t = x0; x0 = x1; x1 = t; t = y0; y0 = y1; y1 = t; }
  const long long dx = x1 - x0, dy = y1 - y0, sy = dy >= 0 ? 1 : -1, ady = dy >= 0 ? dy : -dy;
  const bool ymaj = ady > dx;
  const long long major = ymaj ? ady : dx, minor = ymaj ? dx : ady;
  for (long long k = lane; k <= major; k += 32) {
    const long long st = major == 0 ? 0 : (2 * minor * k + major - 1) / (2 * major);
    if (ymaj) s.put(x0 + st, y0 + sy * k); else s.put(x0 + k, y0 + sy * st);
  }
}

// Line2 (16.16 end points, the outline of FillConvexPoly): clipLine against the grid scaled to 16.16, then the DDA; step i is
// closed-form (x1 + i, y1 + i * y_step)
template <class Sink>
__device__ void line2(const Sink& s, int G, long long x1, long long y1, long long x2, long long y2, int lane) {
  if (!clip_line((long long)G << SHIFT, (long long)G << SHIFT, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long x_step, y_step, ecount;
  if (ax > ay) {
    if (dx < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
    x_step = ONE; y_step = (dy << SHIFT) / (ax | 1); ecount = (x2 - x1) >> SHIFT;
  } else {
    if (dy < 0) { long long t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
    x_step = (dx << SHIFT) / (ay | 1); y_step = ONE; ecount = (y2 - y1) >> SHIFT;
  }
  x1 += ONE >> 1; y1 += ONE >> 1;
  if (lane == 0) s.put((x2 + (ONE >> 1)) >> SHIFT, (y2 + (ONE >> 1)) >> SHIFT);
  if (ax > ay) {
    const long long x = x1 >> SHIFT;
    for (long long i = lane; i <= ecount; i += 32) s.put(x + i, (y1 + i * y_step) >> SHIFT);
  } else {
    const long long y = y1 >> SHIFT;
    for (long long i = lane; i <= ecount; i += 32) s.put((x1 + i * x_step) >> SHIFT, y + i);
  }
}

__device__ __forceinline__ long long pick4(const long long (&a)[4], int i) { return i == 0 ? a[0] : (i == 1 ? a[1] : (i == 2 ? a[2] : a[3])); }

// FillConvexPoly(quad, shift 16): Line2 outline + the two-edge scan.  Every lane replays the scan's edge bookkeeping, jumping
// from edge switch to edge switch (<= 4 of them); between two switches both edge x positions are linear in the row, so the
// rows of such a span are split among the lanes.
template <class Sink>
__device__ void fill_quad(const Sink& s, int G, const long long (&vx)[4], const long long (&vy)[4], int lane) {
#pragma unroll
  for (int i = 0; i < 4; ++i) { const int j = (i + 3) & 3; line2(s, G, vx[j], vy[j], vx[i], vy[i], lane); }
  const long long delta = ONE >> 1;
  int imin = 0;
  long long ymin_f = vy[0], ymax_f = vy[0], xmin_f = vx[0], xmax_f = vx[0];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (vy[i] < ymin_f) { ymin_f = vy[i]; imin = i; }
    ymax_f = vy[i] > ymax_f ? vy[i] : ymax_f; xmax_f = vx[i] > xmax_f ? vx[i] : xmax_f; xmin_f = vx[i] < xmin_f ? vx[i] : xmin_f;
  }
  long long ymin = (ymin_f + delta) >> SHIFT, ymax = (ymax_f + delta) >> SHIFT;
  const long long xmin = (xmin_f + delta) >> SHIFT, xmax = (xmax_f + delta) >> SHIFT;
  if (xmax < 0 || ymax < 0 || xmin >= G || ymin >= G) return;       // OpenCV's early-out refers to the grid
  if (ymax > G - 1) ymax = G - 1;
  struct { int idx, di; long long x, dx, ye; } e[2];
  e[0].idx = e[1].idx = imin; e[0].ye = e[1].ye = ymin; e[0].di = 1; e[1].di = 3;
  e[0].x = e[1].x = -ONE; e[0].dx = e[1].dx = 0;
  int edges = 4;
  long long y = ymin;
  while (y <= ymax) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (y >= e[i].ye) {
        int idx0 = e[i].idx, di = e[i].di, idx = (idx0 + di) & 3;
        for (; edges-- > 0;) {
          const long long ty = (pick4(vy, idx) + delta) >> SHIFT;
          if (ty > y) {
            const long long xs = pick4(vx, idx0), xe = pick4(vx, idx);
            e[i].ye = ty; e[i].dx = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y)); e[i].x = xs; e[i].idx = idx;
            break;
          }
          idx0 = idx; idx = (idx + di) & 3;
        }
      }
    }
    if (edges < 0) break;
    // rows y .. yn-1 use the current pair of edges (the serial loop re-examines an edge only when y reaches its ye)
    long long yn = e[0].ye < e[1].ye ? e[0].ye : e[1].ye;
    if (yn > ymax + 1) yn = ymax + 1;
    if (yn <= y) yn = y + 1;
    for (long long yy = y + lane; yy < yn; yy += 32) {
      if (yy < 0) continue;
      const long long ex0 = e[0].x + (yy - y) * e[0].dx, ex1 = e[1].x + (yy - y) * e[1].dx;
      const bool sw = ex0 > ex1;
      s.span(yy, ((sw ? ex1 : ex0) + delta) >> SHIFT, ((sw ? ex0 : ex1) + delta) >> SHIFT, 0, 1);
    }
    e[0].x += (yn - y) * e[0].dx; e[1].x += (yn - y) * e[1].dx;
    y = yn;
  }
}

// Circle (integer centre): the midpoint walk, outline points (lanes 0..7) or filled spans (all lanes)
template <class Sink>
__device__ void circle(const Sink& s, long long cx, long long cy, int radius, bool fill, int lane) {
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  while (dx >= dy) {
    const long long y11 = cy - dy, y12 = cy + dy, y21 = cy - dx, y22 = cy + dx;
    const long long x11 = cx - dx, x12 = cx + dx, x21 = cx - dy, x22 = cx + dy;
    if (fill) {
      s.span(y11, x11, x12, lane, 32); s.span(y12, x11, x12, lane, 32);
      s.span(y21, x21, x22, lane, 32); s.span(y22, x21, x22, lane, 32);
    } else if (lane < 8) {
      const long long px = (lane & 4) ? ((lane & 1) ? x22 : x21) : ((lane & 1) ? x12 : x11);
      const long long py = (lane & 4) ? ((lane & 2) ? y22 : y21) : ((lane & 2) ? y12 : y11);
      s.put(px, py);
    }
    dy++;
    err += plus;
    plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask;
    dx += mask;
    minus -= mask & 2;
  }
}

// ThickLine (thickness >= 2) between 16.16 points: the quad along the fixed-point normal (half width (t + (t & 1)) / 2) and
// filled Circle caps of radius (t + 1) / 2; `flags` bit 0 / 1: cap at p0 / p1
template <class Sink>
__device__ void thick_line(const Sink& s, int G, long long x0, long long y0, long long x1, long long y1, int thickness, int flags, int lane) {
  const double dx = (double)(x0 - x1) / 65536.0, dy = (double)(y1 - y0) / 65536.0;
  double rr = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  const int odd = thickness & 1;
  const long long th = (long long)thickness << (SHIFT - 1);
  if (fabs(rr) > 2.220446049250313e-16) {
    rr = __ddiv_rn(__dadd_rn((double)th, odd * 32768.0), sqrt(rr));
    const long long dpx = (long long)rint(__dmul_rn(dy, rr)), dpy = (long long)rint(__dmul_rn(dx, rr));
    const long long vx[4] = {x0 + dpx, x0 - dpx, x1 - dpx, x1 + dpx}, vy[4] = {y0 + dpy, y0 - dpy, y1 - dpy, y1 + dpy};
    fill_quad(s, G, vx, vy, lane);
  }
  const int cap = (int)((th + (ONE >> 1)) >> SHIFT);
  if (flags & 1) circle(s, (x0 + (ONE >> 1)) >> SHIFT, (y0 + (ONE >> 1)) >> SHIFT, cap, true, lane);
  if (flags & 2) circle(s, (x1 + (ONE >> 1)) >> SHIFT, (y1 + (ONE >> 1)) >> SHIFT, cap, true, lane);
}

// cv2.line(img, p0, p1, color, thickness, LINE_8, 0) with integer end points
template <class Sink>
__device__ void line(const Sink& s, int G, long long x0, long long y0, long long x1, long long y1, int t, int lane) {
  if (t <= 1) { line8(s, G, x0, y0, x1, y1, lane); return; }
  // cv2 4.13 clips the integer centre line to the image grown by the thickness before building the quad and the caps
  long long a = x0 + t, b = y0 + t, d = x1 + t, e = y1 + t;
  if (!clip_line((long long)G + 2 * t, (long long)G + 2 * t, a, b, d, e)) return;
  thick_line(s, G, (a - t) << SHIFT, (b - t) << SHIFT, (d - t) << SHIFT, (e - t) << SHIFT, t, 3, lane);
}

// OpenCV's SinTable: sin of integer degrees with seven decimals, as float
__device__ __forceinline__ double sin_table(int deg) {
  return (double)(float)(rint(sin(deg * 3.14159265358979323846 / 180.0) * 1e7) / 1e7);
}

// cv2.circle(img, centre, radius, color, thickness, LINE_8, 0); thickness -1 = filled.  Thickness >= 2 is EllipseEx:
// ellipse2Poly(0..360 deg) in 16.16, consecutive duplicates dropped, then an open PolyLine of ThickLines (no centre-line clip
// at shift 16), caps at the first segment's start and every segment's end.
template <class Sink>
__device__ void circle_cv(const Sink& s, int G, long long cx, long long cy, int radius, int t, int lane) {
  if (t <= 1) { circle(s, cx, cy, radius, t < 0, lane); return; }
  const long long CX = cx << SHIFT, CY = cy << SHIFT, AX = (long long)radius << SHIFT;
  const long long dd = (AX + (ONE >> 1)) >> SHIFT;
  const int delta = dd < 3 ? 90 : dd < 10 ? 30 : dd < 15 ? 18 : 5;
  long long qx = 0, qy = 0;
  int np = 0;
  for (int i = 0; i < 360 + delta; i += delta) {
    const int ang = i > 360 ? 360 : i;
    const double fx = __dadd_rn((double)CX, __dmul_rn((double)AX, sin_table(450 - ang)));
    const double fy = __dadd_rn((double)CY, __dmul_rn((double)AX, sin_table(ang)));
    long long vx = (long long)rint(fx / 65536.0) << SHIFT, vy = (long long)rint(fy / 65536.0) << SHIFT;
    vx += (long long)rint(fx - (double)vx); vy += (long long)rint(fy - (double)vy);
    if (np > 0 && vx == qx && vy == qy) continue;
    if (np > 0) thick_line(s, G, qx, qy, vx, vy, t, np == 1 ? 3 : 2, lane);
    qx = vx; qy = vy; ++np;
  }
  if (np == 1) thick_line(s, G, CX, CY, CX, CY, t, 3, lane);   // a zero-size polygon: two copies of the centre
}

}  // namespace cvr
}  // namespace vlfm
