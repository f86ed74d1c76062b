"""Explore half of ObstacleMap.update_map (vlfm/mapping/obstacle_map.py:114-169) and the
two third-party functions it calls.

TEST INFRASTRUCTURE.  PARITY UNPINNED.  ``frontier_exploration`` is an unpinned git
dependency (pyproject.toml:25: git+https://github.com/naokiyokoyama/frontier_exploration.git)
that is NOT in $VLFM_REFERENCE and cannot be fetched here; the reference has no test or
golden vector at this boundary.  ``reveal_fog_of_war`` and ``detect_frontier_waypoints``
below restate that package's published algorithm from its call sites
(obstacle_map.py:117-124, :164-168) and from the rules recorded in SURVEY.md section 8c;
every rule is listed so a maintainer with the package can diff it:

reveal_fog_of_war(top_down_map, fog_mask, current_point(row,col), current_angle, fov_deg, max_line_len)
  R1  cone = cv2.ellipse filled sector, centre (col,row), radius int(max_line_len), heading
      deg(wrap(-angle + pi/2)), spanning +-fov/2.
  R2  obstacles_in_cone = cone AND (1 - top_down_map); external contours (CHAIN_APPROX_SIMPLE).
      No obstacle contour -> return fog_mask unchanged.
  R3  per contour: convex -> the two points with extreme bearing from the agent; otherwise all points.
  R4  visible = cone AND top_down_map; from every such point draw a thickness-2 zero line from the
      point away from the agent to 1.05 x max_line_len (cv2.polylines).
  R5  external contours of what is left; keep the one with the smallest |pointPolygonTest| to the
      agent; if that distance > 3 px return fog_mask unchanged; else fill it into fog_mask.

detect_frontier_waypoints(full_map, explored_mask, area_thresh)
  F1  unexplored = full_map with explored cells zeroed; external contours; those with
      contourArea < area_thresh whose filled interior is uniformly 1 are absorbed into explored (255).
  F2  external contours of explored (CHAIN_APPROX_NONE), closed and Bresenham-interpolated.
  F3  unexplored' = where(explored>0, 0, full_map) -> x255 -> 3x3 cv2.blur; contour points whose
      blurred value is 0 are "bad" and split the contour; pieces with <= 2 points are dropped; first and
      last piece are merged when the contour start is not a bad point (wrap-around).
  F4  waypoint = arc-length midpoint of each piece.
"""
from __future__ import annotations

import numpy as np

from . import contours as _ct
from . import cv_draw as _dr
from . import cv_prims as _pr

# "cv2": call OpenCV exactly where frontier_exploration does.  "numpy": the same steps through the pinned
# restatements in oracle/contours.py, oracle/cv_draw.py, oracle/cv_prims.py (the rules a GPU port follows).
# Both are asserted identical by tests/test_oracle_explore.py.
PRIMS = "cv2"


def _contours(img, simple=True):
    if PRIMS == "cv2":
        import cv2

        return list(cv2.findContours(img, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE if simple else cv2.CHAIN_APPROX_NONE)[0])
    return _ct.find_external_contours(img, simple)


def _fill_contour(img, contour, value):
    if PRIMS == "cv2":
        import cv2

        return cv2.drawContours(img, [contour], 0, value, -1)
    img[_pr.fill_polygon(img.shape[0], img.shape[1], contour.reshape(-1, 2))] = value
    return img


def _ppt(contour, pt):
    if PRIMS == "cv2":
        import cv2

        return cv2.pointPolygonTest(contour, pt, True)
    return _ct.point_polygon_distance(contour, pt)


def _dilate(img, k):
    if PRIMS == "cv2":
        import cv2

        return cv2.dilate(img, np.ones((k, k), np.uint8), iterations=1)
    return _pr.dilate_box(img, k)


def wrap_heading(h: float) -> float:
    return (h + np.pi) % (2 * np.pi) - np.pi


def _extreme_bearing_points(src: np.ndarray, cnt: np.ndarray, yaw: float):
    pts = cnt.reshape(-1, 2) - src
    c, s = np.cos(-yaw), np.sin(-yaw)
    pts = np.matmul(pts, np.array([[c, -s], [s, c]]))
    ang = np.arctan2(pts[:, 1], pts[:, 0])
    return cnt[int(np.argmin(ang))], cnt[int(np.argmax(ang))]


def _ray_segments(src: np.ndarray, pts: np.ndarray, length: float) -> np.ndarray:
    ang = np.arctan2(pts[..., 1] - src[1], pts[..., 0] - src[0])
    ends = np.stack((pts[..., 0] + length * np.cos(ang), pts[..., 1] + length * np.sin(ang)), axis=-1).astype(np.int32)
    return np.stack([pts.reshape(-1, 2), ends.reshape(-1, 2)], axis=1)


def reveal_fog_of_war(top_down_map, current_fog_of_war_mask, current_point, current_angle, fov=90, max_line_len=100):
    src = np.asarray(current_point)[::-1].astype(int)
    heading = np.rad2deg(wrap_heading(-current_angle + np.pi / 2))
    if PRIMS == "cv2":
        import cv2

        cone = cv2.ellipse(np.zeros_like(top_down_map), tuple(int(v) for v in src), (int(max_line_len), int(max_line_len)), 0,
                           heading - fov / 2, heading + fov / 2, 1, -1)                                    # R1
    else:
        cone = _dr.ellipse_sector(top_down_map.shape[0], top_down_map.shape[1], (int(src[0]), int(src[1])), int(max_line_len),
                                  heading - fov / 2, heading + fov / 2).astype(top_down_map.dtype)
    blocked = cone & (1 - top_down_map)
    contours = _contours(blocked)                                                                          # R2
    if len(contours) == 0:
        return current_fog_of_war_mask
    pts = []
    for c in contours:                                                                                     # R3
        if (cv2.isContourConvex(c) if PRIMS == "cv2" else _ct.is_convex(c)):
            a, b = _extreme_bearing_points(src, c, heading)
            pts.append(a.reshape(-1, 2)); pts.append(b.reshape(-1, 2))
        else:
            pts.append(c.reshape(-1, 2))
    pts = np.concatenate(pts, axis=0)
    visible = cone & top_down_map
    segs = _ray_segments(src, pts, max_line_len * 1.05)                                                   # R4
    if PRIMS == "cv2":
        cv2.polylines(visible, segs, isClosed=False, color=0, thickness=2)
    else:
        cut = np.zeros(visible.shape, dtype=bool)
        for a, b in segs:
            _dr.thick_line2(cut, (int(a[0]), int(a[1])), (int(b[0]), int(b[1])))
        visible = np.where(cut, 0, visible).astype(top_down_map.dtype)
    final = _contours(visible)                                                                             # R5
    best, best_d = None, np.inf
    for c in final:
        d = abs(_ppt(c, tuple(int(i) for i in src)))
        if d < best_d:
            best, best_d = c, d
    if best_d > 3:
        return current_fog_of_war_mask
    return _fill_contour(current_fog_of_war_mask, best, 1)


def _bresenham(x0, y0, x1, y1):
    pts = []
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx = 1 if x0 < x1 else -1
    sy = 1 if y0 < y1 else -1
    err = dx - dy
    while True:
        pts.append((x0, y0))
        if x0 == x1 and y0 == y1:
            break
        e2 = 2 * err
        if e2 > -dy:
            err -= dy; x0 += sx
        if e2 < dx:
            err += dx; y0 += sy
    return pts


def _interpolate(contour: np.ndarray) -> np.ndarray:
    p = np.concatenate((contour, contour[:1])).reshape(-1, 2)
    out = []
    for (x0, y0), (x1, y1) in zip(p[:-1], p[1:]):
        out.extend(_bresenham(int(x0), int(y0), int(x1), int(y1)))
    return np.array(out).reshape(-1, 1, 2)


def _absorb_small_unexplored(full_map, explored, area_thresh):
    if area_thresh == -1:
        return explored
    unexplored = full_map.copy()
    unexplored[explored > 0] = 0
    small = []
    for c in _contours(unexplored):                                                                        # F1
        if _ct.contour_area(c) < area_thresh:
            m = _fill_contour(np.zeros_like(explored), c, 1)
            vals = set(unexplored[m.astype(bool)].tolist())
            if 1 in vals and len(vals) == 1:
                small.append(c)
    out = explored.copy()
    for c in small:
        _fill_contour(out, c, 255)
    return out


def _split(contour: np.ndarray, unexplored_blur: np.ndarray):
    n = len(contour)
    bad = [i for i in range(n) if unexplored_blur[contour[i][0][1], contour[i][0][0]] == 0]                # F3
    pieces = np.split(contour, bad)
    wrap = (0 not in bad) and len(bad) > 0 and max(bad) < n - 2
    kept = []
    for i, f in enumerate(pieces):
        if len(f) > 2 or (i == 0 and wrap):
            kept.append(f if i == 0 else f[1:])
    if len(kept) > 1 and wrap:
        last = kept.pop()
        kept[0] = np.concatenate((last, kept[0]))
    return kept


def _midpoint(f: np.ndarray) -> np.ndarray:
    p = f.reshape(-1, 2).astype(np.float64)
    seg = np.sqrt(((p[1:] - p[:-1]) ** 2).sum(1))                                                          # F4
    cum = np.cumsum(seg)
    half = cum[-1] / 2
    i = int(np.argmax(cum > half))
    before = cum[i - 1] if i > 0 else 0.0
    return p[i] + (half - before) / seg[i] * (p[i + 1] - p[i])


def detect_frontier_waypoints(full_map, explored_mask, area_thresh=-1, xy=None):
    explored = _absorb_small_unexplored(full_map, explored_mask, area_thresh)
    contours = _contours(explored, simple=False)                                                           # F2
    unexplored = np.where(explored > 0, 0, full_map)
    u255 = np.where(unexplored > 0, 255, unexplored).astype(np.uint8)
    if PRIMS == "cv2":
        import cv2

        blur = cv2.blur(u255, (3, 3))
    else:
        blur = _dr.blur3(u255)
    fronts = []
    for c in contours:
        fronts.extend(_split(_interpolate(c), blur))
    fronts = [f for f in fronts if len(f) >= 2]
    if not fronts:
        return np.array([])
    return np.array([_midpoint(f) for f in fronts])


def explore_step(m, tf, max_depth, topdown_fov) -> None:
    """obstacle_map.py:114-153 on an ObstacleMapOracle ``m``."""
    agent_px = m.xy_to_px(tf[:2, 3].reshape(1, 2))[0]
    yaw = float(np.arctan2(tf[1, 0], tf[0, 0]))
    new = reveal_fog_of_war(
        top_down_map=np.asarray(m._navigable_map).astype(np.uint8),
        current_fog_of_war_mask=np.zeros_like(m._map, dtype=np.uint8),
        current_point=agent_px[::-1], current_angle=-yaw, fov=np.rad2deg(topdown_fov),
        max_line_len=max_depth * m.ppm)
    new = _dilate(new, 3)
    m.explored_area[new > 0] = 1
    m.explored_area[np.asarray(m._navigable_map) == 0] = 0
    contours = _contours(m.explored_area.astype(np.uint8))
    if len(contours) > 1:
        best, best_d = 0, np.inf
        for i, c in enumerate(contours):
            d = _ppt(c, tuple(int(v) for v in agent_px))
            if d >= 0:
                best = i
                break
            if abs(d) < best_d:
                best, best_d = i, abs(d)
        area = _fill_contour(np.zeros_like(m.explored_area, dtype=np.uint8), contours[best], 1)
        m.explored_area = area.astype(bool)
    grown = _dilate(m.explored_area.astype(np.uint8), 5)
    m._frontiers_px = detect_frontier_waypoints(np.asarray(m._navigable_map).astype(np.uint8), grown, m.area_thresh_px)
    m.frontiers = m.px_to_xy(m._frontiers_px) if len(m._frontiers_px) else np.array([])
