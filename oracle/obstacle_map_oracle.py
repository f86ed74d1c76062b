"""CPU restatement of the VLFM obstacle map (reference: vlfm/mapping/obstacle_map.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).
Obstacle half (:86-109, hole fill -> point cloud -> height band -> np.rint scatter ->
k x k dilation): PINNED bit-for-bit against the real reference class (imported with
``frontier_exploration`` stubbed, tests/test_oracle_obstacle.py + golden fixtures).
Explore half (:114-169): built on oracle/frontier_exploration_oracle.py, whose source
package is absent from $VLFM_REFERENCE -> parity UNPINNED for that half.
"""
from __future__ import annotations

from typing import Optional

import numpy as np


def unproject(depth_m: np.ndarray, keep: np.ndarray, fx: float, fy: float) -> np.ndarray:
    """geometry_utils.py:216-236 -- camera frame (+x fwd, +y left, +z up) = (z, -x, -y)."""
    v, u = np.nonzero(keep)
    z = depth_m[v, u]
    lateral = (u - depth_m.shape[1] // 2) * z / fx
    vertical = (v - depth_m.shape[0] // 2) * z / fy
    return np.stack((z, -lateral, -vertical), axis=-1)


def rigid(tf: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """geometry_utils.py:205-213 -- homogeneous 4x4 via np.dot (BLAS)."""
    hom = np.hstack((pts, np.ones((pts.shape[0], 1))))
    out = np.dot(tf, hom.T).T
    return out[:, :3] / out[:, 3:]


def fill_holes(depth: np.ndarray, area_thresh: int) -> np.ndarray:
    """img_utils.py:361-390 -- zero regions whose cv2.contourArea < thresh become 1."""
    import cv2

    holes = np.where(depth == 0, 1, 0).astype("uint8")
    contours, _ = cv2.findContours(holes, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    fill = np.zeros_like(holes)
    for c in contours:
        if cv2.contourArea(c) < area_thresh:
            cv2.drawContours(fill, [c], 0, 1, -1)
    return np.where(fill == 1, 1, depth)


def fill_holes_numpy(depth: np.ndarray, area_thresh: int) -> np.ndarray:
    """fill_holes without cv2: Suzuki-Abe borders (outer and hole), shoelace area, polygon fill."""
    from . import contours as ct
    from . import cv_prims as pr

    holes = np.where(depth == 0, 1, 0).astype("uint8")
    fill = np.zeros(holes.shape, dtype=bool)
    for c in ct.find_all_contours(holes):
        if ct.contour_area(c) < area_thresh:
            fill |= pr.fill_polygon(holes.shape[0], holes.shape[1], c.reshape(-1, 2))
    return np.where(fill, 1, depth)


class ObstacleMapOracle:
    def __init__(self, min_height: float, max_height: float, agent_radius: float, area_thresh: float = 3.0,
                 hole_area_thresh: int = 100000, size: int = 1000, pixels_per_meter: int = 20):
        self.size, self.ppm = size, pixels_per_meter
        self.origin = np.array([size // 2, size // 2])
        self._map = np.zeros((size, size), dtype=bool)
        self._navigable_map = np.zeros((size, size), dtype=bool)
        self.explored_area = np.zeros((size, size), dtype=bool)
        self.min_h, self.max_h = min_height, max_height
        self.area_thresh_px = area_thresh * pixels_per_meter**2
        self.hole_thresh = hole_area_thresh
        k = pixels_per_meter * agent_radius * 2
        self.k = int(k) + (int(k) % 2 == 0)
        self._frontiers_px = np.array([])
        self.frontiers = np.array([])

    def xy_to_px(self, pts: np.ndarray) -> np.ndarray:  # base_map.py:35-46
        px = np.rint(pts[:, ::-1] * self.ppm) + self.origin
        px[:, 0] = self.size - px[:, 0]
        return px.astype(int)

    def px_to_xy(self, px: np.ndarray) -> np.ndarray:  # base_map.py:48-60
        q = px.copy()
        q[:, 0] = self.size - q[:, 0]
        return ((q - self.origin) / self.ppm)[:, ::-1]

    def update_obstacles(self, depth, tf, min_depth, max_depth, fx, fy) -> None:
        import cv2

        if self.hole_thresh == -1:
            filled = depth.copy()
            filled[depth == 0] = 1.0
        else:
            filled = fill_holes(depth, self.hole_thresh)
        metres = filled * (max_depth - min_depth) + min_depth
        cloud = rigid(tf, unproject(metres, metres < max_depth, fx, fy))
        cloud = cloud[(cloud[:, 2] >= self.min_h) & (cloud[:, 2] <= self.max_h)]
        px = self.xy_to_px(cloud[:, :2])
        self._map[px[:, 1], px[:, 0]] = 1
        grown = cv2.dilate(self._map.astype(np.uint8), np.ones((self.k, self.k), np.uint8), iterations=1)
        self._navigable_map = 1 - grown.astype(bool)

    def update_map(self, depth, tf, min_depth, max_depth, fx, fy, topdown_fov, explore=True, update_obstacles=True):
        if update_obstacles:
            self.update_obstacles(depth, tf, min_depth, max_depth, fx, fy)
        if not explore:
            return
        from .explore_oracle import explore_step

        explore_step(self, tf, max_depth, topdown_fov)
