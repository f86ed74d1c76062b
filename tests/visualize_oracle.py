"""Restatement of ValueMap.visualize / ObstacleMap.visualize and the trajectory overlay as functions of explicit state, drawing
with cv2 (reference: vlfm/mapping/value_map.py:189-219, obstacle_map.py:171-193, traj_visualizer.py).  Test infrastructure:
pinned to frames the reference itself rendered (tests/golden/live_visualize.npz, scripts/make_visualize_golden.py) by
tests/test_oracle_visualize.py, and the reference frames for tests/test_visualize_gpu.py.

The reference caches its path as a mask and adds only the new segments on each call; the union of all segments since the
last reset is the same set of pixels, which is what ``draw_trajectory`` draws.
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import cv2
import numpy as np


def metric_to_pixel(pt: Any, ppm: float, origin: np.ndarray) -> np.ndarray:
    px = pt * ppm * np.array([-1, -1]) + origin
    return px.astype(np.int32)


def draw_trajectory(img: np.ndarray, positions: Sequence[Any], yaw: float, ppm: float, origin: np.ndarray) -> np.ndarray:
    if len(positions) >= 2:
        mask = np.zeros(img.shape[:2], dtype=np.uint8)
        for a, b in zip(positions[:-1], positions[1:]):
            pa, pb = metric_to_pixel(a, ppm, origin), metric_to_pixel(b, ppm, origin)
            if np.array_equal(pa, pb):
                continue
            cv2.line(mask, tuple(pa[::-1]), tuple(pb[::-1]), 255, 3)
        img[mask == 255] = (0, 255, 0)
    p = metric_to_pixel(positions[-1], ppm, origin)
    cv2.circle(img, tuple(p[::-1]), 8, (255, 192, 15), -1)
    end = (int(p[0] - 10 * 1.0 * np.cos(yaw)), int(p[1] - 10 * 1.0 * np.sin(yaw)))
    cv2.line(img, tuple(p[::-1]), tuple(end[::-1]), (0, 0, 0), 3)
    return img


def inferno(image: np.ndarray) -> np.ndarray:
    lo, hi = np.min(image), np.max(image)
    ptp = hi - lo
    norm = np.zeros_like(image) if ptp == 0 else (image - lo) / ptp
    return cv2.applyColorMap((norm * 255).astype(np.uint8), cv2.COLORMAP_INFERNO)


def value_frame(value_grid: np.ndarray, reduce_fn: Callable, explored: Optional[np.ndarray], positions: Sequence[Any], yaw: float,
                markers: Optional[List[Tuple[np.ndarray, Dict[str, Any]]]], ppm: float, origin: np.ndarray) -> np.ndarray:
    """value_grid: [G, G, C] in the dtype the reference's grid has (float64 after a weighted fuse)."""
    reduced = reduce_fn(value_grid).copy()
    if explored is not None:
        reduced[explored == 0] = 0
    img = np.flipud(reduced)
    zero = img == 0
    img[zero] = np.max(img)
    img = inferno(img)
    img[zero] = (255, 255, 255)
    if len(positions) > 0:
        draw_trajectory(img, positions, yaw, ppm, origin)
        for pos, kw in markers or []:
            p = metric_to_pixel(pos, ppm, origin)
            cv2.circle(img, tuple(p[::-1]), **kw)
    return img


def obstacle_frame(obst: np.ndarray, nav: np.ndarray, explored: np.ndarray, frontiers_px: np.ndarray, padding_color: Sequence[int],
                   positions: Sequence[Any], yaw: float, ppm: float, origin: np.ndarray) -> np.ndarray:
    vis = np.ones((*obst.shape[:2], 3), dtype=np.uint8) * 255
    vis[explored == 1] = (200, 255, 200)
    vis[nav == 0] = padding_color
    vis[obst == 1] = (0, 0, 0)
    for f in frontiers_px:
        cv2.circle(vis, tuple([int(i) for i in f]), 5, (200, 0, 0), 2)
    vis = cv2.flip(vis, 0)
    if len(positions) > 0:
        draw_trajectory(vis, positions, yaw, ppm, origin)
    return vis


def itm_v3_reducer(thresh: float) -> Callable:
    """ITMPolicyV3's visualisation reducer (itm_policy.py:275-285)."""
    def reduce(arr: np.ndarray) -> np.ndarray:
        first = arr[:, :, 0]
        return np.where(first > thresh, first, np.max(arr, axis=2))
    return reduce


def max_reducer(i: np.ndarray) -> np.ndarray:
    return np.max(i, axis=-1)
