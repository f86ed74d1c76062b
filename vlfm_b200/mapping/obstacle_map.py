"""GPU obstacle / explored-area map behind the reference's ``ObstacleMap`` surface.

Reference: vlfm/mapping/obstacle_map.py (class :15, update_map :55, reset :48).
Grids are uint8 [1,G,G] tensors in HBM: ``obst`` (ObstacleMap._map), ``nav``
(_navigable_map as 0/1) and ``explored`` (explored_area).  This class is the batch-1 instance of
``ObstacleMapBatch`` (obstacle_batch.py), which a vectorised caller uses directly for B environments per launch sequence.
"""
from __future__ import annotations

from typing import Any, Optional, Union

import numpy as np
import torch

from .. import _lib
from . import render as _render
from .base_map import BaseMap
from .obstacle_batch import ObstacleMapBatch


class ObstacleMap(BaseMap):
    radius_padding_color: tuple = (100, 100, 100)

    def __init__(self, min_height: float, max_height: float, agent_radius: float, area_thresh: float = 3.0,
                 hole_area_thresh: int = 100000, size: int = 1000, pixels_per_meter: int = 20,
                 device: Union[str, torch.device, None] = None):
        super().__init__(size, pixels_per_meter)
        self._eng = ObstacleMapBatch(1, min_height, max_height, agent_radius, area_thresh, hole_area_thresh, size, pixels_per_meter, device)
        self.lib = self._eng.lib
        self.device = self._eng.device
        self._obst, self._nav, self._explored = self._eng.obst, self._eng.nav, self._eng.explored
        self._min_height = min_height
        self._max_height = max_height
        self._area_thresh_in_pixels = self._eng.area_thresh_px  # obstacle_map.py:41
        self._hole_area_thresh = hole_area_thresh
        self._kernel = self._eng.kernel
        self._front_cache: Optional[np.ndarray] = np.array([])
        self._pin: Optional[torch.Tensor] = None
        self._pin_tf: Optional[torch.Tensor] = None
        self._dev_depth: Optional[torch.Tensor] = None
        self._dev_tf = torch.empty((1, 16), dtype=torch.float64, device=self.device)
        self._ev: Optional[torch.cuda.Event] = None

    # ---- numpy views
    @property
    def _map(self) -> np.ndarray:
        self._eng.check_fill(0)
        return self._obst[0].cpu().numpy().astype(bool)

    @property
    def _navigable_map(self) -> np.ndarray:
        self._eng.check_fill(0)
        return self._nav[0].cpu().numpy().astype(np.int64)  # the reference's is int64 0/1 (:105-109)

    @property
    def explored_area(self) -> np.ndarray:
        return self._explored[0].cpu().numpy().astype(bool)

    # frontier waypoints are produced on the device; the host copy is fetched (and the stream synchronised) on access
    @property
    def _frontiers_px(self) -> np.ndarray:
        if self._front_cache is None:
            self._eng.check_fill(0)
            self._front_cache = self._eng.frontiers_px(0)
        return self._front_cache

    @property
    def frontiers(self) -> np.ndarray:
        px = self._frontiers_px
        return np.array([]) if len(px) == 0 else self._px_to_xy(px)      # obstacle_map.py:149-153

    def explored_device(self) -> torch.Tensor:
        return self._explored

    def reset(self) -> None:  # obstacle_map.py:48-53
        super().reset()
        self._eng.reset()
        self._front_cache = np.array([])

    def _upload(self, depth: Optional[np.ndarray], tf: np.ndarray) -> None:
        if self._pin_tf is None:
            self._pin_tf = torch.empty((1, 16), dtype=torch.float64).pin_memory()
            self._ev = torch.cuda.Event()
        else:
            self._ev.synchronize()
        self._pin_tf.numpy()[0, :] = np.asarray(tf, dtype=np.float64).reshape(16)
        if depth is not None:
            h, w = depth.shape
            if self._pin is None or self._pin.shape != (1, h, w):
                self._pin = torch.empty((1, h, w), dtype=torch.float32).pin_memory()
                self._dev_depth = torch.empty((1, h, w), dtype=torch.float32, device=self.device)
            direct = None
            if isinstance(depth, np.ndarray) and depth.dtype == np.float32 and depth.flags.c_contiguous:
                t = torch.from_numpy(depth)
                # page-locked caller frame and an idle stream: DMA straight from it and wait (the caller may reuse the frame);
                # with work queued ahead the wait would stall the host, so the frame is staged instead
                if t.is_pinned() and torch.cuda.current_stream(self.device).query():
                    direct = t
            if direct is None:
                self._pin[0].numpy()[...] = depth
            self._dev_depth.copy_(self._pin if direct is None else direct[None], non_blocking=True)
            self._dev_tf.copy_(self._pin_tf, non_blocking=True)
            self._ev.record()
            if direct is not None:
                self._ev.synchronize()
            return
        self._dev_tf.copy_(self._pin_tf, non_blocking=True)
        self._ev.record()

    def update_map(self, depth: Union[np.ndarray, Any], tf_camera_to_episodic: np.ndarray, min_depth: float,
                   max_depth: float, fx: float, fy: float, topdown_fov: float, explore: bool = True,
                   update_obstacles: bool = True) -> None:
        """obstacle_map.py:55-153."""
        tf = np.asarray(tf_camera_to_episodic, dtype=np.float64)
        with torch.cuda.device(self.device):
            if update_obstacles:
                if depth.ndim == 3:
                    depth = depth.squeeze(2)
                self._upload(depth, tf)
            elif explore:
                self._upload(None, tf)
            else:
                return
            self._eng.update(self._dev_depth if update_obstacles else None, tf[None], self._dev_tf, min_depth, max_depth, fx, fy, topdown_fov,
                             explore=explore, update_obstacles=update_obstacles)
            if explore:
                self._front_cache = None
            if update_obstacles:
                # numpy raises IndexError synchronously (:101); the caller turns it into STOP
                # (base_objectnav_policy.py:157-162).  Only pay for the sync near the border.
                cx, cy = tf[0, 3], tf[1, 3]
                margin = (self._eng._last_half + 2) / self.pixels_per_meter
                lim = self.size / 2 / self.pixels_per_meter
                if abs(cx) + margin >= lim or abs(cy) + margin >= lim:
                    if self._eng.index_error(0):
                        raise IndexError("obstacle cell index out of bounds for the map")

    def visualize_device(self) -> torch.Tensor:
        """obstacle_map.py:171-193 on the device: [G, G, 3] uint8 BGR tensor with the frontier circles and the trajectory."""
        recs = _render.trajectory_records(self._camera_positions, self._last_camera_yaw, self.pixels_per_meter, self._episode_pixel_origin)
        return self._eng.render(padding_color=self.radius_padding_color, draw_lists=[recs])[0]

    def visualize(self) -> np.ndarray:
        """obstacle_map.py:171-193 as a host [G, G, 3] uint8 array."""
        self._eng.check_fill(0)
        if int(self._eng.ex_status[0].item()) != 0:
            raise _lib.VlfmError("explore: a device scratch buffer overflowed (too many contours / points)")
        return self.visualize_device().cpu().numpy()
