"""B environments' obstacle / navigable / explored grids in one set of tensors; one launch SEQUENCE per step for all of them.

Reference: vlfm/mapping/obstacle_map.py:55-169 (``ObstacleMap.update_map`` + ``_get_frontiers``), one instance per environment
in the reference (base_objectnav_policy.py:86-92); the environments are independent (SURVEY.md section 8e), so a vectorised
caller updates them together: fill_small_holes (10 launches), obstacle scatter + dilate (2), explore half + frontiers (~60) --
for the whole batch.  ``ObstacleMap`` (obstacle_map.py here) is the batch-1 instance behind the reference's class surface.

Host-side state per environment: whether the navigable map exists yet, and the COVER rectangle -- the union of every
obstacle-update window and every fog-of-war window of the episode -- from which the S frame of the explore step is derived
(csrc/explore.cu, include/vlfm_b200.h ``VlfmExploreEnv.frame``).
"""
from __future__ import annotations

import ctypes
import math
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .. import _lib
from ..utils.cuda_graph import GraphCache, default_use_graph
from . import render as _render
from . import sframe as _sf

MAX_FRONTIERS = 4096


def wrap_heading(h: float) -> float:
    return (h + np.pi) % (2 * np.pi) - np.pi


class ObstacleMapBatch:
    def __init__(self, batch: int, min_height: float, max_height: float, agent_radius: float, area_thresh: float = 3.0,
                 hole_area_thresh: int = 100000, size: int = 1000, pixels_per_meter: int = 20,
                 device: Union[str, torch.device, None] = None) -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else "cuda")
        self.batch, self.size, self.ppm = batch, size, pixels_per_meter
        dev = self.device
        self.obst = torch.zeros((batch, size, size), dtype=torch.uint8, device=dev)
        self.nav = torch.zeros((batch, size, size), dtype=torch.uint8, device=dev)
        self.explored = torch.zeros((batch, size, size), dtype=torch.uint8, device=dev)
        self.status = torch.zeros((batch,), dtype=torch.int32, device=dev)          # scatter out of bounds (IndexError in the reference)
        self.min_height, self.max_height = min_height, max_height
        self.area_thresh_px = area_thresh * (pixels_per_meter ** 2)                 # obstacle_map.py:41
        self.hole_area_thresh = hole_area_thresh
        k = pixels_per_meter * agent_radius * 2                                     # :43-46
        self.kernel = int(k) + (int(k) % 2 == 0)
        self.nav_valid = [False] * batch
        self.cover: List[Optional[Tuple[int, int, int, int]]] = [None] * batch
        # explore outputs, indexed by SLOT
        self.frontiers = torch.zeros((batch, MAX_FRONTIERS, 2), dtype=torch.float64, device=dev)
        self.count = torch.zeros((batch,), dtype=torch.int32, device=dev)
        self.ex_status = torch.zeros((batch,), dtype=torch.int32, device=dev)
        self._call_front = torch.zeros((batch, MAX_FRONTIERS, 2), dtype=torch.float64, device=dev)   # call-order staging
        self._call_count = torch.zeros((batch,), dtype=torch.int32, device=dev)
        self._call_status = torch.zeros((batch,), dtype=torch.int32, device=dev)
        n = ctypes.c_size_t(0)
        _lib.check(self.lib.vlfm_explore_batch_workspace_bytes(size, batch, ctypes.byref(n)), "vlfm_explore_batch_workspace_bytes")
        self._ex_ws = torch.zeros((n.value + 3) // 4, dtype=torch.int32, device=dev)
        rec = int(self.lib.vlfm_explore_env_record_bytes())
        self._pin = [torch.zeros(rec * batch, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self._pin_ev = [torch.cuda.Event(), torch.cuda.Event()]
        self._pin_used = [False, False]
        self._pin_i = 0
        self._envs = (_lib.ExploreEnv * batch)()
        self._fill: Optional[torch.Tensor] = None
        self._fill_ws: Optional[torch.Tensor] = None
        self._fill_status = torch.zeros((batch,), dtype=torch.int32, device=dev)
        self._slot_ids = torch.arange(batch, dtype=torch.int32, device=dev)
        # CUDA graph of the whole update (hole fill + scatter + dilate + explore): the launch geometry of every C-ABI call depends on
        # the batch size only and the per-environment pose scalars travel in page-locked records, so the second call with the same
        # buffers and parameters captures the sequence and later ones replay it (~75 launches -> one graph launch)
        self.use_graph = default_use_graph()
        self.graphs = GraphCache(max_keys=4)
        self._rec_pin = torch.zeros(rec * batch, dtype=torch.uint8).pin_memory()      # explore records read by the captured upload node
        self._rec_ev = torch.cuda.Event()
        self._rec_used = False
        self._draw: Optional[_render.DrawLists] = None

    # ---------------------------------------------------------------- helpers ----
    def _pinned(self) -> torch.Tensor:
        i = self._pin_i
        self._pin_i ^= 1
        if self._pin_used[i]:
            self._pin_ev[i].synchronize()       # the copy issued from this buffer two calls ago has executed
        self._pin_used[i] = True
        self._cur_pin = i
        return self._pin[i]

    def _pinned_done(self) -> None:
        self._pin_ev[self._cur_pin].record()

    def xy_to_px(self, xy: np.ndarray) -> np.ndarray:                              # base_map.py:35-46
        px = np.rint(xy[:, ::-1] * self.ppm) + np.array([self.size // 2, self.size // 2])
        px[:, 0] = self.size - px[:, 0]
        return px.astype(int)

    def _cover_add(self, slot: int, r: Tuple[int, int, int, int]) -> None:
        self.cover[slot] = _sf.cover_add(self.cover[slot], r, self.size)

    def _frame(self, slot: int) -> Tuple[int, int, int, int]:
        """S frame of the explore step (mapping/sframe.py): cover + margin, sides snapped to the grid edge when closer than D to it."""
        return _sf.sframe(self.cover[slot], self.size, self.area_thresh_px)

    # ------------------------------------------------------------------ update ----
    def _fill_envs(self, n: int, slots, agents, tf_host, max_depth: float, topdown_fov: float) -> None:
        ppm = self.ppm
        L = int(max_depth * ppm)
        envs = self._envs
        for i, s in enumerate(slots):
            col, row = int(agents[i][0]), int(agents[i][1])
            self._cover_add(s, _sf.fog_window(col, row, L))
            tf = tf_host[i]
            yaw = float(np.arctan2(tf[1, 0], tf[0, 0]))
            e = envs[i]
            e.slot, e.agent_col, e.agent_row = s, col, row
            fr = self._frame(s)
            e.frame[0], e.frame[1], e.frame[2], e.frame[3] = fr
            e.heading_deg = float(np.rad2deg(wrap_heading(yaw + np.pi / 2)))     # current_angle = -yaw (:121)
            e.fov_deg = float(np.rad2deg(topdown_fov))
            e.max_line_len = float(max_depth * ppm)
            e.area_thresh_px = float(self.area_thresh_px)

    def _device_sequence(self, n: int, depth, tf_dev, p, slot_t, explore: bool, update_obstacles: bool, pins: Optional[Tuple[torch.Tensor, ...]]) -> None:
        """the launches of one update on the current stream: eager, or for a graph with ``pins`` = its (explore, hole-fill) record buffers"""
        st = _lib.stream_ptr()
        g = self.size
        if update_obstacles:
            h, w = int(depth.shape[1]), int(depth.shape[2])
            fill = None
            if self.hole_area_thresh != -1:          # fill_small_holes (img_utils.py:361-390) on the device
                pin = self._pinned() if pins is None else pins[1]
                rc = self.lib.vlfm_fill_small_holes_batch(_lib.ptr(depth), h, w, n, float(self.hole_area_thresh), _lib.ptr(self._fill),
                                                          _lib.ptr(self._fill_ws), self._fill_ws.numel() * 4, _lib.ptr(self._fill_status),
                                                          pin.data_ptr(), pin.numel(), st)
                if pins is None:
                    self._pinned_done()
                _lib.check(rc, "vlfm_fill_small_holes_batch")
                fill = self._fill
            rc = self.lib.vlfm_obstacle_update(ctypes.byref(p), n, _lib.ptr(slot_t), _lib.ptr(self.obst), _lib.ptr(self.nav),
                                               _lib.ptr(depth), _lib.ptr(tf_dev), _lib.ptr(fill), _lib.ptr(self.status), st)
            _lib.check(rc, "vlfm_obstacle_update")
        if not explore:
            return
        if pins is None:
            pin = self._pinned()
            rc = self.lib.vlfm_explore_update_batch(g, n, self._envs, _lib.ptr(self.explored), _lib.ptr(self.nav), _lib.ptr(self._call_front),
                                                    _lib.ptr(self._call_count), _lib.ptr(self._call_status), _lib.ptr(self._ex_ws),
                                                    self._ex_ws.numel() * 4, pin.data_ptr(), pin.numel(), st)
            self._pinned_done()
            _lib.check(rc, "vlfm_explore_update_batch")
        else:                                        # records already prepared in pins[0] by the caller
            _lib.check(self.lib.vlfm_explore_launch_batch(g, n, _lib.ptr(self._ex_ws), pins[0].data_ptr(), st), "vlfm_explore_launch_batch")
        if slot_t is None:
            self.frontiers[:n].copy_(self._call_front[:n]); self.count[:n].copy_(self._call_count[:n]); self.ex_status[:n].copy_(self._call_status[:n])
        else:
            idx = slot_t.long()
            self.frontiers[idx] = self._call_front[:n]; self.count[idx] = self._call_count[:n]; self.ex_status[idx] = self._call_status[:n]

    def update(self, depth: Optional[torch.Tensor], tf_host: np.ndarray, tf_dev: torch.Tensor, min_depth: float, max_depth: float,
               fx: float, fy: float, topdown_fov: float, slots: Optional[Sequence[int]] = None, explore: bool = True,
               update_obstacles: bool = True) -> None:
        """depth [n,H,W] float32 (device) or None, tf_host [n,4,4] float64 (numpy: the pose scalars of the explore half are
        derived on the host exactly as the reference derives them), tf_dev [n,16] float64 (device, read by the obstacle
        kernels).  ``slots``: grid index of each row (default 0..n-1).  Asynchronous; IndexError conditions are polled by
        ``index_error``."""
        n = len(tf_host)
        slots = list(range(n)) if slots is None else [int(s) for s in slots]
        assert n <= self.batch and len(slots) == n
        g, ppm = self.size, self.ppm
        agents = self.xy_to_px(np.asarray(tf_host, dtype=np.float64)[:, :2, 3])     # (col, row) per env, obstacle_map.py:115-116
        identity = slots == list(range(n))
        with torch.cuda.device(self.device):
            slot_t = None if identity else torch.tensor(slots, dtype=torch.int32, device=self.device)
            p, first = None, False
            if update_obstacles:
                assert depth is not None and depth.dtype == torch.float32 and depth.is_contiguous() and depth.shape[0] == n
                h, w = int(depth.shape[1]), int(depth.shape[2])
                half = int(math.ceil(max_depth * ppm * math.sqrt(1.0 + (w / 2.0 / fx) ** 2))) + self.kernel // 2 + 2
                first = any(not self.nav_valid[s] for s in slots)
                p = _lib.ObstacleParams(h, w, g, ppm, float(np.float32(max_depth - min_depth)), float(np.float32(min_depth)),
                                        float(np.float32(max_depth)), float(fx), float(fy), float(self.min_height), float(self.max_height),
                                        self.kernel, 1 if first else 0, half)
                if self.hole_area_thresh != -1 and (self._fill is None or self._fill.shape[1:] != (h, w)):
                    nb = ctypes.c_size_t(0)
                    _lib.check(self.lib.vlfm_holes_batch_workspace_bytes(h, w, self.batch, ctypes.byref(nb)), "vlfm_holes_batch_workspace_bytes")
                    self._fill = torch.zeros((self.batch, h, w), dtype=torch.uint8, device=self.device)
                    self._fill_ws = torch.zeros((nb.value + 3) // 4, dtype=torch.int32, device=self.device)
                    self.graphs.clear()
                for i, s in enumerate(slots):
                    self._cover_add(s, _sf.obstacle_window(int(agents[i][0]), int(agents[i][1]), half, g))
                    self.nav_valid[s] = True
                self._last_half = half
            if explore:
                self._fill_envs(n, slots, agents, tf_host, max_depth, topdown_fov)
            if not (identity and explore and update_obstacles and not first):
                self._device_sequence(n, depth, tf_dev, p, slot_t, explore, update_obstacles, None)
                return
            key = (n, depth.data_ptr(), tf_dev.data_ptr(), tuple(depth.shape), float(min_depth), float(max_depth), float(fx), float(fy), float(topdown_fov))
            pins = None
            if self.graphs.will_replay(key, self.use_graph):
                if self._rec_used:
                    self._rec_ev.synchronize()           # the previous replay's record upload has executed
                rc = self.lib.vlfm_explore_prepare_batch(g, n, self._envs, _lib.ptr(self.explored), _lib.ptr(self.nav), _lib.ptr(self._call_front),
                                                         _lib.ptr(self._call_count), _lib.ptr(self._call_status), _lib.ptr(self._ex_ws),
                                                         self._ex_ws.numel() * 4, self._rec_pin.data_ptr(), self._rec_pin.numel())
                _lib.check(rc, "vlfm_explore_prepare_batch")
                # a graph uploads its hole-fill records, which hold its depth pointer, from a page-locked buffer of its own: the
                # capturing call allocates it and returns it, so it lives as long as the graph
                holes = None if key in self.graphs.captured else torch.zeros(self._pin[0].numel(), dtype=torch.uint8).pin_memory()
                pins = (self._rec_pin, holes)
            self.graphs(key, self.use_graph, lambda: (self._device_sequence(n, depth, tf_dev, p, None, True, True, pins), pins))
            if pins is not None:
                self._rec_ev.record()
                self._rec_used = True

    # ----------------------------------------------------------------- readback ----
    def check_fill(self, slot: int = 0) -> None:
        if self._fill is not None and int(self._fill_status.max().item()) != 0:     # rows of the last call, not slots: any flag counts
            self._fill_status.zero_()
            raise _lib.VlfmError("fill_small_holes: a device scratch buffer overflowed (too many contours in the depth image)")

    def index_error(self, slot: int) -> bool:
        if int(self.status[slot].item()) & _lib.ST_SCATTER_OOB:
            self.status[slot] = 0
            return True
        return False

    def frontiers_px(self, slot: int) -> np.ndarray:
        n = int(self.count[slot].item())
        if int(self.ex_status[slot].item()) != 0:
            raise _lib.VlfmError("explore: a device scratch buffer overflowed (too many contours / points)")
        if n == 0:
            return np.array([])
        return self.frontiers[slot, :n].cpu().numpy()

    def all_frontiers_px(self, n: Optional[int] = None) -> List[np.ndarray]:
        """frontier lists of slots 0..n-1 with ONE device->host transfer (what a vectorised policy needs every step)"""
        n = self.batch if n is None else n
        cnt = self.count[:n].cpu().numpy()
        if int(self.ex_status[:n].max().item()) != 0:
            raise _lib.VlfmError("explore: a device scratch buffer overflowed (too many contours / points)")
        m = int(cnt.max()) if n else 0
        if m == 0:
            return [np.array([]) for _ in range(n)]
        fr = self.frontiers[:n, :m].cpu().numpy()
        return [fr[i, : cnt[i]].copy() if cnt[i] else np.array([]) for i in range(n)]

    def render(self, slots: Optional[torch.Tensor] = None, padding_color: Sequence[int] = (100, 100, 100),
               draw_lists: Optional[Sequence[Sequence[Sequence[int]]]] = None) -> torch.Tensor:
        """ObstacleMap.visualize frames of n environments: [n, G, G, 3] uint8 BGR on the device.  ``slots`` (int32 [n],
        default 0..batch-1) picks the grids and frontier lists (read on the device, no host round trip);
        ``padding_color`` is the reference's ``radius_padding_color``; ``draw_lists[i]`` holds the draw records
        (mapping/render.py) painted onto frame i after the flip."""
        n = self.batch if slots is None else int(slots.shape[0])
        g = self.size
        pad = [int(c) for c in padding_color]
        out = torch.empty((n, g, g, 3), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            rc = self.lib.vlfm_render_obstacle(g, n, _lib.ptr(slots), _lib.ptr(self.obst), _lib.ptr(self.nav), _lib.ptr(self.explored),
                                               _lib.ptr(self.frontiers), _lib.ptr(self.count), MAX_FRONTIERS, pad[0], pad[1], pad[2],
                                               _lib.ptr(out), _lib.stream_ptr())
        _lib.check(rc, "vlfm_render_obstacle")
        if draw_lists is not None:
            if self._draw is None:
                self._draw = _render.DrawLists(self.device)
            self._draw.draw(out, draw_lists)
        return out

    def px_to_xy(self, px: np.ndarray) -> np.ndarray:                              # base_map.py:48-60
        q = px.copy()
        q[:, 0] = self.size - q[:, 0]
        return ((q - np.array([self.size // 2, self.size // 2])) / self.ppm)[:, ::-1]

    def reset(self, slot: Optional[int] = None) -> None:
        sl = slice(None) if slot is None else slot
        self.obst[sl].zero_(); self.nav[sl].zero_(); self.explored[sl].zero_()
        if slot is None:
            self.status.zero_(); self.count.zero_(); self.ex_status.zero_()
            self.nav_valid = [False] * self.batch
            self.cover = [None] * self.batch
        else:
            self.status[slot] = 0; self.count[slot] = 0; self.ex_status[slot] = 0
            self.nav_valid[slot] = False
            self.cover[slot] = None
