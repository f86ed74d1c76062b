"""GPU value map behind the reference's ``ValueMap`` class surface.

Reference: vlfm/mapping/value_map.py (class :33, update_map :100, sort_waypoints :146,
reset :96).  State lives in HBM (``conf [B,G,G] f32``, ``value [B,G,G,C] f32``); the
per-step work is two CUDA launches through the C-ABI (csrc/value_map.cu).  Host-side
work is argument marshalling only; numpy views of the grids are produced lazily
(``_map`` / ``_value_map`` properties synchronise and copy device -> host).  ``visualize`` renders on the device
(csrc/render.cu, mapping/render.py).
"""
from __future__ import annotations

import math
import os
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .. import _lib
from . import render as _render
from .base_map import BaseMap

MIN_CONFIDENCE = 0.25  # value_map.py:40
DECISION_THRESHOLD = 0.35  # value_map.py:41

_TEMPLATES: Dict[Tuple[float, float, int, str], torch.Tensor] = {}
_TANS: Dict[Tuple[float, int, str], torch.Tensor] = {}
_DISCS: Dict[Tuple[int, str], torch.Tensor] = {}


def build_cone_template(fov: float, max_depth: float, ppm: int, device: torch.device) -> torch.Tensor:
    """Confidence cone (value_map.py:321-355): filled +-fov/2 sector (cv2.ellipse's rasterisation rules) times the cos^2
    falloff remapped to [0.25, 1], float32 -- built on the device by ``vlfm_value_cone_template``.  Configuration-time
    constant per (fov, max_depth, ppm), cached in HBM like the reference's class-level ``_confidence_masks``."""
    half = int(max_depth * ppm)
    side = 2 * half + 1
    out = torch.empty((side, side), dtype=torch.float32, device=device)
    nbytes = side * side + 8 * side * ((side + 31) // 32) + 2304
    scratch = torch.empty((nbytes + 3) // 4, dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        rc = _lib.load().vlfm_value_cone_template(float(fov), float(max_depth), int(ppm), MIN_CONFIDENCE, _lib.ptr(out), _lib.ptr(scratch),
                                                  scratch.numel() * 4, _lib.stream_ptr())
    _lib.check(rc, "vlfm_value_cone_template")
    return out


def _template(fov: float, max_depth: float, ppm: int, device: torch.device) -> torch.Tensor:
    key = (float(fov), float(max_depth), int(ppm), str(device))
    if key not in _TEMPLATES:
        _TEMPLATES[key] = build_cone_template(fov, max_depth, ppm, torch.device(device))
    return _TEMPLATES[key]


def _tan_table(fov: float, width: int, device: torch.device) -> torch.Tensor:
    key = (float(fov), int(width), str(device))
    if key not in _TANS:  # value_map.py:237,242
        _TANS[key] = torch.from_numpy(np.tan(np.linspace(-fov / 2, fov / 2, width))).to(device).contiguous()
    return _TANS[key]


def _disc(radius: int, device: torch.device) -> torch.Tensor:
    key = (int(radius), str(device))
    if key not in _DISCS:  # img_utils.py:247-255
        import cv2

        d = 2 * radius + 1
        m = cv2.circle(np.zeros((d, d), np.uint8), (radius, radius), radius, 255, -1)
        _DISCS[key] = torch.from_numpy(m).to(device).contiguous()
    return _DISCS[key]


def max_channels(i: np.ndarray) -> np.ndarray:
    """ValueMap.visualize's default reduce_fn (value_map.py:192); passing this function keeps the reduction on the device."""
    return np.max(i, axis=-1)


def fusion_code(use_max_confidence: bool, fusion_type: str) -> int:
    if fusion_type == "replace":
        return _lib.FUSE_REPLACE
    code = _lib.FUSE_MAX_CONFIDENCE if use_max_confidence else _lib.FUSE_WEIGHTED
    if fusion_type == "equal_weighting":
        code |= _lib.FUSE_EQUAL
    else:
        assert fusion_type == "default", f"Unknown fusion type {fusion_type}"
    return code


class ValueMapBatch:
    """B environments' value maps in one set of tensors; one C-ABI call per step."""

    def __init__(self, batch: int, value_channels: int, size: int = 1000, pixels_per_meter: int = 20,
                 use_max_confidence: bool = True, fusion_type: str = "default",
                 device: Union[str, torch.device, None] = None) -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else "cuda")
        self.batch, self.channels, self.size, self.ppm = batch, value_channels, size, pixels_per_meter
        self.fusion = fusion_code(use_max_confidence, fusion_type)
        self.conf = torch.zeros((batch, size, size), dtype=torch.float32, device=self.device)
        self.value = torch.zeros((batch, size, size, value_channels), dtype=torch.float32, device=self.device)
        self.status = torch.zeros((batch,), dtype=torch.int32, device=self.device)   # VLFM_ST_* flags per grid SLOT, like conf / value
        self._ws: Optional[torch.Tensor] = None
        self._ws_key: Optional[Tuple[int, int, int]] = None
        self.rows_per_tile = 0
        # The reference's value grid becomes float64 in the first fuse of a weighted map (value_map.py:423) and stays so
        # through reset(); before that fuse it is all zero, which renders white in either dtype.  Frames of such maps are
        # therefore normalised in float64 (an exact upcast of the float32 grid), all others in float32.
        self.ref_float64 = self.fusion in (_lib.FUSE_WEIGHTED, _lib.FUSE_WEIGHTED | _lib.FUSE_EQUAL)
        self._render_ws = _render._Workspace()
        self._draw: Optional[_render.DrawLists] = None

    def _params(self, h: int, w: int, min_depth: float, max_depth: float) -> "_lib.ValueParams":
        side = 2 * int(max_depth * self.ppm) + 1
        return _lib.ValueParams(h, w, self.size, self.channels, side, self.ppm,
                                float(np.float32(max_depth - min_depth)), float(np.float32(min_depth)),
                                float(np.float32(DECISION_THRESHOLD)), self.fusion, self.rows_per_tile)

    def _workspace(self, p: "_lib.ValueParams", n: int) -> torch.Tensor:
        key = (p.H, p.W, p.R)
        if self._ws is None or self._ws_key != key:
            import ctypes

            nbytes = ctypes.c_size_t(0)
            _lib.check(self.lib.vlfm_value_workspace_bytes(ctypes.byref(p), self.batch, ctypes.byref(nbytes)), "workspace")
            self._ws = torch.zeros((max(nbytes.value, 16) + 3) // 4, dtype=torch.int32, device=self.device)
            self._ws_key = key
        return self._ws

    def update(self, values: torch.Tensor, depth: torch.Tensor, tf: torch.Tensor, min_depth: float,
               max_depth: float, fov: float, slots: Optional[torch.Tensor] = None,
               explored: Optional[torch.Tensor] = None) -> None:
        """values [n,C] f64, depth [n,H,W] f32, tf [n,4,4] f64 -- device tensors."""
        import ctypes

        n, h, w = depth.shape
        assert depth.dtype == torch.float32 and depth.is_contiguous() and depth.device.type == "cuda"
        assert tf.dtype == torch.float64 and tf.is_contiguous() and values.dtype == torch.float64 and values.is_contiguous()
        assert n <= self.batch
        p = self._params(h, w, min_depth, max_depth)
        ws = self._workspace(p, n)
        tmpl = _template(fov, max_depth, self.ppm, self.device)
        tan = _tan_table(fov, w, self.device)
        with torch.cuda.device(self.device):
            rc = self.lib.vlfm_value_update(ctypes.byref(p), n, _lib.ptr(slots), _lib.ptr(self.conf), _lib.ptr(self.value),
                                            _lib.ptr(depth), _lib.ptr(tf), _lib.ptr(values), _lib.ptr(tmpl), _lib.ptr(tan),
                                            _lib.ptr(explored), _lib.ptr(ws), _lib.ptr(self.status), _lib.stream_ptr())
        _lib.check(rc, "vlfm_value_update")

    def mask_unexplored(self, explored: torch.Tensor, slots: Optional[torch.Tensor] = None, n: Optional[int] = None) -> None:
        n = self.batch if n is None else n
        with torch.cuda.device(self.device):
            rc = self.lib.vlfm_value_mask_unexplored(self.size, self.channels, n, _lib.ptr(slots), _lib.ptr(self.conf),
                                                     _lib.ptr(self.value), _lib.ptr(explored), _lib.stream_ptr())
        _lib.check(rc, "vlfm_value_mask_unexplored")

    def disc_median(self, slot: int, points_rc: np.ndarray, radius: int) -> np.ndarray:
        """[(row, col)] -> [npoints, C] medians of non-zero cells in the disc (-1 if none), as np.median computes them on the
        reference's grid: an even count's midpoint in float64 for weighted maps, in float32 otherwise (``ref_float64``)."""
        pts = torch.from_numpy(np.ascontiguousarray(points_rc, dtype=np.int32)).to(self.device)
        out = torch.empty((len(points_rc), self.channels), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            rc = self.lib.vlfm_value_disc_median(self.size, self.channels, slot, _lib.ptr(self.value), _lib.ptr(pts),
                                                 len(points_rc), radius, int(self.ref_float64), _lib.ptr(_disc(radius, self.device)),
                                                 _lib.ptr(out), _lib.stream_ptr())
        _lib.check(rc, "vlfm_value_disc_median")
        return out.cpu().numpy()

    def disc_median_batch(self, points_srl: np.ndarray, radius: int) -> np.ndarray:
        """[(slot, row, col)] over any number of environments -> [npoints, C] medians with one launch and one read-back."""
        if len(points_srl) == 0:
            return np.zeros((0, self.channels))
        pts = torch.from_numpy(np.ascontiguousarray(points_srl, dtype=np.int32)).to(self.device)
        out = torch.empty((len(points_srl), self.channels), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            rc = self.lib.vlfm_value_disc_median_batch(self.size, self.channels, _lib.ptr(self.value), _lib.ptr(pts), len(points_srl), radius,
                                                       int(self.ref_float64), _lib.ptr(_disc(radius, self.device)), _lib.ptr(out),
                                                       _lib.stream_ptr())
        _lib.check(rc, "vlfm_value_disc_median_batch")
        return out.cpu().numpy()

    def render(self, slots: Optional[torch.Tensor] = None, reduced: Optional[torch.Tensor] = None, explored: Optional[torch.Tensor] = None,
               draw_lists: Optional[Sequence[Sequence[Sequence[int]]]] = None) -> torch.Tensor:
        """ValueMap.visualize frames of n environments: [n, G, G, 3] uint8 BGR on the device.  ``slots`` (int32 [n], default
        0..batch-1) picks the grids; ``reduced`` [n, G, G] float32 / float64 replaces the default reduction value.amax(-1);
        ``explored`` [nslots, G, G] uint8 (read at the same slots) zeroes unexplored cells; ``draw_lists[i]`` holds the draw
        records (mapping/render.py) painted onto frame i in order."""
        if reduced is None:
            v = self.value if slots is None else self.value[slots.long()]
            reduced = v.amax(-1)
            if self.ref_float64:
                reduced = reduced.double()
        reduced = reduced.contiguous()
        frames = _render.value_frames(reduced, explored, slots, self._render_ws)
        if draw_lists is not None:
            if self._draw is None:
                self._draw = _render.DrawLists(self.device)
            self._draw.draw(frames, draw_lists)
        return frames

    def reset(self, slot: Optional[int] = None) -> None:
        if slot is None:
            self.conf.zero_(); self.value.zero_(); self.status.zero_()
        else:
            self.conf[slot].zero_(); self.value[slot].zero_(); self.status[slot] = 0

    def waypoint_values(self, med: np.ndarray, reduce_fn: Optional[Callable]) -> List[Any]:
        """[npoints, C] disc medians -> the values the reference's sort_waypoints sorts (value_map.py:171-187): np.median's scalar
        type (float64 for weighted maps, float32 otherwise) or the int -1 of an empty disc, one per point when C == 1, else
        ``reduce_fn`` of the per-channel tuples.  The type matters: np.argsort is not stable, and the tie order it produces
        depends on the dtype of the array it sorts."""
        typ = np.float64 if self.ref_float64 else np.float32
        if self.channels == 1:
            return [typ(m[0]) if m[0] != -1 else -1 for m in med]
        assert reduce_fn is not None, "Must provide a reduction function when using multiple value channels."
        return reduce_fn([tuple(typ(v) if v != -1 else -1 for v in m) for m in med])


def frontier_values(omb: Any, vmb: ValueMapBatch, n: int, radius_m: float, reduce_fn: Optional[Callable] = None
                    ) -> List[Tuple[np.ndarray, List[Any]]]:
    """ITMPolicy._sort_frontiers_by_value (itm_policy.py:263-266) for slots 0..n-1 of an ObstacleMapBatch ``omb`` and a ValueMapBatch
    ``vmb``: each environment's frontiers in metres (ObstacleMap.frontiers) sorted and scored exactly as
    ``ValueMap.sort_waypoints(frontiers, radius_m)`` does it -- metres to cells with int() truncation (value_map.py:163-170), the
    disc median of every frontier of every environment in one launch and one read-back, np.argsort of the negated values.
    Returns [(frontiers [F, 2] sorted, values)] per environment.

    A zero-length frontier piece has a NaN midpoint (its arc-length midpoint is 0/0).  The reference's int(NaN) raises ValueError
    there, which would end the step of every environment in the batch; here such a frontier gets the value -1, the value of a
    frontier with no observed cell in its disc, and so sorts behind every frontier that has a value.  A finite point off the grid
    raises AssertionError, as pixel_value_within_radius does (img_utils.py:43)."""
    g, ppm = vmb.size, vmb.ppm
    assert omb.size == g and omb.ppm == ppm
    fronts = omb.all_frontiers_px(n)
    counts = [len(px) for px in fronts]
    out: List[Tuple[np.ndarray, List[Any]]] = [(np.array([]), []) for _ in range(n)]
    if sum(counts) == 0:
        return out
    xy = omb.px_to_xy(np.concatenate([px for px in fronts if len(px)]))      # every environment's frontiers, in metres
    env = np.repeat(np.arange(n), counts)
    ok = ~np.isnan(xy).any(axis=1)
    row = g - (np.trunc(-xy[ok, 0] * ppm) + g // 2)          # size - (int(-x * ppm) + origin[0])
    col = np.trunc(-xy[ok, 1] * ppm) + g // 2                # int(-y * ppm) + origin[1]
    assert ((row >= 0) & (row < g) & (col >= 0) & (col < g)).all(), "Pixel location is outside the image."
    med = np.full((len(xy), vmb.channels), -1.0)
    if ok.any():
        med[ok] = vmb.disc_median_batch(np.stack([env[ok], row, col], axis=1).astype(np.int64), int(radius_m * ppm))
    k = 0
    for e, c in enumerate(counts):
        if c:
            values = vmb.waypoint_values(med[k:k + c], reduce_fn)
            order = np.argsort([-v for v in values])
            out[e] = (xy[k:k + c][order], [values[i] for i in order])
        k += c
    return out


class ValueMap(BaseMap):
    """Drop-in for ``vlfm.mapping.value_map.ValueMap`` (same constructor, methods and
    attributes).  Differences, all documented in DESIGN.md: grids are float32 in HBM
    (the reference's value grid silently becomes float64 after the first weighted fuse,
    value_map.py:423), ``pixels_per_meter`` is honoured, update_map is asynchronous."""

    _min_confidence: float = MIN_CONFIDENCE
    _decision_threshold: float = DECISION_THRESHOLD

    def __init__(self, value_channels: int, size: int = 1000, use_max_confidence: bool = True,
                 fusion_type: str = "default", obstacle_map: Optional[Any] = None,
                 pixels_per_meter: int = 20, device: Union[str, torch.device, None] = None) -> None:
        super().__init__(size, pixels_per_meter)
        self._value_channels = value_channels
        self._use_max_confidence = use_max_confidence
        self._fusion_type = fusion_type
        self._obstacle_map = obstacle_map
        if obstacle_map is not None:  # value_map.py:70-72
            assert obstacle_map.pixels_per_meter == self.pixels_per_meter
            assert obstacle_map.size == self.size
        if os.environ.get("MAP_FUSION_TYPE", "") != "":  # value_map.py:74-75
            self._fusion_type = os.environ["MAP_FUSION_TYPE"]
        self._eng = ValueMapBatch(1, value_channels, size, pixels_per_meter, use_max_confidence, self._fusion_type, device)
        self.device = self._eng.device
        self._stage: List[Optional[Tuple[torch.Tensor, torch.Tensor, torch.cuda.Event]]] = [None, None]
        self._stage_i = 0
        self._dev_depth: Optional[torch.Tensor] = None
        self._dev_small: Optional[torch.Tensor] = None

    # ---- lazily materialised numpy views (device -> host)
    @property
    def _map(self) -> np.ndarray:
        self._raise_pending()
        return self._eng.conf[0].cpu().numpy()

    @property
    def _value_map(self) -> np.ndarray:
        self._raise_pending()
        return self._eng.value[0].cpu().numpy()

    def _raise_pending(self) -> None:
        st = int(self._eng.status[0].item())
        if st & _lib.ST_CAMERA_OFF_GRID:
            self._eng.status.zero_()
            raise AssertionError("Pixel location is outside the image.")  # img_utils.py:43

    def reset(self) -> None:  # value_map.py:96-98
        super().reset()
        self._eng.reset()

    def _staging(self, h: int, w: int):
        i = self._stage_i
        self._stage_i ^= 1
        slot = self._stage[i]
        if slot is None or slot[0].shape != (1, h, w):
            slot = (torch.empty((1, h, w), dtype=torch.float32).pin_memory(),
                    torch.empty((16 + self._value_channels,), dtype=torch.float64).pin_memory(),
                    torch.cuda.Event())
            self._stage[i] = slot
        else:
            slot[2].synchronize()  # the previous H2D from this slot has been consumed
        if self._dev_depth is None or self._dev_depth.shape != (1, h, w):
            self._dev_depth = torch.empty((1, h, w), dtype=torch.float32, device=self.device)
            self._dev_small = torch.empty((16 + self._value_channels,), dtype=torch.float64, device=self.device)
        return slot

    def update_map(self, values: np.ndarray, depth: np.ndarray, tf_camera_to_episodic: np.ndarray,
                   min_depth: float, max_depth: float, fov: float) -> None:
        """value_map.py:100-128.  Host buffers in; H2D copies + 2 kernel launches; async."""
        assert len(values) == self._value_channels, (
            f"Incorrect number of values given ({len(values)}). Expected {self._value_channels}.")
        if depth.ndim == 3:
            depth = depth.squeeze(2)
        ppm = self.pixels_per_meter
        cam = tf_camera_to_episodic[:2, 3] / tf_camera_to_episodic[3, 3]
        row = int(cam[0] * ppm) + int(self._episode_pixel_origin[0])
        col = int(-cam[1] * ppm) + int(self._episode_pixel_origin[1])
        assert 0 <= row < self.size and 0 <= col < self.size, "Pixel location is outside the image."
        h, w = depth.shape
        pin_d, pin_s, ev = self._staging(h, w)
        direct = None
        if isinstance(depth, np.ndarray) and depth.dtype == np.float32 and depth.flags.c_contiguous:
            t = torch.from_numpy(depth)
            # page-locked caller buffer and an idle stream: DMA straight from it and wait (the caller may reuse the buffer);
            # with work queued ahead the wait would stall the host, so the frame is staged instead
            if t.is_pinned() and torch.cuda.current_stream(self.device).query():
                direct = t
        if direct is None:
            pin_d[0].numpy()[...] = depth  # converts to float32 if needed
        s = pin_s.numpy()
        s[:16] = np.asarray(tf_camera_to_episodic, dtype=np.float64).reshape(16)
        s[16:] = np.asarray(values, dtype=np.float64)
        with torch.cuda.device(self.device):
            self._dev_depth.copy_(pin_d if direct is None else direct[None], non_blocking=True)
            self._dev_small.copy_(pin_s, non_blocking=True)
            ev.record()
            if direct is not None:
                ev.synchronize()
            if self._obstacle_map is not None:  # value_map.py:365-375
                exp = self._obstacle_map.explored_device()
                self._eng.mask_unexplored(exp)
            else:
                exp = None
            self._eng.update(self._dev_small[16:].view(1, -1), self._dev_depth, self._dev_small[:16].view(1, 4, 4),
                             min_depth, max_depth, fov, explored=exp)

    def sort_waypoints(self, waypoints: np.ndarray, radius: float, reduce_fn: Optional[Callable] = None
                       ) -> Tuple[np.ndarray, List[float]]:
        """value_map.py:146-187; the per-waypoint disc median runs on the GPU."""
        ppm = self.pixels_per_meter
        radius_px = int(radius * ppm)
        pts = []
        for x, y in waypoints:
            px = int(-x * ppm) + int(self._episode_pixel_origin[0])
            py = int(-y * ppm) + int(self._episode_pixel_origin[1])
            rc = (self.size - px, py)
            assert 0 <= rc[0] < self.size and 0 <= rc[1] < self.size, "Pixel location is outside the image."
            pts.append(rc)
        if len(pts) == 0:
            return np.array([]), []
        med = self._eng.disc_median(0, np.array(pts), radius_px)
        values = self._eng.waypoint_values(med, reduce_fn)
        order = np.argsort([-v for v in values])
        return np.array([waypoints[i] for i in order]), [values[i] for i in order]

    def visualize_device(self, markers: Optional[List[Tuple[np.ndarray, Dict[str, Any]]]] = None,
                         reduce_fn: Callable = max_channels, obstacle_map: Optional[Any] = None) -> torch.Tensor:
        """value_map.py:189-219 on the device: [G, G, 3] uint8 BGR tensor (csrc/render.cu).  The default reduce_fn reduces
        on the device; any other callable runs on the host, as in the reference, on the value grid in the dtype the
        reference's grid has (``ValueMapBatch.ref_float64``), and its result is uploaded."""
        reduced = None
        if reduce_fn is not max_channels:
            grid = self._value_map
            if self._eng.ref_float64:
                grid = grid.astype(np.float64)
            red = np.asarray(reduce_fn(grid))
            if red.dtype not in (np.float32, np.float64):
                red = red.astype(np.float64)
            reduced = torch.from_numpy(np.ascontiguousarray(red)).to(self.device)[None]
        recs: List[List[int]] = []
        if len(self._camera_positions) > 0:           # no trajectory: neither the agent nor the markers (:208-217)
            recs = _render.trajectory_records(self._camera_positions, self._last_camera_yaw, self.pixels_per_meter,
                                              self._episode_pixel_origin)
            recs += _render.marker_records(markers, self.pixels_per_meter, self._episode_pixel_origin)
        explored = obstacle_map.explored_device() if obstacle_map is not None else None
        return self._eng.render(reduced=reduced, explored=explored, draw_lists=[recs])[0]

    def visualize(self, markers: Optional[List[Tuple[np.ndarray, Dict[str, Any]]]] = None, reduce_fn: Callable = max_channels,
                  obstacle_map: Optional[Any] = None) -> np.ndarray:
        """value_map.py:189-219: the inferno frame with the trajectory and the markers, as a host [G, G, 3] uint8 array."""
        return self.visualize_device(markers, reduce_fn, obstacle_map).cpu().numpy()
