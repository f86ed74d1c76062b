"""Map frames for video on the GPU: the value / obstacle map renderings and the trajectory + marker overlay.

Reference: vlfm/mapping/value_map.py:189-219, vlfm/mapping/obstacle_map.py:171-193, vlfm/mapping/traj_visualizer.py.
The frames are produced by csrc/render.cu; this module holds what stays on the host: the inferno LUT, the trajectory style,
the pixel coordinates of the path, agent and markers (computed with the reference's own numpy expressions, so their dtype
flow is the reference's by construction) and the packing of the per-environment draw lists (int32 records, one page-locked
upload per call).
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib

# TrajectoryVisualizer defaults (traj_visualizer.py:14-18, 80-96)
PATH_COLOR = (0, 255, 0)
PATH_THICKNESS = 3
AGENT_RADIUS = 8
AGENT_COLOR = (255, 192, 15)
AGENT_LINE_LENGTH = 10
AGENT_LINE_THICKNESS = 3
AGENT_LINE_COLOR = (0, 0, 0)
SCALE_FACTOR = 1.0

MAX_THICKNESS = 16
MAX_RADIUS = 255
MAX_COORD = 1 << 24

_LUTS: Dict[str, torch.Tensor] = {}


def inferno_lut(device: torch.device) -> torch.Tensor:
    """[256, 3] uint8 BGR: cv2.applyColorMap(arange(256), COLORMAP_INFERNO), cached per device."""
    key = str(device)
    if key not in _LUTS:
        import cv2

        lut = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_INFERNO).reshape(256, 3)
        _LUTS[key] = torch.from_numpy(np.ascontiguousarray(lut)).to(device)
    return _LUTS[key]


def _bgr(color: Any) -> int:
    """cv2's Scalar -> 8-bit BGR: up to four channels, missing ones 0, each rounded and saturated."""
    c = [color] if np.isscalar(color) else list(color)
    if not 1 <= len(c) <= 4:
        raise ValueError(f"colour {color!r}: expected 1 to 4 channels")
    ch = [min(255, max(0, int(np.rint(float(v))))) for v in (c + [0, 0, 0])[:3]]
    return ch[0] | (ch[1] << 8) | (ch[2] << 16)


def _coord(v: Any) -> int:
    v = int(v)
    if not -MAX_COORD < v < MAX_COORD:
        raise ValueError(f"pixel coordinate {v} is outside +-2^24")
    return v


def line_record(p0: Sequence[int], p1: Sequence[int], color: Any, thickness: int) -> List[int]:
    """cv2.line(img, p0, p1, color, thickness) with (x, y) points."""
    t = int(thickness)
    if not 1 <= t <= MAX_THICKNESS:
        raise ValueError(f"line thickness {t} is outside 1..{MAX_THICKNESS}")
    return [_lib.DRAW_LINE, _coord(p0[0]), _coord(p0[1]), _coord(p1[0]), _coord(p1[1]), 0, t, _bgr(color)]


def circle_record(center: Sequence[int], radius: int, color: Any, thickness: int = 1) -> List[int]:
    """cv2.circle(img, center, radius, color, thickness): thickness < 0 fills, 0 draws as 1 (LINE_8, shift 0)."""
    r, t = int(radius), int(thickness)
    t = -1 if t < 0 else max(t, 1)
    if not 0 <= r <= MAX_RADIUS or t > MAX_THICKNESS:
        raise ValueError(f"circle radius {r} / thickness {t} outside 0..{MAX_RADIUS} / -1, 0..{MAX_THICKNESS}")
    return [_lib.DRAW_CIRCLE, _coord(center[0]), _coord(center[1]), 0, 0, r, t, _bgr(color)]


def metric_to_pixel(pt: Any, ppm: float, origin: np.ndarray) -> np.ndarray:
    """traj_visualizer.py:108-114, verbatim: (row, col) int32 of a metric (x, y) point."""
    px = pt * ppm * np.array([-1, -1]) + origin
    return px.astype(np.int32)


def trajectory_records(camera_positions: Sequence[Any], camera_yaw: float, ppm: float, origin: np.ndarray) -> List[List[int]]:
    """TrajectoryVisualizer.draw_trajectory (traj_visualizer.py:28-99) as draw records.  The reference paints the union of
    every path segment since its last reset (a cached mask) in one colour; drawing the segments of all positions since the
    map's reset in order gives the same pixels.  Segments whose end points share a pixel are skipped (:64)."""
    recs: List[List[int]] = []
    if len(camera_positions) == 0:
        return recs
    px = [metric_to_pixel(p, ppm, origin) for p in camera_positions]
    t = int(PATH_THICKNESS * SCALE_FACTOR)
    for a, b in zip(px[:-1], px[1:]):
        if np.array_equal(a, b):
            continue
        recs.append(line_record(a[::-1], b[::-1], PATH_COLOR, t))
    pos = px[-1]
    recs.append(circle_record(pos[::-1], int(AGENT_RADIUS * SCALE_FACTOR), AGENT_COLOR, -1))
    end = (int(pos[0] - AGENT_LINE_LENGTH * SCALE_FACTOR * np.cos(camera_yaw)),
           int(pos[1] - AGENT_LINE_LENGTH * SCALE_FACTOR * np.sin(camera_yaw)))
    recs.append(line_record(pos[::-1], end[::-1], AGENT_LINE_COLOR, int(AGENT_LINE_THICKNESS * SCALE_FACTOR)))
    return recs


_MARKER_KEYS = {"radius", "color", "thickness"}


def marker_records(markers: Optional[Sequence[Tuple[Any, Dict[str, Any]]]], ppm: float, origin: np.ndarray) -> List[List[int]]:
    """TrajectoryVisualizer.draw_circle for each (position, kwargs) (traj_visualizer.py:101-106); kwargs are cv2.circle's
    radius, color and thickness."""
    recs: List[List[int]] = []
    for pos, kw in markers or []:
        extra = set(kw) - _MARKER_KEYS
        if extra:
            raise TypeError(f"marker keyword(s) {sorted(extra)} not supported (radius, color, thickness)")
        if "radius" not in kw or "color" not in kw:
            raise TypeError("a marker needs 'radius' and 'color'")
        px = metric_to_pixel(pos, ppm, origin)
        recs.append(circle_record(px[::-1], kw["radius"], kw["color"], kw.get("thickness", 1)))
    return recs


class DrawLists:
    """Packs per-environment draw lists into one page-locked int32 buffer and draws them with vlfm_render_draw.  Two
    buffers alternate; a buffer is refilled only after the upload issued from it has executed."""

    def __init__(self, device: torch.device) -> None:
        self.device = device
        self._pin: List[Optional[torch.Tensor]] = [None, None]
        self._ev = [torch.cuda.Event(), torch.cuda.Event()]
        self._used = [False, False]
        self._i = 0
        self._dev: Optional[torch.Tensor] = None

    def draw(self, frames: torch.Tensor, lists: Sequence[Sequence[Sequence[int]]]) -> None:
        n, g = int(frames.shape[0]), int(frames.shape[1])
        assert frames.dtype == torch.uint8 and frames.is_contiguous() and tuple(frames.shape[1:]) == (g, g, 3) and len(lists) == n
        counts = [len(l) for l in lists]
        total = sum(counts)
        if total == 0:
            return
        nints = n + 1 + _lib.DRAW_RECORD_INTS * total
        i = self._i
        self._i ^= 1
        if self._used[i]:
            self._ev[i].synchronize()
        if self._pin[i] is None or self._pin[i].numel() < nints:
            self._pin[i] = torch.empty(max(nints, 1024), dtype=torch.int32).pin_memory()
        buf = self._pin[i].numpy()
        buf[0] = 0
        buf[1 : n + 1] = np.cumsum(counts)
        buf[n + 1 : nints] = np.asarray([r for l in lists for r in l], dtype=np.int64).reshape(-1)
        if self._dev is None or self._dev.numel() < nints:
            self._dev = torch.empty(max(nints, 1024), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.load().vlfm_render_draw(g, n, _lib.ptr(frames), self._pin[i].data_ptr(), nints, _lib.ptr(self._dev),
                                              self._dev.numel(), _lib.stream_ptr())
            self._ev[i].record()
        self._used[i] = True
        _lib.check(rc, "vlfm_render_draw")


class _Workspace:
    def __init__(self) -> None:
        self.t: Optional[torch.Tensor] = None

    def get(self, n: int, device: torch.device) -> torch.Tensor:
        nb = ctypes.c_size_t(0)
        _lib.check(_lib.load().vlfm_render_workspace_bytes(n, ctypes.byref(nb)), "vlfm_render_workspace_bytes")
        if self.t is None or self.t.numel() * 8 < nb.value:
            self.t = torch.empty((nb.value + 7) // 8, dtype=torch.float64, device=device)
        return self.t


def value_frames(reduced: torch.Tensor, explored: Optional[torch.Tensor], slots: Optional[torch.Tensor], ws: _Workspace,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[n, G, G] float32 / float64 reduced maps (call order) -> [n, G, G, 3] uint8 frames (vlfm_render_value)."""
    n, g = int(reduced.shape[0]), int(reduced.shape[1])
    assert reduced.dtype in (torch.float32, torch.float64) and reduced.is_contiguous() and reduced.shape == (n, g, g)
    if explored is not None:
        assert explored.dtype == torch.uint8 and explored.is_contiguous() and tuple(explored.shape[1:]) == (g, g)
    dev = reduced.device
    out = torch.empty((n, g, g, 3), dtype=torch.uint8, device=dev) if out is None else out
    with torch.cuda.device(dev):
        rc = _lib.load().vlfm_render_value(g, n, _lib.ptr(slots), _lib.ptr(reduced), int(reduced.dtype == torch.float64), _lib.ptr(explored),
                                           _lib.ptr(inferno_lut(dev)), _lib.ptr(out), _lib.ptr(ws.get(n, dev)), ws.t.numel() * 8,
                                           _lib.stream_ptr())
    _lib.check(rc, "vlfm_render_value")
    return out
