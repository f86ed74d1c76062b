"""BaseMap conversions (vlfm/mapping/base_map.py:35-60): explicit formulae, and what the reference class returned (stored fixtures)."""
import numpy as np
import pytest

from oracle.live_cases import base_map_points
from vlfm_b200.mapping.base_map import BaseMap


def _ref_xy_to_px(points, size, ppm):          # the reference's arithmetic, array form
    origin = np.array([size // 2, size // 2])
    px = np.rint(points[:, ::-1] * ppm) + origin
    px[:, 0] = size - px[:, 0]
    return px.astype(int)


def _ref_px_to_xy(px, size, ppm):
    origin = np.array([size // 2, size // 2])
    q = px.copy()
    q[:, 0] = size - q[:, 0]
    return ((q - origin) / ppm)[:, ::-1]


@pytest.mark.parametrize("size,ppm", [(1000, 20), (2500, 50), (301, 20), (4000, 40)])
def test_conversions_match_reference_arithmetic(size, ppm):
    rng = np.random.default_rng(size + ppm)
    m = BaseMap(size=size, pixels_per_meter=ppm)
    pts = rng.uniform(-size / ppm / 2, size / ppm / 2, (500, 2))
    pts[:8] = np.array([[0.0, 0.0], [0.025, -0.025], [0.075, 0.125], [1.0, -1.0], [-0.5, 0.5], [2.5 / ppm, 0.5 / ppm], [-1.5 / ppm, 3.5 / ppm], [12.3, -7.7]])
    got = m._xy_to_px(pts)
    assert got.dtype.kind == "i" and np.array_equal(got, _ref_xy_to_px(pts, size, ppm))       # incl. the half-to-even ties
    cells_i = rng.integers(0, size, (200, 2))
    cells_f = rng.uniform(0, size, (200, 2))                                                   # frontier midpoints are fractional
    for cells in (cells_i, cells_f):
        assert np.array_equal(m._px_to_xy(cells), _ref_px_to_xy(cells, size, ppm))
    m.update_agent_traj(np.array([1.0, 2.0]), 0.3)
    assert len(m._camera_positions) == 1 and m._last_camera_yaw == 0.3
    m.reset()
    assert m._camera_positions == []


def test_conversions_match_live_reference_class(live_golden):
    ref, got = live_golden("base_map"), BaseMap(size=1000)
    pts, cells = base_map_points()
    px = got._xy_to_px(pts)
    assert px.dtype.kind == ref["px"].dtype.kind and np.array_equal(px, ref["px"])
    assert np.array_equal(got._px_to_xy(cells), ref["xy"])
    assert np.array_equal(got._episode_pixel_origin, ref["origin"]) and got.pixels_per_meter == ref["ppm"]
