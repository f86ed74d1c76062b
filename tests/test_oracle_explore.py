"""Explore half of the obstacle map: the cv2-based restatement and the cv2-free one agree, and the reference's
own ObstacleMap code (run with the restated frontier_exploration functions injected; its outputs are stored fixtures) agrees
with both."""
import numpy as np
import pytest

import oracle.explore_oracle as ex
from oracle.live_cases import explore_frames
from oracle.obstacle_map_oracle import ObstacleMapOracle
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory


def _run(prims, seed, steps, hw, size, start=(0.0, 0.0), bound=4.0, depth_scale=1.0):
    ex.PRIMS = prims
    try:
        o = ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=-1, size=size)
        fx = focal_from_hfov(hw[1])
        out = []
        for f in trajectory(seed, steps, h=hw[0], w=hw[1], bound_m=bound, start_xy=start):
            o.update_map(f.depth * np.float32(depth_scale), f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79))
            out.append((o.explored_area.copy(), np.asarray(o._frontiers_px).copy(), np.asarray(o.frontiers).copy()))
        return out
    finally:
        ex.PRIMS = "cv2"


def test_cv2_and_numpy_backends_agree():
    for seed in range(3):
        a = _run("cv2", seed, 6, (120, 160), 400)
        b = _run("numpy", seed, 6, (120, 160), 400)
        assert a[-1][0].sum() > 100
        for (ea, fa, xa), (eb, fb, xb) in zip(a, b):
            assert np.array_equal(ea, eb) and fa.shape == fb.shape and np.array_equal(fa, fb) and np.array_equal(xa, xb)


def test_backends_agree_at_the_map_border():
    """agent within max_depth of the grid edge (walls close enough that no obstacle cell leaves the grid, which would be the
    reference's IndexError): the 5 m cone and the occlusion rays are clipped by cv2 (clipLine rules)"""
    for seed, start in ((0, (8.2, 8.2)), (1, (-8.2, 8.2)), (2, (8.2, -8.2)), (3, (-8.2, -8.2)), (4, (0.0, 8.3)), (5, (-8.3, 0.5))):
        a = _run("cv2", seed, 6, (120, 160), 400, start=start, bound=0.4, depth_scale=0.15)
        b = _run("numpy", seed, 6, (120, 160), 400, start=start, bound=0.4, depth_scale=0.15)
        assert a[-1][0].sum() > 50
        for (ea, fa, xa), (eb, fb, xb) in zip(a, b):
            assert np.array_equal(ea, eb) and fa.shape == fb.shape and np.array_equal(fa, fb) and np.array_equal(xa, xb)


def test_reference_class_with_injected_functions(live_golden):
    ref = live_golden("explore")
    o = ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=-1, size=400)
    fx = focal_from_hfov(160)
    for k, f in enumerate(explore_frames()):
        o.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79))
        explored = np.unpackbits(ref[f"explored{k}"])[: 400 * 400].reshape(400, 400)
        assert explored.any()
        assert np.array_equal(explored.astype(bool), np.asarray(o.explored_area, dtype=bool))
        assert np.array_equal(ref[f"frontiers_px{k}"], np.asarray(o._frontiers_px))
        assert np.array_equal(ref[f"frontiers{k}"], np.asarray(o.frontiers))
