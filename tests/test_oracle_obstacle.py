import numpy as np
import pytest

from oracle.live_cases import OBSTACLE_CASES, OBSTACLE_HOLES
from oracle.obstacle_map_oracle import ObstacleMapOracle
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory


@pytest.mark.parametrize("hole", OBSTACLE_HOLES)
def test_obstacle_half_matches_live_reference(hole, live_golden):
    ref = live_golden("obstacle")
    for i, (seed, (h, w), size, ppm) in enumerate(OBSTACLE_CASES):
        o = ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=hole, size=size, pixels_per_meter=ppm)
        fx = focal_from_hfov(w)
        for f in trajectory(seed, 4, h=h, w=w, bound_m=5):
            o.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79), explore=False)
        r_map = np.unpackbits(ref[f"h{hole}_map{i}"])[: size * size].reshape(size, size).astype(bool)
        r_nav = np.unpackbits(ref[f"h{hole}_nav{i}"])[: size * size].reshape(size, size).astype(bool)
        assert r_map.any() and not r_nav.all()
        assert np.array_equal(r_map, o._map) and np.array_equal(r_nav, o._navigable_map)


def _depth_with_holes(seed, h=60, w=80):
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.05, 1.0, (h, w)).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    for _ in range(int(rng.integers(2, 6))):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(3, 14)
        d[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 0
        if r > 6:
            d[(yy - cy) ** 2 + (xx - cx) ** 2 <= (r // 2) ** 2] = 0.5
            d[(yy - cy) ** 2 + (xx - cx) ** 2 <= (r // 4) ** 2] = 0
    d[rng.random((h, w)) < 0.02] = 0
    return d


@pytest.mark.parametrize("thresh", [5, 40, 200, 100000])
def test_fill_holes_restatement_matches_cv2(thresh):
    """oracle.fill_holes_numpy (the rules the GPU kernel follows) against the cv2 calls the reference makes
    (vlfm/utils/img_utils.py:361-390)."""
    cv2 = pytest.importorskip("cv2")
    from oracle import contours as ct
    from oracle.obstacle_map_oracle import fill_holes, fill_holes_numpy

    for seed in range(12):
        d = _depth_with_holes(seed * 13 + thresh)
        assert np.array_equal(fill_holes(d, thresh), fill_holes_numpy(d, thresh))
        holes = (d == 0).astype(np.uint8)
        want = sorted(tuple(map(tuple, c.reshape(-1, 2))) for c in cv2.findContours(holes, cv2.RETR_TREE, cv2.CHAIN_APPROX_NONE)[0])
        got = sorted(tuple(map(tuple, c.reshape(-1, 2))) for c in ct.find_all_contours(holes))
        assert got == want
