"""Pin oracle/value_map_oracle.py: (1) against the committed fixtures generated from the
real reference, (2) against what the reference class computed on two more scenarios (stored fixtures),
(3) cv2 and numpy primitive back-ends agree bit for bit."""
import glob
import hashlib
import os

import numpy as np
import pytest

from oracle.live_cases import VALUE_CASES
from oracle.value_map_oracle import ValueMapOracle
from vlfm_b200.utils.synthetic import trajectory

FOV = float(np.deg2rad(79.0))


def _digest(frames):
    h = hashlib.sha256()
    for f in frames:
        h.update(np.ascontiguousarray(f.depth).tobytes())
        h.update(np.ascontiguousarray(f.tf).tobytes())
    return h.hexdigest()


def load_case(path):
    z = np.load(path)
    h, w = (int(v) for v in z["hw"])
    frames = trajectory(int(z["seed"]), int(z["steps"]), h=h, w=w, bound_m=float(z["bound"]))
    assert _digest(frames) == str(z["input_sha256"]), "synthetic generator drifted from the fixtures"
    return z, frames


def dense(idx, val, shape, dtype):
    out = np.zeros(int(np.prod(shape)), dtype=dtype)
    out[idx] = val
    return out.reshape(shape)


@pytest.mark.parametrize("prims", ["cv2", "numpy"])
def test_oracle_matches_golden(golden_dir, prims):
    paths = sorted(glob.glob(os.path.join(golden_dir, "vm_*.npz")))
    assert paths
    for path in paths:
        z, frames = load_case(path)
        size, ch = int(z["size"]), int(z["channels"])
        o = ValueMapOracle(ch, size=size, use_max_confidence=bool(z["use_max_confidence"]), fusion_type=str(z["fusion"]), prims=prims)
        for f, v in zip(frames, z["values"]):
            o.update_map(v, f.depth, f.tf, 0.5, 5.0, FOV)
        conf = dense(z["conf_idx"], z["conf_val"], (size, size), np.float32)
        val = dense(z["value_idx"], z["value_val"], (size, size, ch), np.float64)
        assert np.array_equal(o._map, conf), path
        assert np.array_equal(o._value_map.astype(np.float64), val), path
        red = (lambda s: [max(t) for t in s]) if ch > 1 else None
        sw, sv = o.sort_waypoints(z["waypoints"], 0.5, reduce_fn=red)
        assert np.array_equal(sw, z["sorted_wp"]) and np.allclose(np.asarray(sv, float), z["sorted_val"], rtol=0, atol=0)


def test_oracle_matches_live_reference(live_golden):
    ref = live_golden("value_map")
    for i, (ch, maxc, fus, size, seed) in enumerate(VALUE_CASES):
        o = ValueMapOracle(ch, size=size, use_max_confidence=maxc, fusion_type=fus, prims="numpy")
        rng = np.random.default_rng(seed)
        for f in trajectory(seed, 5, bound_m=size / 40 - 6):
            o.update_map(rng.random(ch), f.depth, f.tf, 0.5, 5.0, FOV)
        r_map, r_value = ref[f"map{i}"], ref[f"value{i}"]
        assert r_map.any() and r_map.dtype == o._map.dtype and r_value.dtype == o._value_map.dtype
        assert np.array_equal(r_map, o._map) and np.array_equal(r_value, o._value_map)


def test_oracle_ppm40_matches_patched_reference(live_golden):
    """configs[4]/[5] geometry: the reference needs `pixels_per_meter` patched and its cone cache cleared
    (value_map.py:65, :339); the oracle takes ppm as a parameter."""
    ref = live_golden("value_map")
    o = ValueMapOracle(1, size=1000, use_max_confidence=False, pixels_per_meter=40, prims="numpy")
    rng = np.random.default_rng(9)
    for f in trajectory(62, 2, h=128, w=128, bound_m=6.0):
        o.update_map(rng.random(1), f.depth, f.tf, 0.5, 5.0, FOV)
    assert ref["ppm40_map"].any()
    assert np.array_equal(ref["ppm40_map"], o._map) and np.array_equal(ref["ppm40_value"], o._value_map)
