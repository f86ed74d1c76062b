"""Scenarios on which the reference's own classes were run to make tests/golden/live_*.npz, and the helpers to compare with them.

Imported by ``oracle/make_golden.py`` (which runs the reference on them) and by the tests (which run the oracle / the host
classes on them and compare with the stored results), so the two sides cannot drift apart.  Needs numpy only.
"""
from __future__ import annotations

import hashlib

import numpy as np

from vlfm_b200.utils.synthetic import focal_from_hfov, make_object_mask, trajectory

# ---- value map: channels, use_max_confidence, fusion, grid size, seed
VALUE_CASES = [(1, False, "default", 700, 21), (2, True, "default", 500, 22)]

# ---- obstacle half: hole_area_thresh values; seed, (H, W), grid size, pixels per metre
OBSTACLE_HOLES = [-1, 100000]
OBSTACLE_CASES = [(0, (240, 320), 600, 20), (2, (240, 320), 1500, 50)]

# ---- frontier map: stream seeds
FRONTIER_SEEDS = [0, 1, 2]


def fingerprint(a: np.ndarray) -> dict:
    """A large array as shape + dtype + SHA-256 of its bytes (equality of the whole array is still decidable) and every 97th
    row, so that a mismatch can be looked at."""
    a = np.ascontiguousarray(a)
    return {"shape": np.array(a.shape), "dtype": np.array(str(a.dtype)), "sha256": np.array(hashlib.sha256(a.tobytes()).hexdigest()),
            "rows": a[::97].copy()}


def explore_frames():
    return trajectory(7, 6, h=120, w=160, bound_m=4)


def object_scenario(seed, steps=6, h=240, w=320):
    """(depth, mask, camera transform, focal length) per step: detections on either image side, every third one out of range."""
    rng = np.random.default_rng(100 + seed)
    fx = focal_from_hfov(w)
    out = []
    for i, f in enumerate(trajectory(seed, steps, h=h, w=w, bound_m=6.0)):
        side = ["any", "left", "any", "right", "any"][i % 5]
        mask = make_object_mask(rng, h, w, side)
        depth = f.depth.copy()
        if i % 3 == 2:
            depth[mask > 0] = np.float32(0.98)                                # a far detection: out-of-range ids
        out.append((depth, mask, f.tf, fx))
    return out


def base_map_points():
    rng = np.random.default_rng(5)
    return rng.uniform(-20, 20, (1000, 2)), rng.uniform(0, 1000, (300, 2))


class ScriptedEncoder:
    """Stands in for the image-text encoder of FrontierMap: a cosine that depends on the call count and the image only."""

    def __init__(self):
        self.calls = 0

    def cosine(self, image, text):
        self.calls += 1
        return 0.1 * self.calls + float(image.sum() % 7) * 1e-3


def frontier_stream(seed, steps=30):
    rng = np.random.default_rng(seed)
    pool = [rng.uniform(-5, 5, 2).round(2) for _ in range(12)]
    out = []
    for _ in range(steps):
        k = int(rng.integers(0, 6))
        idx = rng.choice(len(pool), size=k, replace=False)
        out.append(([pool[i].copy() for i in idx], rng.integers(0, 255, (4, 4, 3), dtype=np.uint8)))
    return out
