"""The visualize oracle (tests/visualize_oracle.py) reproduces, bit for bit, the frames the reference's own ValueMap.visualize /
ObstacleMap.visualize rendered (tests/golden/live_visualize.npz, scripts/make_visualize_golden.py): weighted (float64) and
max-confidence (float32) maps, C = 2 with an ITMPolicyV3 reducer, obstacle-map masking, repeated trajectory cells, a reset
mid-episode, markers and path off the map, black padding, an all-zero map, a one-point trajectory and negative values."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

import make_visualize_golden as mg  # noqa: E402
import visualize_oracle as vo  # noqa: E402


@pytest.fixture(scope="module")
def golden(live_golden):
    return live_golden("visualize")


def replay(z, case, force_float32=False):
    """the oracle's frame at every step of a golden case (force_float32: normalise a weighted map in float32, which is wrong)"""
    name, kind, ch, maxconf, red, masked, _neg, _zero, pad = case
    g = mg.grids_of(z, name)
    xy, yaw, reset_at = z[f"{name}/xy"], z[f"{name}/yaw"], int(z[f"{name}/reset_at"][0])
    markers = [(z[f"{name}/marker_xy"][k], {"radius": int(z[f"{name}/marker_radius"][k]), "thickness": int(z[f"{name}/marker_thickness"][k]),
                                            "color": tuple(int(c) for c in z[f"{name}/marker_color"][k])}) for k in range(len(z[f"{name}/marker_xy"]))]
    origin = np.array([mg.G // 2, mg.G // 2])
    frames, start = [], 0
    for t in range(len(xy)):
        if t == reset_at:
            start = t
        pos = list(xy[start : t + 1])
        if kind == "value":
            grid = g["value"].astype(np.float32 if maxconf or force_float32 else np.float64)
            fn = vo.max_reducer if red == "max" else vo.itm_v3_reducer(mg.THRESH)
            frames.append(vo.value_frame(grid, fn, g["explored"] if masked else None, pos, float(yaw[t]), markers, mg.PPM, origin))
        else:
            frames.append(vo.obstacle_frame(g["obst"], g["nav"], g["explored"], z[f"{name}/frontiers_px"], pad, pos, float(yaw[t]), mg.PPM, origin))
    return np.stack(frames)


@pytest.mark.parametrize("case", mg.CASES, ids=[c[0] for c in mg.CASES])
def test_oracle_matches_reference_frames(golden, case):
    ref = mg.frames_of(golden, case[0])
    got = replay(golden, case)
    assert got.shape == ref.shape
    for t in range(len(ref)):
        assert np.array_equal(got[t], ref[t]), f"{case[0]} step {t}: {(got[t] != ref[t]).any(-1).sum()} pixels differ"


def test_fixture_covers_the_scenarios(golden):
    f = mg.frames_of(golden, "weighted")
    assert (f[1:] != f[0]).any()                                           # the trajectory changes the frames
    assert len(golden["all_zero/xy"]) == 1 and not golden["all_zero/value_idx"].size
    assert golden["weighted/xy"].dtype == np.float64 and golden["maxconf/xy"].dtype == np.float32
    assert (golden["negative/value_val"] < 0).any()
    assert int(golden["weighted/reset_at"][0]) > 0


@pytest.mark.parametrize("case", [c for c in mg.CASES if c[1] == "value" and not c[3] and not c[7]], ids=lambda c: c[0])
def test_weighted_maps_need_float64(golden, case):
    """the weighted cases hold cells whose LUT index depends on the normalisation dtype, so the float64 rule is pinned"""
    ref = mg.frames_of(golden, case[0])
    wrong = replay(golden, case, force_float32=True)
    assert (wrong != ref).any(-1).sum() >= 3 * len(ref)
