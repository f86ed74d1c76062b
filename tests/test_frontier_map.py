"""FrontierMap (vlfm/mapping/frontier_map.py:10-77): host bookkeeping around one cosine call per update that introduces a
new frontier.  Checked against explicit expectations, and against what the REAL reference class (its HTTP encoder replaced by
the same scripted one) did on the same streams (stored fixtures)."""
import numpy as np
import pytest

from oracle.live_cases import FRONTIER_SEEDS, ScriptedEncoder, frontier_stream
from vlfm_b200.mapping.frontier_map import FrontierMap


def test_update_sort_reset_semantics():
    enc = ScriptedEncoder()
    fm = FrontierMap(encoder=enc)
    img = np.zeros((2, 2, 3), np.uint8)
    a, b, c = np.array([1.0, 2.0]), np.array([3.0, 4.0]), np.array([5.0, 6.0])
    fm.update([a, b], img, "x")
    assert enc.calls == 1 and [f.cosine for f in fm.frontiers] == [0.1, 0.1]            # one encode for both new frontiers
    fm.update([b.copy(), c], img, "x")                                                  # a vanished, b kept (array_equal), c new
    assert enc.calls == 2 and len(fm.frontiers) == 2
    assert np.array_equal(fm.frontiers[0].xyz, b) and fm.frontiers[0].cosine == 0.1 and fm.frontiers[1].cosine == 0.2
    fm.update([b, c], img, "x")
    assert enc.calls == 2                                                               # nothing new: no encode
    pts, vals = fm.sort_waypoints()
    assert vals == [0.2, 0.1] and np.array_equal(pts, np.array([c, b]))
    fm.reset()
    assert fm.frontiers == []
    fm.update([], img, "x")
    assert enc.calls == 2 and fm.frontiers == []


@pytest.mark.parametrize("seed", FRONTIER_SEEDS)
def test_matches_live_reference(seed, live_golden):
    ref, got = live_golden("frontier_map"), FrontierMap(encoder=ScriptedEncoder())
    for k, (locs, img) in enumerate(frontier_stream(seed)):
        got.update(locs, img, "a chair")
        key = f"s{seed}_t{k}_"
        r_xyz, r_cos = ref[key + "xyz"], ref[key + "cos"]
        assert len(r_cos) == len(got.frontiers)
        for x, c, g in zip(r_xyz, r_cos, got.frontiers):
            assert np.array_equal(x, g.xyz) and c == g.cosine
        if got.frontiers:
            gp, gv = got.sort_waypoints()
            assert list(ref[key + "sorted_vals"]) == gv and np.array_equal(ref[key + "sorted_pts"], gp)
    assert int(ref[f"s{seed}_calls"]) == got.encoder.calls and got.encoder.calls > 3
