"""oracle/object_map_oracle.py: DBSCAN restatement vs scikit-learn's implementation; the whole class vs the REAL reference
class (vlfm/mapping/object_point_cloud_map.py, run with a stub open3d; its outputs are stored fixtures)."""
import cv2
import numpy as np
import pytest

from oracle import object_map_oracle as om
from oracle.live_cases import fingerprint, object_scenario
from vlfm_b200.utils.synthetic import make_object_mask


def _clustered(rng, n):
    k = int(rng.integers(1, 5))
    parts = []
    for _ in range(k):
        c = rng.uniform(-2, 2, 3)
        parts.append(c + rng.normal(0, rng.uniform(0.03, 0.25), (int(n // k), 3)))
    parts.append(rng.uniform(-3, 3, (n // 10, 3)))
    p = np.concatenate(parts)
    return p[rng.permutation(len(p))]


def test_dbscan_labels_match_sklearn():
    from sklearn.cluster import DBSCAN

    rng = np.random.default_rng(0)
    for t in range(12):
        pts = _clustered(rng, int(rng.integers(300, 2500)))
        mp = [100, 40, 10][t % 3]
        ref = DBSCAN(eps=0.2, min_samples=mp, algorithm="brute").fit(pts).labels_
        got = om.dbscan_labels(pts, 0.2, mp)
        assert np.array_equal(ref, got), (t, (ref != got).sum())
    assert len(om.dbscan_filter(rng.uniform(-50, 50, (500, 3)))) == 0          # only noise


def test_erode_restatement():
    rng = np.random.default_rng(1)
    for k in (0, 1, 2, 3):
        m = make_object_mask(rng, 120, 160)
        m[:, :3] = 1                                                           # touches the image edge: the border does not erode
        assert np.array_equal(cv2.erode(m * 255, None, iterations=k), om.erode_mask_numpy(m, k))


def _same(ref, key, a):
    """`a` against the fingerprint oracle/make_golden.py stored of the reference's array: shape, dtype and the SHA-256 of the
    bytes, i.e. equality of the whole array (clouds of 10^4..10^5 points are too large to store)."""
    got = fingerprint(np.asarray(a))
    assert np.array_equal(got["shape"], ref[key + "_shape"]) and str(got["dtype"]) == str(ref[key + "_dtype"]), key
    assert np.array_equal(got["rows"], ref[key + "_rows"]), key
    return str(got["sha256"]) == str(ref[key + "_sha256"])


@pytest.mark.parametrize("use_dbscan", [True, False])
def test_oracle_class_matches_the_reference_class(use_dbscan, live_golden):
    ref = live_golden("object_map")
    seen = 0
    for seed in range(3):
        o = om.ObjectPointCloudMapOracle(erosion_size=2)
        o.use_dbscan = use_dbscan
        for k, (depth, mask, tf, fx) in enumerate(object_scenario(seed)):
            np.random.seed(7 + seed)
            o.update_map("chair", depth, mask, tf, 0.5, 5.0, fx, fx)
            o.update_explored(tf, 5.0, np.deg2rad(79))
            key = f"d{int(use_dbscan)}_s{seed}_t{k}_"
            assert bool(ref[key + "has"]) == o.has_object("chair")
            if o.has_object("chair"):
                seen += 1
                assert _same(ref, key + "cloud", o.clouds["chair"])
                pos = tf[:2, 3] + 0.3
                assert np.array_equal(ref[key + "best"], o.get_best_object("chair", pos))
                assert _same(ref, key + "target", o.get_target_cloud("chair"))
    assert seen >= 6
