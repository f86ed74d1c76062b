"""Generate tests/golden/*.npz by running the REAL reference.

Usage:  VLFM_REFERENCE=<checkout of bdaiinstitute/vlfm> python oracle/make_golden.py
vm_*.npz: inputs are regenerated from vlfm_b200.utils.synthetic with the recorded seeds (an input checksum is stored so
generator drift is detected); outputs are stored sparsely (flat indices + values of non-zero cells).
live_*.npz: what the reference's own classes computed on the scenarios of the tests that compare the oracle / the host classes
with them (scenario definitions: oracle/live_cases.py, shared with those tests).
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import live_cases as lc  # noqa: E402
from oracle import ref_import  # noqa: E402
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
FOV = float(np.deg2rad(79.0))

VALUE_CASES = [
    # name, channels, use_max_conf, fusion, size, seed, steps, (H, W), bound
    ("vm_weighted", 1, False, "default", 480, 11, 6, (480, 640), 5.0),
    ("vm_maxconf_c2", 2, True, "default", 480, 12, 6, (480, 640), 5.0),
    ("vm_edge_clip", 1, False, "default", 260, 13, 5, (240, 320), 6.2),
    ("vm_replace", 1, False, "replace", 400, 14, 4, (120, 160), 3.0),
    ("vm_equal", 1, False, "equal_weighting", 400, 15, 4, (120, 160), 3.0),
]


def digest(frames) -> str:
    h = hashlib.sha256()
    for f in frames:
        h.update(np.ascontiguousarray(f.depth).tobytes())
        h.update(np.ascontiguousarray(f.tf).tobytes())
    return h.hexdigest()


def sparse(a: np.ndarray):
    flat = a.reshape(-1)
    idx = np.flatnonzero(flat)
    return idx.astype(np.int32), flat[idx]


def value_cases() -> None:
    RV = ref_import.value_map_class()
    for name, ch, maxc, fus, size, seed, steps, (h, w), bound in VALUE_CASES:
        RV._confidence_masks.clear()
        ref = RV(ch, size=size, use_max_confidence=maxc, fusion_type=fus)
        frames = trajectory(seed, steps, h=h, w=w, bound_m=bound)
        rng = np.random.default_rng(seed)
        vals = rng.random((steps, ch))
        for f, v in zip(frames, vals):
            ref.update_map(v, f.depth, f.tf, 0.5, 5.0, FOV)
        ci, cv = sparse(ref._map)
        vi, vv = sparse(ref._value_map)
        wps = np.array([[f.xy[0] + 0.4, f.xy[1] - 0.3] for f in frames])
        red = (lambda s: [max(t) for t in s]) if ch > 1 else None
        sw, sv = ref.sort_waypoints(wps, 0.5, reduce_fn=red)
        np.savez_compressed(
            os.path.join(OUT, name + ".npz"),
            channels=ch, use_max_confidence=maxc, fusion=fus, size=size, seed=seed, steps=steps,
            hw=np.array([h, w]), bound=bound, values=vals, input_sha256=digest(frames),
            conf_idx=ci, conf_val=cv, value_idx=vi, value_val=vv.astype(np.float64),
            value_dtype=str(ref._value_map.dtype), waypoints=wps, sorted_wp=sw,
            sorted_val=np.asarray(sv, dtype=np.float64),
        )
        print(name, "conf nz", ci.size, "value nz", vi.size)


def save(name: str, arrays: dict) -> None:
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(name, len(arrays), "arrays", os.path.getsize(path), "bytes")


def live_value_map() -> None:
    RV = ref_import.value_map_class()
    out = {}
    for i, (ch, maxc, fus, size, seed) in enumerate(lc.VALUE_CASES):
        RV._confidence_masks.clear()
        r = RV(ch, size=size, use_max_confidence=maxc, fusion_type=fus)
        rng = np.random.default_rng(seed)
        for f in trajectory(seed, 5, bound_m=size / 40 - 6):
            r.update_map(rng.random(ch), f.depth, f.tf, 0.5, 5.0, FOV)
        out[f"map{i}"], out[f"value{i}"] = r._map, r._value_map
    RV._confidence_masks.clear()
    r = RV(1, size=1000, use_max_confidence=False)
    r.pixels_per_meter = 40
    rng = np.random.default_rng(9)
    for f in trajectory(62, 2, h=128, w=128, bound_m=6.0):
        r.update_map(rng.random(1), f.depth, f.tf, 0.5, 5.0, FOV)
    RV._confidence_masks.clear()
    out["ppm40_map"], out["ppm40_value"] = r._map, r._value_map
    save("live_value_map", out)


def live_obstacle() -> None:
    RO = ref_import.obstacle_map_class()
    out = {}
    for hole in lc.OBSTACLE_HOLES:
        for i, (seed, (h, w), size, ppm) in enumerate(lc.OBSTACLE_CASES):
            r = RO(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=hole, size=size, pixels_per_meter=ppm)
            fx = focal_from_hfov(w)
            for f in trajectory(seed, 4, h=h, w=w, bound_m=5):
                r.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79), explore=False)
            out[f"h{hole}_map{i}"] = np.packbits(np.asarray(r._map, dtype=bool))
            out[f"h{hole}_nav{i}"] = np.packbits(np.asarray(r._navigable_map, dtype=bool))
    save("live_obstacle", out)
    r = RO(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=-1, size=400)
    fx = focal_from_hfov(160)
    out = {}
    for k, f in enumerate(lc.explore_frames()):
        r.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79))
        out[f"explored{k}"] = np.packbits(np.asarray(r.explored_area, dtype=bool))
        out[f"frontiers_px{k}"], out[f"frontiers{k}"] = np.asarray(r._frontiers_px), np.asarray(r.frontiers)
    save("live_explore", out)


def live_object_map() -> None:
    R = ref_import.object_map_module().ObjectPointCloudMap
    out = {}
    for use_dbscan in (True, False):
        for seed in range(3):
            r = R(erosion_size=2)
            r.reset()
            r.use_dbscan = use_dbscan
            for k, (depth, mask, tf, fx) in enumerate(lc.object_scenario(seed)):
                np.random.seed(7 + seed)
                r.update_map("chair", depth, mask, tf, 0.5, 5.0, fx, fx)
                r.update_explored(tf, 5.0, np.deg2rad(79))
                key = f"d{int(use_dbscan)}_s{seed}_t{k}_"
                out[key + "has"] = np.array(r.has_object("chair"))
                if r.has_object("chair"):
                    out[key + "best"] = np.asarray(r.get_best_object("chair", tf[:2, 3] + 0.3))
                    for name, a in (("cloud", r.clouds["chair"]), ("target", r.get_target_cloud("chair"))):
                        out.update({key + name + "_" + k2: v for k2, v in lc.fingerprint(np.asarray(a)).items()})
    save("live_object_map", out)


def live_host_maps() -> None:
    ref = ref_import.base_map_class()(size=1000)
    pts, cells = lc.base_map_points()
    save("live_base_map", {"px": ref._xy_to_px(pts), "xy": ref._px_to_xy(cells), "origin": np.asarray(ref._episode_pixel_origin),
                           "ppm": np.array(ref.pixels_per_meter)})
    RF = ref_import.frontier_map_class(lc.ScriptedEncoder)
    out = {}
    for seed in lc.FRONTIER_SEEDS:
        ref = RF()
        ref.frontiers = []
        for k, (locs, img) in enumerate(lc.frontier_stream(seed)):
            ref.update(locs, img, "a chair")
            key = f"s{seed}_t{k}_"
            out[key + "xyz"] = np.array([f.xyz for f in ref.frontiers], dtype=np.float64).reshape(len(ref.frontiers), 2)
            out[key + "cos"] = np.array([f.cosine for f in ref.frontiers], dtype=np.float64)
            if ref.frontiers:
                sp, sv = ref.sort_waypoints()
                out[key + "sorted_pts"], out[key + "sorted_vals"] = np.asarray(sp), np.asarray(sv, dtype=np.float64)
        out[f"s{seed}_calls"] = np.array(ref.encoder.calls)
    save("live_frontier_map", out)


if __name__ == "__main__":
    assert ref_import.available(), "set VLFM_REFERENCE to a checkout of the reference"
    os.makedirs(OUT, exist_ok=True)
    value_cases()
    live_value_map()
    live_obstacle()
    live_object_map()
    live_host_maps()
