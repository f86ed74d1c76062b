"""Write tests/golden/live_visualize.npz: frames the REAL reference's ValueMap.visualize / ObstacleMap.visualize rendered.

Usage:  VLFM_REFERENCE=<checkout of bdaiinstitute/vlfm> python scripts/make_visualize_golden.py

The scenarios (``CASES``) set the reference maps' grids directly (stored sparsely), feed a trajectory through
update_agent_traj -- with repeated cells, a reset mid-episode, points off the map -- and record the frame of every step.
tests/test_oracle_visualize.py replays them through tests/visualize_oracle.py; tests/test_visualize_gpu.py through the
GPU maps.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

G = 256
PPM = 20
THRESH = 0.3      # ITMPolicyV3-style reducer threshold
FOV = float(np.deg2rad(79.0))

# name, kind, channels, use_max_confidence, reducer, masked by an obstacle map, negative values, all zero, padding colour
CASES = [
    ("weighted", "value", 1, False, "max", False, False, False, None),
    ("maxconf", "value", 1, True, "max", True, False, False, None),
    ("c2_v3", "value", 2, True, "v3", True, False, False, None),
    ("weighted_c2_v3", "value", 2, False, "v3", False, True, False, None),
    ("negative", "value", 1, False, "max", False, True, False, None),
    ("all_zero", "value", 1, False, "max", False, False, True, None),
    ("obstacle", "obstacle", 0, False, "", False, False, False, (100, 100, 100)),
    ("obstacle_black", "obstacle", 0, False, "", False, False, False, (0, 0, 0)),
]


def blobs(rng: np.random.Generator, n: int, rmax: int = 30) -> np.ndarray:
    """[G, G] mask of n random discs"""
    yy, xx = np.mgrid[:G, :G]
    m = np.zeros((G, G), bool)
    for _ in range(n):
        cy, cx, r = rng.integers(0, G), rng.integers(0, G), rng.integers(4, rmax)
        m |= (yy - cy) ** 2 + (xx - cx) ** 2 <= r * r
    return m


def plant_dtype_sensitive(v: np.ndarray) -> None:
    """Plant cells (equal in every channel, so any reducer keeps them) whose LUT index differs between a float32 and a
    float64 normalisation: float32 neighbours of lo + k * (hi - lo) / 255, inside [lo, hi] so lo and hi stay put.  The
    reference's grid dtype then shows in the frames."""
    red = v.max(axis=-1)
    nz = red[red != 0]
    lo, hi = nz.min(), red.max()

    def idx(x, dt):
        x, l, h = dt(x), dt(lo), dt(hi)
        return int(((x - l) / (h - l)) * dt(255))

    found = []
    for k in range(1, 255):
        x0 = np.float32(np.float64(lo) + k * (np.float64(hi) - np.float64(lo)) / 255)
        for d in range(-3, 4):
            x = np.float32(x0 + d * np.spacing(x0))
            if lo < x < hi and x != 0 and idx(x, np.float32) != idx(x, np.float64):
                found.append(x)
                break
        if len(found) == 8:
            break
    assert len(found) >= 3, "no dtype-sensitive values found"
    v[5, 5 : 5 + len(found)] = np.asarray(found, np.float32)[:, None]


def scenario(seed: int, kind: str, channels: int, negative: bool, all_zero: bool, weighted: bool = False):
    """Grids, trajectory and markers of one case (deterministic in the seed)."""
    rng = np.random.default_rng(seed)
    out = {}
    if kind == "value":
        v = np.zeros((G, G, channels), np.float32)
        if not all_zero:
            m = blobs(rng, 3, 12)
            lo = -0.5 if negative else 0.0
            v[m] = rng.uniform(lo, 1.0, (int(m.sum()), channels)).astype(np.float32)
            if weighted:
                plant_dtype_sensitive(v)
        out["value"] = v
    out["explored"] = blobs(rng, 6, 20).astype(np.uint8)
    out["obst"] = (blobs(rng, 12, 12) & ~blobs(rng, 12, 10)).astype(np.uint8)
    out["nav"] = (~blobs(rng, 5, 20)).astype(np.uint8)
    nf = 8
    fr = np.concatenate([rng.uniform(-3, G + 3, (nf, 2)), [[0.5, 0.5], [G - 0.5, 100.25], [3.7, G - 1.2]]])
    out["frontiers_px"] = fr
    # trajectory: a walk that leaves the map on one side, with repeated cells (sub-pixel steps) and a reset at step 6
    steps = 11 if not all_zero else 1
    xy = np.cumsum(rng.normal(0, 0.6, (steps, 2)), axis=0)
    if steps > 8:
        xy[3] = xy[2] + 0.01                    # same pixel as the previous point
        xy[8] = [7.3, -2.0]                     # off the map (half size 6.4 m)
        xy[9] = [6.5, -6.9]
    dtype = np.float32 if seed % 2 else np.float64
    out["xy"] = xy.astype(dtype)
    out["yaw"] = rng.uniform(-np.pi, np.pi, steps)
    out["reset_at"] = np.array([6 if steps > 8 else -1])
    mk = np.concatenate([rng.uniform(-7, 7, (4, 2)), [[6.35, 0.0], [0.0, -6.45]]])
    out["marker_xy"] = mk
    out["marker_color"] = rng.integers(0, 256, (len(mk), 3))
    out["marker_thickness"] = np.array([2, 2, -1, 1, 2, 3])
    out["marker_radius"] = np.array([5, 5, 5, 7, 5, 0])
    return out


def markers_of(s):
    return [(s["marker_xy"][k], {"radius": int(s["marker_radius"][k]), "thickness": int(s["marker_thickness"][k]),
                                 "color": tuple(int(c) for c in s["marker_color"][k])}) for k in range(len(s["marker_xy"]))]


def frames_of(z, name: str) -> np.ndarray:
    """[T, G, G, 3] frames of a case stored by main()"""
    f0 = z[f"{name}/frame0"]
    out = []
    for t in range(len(z[f"{name}/xy"])):
        f = f0.copy()
        f[np.unpackbits(z[f"{name}/diff_mask_{t}"], count=G * G).reshape(G, G).astype(bool)] = z[f"{name}/diff_val_{t}"]
        out.append(f)
    return np.stack(out)


def grids_of(z, name: str) -> dict:
    """the grids of a case stored by main(): value [G, G, C] float32 (value cases), explored / obst / nav [G, G] uint8"""
    out = {}
    if f"{name}/value_idx" in z:
        ch = max(CASES[[c[0] for c in CASES].index(name)][2], 1)
        v = np.zeros(G * G * ch, np.float32)
        v[z[f"{name}/value_idx"]] = z[f"{name}/value_val"]
        out["value"] = v.reshape(G, G, ch)
    for k in ("explored", "obst"):
        a = np.zeros(G * G, np.uint8)
        a[z[f"{name}/{k}_idx"]] = 1
        out[k] = a.reshape(G, G)
    nav = np.ones(G * G, np.uint8)
    nav[z[f"{name}/nav0_idx"]] = 0
    out["nav"] = nav.reshape(G, G)
    return out


def main() -> None:
    from oracle import ref_import
    from vlfm_b200.utils.synthetic import trajectory
    import visualize_oracle as vo

    assert ref_import.available(), "set VLFM_REFERENCE to a checkout of the reference"
    VM, OM = ref_import.value_map_class(), ref_import.obstacle_map_class()
    arrays = {}
    for ci, (name, kind, ch, maxconf, red, masked, neg, zero, pad) in enumerate(CASES):
        s = scenario(100 + ci, kind, max(ch, 1), neg, zero, weighted=kind == "value" and not maxconf)
        # reset() gives each instance its own trajectory list (the reference's BaseMap starts with a class-level one, shared by
        # every map until its first reset; the policies reset their maps at the start of each episode)
        om = OM(0.61, 0.88, 0.18, size=G, pixels_per_meter=PPM)
        om.reset()

        def set_obstacle():
            om._map = s["obst"].astype(bool)
            om._navigable_map = s["nav"].astype(np.int64)
            om.explored_area = s["explored"].astype(bool)
            om._frontiers_px = s["frontiers_px"]

        set_obstacle()
        if pad is not None:
            om.radius_padding_color = pad
        if kind == "value":
            vm = VM(ch, size=G, use_max_confidence=maxconf)
            vm.reset()
            # one real fuse lets the reference pick its grid's dtype (float64 for a weighted map, value_map.py:423); the grid
            # is then overwritten in place, which keeps that dtype
            f = trajectory(ci, 1, h=120, w=160, bound_m=2.0)[0]
            vm.update_map(np.full(ch, 0.5), f.depth, f.tf, 0.5, 5.0, FOV)
            assert vm._value_map.dtype == (np.float32 if maxconf else np.float64)
            vm._value_map[...] = s["value"]
            fn = vo.max_reducer if red == "max" else vo.itm_v3_reducer(THRESH)
        frames = []
        for t in range(len(s["xy"])):
            if t == int(s["reset_at"][0]):
                if kind == "value":
                    vm.reset()
                    vm._value_map[...] = s["value"]
                else:
                    om.reset()
                    set_obstacle()
            m = vm if kind == "value" else om
            m.update_agent_traj(s["xy"][t], float(s["yaw"][t]))
            if kind == "value":
                frames.append(vm.visualize(markers_of(s), reduce_fn=fn, obstacle_map=om if masked else None))
            else:
                frames.append(om.visualize())
        if kind == "value":
            nz = np.flatnonzero(s["value"])
            arrays[f"{name}/value_idx"] = nz.astype(np.int32)
            arrays[f"{name}/value_val"] = s["value"].reshape(-1)[nz]
        arrays[f"{name}/explored_idx"] = np.flatnonzero(s["explored"]).astype(np.int32)
        arrays[f"{name}/obst_idx"] = np.flatnonzero(s["obst"]).astype(np.int32)
        arrays[f"{name}/nav0_idx"] = np.flatnonzero(s["nav"] == 0).astype(np.int32)
        for k in ("frontiers_px", "xy", "yaw", "reset_at", "marker_xy", "marker_color", "marker_thickness", "marker_radius"):
            arrays[f"{name}/{k}"] = s[k]
        # frames: the first one, then the bytes in which each frame differs from it (the trajectory and the markers)
        arrays[f"{name}/frame0"] = frames[0]
        for t in range(len(frames)):
            d = (frames[t] != frames[0]).any(-1)
            arrays[f"{name}/diff_mask_{t}"] = np.packbits(d)
            arrays[f"{name}/diff_val_{t}"] = frames[t][d]
    path = os.path.join(ROOT, "tests", "golden", "live_visualize.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
