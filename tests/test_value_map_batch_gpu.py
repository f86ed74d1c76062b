"""ValueMapBatch (csrc/value_map.cu) against one ValueMapOracle per environment, at the batches and geometries the workloads run:
B = 32 (the automatic 23-row fuse tiling), the >48 KB value_geom_kernel shared-memory path (1024^2 depth at ppm 40, ppm 50),
C = 1..8 channels, every fusion mode, cameras next to the grid edge, permuted slots, partial batches, resets, explored masks and
an off-grid camera.  The disc median and the frontier scoring are checked against np.median of the reference's crop-and-disc
selection, in the dtype the reference's value grid has.

Comparison rule: confidence grid bit-exact; value grid bit-exact for max-confidence, replace and equal-weighting-with-max-
confidence maps (the reference keeps those grids float32 and stores the same float32 cast of the value); value grid within 1e-6
of the reference's float64 grid for weighted maps."""
import ctypes
import dataclasses

import cv2
import numpy as np
import pytest
import torch

from oracle.obstacle_map_oracle import ObstacleMapOracle
from oracle.value_map_oracle import ValueMapOracle, disc_reduce
from vlfm_b200 import _lib
from vlfm_b200.utils.synthetic import focal_from_hfov, tf_from_pose, trajectory

pytestmark = pytest.mark.gpu
FOV = float(np.deg2rad(79))
MIN_D, MAX_D = 0.5, 5.0
VAL_TOL = 1e-6
VLFM_E_INVALID = 1
# (use_max_confidence, fusion_type)
FUSIONS = {
    "weighted": (False, "default"),
    "max_confidence": (True, "default"),
    "replace": (False, "replace"),
    "equal_weighted": (False, "equal_weighting"),
    "equal_max_confidence": (True, "equal_weighting"),
}


def _engine(B, C, G, ppm, fusion):
    from vlfm_b200.mapping.value_map import ValueMapBatch

    maxc, fus = FUSIONS[fusion]
    return ValueMapBatch(B, C, size=G, pixels_per_meter=ppm, use_max_confidence=maxc, fusion_type=fus)


def _oracle(C, G, ppm, fusion, explored_fn=None):
    maxc, fus = FUSIONS[fusion]
    return ValueMapOracle(C, size=G, use_max_confidence=maxc, fusion_type=fus, pixels_per_meter=ppm, explored_fn=explored_fn)


def _check(eng, slot, o, tag):
    conf = eng.conf[slot].cpu().numpy()
    val = eng.value[slot].cpu().numpy()
    assert np.array_equal(conf.view(np.uint32), o._map.view(np.uint32)), f"{tag}: confidence grid differs in {(conf != o._map).sum()} cells"
    if eng.ref_float64:
        d = np.abs(val.astype(np.float64) - o._value_map.astype(np.float64)).max()
        assert d <= VAL_TOL, f"{tag}: value grid off by {d}"
    else:
        assert o._value_map.dtype == np.float32
        bad = (val.view(np.uint32) != o._value_map.view(np.uint32)).sum()
        assert bad == 0, f"{tag}: value grid differs in {bad} cells"


def _step(eng, orcs, frames, values, slots=None, explored=None):
    """One batched update of the rows ``frames`` (row i -> grid slot slots[i]) and the same update on their oracles."""
    n = len(frames)
    slots = list(range(n)) if slots is None else slots
    for i, s in enumerate(slots):
        orcs[s].update_map(values[i], frames[i].depth, frames[i].tf, MIN_D, MAX_D, FOV)
    depth = torch.from_numpy(np.stack([f.depth for f in frames])).cuda()
    tf = torch.from_numpy(np.stack([f.tf for f in frames])).cuda()
    vals = torch.from_numpy(np.ascontiguousarray(values, dtype=np.float64)).cuda()
    slot_t = None if slots == list(range(n)) else torch.tensor(slots, dtype=torch.int32, device="cuda")
    if explored is not None:
        eng.mask_unexplored(explored, slot_t, n)
    eng.update(vals, depth, tf, MIN_D, MAX_D, FOV, slots=slot_t, explored=explored)


def _geom_smem_bytes(W, R):
    """value_geom_kernel's dynamic shared memory (k1_smem in csrc/value_map.cu): vertices, two R x ceil(R/32) bit planes, long-edge list."""
    E, WPR = W + 2, (R + 31) // 32
    return max(4 * (2 * ((E + 1) & ~1) + 2 * R * WPR + E), 8 * 128 * 4)


def _auto_rows_per_tile(B, R):
    """The fuse kernel's row tiling when rows_per_tile = 0 (vlfm_value_update)."""
    tiles = min(max((264 + B - 1) // B, 1), R)
    return max((R + tiles - 1) // tiles, 4)


# ------------------------------------------------------------------------------------------------ batch vs per-env oracles
BATCH_CASES = {
    # configs[1]@32 / configs[2]: 32 environments, 640x480, 1000^2 grid at ppm 20 -> the automatic tiling is 23 rows
    "b32_640x480": dict(B=32, hw=(480, 640), G=1000, ppm=20, steps=3, bound=12.0, fusion="weighted", C=1),
    # configs[4] geometry: 1024^2 depth, ppm 40 (R = 401) -> value_geom_kernel needs > 48 KB of shared memory
    "b3_1024sq_ppm40": dict(B=3, hw=(1024, 1024), G=1400, ppm=40, steps=3, bound=8.0, fusion="weighted", C=1),
    "b2_1024sq_ppm40_g4000": dict(B=2, hw=(1024, 1024), G=4000, ppm=40, steps=1, bound=8.0, fusion="max_confidence", C=1),
    # ppm 50 (R = 501), 480x640 depth
    "b2_ppm50": dict(B=2, hw=(480, 640), G=1000, ppm=50, steps=3, bound=4.0, fusion="max_confidence", C=1),
}


@pytest.mark.parametrize("name", list(BATCH_CASES))
def test_batch_vs_per_env_oracles(name):
    cfg = BATCH_CASES[name]
    B, (h, w), G, ppm, C = cfg["B"], cfg["hw"], cfg["G"], cfg["ppm"], cfg["C"]
    R = 2 * int(MAX_D * ppm) + 1
    if name == "b32_640x480":
        assert _auto_rows_per_tile(B, R) == 23
    if ppm >= 40:
        assert _geom_smem_bytes(w, R) > 48 * 1024
    eng = _engine(B, C, G, ppm, cfg["fusion"])
    orcs = [_oracle(C, G, ppm, cfg["fusion"]) for _ in range(B)]
    frames = [trajectory(300 + e, cfg["steps"], h=h, w=w, bound_m=cfg["bound"], start_xy=(0.3 * e, -0.2 * e)) for e in range(B)]
    rng = np.random.default_rng(len(name))
    for i in range(cfg["steps"]):
        _step(eng, orcs, [frames[e][i] for e in range(B)], rng.random((B, C)))
        for e in range(B):
            _check(eng, e, orcs[e], f"{name} step {i} env {e}")
    assert int(eng.status.abs().sum()) == 0
    assert all(o._map.any() for o in orcs)


@pytest.mark.parametrize("fusion", list(FUSIONS))
@pytest.mark.parametrize("C,G", [(1, 400), (1, 403), (2, 400), (5, 400), (8, 400)])
def test_channels_and_fusion_modes(C, G, fusion):
    """C = 1 on a grid with G % 4 == 0 takes the float4 fuse path, every other case the per-cell path; C = 8 is the largest C."""
    B, steps = 3, 4
    eng = _engine(B, C, G, 20, fusion)
    orcs = [_oracle(C, G, 20, fusion) for _ in range(B)]
    frames = [trajectory(400 + 10 * C + e, steps, h=120, w=160, bound_m=4.0, start_xy=(0.5 * e, 0.4 * e)) for e in range(B)]
    rng = np.random.default_rng(G + C)
    for i in range(steps):
        _step(eng, orcs, [frames[e][i] for e in range(B)], rng.random((B, C)))
        for e in range(B):
            _check(eng, e, orcs[e], f"C={C} G={G} {fusion} step {i} env {e}")


@pytest.mark.parametrize("fusion", ["weighted", "max_confidence", "replace"])
def test_cameras_at_the_grid_edge(fusion):
    """Cameras closer than R/2 to every edge and corner: the fuse window is clipped on each side in turn."""
    G, ppm = 300, 20
    lim = (G // 2 - 1) / ppm                      # the last cell row / column inside the grid
    poses = [(lim, 0.0), (-G // 2 / ppm, 0.0), (0.0, lim), (0.0, -lim), (lim, lim), (-lim, -lim), (lim, -lim), (-lim, lim), (3.1, -4.2)]
    B = len(poses)
    eng = _engine(B, 1, G, ppm, fusion)
    orcs = [_oracle(1, G, ppm, fusion) for _ in range(B)]
    base = trajectory(500, 3, h=120, w=160)
    rng = np.random.default_rng(5)
    for i in range(3):
        frames = []
        for e, (x, y) in enumerate(poses):
            frames.append(dataclasses.replace(base[i], tf=tf_from_pose(x, y, 0.88, 0.9 * e + 1.3 * i)))
        _step(eng, orcs, frames, rng.random((B, 1)))
        for e in range(B):
            _check(eng, e, orcs[e], f"{fusion} step {i} pose {poses[e]}")
    assert int(eng.status.abs().sum()) == 0


# --------------------------------------------------------------------------------------------------------- tiling invariance
@pytest.mark.parametrize("fusion", ["weighted", "max_confidence"])
def test_fuse_tiling_invariance(fusion):
    """The fuse kernel's row tiling changes which block writes which cell, never a result: explicit tilings 1, 3, 4, 23, R - 1, R
    and the automatic choice at B = 1, 5, 32 and 300 (above 264 the whole window is one tile) give the same bits as each other and
    match the oracles."""
    G, ppm, h, w, steps = 300, 20, 60, 80, 2
    R = 2 * int(MAX_D * ppm) + 1
    assert [_auto_rows_per_tile(b, R) for b in (1, 5, 32, 300)] == [4, 4, 23, R]
    Bmax = 300
    frames = [trajectory(600 + e, steps, h=h, w=w, bound_m=4.0, start_xy=(0.01 * (e % 17), -0.01 * (e % 13))) for e in range(Bmax)]
    values = np.random.default_rng(6).random((steps, Bmax, 1))
    orcs = [_oracle(1, G, ppm, fusion) for _ in range(Bmax)]
    for i in range(steps):
        for e in range(Bmax):
            orcs[e].update_map(values[i, e], frames[e][i].depth, frames[e][i].tf, MIN_D, MAX_D, FOV)
    runs = [(5, rpt) for rpt in (1, 3, 4, 23, R - 1, R)] + [(b, 0) for b in (1, 5, 32, 300)]
    first = None
    for B, rpt in runs:
        eng = _engine(B, 1, G, ppm, fusion)
        eng.rows_per_tile = rpt
        for i in range(steps):
            depth = torch.from_numpy(np.stack([frames[e][i].depth for e in range(B)])).cuda()
            tf = torch.from_numpy(np.stack([frames[e][i].tf for e in range(B)])).cuda()
            eng.update(torch.from_numpy(values[i, :B].copy()).cuda(), depth, tf, MIN_D, MAX_D, FOV)
        for e in range(B):
            _check(eng, e, orcs[e], f"B={B} rows_per_tile={rpt} env {e}")
        k = min(B, 5)                                 # the environments every run has
        conf, val = eng.conf[:k].cpu().numpy(), eng.value[:k].cpu().numpy()
        if first is None:
            first = (conf, val)
        assert np.array_equal(conf.view(np.uint32), first[0][:k].view(np.uint32)), f"B={B} rows_per_tile={rpt}: confidence bits"
        assert np.array_equal(val.view(np.uint32), first[1][:k].view(np.uint32)), f"B={B} rows_per_tile={rpt}: value bits"
        del eng
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------- slots, partial batches, resets, explored
@pytest.mark.parametrize("fusion", ["weighted", "max_confidence"])
def test_slots_partial_batches_reset_and_explored(fusion):
    B, G, C, steps = 4, 400, 2, 9
    explored = torch.zeros((B, G, G), dtype=torch.uint8, device="cuda")
    host = [np.zeros((G, G), bool) for _ in range(B)]
    eng = _engine(B, C, G, 20, fusion)
    mk = lambda s: _oracle(C, G, 20, fusion, explored_fn=lambda: host[s])
    orcs = [mk(s) for s in range(B)]
    frames = [trajectory(700 + s, steps, h=120, w=160, bound_m=4.0) for s in range(B)]
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:G, 0:G]
    for i in range(steps):
        slots = [[2, 0, 3, 1], [1, 3], [0, 1, 2, 3], [3], [2, 1]][i % 5]
        if i == 5:
            eng.reset(1)
            orcs[1] = mk(1)
        for s in range(B):                            # a moving, growing explored disc per slot
            cy, cx = G / 2 + 50 * np.cos(i + s), G / 2 + 50 * np.sin(i - s)
            host[s] = ((yy - cy) ** 2 + (xx - cx) ** 2) < (80 + 12 * i) ** 2
            explored[s] = torch.from_numpy(host[s].astype(np.uint8))
        before = {s: (eng.conf[s].clone(), eng.value[s].clone()) for s in range(B) if s not in slots}
        _step(eng, orcs, [frames[s][i] for s in slots], rng.random((len(slots), C)), slots=slots, explored=explored)
        for s, (cf, vl) in before.items():
            assert torch.equal(eng.conf[s].view(torch.int32), cf.view(torch.int32)), f"step {i}: slot {s} not in the call changed"
            assert torch.equal(eng.value[s].view(torch.int32), vl.view(torch.int32)), f"step {i}: slot {s} not in the call changed"
        for s in range(B):
            _check(eng, s, orcs[s], f"{fusion} step {i} slot {s}")
    assert all(o._map.any() for o in orcs)
    assert all((~h & (o._map > 0)).sum() == 0 for h, o in zip(host, orcs) if o is not orcs[1])


def test_off_grid_camera_in_a_batch():
    """Row 0 of a call with permuted slots has its camera off the grid: the flag lands on that row's SLOT (status is per slot,
    like the grids, so reset(slot) clears it), its grids are untouched and the other rows still match their oracles."""
    B, G, steps = 3, 400, 3
    eng = _engine(B, 1, G, 20, "max_confidence")
    orcs = [_oracle(1, G, 20, "max_confidence") for _ in range(B)]
    frames = [trajectory(800 + s, steps, h=120, w=160, bound_m=4.0) for s in range(B)]
    rng = np.random.default_rng(8)
    _step(eng, orcs, [frames[s][0] for s in range(B)], rng.random((B, 1)))
    slots = [2, 0, 1]
    off = dataclasses.replace(frames[2][1], tf=tf_from_pose(40.0, -3.0, 0.88, 0.4))      # 800 cells past the grid's edge
    before = (eng.conf[2].clone(), eng.value[2].clone())
    vals = rng.random((B, 1))
    for i, s in enumerate(slots[1:], 1):
        orcs[s].update_map(vals[i], frames[s][1].depth, frames[s][1].tf, MIN_D, MAX_D, FOV)
    rows = [off, frames[0][1], frames[1][1]]
    eng.update(torch.from_numpy(vals).cuda(), torch.from_numpy(np.stack([r.depth for r in rows])).cuda(),
               torch.from_numpy(np.stack([r.tf for r in rows])).cuda(), MIN_D, MAX_D, FOV,
               slots=torch.tensor(slots, dtype=torch.int32, device="cuda"))
    st = eng.status.cpu().numpy()
    assert st[2] == _lib.ST_CAMERA_OFF_GRID and st[0] == 0 and st[1] == 0, st
    assert torch.equal(eng.conf[2], before[0]) and torch.equal(eng.value[2], before[1])
    for s in range(B):
        _check(eng, s, orcs[s], f"slot {s}")
    eng.reset(2)
    orcs[2] = _oracle(1, G, 20, "max_confidence")
    assert int(eng.status.abs().sum()) == 0
    _step(eng, orcs, [frames[s][2] for s in range(B)], rng.random((B, 1)))
    for s in range(B):
        _check(eng, s, orcs[s], f"after reset, slot {s}")
    assert int(eng.status.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------------------- disc median
def _median_points(G, radius, rng):
    """Centres on every edge and corner (the crop is clipped), one cell inside the clipping distance, and random interior cells."""
    e = [0, 1, max(radius - 1, 0), radius, G // 2, G - 1 - radius, G - 2, G - 1]
    pts = [(r, c) for r in e for c in e]
    pts += [tuple(p) for p in rng.integers(0, G, (40, 2))]
    return np.array(pts)


def _want(grid, pts, radius, dtype):
    """np.median of the reference's crop-and-disc selection on the grid in the reference's dtype, per channel (-1: empty disc)."""
    g = grid.astype(dtype)
    return np.array([[float(disc_reduce(g[..., c], tuple(int(v) for v in p), radius)) for c in range(g.shape[-1])] for p in pts])


def _synthetic_grid(G, C, rng):
    """Random float32 values with regions of different density: dense, sparse (discs of 1, 2, 3 ... cells), and an all-zero block
    holding a single non-zero cell at its centre."""
    v = rng.random((G, G, C), dtype=np.float32) + np.float32(1e-3)
    dens = np.full((G, G), 0.5)
    dens[:, : G // 3] = 0.9
    dens[G // 2 :, G // 3 : 2 * G // 3] = 0.004
    v[rng.random((G, G)) >= dens] = 0
    z0 = 2 * G // 3 + 8
    v[z0 - 40 : z0 + 40, z0 - 40 : z0 + 40] = 0
    v[z0, z0] = np.float32(0.625)
    return v, (z0, z0)


@pytest.mark.parametrize("fusion", ["weighted", "max_confidence", "replace", "equal_max_confidence"])
def test_disc_median_is_np_median(fusion):
    """disc_median and disc_median_batch equal np.median exactly: the midpoint of an even count is averaged in float64 for weighted
    maps and in float32 for the others, as np.median does on the reference's grid.  Radii 0..31 cover both kernel instantiations
    (1024 and 4096 candidates) and the switch between them at 15 / 16."""
    B, C, G = 3, 2, 200
    eng = _engine(B, C, G, 20, fusion)
    dtype = np.float64 if eng.ref_float64 else np.float32
    rng = np.random.default_rng(9)
    # grids built by the engine ...
    frames = [trajectory(900 + s, 6, h=120, w=160, bound_m=3.0) for s in range(B)]
    for i in range(6):
        depth = torch.from_numpy(np.stack([frames[s][i].depth for s in range(B)])).cuda()
        tf = torch.from_numpy(np.stack([frames[s][i].tf for s in range(B)])).cuda()
        eng.update(torch.from_numpy(rng.random((B, C))).cuda(), depth, tf, MIN_D, MAX_D, FOV)
    built = eng.value.cpu().numpy()
    # ... and random grids with controlled densities (distinct float32 values, so even counts separate the two precisions)
    synth, lone = zip(*[_synthetic_grid(G, C, rng) for _ in range(B)])
    counts = {"zero": 0, "one": 0, "odd": 0, "even": 0}
    for grids in (built, np.stack(synth)):
        eng.value.copy_(torch.from_numpy(np.ascontiguousarray(grids)))
        for radius in (0, 10, 15, 16, 20, 25, 31):
            srl = []
            for s in range(B):
                pts = _median_points(G, radius, rng)
                if grids is not built:
                    pts = np.concatenate([pts, [lone[s], (lone[s][0] + 3, lone[s][1] - 2), (lone[s][0] - 30, lone[s][1] + 30)]])
                got = eng.disc_median(s, pts, radius)
                want = _want(grids[s], pts, radius, dtype)
                bad = np.flatnonzero((got != want).any(axis=1))
                assert bad.size == 0, f"slot {s} radius {radius}: {bad.size} points differ, e.g. {pts[bad[0]]}: {got[bad[0]]} vs {want[bad[0]]}"
                srl.append(np.concatenate([np.full((len(pts), 1), s), pts], axis=1))
                for p in pts:
                    g = grids[s]
                    r0, c0 = max(0, p[0] - radius), max(0, p[1] - radius)
                    crop = g[r0 : p[0] + radius + 1, c0 : p[1] + radius + 1, 0]
                    disc = cv2.circle(np.zeros(crop.shape, np.uint8), (radius, radius), radius, 255, -1)
                    n = int(((crop > 0) & (disc > 0)).sum())
                    counts["zero" if n == 0 else "one" if n == 1 else "odd" if n & 1 else "even"] += 1
            srl = np.concatenate(srl)
            perm = rng.permutation(len(srl))                       # slots interleaved in one launch
            got = eng.disc_median_batch(srl[perm], radius)
            want = np.concatenate([_want(grids[s], srl[srl[:, 0] == s, 1:], radius, dtype) for s in range(B)])[perm]
            assert np.array_equal(got, want), f"disc_median_batch radius {radius}: {(got != want).any(axis=1).sum()} points differ"
    assert min(counts.values()) > 0, counts


# --------------------------------------------------------------------------------------------------------- frontier scoring
def _ref_sorted(o, fr, radius):
    """ValueMap.sort_waypoints(fr, radius) on the oracle, with a NaN frontier scored -1 (the documented choice of frontier_values;
    the reference's int(NaN) raises ValueError)."""
    ok = ~np.isnan(fr).any(axis=1)
    if ok.all():
        return o.sort_waypoints(fr, radius)
    with pytest.raises(ValueError):
        o.sort_waypoints(fr, radius)
    values = [o.sort_waypoints(fr[i : i + 1], radius)[1][0] if ok[i] else -1 for i in range(len(fr))]
    order = np.argsort([-v for v in values])
    return np.array([fr[i] for i in order]), [values[i] for i in order]


@pytest.mark.parametrize("link", [False, True], ids=["plain", "explored_link"])
@pytest.mark.parametrize("fusion", ["weighted", "max_confidence"])
def test_frontier_values_is_sort_waypoints(fusion, link):
    """frontier_values (what FullStep's frontier scoring runs) returns every environment's frontiers and values as
    ValueMap.sort_waypoints(frontiers, 0.5) does: cells by int() truncation of the metre coordinates."""
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
    from vlfm_b200.mapping.value_map import frontier_values

    B, G, ppm, (h, w), steps = 3, 400, 20, (120, 160), 6
    fx = focal_from_hfov(w)
    omb = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=-1, size=G)
    oo = [ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=-1, size=G) for _ in range(B)]
    vmb = _engine(B, 1, G, ppm, fusion)
    vo = [_oracle(1, G, ppm, fusion, explored_fn=(lambda e=e: oo[e].explored_area) if link else None) for e in range(B)]
    frames = [trajectory(40 + e, steps, h=h, w=w, bound_m=2.5) for e in range(B)]
    rng = np.random.default_rng(10)
    scored = 0
    for i in range(steps):
        rows = [frames[e][i] for e in range(B)]
        for e in range(B):
            oo[e].update_map(rows[e].depth, rows[e].tf, MIN_D, MAX_D, fx, fx, FOV)
        depth = torch.from_numpy(np.stack([r.depth for r in rows])).cuda()
        tfs = np.stack([r.tf for r in rows])
        omb.update(depth, tfs, torch.from_numpy(tfs.reshape(B, 16)).cuda(), MIN_D, MAX_D, fx, fx, FOV)
        _step(vmb, vo, rows, rng.random((B, 1)), explored=omb.explored if link else None)
        got = frontier_values(omb, vmb, B, 0.5)
        grids = vmb.value.cpu().numpy()
        for e in range(B):
            fr = np.asarray(oo[e].frontiers)
            gw, gv = got[e]
            if len(fr) == 0:
                assert len(gw) == 0 and gv == []
                continue
            scored += len(fr)
            if not vmb.ref_float64:                       # bit-exact grids: the reference's own order and values
                ww, wv = _ref_sorted(vo[e], fr, 0.5)
                assert np.array_equal(gw, ww, equal_nan=True), f"step {i} env {e}: order"
                assert [float(v) for v in gv] == [float(v) for v in wv], f"step {i} env {e}: values"
                continue
            # weighted: exactly np.median on the read-back grid (float64, as the reference's grid) at the same cells ...
            rb = ValueMapOracle(1, size=G, use_max_confidence=False, pixels_per_meter=ppm)
            rb._value_map = grids[e].astype(np.float64)
            ww, wv = _ref_sorted(rb, fr, 0.5)
            assert np.array_equal(gw, ww, equal_nan=True), f"step {i} env {e}: order"
            assert [float(v) for v in gv] == [float(v) for v in wv], f"step {i} env {e}: values"
            # ... and within 1e-6 of the reference's float64 grid, frontier by frontier
            rw, rv = _ref_sorted(vo[e], fr, 0.5)
            key = lambda ws, vs: {tuple(np.nan_to_num(p, nan=-1e9)): float(v) for p, v in zip(ws, vs)}
            kg, kr = key(gw, gv), key(rw, rv)
            assert kg.keys() == kr.keys() and max(abs(kg[k] - kr[k]) for k in kg) <= VAL_TOL, f"step {i} env {e}"
    assert scored > 10


def test_frontier_values_nan_midpoint_scores_minus_one():
    """A zero-length frontier piece has a NaN midpoint; frontier_values scores it -1 (the reference's int(NaN) would raise) and the
    other frontiers of every environment keep their values."""
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
    from vlfm_b200.mapping.value_map import frontier_values

    B, G = 2, 200
    omb = ObstacleMapBatch(B, 0.61, 0.88, 0.18, size=G)
    vmb = _engine(B, 1, G, 20, "max_confidence")
    v = np.zeros((B, G, G, 1), np.float32)
    v[0, 90:110, 90:110] = 0.25
    v[1, 40:60, 120:140] = 0.75
    vmb.value.copy_(torch.from_numpy(v))
    px = [np.array([[100.0, 100.0], [np.nan, np.nan], [10.0, 10.0]]), np.array([[np.nan, np.nan], [130.5, 50.5]])]
    for e, p in enumerate(px):
        omb.frontiers[e, : len(p)] = torch.from_numpy(p).cuda()
        omb.count[e] = len(p)
    got = frontier_values(omb, vmb, B, 0.5)
    vals = [[float(x) for x in gv] for _, gv in got]
    assert vals == [[0.25, -1.0, -1.0], [0.75, -1.0]], vals
    assert np.isnan(got[0][0][1:]).any() and np.isnan(got[1][0][1]).all()
    o = ValueMapOracle(1, size=G)
    with pytest.raises(ValueError):
        o.sort_waypoints(omb.px_to_xy(px[1]), 0.5)


# ------------------------------------------------------------------------------------------------------ refused arguments
def test_bad_arguments_are_refused_without_a_launch():
    lib = _lib.load()
    st = _lib.stream_ptr()
    buf = torch.zeros(1 << 16, dtype=torch.float64, device="cuda")
    P = buf.data_ptr()

    def params(C=1, R=201):
        return _lib.ValueParams(48, 64, 300, C, R, 20, 4.5, 0.5, 0.35, 0, 0)

    def update(p, batch):
        return lib.vlfm_value_update(ctypes.byref(p), batch, None, P, P, P, P, P, P, P, None, P, P, st)

    refused = [
        ("C 9", lambda: update(params(C=9), 1)),
        ("C 0", lambda: update(params(C=0), 1)),
        ("even R", lambda: update(params(R=200), 1)),
        ("batch 65536", lambda: update(params(), 65536)),
        ("median radius 32", lambda: lib.vlfm_value_disc_median(300, 1, 0, P, P, 1, 32, 0, P, P, st)),
        ("median radius -1", lambda: lib.vlfm_value_disc_median(300, 1, 0, P, P, 1, -1, 1, P, P, st)),
        ("batch median radius 32", lambda: lib.vlfm_value_disc_median_batch(300, 1, P, P, 1, 32, 0, P, P, st)),
        ("batch median radius -1", lambda: lib.vlfm_value_disc_median_batch(300, 1, P, P, 1, -1, 1, P, P, st)),
    ]
    empty = [
        ("update batch 0", lambda: update(params(), 0)),
        ("update batch -1", lambda: update(params(), -1)),
        ("mask batch 0", lambda: lib.vlfm_value_mask_unexplored(300, 1, 0, None, P, P, P, st)),
        ("median npoints 0", lambda: lib.vlfm_value_disc_median(300, 1, 0, P, P, 0, 10, 0, P, P, st)),
        ("median npoints -3", lambda: lib.vlfm_value_disc_median(300, 1, 0, P, P, -3, 10, 1, P, P, st)),
        ("batch median npoints 0", lambda: lib.vlfm_value_disc_median_batch(300, 1, P, P, 0, 10, 0, P, P, st)),
        ("batch median npoints -3", lambda: lib.vlfm_value_disc_median_batch(300, 1, P, P, -3, 20, 1, P, P, st)),
    ]
    torch.cuda.synchronize()
    for want, calls in ((VLFM_E_INVALID, refused), (_lib.VLFM_OK, empty)):
        for name, call in calls:
            before = _lib.launch_count()
            rc = call()
            assert rc == want, f"{name} returned {rc}"
            assert _lib.launch_count() == before, f"{name}: a kernel was launched"
    torch.cuda.synchronize()
    assert int(buf.abs().sum()) == 0, "a refused call wrote to memory"
