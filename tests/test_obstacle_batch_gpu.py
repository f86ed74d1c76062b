"""ObstacleMapBatch: B environments per launch sequence (hole fill, scatter + dilate, explore half, frontiers) vs one oracle per
environment -- obstacle / navigable / explored grids bit-exact, ORDERED frontier lists identical; slots permuted, partial
batches, resets in the middle, S frames that grow with the episode."""
import numpy as np
import pytest
import torch

from oracle.obstacle_map_oracle import ObstacleMapOracle
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory

pytestmark = pytest.mark.gpu
FOV = np.deg2rad(79)


def _check(eng, slot, o, tag):
    assert np.array_equal(eng.obst[slot].cpu().numpy().astype(bool), o._map), f"{tag}: obstacle grid"
    assert np.array_equal(eng.nav[slot].cpu().numpy().astype(np.int64), np.asarray(o._navigable_map).astype(np.int64)), f"{tag}: navigable grid"
    assert np.array_equal(eng.explored[slot].cpu().numpy().astype(bool), o.explored_area), f"{tag}: explored area"
    fo, fg = np.asarray(o._frontiers_px), eng.frontiers_px(slot)
    assert fo.shape == fg.shape and np.array_equal(fo, fg), f"{tag}: frontiers {fg.shape} vs {fo.shape}"


@pytest.mark.parametrize("cfg", [
    dict(B=4, hw=(120, 160), size=400, steps=8, bound=2.5, hole=-1),
    dict(B=5, hw=(240, 320), size=1000, steps=7, bound=12.0, hole=100000),
    dict(B=3, hw=(240, 320), size=2000, steps=5, bound=30.0, hole=100000),
])
def test_batch_vs_per_env_oracles(cfg):
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch

    B, (h, w), G = cfg["B"], cfg["hw"], cfg["size"]
    fx = focal_from_hfov(w)
    eng = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=cfg["hole"], size=G)
    orc = [ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=cfg["hole"], size=G) for _ in range(B)]
    frames = [trajectory(40 + e, cfg["steps"], h=h, w=w, bound_m=cfg["bound"], start_xy=(0.002 * G * e / 2, -0.003 * G * e / 2)) for e in range(B)]
    for i in range(cfg["steps"]):
        for e in range(B):
            orc[e].update_map(frames[e][i].depth, frames[e][i].tf, 0.5, 5.0, fx, fx, FOV)
        depth = torch.from_numpy(np.stack([frames[e][i].depth for e in range(B)])).cuda()
        tfs = np.stack([frames[e][i].tf for e in range(B)])
        eng.update(depth, tfs, torch.from_numpy(tfs.reshape(B, 16)).cuda(), 0.5, 5.0, fx, fx, FOV)
        for e in range(B):
            _check(eng, e, orc[e], f"step {i} env {e}")
        fr = eng.all_frontiers_px()
        for e in range(B):
            assert np.array_equal(np.asarray(orc[e]._frontiers_px), fr[e])
    assert all(o.explored_area.sum() > 100 for o in orc)
    # the S frame is a strict sub-rectangle of the grid on the larger maps (that is what is being tested)
    if G >= 1000:
        fr = eng._frame(0)
        assert (fr[2] - fr[0]) * (fr[3] - fr[1]) < G * G // 2


def test_slots_partial_batches_and_reset():
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch

    B, h, w, G = 4, 120, 160, 600
    fx = focal_from_hfov(w)
    eng = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=60, size=G)
    orc = [ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=60, size=G) for _ in range(B)]
    frames = [trajectory(70 + e, 9, h=h, w=w, bound_m=6.0) for e in range(B)]
    for i in range(9):
        slots = [[2, 0, 3, 1], [1, 3], [0, 1, 2, 3], [3]][i % 4]           # rows of the call -> grid slots
        if i == 5:
            eng.reset(1)
            orc[1] = ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=60, size=G)
        for s in slots:
            orc[s].update_map(frames[s][i].depth, frames[s][i].tf, 0.5, 5.0, fx, fx, FOV)
        depth = torch.from_numpy(np.stack([frames[s][i].depth for s in slots])).cuda()
        tfs = np.stack([frames[s][i].tf for s in slots])
        eng.update(depth, tfs, torch.from_numpy(tfs.reshape(len(slots), 16)).cuda(), 0.5, 5.0, fx, fx, FOV, slots=slots)
        for s in range(B):
            if orc[s]._map.any() or s in slots:
                _check(eng, s, orc[s], f"step {i} slot {s}")


def test_graph_replay_with_static_buffers():
    """The steady state of an episode loop -- same device buffers every step -- is captured in a CUDA graph after two eager calls
    (launch geometry depends on the batch size only; the per-environment records travel in page-locked memory): every replayed
    step still matches the per-environment oracles, while the S frames grow."""
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch

    B, h, w, G = 3, 240, 320, 1000
    fx = focal_from_hfov(w)
    eng = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=100000, size=G)
    orc = [ObstacleMapOracle(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=100000, size=G) for _ in range(B)]
    frames = [trajectory(90 + e, 9, h=h, w=w, bound_m=12.0, start_xy=(2.0 * e, -1.0 * e)) for e in range(B)]
    depth = torch.empty(B, h, w, dtype=torch.float32, device="cuda")
    tfd = torch.empty(B, 16, dtype=torch.float64, device="cuda")
    for i in range(9):
        for e in range(B):
            orc[e].update_map(frames[e][i].depth, frames[e][i].tf, 0.5, 5.0, fx, fx, FOV)
        tfs = np.stack([frames[e][i].tf for e in range(B)])
        depth.copy_(torch.from_numpy(np.stack([frames[e][i].depth for e in range(B)])))
        tfd.copy_(torch.from_numpy(tfs.reshape(B, 16)))
        eng.update(depth, tfs, tfd, 0.5, 5.0, fx, fx, FOV)
        for e in range(B):
            _check(eng, e, orc[e], f"step {i} env {e}")
    assert eng.use_graph and len(eng.graphs.captured) == 1, "the update was never captured"
