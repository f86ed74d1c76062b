"""Map frames on the GPU (csrc/render.cu, mapping/render.py) against cv2 and the reference, bit for bit."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

import make_visualize_golden as mg  # noqa: E402
import visualize_oracle as vo  # noqa: E402
from vlfm_b200 import _lib  # noqa: E402
from vlfm_b200.mapping import render  # noqa: E402

pytestmark = pytest.mark.gpu


def random_primitive(rng, g):
    def pt(far):
        if far:
            return [int(v) for v in rng.integers(-50 * g, 51 * g, 2)]
        edge = rng.random() < 0.3
        if edge:
            return [int(rng.choice([-1, 0, g - 1, g])), int(rng.integers(-3, g + 3))][:: 1 if rng.random() < 0.5 else -1]
        return [int(v) for v in rng.integers(-25, g + 25, 2)]

    color = tuple(int(c) for c in rng.integers(0, 256, 3))
    if rng.random() < 0.55:
        p0 = pt(rng.random() < 0.15)
        r = rng.random()
        p1 = list(p0) if r < 0.1 else ([p0[0] + int(rng.integers(-4, 5)), p0[1] + int(rng.integers(-4, 5))] if r < 0.3 else pt(rng.random() < 0.15))
        return ("line", tuple(p0), tuple(p1), color, int(rng.integers(1, 8)) if rng.random() < 0.8 else int(rng.integers(8, render.MAX_THICKNESS + 1)))
    c = pt(False)
    r = int(rng.integers(0, 21)) if rng.random() < 0.8 else int(rng.integers(21, render.MAX_RADIUS + 1))
    t = int(rng.choice([-1, 1, 2, 3])) if rng.random() < 0.8 else int(rng.integers(4, render.MAX_THICKNESS + 1))
    return ("circle", tuple(c), r, color, t)


def cv2_draw(img, prims):
    for p in prims:
        if p[0] == "line":
            cv2.line(img, p[1], p[2], p[3], p[4])
        else:
            cv2.circle(img, p[1], p[2], p[3], p[4])
    return img


def records(prims):
    return [render.line_record(p[1], p[2], p[3], p[4]) if p[0] == "line" else render.circle_record(p[1], p[2], p[3], p[4]) for p in prims]


@pytest.mark.parametrize("g,n", [(64, 160), (257, 120), (1000, 24)])
def test_draw_list_matches_cv2(g, n):
    rng = np.random.default_rng(g)
    base = rng.integers(0, 256, (n, g, g, 3), dtype=np.uint8)
    lists = [[random_primitive(rng, g) for _ in range(int(rng.integers(0, 14)))] for _ in range(n)]
    frames = torch.from_numpy(base.copy()).cuda()
    render.DrawLists(frames.device).draw(frames, [records(l) for l in lists])
    got = frames.cpu().numpy()
    bad = [i for i in range(n) if not np.array_equal(got[i], cv2_draw(base[i].copy(), lists[i]))]
    assert not bad, f"{len(bad)} of {n} frames differ from cv2, first {bad[0]}: {lists[bad[0]]}"


def value_map_from(grid, maxconf, size):
    from vlfm_b200.mapping.value_map import ValueMap

    vm = ValueMap(grid.shape[-1], size=size, use_max_confidence=maxconf)
    vm._eng.value[0].copy_(torch.from_numpy(grid))
    return vm


def obstacle_map_from(g, size, frontiers):
    from vlfm_b200.mapping.obstacle_map import ObstacleMap

    om = ObstacleMap(0.61, 0.88, 0.18, size=size)
    set_obstacle(om, g, frontiers)
    return om


def set_obstacle(om, g, frontiers):
    om._eng.obst[0].copy_(torch.from_numpy(g["obst"]))
    om._eng.nav[0].copy_(torch.from_numpy(g["nav"]))
    om._eng.explored[0].copy_(torch.from_numpy(g["explored"]))
    if len(frontiers):
        om._eng.frontiers[0, : len(frontiers)].copy_(torch.from_numpy(np.asarray(frontiers, np.float64)))
    om._eng.count[0] = len(frontiers)
    om._front_cache = None


@pytest.mark.parametrize("case", mg.CASES, ids=[c[0] for c in mg.CASES])
def test_visualize_matches_reference_frames(live_golden, case):
    """ValueMap.visualize / ObstacleMap.visualize equal the frames the reference rendered on the same grids and trajectory."""
    z = live_golden("visualize")
    name, kind, ch, maxconf, red, masked, _neg, _zero, pad = case
    g = mg.grids_of(z, name)
    ref = mg.frames_of(z, name)
    xy, yaw, reset_at = z[f"{name}/xy"], z[f"{name}/yaw"], int(z[f"{name}/reset_at"][0])
    markers = [(z[f"{name}/marker_xy"][k], {"radius": int(z[f"{name}/marker_radius"][k]), "thickness": int(z[f"{name}/marker_thickness"][k]),
                                            "color": tuple(int(c) for c in z[f"{name}/marker_color"][k])}) for k in range(len(z[f"{name}/marker_xy"]))]
    om = obstacle_map_from(g, mg.G, z[f"{name}/frontiers_px"])
    if pad is not None:
        om.radius_padding_color = pad
    if kind == "value":
        from vlfm_b200.mapping.value_map import max_channels

        vm = value_map_from(g["value"], maxconf, mg.G)
        fn = max_channels if red == "max" else vo.itm_v3_reducer(mg.THRESH)
    for t in range(len(xy)):
        if t == reset_at:
            if kind == "value":
                vm.reset()
                vm._eng.value[0].copy_(torch.from_numpy(g["value"]))
            else:
                om.reset()
                set_obstacle(om, g, z[f"{name}/frontiers_px"])
        m = vm if kind == "value" else om
        m.update_agent_traj(xy[t], float(yaw[t]))
        got = vm.visualize(markers, reduce_fn=fn, obstacle_map=om if masked else None) if kind == "value" else om.visualize()
        assert got.dtype == np.uint8 and got.flags.c_contiguous
        assert np.array_equal(got, ref[t]), f"{name} step {t}: {(got != ref[t]).any(-1).sum()} pixels differ"


def synthetic_value(rng, size, ch, negative=False):
    v = np.zeros((size, size, ch), np.float32)
    yy, xx = np.mgrid[:size, :size]
    m = np.zeros((size, size), bool)
    for _ in range(12):
        cy, cx, r = rng.integers(0, size), rng.integers(0, size), rng.integers(10, size // 6)
        m |= (yy - cy) ** 2 + (xx - cx) ** 2 <= r * r
    v[m] = rng.uniform(-0.3 if negative else 0.0, 1.0, (int(m.sum()), ch)).astype(np.float32)
    return v


@pytest.mark.parametrize("size,ch,maxconf,host_fn,masked", [
    (1000, 1, False, False, False), (1000, 1, True, False, True), (1000, 2, True, False, False), (1000, 2, False, True, True),
    (260, 1, False, False, True), (260, 2, True, True, False)])
def test_value_visualize_trajectories(size, ch, maxconf, host_fn, masked):
    """every step of a synthetic trajectory (ITMPolicy-style markers; at G 260 the path and markers leave the map)"""
    from vlfm_b200.mapping.value_map import max_channels

    rng = np.random.default_rng(size + ch + 10 * maxconf + 100 * host_fn)
    grid = synthetic_value(rng, size, ch, negative=not maxconf)
    vm = value_map_from(grid, maxconf, size)
    ref_grid = grid.astype(np.float32 if maxconf else np.float64)
    explored = (rng.random((size, size)) < 0.97).astype(np.uint8) if masked else None
    om = None
    if masked:
        om = obstacle_map_from({"obst": np.zeros((size, size), np.uint8), "nav": np.ones((size, size), np.uint8), "explored": explored}, size, [])
    half = size / 2 / 20
    xy = np.cumsum(rng.normal(0, 0.4, (24, 2)), axis=0) + (half * 0.8 if size == 260 else 0)
    fn_dev = vo.itm_v3_reducer(0.4) if host_fn else max_channels
    fn_ref = vo.itm_v3_reducer(0.4) if host_fn else vo.max_reducer
    for t in range(len(xy)):
        front = xy[t] + rng.normal(0, 2.0, (5, 2))
        markers = [(f, {"radius": 5, "thickness": 2, "color": (0, 0, 255)}) for f in front]
        markers.append((front[2], {"radius": 5, "thickness": 2, "color": (0, 255, 255)}))
        yaw = float(rng.uniform(-np.pi, np.pi))
        vm.update_agent_traj(xy[t], yaw)
        got = vm.visualize(markers, reduce_fn=fn_dev, obstacle_map=om)
        ref = vo.value_frame(ref_grid, fn_ref, explored, list(xy[: t + 1]), yaw, markers, 20, np.array([size // 2, size // 2]))
        assert np.array_equal(got, ref), f"step {t}: {(got != ref).any(-1).sum()} pixels differ"


@pytest.mark.parametrize("edge,pad", [(False, (100, 100, 100)), (True, (0, 0, 0))])
def test_obstacle_visualize_explore(edge, pad):
    """ObstacleMap.visualize on explore trajectories (real frontiers from the device) against the oracle on the same grids"""
    from vlfm_b200.mapping.obstacle_map import ObstacleMap
    from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory

    size = 400
    fov = float(np.deg2rad(79.0))
    fx = focal_from_hfov(160)
    om = ObstacleMap(0.61, 0.88, 0.18, area_thresh=1.5, size=size)
    om.radius_padding_color = pad
    positions, drawn = [], 0
    for f in trajectory(7 if edge else 3, 8, h=120, w=160, bound_m=9.0 if edge else 3.0):
        try:
            om.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, fov)
        except IndexError:
            continue
        xy, yaw = f.tf[:2, 3].copy(), float(np.arctan2(f.tf[1, 0], f.tf[0, 0]))
        om.update_agent_traj(xy, yaw)
        positions.append(xy)
        got = om.visualize()
        ref = vo.obstacle_frame(om._map.astype(np.uint8), om._navigable_map, om.explored_area.astype(np.uint8), om._frontiers_px, pad,
                                positions, yaw, 20, np.array([size // 2, size // 2]))
        assert np.array_equal(got, ref), f"{(got != ref).any(-1).sum()} pixels differ"
        drawn += len(om._frontiers_px)
    assert drawn > 0


def test_batch_slots_and_side_effects():
    """B = 5 with permuted slots and one slot reset equals the per-environment renders; grids are untouched; repeats equal"""
    from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
    from vlfm_b200.mapping.value_map import ValueMapBatch

    rng = np.random.default_rng(5)
    b, size = 5, 300
    vb = ValueMapBatch(b, 2, size, use_max_confidence=False)
    for s in range(b):
        vb.value[s].copy_(torch.from_numpy(synthetic_value(rng, size, 2)))
    vb.reset(3)
    ob = ObstacleMapBatch(b, 0.61, 0.88, 0.18, size=size)
    ob.obst.copy_(torch.from_numpy((rng.random((b, size, size)) < 0.02).astype(np.uint8)))
    ob.nav.copy_(torch.from_numpy((rng.random((b, size, size)) < 0.9).astype(np.uint8)))
    ob.explored.copy_(torch.from_numpy((rng.random((b, size, size)) < 0.5).astype(np.uint8)))
    for s in range(b):
        k = int(rng.integers(0, 20))
        ob.frontiers[s, :k] = torch.from_numpy(rng.uniform(-5, size + 5, (k, 2)))
        ob.count[s] = k
    lists = [records([random_primitive(rng, size) for _ in range(6)]) for _ in range(b)]
    before = [t.clone() for t in (vb.value, vb.conf, ob.obst, ob.nav, ob.explored, ob.frontiers, ob.count)]
    perm = [3, 0, 4, 1, 2]
    slots = torch.tensor(perm, dtype=torch.int32, device="cuda")
    v_all = vb.render(slots=slots, explored=ob.explored, draw_lists=lists).cpu().numpy()
    o_all = ob.render(slots=slots, padding_color=(10, 20, 30), draw_lists=lists).cpu().numpy()
    for i, s in enumerate(perm):
        one = torch.tensor([s], dtype=torch.int32, device="cuda")
        assert np.array_equal(v_all[i], vb.render(slots=one, explored=ob.explored, draw_lists=[lists[i]]).cpu().numpy()[0])
        assert np.array_equal(o_all[i], ob.render(slots=one, padding_color=(10, 20, 30), draw_lists=[lists[i]]).cpu().numpy()[0])
    assert np.array_equal(v_all, vb.render(slots=slots, explored=ob.explored, draw_lists=lists).cpu().numpy())
    assert np.array_equal(o_all, ob.render(slots=slots, padding_color=(10, 20, 30), draw_lists=lists).cpu().numpy())
    for a, t in zip(before, (vb.value, vb.conf, ob.obst, ob.nav, ob.explored, ob.frontiers, ob.count)):
        assert torch.equal(a, t)


def test_empty_trajectory_equals_previous_host_rendering():
    """no trajectory: no agent and no markers -- the frame the former host implementation returned (it normalised in
    float32, so the map is a max-confidence one)"""
    rng = np.random.default_rng(9)
    size = 300
    grid = synthetic_value(rng, size, 1)
    vm = value_map_from(grid, True, size)        # max-confidence: float32 on both sides, as the former host rendering
    got = vm.visualize([(np.zeros(2), {"radius": 5, "color": (0, 0, 255), "thickness": 2})])
    reduced = np.max(grid, axis=-1)
    img = np.flipud(reduced)
    zero = img == 0
    img = img.copy()
    img[zero] = np.max(img)
    lo, hi = float(img.min()), float(img.max())
    norm = ((img - lo) / (hi - lo) * 255).astype(np.uint8) if hi > lo else np.zeros_like(img, np.uint8)
    old = cv2.applyColorMap(norm, cv2.COLORMAP_INFERNO)
    old[zero] = (255, 255, 255)
    assert np.array_equal(got, old)
    with pytest.raises(TypeError):
        vm.update_agent_traj(np.zeros(2), 0.0)
        vm.visualize([(np.zeros(2), {"radius": 5, "color": (0, 0, 255), "lineType": 8})])


def test_argument_errors_launch_nothing():
    lib = _lib.load()
    g, n = 64, 2
    frames = torch.zeros((n, g, g, 3), dtype=torch.uint8, device="cuda")
    red = torch.zeros((n, g, g), dtype=torch.float32, device="cuda")
    lut = render.inferno_lut(frames.device)
    ws = torch.zeros(4096, dtype=torch.float64, device="cuda")
    u8 = torch.zeros((n, g, g), dtype=torch.uint8, device="cuda")
    fr = torch.zeros((n, 16, 2), dtype=torch.float64, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    dev = torch.zeros(4096, dtype=torch.int32, device="cuda")
    st = _lib.stream_ptr()
    p = _lib.ptr
    torch.cuda.synchronize()
    before = _lib.launch_count()

    def draw(recs, offsets=None):
        offs = [0, len(recs), len(recs)] if offsets is None else offsets
        h = np.ascontiguousarray(np.asarray(offs + [v for r in recs for v in r], np.int32))
        return lib.vlfm_render_draw(g, n, p(frames), h.ctypes.data, h.size, p(dev), dev.numel(), st)

    good_line = [_lib.DRAW_LINE, 0, 0, 5, 5, 0, 2, 0xff]
    bad = [
        lib.vlfm_render_value(0, n, None, p(red), 0, None, p(lut), p(frames), p(ws), ws.numel() * 8, st),
        lib.vlfm_render_value(g, n, None, p(red), 2, None, p(lut), p(frames), p(ws), ws.numel() * 8, st),
        lib.vlfm_render_value(g, n, None, p(red), 0, None, p(lut), p(frames), p(ws), 8, st),
        lib.vlfm_render_value(g, n, None, None, 0, None, p(lut), p(frames), p(ws), ws.numel() * 8, st),
        lib.vlfm_render_obstacle(g, n, None, p(u8), p(u8), p(u8), p(fr), p(cnt), 16, 256, 0, 0, p(frames), st),
        lib.vlfm_render_obstacle(g, 0, None, p(u8), p(u8), p(u8), p(fr), p(cnt), 16, 0, 0, 0, p(frames), st),
        lib.vlfm_render_obstacle(g, n, None, p(u8), p(u8), p(u8), p(fr), p(cnt), 0, 0, 0, 0, p(frames), st),
        draw([good_line[:6] + [0] + good_line[7:]]),                    # line thickness 0
        draw([good_line[:6] + [17] + good_line[7:]]),                   # line thickness 17
        draw([[_lib.DRAW_CIRCLE, 3, 3, 0, 0, 256, 1, 0]]),              # radius 256
        draw([[_lib.DRAW_CIRCLE, 3, 3, 0, 0, 5, -2, 0]]),               # thickness -2
        draw([[7, 3, 3, 0, 0, 5, 1, 0]]),                               # unknown op
        draw([[_lib.DRAW_LINE, 1 << 24, 0, 0, 0, 0, 1, 0]]),            # coordinate out of range
        draw([good_line[:7] + [1 << 24]]),                              # colour above 24 bits
        draw([good_line], offsets=[0, 1, 0]),                           # decreasing offsets
        draw([good_line], offsets=[1, 1, 1]),                           # offsets[0] != 0
    ]
    assert all(rc == 1 for rc in bad), bad                              # VLFM_E_INVALID
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert not frames.any()
    with pytest.raises(ValueError):
        render.line_record((0, 0), (1, 1), (0, 0, 0), 17)
    with pytest.raises(ValueError):
        render.circle_record((0, 0), 300, (0, 0, 0), 1)
