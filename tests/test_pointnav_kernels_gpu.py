"""Every PointNav kernel of csrc/pointnav.cu on its own, against a float64 reference of the same operation (or bit-exact), at the
engine's shapes and at edges: identity, down- and up-scaling and odd frame sizes, 2 and 16 channels per group and a single
group, each residual kind, odd maps, GEMV batches around the warp and tile sizes.  Outputs are prefilled with NaN so an
unwritten element fails; launches are repeated and must reproduce their bits.  Plus a bad-argument table and a ptxas check."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.pointnav_oracle import area_resize
from vlfm_b200 import build

VLFM_E_INVALID = 1
U = 2.0 ** -24
f64 = torch.float64


def _lib():
    from vlfm_b200 import _lib as lib

    return lib


def _call(name, *args):
    lib = _lib()
    lib.check(getattr(lib.load(), name)(*args), name)


def _st():
    return _lib().stream_ptr()


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


# ------------------------------------------------------------------------------------------------------------ depth in
@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", [((224, 224), (224, 224)), ((480, 640), (224, 224)), ((120, 160), (212, 240)), ((97, 131), (30, 22)),
                                     ((212, 240), (212, 240))])
def test_depth_in(src, dst):
    B = 2
    g = torch.Generator().manual_seed(1)
    depth = torch.rand(B, *src, generator=g)
    depth[:, 5:9, 7:12] = 0
    IH, IW = dst
    PH, PW = IH // 2, IW // 2
    OH, OW = (PH - 1) // 2 + 1, (PW - 1) // 2 + 1
    col = _nan(B * OH * OW, 56, dtype=torch.float16)
    resized = _nan(B, IH, IW)
    d = depth.cuda()
    _call("vlfm_pointnav_depth_in", d.data_ptr(), B, src[0], src[1], IH, IW, col.data_ptr(), 56, resized.data_ptr(), _st())
    ref_r = area_resize(depth, dst)
    if src == dst:
        assert torch.equal(resized.cpu(), depth)
    else:
        # fp32 window sum of <= k terms then one division: <= (k + 1) u relative, values in [0, 1]
        k = -(-src[0] // IH + 1) * -(-src[1] // IW + 1)
        assert (resized.cpu().double() - F.adaptive_avg_pool2d(depth.double()[:, None], dst)[:, 0]).abs().max() <= (k + 2) * U
    pooled = F.avg_pool2d(ref_r.double()[:, None], 2)
    ref_col = F.unfold(pooled, 7, padding=3, stride=2).transpose(1, 2).reshape(B * OH * OW, 49)
    got = col.cpu().double()
    assert torch.equal(got[:, 49:], torch.zeros_like(got[:, 49:]))
    # the pooled value in fp32 (3 adds + exact /4: 4u relative to the resized values' rounding) then one fp16 rounding
    err = (got[:, :49] - ref_col).abs()
    assert (err <= ref_col.abs() * (2.0 ** -11 + 8 * U) + 64 * U).all()
    col2 = _nan(B * OH * OW, 56, dtype=torch.float16)
    _call("vlfm_pointnav_depth_in", d.data_ptr(), B, src[0], src[1], IH, IW, col2.data_ptr(), 56, None, _st())
    assert torch.equal(_bits(col), _bits(col2))


# ----------------------------------------------------------------------------------------------------------- GroupNorm
def _gn64(x, gamma, beta, G):
    B, HW, C = x.shape
    return F.group_norm(x.double().permute(0, 2, 1), G, gamma.double(), beta.double(), eps=1e-5).permute(0, 2, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("C,G,HW", [(32, 16, 112 * 112), (256, 16, 16), (128, 1, 16), (64, 16, 27 * 30), (48, 16, 7)])
@pytest.mark.parametrize("rmode", [0, 1, 2])
def test_groupnorm(C, G, HW, rmode):
    B = 3
    g = torch.Generator().manual_seed(C + G + rmode)
    x = torch.randn(B, HW, C, generator=g) * 3 + 1
    y = torch.randn(B, HW, C, generator=g) * 2 - 0.5
    r = torch.randn(B, HW, C, generator=g)
    ga, ba = 1 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    gb, bb = 1 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    dx, dy, dr = x.cuda(), y.cuda(), r.cuda()
    dga, dba, dgb, dbb = ga.cuda(), ba.cuda(), gb.cuda(), bb.cuda()
    o32, o16 = _nan(B, HW, C), _nan(B, HW, C, dtype=torch.float16)
    args = lambda out32, out16: (dx.data_ptr(), dga.data_ptr(), dba.data_ptr(), rmode, dr.data_ptr() if rmode == 1 else None,
                                 dy.data_ptr() if rmode == 2 else None, dgb.data_ptr() if rmode == 2 else None,
                                 dbb.data_ptr() if rmode == 2 else None, out32.data_ptr(), out16.data_ptr(), B, HW, C, G, 1e-5, 1, _st())
    _call("vlfm_pointnav_groupnorm", *args(o32, o16))
    ref = _gn64(x, ga, ba, G)
    if rmode == 1:
        ref = ref + r.double()
    elif rmode == 2:
        ref = ref + _gn64(y, gb, bb, G)
    ref = ref.clamp_min(0)
    # fp32 statistics over n = HW*C/G values: the mean's and variance's rounding ~ log2(n) u relative, times |x - mean| / std
    # ~ 4 here; a handful of fp32 operations per element after
    bar = 1e-5 * (1 + ref.abs())
    assert ((o32.cpu().double() - ref).abs() <= bar).all()
    assert torch.equal(o16.cpu(), o32.cpu().half())
    o32b, o16b = _nan(B, HW, C), _nan(B, HW, C, dtype=torch.float16)
    _call("vlfm_pointnav_groupnorm", *args(o32b, o16b))
    assert torch.equal(_bits(o32), _bits(o32b))


@pytest.mark.gpu
def test_groupnorm_in_place_residual():
    """out32 may alias the identity residual (the engine's block output)."""
    B, HW, C, G = 2, 50, 32, 16
    x, r = torch.randn(B, HW, C).cuda(), torch.randn(B, HW, C).cuda()
    ga, ba = torch.ones(C).cuda(), torch.zeros(C).cuda()
    out = _nan(B, HW, C)
    _call("vlfm_pointnav_groupnorm", x.data_ptr(), ga.data_ptr(), ba.data_ptr(), 1, r.data_ptr(), None, None, None, out.data_ptr(), None,
          B, HW, C, G, 1e-5, 0, _st())
    r2 = r.clone()
    _call("vlfm_pointnav_groupnorm", x.data_ptr(), ga.data_ptr(), ba.data_ptr(), 1, r2.data_ptr(), None, None, None, r2.data_ptr(), None,
          B, HW, C, G, 1e-5, 0, _st())
    assert torch.equal(out, r2)


# ------------------------------------------------------------------------------------------------------ pool and gather
@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C", [(112, 112, 32), (106, 120, 32), (7, 9, 8), (1, 3, 16)])
def test_maxpool_and_gather(H, W, C):
    B = 2
    x = torch.randn(B, H, W, C)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    o32, o16 = _nan(B, Ho, Wo, C), _nan(B, Ho, Wo, C, dtype=torch.float16)
    dx = x.cuda()
    _call("vlfm_pointnav_maxpool3s2", dx.data_ptr(), o32.data_ptr(), o16.data_ptr(), B, H, W, C, _st())
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(o32.cpu(), ref)
    assert torch.equal(o16.cpu(), ref.half())
    if C % 8 == 0:
        x16 = dx.half()
        g = _nan(B * Ho * Wo, C, dtype=torch.float16)
        _call("vlfm_pointnav_gather_s2", x16.data_ptr(), g.data_ptr(), B, H, W, C, _st())
        assert torch.equal(g.cpu(), x16.cpu()[:, ::2, ::2, :].reshape(-1, C))


# ---------------------------------------------------------------------------------------------------------------- GEMV
@pytest.mark.gpu
@pytest.mark.parametrize("N,K", [(2048, 1088), (512, 2048), (2048, 1024), (13, 36)])
def test_gemv_f32(N, K):
    g = torch.Generator().manual_seed(N + K)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    X = torch.randn(65, K + 4, generator=g)
    dW, db, dX = W.cuda(), bias.cuda(), X.cuda()
    ref = X[:, :K].double() @ W.double().T + bias.double()
    rows = {}
    for B in (1, 2, 31, 32, 33, 64):
        y = _nan(B, N + 3)
        _call("vlfm_pointnav_gemv_f32", dX.data_ptr(), K + 4, dW.data_ptr(), K, db.data_ptr(), y.data_ptr(), N + 3, B, N, K, 0, _st())
        yc = y.cpu()
        assert torch.isnan(yc[:, N:]).all()
        # fp32 dot product of K terms: |err| <= ~ (K/32 + 5) u sum |x w| per lane-and-tree order
        bound = (K / 32 + 8) * U * (X[:B, :K].double().abs() @ W.double().abs().T) + 2 * U * ref[:B].abs()
        assert ((yc[:, :N].double() - ref[:B]).abs() <= bound).all()
        for b in range(B):
            rows.setdefault(b, yc[b, :N]).equal(yc[b, :N]) or pytest.fail(f"row {b} differs at B={B}")
        y2 = _nan(B, N + 3)
        _call("vlfm_pointnav_gemv_f32", dX.data_ptr(), K + 4, dW.data_ptr(), K, db.data_ptr(), y2.data_ptr(), N + 3, B, N, K, 0, _st())
        assert torch.equal(_bits(y), _bits(y2))
    yr = _nan(3, N)
    _call("vlfm_pointnav_gemv_f32", dX.data_ptr(), K + 4, dW.data_ptr(), K, db.data_ptr(), yr.data_ptr(), N, 3, N, K, 1, _st())
    assert torch.equal(yr.cpu(), torch.stack([rows[i] for i in range(3)]).clamp_min(0))
    bad = _lib().load().vlfm_pointnav_gemv_f32(dX.data_ptr(), K + 4, dW.data_ptr(), K, db.data_ptr(), yr.data_ptr(), N, 65, N, K, 0, _st())
    assert bad == VLFM_E_INVALID


# ---------------------------------------------------------------------------------------------------------------- LSTM
@pytest.mark.gpu
@pytest.mark.parametrize("discrete", [True, False])
def test_lstm_prep_cell_head(discrete):
    """prep (mask, goal and prev-action features, permuted env slots) -> layer-0 cell -> layer-1 cell + head + write-back,
    with the gate pre-activations given (the GEMVs are tested above), against float64."""
    B, E, H = 3, 5, 512
    g = torch.Generator().manual_seed(int(discrete))
    state = torch.randn(E, 4, H, generator=g) * 2
    prev = torch.tensor([[1], [3], [0], [2], [1]]) if discrete else torch.randn(E, 2, generator=g).tanh()
    env_ids = torch.tensor([4, 0, 2], dtype=torch.int32)
    masks = torch.tensor([1, 0, 1], dtype=torch.uint8)
    goal = torch.tensor([[1.5, 0.3], [4.0, -2.9], [0.2, 3.1]])
    wg, bg = torch.randn(32, 3, generator=g), torch.randn(32, generator=g)
    wp = torch.randn(5, 32, generator=g) if discrete else torch.randn(32, 2, generator=g)
    bp = None if discrete else torch.randn(32, generator=g)
    gates0, gates1 = torch.randn(B, 4 * H, generator=g) * 2, torch.randn(B, 4 * H, generator=g) * 2
    wh, bh = torch.randn(4, H, generator=g) / 8, torch.randn(4, generator=g)
    cu = lambda t: None if t is None else t.cuda()
    d = {k: cu(v) for k, v in dict(state=state, prev=prev, env_ids=env_ids, masks=masks, goal=goal, wg=wg, bg=bg, wp=wp, bp=bp,
                                   gates0=gates0, gates1=gates1, wh=wh, bh=bh).items()}
    xin0, xin1, cbuf = _nan(B, 1088), _nan(B, 1024), _nan(B, 1024)
    xin0[:, :512] = 0
    _call("vlfm_pointnav_lstm_prep", d["env_ids"].data_ptr(), d["state"].data_ptr(), d["prev"].data_ptr(), int(discrete),
          d["masks"].data_ptr(), d["goal"].data_ptr(), d["wg"].data_ptr(), d["bg"].data_ptr(), d["wp"].data_ptr(), _lib().ptr(d["bp"]),
          xin0.data_ptr(), xin1.data_ptr(), cbuf.data_ptr(), B, _st())
    m = masks.bool()
    s = state[env_ids.long()].double() * m[:, None, None]
    gf = torch.stack([goal[:, 0], torch.cos(-goal[:, 1]), torch.sin(-goal[:, 1])], -1).double()
    ref_goal = gf @ wg.double().T + bg.double()
    if discrete:
        ref_prev = wp.double()[torch.where(m, prev[env_ids.long(), 0] + 1, 0)]
    else:
        ref_prev = (prev[env_ids.long()].double() * m[:, None]) @ wp.double().T + bp.double()
    x0 = xin0.cpu().double()
    assert (x0[:, 512:544] - ref_goal).abs().max() < 1e-5
    assert (x0[:, 544:576] - ref_prev).abs().max() < 1e-5
    assert torch.equal(x0[:, 576:], s[:, 0]) and torch.equal(xin1.cpu().double()[:, 512:], s[:, 1])
    assert torch.equal(cbuf.cpu().double(), torch.cat([s[:, 2], s[:, 3]], 1))

    def cell(gt, c):
        i, f, gg, o = gt.double().chunk(4, 1)
        c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        return torch.sigmoid(o) * torch.tanh(c2), c2

    _call("vlfm_pointnav_lstm_cell", d["gates0"].data_ptr(), cbuf.data_ptr(), xin1.data_ptr(), B, _st())
    h0, c0 = cell(gates0, s[:, 2])
    assert (xin1.cpu().double()[:, :512] - h0).abs().max() < 1e-5 and (cbuf.cpu().double()[:, :512] - c0).abs().max() < 1e-5
    feat, head = _nan(B, H), _nan(B, 4)
    action = torch.full((B, 1), -7, dtype=torch.long, device="cuda") if discrete else _nan(B, 2)
    _call("vlfm_pointnav_lstm_head", d["gates1"].data_ptr(), cbuf.data_ptr(), xin1.data_ptr(), d["wh"].data_ptr(), d["bh"].data_ptr(),
          int(discrete), d["env_ids"].data_ptr(), d["state"].data_ptr(), d["prev"].data_ptr(), feat.data_ptr(), head.data_ptr(),
          action.data_ptr(), B, _st())
    h1, c1 = cell(gates1, s[:, 3])
    ref_head = h1 @ wh.double().T + bh.double()
    assert (feat.cpu().double() - h1).abs().max() < 1e-5
    assert (head.cpu().double() - ref_head).abs().max() < 1e-4
    new = d["state"].cpu().double()
    ref_state = torch.stack([h0, h1, c0, c1], 1)
    assert (new[env_ids.long()] - ref_state).abs().max() < 1e-5
    untouched = [1, 3]
    assert torch.equal(new[untouched], state[untouched].double())
    hc = head.cpu()
    if discrete:
        assert torch.equal(action.cpu()[:, 0], hc.argmax(1))
        assert torch.equal(d["prev"].cpu()[env_ids.long()], action.cpu())
    else:
        assert (action.cpu() - torch.tanh(hc[:, :2])).abs().max() < 1e-6
        assert torch.equal(d["prev"].cpu()[env_ids.long()], action.cpu())


@pytest.mark.gpu
def test_head_argmax_first_index_on_ties():
    B, H = 1, 512
    gates = torch.zeros(B, 4 * H, device="cuda")
    cbuf, xin1 = torch.zeros(B, 1024, device="cuda"), torch.zeros(B, 1024, device="cuda")
    wh = torch.zeros(4, H, device="cuda")
    bh = torch.tensor([0.5, 2.0, 2.0, 1.0], device="cuda")
    state = torch.zeros(1, 4, H, device="cuda")
    prev = torch.zeros(1, 1, dtype=torch.long, device="cuda")
    ids = torch.zeros(1, dtype=torch.int32, device="cuda")
    action = torch.full((1, 1), -1, dtype=torch.long, device="cuda")
    _call("vlfm_pointnav_lstm_head", gates.data_ptr(), cbuf.data_ptr(), xin1.data_ptr(), wh.data_ptr(), bh.data_ptr(), 1, ids.data_ptr(),
          state.data_ptr(), prev.data_ptr(), None, None, action.data_ptr(), B, _st())
    assert action.item() == 1 and prev.item() == 1


# --------------------------------------------------------------------------------------------------------- bad arguments
@pytest.mark.gpu
def test_bad_arguments():
    lib = _lib().load()
    p = torch.zeros(4096, device="cuda")
    a = p.data_ptr()
    st = _st()
    calls = [
        lambda: lib.vlfm_pointnav_depth_in(a, 1, 10, 10, 8, 8, a, 50, None, st),          # ldk % 8
        lambda: lib.vlfm_pointnav_depth_in(None, 1, 10, 10, 8, 8, a, 56, None, st),
        lambda: lib.vlfm_pointnav_depth_in(a, 1, 10, 10, 1, 8, a, 56, None, st),          # input too small
        lambda: lib.vlfm_pointnav_groupnorm(a, a, a, 0, None, None, None, None, a, None, 1, 4, 30, 16, 1e-5, 1, st),   # C % G
        lambda: lib.vlfm_pointnav_groupnorm(a, a, a, 1, None, None, None, None, a, None, 1, 4, 32, 16, 1e-5, 1, st),   # no r
        lambda: lib.vlfm_pointnav_groupnorm(a, a, a, 2, None, a, None, None, a, None, 1, 4, 32, 16, 1e-5, 1, st),      # no GN_b
        lambda: lib.vlfm_pointnav_groupnorm(a, a, a, 3, None, None, None, None, a, None, 1, 4, 32, 16, 1e-5, 1, st),
        lambda: lib.vlfm_pointnav_groupnorm(a, a, a, 0, None, None, None, None, None, None, 1, 4, 32, 16, 1e-5, 1, st),  # no output
        lambda: lib.vlfm_pointnav_maxpool3s2(a, None, None, 1, 4, 4, 8, st),
        lambda: lib.vlfm_pointnav_gather_s2(a, a, 1, 4, 4, 12, st),                        # C % 8
        lambda: lib.vlfm_pointnav_gather_s2(a + 2, a, 1, 4, 4, 16, st),                    # misaligned
        lambda: lib.vlfm_pointnav_gemv_f32(a, 8, a, 8, None, a, 8, 0, 8, 8, 0, st),
        lambda: lib.vlfm_pointnav_gemv_f32(a, 8, a, 8, None, a, 8, 65, 8, 8, 0, st),
        lambda: lib.vlfm_pointnav_gemv_f32(a, 8, a, 8, None, a, 8, 1, 8, 6, 0, st),        # K % 4
        lambda: lib.vlfm_pointnav_gemv_f32(a + 4, 8, a, 8, None, a, 8, 1, 8, 8, 0, st),    # misaligned x
        lambda: lib.vlfm_pointnav_gemv_f32(a, 4, a, 8, None, a, 8, 1, 8, 8, 0, st),        # ldx < K
        lambda: lib.vlfm_pointnav_lstm_prep(a, a, a, 0, a, a, a, a, a, None, a, a, a, 1, st),   # continuous without bias
        lambda: lib.vlfm_pointnav_lstm_cell(a, a, None, 1, st),
        lambda: lib.vlfm_pointnav_lstm_head(a, a, a, a, a, 1, a, a, a, None, None, None, 1, st),
        lambda: lib.vlfm_pointnav_lstm_head(a, a, a, a, a, 1, a, a, a, None, None, a, 0, st),
    ]
    n0 = _lib().launch_count()
    for i, c in enumerate(calls):
        assert c() == VLFM_E_INVALID, f"call {i}"
    assert _lib().launch_count() == n0


def test_pointnav_ptxas_no_spills(tmp_path):
    if not shutil.which(build.NVCC) and not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "pointnav.cu")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "pointnav.o")], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    kernels = [p for p in props if "pointnav" in p[0]]
    assert len(kernels) >= 14        # 7 GEMV instantiations + 7 others
    for name, _, st, ld in kernels:
        assert st == "0" and ld == "0", f"{name} spills ({st} B stores, {ld} B loads)"
