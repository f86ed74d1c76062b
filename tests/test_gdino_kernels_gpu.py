"""GroundingDINO's Swin-T and deformable-attention kernels against float64 references, with the parts a freshly initialised
model leaves at zero made non-zero: relative-position bias tables, q/k/v biases (what a padded token attends with), batches
above one, maps that are multiples of the 7x7 window, and the runtime-shaped / clamped / strided paths of the fused
deformable-attention gather.

The window-attention reference is itself checked against HF's SwinLayer in float64 (no GPU needed), and each window-attention
case proves it can fail: references with a transposed bias index, zero padded tokens or mask regions taken on the unpadded map
must all miss the kernel by far more than the bar."""
import contextlib
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.gdino_oracle import GdinoOracle, preprocess
from vlfm_b200.utils.synthetic import make_rgb

WS = 7
VLFM_E_INVALID = 1
BACKBONE = "model.backbone.conv_encoder.model."


# ------------------------------------------------------------------------------------------------ float64 references ----
def _regions(n: int, size: int, shift: int) -> torch.Tensor:
    """Shift-mask region of each coordinate of the shifted frame: [0, size-7) -> 0, [size-7, size-shift) -> 1, rest -> 2."""
    y = torch.arange(n)
    return torch.where(y < size - WS, 0, torch.where(y < size - shift, 1, 2))


def ref_window_attention(qkv, qkv_bias, rel_table, B, H, W, C, heads, shift, transpose_bias=False, zero_pad=False,
                         unpadded_mask=False):
    """(Shifted-)window attention in float64.  qkv [B*H*W, 3C] (q | k | v, head h at columns h*hd), qkv_bias [3C],
    rel_table [169, heads] -> [B*H*W, C].  The keyword arguments build the deliberately wrong variants the GPU test must
    be able to tell apart from the right one."""
    dev, f64 = qkv.device, torch.float64
    hd = C // heads
    Hp, Wp = -(-H // WS) * WS, -(-W // WS) * WS
    nwy, nwx = Hp // WS, Wp // WS
    # 1. pad to multiples of 7: a padded token is a zero LayerNorm output, so its projection is the bias
    full = torch.zeros(B, Hp, Wp, 3 * C, dtype=f64, device=dev)
    if not zero_pad:
        full[:] = qkv_bias.to(dev, f64)
    full[:, :H, :W] = qkv.to(f64).view(B, H, W, 3 * C)
    # 2. cyclic shift, 3. window partition -> [3, B, nwy, nwx, heads, 49, hd]
    full = torch.roll(full, (-shift, -shift), (1, 2))
    q, k, v = full.view(B, nwy, WS, nwx, WS, 3, heads, hd).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, B, nwy, nwx, heads, WS * WS, hd)
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    # 4. relative-position bias: idx = (dy + 6) * 13 + (dx + 6), dy / dx = query minus key coordinate inside the window
    ty, tx = torch.arange(WS * WS) // WS, torch.arange(WS * WS) % WS
    dy, dx = ty[:, None] - ty[None, :] + WS - 1, tx[:, None] - tx[None, :] + WS - 1
    idx = (dx * (2 * WS - 1) + dy) if transpose_bias else (dy * (2 * WS - 1) + dx)
    s = s + rel_table.to(dev, f64)[idx.to(dev)].permute(2, 0, 1)
    # 5. shift mask: -100 between regions of the PADDED map
    if shift > 0:
        hh, ww = (H, W) if unpadded_mask else (Hp, Wp)
        reg = _regions(Hp, hh, shift)[:, None] * 3 + _regions(Wp, ww, shift)[None, :]
        reg = reg.view(nwy, WS, nwx, WS).permute(0, 2, 1, 3).reshape(nwy, nwx, WS * WS).to(dev)
        s = s + torch.where(reg[..., :, None] != reg[..., None, :], -100.0, 0.0).to(f64)[None, :, :, None]
    # 6. softmax, PV, window reverse, reverse shift, crop
    o = torch.softmax(s, -1) @ v
    o = o.view(B, nwy, nwx, heads, WS, WS, hd).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, Hp, Wp, C)
    o = torch.roll(o, (shift, shift), (1, 2))[:, :H, :W]
    return o.reshape(B * H * W, C)


def _f32(x):
    return np.asarray(x, dtype=np.float32)


def ref_msda_fused(value16, offlog, ld, logit_col, ref, ref_dim, B, Q, heads, levels, points, shapes):
    """vlfm_msda_fused's operation from its own input layout, on the CPU: offsets at column 0 and logits at `logit_col` of
    rows of width `ld`; a softmax per head over the levels*points logits; sampling locations; grid_sample's bilinear
    unnormalisation (align_corners=False, zero padding) of the fp16 values.  The location arithmetic is float32, one
    rounding per operation in the order HF's module computes it (a one-ulp move of a location is amplified by the value
    gradient, so it is part of the operation's definition, not of its error); the softmax and the sampling are float64."""
    LP = levels * points
    rows = offlog.detach().cpu().numpy().reshape(B * Q, ld)
    off = _f32(rows[:, : heads * LP * 2]).reshape(B * Q, heads, levels, points, 2)
    logit = torch.from_numpy(rows[:, logit_col: logit_col + heads * LP].astype(np.float64)).view(B * Q, heads, LP)
    w = torch.softmax(logit, -1).view(B * Q, heads, levels, points)
    rp = _f32(ref.detach().cpu().numpy()).reshape(B * Q, levels, ref_dim)
    val = value16.detach().cpu().double().view(B, -1, heads, 32)
    out = torch.zeros(B * Q, heads, 32, dtype=torch.float64)
    bidx = torch.arange(B * Q)[:, None, None].expand(B * Q, heads, points) // Q
    hidx = torch.arange(heads)[None, :, None].expand(B * Q, heads, points)
    start = 0
    for l, (Hl, Wl) in enumerate(shapes):
        o, r = off[:, :, l], rp[:, l][:, None, None, :]
        if ref_dim == 2:
            lx = r[..., 0] + o[..., 0] / np.float32(Wl)
            ly = r[..., 1] + o[..., 1] / np.float32(Hl)
        else:
            lx = r[..., 0] + o[..., 0] / np.float32(points) * r[..., 2] * np.float32(0.5)
            ly = r[..., 1] + o[..., 1] / np.float32(points) * r[..., 3] * np.float32(0.5)
        ix = ((np.float32(2) * lx - np.float32(1)) + np.float32(1)) * np.float32(0.5) * np.float32(Wl) - np.float32(0.5)
        iy = ((np.float32(2) * ly - np.float32(1)) + np.float32(1)) * np.float32(0.5) * np.float32(Hl) - np.float32(0.5)
        assert ix.dtype == iy.dtype == np.float32
        ix, iy = torch.from_numpy(ix.astype(np.float64)), torch.from_numpy(iy.astype(np.float64))
        x0, y0 = torch.floor(ix), torch.floor(iy)
        fx, fy = ix - x0, iy - y0
        for ty in (0, 1):
            for tx in (0, 1):
                px, py = x0 + tx, y0 + ty
                ok = (px >= 0) & (px < Wl) & (py >= 0) & (py < Hl)
                pos = torch.where(ok, py * Wl + px, 0).long() + start
                tap = (fx if tx else 1 - fx) * (fy if ty else 1 - fy) * ok
                out += ((w[:, :, l] * tap)[..., None] * val[bidx, pos, hidx]).sum(2)
        start += Hl * Wl
    return out.view(B * Q, heads * 32)


# ---------------------------------------------------------------------------------- 1. the reference, anchored to HF ----
@pytest.mark.parametrize("H,W,B,heads,shift", [(15, 20, 2, 3, 3), (14, 21, 1, 6, 3), (8, 10, 2, 3, 0), (29, 40, 1, 3, 3)])
def test_window_reference_matches_hf_swin_layer(H, W, B, heads, shift):
    """ref_window_attention against the attention of HF's SwinLayer in float64, with non-zero position-bias table and
    q/k/v biases.  The layer's attention output (the input of attention.output, in window order) is taken with a hook and
    brought back to image order by undoing the window partition, the shift and the padding."""
    from transformers import SwinConfig
    from transformers.models.swin.modeling_swin import SwinLayer, window_reverse

    C = heads * 32
    torch.manual_seed(H * 1000 + W)
    layer = SwinLayer(SwinConfig(embed_dim=C, window_size=WS), dim=C, input_resolution=(H, W), num_heads=heads, shift_size=shift)
    layer = layer.double().eval()
    sa = layer.attention.self
    g = torch.Generator().manual_seed(H * 31 + W)
    with torch.no_grad():
        sa.relative_position_bias_table.copy_(torch.randn(sa.relative_position_bias_table.shape, generator=g, dtype=torch.float64) * 2)
        for lin in (sa.query, sa.key, sa.value):
            lin.bias.copy_(torch.randn(C, generator=g, dtype=torch.float64) * 0.5)
    x = torch.randn(B, H * W, C, generator=g, dtype=torch.float64)
    cap = {}
    hook = layer.attention.output.register_forward_pre_hook(lambda m, args: cap.__setitem__("ctx", args[0].detach().clone()))
    try:
        with torch.no_grad():
            layer(x, (H, W))
            ln = layer.layernorm_before(x).reshape(B * H * W, C)
            qkv = torch.cat([sa.query(ln), sa.key(ln), sa.value(ln)], -1)
            qkv_bias = torch.cat([sa.query.bias, sa.key.bias, sa.value.bias])
    finally:
        hook.remove()
    assert layer.shift_size == shift and float(sa.relative_position_bias_table.detach().abs().min()) > 0
    Hp, Wp = -(-H // WS) * WS, -(-W // WS) * WS
    want = window_reverse(cap["ctx"].view(-1, WS, WS, C), WS, Hp, Wp)
    want = torch.roll(want, (shift, shift), (1, 2))[:, :H, :W].reshape(B * H * W, C)
    got = ref_window_attention(qkv, qkv_bias, sa.relative_position_bias_table.detach(), B, H, W, C, heads, shift)
    err = float((got - want).abs().max())
    print(f"reference vs HF SwinLayer {H}x{W} B{B} heads {heads} shift {shift}: max {err:.3g} on outputs up to {float(want.abs().max()):.3g}")
    assert err <= 1e-10


# ------------------------------------------------------------------------------------- 2. window attention on the GPU ----
def _lib():
    from vlfm_b200 import _lib as lib

    return lib


def _window_inputs(B, H, W, heads, seed):
    g = torch.Generator().manual_seed(seed)
    C = heads * 32
    qkv = torch.randn(B * H * W, 3 * C, generator=g).half()
    qkv_bias = torch.randn(3 * C, generator=g)
    rel = torch.randn((2 * WS - 1) ** 2, heads, generator=g) * 2
    return qkv.cuda(), qkv_bias.cuda(), rel.cuda()


SENTINEL_ROWS = 64


def _run_window(qkv, qkv_bias, rel, B, H, W, heads, shift):
    """Output rows prefilled with NaN and followed by SENTINEL_ROWS rows of random values; returns (out, sentinel)."""
    lib = _lib()
    C = heads * 32
    out = torch.full((B * H * W + SENTINEL_ROWS, C), float("nan"), dtype=torch.float16, device="cuda")
    out[B * H * W:] = torch.randn(SENTINEL_ROWS, C, generator=torch.Generator().manual_seed(1)).half().cuda()
    sentinel = out[B * H * W:].clone()
    rc = lib.load().vlfm_swin_window_attention(qkv.data_ptr(), qkv_bias.data_ptr(), rel.data_ptr(), out.data_ptr(), B, H, W, C, heads, shift,
                                               lib.stream_ptr())
    lib.check(rc, "vlfm_swin_window_attention")
    torch.cuda.synchronize()
    return out, sentinel


# every stage of a 480x640 frame (120x160 ... 15x20) and of a 225x318 frame (57x80 ... 8x10), and maps that need no padding
WIN_MAPS = [(120, 160, 3), (60, 80, 6), (30, 40, 12), (15, 20, 24), (57, 80, 3), (29, 40, 6), (15, 20, 12), (8, 10, 24), (14, 21, 6), (112, 112, 3)]
WIN_CASES = [(B, H, W, heads, shift) for H, W, heads in WIN_MAPS for B in (1, 3) for shift in (0, 3)] + [(3, 29, 40, 6, 5)]
WIN_BAR = 4e-3     # fp16 P, fp16 output store, fp16 rounding of a padded token's bias (the same bar as test_attention_matches_torch)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,heads,shift", WIN_CASES)
def test_window_attention_matches_reference(B, H, W, heads, shift):
    C = heads * 32
    qkv, qkv_bias, rel = _window_inputs(B, H, W, heads, seed=B * 100000 + H * 1000 + W * 10 + shift)
    out, sentinel = _run_window(qkv, qkv_bias, rel, B, H, W, heads, shift)
    n = B * H * W
    assert not bool(out[:n].isnan().any()), "rows left unwritten"
    assert torch.equal(out[n:].view(torch.int16), sentinel.view(torch.int16)), "rows past the end were written"
    got = out[:n].double()
    ref = ref_window_attention(qkv, qkv_bias, rel, B, H, W, C, heads, shift)
    err = float((got - ref).abs().max())
    mutants = {"transposed bias index": dict(transpose_bias=True)}
    padded = H % WS or W % WS
    if padded:
        mutants["zero padded tokens"] = dict(zero_pad=True)
        if shift:
            mutants["mask on the unpadded map"] = dict(unpadded_mask=True)
    miss = {name: float((got - ref_window_attention(qkv, qkv_bias, rel, B, H, W, C, heads, shift, **kw)).abs().max())
            for name, kw in mutants.items()}
    print(f"window attention B{B} {H}x{W} heads {heads} shift {shift}: max {err:.3g} (bar {WIN_BAR}); wrong references miss by", miss)
    assert err <= WIN_BAR
    for name, d in miss.items():
        assert d > 10 * WIN_BAR, f"the test cannot tell the kernel from a reference with a {name} ({d:.3g})"


@pytest.mark.gpu
def test_window_attention_is_deterministic():
    args = (3, 57, 80, 3, 3)
    qkv, qkv_bias, rel = _window_inputs(*args[:4], seed=4242)
    a, _ = _run_window(qkv, qkv_bias, rel, *args)
    b, _ = _run_window(qkv, qkv_bias, rel, *args)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# --------------------------------------------------------------------------------------------- 6. argument validation ----
@pytest.mark.gpu
def test_window_attention_rejects_bad_arguments():
    lib = _lib()
    L = lib.load()
    B, H, W, heads = 1, 14, 14, 2
    C = heads * 32
    qkv, qkv_bias, rel = _window_inputs(B, H, W, heads, seed=3)
    out = torch.zeros(B * H * W, C, dtype=torch.float16, device="cuda")
    p = (qkv.data_ptr(), qkv_bias.data_ptr(), rel.data_ptr(), out.data_ptr())
    st = lib.stream_ptr()
    torch.cuda.synchronize()
    bad = {
        "C != heads * 32": (*p, B, H, W, C + 32, heads, 0, st),
        "C = heads * 16": (*p, B, H, W, heads * 16, heads, 0, st),
        "shift 7": (*p, B, H, W, C, heads, 7, st),
        "shift -1": (*p, B, H, W, C, heads, -1, st),
        "NULL qkv": (None, *p[1:], B, H, W, C, heads, 0, st),
        "NULL bias": (p[0], None, *p[2:], B, H, W, C, heads, 0, st),
        "NULL table": (*p[:2], None, p[3], B, H, W, C, heads, 0, st),
        "NULL out": (*p[:3], None, B, H, W, C, heads, 0, st),
    }
    for name, args in bad.items():
        before = lib.launch_count()
        rc = L.vlfm_swin_window_attention(*args)
        assert rc == VLFM_E_INVALID, name
        assert lib.launch_count() == before, f"{name}: a kernel was launched"
    torch.cuda.synchronize()
    assert float(out.abs().max()) == 0.0
    before = lib.launch_count()
    lib.check(L.vlfm_swin_window_attention(*p, B, H, W, C, heads, 3, st), "vlfm_swin_window_attention")
    assert lib.launch_count() == before + 1


# ------------------------------------------------------------------------------------------------ 3. bit-exact gathers ----
@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C", [(120, 160, 96), (57, 80, 96), (29, 40, 192), (15, 20, 384), (15, 21, 96), (60, 81, 192), (8, 11, 384)])
def test_patch_merge_is_the_2x2_gather(H, W, C):
    lib = _lib()
    B = 2
    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(H * W + C)).cuda()
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    out = torch.full((B * H2 * W2, 4 * C), float("nan"), device="cuda")
    lib.check(lib.load().vlfm_swin_patch_merge(x.data_ptr(), out.data_ptr(), B, H, W, C, lib.stream_ptr()), "vlfm_swin_patch_merge")
    xp = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    ref = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1).reshape(B * H2 * W2, 4 * C)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(480, 640), (225, 318), (481, 643)])
def test_patch_im2col_is_the_preprocessed_unfold(H, W):
    """The uint8 frame -> fp16 rows of the 4x4/4 patch-embedding GEMM, against the oracle's own preprocessing (fp32
    to_tensor + ImageNet normalise) rounded to fp16, zero-padded to a multiple of 4 and unfolded in c*16 + ky*4 + kx order."""
    from vlfm_b200.vlm.swin_engine import IMAGENET_MEAN, IMAGENET_STD

    lib = _lib()
    B = 2
    rng = np.random.default_rng(H + W)
    imgs = np.stack([make_rgb(rng, H, W) for _ in range(B)])
    imgs[0, 0, :8] = 0                       # the extremes of the uint8 range
    imgs[1, -1, -8:] = 255
    Hp, Wp = (H + 3) // 4, (W + 3) // 4
    out = torch.full((B * Hp * Wp, 48), float("nan"), dtype=torch.float16, device="cuda")
    mean, std = (ctypes.c_float * 3)(*IMAGENET_MEAN), (ctypes.c_float * 3)(*IMAGENET_STD)
    d_img = torch.from_numpy(imgs).cuda()
    lib.check(lib.load().vlfm_swin_patch_im2col(d_img.data_ptr(), out.data_ptr(), B, H, W, mean, std, lib.stream_ptr()), "vlfm_swin_patch_im2col")
    refs = []
    for img in imgs:
        px = F.pad(preprocess(img), (0, 4 * Wp - W, 0, 4 * Hp - H))
        refs.append(px.view(3, Hp, 4, Wp, 4).permute(1, 3, 0, 2, 4).reshape(Hp * Wp, 48))
    ref = torch.cat(refs).half()
    torch.cuda.synchronize()
    got = out.cpu()
    assert not bool(got.isnan().any())
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), f"{int((got != ref).sum())} of {ref.numel()} values differ"


# --------------------------------------------------------------------------- 4. the backbone with realistic biases, B > 1 ----
@pytest.fixture(scope="module")
def biased():
    """GdinoOracle(0) with the Swin parameters a fresh HF initialisation leaves at zero / one made non-zero, loaded into the
    oracle and into the GPU detector: relative-position tables ~ N(0, 1), q/k/v/proj/fc biases ~ N(0, 0.1), every LayerNorm
    weight and bias moved by ~0.1."""
    from vlfm_b200.vlm.grounding_dino import GroundingDINO

    orc = GdinoOracle(0)
    g = torch.Generator().manual_seed(2024)
    biases = ("attention.self.query.bias", "attention.self.key.bias", "attention.self.value.bias", "attention.output.dense.bias",
              "intermediate.dense.bias", "output.dense.bias")
    with torch.no_grad():
        for k, v in orc.state_dict().items():
            if not k.startswith(BACKBONE):
                continue
            if k.endswith("relative_position_bias_table"):
                v.copy_(torch.randn(v.shape, generator=g))
            elif ".blocks." in k and k.endswith(biases):
                v.copy_(torch.randn(v.shape, generator=g) * 0.1)
            elif "norm" in k[len(BACKBONE):]:            # layernorm_before / _after, embeddings.norm, downsample.norm, hidden_states_norms
                v.add_(torch.randn(v.shape, generator=g) * 0.1)
    det = GroundingDINO(state_dict={k: v.clone() for k, v in orc.state_dict().items()}, seed=0, synthetic=True)
    return orc, det


def _swin_attention_modules(orc):
    return [m for m in orc.model.model.backbone.conv_encoder.model.modules() if type(m).__name__ == "SwinSelfAttention"]


@contextlib.contextmanager
def _tables_zeroed(orc):
    mods = _swin_attention_modules(orc)
    saved = [m.relative_position_bias_table.detach().clone() for m in mods]
    try:
        with torch.no_grad():
            for m in mods:
                m.relative_position_bias_table.zero_()
        yield
    finally:
        with torch.no_grad():
            for m, t in zip(mods, saved):
                m.relative_position_bias_table.copy_(t)


@contextlib.contextmanager
def _padded_tokens_zeroed(orc):
    """q/k/v of padded tokens (the all-zero rows the window padding inserts before the projections) set to zero, not the bias."""
    def hook(m, args, out):
        return out.masked_fill((args[0] == 0).all(-1, keepdim=True), 0.0)

    hs = [lin.register_forward_hook(hook) for m in _swin_attention_modules(orc) for lin in (m.query, m.key, m.value)]
    try:
        yield
    finally:
        for h in hs:
            h.remove()


def _stage_errors(got, ref):
    return [(float((o - r).abs().mean()), float((o - r).abs().max())) for o, r in zip(got, ref)]


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(480, 640), (225, 318), (448, 448)])     # 448: stage maps 112 / 56 / 28 / 14, no padding anywhere
def test_backbone_with_position_biases_matches_oracle(biased, hw):
    orc, det = biased
    img = make_rgb(np.random.default_rng(hw[0] + 7), *hw)
    ref = orc.backbone_features(img)
    with _tables_zeroed(orc):
        ref0 = orc.backbone_features(img)
    with _padded_tokens_zeroed(orc):
        refp = orc.backbone_features(img)
    got = [o[0].cpu() for o in det.backbone.forward(torch.from_numpy(img[None]).cuda())]
    torch.cuda.synchronize()
    assert len(got) == len(ref) == 3 and all(o.shape == r.shape for o, r in zip(got, ref))
    err = _stage_errors(got, ref)
    no_table = [m for m, _ in _stage_errors(ref0, ref)]
    no_pad = _stage_errors(refp, ref)
    print(f"backbone {hw}: (mean, max) error per stage {err}; oracle moves by {no_table} (mean) without tables, by {no_pad} "
          "(mean, max) with zero padded tokens")
    for (mean, mx), d in zip(err, no_table):
        assert mean <= 5e-3 and mx <= 1e-1
        assert d >= 2e-2, "zeroing the tables barely moves the oracle: the comparison cannot see the bias lookup"
        assert mean <= d / 10


@pytest.mark.gpu
def test_backbone_batch_matches_single_frames(biased):
    orc, det = biased
    rng = np.random.default_rng(77)
    imgs = np.stack([make_rgb(rng, 480, 640) for _ in range(3)])
    batch = [o.cpu() for o in det.backbone.forward(torch.from_numpy(imgs).cuda())]
    singles = [[o[0].cpu() for o in det.backbone.forward(torch.from_numpy(img[None]).cuda())] for img in imgs]
    torch.cuda.synchronize()
    for i, img in enumerate(imgs):
        mine = [o[i] for o in batch]
        d = max(float((a - b).abs().max()) for a, b in zip(mine, singles[i]))
        err = _stage_errors(mine, orc.backbone_features(img))
        print(f"image {i} of 3: batch vs batch-1 max {d:.3g}; vs oracle (mean, max) {err}")
        assert d <= 1e-2
        assert all(mean <= 5e-3 and mx <= 1e-1 for mean, mx in err)


def _detection_metrics(la, ba, lb, bb):
    """Sorted-confidence mean difference and box-set distance: with random weights the 900 queries come from a top-k over
    near-tied scores, so rows permute between two computations and are not compared one by one."""
    ca, cb = la.max(dim=1)[0].sort()[0], lb.max(dim=1)[0].sort()[0]
    dist = (bb[:, None, :] - ba[None, :, :]).abs().sum(-1).min(dim=1)[0]
    return float((ca - cb).abs().mean()), float(dist.mean())


@pytest.mark.gpu
def test_detector_batches_match_single_frames(biased):
    """raw_outputs_device at B = 2 (CUDA-graph replay) and B = 5 (above the graph batch limit: eager) against each frame's
    batch-1 raw_outputs, held to max(floor, 3x) what two eager batch-1 runs of one frame differ by."""
    _, det = biased
    ids = det.tokenizer.encode("chair . couch . tv .")
    rng = np.random.default_rng(31)
    imgs = np.stack([make_rgb(rng, 480, 640) for _ in range(5)])
    use_graph = det.use_graph
    try:
        det.use_graph = False
        e0 = [t.clone() for t in det.raw_outputs(imgs[0], ids)]
        e1 = [t.clone() for t in det.raw_outputs(imgs[0], ids)]
    finally:
        det.use_graph = use_graph
    ee = _detection_metrics(e0[0], e0[1], e1[0], e1[1])
    bar = (max(5e-3, 3 * ee[0]), max(1e-3, 3 * ee[1]))
    # back to back, as a policy loop calls it: the graph replays are enqueued faster than they run, so each call must keep
    # its own frame even though the next call refills the same page-locked staging buffer
    single = [[t.clone() for t in det.raw_outputs(img, ids)] for img in imgs]
    from vlfm_b200.vlm.grounding_dino import GRAPH_MAX_BATCH

    assert GRAPH_MAX_BATCH == 4
    other = _detection_metrics(single[0][0], single[0][1], single[1][0], single[1][1])
    res = []
    for b in (2, 5):
        d_imgs = torch.from_numpy(imgs[:b]).cuda()
        det.raw_outputs_device(d_imgs, ids)
        lg, bx = (t.clone() for t in det.raw_outputs_device(d_imgs, ids))
        graph = (b, 480, 640, tuple(ids)) in det.graphs.captured
        assert graph == (b <= 4) and det.graphs.error is None, det.graphs.error
        for i in range(b):
            res.append(_detection_metrics(single[i][0], single[i][1], lg[i], bx[i]))
            print(f"B={b} ({'graph' if graph else 'eager'}) image {i}: (confidence, box-set) {res[-1]}; eager vs eager {ee}; "
                  f"two different frames {other}")
    for m in res:
        assert m[0] <= bar[0] and m[1] <= bar[1]


@pytest.mark.gpu
def test_backbone_refuses_frames_below_225_px(biased):
    from vlfm_b200._lib import VlfmError

    _, det = biased
    small = torch.from_numpy(make_rgb(np.random.default_rng(0), 224, 224)[None]).cuda()
    with pytest.raises(VlfmError, match="225 px"):
        det.backbone.forward(small)
    ok = det.backbone.forward(torch.from_numpy(make_rgb(np.random.default_rng(0), 225, 225)[None]).cuda())
    torch.cuda.synchronize()
    assert [tuple(o.shape[2:]) for o in ok] == [(29, 29), (15, 15), (8, 8)]
    assert all(bool(o.isfinite().all()) for o in ok)


# ----------------------------------------------------------------------------------------- 5. fused deformable attention ----
MSDA_CASES = [
    # ref_dim, levels, points, B, Q, heads, shapes, gap before logit_col, spare columns at the end of a row
    (2, 4, 4, 2, 100, 8, [(20, 32), (10, 16), (5, 8), (3, 4)], 0, 0),           # the specialised 4x4 template, tight rows
    (4, 4, 4, 2, 100, 8, [(60, 80), (30, 40), (15, 20), (8, 10)], 6, 10),
    (4, 4, 4, 3, 37, 3, [(20, 32), (10, 16), (5, 8), (3, 4)], 2, 4),             # 333 warps: a partial block of 8
    (2, 3, 5, 3, 37, 8, [(24, 32), (12, 16), (7, 9)], 4, 2),                     # runtime levels / points from here on
    (4, 2, 8, 2, 50, 5, [(16, 16), (9, 13)], 0, 6),
    (2, 1, 1, 3, 37, 3, [(32, 64)], 8, 0),
    (4, 1, 1, 1, 64, 8, [(11, 7)], 2, 2),
]


def _msda_inputs(ref_dim, levels, points, B, Q, heads, shapes, gap, spare, seed):
    g = torch.Generator().manual_seed(seed)
    LP = levels * points
    S = sum(h * w for h, w in shapes)
    logit_col = heads * LP * 2 + gap
    ld = logit_col + heads * LP + spare
    ld += ld & 1                                                    # the float2 offset loads need even rows
    value = torch.randn(B, S, heads, 32, generator=g).half()
    rows = torch.full((B * Q, ld), float("nan"))                    # gap and spare columns must never be read
    off = torch.randn(B * Q, heads, levels, points, 2, generator=g) * 2
    logit = torch.randn(B * Q, heads, LP, generator=g) * 2
    if ref_dim == 2:
        ref = torch.rand(B * Q, levels, 2, generator=g) * 1.2 - 0.1
    else:
        ref = torch.rand(B * Q, levels, 4, generator=g)
        ref[..., 2:] = ref[..., 2:] * 0.4 + 0.05
    # query 0 of every image: exact pixel centres and the -1 / W-1 (H-1) borders; ref 0 and (for ref_dim 4) w = h = 2 make the
    # location off / W (off / points), exact for the power-of-two sizes above
    for b in range(B):
        r = b * Q
        ref[r] = 0.0
        if ref_dim == 4:
            ref[r, :, 2:] = 2.0
        for l, (Hl, Wl) in enumerate(shapes):
            nx, ny = (Wl, Hl) if ref_dim == 2 else (points, points)
            targets = [(0.5, 0.5), (Wl - 0.5, Hl - 0.5), (-0.5, 2.5), (Wl - 0.5, 1.5), (3.5, -0.5), (1.5, Hl - 0.5), (-0.5, -0.5), (Wl + 0.5, Hl)]
            for j in range(points):
                for h in range(heads):
                    tx, ty = targets[(j + h + l) % len(targets)]
                    off[r, h, l, j] = torch.tensor([tx / Wl * nx, ty / Hl * ny])
    # far samples: offsets of 1e4 (both signs) and 1e7, which the kernel clamps before its int conversion
    far = torch.randint(1, B * Q, (max(8, B * Q // 10),), generator=g)
    off[far, far % heads, far % levels, far % points] = torch.tensor([1e4, -1e4, 1e7, -1e7])[far % 4, None] * torch.tensor([1.0, -0.5])
    rows[:, : heads * LP * 2] = off.reshape(B * Q, -1)
    rows[:, logit_col: logit_col + heads * LP] = logit.reshape(B * Q, -1)
    return value, rows, ld, logit_col, ref, S


def _run_msda(value, rows, ld, logit_col, ref, ref_dim, B, S, Q, heads, levels, points, shapes):
    lib = _lib()
    out = torch.full((B * Q * heads * 32,), float("nan"), dtype=torch.float16, device="cuda")
    flat = [int(v) for hw in shapes for v in hw]
    sh = (ctypes.c_int32 * len(flat))(*flat)
    rc = lib.load().vlfm_msda_fused(value.data_ptr(), rows.data_ptr(), ld, logit_col, ref.data_ptr(), ref_dim, out.data_ptr(), B, S, Q, heads,
                                    levels, points, ctypes.cast(sh, ctypes.c_void_p), lib.stream_ptr())
    return rc, out


@pytest.mark.gpu
@pytest.mark.parametrize("ref_dim,levels,points,B,Q,heads,shapes,gap,spare", MSDA_CASES)
def test_msda_fused_matches_reference(ref_dim, levels, points, B, Q, heads, shapes, gap, spare):
    value, rows, ld, logit_col, ref, S = _msda_inputs(ref_dim, levels, points, B, Q, heads, shapes, gap, spare,
                                                      seed=ref_dim * 1000 + levels * 100 + points * 10 + B)
    rc, out = _run_msda(value.cuda(), rows.cuda(), ld, logit_col, ref.cuda(), ref_dim, B, S, Q, heads, levels, points, shapes)
    _lib().check(rc, "vlfm_msda_fused")
    torch.cuda.synchronize()
    got = out.cpu().double().view(B * Q, heads * 32)
    want = ref_msda_fused(value, rows, ld, logit_col, ref, ref_dim, B, Q, heads, levels, points, shapes)
    err = (got - want).abs()
    excess = float((err - (2.0 ** -11 * want.abs() + 1e-5)).max())
    print(f"msda_fused ref_dim {ref_dim} {levels}x{points} B{B} Q{Q} heads {heads} ld {ld} logit_col {logit_col}: max {float(err.max()):.3g}, "
          f"max err / |ref| {float((err / want.abs().clamp_min(1e-3)).max()):.3g}, worst excess over the bar {excess:.3g}")
    assert not bool(got.isnan().any())
    assert excess <= 0.0


@pytest.mark.gpu
def test_msda_fused_rejects_bad_arguments():
    lib = _lib()
    shapes = [(8, 8), (4, 4), (2, 2), (1, 1)]
    value, rows, ld, logit_col, ref, S = _msda_inputs(2, 4, 4, 1, 8, 2, shapes, 0, 0, seed=9)
    value, rows, ref = value.cuda(), rows.cuda(), ref.cuda()
    torch.cuda.synchronize()
    for name, (l_d, rd, lv, pt) in {"levels * points > 16": (ld, 2, 4, 5), "odd ld": (ld - 1, 2, 4, 4), "ref_dim 3": (ld, 3, 4, 4)}.items():
        before = lib.launch_count()
        rc, out = _run_msda(value, rows, l_d, logit_col, ref, rd, 1, S, 8, 2, lv, pt, shapes)
        assert rc == VLFM_E_INVALID and lib.launch_count() == before, name
