"""Every MobileSAM kernel of csrc/sam_ops.cu on its own, against a float64 (or bit-exact) reference of the same operation, at
the engine's vit_t / TINY shapes and at the edges where such kernels go wrong: partial windows and key chunks, odd maps,
strided views, off-frame boxes, frames with a side above S.

Conventions (as tests/test_gdino_kernels_gpu.py): outputs are prefilled with NaN (uint8 outputs with 0xAB) and followed by
sentinel rows, so an unwritten element or a write past the end fails; every launch is repeated and must reproduce its bits;
bad arguments return VLFM_E_INVALID without a launch.  Every bar below is derived from rounding analysis in its docstring
(u = 2^-24, the fp32 unit roundoff).  Where a bar is not exact, "mutant" references, plausible wrong versions of the
reference, must miss the kernel by more than 10x the bar, which shows the bar is tight enough to catch such a bug.

CPU tests (unmarked) pin the references to the oracle (oracle/sam_oracle.py) and the Pillow pass order."""
import ctypes
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.sam_oracle import SamOracle, apply_box, preprocess, preshape
from vlfm_b200.vlm.preprocess import bilinear_tables, pillow_vertical_first
from vlfm_b200.vlm.sam_config import TINY, VIT_T, random_state_dict
from vlfm_b200.vlm.sam_weights import convert_state_dict

VLFM_E_INVALID = 1
U = 2.0 ** -24
SENT = 64            # sentinel rows after every output
f64 = torch.float64


def _lib():
    from vlfm_b200 import _lib as lib

    return lib


def _call(name, *args):
    lib = _lib()
    lib.check(getattr(lib.load(), name)(*args), name)


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """spacing of fp16 numbers at |x| (2^-24 in the subnormal range)"""
    a = x.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def _out(rows, cols, dtype, seed=7):
    """[rows + SENT, cols] output: rows NaN, then SENT rows of random sentinel values; -> (buffer, sentinel copy)"""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((rows + SENT, cols), float("nan"), dtype=dtype)
    buf[rows:] = torch.randn(SENT, cols, generator=g).to(dtype)
    buf = buf.cuda()
    return buf, buf[rows:].clone()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32) if t.dtype == torch.float32 else t


def _check_written(buf, sentinel, rows, what):
    torch.cuda.synchronize()
    assert not bool(buf[:rows].isnan().any()), f"{what}: output elements left unwritten"
    assert torch.equal(_bits(buf[rows:]), _bits(sentinel)), f"{what}: rows past the end were written"


def _report(what, err, bar, miss=None):
    ratio = float((err / bar).max()) if torch.is_tensor(err) else err / bar
    print(f"{what}: max err/bar {ratio:.3g}" + (f"; mutants miss by x bar: {miss}" if miss else ""))
    return ratio


# =========================================================================================== 1. window attention ====
def ref_window_attention(qkv, pad, bias, B, H, W, heads, ws, scale, transpose_bias=False, mask_pad=False, zero_pad=False,
                         head0_bias=False):
    """TinyViT window attention in float64 on the engine's layout.  qkv [B*H*W, 3C] ([q | k | v], head h at h*32 in each),
    pad [3C] the q/k/v row of a padding token, bias [heads, ws*ws] indexed by |dy|*ws + |dx|.  The map is padded to a
    window multiple with `pad` rows (unmasked keys), padded queries are cropped.  Returns (out [B*H*W, C], stats) where
    stats = (max scale*sum_d |q_d k_d|, max |score|, max |v|) feed the bar.  The keyword arguments build the mutants."""
    dev = qkv.device
    C = heads * 32
    N = ws * ws
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    nwy, nwx = Hp // ws, Wp // ws
    full = torch.zeros(B, Hp, Wp, 3 * C, dtype=f64, device=dev)
    if not zero_pad:
        full[:] = pad.to(dev, f64)
    full[:, :H, :W] = qkv.to(f64).view(B, H, W, 3 * C)
    q, k, v = full.view(B, nwy, ws, nwx, ws, 3, heads, 32).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, B, nwy, nwx, heads, N, 32)
    s = q @ k.transpose(-1, -2) * scale
    t = torch.arange(N, device=dev)
    dy, dx = (t[:, None] // ws - t[None] // ws).abs(), (t[:, None] % ws - t[None] % ws).abs()
    idx = dx * ws + dy if transpose_bias else dy * ws + dx
    bt = bias.to(dev, f64)
    if head0_bias:
        bt = bt[:1].expand(heads, N)
    s = s + bt[:, idx]
    if mask_pad:
        valid = torch.zeros(Hp, Wp, dtype=torch.bool, device=dev)
        valid[:H, :W] = True
        valid = valid.view(nwy, ws, nwx, ws).permute(0, 2, 1, 3).reshape(nwy, nwx, N)
        s = s.masked_fill(~valid[None, :, :, None, None, :], float("-inf"))
    o = torch.softmax(s, -1) @ v
    o = o.view(B, nwy, nwx, heads, ws, ws, 32).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, Hp, Wp, C)[:, :H, :W]
    stats = (float((q.abs() @ k.abs().transpose(-1, -2)).max()) * scale, float(s[s.isfinite()].abs().max()), float(v.abs().max()))
    return o.reshape(B * H * W, C), stats


def window_bar(ref, stats, ws, n_keys):
    """fp32 kernel, fp16 operands (exact in fp32).  A score is a 32-term fp32 FMA chain times scale plus the bias:
    |ds| <= u (33 scale sum|q k| + 2 |s|).  Each __expf(x) is within (2 + 1.16|x|) fp32 ulps (CUDA C Programming Guide,
    intrinsic functions), |x| <= 2 max|s|; a key's weight goes through its own exp and up to ws online rescales, so its
    relative error is d <= |ds| + (ws + 1) 2u (2 + 2.32 max|s|).  Relative weight errors d move the normalised average by at
    most 2 d max|v - o| <= 4 d max|v|; the fp32 sums over n_keys terms add (n_keys + 2) 2u max|v|.  The fp16 store adds half
    an ulp of the result: one fp16 ulp of the reference covers it and a crossing of a binade boundary."""
    sabs, smax, vmax = stats
    ds = U * (33 * sabs + 2 * smax)
    d = ds + (ws + 1) * 2 * U * (2 + 2.32 * smax)
    return ulp16(ref) + 4 * d * vmax + (n_keys + 2) * 2 * U * vmax


def _window_inputs(B, H, W, heads, ws, seed):
    g = torch.Generator().manual_seed(seed)
    C = heads * 32
    qkv = torch.randn(B * H * W, 3 * C, generator=g).half()
    pad = torch.cat([torch.randn(C, generator=g), 3 * torch.randn(C, generator=g), 4 + 3 * torch.randn(C, generator=g)]).half()
    bias = torch.randn(heads, ws * ws, generator=g)
    return qkv.cuda(), pad.cuda(), bias.cuda()


def _run_window(qkv, pad, bias, B, H, W, heads, ws, scale):
    C = heads * 32
    out, sent = _out(B * H * W, C, torch.float16)
    _call("vlfm_sam_window_attention", qkv.data_ptr(), pad.data_ptr(), bias.data_ptr(), out.data_ptr(), B, H, W, C, heads, ws,
          scale, _lib().stream_ptr())
    _check_written(out, sent, B * H * W, "window attention")
    return out[: B * H * W]


# (B, H, W, heads, ws): vit_t's three attention stages, TINY's three, window multiples, maps smaller than a window,
# a non-square map, B = 3
WIN_CASES = [(1, 128, 128, 4, 7), (1, 64, 64, 5, 14), (1, 64, 64, 10, 7), (1, 32, 32, 2, 7), (1, 16, 16, 2, 14), (1, 16, 16, 3, 7),
             (2, 7, 7, 2, 7), (1, 14, 14, 3, 14), (2, 28, 28, 1, 14), (1, 28, 28, 2, 7), (2, 5, 3, 2, 7), (1, 1, 1, 3, 7),
             (1, 5, 3, 2, 14), (1, 1, 1, 2, 14), (1, 13, 29, 2, 7), (1, 13, 29, 2, 14), (3, 13, 29, 3, 7), (3, 20, 17, 2, 14)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,heads,ws", WIN_CASES)
def test_window_attention_matches_reference(B, H, W, heads, ws):
    scale = float(np.float32(32 ** -0.5))
    qkv, pad, bias = _window_inputs(B, H, W, heads, ws, seed=B * 10 ** 6 + H * 1000 + W * 10 + heads + ws)
    got = _run_window(qkv, pad, bias, B, H, W, heads, ws, scale)
    again = _run_window(qkv, pad, bias, B, H, W, heads, ws, scale)
    assert torch.equal(_bits(got), _bits(again)), "not bitwise reproducible"
    ref, stats = ref_window_attention(qkv, pad, bias, B, H, W, heads, ws, scale)
    bar = window_bar(ref, stats, ws, ws * ws)
    err = (got.double() - ref).abs()
    mutants = {"transposed bias": dict(transpose_bias=True)}
    if H % ws or W % ws:
        mutants.update({"padded keys masked": dict(mask_pad=True), "padded K/V zeroed": dict(zero_pad=True)})
    if heads > 1:
        mutants["head 0's bias"] = dict(head0_bias=True)
    if H * W == 1:
        # one real key, every other key the same pad row: the output depends on the bias only through bias[0] and the sum of
        # exp(bias) over the other offsets, which a transposed index leaves unchanged and another head's row barely moves
        mutants = {n: kw for n, kw in mutants.items() if n not in ("transposed bias", "head 0's bias")}
    miss = {n: round(float((got.double() - ref_window_attention(qkv, pad, bias, B, H, W, heads, ws, scale, **kw)[0]).abs().max())
                     / float(bar.max()), 1) for n, kw in mutants.items()}
    _report(f"window attention B{B} {H}x{W} heads {heads} ws {ws}", err, bar, miss)
    assert bool((err <= bar).all())
    for n, m in miss.items():
        assert m > 10, f"the test cannot tell the kernel from a reference with {n}"


def test_window_reference_matches_oracle():
    """LN -> qkv (sam_weights' [q | k | v] row permutation) -> ref_window_attention with the engine's pad row
    W.fp16(beta) + b -> proj equals SamOracle.window_attention on the zero-padded windows, in float64.  beta is made
    fp16-exact so that the engine's formula and the oracle's LayerNorm of a zero token agree to the last bit."""
    d = TINY
    sd = random_state_dict(d, 4)
    s, ws = 1, d.windows[1]
    heads, C = d.heads[s], d.embed_dims[s]
    name = f"image_encoder.layers.{s}.blocks.0.attn"
    sd[name + ".norm.bias"] = sd[name + ".norm.bias"].half().float() * 8
    w = convert_state_dict(sd, d)
    orc = SamOracle(d, sd)
    orc.sd = {k: v.double() for k, v in orc.sd.items()}
    p = {k[len(f"l{s}.b0."):]: v.double() for k, v in w.items() if k.startswith(f"l{s}.b0.")}
    B, H, W = 2, 10, 12
    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(5), dtype=f64)
    xn = F.layer_norm(x, (C,), p["ln1.w"], p["ln1.b"], 1e-5)
    qkv = (xn @ p["qkv.w"].T + p["qkv.b"]).reshape(B * H * W, 3 * C)
    pad_row = p["qkv.w"] @ p["ln1.b"].half().double() + p["qkv.b"]
    o, _ = ref_window_attention(qkv, pad_row, p["bias"], B, H, W, heads, ws, (C // heads) ** -0.5)
    ours = (o @ p["proj.w"].T + p["proj.b"]).view(B, H, W, C)
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    xp = F.pad(x, (0, 0, 0, Wp - W, 0, Hp - H))
    t = xp.view(B, Hp // ws, ws, Wp // ws, ws, C).transpose(2, 3).reshape(-1, ws * ws, C)
    want = orc.window_attention(t, name, heads, ws)
    want = want.view(B, Hp // ws, Wp // ws, ws, ws, C).transpose(2, 3).reshape(B, Hp, Wp, C)[:, :H, :W]
    err = float((ours - want).abs().max())
    print(f"window reference vs oracle: {err:.3g}")
    assert err <= 1e-10


# ====================================================================================== 2. token -> image attention ====
def ref_t2i(q, k, v, M, heads, Nq, Nk, scale, drop_tail=False, no_rescale=False):
    """softmax(scale q k^T) v per (box, head) in float64 from the strided fp16 operands -> ([M*Nq, heads*16], stats).
    drop_tail: keys past the last whole 256-key chunk ignored; no_rescale: 256-key chunks merged as sum(acc_c) / sum(l_c)
    with each chunk relative to its own max."""
    D = heads * 16
    qq = q[:, :D].double().view(M, Nq, heads, 16).transpose(1, 2)
    kk = k[:, :D].double().view(M, Nk, heads, 16).transpose(1, 2)
    vv = v[:, :D].double().view(M, Nk, heads, 16).transpose(1, 2)
    s = qq @ kk.transpose(-1, -2) * scale
    stats = (float((qq.abs() @ kk.abs().transpose(-1, -2)).max()) * scale, float(s.abs().max()), float(vv.abs().max()))
    if drop_tail:
        n = Nk // 256 * 256
        s, vv = s[..., :n], vv[:, :, :n]
    if no_rescale:
        a, l = 0, 0
        for c0 in range(0, s.shape[-1], 256):
            sc = s[..., c0:c0 + 256]
            p = torch.exp(sc - sc.max(-1, keepdim=True).values)
            a, l = a + p @ vv[:, :, c0:c0 + 256], l + p.sum(-1, keepdim=True)
        o = a / l
    else:
        o = torch.softmax(s, -1) @ vv
    return o.transpose(1, 2).reshape(M * Nq, D), stats


def t2i_bar(ref, stats):
    """Scores: q*scale rounded, then a 16-term FMA chain: |ds| <= u (18 scale sum|q k|).  A key's weight passes through at
    most 16 __expf calls (its own, <= 8 online rescales in its lane, 5 butterfly merges, the chunk merge), each within
    (2 + 1.16|x|) ulps with |x| <= 2 max|s|, and about 32 fp32 products: d <= |ds| + 16 * 2u (2 + 2.32 max|s|) + 32u.  As
    for the window attention the average moves by <= 4 d max|v|; the sums (<= 8 lane terms, 5 merges, <= 17 chunks) add
    64 u max|v|; the fp16 store one ulp of the reference."""
    sabs, smax, vmax = stats
    d = U * 18 * sabs + 16 * 2 * U * (2 + 2.32 * smax) + 32 * U
    return ulp16(ref) + 4 * d * vmax + 64 * U * vmax


def _t2i_inputs(M, heads, Nq, Nk, seed, spike=None, score=30.0):
    """q [M*Nq, ldq], k / v [M*Nk, ldk / ldv] fp16 with padded leading dimensions.  spike = key index whose score is
    +score for every query (one other key gets -score), so that the global max sits in that key's chunk."""
    g = torch.Generator().manual_seed(seed)
    D = heads * 16
    q = 2 * torch.randn(M * Nq, D + 24, generator=g)
    k = torch.randn(M * Nk, D + 8, generator=g)
    v = torch.randn(M * Nk, D + 40, generator=g)
    scale = float(np.float32(16 ** -0.5))
    if spike is not None:
        u = torch.randn(M, 1, D, generator=g).half().float()
        q[:, :D] = u.expand(M, Nq, D).reshape(M * Nq, D)
        uh = u.view(M, heads, 16)
        for m in range(M):
            for sgn, j in ((1, spike), (-1, (spike + Nk // 2) % Nk)):
                row = m * Nk + j
                if sgn < 0 and j == spike:
                    continue
                k[row, :D] = (sgn * score / scale * uh[m] / (uh[m] ** 2).sum(-1, keepdim=True)).reshape(D)
    return q.half().cuda(), k.half().cuda(), v.half().cuda(), scale


def _run_t2i(q, k, v, M, heads, Nq, Nk, scale):
    D = heads * 16
    ldo = D + 16
    o, _ = _out(M * Nq, ldo, torch.float16)
    o[: M * Nq, D:] = torch.randn(M * Nq, ldo - D, generator=torch.Generator().manual_seed(3)).half().cuda()   # outside the view
    before = o.clone()
    chunks = (Nk + 255) // 256
    part = torch.full((M * heads * chunks * Nq * 18,), float("nan"), device="cuda")
    _call("vlfm_sam_t2i_attention", q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), M, heads, Nq, Nk, q.stride(0), k.stride(0),
          v.stride(0), ldo, scale, part.data_ptr(), part.numel(), _lib().stream_ptr())
    torch.cuda.synchronize()
    assert not bool(o[: M * Nq, :D].isnan().any()), "output elements left unwritten"
    assert torch.equal(_bits(o[: M * Nq, D:]), _bits(before[: M * Nq, D:])), "columns outside the strided view were written"
    assert torch.equal(_bits(o[M * Nq:]), _bits(before[M * Nq:])), "rows past the end were written"
    return o[: M * Nq, :D]


T2I_NK = [1, 5, 31, 32, 255, 256, 257, 4095, 4096, 4097]
T2I_CASES = [(Nk, Nq, (1, 4, 8)[i % 3], (1, 3)[(i // 3) % 2]) for i, (Nk, Nq) in enumerate((a, b) for a in T2I_NK for b in (1, 7, 8))]
T2I_CASES += [(4096, 7, 8, 3), (256, 7, 4, 3)]       # vit_t and TINY decoder shapes, three boxes


def _t2i_case(M, heads, Nq, Nk, seed, spike=None):
    score = 30.0
    if spike is None and Nk > 256 and Nk % 256:
        spike, score = Nk - 1, 8.0          # a key of the partial last chunk that carries weight: dropping it shows
    q, k, v, scale = _t2i_inputs(M, heads, Nq, Nk, seed, spike, score)
    got = _run_t2i(q, k, v, M, heads, Nq, Nk, scale)
    again = _run_t2i(q, k, v, M, heads, Nq, Nk, scale)
    assert torch.equal(_bits(got), _bits(again)), "not bitwise reproducible"
    ref, stats = ref_t2i(q, k, v, M, heads, Nq, Nk, scale)
    bar = t2i_bar(ref, stats)
    err = (got.double() - ref).abs()
    mutants = {}
    if Nk > 256 and Nk % 256 and spike >= Nk // 256 * 256:
        mutants["tail keys dropped"] = dict(drop_tail=True)
    if Nk > 256:
        mutants["chunks merged without rescaling"] = dict(no_rescale=True)
    miss = {n: round(float((got.double() - ref_t2i(q, k, v, M, heads, Nq, Nk, scale, **kw)[0]).abs().max()) / float(bar.max()), 1)
            for n, kw in mutants.items()}
    _report(f"t2i M{M} heads {heads} Nq {Nq} Nk {Nk}" + (f" spike at key {spike}" if spike is not None else "")
            + f" (max |s| {stats[1]:.1f})", err, bar, miss)
    assert bool((err <= bar).all())
    for n, m in miss.items():
        assert m > 10, f"the test cannot tell the kernel from a reference with {n}"


@pytest.mark.gpu
@pytest.mark.parametrize("Nk,Nq,heads,M", T2I_CASES)
def test_t2i_attention_matches_reference(Nk, Nq, heads, M):
    _t2i_case(M, heads, Nq, Nk, seed=Nk * 100 + Nq * 10 + heads + M)


@pytest.mark.gpu
@pytest.mark.parametrize("Nk,spike", [(4097, 3), (4097, 4096), (4096, 4095), (1000, 0), (1000, 999), (257, 256)])
def test_t2i_attention_global_max_in_first_or_last_chunk(Nk, spike):
    _t2i_case(2, 8, 7, Nk, seed=Nk + spike, spike=spike)


# ============================================================================================ 3. depthwise conv ====
def ref_dwconv(x, w, b, stride, gelu, transpose_taps=False):
    """float64 conv2d(groups=C) of NHWC x with tap-major w [9, C] (tap ky*3+kx), + b, optional GELU (erf); -> (y, bound
    input) where the second is the same conv with |x|, |w| plus |b| (the scale of the fp32 rounding)."""
    C = x.shape[-1]
    wt = w.double().t().reshape(C, 1, 3, 3)
    if transpose_taps:
        wt = wt.transpose(2, 3)
    xc = x.double().permute(0, 3, 1, 2)
    y = F.conv2d(xc, wt, b.double(), stride, 1, 1, C)
    a = F.conv2d(xc.abs(), wt.abs(), b.double().abs(), stride, 1, 1, C)
    if gelu:
        y = F.gelu(y)
    return y.permute(0, 2, 3, 1).reshape(-1, C), a.permute(0, 2, 3, 1).reshape(-1, C)


def dwconv_bar(ref, a, gelu, out_f32):
    """Nine FMAs and the bias add in fp32: |e| <= 10u a, a = sum |x w| + |b|.  GELU's slope is below 1.13 and its own fp32
    evaluation (x*c, erff within 2 ulps, 1 + erf, two products) adds <= u (2|y| + 6|ref|) (the erff ulp error times 0.5|y|,
    relative roundings on the result).  The store: u|ref| for fp32, one fp16 ulp of the reference for fp16."""
    e = 10 * U * a * (1.13 if gelu else 1.0)
    if gelu:
        e = e + U * (2 * a + 6 * ref.abs())
    return e + (U * ref.abs() if out_f32 else ulp16(ref))


DW_MAPS = [(1, 1), (2, 3), (7, 9), (13, 13)]


def _dw_case(B, H, W, C, stride, gelu, in_f32, out_f32, seed):
    g = torch.Generator().manual_seed(seed)
    x = (2 * torch.randn(B, H, W, C, generator=g)).to(torch.float32 if in_f32 else torch.float16).cuda()
    w = (torch.randn(9, C, generator=g) / 3).cuda()
    b = (0.5 * torch.randn(C, generator=g)).cuda()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    n = B * Ho * Wo
    dt = torch.float32 if out_f32 else torch.float16
    outs = []
    for _ in range(2):
        out, sent = _out(n, C, dt, seed=seed)
        _call("vlfm_sam_dwconv3x3", x.data_ptr(), in_f32, w.data_ptr(), b.data_ptr(), out.data_ptr(), out_f32, B, H, W, C, stride, gelu,
              _lib().stream_ptr())
        _check_written(out, sent, n, "dwconv")
        outs.append(out[:n])
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "not bitwise reproducible"
    ref, a = ref_dwconv(x, w, b, stride, gelu)
    bar = dwconv_bar(ref, a, gelu, out_f32)
    err = (outs[0].double() - ref).abs()
    miss = None
    if H > 1 and W > 1:
        m = float(((outs[0].double() - ref_dwconv(x, w, b, stride, gelu, transpose_taps=True)[0]).abs() / bar).max())
        miss = {"ky/kx transposed": round(m, 1)}
        assert m > 10, "the test cannot tell the kernel from a reference with transposed taps"
    return _report(f"dwconv B{B} {H}x{W} C{C} s{stride} gelu {gelu} in {'f32' if in_f32 else 'f16'} out {'f32' if out_f32 else 'f16'}",
                   err, bar, miss), bool((err <= bar).all())


@pytest.mark.gpu
@pytest.mark.parametrize("in_f32", [0, 1])
@pytest.mark.parametrize("out_f32", [0, 1])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("gelu", [0, 1])
def test_dwconv3x3_matches_reference(in_f32, out_f32, stride, gelu):
    bad = []
    for H, W in DW_MAPS:
        for C in (3, 20, 256):
            _, ok = _dw_case(2, H, W, C, stride, gelu, in_f32, out_f32, seed=H * 1000 + W * 10 + C + stride)
            if not ok:
                bad.append((H, W, C))
    assert not bad, f"over the bar at {bad}"


# the engine's depthwise convs: MBConv (vit_t 256^2 x 256 and TINY 64^2 x 128, fp16, GELU), PatchMerging (stride 2 and the
# stride-1 merge into the last stage), local_conv (fp32 in / out, no GELU)
DW_ENGINE = [(256, 256, 256, 1, 1, 0, 0), (64, 64, 128, 1, 1, 0, 0), (256, 256, 128, 2, 1, 0, 0), (64, 64, 320, 1, 1, 0, 0),
             (128, 128, 128, 1, 0, 1, 1), (64, 64, 160, 1, 0, 1, 1), (16, 16, 96, 1, 0, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,C,stride,gelu,in_f32,out_f32", DW_ENGINE)
def test_dwconv3x3_engine_shapes(H, W, C, stride, gelu, in_f32, out_f32):
    _, ok = _dw_case(1, H, W, C, stride, gelu, in_f32, out_f32, seed=H + C)
    assert ok


# ============================================================================================= 4. box tokens ====
def ref_box_tokens(boxes, hw, S, gauss, fixed, half_shift=True, scale=True, swap_xy=False, clamp=False):
    """apply_boxes in float64, cast to float32; then +0.5, /S, 2x - 1 and the Gaussian projection in float32 (HF's
    PositionEmbeddingRandom: a float32 matmul, so u*g0 and v*g1 rounded, then summed), 2 pi a in float32; sin / cos in float64
    of that float32 argument, plus `fixed` -> (tokens [M*7, D] float64, bound term per element)."""
    H, W = hw
    newh, neww = preshape(H, W, S)
    b = np.asarray(boxes, np.float64).reshape(-1, 2, 2).copy()
    if clamp:
        b[..., 0] = np.clip(b[..., 0], 0, W)
        b[..., 1] = np.clip(b[..., 1], 0, H)
    if scale:
        b[..., 0] *= neww / W
        b[..., 1] *= newh / H
    c = b.astype(np.float32)
    if swap_xy:
        c = c[..., ::-1]
    f = np.float32
    if half_shift:
        c = c + f(0.5)
    c = c / f(S)
    c = f(2) * c - f(1)
    g = gauss.cpu().numpy().astype(np.float32)
    ug, vg = c[..., 0:1] * g[0], c[..., 1:2] * g[1]
    a = ug + vg
    arg = f(2 * np.pi) * a
    assert arg.dtype == np.float32
    M, D = b.shape[0], fixed.shape[1]
    fx = fixed.cpu().double().numpy()
    tok = np.repeat(fx[None], M, 0)
    arg64 = arg.astype(np.float64)
    tok[:, 5:7, : D // 2] += np.sin(arg64)
    tok[:, 5:7, D // 2:] += np.cos(arg64)
    # argument: the kernel's fma and the reference's separate products round differently (<= u (|ug| + |vg| + |a|) each
    # side), and 2 pi a rounds once on each side: |d arg| <= 2 u (2 pi (|ug| + |vg| + |a|) + |arg|); sinf / cosf within 2 ulps
    # (<= 2u of a value <= 1, doubled for the ulp of [0.5, 1)), the fp32 add of `fixed` half an ulp of the result
    darg = 2 * U * (2 * np.pi * (np.abs(ug) + np.abs(vg) + np.abs(a)) + np.abs(arg))
    bound = np.zeros_like(tok)
    bound[:, 5:7] = np.concatenate([darg, darg], -1) + 4 * U + U * np.abs(tok[:, 5:7])
    return torch.from_numpy(tok.reshape(M * 7, D)), torch.from_numpy(bound.reshape(M * 7, D))


def _boxes(H, W, M, seed):
    rng = np.random.default_rng(seed)
    fixed = [[W * 0.2, H * 0.25, W * 0.7, H * 0.8], [-W * 0.3, -H * 0.2, W * 1.4, H * 1.1], [W * 0.4, H * 0.2, W * 0.4, H * 0.7],
             [W * 0.13 + 0.37, H * 0.31 + 0.61, W * 0.58 + 0.29, H * 0.77 + 0.13], [0, 0, W - 1, H - 1], [W * 2, H * 2, W * 3, H * 3],
             [-5.5, -7.25, -1.125, -0.5]]
    more = rng.uniform(-0.3, 1.3, (M - len(fixed), 4)) * [W, H, W, H]
    return np.concatenate([np.array(fixed), more])


def test_box_token_reference_matches_oracle():
    """ref_box_tokens rows 5, 6 equal the oracle's HF prompt-encoder sparse embedding of the box (and rows 0..4 the fixed
    tokens) at vit_t and TINY size, frames above and below S."""
    for d, hw in ((VIT_T, (480, 640)), (VIT_T, (2000, 1500)), (TINY, (120, 160)), (TINY, (300, 200))):
        sd = random_state_dict(d, 2)
        orc = SamOracle(d, sd)
        w = convert_state_dict(sd, d)
        for box in _boxes(*hw, 8, seed=hw[0]):
            ref, bound = ref_box_tokens([box], hw, d.img_size, w["pe.gauss"], w["fixed"])
            with torch.no_grad():
                sparse, _ = orc.pe(None, None, apply_box(box, hw, d.img_size)[None], None)
            # HF's float32 matmul may fuse u g0 + v g1 like the kernel: the same argument bound as the GPU test's bar
            err = (ref[5:7] - sparse[0, 0].double()).abs()
            assert bool((err <= bound[5:7]).all()), (d.img_size, hw, box, float(err.max()))
            assert torch.equal(ref[:5], w["fixed"][:5].double())


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,S,D", [(480, 640, 1024, 256), (2000, 1500, 1024, 256), (1, 1, 1024, 256), (7, 2000, 1024, 256),
                                     (120, 160, 256, 128), (300, 200, 256, 128)])
def test_box_tokens_match_reference(H, W, S, D):
    M = 17
    g = torch.Generator().manual_seed(H + W + D)
    gauss = torch.randn(2, D // 2, generator=g).cuda()
    fixed = torch.randn(7, D, generator=g).cuda()
    boxes = _boxes(H, W, M, seed=H * W)
    d_boxes = torch.from_numpy(boxes).cuda()
    newh, neww = preshape(H, W, S)
    outs = []
    for _ in range(2):
        tok, sent = _out(M * 7, D, torch.float32)
        _call("vlfm_sam_box_tokens", d_boxes.data_ptr(), M, H, W, newh, neww, S, gauss.data_ptr(), fixed.data_ptr(), tok.data_ptr(), D,
              _lib().stream_ptr())
        _check_written(tok, sent, M * 7, "box tokens")
        outs.append(tok[: M * 7].cpu())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
    got = outs[0]
    fixed_rows = torch.arange(M * 7) % 7 < 5
    assert torch.equal(got[fixed_rows], fixed.cpu().repeat(M, 1)[fixed_rows]), "iou / mask token rows are not copies of `fixed`"
    ref, bar = ref_box_tokens(boxes, (H, W), S, gauss, fixed)
    bar = bar.clamp_min(1e-30)
    err = (got.double() - ref).abs()
    mut = {"no +0.5": dict(half_shift=False), "no neww/W scale": dict(scale=False), "x and y swapped": dict(swap_xy=True),
           "box clamped to the frame": dict(clamp=True)}
    miss = {}
    for n, kw in mut.items():
        if n == "no neww/W scale" and (newh, neww) == (H, W):
            continue
        miss[n] = round(float((got.double() - ref_box_tokens(boxes, (H, W), S, gauss, fixed, **kw)[0]).abs().max()) / float(bar.max()), 1)
    _report(f"box tokens {H}x{W} S {S} D {D}", err, bar, miss)
    assert bool((err <= bar).all())
    for n, m in miss.items():
        assert m > 10, f"the test cannot tell the kernel from a reference with {n}"


# ============================================================================================ 5. mask finish ====
def _lerp(o_size, in_size, align_corners=False):
    """torch upsample_bilinear2d's source indices and float32 weights for in_size -> o_size"""
    o = np.arange(o_size, dtype=np.float32)
    if align_corners:
        sc = np.float32((in_size - 1) / (o_size - 1)) if o_size > 1 else np.float32(0)
        src = sc * o
    else:
        sc = np.float32(in_size) / np.float32(o_size)
        src = np.maximum(sc * (o + np.float32(0.5)) - np.float32(0.5), np.float32(0))
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < in_size - 1)
    w1 = (src - i0.astype(np.float32)).astype(np.float32)
    w0 = (np.float32(1) - w1).astype(np.float32)
    return i0, i1, torch.from_numpy(w0.astype(np.float64)), torch.from_numpy(w1.astype(np.float64))


def _resize(x, oh, ow, align_corners=False):
    """[M, h, w] float64 -> [M, oh, ow] with float32 indices / weights, blend in float64"""
    dev = x.device
    i0, i1, w0, w1 = (torch.as_tensor(a).to(dev) for a in _lerp(oh, x.shape[1], align_corners))
    y = x[:, i0] * w0[None, :, None] + x[:, i1] * w1[None, :, None]
    i0, i1, w0, w1 = (torch.as_tensor(a).to(dev) for a in _lerp(ow, x.shape[2], align_corners))
    return y[:, :, i0] * w0[None, None] + y[:, :, i1] * w1[None, None]


def ref_mask_finish(low, S, hw, align_corners=False, crop=True):
    """low-res logits [M, L, L] -> bilinear to S x S -> crop [:newh, :neww] -> bilinear to hw, before the threshold"""
    newh, neww = preshape(hw[0], hw[1], S)
    up = _resize(low.double(), S, S, align_corners)
    if crop:
        up = up[:, :newh, :neww]
    return _resize(up, hw[0], hw[1], align_corners)


def mask_eps(low):
    """Each of the two fp32 blends w0 (w0' A + w1' B) + w1 (...) rounds 4 times on the way to a convex combination: <= 4u
    max|input|; the second blend carries the first's error convexly: the kernel's pre-threshold value is within 8u max|low|
    of the reference (the weights and indices are the same float32 numbers on both sides).  One more u for second-order
    terms: eps = 9u max|low|."""
    return 9 * U * float(low.abs().max())


def _low(M, L, seed):
    """smooth random logits with sign changes: a coarse random field upsampled, plus noise"""
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(M, 1, 6, 6, generator=g)
    return (F.interpolate(c, (L, L), mode="bicubic", align_corners=False)[:, 0] + 0.1 * torch.randn(M, L, L, generator=g)).float()


def test_mask_finish_reference_matches_oracle_postprocess():
    """ref_mask_finish equals SamOracle.postprocess (F.interpolate twice, float32) before the threshold, to float32 rounding"""
    for L, S in ((64, 256), (256, 1024)):
        orc = types.SimpleNamespace(d=types.SimpleNamespace(img_size=S))
        low = _low(1, L, seed=L)
        for hw in ((120, 160), (160, 120), (7, 300), (300, 7), (1, 1), (S + 37, S // 2 + 3)):
            want = SamOracle.postprocess(orc, low[0], hw).double()
            got = ref_mask_finish(low, S, hw)[0]
            err = float((got - want).abs().max())
            assert err <= 16 * U * float(low.abs().max()), (L, S, hw, err)


MF_FRAMES = [(480, 640), (640, 480), (1536, 2048), (2048, 1536), (7, 2000), (2000, 7), (1, 1), (120, 160)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", MF_FRAMES)
@pytest.mark.parametrize("L,S", [(256, 1024), (64, 256)])
def test_mask_finish_matches_reference(H, W, L, S):
    M = 3
    low = _low(M, L, seed=H * 7 + W + L)
    dl = low.cuda()
    newh, neww = preshape(H, W, S)
    outs = []
    for _ in range(2):
        out = torch.full((M * H * W + SENT,), 0xAB, dtype=torch.uint8, device="cuda")
        _call("vlfm_sam_mask_finish", dl.data_ptr(), out.data_ptr(), M, L, S, newh, neww, H, W, _lib().stream_ptr())
        torch.cuda.synchronize()
        assert bool((out[: M * H * W] <= 1).all()), "mask elements left unwritten"
        assert bool((out[M * H * W:] == 0xAB).all()), "elements past the end were written"
        outs.append(out[: M * H * W].view(M, H, W))
    assert torch.equal(outs[0], outs[1])
    got = outs[0].bool()
    ref = ref_mask_finish(dl, S, (H, W))
    eps = mask_eps(low)
    sure = ref.abs() > eps
    bad = int((got != (ref > 0))[sure].sum())
    orc = types.SimpleNamespace(d=types.SimpleNamespace(img_size=S))
    for m in range(M):
        post = (SamOracle.postprocess(orc, low[m], (H, W)) > 0).cuda()
        assert torch.equal(post[sure[m]], got[m][sure[m]]), "disagrees with SamOracle.postprocess"
    miss = {}
    if H * W >= 100:
        mutants = {"align_corners=True": dict(align_corners=True)}
        if newh < S or neww < S:
            mutants["crop skipped"] = dict(crop=False)
        for n, kw in mutants.items():
            mref = ref_mask_finish(dl, S, (H, W), **kw)
            miss[n] = int(((mref > 0) != got)[mref.abs() > 10 * eps].sum())
    print(f"mask finish {H}x{W} L{L} S{S}: eps {eps:.3g}, pixels compared {float(sure.double().mean()):.4f}, disagreeing {bad}; "
          f"pixels where a mutant beyond 10 eps disagrees: {miss}")
    assert bad == 0
    for n, c in miss.items():
        assert c > 0, f"the test cannot tell the kernel from a reference with {n}"


@pytest.mark.gpu
def test_mask_finish_nan_low_gives_empty_mask():
    M, L, S, H, W = 3, 64, 256, 120, 160
    low = _low(M, L, seed=1)
    low[1] = float("nan")
    dl = low.cuda()
    out = torch.full((M, H, W), 0xAB, dtype=torch.uint8, device="cuda")
    _call("vlfm_sam_mask_finish", dl.data_ptr(), out.data_ptr(), M, L, S, *preshape(H, W, S), H, W, _lib().stream_ptr())
    torch.cuda.synchronize()
    assert int(out[1].sum()) == 0 and bool((out <= 1).all()) and int(out[0].sum()) > 0


# ============================================================================================ 6. mask logits ====
def ref_mask_logits(up, hyper, M, h, w, C):
    """logits[m, Y, X] = sum_c hyper[m, c] GELU(up[m, Y/2, X/2, (Y%2, X%2), c]) in float64 -> (logits, bar)"""
    u = up.double().view(M, h, w, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(M, 2 * h, 2 * w, C)
    hy = hyper.double().view(M, 1, 1, C)
    gl = F.gelu(u)
    out = (gl * hy).sum(-1)
    # C fp32 FMAs: <= C 2^-23 sum|h gelu(u)| (the issue's bar), plus the fp32 GELU of each term: erff is within 2 ulps of a
    # value in (-1, 1), an absolute 2^-23 that 0.5|u| carries into gelu(u) even where 1 + erf cancels (u < 0), and <= 4
    # relative roundings: |d gelu| <= u (|u| + 4|gelu(u)|) per term, weighted by |h|
    bar = C * 2.0 ** -23 * (gl * hy).abs().sum(-1) + (hy.abs() * U * (u.abs() + 4 * gl.abs())).sum(-1)
    return out.reshape(-1), bar.reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("M,h,w,C", [(2, 5, 7, 1), (2, 5, 7, 16), (2, 9, 4, 32), (2, 3, 11, 64), (3, 128, 128, 32), (3, 32, 32, 16)])
def test_mask_logits_match_reference(M, h, w, C):
    g = torch.Generator().manual_seed(h * w + C)
    up = (2 * torch.randn(M * h * w, 4 * C, generator=g)).cuda()
    hyper = torch.randn(M, C, generator=g).cuda()
    n = M * 4 * h * w
    outs = []
    for _ in range(2):
        lo, sent = _out(n, 1, torch.float32)
        _call("vlfm_sam_mask_logits", up.data_ptr(), hyper.data_ptr(), lo.data_ptr(), M, h, w, C, _lib().stream_ptr())
        _check_written(lo, sent, n, "mask logits")
        outs.append(lo[:n, 0])
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
    ref, bar = ref_mask_logits(up, hyper, M, h, w, C)
    err = (outs[0].double() - ref).abs()
    _report(f"mask logits M{M} {h}x{w} C{C}", err, bar)
    assert bool((err <= bar).all())


# ========================================================================================= 7. bit-exact ports ====
@pytest.mark.gpu
@pytest.mark.parametrize("B,h,w,C", [(2, 3, 5, 7), (1, 64, 64, 64), (2, 16, 16, 32), (1, 1, 2, 1)])
def test_pixel_shuffle2_scatter(B, h, w, C):
    x = torch.randn(B * h * w, 4 * C, generator=torch.Generator().manual_seed(h * w * C)).cuda()
    out, sent = _out(B * 4 * h * w, C, torch.float32)
    _call("vlfm_sam_pixel_shuffle2", x.data_ptr(), out.data_ptr(), B, h, w, C, _lib().stream_ptr())
    _check_written(out, sent, B * 4 * h * w, "pixel shuffle")
    ref = x.view(B, h, w, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * 4 * h * w, C)
    assert torch.equal(_bits(out[: B * 4 * h * w]), _bits(ref))


@pytest.mark.gpu
@pytest.mark.parametrize("rows,pe_rows,D", [(7 * 128, 7 * 128, 256), (3 * 4096, 4096, 256), (5 * 7, 7, 33), (1000, 1, 128)])
@pytest.mark.parametrize("which", ["both", "out16", "outp16"])
def test_add_pe_f16(rows, pe_rows, D, which):
    g = torch.Generator().manual_seed(rows + D)
    x = (10 * torch.randn(rows, D, generator=g)).cuda()
    pe = torch.randn(pe_rows, D, generator=g).cuda()
    o16, s16 = _out(rows, D, torch.float16)
    op16, sp16 = _out(rows, D, torch.float16, seed=8)
    a = o16 if which in ("both", "out16") else None
    b = op16 if which in ("both", "outp16") else None
    _call("vlfm_sam_add_pe_f16", x.data_ptr(), pe.data_ptr(), _lib().ptr(a), _lib().ptr(b), rows, pe_rows, D, _lib().stream_ptr())
    torch.cuda.synchronize()
    ref_p = (x + pe.repeat(rows // pe_rows, 1)).half()
    for buf, sent, ref, used in ((o16, s16, x.half(), a is not None), (op16, sp16, ref_p, b is not None)):
        if used:
            _check_written(buf, sent, rows, "add_pe")
            assert torch.equal(_bits(buf[:rows]), _bits(ref))
        else:
            assert bool(buf[:rows].isnan().all()), "a NULL output's buffer was written"


@pytest.mark.gpu
def test_decoder_init_frame_indices():
    M, F_, HW, D = 6, 3, 64, 32
    g = torch.Generator().manual_seed(0)
    emb = torch.randn(F_, HW, D, generator=g).cuda()
    nomask = torch.randn(D, generator=g).cuda()
    frame = torch.tensor([2, 0, -1, 1, 3, 2], dtype=torch.int32).cuda()
    keys, sent = _out(M * HW, D, torch.float32)
    keys[: M * HW] = 7.0                # finite, so that the NaN rows of invalid frames show they were written
    _call("vlfm_sam_decoder_init", emb.data_ptr(), frame.data_ptr(), nomask.data_ptr(), keys.data_ptr(), M, F_, HW, D, _lib().stream_ptr())
    torch.cuda.synchronize()
    k = keys[: M * HW].view(M, HW, D)
    for m, f in enumerate(frame.tolist()):
        if 0 <= f < F_:
            assert torch.equal(_bits(k[m]), _bits(emb[f] + nomask)), m
        else:
            assert bool(k[m].isnan().all()), f"box {m} (frame {f}) is not NaN"
    assert torch.equal(_bits(keys[M * HW:]), _bits(sent))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 257, 65536 + 77])
@pytest.mark.parametrize("with_b,gelu", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("inplace", [0, 1])
def test_add_act(n, with_b, gelu, inplace):
    """fp32 a (+ b), GELU as 0.5 x (1 + erf(x / sqrt 2)) in fp32 (the same operations as torch's CUDA ops, hence bitwise);
    the in-place form writes out32 over b (the engine's MBConv shortcut)."""
    if inplace and not with_b:
        pytest.skip("the in-place form needs b")
    g = torch.Generator().manual_seed(n + 10 * with_b + gelu)
    a = (3 * torch.randn(n, generator=g)).cuda()
    b = (3 * torch.randn(n, generator=g)).cuda() if with_b else None
    v = a + b if with_b else a.clone()
    ref = 0.5 * v * (1 + torch.erf(v * 0.70710678118654752)) if gelu else v
    o16, s16 = _out(n, 1, torch.float16)
    if inplace:
        o32 = b
        sent32 = None
    else:
        o32, sent32 = _out(n, 1, torch.float32, seed=9)
    _call("vlfm_sam_add_act", a.data_ptr(), _lib().ptr(b), o32.data_ptr(), o16.data_ptr(), n, gelu, _lib().stream_ptr())
    _check_written(o16, s16, n, "add_act fp16")
    assert torch.equal(_bits(o16[:n, 0]), _bits(ref.half()))
    if inplace:
        assert torch.equal(_bits(b), _bits(ref))
    else:
        _check_written(o32, sent32, n, "add_act fp32")
        assert torch.equal(_bits(o32[:n, 0]), _bits(ref))


# ============================================================================================= 8. preprocess ====
def _tables_dev(H, W, S):
    newh, neww = preshape(H, W, S)
    hb, hk, hks = bilinear_tables(W, neww)
    vb, vk, vks = bilinear_tables(H, newh)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return newh, neww, (t(hb), t(hk), hks, t(vb), t(vk), vks), int(pillow_vertical_first(H, W, newh))


def _run_preprocess(imgs, S):
    from vlfm_b200.vlm.sam_engine import PIXEL_MEAN, PIXEL_STD

    B, H, W, _ = imgs.shape
    newh, neww, (hb, hk, hks, vb, vk, vks), v_first = _tables_dev(H, W, S)
    mid = torch.empty(B * (newh * W if v_first else H * neww) * 3, dtype=torch.uint8, device="cuda")
    out, sent = _out(B * S * S, 3, torch.float16)
    d = torch.from_numpy(imgs).cuda()
    _call("vlfm_sam_preprocess", d.data_ptr(), mid.data_ptr(), out.data_ptr(), B, H, W, newh, neww, S, hb.data_ptr(), hk.data_ptr(), hks,
          vb.data_ptr(), vk.data_ptr(), vks, v_first, (ctypes.c_float * 3)(*PIXEL_MEAN), (ctypes.c_float * 3)(*PIXEL_STD),
          _lib().stream_ptr())
    _check_written(out, sent, B * S * S, "preprocess")
    return out[: B * S * S].view(B, S, S, 3).cpu()


# Pillow resizes these vertically first (more than 100x taller than wide, shrinking vertically)
TALL_NARROW = [(2000, 8), (1200, 7), (1200, 8), (1536, 3), (2048, 3), (2048, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1536, 2048), (2048, 1536), (7, 2000), (1, 1), (333, 517), (1000, 8), (150, 1), (1100, 11),
                                 (1025, 10)] + TALL_NARROW)
def test_preprocess_matches_oracle(H, W):
    """fp16 NHWC = the oracle's (torchvision -> Pillow) fp32 tensor rounded to fp16, bitwise; repeat launches equal"""
    S = 1024
    rng = np.random.default_rng(H * 3 + W)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    img[: H // 3] = (img[: H // 3] // 64) * 64
    ref, _ = preprocess(img, S)
    got = _run_preprocess(img[None], S)
    assert torch.equal(_bits(got), _bits(_run_preprocess(img[None], S)))
    ref16 = ref[0].permute(1, 2, 0).half()
    assert torch.equal(_bits(got[0]), _bits(ref16)), f"{int((got[0] != ref16).sum())} values differ"


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(480, 640), (2000, 8)])
def test_preprocess_batch_equals_single_frames(H, W):
    rng = np.random.default_rng(H + W)
    imgs = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    many = _run_preprocess(imgs, 1024)
    for b in range(3):
        assert torch.equal(_bits(many[b]), _bits(_run_preprocess(imgs[b:b + 1], 1024)[0])), b


# ====================================================================================== bad-argument table ====
def _bad_calls():
    """(kernel, name, args) of calls every entry point must refuse without a launch; buffers are small valid tensors"""
    lib = _lib()
    st = lib.stream_ptr()
    h = torch.zeros(8192, dtype=torch.float16, device="cuda")
    f = torch.zeros(4096, device="cuda")
    i = torch.zeros(64, dtype=torch.int32, device="cuda")
    u8 = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    P = h.data_ptr()
    Pf, Pi, Pu = f.data_ptr(), i.data_ptr(), u8.data_ptr()
    mean = (ctypes.c_float * 3)(0, 0, 0)
    std = (ctypes.c_float * 3)(1, 1, 1)
    pre = lambda B=1, H=4, W=4, OH=2, OW=2, S=4, hks=3, vks=3, vf=0, img=Pu: (img, Pu, P, B, H, W, OH, OW, S, Pi, Pi, hks, Pi, Pi, vks, vf,
                                                                           mean, std, st)
    t2i = lambda M=1, heads=1, Nq=7, Nk=300, ldq=16, part=None: (P, P, P, P, M, heads, Nq, Nk, ldq, 16, 16, 16, 0.25, Pf,
                                                                 part if part is not None else M * heads * 2 * Nq * 18, st)
    win = lambda C=64, heads=2, ws=7, B=1, qkv=P: (qkv, P, Pf, P, B, 7, 7, C, heads, ws, 0.17, st)
    return [
        ("vlfm_sam_preprocess", "OH > S", pre(OH=5)),
        ("vlfm_sam_preprocess", "OW < 1", pre(OW=0)),
        ("vlfm_sam_preprocess", "v_first 2", pre(vf=2)),
        ("vlfm_sam_preprocess", "hksize 0", pre(hks=0)),
        ("vlfm_sam_preprocess", "NULL image", pre(img=None)),
        ("vlfm_sam_dwconv3x3", "stride 0", (P, 0, Pf, Pf, P, 0, 1, 4, 4, 8, 0, 1, st)),
        ("vlfm_sam_dwconv3x3", "C 0", (P, 0, Pf, Pf, P, 0, 1, 4, 4, 0, 1, 1, st)),
        ("vlfm_sam_dwconv3x3", "NULL bias", (P, 0, Pf, None, P, 0, 1, 4, 4, 8, 1, 1, st)),
        ("vlfm_sam_add_act", "no output", (Pf, Pf, None, None, 16, 0, st)),
        ("vlfm_sam_add_act", "n 0", (Pf, Pf, Pf, None, 0, 0, st)),
        ("vlfm_sam_window_attention", "C != heads*32", win(C=96)),
        ("vlfm_sam_window_attention", "window 8", win(ws=8)),
        ("vlfm_sam_window_attention", "B 0", win(B=0)),
        ("vlfm_sam_window_attention", "NULL qkv", win(qkv=None)),
        ("vlfm_sam_box_tokens", "odd D", (Pf, 1, 4, 4, 4, 4, 4, Pf, Pf, Pf, 7, st)),
        ("vlfm_sam_box_tokens", "M 0", (Pf, 0, 4, 4, 4, 4, 4, Pf, Pf, Pf, 8, st)),
        ("vlfm_sam_add_pe_f16", "no output", (Pf, Pf, None, None, 4, 4, 8, st)),
        ("vlfm_sam_add_pe_f16", "pe NULL with outp16", (Pf, None, None, P, 4, 4, 8, st)),
        ("vlfm_sam_add_pe_f16", "pe_rows 0 with outp16", (Pf, Pf, None, P, 4, 0, 8, st)),
        ("vlfm_sam_decoder_init", "F 0", (Pf, Pi, Pf, Pf, 1, 0, 4, 8, st)),
        ("vlfm_sam_t2i_attention", "part_floats one short", t2i(part=1 * 1 * 2 * 7 * 18 - 1)),
        ("vlfm_sam_t2i_attention", "Nq 9", t2i(Nq=9)),
        ("vlfm_sam_t2i_attention", "ldq < heads*16", t2i(ldq=8)),
        ("vlfm_sam_t2i_attention", "Nk 0", t2i(Nk=0)),
        ("vlfm_sam_pixel_shuffle2", "w 0", (Pf, Pf, 1, 2, 0, 4, st)),
        ("vlfm_sam_mask_logits", "C 0", (Pf, Pf, Pf, 1, 2, 2, 0, st)),
        ("vlfm_sam_mask_finish", "newh > S", (Pf, Pu, 1, 4, 8, 9, 8, 4, 4, st)),
        ("vlfm_sam_mask_finish", "W 0", (Pf, Pu, 1, 4, 8, 8, 8, 4, 0, st)),
    ], (h, f, i, u8)


@pytest.mark.gpu
def test_bad_arguments_launch_nothing():
    lib = _lib()
    L = lib.load()
    calls, bufs = _bad_calls()
    torch.cuda.synchronize()
    for fn, name, args in calls:
        before = lib.launch_count()
        rc = getattr(L, fn)(*args)
        assert rc == VLFM_E_INVALID, f"{fn}: {name} returned {rc}"
        assert lib.launch_count() == before, f"{fn}: {name}: a kernel was launched"
    torch.cuda.synchronize()
    for b in bufs:
        assert int(b.double().abs().sum()) == 0, "a refused call wrote its output"
    # the same t2i call with the exact part size goes through
    before = lib.launch_count()
    args = list(next(a for fn, n, a in calls if n == "part_floats one short"))
    args[-2] += 1
    lib.check(L.vlfm_sam_t2i_attention(*args), "vlfm_sam_t2i_attention")
    assert lib.launch_count() == before + 2


# ========================================================================================== engine edge cases ====
@pytest.fixture(scope="module")
def tiny_engine():
    from vlfm_b200.vlm.sam_engine import MobileSamEngine

    eng = MobileSamEngine(TINY, convert_state_dict(random_state_dict(TINY, 0), TINY), max_batch=2)
    rng = np.random.default_rng(0)
    eng.encode(torch.from_numpy(rng.integers(0, 256, (2, 120, 160, 3), dtype=np.uint8)).cuda())
    return eng


def _decode(eng, boxes, fidx):
    m, low = eng.decode(torch.tensor(boxes, dtype=torch.float64).cuda(), torch.tensor(fidx, dtype=torch.int32).cuda(), (120, 160),
                        low_out=True)
    torch.cuda.synchronize()
    return m.clone(), low.clone()


@pytest.mark.gpu
def test_decode_invalid_frame_index_and_stale_rows(tiny_engine):
    """frame_idx [0, frames, 0, -1]: the invalid boxes give NaN low-res logits and an all-False mask, the valid ones are
    bitwise the decode without them; a later 2-box decode (on the same buffers, whose padded rows the NaN decode left
    behind) is bitwise the same decode run before it."""
    eng = tiny_engine
    boxes = [[20, 30, 100, 90], [10, 10, 150, 110], [60.5, 5.25, 140.75, 100.5], [0, 0, 159, 119]]
    _decode(eng, boxes, [0, 1, 0, 1])                               # buffers for 4 boxes, every row written with finite values
    two = [[30, 20, 120, 100], [5, 40, 80, 110]]
    m_before, l_before = _decode(eng, two, [1, 0])
    m, low = _decode(eng, boxes, [0, eng.frames, 0, -1])
    assert bool(low[1].isnan().all()) and bool(low[3].isnan().all())
    assert int(m[1].sum()) == 0 and int(m[3].sum()) == 0
    mv, lv = _decode(eng, [boxes[0], boxes[2]], [0, 0])
    assert torch.equal(_bits(low[[0, 2]]), _bits(lv)) and torch.equal(m[[0, 2]], mv)
    assert not bool(lv.isnan().any()) and int(mv.sum()) > 0
    _decode(eng, boxes, [0, eng.frames, 0, -1])                     # leave NaN rows behind again
    m_after, l_after = _decode(eng, two, [1, 0])
    assert torch.equal(_bits(l_after), _bits(l_before)) and torch.equal(m_after, m_before)
