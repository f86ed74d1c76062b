"""Attention and LayerNorm kernels vs high-precision references of the same op."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN16 = 0x7E5A        # fp16 NaN with a payload: an untouched spare element still holds exactly this bit pattern

# vlfm_attention_f16 picks its variant from items = B * heads * ceil(Nq / 32) (vit_ops.cu; VLFM_ATT_KH4 unset): KH = 1 (64-row
# blocks, every warp sees all keys) above two waves of 264 items, KH = 4 (four key parts) up to one wave when Nk >= 64, else KH = 2.


def _variant(B, heads, Nq, Nk, hd):
    items = B * heads * ((Nq + 31) // 32)
    kh = 1 if items > 2 * 264 else (4 if items <= 264 and Nk >= 64 else 2)
    return kh, 64 if hd <= 64 else 96


VIT = [(1, 16, 257, 257, 88), (2, 16, 257, 257, 88), (3, 16, 257, 257, 88), (4, 16, 257, 257, 88), (32, 16, 257, 257, 88)]
QFORMER = [(1, 12, 32, 257, 64), (24, 12, 32, 257, 64), (64, 12, 32, 32, 64)]
LEGACY = [(1, 16, 257, 257, 88), (8, 16, 257, 257, 88), (4, 12, 32, 257, 64), (64, 12, 32, 32, 64), (1, 12, 7, 7, 64), (3, 2, 17, 16, 16)]
NQS, NKS, HDS = (1, 31, 33, 65, 257), (1, 16, 17, 63, 64, 65, 257, 271, 272), (8, 40, 64, 72, 88, 96)
EDGE = ([(1, 2, nq, nk, 40) for nq in NQS for nk in NKS]             # KH 4 (Nk >= 64) / KH 2, zero columns 40..63 of HDP 64
        + [(6, 24, 33, nk, 96) for nk in NKS]                       # KH 2 (288 items)
        + [(12, 16, 65, nk, 72) for nk in NKS]                      # KH 1 (576 items), zero columns 72..95 of HDP 96
        + [c for hd in HDS for c in ((1, 2, 31, 257, hd), (6, 24, 33, 257, hd), (12, 16, 65, 257, hd))])
CASES = list(dict.fromkeys(VIT + QFORMER + LEGACY + EDGE))

# a dominant key at every boundary of the key partition for Nk = 257 (17 tiles of 16): 64-key blocks (63/64, 127/128), the KH 4
# parts of 5 + 4 + 4 + 4 tiles (79/80, 143/144, 207/208), the KH 2 parts of 9 + 8 tiles (143/144), and key 256, the only live key
# of the last (padded) tile
PLANT = (0, 63, 64, 79, 80, 127, 128, 143, 144, 207, 208, 256)


def test_case_list_covers_every_variant():
    assert {_variant(*c) for c in CASES} == {(kh, hdp) for kh in (4, 2, 1) for hdp in (64, 96)}
    assert [_variant(*c)[0] for c in VIT] == [4, 2, 2, 1, 1] and [_variant(*c)[0] for c in QFORMER] == [4, 2, 1]
    assert _variant(1, 2, 31, 63, 40)[0] == 2 and _variant(1, 2, 31, 64, 40)[0] == 4


def _lib():
    from vlfm_b200 import _lib

    return _lib, _lib.load()


def _inputs(B, heads, Nq, Nk, hd, mode, g):
    """q, k, v as column slices of one [B * max(Nq, Nk), 3 * heads * hd] fp16 buffer (the engine's qkv GEMM output), and the
    planted key of every (b, h, query) row (or None)."""
    D = heads * hd
    buf = torch.randn(B * max(Nq, Nk), 3 * D, generator=g).half()
    q, k, v = buf[: B * Nq, :D], buf[: B * Nk, D : 2 * D], buf[: B * Nk, 2 * D :]
    scale = hd ** -0.5
    plant = None
    if mode == "peaky":       # |scale * s| up to ~30
        q.mul_(6.0)
    elif mode == "plant":     # q_row = t * k_j / (scale |k_j|^2): the scaled logit of key j is t in [6, 10], the others ~ t / sqrt(hd)
        kk = k.float().view(B, Nk, heads, hd)
        qq = q.view(B, Nq, heads, hd)
        r = torch.arange(Nq)
        plant = torch.empty(B, heads, Nq, dtype=torch.long)
        for b in range(B):
            for h in range(heads):
                j = torch.tensor(PLANT)[(r + 5 * b + 3 * h) % len(PLANT)]
                t = 6.0 + 4.0 * torch.rand(Nq, generator=g)
                kj = kk[b, j, h]
                qq[b, :, h] = (kj * (t / (scale * (kj * kj).sum(-1)))[:, None]).half()
                plant[b, h] = j
    return buf, q, k, v, plant


def _ref(q, k, v, B, heads, Nq, Nk, hd, scale, drop=None):
    """float64 softmax(scale q k^T) v on the fp16 operands -> out [B*Nq, heads*hd], weights pi [B, heads, Nq, Nk]"""
    qd = q.double().view(B, Nq, heads, hd).transpose(1, 2)
    kd = k.double().view(B, Nk, heads, hd).transpose(1, 2)
    vd = v.double().view(B, Nk, heads, hd).transpose(1, 2)
    s = qd @ kd.transpose(-1, -2) * scale
    if drop is not None:
        s.scatter_(-1, drop[..., None], -math.inf)
    pi = torch.softmax(s, -1)
    return (pi @ vd).transpose(1, 2).reshape(B * Nq, heads * hd), pi, qd, kd, vd


def _call(lib, L, q, k, v, o, B, heads, Nq, Nk, hd, scale, ldq=None, ldo=None):
    return lib.vlfm_attention_f16(q.data_ptr() if q is not None else None, k.data_ptr(), v.data_ptr(), o.data_ptr(), B, heads, Nq, Nk, hd,
                                  ldq if ldq is not None else q.stride(0), k.stride(0), v.stride(0), ldo if ldo is not None else o.stride(0),
                                  ctypes.c_float(scale), L.stream_ptr())


@pytest.mark.parametrize("mode", ["randn", "peaky", "plant"])
@pytest.mark.parametrize("B,heads,Nq,Nk,hd", CASES)
def test_attention_f16_vs_float64(B, heads, Nq, Nk, hd, mode):
    """vlfm_attention_f16 on the engine's strided q / k / v against a float64 reference.

    Error model.  The kernel computes the scores in fp32 (mma.sync, fp16 products exact), scales them by fp32 scale * log2(e),
    takes exp2 against a running max, rounds P to fp16 for the P.V mma (relative error 2^-11; below 2^-14 an absolute 2^-25), keeps
    l as the sum of the unrounded fp32 P, accumulates P.V in fp32 and rounds the output to fp16 (2^-11 relative).  So

        bar = 2^-11 |ref| + (2^-11 + eps_s) sum_j pi_j |v_j| + Nk 2^-25 max|v|

    with pi the float64 softmax and eps_s the relative error of P_j / l from the fp32 arithmetic:

        eps_s = 2^-23 (2 (hd + 5) scale S + Nk + 4),   S = max over (row, key) of sum_d |q_d k_d|.

    2 (hd + 5) scale S 2^-23 bounds the error of the exponent (natural-log units): the fp32 accumulation of hd products (one ulp
    per add), the roundings of scale * log2(e), of the scaled score and of the subtraction of the running max, counted twice since
    P_j / l is a ratio; Nk 2^-23 covers the fp32 sums of l and of P.V, and 4 * 2^-23 the exp2f error.  Observed err / bar: printed.

    A small bar proves little unless wrong answers miss it: for planted keys, three wrong references (planted key dropped, keys of
    head h + 1, unscaled logits) must each miss the kernel by more than 10x the bar somewhere."""
    if mode == "plant" and (Nk != 257 or hd < 40):
        pytest.skip("keys are planted at the partition boundaries of Nk = 257; at hd 8 the other logits are too close to dominate")
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(B * 7919 + heads * 131 + Nq * 17 + Nk * 3 + hd + len(mode))
    D, scale = heads * hd, hd ** -0.5
    buf, q, k, v, plant = _inputs(B, heads, Nq, Nk, hd, mode, g)
    buf = buf.cuda()
    q, k, v = buf[: B * Nq, :D], buf[: B * Nk, D : 2 * D], buf[: B * Nk, 2 * D :]
    outs = []
    for _ in range(3):
        o = torch.full((B * Nq + 8, D + 8), NAN16, dtype=torch.int16, device="cuda").view(torch.float16)
        L.check(_call(lib, L, q, k, v, o, B, heads, Nq, Nk, hd, scale), "vlfm_attention_f16")
        torch.cuda.synchronize()
        outs.append(o)
    o = outs[0]
    for other in outs[1:]:
        assert torch.equal(other.view(torch.int16), o.view(torch.int16)), "repeat calls differ"
    bits = o.view(torch.int16)
    assert bool((bits[B * Nq :] == NAN16).all()) and bool((bits[:, D:] == NAN16).all()), "spare rows / columns were written"
    got = o[: B * Nq, :D]
    assert bool(torch.isfinite(got).all()), "non-finite output"
    if Nk == 1:   # one key: P = 1, l = 1, the output is V itself
        assert torch.equal(got.view(B, Nq, D), v.view(B, 1, D).expand(B, Nq, D)), "Nk = 1: the output must be V"
    got = got.double()
    ref, pi, qd, kd, vd = _ref(q, k, v, B, heads, Nq, Nk, hd, scale)
    S = float((qd.abs() @ kd.abs().transpose(-1, -2)).max())
    eps_s = 2.0 ** -23 * (2 * (hd + 5) * scale * S + Nk + 4)
    piv = (pi @ vd.abs()).transpose(1, 2).reshape(B * Nq, D)
    bar = 2.0 ** -11 * ref.abs() + (2.0 ** -11 + eps_s) * piv + Nk * 2.0 ** -25 * float(vd.abs().max())
    ratio = float(((got - ref).abs() / bar).max())
    kh, hdp = _variant(B, heads, Nq, Nk, hd)
    msg = f"KH {kh} HDP {hdp} {mode} B {B} heads {heads} Nq {Nq} Nk {Nk} hd {hd}: max err/bar {ratio:.3f} (eps_s {eps_s:.2e})"
    if plant is not None:
        pw = pi.gather(-1, plant.cuda()[..., None])
        assert float(pw.min()) >= 0.3, "a planted key carries under 30 % of its row"
        kroll = k.view(B * Nk, heads, hd).roll(-1, dims=1).reshape(B * Nk, D)
        wrong = {"dropped": _ref(q, k, v, B, heads, Nq, Nk, hd, scale, drop=plant.cuda())[0],
                 "head+1": _ref(q, kroll, v, B, heads, Nq, Nk, hd, scale)[0],
                 "unscaled": _ref(q, k, v, B, heads, Nq, Nk, hd, 1.0)[0]}
        miss = {n: float(((got - w).abs() / bar).max()) for n, w in wrong.items()}
        msg += ", controls miss by " + ", ".join(f"{n} {m:.0f}x" for n, m in miss.items())
        for n, m in miss.items():
            assert m > 10.0, (n, m)
    print(msg)
    assert ratio <= 1.0, msg


def test_attention_f16_argument_errors():
    """Unsupported shapes / strides return VLFM_E_UNSUPPORTED (3), bad arguments VLFM_E_INVALID (1); neither launches."""
    L, lib = _lib()
    buf = torch.zeros(4 * 273, 3 * 2 * 104, dtype=torch.float16, device="cuda")
    o = torch.zeros(4 * 273, 2 * 104 + 8, dtype=torch.float16, device="cuda")

    def call(B=1, Nk=16, hd=64, ldq=None, ldo=None, q=buf):
        return _call(lib, L, q, buf, buf, o, B, 2, 16, Nk, hd, 0.125, ldq=ldq if ldq is not None else buf.stride(0), ldo=ldo)

    n0 = L.launch_count()
    assert call(Nk=273) == 3
    assert call(hd=100) == 3
    assert call(hd=12) == 3
    assert call(ldq=4) == 3
    assert call(ldo=o.stride(0) - 1) == 3
    assert call(B=0) == 1
    assert call(q=None) == 1
    assert L.launch_count() == n0
    assert call(Nk=272, hd=96) == 0
    torch.cuda.synchronize()
    assert L.launch_count() == n0 + 1


# D = 4, 256 / 260, 768 / 772, 1536: both sides of the <2> / <6> / <12> float4-per-lane instantiations of layernorm_kernel;
# rows = 1, 3, 5 around its four rows per block
@pytest.mark.parametrize("rows,D,eps", [(257, 1408, 1e-6), (32, 768, 1e-12), (19200, 96, 1e-5), (5, 1536, 1e-5), (100, 64, 1e-5),
                                        (1, 4, 1e-5), (5, 4, 1e-5), (3, 256, 1e-5), (1, 260, 1e-5), (5, 768, 1e-6), (3, 772, 1e-6),
                                        (1, 1536, 1e-5), (3, 1536, 1e-6)])
def test_layernorm_matches_torch(rows, D, eps):
    from vlfm_b200.vlm.dense import layernorm

    g = torch.Generator(device="cpu").manual_seed(rows + D)
    x = (torch.randn(rows, D, generator=g) * 3 + 0.7).cuda()
    gamma = (1 + 0.1 * torch.randn(D, generator=g)).cuda()
    beta = (0.1 * torch.randn(D, generator=g)).cuda()
    o16, o32 = layernorm(x, gamma, beta, eps, True, True)
    ref = torch.nn.functional.layer_norm(x, (D,), gamma, beta, eps)
    assert (o32 - ref).abs().max().item() <= 2e-5
    assert (o16.float() - ref).abs().max().item() <= 4e-3
    # the same rows as column windows of wider buffers (ldx, ldo16, ldo32 = D + 12, a spare row below): the same bits, and every
    # spare element of x (NaN) stays unread and every spare element of the outputs keeps its payload-NaN bits
    ld = D + 12
    win = (slice(0, rows), slice(4, 4 + D))
    xb = torch.full((rows + 1, ld), float("nan"), device="cuda")
    xb[win] = x
    o16b = torch.full((rows + 1, ld), NAN16, dtype=torch.int16, device="cuda")
    o32b = torch.full((rows + 1, ld), 0x7FC05A5A, dtype=torch.int32, device="cuda")
    layernorm(xb[win], gamma, beta, eps, o16b.view(torch.float16)[win], o32b.view(torch.float32)[win])
    torch.cuda.synchronize()
    assert torch.equal(o16b[win], o16.view(torch.int16)) and torch.equal(o32b[win], o32.view(torch.int32))
    spare = torch.ones(rows + 1, ld, dtype=torch.bool, device="cuda")
    spare[win] = False
    assert bool((o16b[spare] == NAN16).all()) and bool((o32b[spare] == 0x7FC05A5A).all())
