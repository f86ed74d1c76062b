"""The float32-grade "x2" path of the Q-Former (fp16 pairs hi + lo/2048 on the wgmma GEMM, float32 attention) against
float64 references of the same ops.  Tolerances are float32-arithmetic sized (1e-6 of the output scale), three orders of magnitude
below the plain fp16-operand GEMM's 2e-3."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(t):
    hi = t.half()
    lo = ((t - hi.float()) * 2048.0).half()
    return hi.contiguous(), lo.contiguous()


def _lib():
    from vlfm_b200 import _lib

    return _lib, _lib.load()


@pytest.mark.parametrize("M,N,K", [(32, 768, 768), (32, 3072, 768), (32, 2304, 768), (11, 768, 768), (257, 4608, 1408), (1024, 768, 768), (64, 256, 768)])
@pytest.mark.parametrize("epi", ["f32", "resid", "gelu_x2"])
def test_gemm_x2_vs_float64(M, N, K, epi):
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(M + 3 * N + 7 * K)
    a = (torch.randn(M, K, generator=g) * 0.7).cuda()
    a[0, :5] = torch.tensor([40.0, -25.0, 1e-4, 3e-6, 0.0])             # outliers / tiny values
    w = (torch.randn(N, K, generator=g) * 0.04).cuda()
    bias = torch.randn(N, generator=g).cuda()
    ahi, alo = _split(a)
    whi, wlo = _split(w)
    ref = a.double() @ w.double().t() + bias.double()
    st = L.stream_ptr()
    if epi == "f32":
        out = torch.empty(M, N, device="cuda")
        L.check(lib.vlfm_gemm_f16x2(ahi.data_ptr(), alo.data_ptr(), whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), out.data_ptr(), None,
                                    M, N, K, K, K, N, L.EPI_BIAS_F32, st), "gemm x2")
        got = out.double()
    elif epi == "resid":
        x = torch.randn(M, N, generator=g).cuda()
        ref = ref + x.double()
        L.check(lib.vlfm_gemm_f16x2(ahi.data_ptr(), alo.data_ptr(), whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), x.data_ptr(), None,
                                    M, N, K, K, K, N, L.EPI_BIAS_RESID_F32, st), "gemm x2")
        got = x.double()
    else:
        ref = torch.nn.functional.gelu(ref)
        ohi, olo = torch.empty(M, N, dtype=torch.float16, device="cuda"), torch.empty(M, N, dtype=torch.float16, device="cuda")
        L.check(lib.vlfm_gemm_f16x2(ahi.data_ptr(), alo.data_ptr(), whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), ohi.data_ptr(), olo.data_ptr(),
                                    M, N, K, K, K, N, L.EPI_BIAS_GELU_F16X2, st), "gemm x2")
        got = ohi.double() + olo.double() / 2048.0
    torch.cuda.synchronize()
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max())
    assert err <= 5e-6 * scale, f"max err {err:.3e} vs scale {scale:.3e}"


@pytest.mark.parametrize("M,N,K", [(32, 768, 768), (32, 768, 3072), (9, 768, 3072), (1024, 768, 3072)])
def test_gemm_x2_resid_layernorm(M, N, K):
    """x += A W^T + b; LayerNorm(x) as x2 operands: float64 reference, bitwise reproducible (deterministic split-K)."""
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a, w = (torch.randn(M, K, generator=g) * 0.5).cuda(), (torch.randn(N, K, generator=g) * 0.03).cuda()
    bias, x0 = torch.randn(N, generator=g).cuda(), torch.randn(M, N, generator=g).cuda()
    gam, bet = (1 + 0.1 * torch.randn(N, generator=g)).cuda(), (0.1 * torch.randn(N, generator=g)).cuda()
    ahi, alo = _split(a)
    whi, wlo = _split(w)
    part = torch.empty(8 * M * N, device="cuda")
    outs = []
    for _ in range(3):
        x = x0.clone()
        hi, lo = torch.empty(M, N, dtype=torch.float16, device="cuda"), torch.empty(M, N, dtype=torch.float16, device="cuda")
        o32 = torch.empty(M, N, device="cuda")
        L.check(lib.vlfm_gemm_f16x2_resid_ln(ahi.data_ptr(), alo.data_ptr(), whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), x.data_ptr(), M, N, K, K, K, N,
                                             gam.data_ptr(), bet.data_ptr(), hi.data_ptr(), lo.data_ptr(), N, o32.data_ptr(), N, 1e-12,
                                             part.data_ptr(), part.numel() * 4, L.stream_ptr()), "x2 resid ln")
        torch.cuda.synchronize()
        outs.append((x.clone(), hi.clone(), lo.clone(), o32.clone()))
    xr = x0.double() + a.double() @ w.double().t() + bias.double()
    yr = torch.nn.functional.layer_norm(xr, (N,), gam.double(), bet.double(), 1e-12)
    x, hi, lo, o32 = outs[0]
    assert float((x.double() - xr).abs().max()) <= 6e-6 * float(xr.abs().max())      # fp32 accumulation over K = 3072
    assert float((o32.double() - yr).abs().max()) <= 2e-5
    assert float((hi.double() + lo.double() / 2048.0 - o32.double()).abs().max()) <= 2e-6          # the pair carries the fp32 value
    for o in outs[1:]:
        assert all(torch.equal(p, q) for p, q in zip(o, outs[0]))


# 12 heads x 64 at 32 queries: the row-group count z of vlfm_attention_f32 is 4 up to B = 5, 3 at B = 6 (passes of 24 rows: the
# second one is partial), 2 at B = 8 and 1 from B = 12 (each warp loops over four query rows)
@pytest.mark.parametrize("B,heads,Nq,Nk,hd", [(1, 12, 32, 32, 64), (1, 12, 32, 257, 64), (3, 12, 32, 257, 64), (1, 2, 9, 9, 32), (2, 2, 8, 17, 32),
                                               (6, 12, 32, 257, 64), (8, 12, 32, 257, 64), (12, 12, 32, 257, 64), (32, 12, 32, 257, 64),
                                               (2, 12, 32, 1, 64), (2, 12, 32, 272, 64), (3, 12, 1, 257, 64), (3, 12, 33, 257, 64)])
def test_attention_f32_vs_float64(B, heads, Nq, Nk, hd):
    """The engine's strides: q a column slice of the [B*Nq, 3*H] q/k/v buffer, K / V one layer's slices of the cross-attention
    buffer [B*Nk, 6*2*H] (all layers' K|V side by side); hi / lo NaN-filled with 8 spare rows and columns that must stay NaN."""
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(Nq * 3 + Nk + 1000 * B)
    H = heads * hd
    qbuf = torch.randn(B * Nq, 3 * H, generator=g).cuda()
    kvbuf = torch.randn(B * Nk, 6 * 2 * H, generator=g).cuda()
    j = B % 6
    q, k, v = qbuf[:, :H], kvbuf[:, 2 * j * H : (2 * j + 1) * H], kvbuf[:, (2 * j + 1) * H : (2 * j + 2) * H]
    hi, lo = (torch.full((B * Nq + 8, H + 8), float("nan"), dtype=torch.float16, device="cuda") for _ in range(2))
    sc = hd ** -0.5
    L.check(lib.vlfm_attention_f32(q.data_ptr(), k.data_ptr(), v.data_ptr(), hi.data_ptr(), lo.data_ptr(), B, heads, Nq, Nk, hd, q.stride(0),
                                   k.stride(0), v.stride(0), hi.stride(0), ctypes.c_float(sc), L.stream_ptr()), "attention f32")
    torch.cuda.synchronize()
    for t in (hi, lo):
        assert bool(torch.isnan(t[B * Nq :]).all()) and bool(torch.isnan(t[:, H:]).all()), "spare rows / columns were written"
        assert bool(torch.isfinite(t[: B * Nq, :H]).all()), "output rows left unwritten or non-finite"
    qd, kd, vd = (t.double().reshape(B, -1, heads, hd).transpose(1, 2) for t in (q, k, v))
    ref = (torch.softmax(qd @ kd.transpose(-1, -2) * sc, -1) @ vd).transpose(1, 2).reshape(B * Nq, H)
    got = hi[: B * Nq, :H].double() + lo[: B * Nq, :H].double() / 2048.0
    assert float((got - ref).abs().max()) <= 2e-6 * max(1.0, float(ref.abs().max()))


def test_layernorm_x2_and_split():
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(5)
    x = (torch.randn(70, 768, generator=g) * 3).cuda()
    gam, bet = (1 + 0.1 * torch.randn(768, generator=g)).cuda(), (0.1 * torch.randn(768, generator=g)).cuda()
    hi, lo = torch.empty(70, 768, dtype=torch.float16, device="cuda"), torch.empty(70, 768, dtype=torch.float16, device="cuda")
    o32 = torch.empty(70, 768, device="cuda")
    L.check(lib.vlfm_layernorm_x2(x.data_ptr(), gam.data_ptr(), bet.data_ptr(), hi.data_ptr(), lo.data_ptr(), o32.data_ptr(), 70, 768, 768, 768, 768,
                                  ctypes.c_float(1e-12), L.stream_ptr()), "ln x2")
    ref = torch.nn.functional.layer_norm(x.double(), (768,), gam.double(), bet.double(), 1e-12)
    assert float((o32.double() - ref).abs().max()) <= 2e-6 * float(ref.abs().max())
    assert torch.equal(hi, o32.half())
    assert float((hi.double() + lo.double() / 2048.0 - o32.double()).abs().max()) <= 1e-6
    h2, l2 = torch.empty_like(hi), torch.empty_like(lo)
    L.check(lib.vlfm_split_x2(o32.data_ptr(), h2.data_ptr(), l2.data_ptr(), o32.numel(), L.stream_ptr()), "split")
    torch.cuda.synchronize()
    assert torch.equal(h2, hi) and torch.equal(l2, lo)
