"""The batch-1 variant of the attention kernel (attention_kernel<HDP, 4, true>, vit_ops.cu) behind vlfm_attention_f16.

It runs one CTA per (batch, head, 64-query block), 16 warps = 4 row groups x the 4 key parts of attention_kernel<HDP, 4>, with
each part's K / V behind its own mbarrier.  vlfm_attention_f16 picks it when B * heads * ceil(Nq / 64) <= 132 and Nk >= 64 (the
ViT-g at batch 1); VLFM_ATT_IMPL=b1 runs it for every shape (the edge shapes below), VLFM_ATT_IMPL=legacy never.  Its key parts,
64-key blocks and merge order are those of the 4-part legacy variant, so wherever that variant runs the bits must be equal."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from test_attention_ln_gpu import NAN16, _call, _inputs, _ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_legacy_sha256.json")

VIT = [(1, 16, 257, 257, 88), (2, 16, 257, 257, 88), (4, 16, 257, 257, 88)]
EDGE_N = (1, 63, 64, 65, 257, 272)
EDGE = ([(1, 2, nq, nk, 88) for nq in EDGE_N for nk in EDGE_N]
        + [(1, 2, nq, nk, hd) for hd in (8, 64, 96) for nq, nk in ((65, 257), (257, 272), (63, 64), (1, 1))])
CASES = list(dict.fromkeys(VIT + EDGE))


def _legacy_quad(B, heads, Nq, Nk):
    """vlfm_attention_f16's legacy choice of attention_kernel<HDP, 4> (four key parts)"""
    items = B * heads * ((Nq + 31) // 32)
    return items <= 264 and Nk >= 64


def _lib():
    from vlfm_b200 import _lib

    return _lib, _lib.load()


def _run(L, lib, buf, B, heads, Nq, Nk, hd, repeats=1):
    """The kernel on the strided q / k / v views (ld = 3 * heads * hd) into a NaN-filled output with 8 spare rows and columns
    (output stride != input stride); every repeat must give the same bits."""
    D = heads * hd
    q, k, v = buf[: B * Nq, :D], buf[: B * Nk, D : 2 * D], buf[: B * Nk, 2 * D :]
    outs = []
    for _ in range(repeats):
        o = torch.full((B * Nq + 8, D + 8), NAN16, dtype=torch.int16, device="cuda").view(torch.float16)
        L.check(_call(lib, L, q, k, v, o, B, heads, Nq, Nk, hd, hd ** -0.5), "vlfm_attention_f16")
        torch.cuda.synchronize()
        outs.append(o)
    for other in outs[1:]:
        assert torch.equal(other.view(torch.int16), outs[0].view(torch.int16)), "repeat calls differ"
    bits = outs[0].view(torch.int16)
    assert bool((bits[B * Nq :] == NAN16).all()) and bool((bits[:, D:] == NAN16).all()), "spare rows / columns were written"
    return outs[0][: B * Nq, :D]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["randn", "peaky", "plant"])
@pytest.mark.parametrize("B,heads,Nq,Nk,hd", CASES)
def test_attention_b1_vs_float64(B, heads, Nq, Nk, hd, mode, monkeypatch):
    """The batch-1 kernel against float64 with test_attention_f16_vs_float64's bar (same numerics: fp32 scores, exp2 online
    softmax, P rounded to fp16, fp32 P.V, output scaled by 1 / l in fp32), and bitwise equal to the 4-part legacy variant where
    that one runs; planted keys at every boundary of the key parts and their 64-key blocks (test_attention_ln_gpu.PLANT), and three
    wrong references (planted key dropped, keys of head h + 1, unscaled logits) must each miss by more than 10x the bar."""
    if mode == "plant" and (Nk != 257 or hd < 40):
        pytest.skip("keys are planted at the partition boundaries of Nk = 257; at hd 8 the other logits are too close to dominate")
    monkeypatch.setenv("VLFM_ATT_IMPL", "b1")
    L, lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(B * 7919 + heads * 131 + Nq * 17 + Nk * 3 + hd + len(mode) + 1)
    D, scale = heads * hd, hd ** -0.5
    buf, _, _, _, plant = _inputs(B, heads, Nq, Nk, hd, mode, g)
    buf = buf.cuda()
    q, k, v = buf[: B * Nq, :D], buf[: B * Nk, D : 2 * D], buf[: B * Nk, 2 * D :]
    got = _run(L, lib, buf, B, heads, Nq, Nk, hd, repeats=2)
    assert bool(torch.isfinite(got).all()), "non-finite output"
    if _legacy_quad(B, heads, Nq, Nk):
        monkeypatch.setenv("VLFM_ATT_IMPL", "legacy")
        assert torch.equal(_run(L, lib, buf, B, heads, Nq, Nk, hd).view(torch.int16), got.view(torch.int16)), "bits differ from <HDP, 4>"
    if Nk == 1:
        assert torch.equal(got.view(B, Nq, D), v.view(B, 1, D).expand(B, Nq, D)), "Nk = 1: the output must be V"
    got = got.double()
    ref, pi, qd, kd, vd = _ref(q, k, v, B, heads, Nq, Nk, hd, scale)
    S = float((qd.abs() @ kd.abs().transpose(-1, -2)).max())
    eps_s = 2.0 ** -23 * (2 * (hd + 5) * scale * S + Nk + 4)
    piv = (pi @ vd.abs()).transpose(1, 2).reshape(B * Nq, D)
    bar = 2.0 ** -11 * ref.abs() + (2.0 ** -11 + eps_s) * piv + Nk * 2.0 ** -25 * float(vd.abs().max())
    ratio = float(((got - ref).abs() / bar).max())
    msg = f"b1 {mode} B {B} heads {heads} Nq {Nq} Nk {Nk} hd {hd}: max err/bar {ratio:.3f} (eps_s {eps_s:.2e})"
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


def _legacy_cases():
    """(B, heads, Nq, Nk, hd, seed): the ViT-g at batch 1 (attention_kernel<96, 4>) and 2 (<96, 2>), MobileSAM's 7-key shape."""
    return [(1, 16, 257, 257, 88, 1), (2, 16, 257, 257, 88, 2), (4, 8, 7, 7, 32, 3)]


def _legacy_inputs(B, heads, Nq, Nk, hd, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(B * max(Nq, Nk), 3 * heads * hd, generator=g).half()


def _sha(t):
    return hashlib.sha256(t.contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest()


@pytest.mark.gpu
def test_attention_legacy_bits_and_selection(monkeypatch):
    """VLFM_ATT_IMPL=legacy gives the bits the mma.sync variants gave before the batch-1 kernel existed (sha256 of the output,
    tests/golden/attention_legacy_sha256.json); the default picks the batch-1 kernel at the ViT's batch 1 only."""
    L, lib = _lib()
    with open(GOLDEN) as f:
        golden = json.load(f)
    for B, heads, Nq, Nk, hd, seed in _legacy_cases():
        buf = _legacy_inputs(B, heads, Nq, Nk, hd, seed).cuda()
        monkeypatch.setenv("VLFM_ATT_IMPL", "legacy")
        legacy = _run(L, lib, buf, B, heads, Nq, Nk, hd)
        assert _sha(legacy) == golden[f"{B}x{heads}x{Nq}x{Nk}x{hd}"], (B, heads, Nq, Nk, hd)
        monkeypatch.setenv("VLFM_ATT_IMPL", "b1")
        b1 = _run(L, lib, buf, B, heads, Nq, Nk, hd)
        monkeypatch.delenv("VLFM_ATT_IMPL")
        default = _run(L, lib, buf, B, heads, Nq, Nk, hd)
        assert torch.equal(default.view(torch.int16), (b1 if (B, Nk) == (1, 257) else legacy).view(torch.int16)), (B, heads, Nq, Nk, hd)
    monkeypatch.setenv("VLFM_ATT_IMPL", "bogus")
    buf = _legacy_inputs(1, 2, 16, 16, 64, 0).cuda()
    o = torch.empty(16, 128, dtype=torch.float16, device="cuda")
    assert _call(lib, L, buf[:, :128], buf[:, 128:256], buf[:, 256:], o, 1, 2, 16, 16, 64, 0.125) == 1


def test_attention_b1_ptxas_no_spills(tmp_path):
    """The batch-1 variant (512 threads: at most 128 registers) compiles for sm_90a without spills (no GPU needed)."""
    from vlfm_b200 import build

    if not shutil.which(build.NVCC) and not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "vit_ops.cu")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "vit_ops.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert not [l for l in log.splitlines() if "C7518" in l]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    kernels = [p for p in props if re.match(r"_ZN4vlfm16attention_kernelILi\d+ELi4ELb1E", p[0])]
    assert len(kernels) == 2
    for name, _, st, ld in kernels:
        assert st == "0" and ld == "0", f"{name} spills ({st} B stores, {ld} B loads)"
