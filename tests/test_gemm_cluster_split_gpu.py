"""The batch-1 ViT plan of the wgmma GEMM (VLFM_EPI_CLUSTER_SPLIT): 256 < M <= 258 rows in one 256-row tile per column block,
K split over a thread-block cluster and reduced in shared memory.  Against float64 at the fp16 GEMM's tolerances (2e-3 of the
output scale for fp16 outputs, 2e-4 for fp32), every epilogue, ragged N and K, the unsplit (one K-block) case, bitwise repeats
and CUDA-graph replay, and the rows where the flag must change nothing."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

FLAG = 256   # VLFM_EPI_CLUSTER_SPLIT


@pytest.fixture(autouse=True)
def every_shape(monkeypatch):
    """By default the plan runs for weights of at least 8 Mi elements only (ViT fc1 and fc2); =2 runs it for every shape it can
    take, so that the small and ragged shapes below exercise it too."""
    monkeypatch.setenv("VLFM_GEMM_CSPLIT", "2")

# the four ViT-g layer GEMMs at batch 1 (qkv, proj, fc1, fc2) with the epilogue the forward runs them with
VIT = [(257, 4224, 1408, 0), (257, 1408, 1408, 2), (257, 6144, 1408, 1), (257, 1408, 6144, 2)]
# M = 258 (two tail rows), N not a multiple of any tile width, K not a multiple of 64, few K-blocks (cluster capped at nk),
# one K-block (no split: the epilogue runs straight from the fragments), K = 8.  (The residual epilogue of vlfm_gemm_f16 without
# the flag splits K with atomics at some of the shapes of the next test, so that one compares fp32 outputs instead.)
EDGE = [(M, N, K, e) for (M, N, K) in [(258, 1000, 1000), (257, 520, 200), (258, 1408, 64), (257, 296, 8), (258, 4224, 1408)]
        for e in range(5)]


def _inputs(M, N, K, epi):
    g = torch.Generator(device="cpu").manual_seed(M * 13 + N * 5 + K + epi)
    a = (torch.randn(M, K, generator=g) * 0.5).half().cuda()
    w = (torch.randn(N, K, generator=g) * 0.05).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    resid = (torch.randn(M, N, generator=g) * 3).float().cuda()
    return a, w, bias, resid


def _reference(a, w, bias, resid, epi):
    ref = a.double() @ w.double().t() + bias.double()
    if epi == 1:
        ref = torch.nn.functional.gelu(ref)
    elif epi == 4:
        ref = torch.relu(ref)
    elif epi == 2:
        ref = ref + resid.double()
    return ref


def _run(a, w, bias, resid, epi, flag):
    """One call into a fresh output: the residual stream copied from `resid`, every other output prefilled with NaN."""
    from vlfm_b200.vlm.dense import gemm_f16

    M, N = a.shape[0], w.shape[0]
    if epi == 2:
        out = resid.clone()
    else:
        out = torch.full((M, N), float("nan"), dtype=torch.float32 if epi == 3 else torch.float16, device="cuda")
    gemm_f16(a, w, bias, epi | flag, out)
    return out


@pytest.mark.parametrize("M,N,K,epi", VIT + EDGE)
def test_cluster_split_matches_float64(M, N, K, epi):
    a, w, bias, resid = _inputs(M, N, K, epi)
    ref = _reference(a, w, bias, resid, epi)
    outs = [_run(a, w, bias, resid, epi, FLAG) for _ in range(3)]
    torch.cuda.synchronize()
    got = outs[0].double()
    assert torch.isfinite(got).all(), "an output element was not written"
    scale = ref.abs().max().item()
    tol = (2e-3 if epi in (0, 1, 4) else 2e-4) * scale
    err = (got - ref).abs()
    assert err.max().item() <= tol, f"max err {err.max().item()} vs tol {tol}"
    assert err[256:].max().item() <= tol, "tail rows"
    for o in outs[1:]:
        assert torch.equal(outs[0], o)
    # the same call captured in a CUDA graph and replayed twice: bit-identical to the eager calls
    out_g = resid.clone() if epi == 2 else torch.empty_like(outs[0])
    from vlfm_b200.vlm.dense import gemm_f16

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            gemm_f16(a, w, bias, epi | FLAG, out_g)
        for _ in range(2):
            if epi == 2:
                out_g.copy_(resid)
            else:
                out_g.fill_(float("nan"))
            graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], out_g)


@pytest.mark.parametrize("M", [256, 259, 385])
@pytest.mark.parametrize("N,K,epi", [(4224, 1408, 0), (1408, 6144, 3), (1000, 1000, 1)])
def test_flag_changes_nothing_outside_257_258_rows(M, N, K, epi):
    """The cluster split changes the order of a row's sums.  Outside 257-258 rows the flag must leave the plan alone, so that a
    row's bits do not depend on M for callers that pad (MobileSAM) or batch."""
    a, w, bias, resid = _inputs(M, N, K, epi)
    with_flag = _run(a, w, bias, resid, epi, FLAG)
    without = _run(a, w, bias, resid, epi, 0)
    torch.cuda.synchronize()
    assert torch.equal(with_flag, without)


@pytest.mark.parametrize("K", [1408, 6144])
def test_resid_ln_with_workspace_takes_the_cluster_split(K):
    """vlfm_gemm_f16_resid_ln with a workspace at 257 rows runs the cluster split: the LayerNorm launch reads x only, so the
    NaN-prefilled workspace stays untouched, and the result matches float64."""
    from vlfm_b200 import _lib
    from vlfm_b200.vlm.dense import gemm_f16_resid_ln

    M, N = 257, 1408
    a, w, bias, x0 = _inputs(M, N, K, 2)
    g = torch.Generator(device="cpu").manual_seed(K)
    gamma = (1 + 0.1 * torch.randn(N, generator=g)).float().cuda()
    beta = (0.1 * torch.randn(N, generator=g)).float().cuda()
    partials = torch.full((8 * M * N,), float("nan"), device="cuda")
    x = x0.clone()
    y32 = torch.empty(M, N, device="cuda")
    gemm_f16_resid_ln(a, w, bias, x, gamma, beta, 1e-6, out32=y32, partials=partials)
    torch.cuda.synchronize()
    bn, s, nbytes = ctypes.c_int(), ctypes.c_int(), ctypes.c_double()
    _lib.load().vlfm_gemm_csplit_plan(M, N, K, ctypes.addressof(bn), ctypes.addressof(s), ctypes.addressof(nbytes))
    if bn.value:
        assert bool(torch.isnan(partials).all())
    ref_x = _reference(a, w, bias, x0, 2)
    ref_y = torch.nn.functional.layer_norm(ref_x, (N,), gamma.double(), beta.double(), 1e-6)
    assert (x.double() - ref_x).abs().max().item() <= 2e-4 * ref_x.abs().max().item()
    assert (y32.double() - ref_y).abs().max().item() <= 1e-3 * ref_y.abs().max().item()
    # the same as vlfm_gemm_f16 with the flag and the residual epilogue, then LayerNorm: one plan for both entry points
    assert torch.equal(x, _run(a, w, bias, x0, 2, FLAG))
