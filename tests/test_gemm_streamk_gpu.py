"""Stream-K residual GEMM + LayerNorm (vlfm_gemm_f16_resid_ln below one wave of 128 x 128 tiles) and the sub-wave tile widths
(BN 96 / 64) of the other epilogues, against torch fp32.  The stream-K partial sums are reduced in a fixed order by the LayerNorm
launch, so repeated calls and a CUDA-graph replay give bit-identical results."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SLAB_BYTES = 130 * 128 * 4      # one 128 x 128 tile + 2 tail rows, fp32 (SK_SLAB in common.cuh)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(M, N, K):
    g = torch.Generator(device="cpu").manual_seed(M + 3 * N + 7 * K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().cuda()
    w = (torch.randn(N, K, generator=g) * 0.05).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    x0 = (torch.randn(M, N, generator=g) * 3).float().cuda()
    gamma = (1 + 0.1 * torch.randn(N, generator=g)).float().cuda()
    beta = (0.1 * torch.randn(N, generator=g)).float().cuda()
    return a, w, bias, x0, gamma, beta


def _call(lib, a, w, bias, x, gamma, beta, y16, y32, partials, nbytes):
    from vlfm_b200 import _lib

    M, K = a.shape
    N = w.shape[0]
    rc = lib.vlfm_gemm_f16_resid_ln(a.data_ptr(), w.data_ptr(), bias.data_ptr(), x.data_ptr(), M, N, K, K, K, N, gamma.data_ptr(),
                                    beta.data_ptr(), y16.data_ptr(), N, y32.data_ptr(), N, 1e-6, partials.data_ptr(), nbytes,
                                    _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16_resid_ln")


# (M, N, K, workspace slabs or None for P = SMs + tiles - 1): the ViT-g batch-1 shapes (proj, fc2), batch 2, M = 257 tail rows with
# a K of a few blocks (every CTA covers parts of two tiles), a K of one block (too few K-blocks to split: runs unsplit), rows that
# are not a tail (M = 300: the last row tile is partly past M), a workspace too small for P = SMs, and an N that is not a multiple of 128
CASES = [(257, 1408, 1408, None), (257, 1408, 6144, None), (514, 1408, 6144, None), (257, 1408, 256, None), (257, 1408, 64, None),
         (300, 1408, 1408, None), (257, 1408, 1408, 100), (257, 1408, 6144, 60), (257, 1000, 1408, None), (32, 768, 3072, None)]


@pytest.mark.parametrize("M,N,K,slabs", CASES)
def test_streamk_resid_layernorm(M, N, K, slabs):
    from vlfm_b200 import _lib

    lib = _lib.load()
    a, w, bias, x0, gamma, beta = _inputs(M, N, K)
    tiles = (M // 128 if M % 128 <= 2 and M > 128 else (M + 127) // 128) * ((N + 127) // 128)
    nslabs = slabs if slabs is not None else _sms() + tiles - 1
    partials = torch.empty(nslabs * SLAB_BYTES // 4, dtype=torch.float32, device="cuda")
    ref_x = x0 + a.float() @ w.float().t() + bias
    ref_y = torch.nn.functional.layer_norm(ref_x, (N,), gamma, beta, 1e-6)
    outs = []
    for rep in range(3):
        x = x0.clone()
        y16 = torch.empty(M, N, dtype=torch.float16, device="cuda")
        y32 = torch.empty(M, N, dtype=torch.float32, device="cuda")
        partials.fill_(float("nan"))                      # every slab the reduction reads must have been written by this call
        _call(lib, a, w, bias, x, gamma, beta, y16, y32, partials, partials.numel() * 4)
        torch.cuda.synchronize()
        outs.append((x, y32, y16))
    x, y32, y16 = outs[0]
    sx, sy = ref_x.abs().max().item(), ref_y.abs().max().item()
    assert torch.isfinite(x).all() and torch.isfinite(y32).all()
    assert (x - ref_x).abs().max().item() <= 2e-4 * sx
    assert (y32 - ref_y).abs().max().item() <= 1e-3 * sy and (y16.float() - ref_y).abs().max().item() <= 3e-3 * sy
    for x2, y2, h2 in outs[1:]:
        assert torch.equal(x, x2) and torch.equal(y32, y2) and torch.equal(y16, h2)
    # the same call captured in a CUDA graph and replayed: bit-identical to the eager calls
    xg = x0.clone()
    y16g = torch.empty(M, N, dtype=torch.float16, device="cuda")
    y32g = torch.empty(M, N, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            _call(lib, a, w, bias, xg, gamma, beta, y16g, y32g, partials, partials.numel() * 4)
        for _ in range(2):
            xg.copy_(x0)
            partials.fill_(float("nan"))
            graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(x, xg) and torch.equal(y32, y32g) and torch.equal(y16, y16g)


@pytest.mark.parametrize("M,N,K", [(257, 6144, 1408), (257, 4224, 1408), (300, 1000, 520), (257, 1520, 200)])
@pytest.mark.parametrize("epi", [0, 1, 2, 3, 4])
def test_sub_wave_tile_widths(M, N, K, epi):
    """Below one wave the non-residual epilogues pick BN 96 (ViT fc1: 6144 columns) or 64 (qkv: 4224 columns): every epilogue at
    those widths, with tail rows and ragged N / K, at the tolerances of test_gemm_gpu.py."""
    from vlfm_b200.vlm.dense import gemm_f16

    g = torch.Generator(device="cpu").manual_seed(M * 13 + N + K + epi)
    a = (torch.randn(M, K, generator=g) * 0.5).half().cuda()
    w = (torch.randn(N, K, generator=g) * 0.05).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    ref = a.float() @ w.float().t() + bias
    if epi == 1:
        ref = torch.nn.functional.gelu(ref)
    if epi == 4:
        ref = torch.relu(ref)
    resid = None
    if epi == 2:
        resid = torch.randn(M, N, generator=g).float().cuda()
        ref = ref + resid
    got = gemm_f16(a, w, bias, epi, resid).float()
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    tol = 2e-3 * scale if epi in (0, 1, 4) else 2e-4 * scale
    assert torch.isfinite(got).all()
    assert (got - ref).abs().max().item() <= tol
