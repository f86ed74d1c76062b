"""wgmma GEMM vs a plain PyTorch fp32 reference of the same op (fp16 inputs, fp32
accumulation): tolerance 2e-3 relative to the output scale."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def run_gemm(a, w, bias, epi, resid=None):
    from vlfm_b200.vlm.dense import gemm_f16

    return gemm_f16(a, w, bias, epi, resid)


@pytest.mark.parametrize("M,N,K", [(257, 4224, 1408), (257, 1408, 6144), (128, 128, 64), (1, 256, 768),
                                   (300, 1408, 592), (32, 768, 768), (1000, 6144, 1408), (257, 9216, 1408),
                                   (77, 264, 72), (8224, 4224, 1408), (2100, 2312, 520)])
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
def test_gemm_matches_torch(M, N, K, epi):
    if epi in (1, 2) and (M, N, K) not in [(257, 4224, 1408), (300, 1408, 592), (77, 264, 72), (32, 768, 768), (8224, 4224, 1408), (2100, 2312, 520)]:
        pytest.skip("epilogue variants checked on a subset of shapes")
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K + epi)
    a = (torch.randn(M, K, generator=g) * 0.5).half().cuda()
    w = (torch.randn(N, K, generator=g) * 0.05).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    ref = a.float() @ w.float().t() + bias
    if epi == 1:
        ref = torch.nn.functional.gelu(ref)
    resid = None
    if epi == 2:
        resid = torch.randn(M, N, generator=g).float().cuda()
        ref = ref + resid
    out = run_gemm(a, w, bias, epi, resid)
    torch.cuda.synchronize()
    got = out.float()
    scale = ref.abs().max().item()
    tol = 2e-3 * scale if epi in (0, 1) else 2e-4 * scale
    assert torch.isfinite(got).all()
    assert (got - ref).abs().max().item() <= tol, f"max err {(got - ref).abs().max().item()} vs tol {tol}"


@pytest.mark.parametrize("M,N,K", [(257, 4224, 1408), (257, 1408, 6144), (129, 96, 72), (258, 1408, 1408), (386, 264, 200), (257, 6144, 1408)])
@pytest.mark.parametrize("epi", [0, 1, 2, 3, 4])
def test_tail_rows_on_cuda_cores(M, N, K, epi):
    """M = 128*q + r, r <= 2: the r tail rows are computed by the last row tile's CTAs on CUDA cores from the swizzled W stages
    (incl. split-K atomics for the residual epilogue, K and N tails).  Same tolerance as the tensor-core rows; the tail rows
    are also checked on their own."""
    g = torch.Generator(device="cpu").manual_seed(M * 11 + N * 5 + K + epi)
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
    out = run_gemm(a, w, bias, epi, resid)
    torch.cuda.synchronize()
    got = out.float()
    scale = ref.abs().max().item()
    tol = 2e-3 * scale if epi in (0, 1, 4) else 2e-4 * scale
    q = (M // 128) * 128
    assert torch.isfinite(got).all()
    assert (got[q:] - ref[q:]).abs().max().item() <= tol, f"tail rows: max err {(got[q:] - ref[q:]).abs().max().item()} vs tol {tol}"
    assert (got - ref).abs().max().item() <= tol


@pytest.mark.parametrize("M,N,K", [(257, 1408, 6144), (257, 1408, 1408), (32, 768, 3072), (10, 768, 768), (514, 1408, 6144), (300, 264, 520)])
def test_resid_layernorm_is_exact_and_bitwise_reproducible(M, N, K):
    """vlfm_gemm_f16_resid_ln: x += A W^T + b, y = LayerNorm(x).  The split-K partial sums are reduced in a fixed order by the
    LayerNorm launch: two runs give bit-identical x and y (round 1's red.add reduction did not), and both match torch fp32."""
    import ctypes
    from vlfm_b200 import _lib

    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(M + 3 * N + 5 * K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().cuda()
    w = (torch.randn(N, K, generator=g) * 0.05).half().cuda()
    bias = torch.randn(N, generator=g).float().cuda()
    x0 = (torch.randn(M, N, generator=g) * 3).float().cuda()
    gamma = (1 + 0.1 * torch.randn(N, generator=g)).float().cuda()
    beta = (0.1 * torch.randn(N, generator=g)).float().cuda()
    partials = torch.empty(8 * M * N, dtype=torch.float32, device="cuda")
    ref_x = x0 + a.float() @ w.float().t() + bias
    ref_y = torch.nn.functional.layer_norm(ref_x, (N,), gamma, beta, 1e-6)
    outs = []
    for rep in range(3):
        x = x0.clone()
        y16 = torch.empty(M, N, dtype=torch.float16, device="cuda")
        y32 = torch.empty(M, N, dtype=torch.float32, device="cuda")
        partials.fill_(float("nan"))                      # every slab the reduction reads must have been written by this call
        rc = lib.vlfm_gemm_f16_resid_ln(a.data_ptr(), w.data_ptr(), bias.data_ptr(), x.data_ptr(), M, N, K, K, K, N, gamma.data_ptr(),
                                        beta.data_ptr(), y16.data_ptr(), N, y32.data_ptr(), N, 1e-6, partials.data_ptr(), partials.numel() * 4,
                                        _lib.stream_ptr())
        _lib.check(rc, "vlfm_gemm_f16_resid_ln")
        torch.cuda.synchronize()
        outs.append((x, y32, y16))
    x, y32, y16 = outs[0]
    sx, sy = ref_x.abs().max().item(), ref_y.abs().max().item()
    assert torch.isfinite(x).all() and torch.isfinite(y32).all()
    assert (x - ref_x).abs().max().item() <= 2e-4 * sx
    assert (y32 - ref_y).abs().max().item() <= 1e-3 * sy and (y16.float() - ref_y).abs().max().item() <= 3e-3 * sy
    for x2, y2, h2 in outs[1:]:
        assert torch.equal(x, x2) and torch.equal(y32, y2) and torch.equal(y16, h2)
    # post-LN form: the fp32 output aliases the residual stream (Q-Former blocks)
    x = x0.clone()
    rc = lib.vlfm_gemm_f16_resid_ln(a.data_ptr(), w.data_ptr(), bias.data_ptr(), x.data_ptr(), M, N, K, K, K, N, gamma.data_ptr(), beta.data_ptr(),
                                    None, 0, x.data_ptr(), N, 1e-6, partials.data_ptr(), partials.numel() * 4, _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16_resid_ln")
    torch.cuda.synchronize()
    assert torch.equal(x, y32)
