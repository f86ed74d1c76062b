"""The conv-row contract shared by every conv net here: ``vlfm_im2col_f16`` (csrc/im2col.cu, through ``dense.im2col``) writes
exactly ``F.unfold`` reordered to (ky, kx, c) columns and zero-padded to ldk, bit for bit, and ``dense.conv_rows`` lays a conv
weight out in the same column order.

GPU outputs are prefilled with NaN and followed by NaN sentinel rows, so an unwritten element or a write past the end fails;
every launch is repeated and must reproduce its bits; bad arguments return VLFM_E_INVALID without a launch."""
import pytest
import torch
import torch.nn.functional as F

from vlfm_b200 import _lib
from vlfm_b200.vlm.dense import conv_rows, im2col

VLFM_E_INVALID = 1
SENT = 4             # sentinel rows after the output


def unfold_rows(x: torch.Tensor, k: int, stride: int, ldk: int) -> torch.Tensor:
    """x [B,H,W,C] -> [B*Ho*Wo, ldk]: F.unfold (pad k // 2) reordered to columns (ky, kx, c), zero-padded to ldk."""
    B, H, W, C = x.shape
    u = F.unfold(x.permute(0, 3, 1, 2), k, padding=k // 2, stride=stride)               # [B, C*k*k, L], rows (c, ky, kx)
    L = u.shape[-1]
    r = u.view(B, C, k * k, L).permute(0, 3, 2, 1).reshape(B * L, k * k * C)
    return F.pad(r, (0, ldk - k * k * C))


# --------------------------------------------------------------------------------------------------------- conv_rows (CPU)
@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("C,stride", [(3, 1), (5, 2), (16, 2)])
def test_conv_rows_times_unfold_rows_is_conv2d(k, C, stride):
    g = torch.Generator().manual_seed(k * 100 + C)
    B, H, W, O = 2, 9, 11, 6
    x = torch.randn(B, H, W, C, generator=g, dtype=torch.float64)
    w = torch.randn(O, C, k, k, generator=g, dtype=torch.float64)
    wr = conv_rows(w)
    ldk = (k * k * C + 7) // 8 * 8
    assert wr.shape == (O, ldk) and wr.dtype == w.dtype and wr.is_contiguous()
    assert torch.equal(wr[:, k * k * C:], torch.zeros(O, ldk - k * k * C, dtype=w.dtype))
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, stride=stride, padding=k // 2)             # [B, O, Ho, Wo]
    got = unfold_rows(x, k, stride, ldk) @ wr.T
    assert torch.allclose(got, ref.permute(0, 2, 3, 1).reshape(-1, O), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------ kernel (GPU)
# (B, H, W, C, k, stride, ldx, channel offset, ldk): x is channels [off, off + C) of [B, H, W, ldx] rows
CASES = [
    # MobileSAM: the stem (C = 3, K 27 -> 32), the neck (C = 256), odd maps, a 1 x 1 map, K padding
    (2, 17, 23, 3, 3, 2, 3, 0, 32), (1, 64, 64, 3, 3, 2, 3, 0, 32), (2, 9, 11, 256, 3, 1, 256, 0, 2304),
    (1, 16, 16, 256, 3, 1, 256, 0, 2304), (2, 7, 5, 5, 3, 1, 5, 0, 48), (2, 7, 5, 5, 3, 2, 5, 0, 48),
    (1, 1, 1, 5, 3, 2, 5, 0, 48), (3, 13, 8, 32, 3, 2, 32, 0, 288),
    # YOLOv7: a channel slice of a wider concat buffer
    (2, 9, 12, 24, 3, 1, 40, 8, 216), (2, 9, 12, 24, 3, 2, 40, 8, 216),
    # PointNav: the stride-2 1x1 downsample rows
    (2, 112, 112, 32, 1, 2, 32, 0, 32), (2, 106, 120, 32, 1, 2, 32, 0, 32), (2, 7, 9, 8, 1, 2, 8, 0, 8), (2, 1, 3, 16, 1, 2, 16, 0, 16),
    # GroundingDINO: the fourth neck level's 3x3 stride-2 conv on the last backbone stage
    (3, 15, 20, 768, 3, 2, 768, 0, 6912),
    # one column at a time: C % 8, ldx % 8, an input not 16-byte aligned; with ldk above k*k*C
    (1, 4, 4, 12, 3, 1, 12, 0, 112), (1, 4, 4, 12, 1, 2, 12, 0, 16), (1, 4, 4, 16, 1, 2, 24, 1, 16),
    (2, 9, 7, 12, 3, 1, 16, 1, 112), (2, 9, 7, 8, 3, 2, 12, 1, 72), (2, 5, 6, 3, 3, 1, 3, 0, 40), (1, 5, 6, 12, 1, 1, 12, 0, 24),
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C,k,stride,ldx,off,ldk", CASES)
def test_im2col_is_the_unfold(B, H, W, C, k, stride, ldx, off, ldk):
    full = torch.randn(B, H, W, ldx, generator=torch.Generator().manual_seed(H * W + C)).half()
    xs = full[..., off:off + C]
    x = full.cuda().view(B * H * W, ldx)[:, off:off + C]
    n = B * ((H - 1) // stride + 1) * ((W - 1) // stride + 1)
    outs = []
    for _ in range(2):
        col = torch.full((n + SENT, ldk), float("nan"), dtype=torch.float16, device="cuda")
        assert im2col(x, B, H, W, k, stride, col[:n]).data_ptr() == col.data_ptr()
        torch.cuda.synchronize()
        assert bool(col[n:].isnan().all()), "rows past the end were written"
        outs.append(col[:n].cpu())
    ref = unfold_rows(xs.float(), k, stride, ldk).half()
    assert torch.equal(outs[0].view(torch.int16), ref.view(torch.int16)), f"{int((outs[0] != ref).sum())} of {ref.numel()} values differ"
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))


@pytest.mark.gpu
def test_im2col_new_output_has_padded_ldk():
    x = torch.randn(2 * 5 * 6, 3, device="cuda").half()
    col = im2col(x, 2, 5, 6, 3, 2)
    assert col.shape == (2 * 3 * 3, 32)
    assert torch.equal(col.cpu(), unfold_rows(x.cpu().float().view(2, 5, 6, 3), 3, 2, 32).half())


@pytest.mark.gpu
def test_bad_arguments_are_refused_without_a_launch():
    lib = _lib.load()
    st = _lib.stream_ptr()
    buf = torch.zeros(8192, dtype=torch.float16, device="cuda")
    P = buf.data_ptr()
    # (name, (d_x16, ldx, d_col16, B, H, W, C, k, stride, ldk))
    calls = [
        ("ldk < k*k*C", (P, 3, P, 1, 4, 4, 3, 3, 1, 24)),
        ("ldk % 8", (P, 3, P, 1, 4, 4, 3, 3, 1, 36)),
        ("stride 3", (P, 3, P, 1, 4, 4, 3, 3, 3, 32)),
        ("stride 3, C % 8 == 0", (P, 16, P, 1, 4, 4, 16, 3, 3, 144)),
        ("k 2", (P, 8, P, 1, 4, 4, 8, 2, 1, 32)),
        ("ldx < C", (P, 4, P, 1, 4, 4, 8, 3, 1, 72)),
        ("NULL input", (None, 8, P, 1, 4, 4, 8, 3, 1, 72)),
        ("NULL output", (P, 8, None, 1, 4, 4, 8, 3, 1, 72)),
        ("misaligned output", (P, 8, P + 2, 1, 4, 4, 8, 3, 1, 72)),
        ("B 0", (P, 8, P, 0, 4, 4, 8, 3, 1, 72)),
        ("C 0", (P, 8, P, 1, 4, 4, 0, 3, 1, 8)),
    ]
    torch.cuda.synchronize()
    for name, args in calls:
        before = _lib.launch_count()
        rc = lib.vlfm_im2col_f16(*args, st)
        assert rc == VLFM_E_INVALID, f"{name} returned {rc}"
        assert _lib.launch_count() == before, f"{name}: a kernel was launched"
    torch.cuda.synchronize()
    assert int(buf.double().abs().sum()) == 0, "a refused call wrote its output"
