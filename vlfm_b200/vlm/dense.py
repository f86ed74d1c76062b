"""Torch-tensor wrappers over the dense C-ABI entry points (csrc/gemm_wgmma.cu, vit_ops.cu, gdino_ops.cu, im2col.cu): the only
Python code that calls them.  Every engine (BLIP-2, Swin, GroundingDINO, MobileSAM, PointNav, YOLOv7) goes through these.

Each wrapper writes into the outputs the caller gives and allocates a required output only when it is not given, so a CUDA-graph
captured forward can pass preallocated buffers.  An optional output of the ABI (a NULL pointer there) is left out by passing
None.  ``rows`` runs a launch on the first ``rows`` rows of its operands instead of ``a.shape[0]``.  No checks beyond the
C-ABI's own: these sit on host-bound launch sequences (the MobileSAM decoder issues ~60 of them per call).

Operands are fp16 with unit column stride; row strides are passed through, so row slices and column views of wider buffers
are fine.  Residual streams, LayerNorm inputs and fp32 outputs are fp32.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _lib

F16, F32 = torch.float16, torch.float32
Tensor = torch.Tensor


def gemm_f16(a: Tensor, w: Tensor, bias: Optional[Tensor], epilogue: int, out: Optional[Tensor] = None,
             rows: Optional[int] = None) -> Tensor:
    """out = epilogue(a[M,K] @ w[N,K]^T + bias).  For EPI_BIAS_RESID_F32 ``out`` is the fp32 residual stream updated in place.
    ``epilogue`` may carry the EPI_CLUSTER_SPLIT flag (the batch-1 ViT plan is allowed)."""
    M, K = a.shape
    if rows is not None:
        M = rows
    if out is None:
        epi = epilogue & ~_lib.EPI_CLUSTER_SPLIT
        assert epi != _lib.EPI_BIAS_RESID_F32, "the residual epilogue updates a caller-given stream"
        out = torch.empty((M, w.shape[0]), dtype=F32 if epi == _lib.EPI_BIAS_F32 else F16, device=a.device)
    rc = _lib.load().vlfm_gemm_f16(a.data_ptr(), w.data_ptr(), _lib.ptr(bias), out.data_ptr(), M, w.shape[0], K, a.stride(0),
                                   w.stride(0), out.stride(0), epilogue, _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16")
    return out


def gemm_f16_resid_ln(a: Tensor, w: Tensor, bias: Optional[Tensor], x: Tensor, gamma: Tensor, beta: Tensor, eps: float,
                      out16: Optional[Tensor] = None, out32: Optional[Tensor] = None, partials: Optional[Tensor] = None,
                      rows: Optional[int] = None) -> None:
    """x += a @ w^T + bias ; LayerNorm(x) -> out16 (fp16) and / or out32 (fp32; may be x itself).  ``partials`` is the fp32
    split-K workspace: without one the GEMM does not split K.  Bitwise reproducible either way."""
    M, K = a.shape
    if rows is not None:
        M = rows
    ws, ws_bytes = (None, 0) if partials is None else (partials.data_ptr(), partials.numel() * 4)
    rc = _lib.load().vlfm_gemm_f16_resid_ln(a.data_ptr(), w.data_ptr(), _lib.ptr(bias), x.data_ptr(), M, w.shape[0], K, a.stride(0),
                                            w.stride(0), x.stride(0), gamma.data_ptr(), beta.data_ptr(),
                                            _lib.ptr(out16), 0 if out16 is None else out16.stride(0),
                                            _lib.ptr(out32), 0 if out32 is None else out32.stride(0), eps, ws, ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16_resid_ln")


def gemm_f16x2(a: Tensor, a_lo: Tensor, w: Tensor, w_lo: Tensor, bias: Optional[Tensor], epilogue: int, out: Tensor,
               out_lo: Optional[Tensor] = None) -> None:
    """x2 operands (hi, lo) on both sides -> fp32 ``out`` (EPI_BIAS_F32 / EPI_BIAS_RESID_F32) or GELU as x2 operands
    ``out`` / ``out_lo`` (EPI_BIAS_GELU_F16X2)."""
    M, K = a.shape
    rc = _lib.load().vlfm_gemm_f16x2(a.data_ptr(), a_lo.data_ptr(), w.data_ptr(), w_lo.data_ptr(), _lib.ptr(bias), out.data_ptr(),
                                     _lib.ptr(out_lo), M, w.shape[0], K, a.stride(0), w.stride(0), out.stride(0), epilogue,
                                     _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16x2")


def gemm_f16x2_resid_ln(a: Tensor, a_lo: Tensor, w: Tensor, w_lo: Tensor, bias: Optional[Tensor], x: Tensor, gamma: Tensor,
                        beta: Tensor, eps: float, out_hi: Tensor, out_lo: Tensor, out32: Optional[Tensor] = None,
                        partials: Optional[Tensor] = None) -> None:
    """x += (x2 product) + bias ; LayerNorm(x) -> x2 operands out_hi / out_lo (same stride) and optionally fp32 out32."""
    M, K = a.shape
    ws, ws_bytes = (None, 0) if partials is None else (partials.data_ptr(), partials.numel() * 4)
    rc = _lib.load().vlfm_gemm_f16x2_resid_ln(a.data_ptr(), a_lo.data_ptr(), w.data_ptr(), w_lo.data_ptr(), _lib.ptr(bias), x.data_ptr(),
                                              M, w.shape[0], K, a.stride(0), w.stride(0), x.stride(0), gamma.data_ptr(), beta.data_ptr(),
                                              out_hi.data_ptr(), out_lo.data_ptr(), out_hi.stride(0),
                                              _lib.ptr(out32), 0 if out32 is None else out32.stride(0), eps, ws, ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16x2_resid_ln")


def layernorm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, out16=None, out32=None):
    """LayerNorm over the rows of x -> out16 (fp16) and / or out32 (fp32; may be x itself).  Each output is a tensor to write,
    True for a new one, or None / False for none.  Returns (out16, out32)."""
    rows, D = x.shape
    if out16 is True:
        out16 = torch.empty((rows, D), dtype=F16, device=x.device)
    elif out16 is False:
        out16 = None
    if out32 is True:
        out32 = torch.empty((rows, D), dtype=F32, device=x.device)
    elif out32 is False:
        out32 = None
    rc = _lib.load().vlfm_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _lib.ptr(out16), _lib.ptr(out32), rows, D,
                                    x.stride(0), 0 if out16 is None else out16.stride(0), 0 if out32 is None else out32.stride(0), eps,
                                    _lib.stream_ptr())
    _lib.check(rc, "vlfm_layernorm")
    return out16, out32


def layernorm_x2(x: Tensor, gamma: Tensor, beta: Tensor, eps: float, out_hi: Tensor, out_lo: Tensor,
                 out32: Optional[Tensor] = None) -> None:
    """LayerNorm over the rows of x -> x2 operands out_hi / out_lo (same stride) and optionally fp32 out32."""
    rows, D = x.shape
    rc = _lib.load().vlfm_layernorm_x2(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out_hi.data_ptr(), out_lo.data_ptr(),
                                       _lib.ptr(out32), rows, D, x.stride(0), out_hi.stride(0), 0 if out32 is None else out32.stride(0), eps,
                                       _lib.stream_ptr())
    _lib.check(rc, "vlfm_layernorm_x2")


def attention_f16(q: Tensor, k: Tensor, v: Tensor, B: int, heads: int, Nq: int, Nk: int, hd: int, scale: float,
                  out: Optional[Tensor] = None) -> Tensor:
    """softmax(scale * q k^T) v per (batch, head); q [B*Nq, >=heads*hd], k/v [B*Nk, ...] fp16 (strided views allowed)."""
    if out is None:
        out = torch.empty((B * Nq, heads * hd), dtype=F16, device=q.device)
    rc = _lib.load().vlfm_attention_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, heads, Nq, Nk, hd, q.stride(0),
                                        k.stride(0), v.stride(0), out.stride(0), scale, _lib.stream_ptr())
    _lib.check(rc, "vlfm_attention_f16")
    return out


def attention_f32(q: Tensor, k: Tensor, v: Tensor, B: int, heads: int, Nq: int, Nk: int, hd: int, scale: float, out_hi: Tensor,
                  out_lo: Tensor) -> None:
    """attention_f16 in float32 on fp32 q / k / v, with the output as x2 operands out_hi / out_lo (same stride)."""
    rc = _lib.load().vlfm_attention_f32(q.data_ptr(), k.data_ptr(), v.data_ptr(), out_hi.data_ptr(), out_lo.data_ptr(), B, heads, Nq,
                                        Nk, hd, q.stride(0), k.stride(0), v.stride(0), out_hi.stride(0), scale, _lib.stream_ptr())
    _lib.check(rc, "vlfm_attention_f32")


def split_x2(x: Tensor, out_lo: Tensor) -> None:
    """out_lo = the lo half of x's x2 operands (x fp32 contiguous; the hi half is fp16(x), which the caller already has)."""
    rc = _lib.load().vlfm_split_x2(x.data_ptr(), None, out_lo.data_ptr(), x.numel(), _lib.stream_ptr())
    _lib.check(rc, "vlfm_split_x2")


def cast_f16(x: Tensor, out: Optional[Tensor] = None) -> Tensor:
    """fp32 contiguous -> fp16."""
    if out is None:
        out = torch.empty(x.shape, dtype=F16, device=x.device)
    rc = _lib.load().vlfm_cast_f32_f16(x.data_ptr(), out.data_ptr(), x.numel(), _lib.stream_ptr())
    _lib.check(rc, "vlfm_cast_f32_f16")
    return out


def cast_addpos_f16(x: Tensor, pos: Optional[Tensor], out: Optional[Tensor] = None, out_pos: Optional[Tensor] = None) -> Tensor:
    """fp32 contiguous x (and pos of the same shape, or None for zero) -> out_pos = fp16(x + pos), returned, and, when ``out``
    is given, out = fp16(x)."""
    if out_pos is None:
        out_pos = torch.empty(x.shape, dtype=F16, device=x.device)
    rc = _lib.load().vlfm_cast_addpos_f16(x.data_ptr(), _lib.ptr(pos), _lib.ptr(out), out_pos.data_ptr(), x.numel(), _lib.stream_ptr())
    _lib.check(rc, "vlfm_cast_addpos_f16")
    return out_pos


def im2col(x: Tensor, B: int, H: int, W: int, k: int, stride: int, out: Optional[Tensor] = None) -> Tensor:
    """Rows of a k x k conv (pad k // 2) over x [B*H*W, C] NHWC rows -> out [B*Ho*Wo, ldk] (contiguous), the A operand of a GEMM
    with the weight ``conv_rows(w)``.  A new ``out`` has ldk = k*k*C rounded up to a multiple of 8."""
    C = x.shape[1]
    if out is None:
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        out = torch.empty((B * Ho * Wo, (k * k * C + 7) // 8 * 8), dtype=F16, device=x.device)
    rc = _lib.load().vlfm_im2col_f16(x.data_ptr(), x.stride(0), out.data_ptr(), B, H, W, C, k, stride, out.shape[1], _lib.stream_ptr())
    _lib.check(rc, "vlfm_im2col_f16")
    return out


def conv_rows(w: Tensor) -> Tensor:
    """Conv weight [O, C, k, k] -> GEMM rows [O, ldk] in w's dtype, columns (ky, kx, c) zero-padded to ldk = k*k*C rounded up to a
    multiple of 8: the column order of ``im2col``."""
    O, C, k, _ = w.shape
    r = w.permute(0, 2, 3, 1).reshape(O, k * k * C)
    return torch.nn.functional.pad(r, (0, (k * k * C + 7) // 8 * 8 - k * k * C)).contiguous()
