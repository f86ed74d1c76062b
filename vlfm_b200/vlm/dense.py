"""Thin torch-tensor wrappers over the dense C-ABI entry points (csrc/gemm_wgmma.cu ...)."""
from __future__ import annotations

from typing import Optional

import torch

from .. import _lib


def gemm_f16(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], epilogue: int,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(a[M,K] @ w[N,K]^T + bias).  For epilogue 2 ``out`` is the fp32
    residual stream updated in place."""
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and a.stride(1) == 1 and w.stride(1) == 1
    if out is None:
        assert epilogue != _lib.EPI_BIAS_RESID_F32
        out = torch.empty((M, N), dtype=torch.float32 if epilogue == _lib.EPI_BIAS_F32 else torch.float16, device=a.device)
    rc = lib.vlfm_gemm_f16(_lib.ptr(a), _lib.ptr(w), _lib.ptr(bias), _lib.ptr(out), M, N, K, a.stride(0), w.stride(0),
                           out.stride(0), epilogue, _lib.stream_ptr())
    _lib.check(rc, "vlfm_gemm_f16")
    return out


def attention_f16(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, heads: int, Nq: int, Nk: int, hd: int,
                  scale: float) -> torch.Tensor:
    """softmax(scale * q k^T) v per (batch, head); q [B*Nq, >=heads*hd], k/v [B*Nk, ...] fp16 (strided views allowed)."""
    lib = _lib.load()
    out = torch.empty((B * Nq, heads * hd), dtype=torch.float16, device=q.device)
    rc = lib.vlfm_attention_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, heads, Nq, Nk, hd, q.stride(0),
                                k.stride(0), v.stride(0), out.stride(0), scale, _lib.stream_ptr())
    _lib.check(rc, "vlfm_attention_f16")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, want16: bool = True, want32: bool = False):
    lib = _lib.load()
    rows, D = x.shape
    o16 = torch.empty((rows, D), dtype=torch.float16, device=x.device) if want16 else None
    o32 = torch.empty((rows, D), dtype=torch.float32, device=x.device) if want32 else None
    rc = lib.vlfm_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _lib.ptr(o16), _lib.ptr(o32), rows, D, x.stride(0),
                            D if want16 else 0, D if want32 else 0, eps, _lib.stream_ptr())
    _lib.check(rc, "vlfm_layernorm")
    return o16, o32
