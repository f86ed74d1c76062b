"""Kernel interface of ``GdinoForward`` (vlm/gdino_forward.py) on the C-ABI library: every method is one or two launches of
csrc/gdino_head.cu / gemm_wgmma.cu / vit_ops.cu kernels over torch-owned buffers.  No torch arithmetic here."""
from __future__ import annotations

from typing import Optional

import torch

from .. import _lib
from .dense import cast_f16, gemm_f16, im2col, layernorm as _layernorm

F16, F32 = torch.float16, torch.float32


class LibOps:
    def __init__(self) -> None:
        self.lib = _lib.load()

    # ---- operands
    def weight(self, w: torch.Tensor) -> torch.Tensor:
        w = w.to("cuda", F16).contiguous()
        assert w.shape[1] % 8 == 0, "GEMM K must be a multiple of 8"
        return w

    def to_operand(self, x: torch.Tensor) -> torch.Tensor:
        return x if x.dtype == F16 else cast_f16(x)

    def linear_operand(self, a16: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
        return gemm_f16(a16, w16, bias, _lib.EPI_BIAS_F32)

    def linear(self, x: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor], relu: bool = False) -> torch.Tensor:
        """fp32 or fp16 rows in; fp16 out after a ReLU (the next layer's operand), fp32 otherwise."""
        return gemm_f16(self.to_operand(x.contiguous()), w16, bias, _lib.EPI_BIAS_RELU_F16 if relu else _lib.EPI_BIAS_F32)

    def layernorm(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
        return _layernorm(x, g, b, eps, out32=True)[1]

    # ---- neck
    def im2col3x3s2(self, rows: torch.Tensor, B: int, h: int, w: int) -> torch.Tensor:
        """Rows of the fourth level's 3x3 stride-2 conv; fp32 rows are cast to the fp16 operand first."""
        return im2col(self.to_operand(rows), B, h, w, 3, 2)

    def groupnorm_rows(self, y: torch.Tensor, B: int, HW: int, C: int, groups: int, g: torch.Tensor, b: torch.Tensor, eps: float,
                       out: torch.Tensor, row_off: int, S: int) -> None:
        _lib.check(self.lib.vlfm_groupnorm_rows(y.data_ptr(), B, HW, C, groups, g.data_ptr(), b.data_ptr(), float(eps), out.data_ptr(), row_off, S,
                                                _lib.stream_ptr()), "vlfm_groupnorm_rows")

    # ---- two-stage selection
    def mask_rows(self, x: torch.Tensor, valid_u8: torch.Tensor) -> torch.Tensor:
        out = torch.empty(x.shape, dtype=F16, device=x.device)
        _lib.check(self.lib.vlfm_mask_rows_f16(x.data_ptr(), valid_u8.data_ptr(), out.data_ptr(), x.shape[0], x.shape[1], _lib.stream_ptr()),
                   "vlfm_mask_rows_f16")
        return out

    def proposal_scores(self, q: torch.Tensor, text: torch.Tensor, B: int, S: int, T: int) -> torch.Tensor:
        out = torch.empty((B, S), dtype=F32, device=q.device)
        _lib.check(self.lib.vlfm_proposal_scores(q.data_ptr(), text.data_ptr(), B, S, T, q.shape[1], out.data_ptr(), _lib.stream_ptr()),
                   "vlfm_proposal_scores")
        return out

    def topk_rows(self, scores: torch.Tensor, k: int) -> torch.Tensor:
        B, S = scores.shape
        idx = torch.empty((B, k), dtype=torch.int64, device=scores.device)
        _lib.check(self.lib.vlfm_topk_rows(scores.data_ptr(), B, S, k, idx.data_ptr(), _lib.stream_ptr()), "vlfm_topk_rows")
        return idx

    def decoder_query_pos(self, ref: torch.Tensor, valid_ratios: torch.Tensor, dim_t: torch.Tensor):
        """ref [B, nq, 4], valid_ratios [B, L, 2], dim_t [P] -> (reference_points_input [B, nq, L, 4] fp32, sine embedding operand [B*nq, 4P])"""
        B, nq, _ = ref.shape
        L, P = valid_ratios.shape[1], dim_t.shape[0]
        ref_in = torch.empty((B, nq, L, 4), dtype=F32, device=ref.device)
        emb = torch.empty((B * nq, 4 * P), dtype=F16, device=ref.device)
        _lib.check(self.lib.vlfm_decoder_query_pos(ref.contiguous().data_ptr(), valid_ratios.contiguous().data_ptr(), dim_t.data_ptr(), B, nq, L, P,
                                                   ref_in.data_ptr(), emb.data_ptr(), _lib.stream_ptr()), "vlfm_decoder_query_pos")
        return ref_in, emb

    def gather_rows(self, src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
        B, S, C = src.shape
        K = idx.shape[1]
        out = torch.empty((B, K, C), dtype=F32, device=src.device)
        _lib.check(self.lib.vlfm_gather_rows(src.data_ptr(), idx.data_ptr(), B, S, K, C, out.data_ptr(), _lib.stream_ptr()), "vlfm_gather_rows")
        return out

    # ---- heads
    def box_finish(self, delta: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
        out = torch.empty_like(delta)
        _lib.check(self.lib.vlfm_box_finish(delta.data_ptr(), ref.data_ptr(), out.data_ptr(), delta.numel(), _lib.stream_ptr()), "vlfm_box_finish")
        return out

    def contrastive_sigmoid(self, hs: torch.Tensor, text: torch.Tensor, L: int) -> torch.Tensor:
        B, Q, D = hs.shape
        T = text.shape[1]
        out = torch.empty((B, Q, L), dtype=F32, device=hs.device)
        _lib.check(self.lib.vlfm_contrastive_sigmoid(hs.data_ptr(), text.data_ptr(), B, Q, T, D, L, out.data_ptr(), _lib.stream_ptr()),
                   "vlfm_contrastive_sigmoid")
        return out
