"""GroundingDINO's Swin-T backbone on hand-written sm_90a kernels (through the C-ABI).

Reference: the image branch of ``groundingdino.util.inference.predict`` called at
vlfm/vlm/grounding_dino.py:61-67, preceded by to_tensor + ImageNet normalise (:52-54; no
resize -- the native 480x640 frame goes in).  GEMMs (patch embedding, QKV, projection, MLP,
patch-merging reduction) run on the wgmma GEMM; LayerNorms on the shared LayerNorm kernel;
window attention / patch merging / patch im2col are csrc/swin_ops.cu.

Weights use the HF ``SwinBackbone`` naming (the prefix inside a GroundingDINO checkpoint is
``model.backbone.conv_encoder.model.``).
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Sequence, Tuple

import torch

from .. import _lib

F16, F32 = torch.float16, torch.float32
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


class SwinBackboneEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], prefix: str = "", embed_dim: int = 96, depths: Sequence[int] = (2, 2, 6, 2),
                 heads: Sequence[int] = (3, 6, 12, 24), out_stages: Sequence[int] = (2, 3, 4), eps: float = 1e-5,
                 device="cuda") -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.dev = torch.device(device)
        self.depths, self.heads, self.out_stages, self.eps, self.C0 = tuple(depths), tuple(heads), tuple(out_stages), eps, embed_dim
        self._mean = (ctypes.c_float * 3)(*IMAGENET_MEAN)
        self._std = (ctypes.c_float * 3)(*IMAGENET_STD)
        g = lambda k: sd[prefix + k]
        h = lambda t: t.to(self.dev, F16).contiguous()
        f = lambda t: t.to(self.dev, F32).contiguous()
        self.pe_w = h(g("embeddings.patch_embeddings.projection.weight").reshape(embed_dim, 48))
        self.pe_b = f(g("embeddings.patch_embeddings.projection.bias"))
        self.pe_ln = (f(g("embeddings.norm.weight")), f(g("embeddings.norm.bias")))
        self.stages: List[Dict] = []
        for s, depth in enumerate(depths):
            blocks = []
            for i in range(depth):
                p = f"encoder.layers.{s}.blocks.{i}."
                a = p + "attention.self."
                blocks.append(dict(
                    ln1=(f(g(p + "layernorm_before.weight")), f(g(p + "layernorm_before.bias"))),
                    qkv_w=h(torch.cat([g(a + "query.weight"), g(a + "key.weight"), g(a + "value.weight")], 0)),
                    qkv_b=f(torch.cat([g(a + "query.bias"), g(a + "key.bias"), g(a + "value.bias")], 0)),
                    rel=f(g(a + "relative_position_bias_table")),
                    proj_w=h(g(p + "attention.output.dense.weight")), proj_b=f(g(p + "attention.output.dense.bias")),
                    ln2=(f(g(p + "layernorm_after.weight")), f(g(p + "layernorm_after.bias"))),
                    fc1_w=h(g(p + "intermediate.dense.weight")), fc1_b=f(g(p + "intermediate.dense.bias")),
                    fc2_w=h(g(p + "output.dense.weight")), fc2_b=f(g(p + "output.dense.bias")),
                    shift=0 if i % 2 == 0 else 3,
                ))
            st = dict(blocks=blocks)
            if s < len(depths) - 1:
                d = f"encoder.layers.{s}.downsample."
                st["merge_w"] = h(g(d + "reduction.weight"))
                st["merge_ln"] = (f(g(d + "norm.weight")), f(g(d + "norm.bias")))
            if (s + 1) in self.out_stages:
                st["out_ln"] = (f(g(f"hidden_states_norms.stage{s + 1}.weight")), f(g(f"hidden_states_norms.stage{s + 1}.bias")))
            self.stages.append(st)
        self._bufs: Dict[Tuple[int, int, int], Dict[str, torch.Tensor]] = {}

    # ---- primitives
    def _gemm(self, a, w, bias, epi, out):
        rc = self.lib.vlfm_gemm_f16(a.data_ptr(), w.data_ptr(), _lib.ptr(bias), out.data_ptr(), a.shape[0], w.shape[0], a.shape[1],
                                    a.stride(0), w.stride(0), out.stride(0), epi, _lib.stream_ptr())
        _lib.check(rc, "vlfm_gemm_f16")

    def _ln(self, x, wb, out16, out32):
        rows, D = x.shape
        rc = self.lib.vlfm_layernorm(x.data_ptr(), wb[0].data_ptr(), wb[1].data_ptr(), _lib.ptr(out16), _lib.ptr(out32), rows, D,
                                     x.stride(0), out16.stride(0) if out16 is not None else 0,
                                     out32.stride(0) if out32 is not None else 0, self.eps, _lib.stream_ptr())
        _lib.check(rc, "vlfm_layernorm")

    def _buffers(self, B: int, H: int, W: int) -> Dict[str, torch.Tensor]:
        key = (B, H, W)
        if key not in self._bufs:
            Hp, Wp = (H + 3) // 4, (W + 3) // 4
            n0 = B * Hp * Wp
            e = lambda *s, dt=F16: torch.empty(*s, dtype=dt, device=self.dev)
            C = self.C0
            self._bufs[key] = dict(col=e(n0, 48), x=e(n0, C, dt=F32), xn=e(n0, 4 * C), qkv=e(n0, 3 * C), ao=e(n0, C), h=e(n0, 4 * C),
                                   mg=e(n0 // 4 + B * (Hp + Wp) + B, 4 * C, dt=F32), x2=e(n0, C, dt=F32))
        return self._bufs[key]

    @torch.inference_mode()
    def forward_rows(self, images: torch.Tensor):
        """images [B,H,W,3] uint8 (device) -> [(rows [B*h*w, C] fp32 in NHWC order, h, w)] per out stage: what the neck's row GEMMs
        consume (vlm/gdino_forward.py) -- no NCHW permute / copy."""
        return self.forward(images, rows=True)

    @torch.inference_mode()
    def forward(self, images: torch.Tensor, rows: bool = False) -> List[torch.Tensor]:
        """images [B,H,W,3] uint8 (device) -> feature maps [B,C_s,H_s,W_s] fp32 for the configured out stages."""
        B, H, W, _ = images.shape
        assert images.dtype == torch.uint8 and images.is_contiguous()
        bufs = self._buffers(B, H, W)
        lib, st = self.lib, _lib.stream_ptr()
        with torch.cuda.device(self.dev):
            rc = lib.vlfm_swin_patch_im2col(images.data_ptr(), bufs["col"].data_ptr(), B, H, W, self._mean, self._std, st)
            _lib.check(rc, "vlfm_swin_patch_im2col")
            h, w, C = (H + 3) // 4, (W + 3) // 4, self.C0
            n = B * h * w
            flat = lambda t, rows, cols: t.view(-1)[: rows * cols].view(rows, cols)
            x = flat(bufs["x"], n, C)
            self._gemm(bufs["col"], self.pe_w, self.pe_b, _lib.EPI_BIAS_F32, x)
            self._ln(x, self.pe_ln, None, x)
            feats: List[torch.Tensor] = []
            cur, other = "x", "x2"
            for s, stage in enumerate(self.stages):
                if min(h, w) <= 7:
                    # HF's Swin (set_shift_and_window_size) drops the shift and shrinks the window when a stage's map is not larger
                    # than the 7x7 window; that variant is not built: refuse instead of silently computing something else
                    raise _lib.VlfmError(f"Swin backbone: stage {s + 1} feature map {h}x{w} is not larger than the 7x7 window "
                                         f"(image {H}x{W} too small; the minimum side is 225 px)")
                n = B * h * w
                x = flat(bufs[cur], n, C)
                xn, qkv, ao, hh = flat(bufs["xn"], n, C), flat(bufs["qkv"], n, 3 * C), flat(bufs["ao"], n, C), flat(bufs["h"], n, 4 * C)
                for blk in stage["blocks"]:
                    self._ln(x, blk["ln1"], xn, None)
                    self._gemm(xn, blk["qkv_w"], blk["qkv_b"], _lib.EPI_BIAS_F16, qkv)
                    rc = lib.vlfm_swin_window_attention(qkv.data_ptr(), blk["qkv_b"].data_ptr(), blk["rel"].data_ptr(), ao.data_ptr(),
                                                        B, h, w, C, self.heads[s], blk["shift"], st)
                    _lib.check(rc, "vlfm_swin_window_attention")
                    self._gemm(ao, blk["proj_w"], blk["proj_b"], _lib.EPI_BIAS_RESID_F32, x)
                    self._ln(x, blk["ln2"], xn, None)
                    self._gemm(xn, blk["fc1_w"], blk["fc1_b"], _lib.EPI_BIAS_GELU_F16, hh)
                    self._gemm(hh, blk["fc2_w"], blk["fc2_b"], _lib.EPI_BIAS_RESID_F32, x)
                if "out_ln" in stage:
                    o = torch.empty(n, C, dtype=F32, device=self.dev)
                    self._ln(x, stage["out_ln"], None, o)
                    feats.append((o, h, w) if rows else o.view(B, h, w, C).permute(0, 3, 1, 2).contiguous())
                if "merge_w" in stage:
                    h2, w2 = (h + 1) // 2, (w + 1) // 2
                    n2 = B * h2 * w2
                    mg = flat(bufs["mg"], n2, 4 * C)
                    rc = lib.vlfm_swin_patch_merge(x.data_ptr(), mg.data_ptr(), B, h, w, C, st)
                    _lib.check(rc, "vlfm_swin_patch_merge")
                    mn = flat(bufs["xn"], n2, 4 * C)
                    self._ln(mg, stage["merge_ln"], mn, None)
                    nx = flat(bufs[other], n2, 2 * C)
                    self._gemm(mn, stage["merge_w"], None, _lib.EPI_BIAS_F32, nx)
                    cur, other = other, cur
                    h, w, C = h2, w2, 2 * C
        return feats
