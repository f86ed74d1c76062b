"""BLIP-2 ITC forward on hand-written sm_90a kernels (through the C-ABI).

Replaces what ``self.model({"image": img, "text_input": txt}, match_head="itc")`` does
inside ``BLIP2ITM.cosine`` (vlfm/vlm/blip2itm.py:52) together with the preprocessing at
:48-49.  Python here only sequences C-ABI launches over preallocated buffers; the whole
per-batch forward is captured once in a CUDA graph and replayed.

Numerics: fp16 GEMM/attention operands (lavis runs the ViT under fp16 autocast too),
fp32 accumulation (registers), fp32 residual stream, fp32 LayerNorm / softmax statistics.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from .. import _lib
from . import dense
from .blip2_config import Blip2Dims
from .preprocess import CLIP_MEAN, CLIP_STD, bicubic_tables

F16, F32 = torch.float16, torch.float32


def partials_floats(dims: Blip2Dims, max_batch: int) -> int:
    """Size (floats) of the split-K workspace of the residual GEMM + LayerNorm calls: eight slabs of the residual stream for at
    most 1024 rows (every stream-K plan, below one wave of tiles, and the uniform splits of the smaller batches), and at least
    three for the whole batch: above one wave the GEMM plan splits the ViT's fc2 (K = 6144) two or three ways at some batches
    (at B = 32: two), which is faster there than unsplit.  A split that does not fit runs unsplit (vlfm_gemm_f16_resid_ln never
    reduces with atomics), so this size trades memory (139 MB at max_batch 32) for speed, not correctness."""
    rows = max_batch * dims.tokens
    return max(8 * min(rows, 1024), 3 * rows) * max(dims.v_hidden, dims.q_hidden)


class Blip2ITCEngine:
    def __init__(self, dims: Blip2Dims, state_dict: Dict[str, torch.Tensor], device="cuda", max_batch: int = 1,
                 use_graph: bool = True) -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.d = dims
        self.dev = torch.device(device)
        self.max_batch = max_batch
        self.use_graph = use_graph and os.environ.get("VLFM_NO_GRAPH", "") != "1"
        self._graphs: Dict[Tuple[int, int, int], Tuple[torch.cuda.CUDAGraph, torch.Tensor]] = {}
        self._tables: Dict[Tuple[int, int], Tuple[torch.Tensor, ...]] = {}
        self._mean = (ctypes.c_float * 3)(*CLIP_MEAN)
        self._std = (ctypes.c_float * 3)(*CLIP_STD)
        # the Q-Former runs in float32-grade arithmetic (x2 operands on the fp16 tensor path, fp32 attention): the reference runs it
        # in fp32 (only the ViT is half precision in lavis) and fp16 operands there alone cost ~3e-5 on the cosine
        self._load(state_dict)
        self._alloc(max_batch)
        self.text_feat = torch.zeros(dims.proj, dtype=F32, device=self.dev)
        # residual GEMM + LayerNorm as one C-ABI call with a deterministic split-K reduction (partial sums stored side by side, added
        # to the residual stream in split order by the LayerNorm launch): the cosine is bitwise reproducible run to run.  False runs
        # them as a plain residual GEMM (self._gemm / self._gemm_x2) and a LayerNorm launch: bench.py's GEMM replay records them so.
        self.fuse_ln = True
        self._partials = torch.empty(partials_floats(dims, max_batch), dtype=F32, device=self.dev)
        self._fold_layer0()
        self._many_out: Dict[int, torch.Tensor] = {}   # forward_many / head outputs [max_batch, P], one per P
        # bumped by every forward / forward_many / encode_text: q_proj holds the image features of the forward that set the
        # current value, so a caller that recorded it can score that forward's images against new prompts with head() alone
        self.generation = 0

    # ------------------------------------------------------------------ weights ----
    def _load(self, sd: Dict[str, torch.Tensor]) -> None:
        d, dev = self.d, self.dev

        def h(t):  # fp16 GEMM operand
            return t.to(dev, F16).contiguous()

        def f(t):
            return t.to(dev, F32).contiguous()

        def lo(t):  # x2 residual of an fp32 weight: (w - fp16(w)) * 2048 as fp16
            t = t.to(dev, F32)
            return ((t - t.to(F16).to(F32)) * 2048.0).to(F16).contiguous()

        D = d.v_hidden
        pw = sd["vision_model.embeddings.patch_embedding.weight"].reshape(D, d.patch_k)
        pwp = torch.zeros(D, d.patch_k_padded)
        pwp[:, : d.patch_k] = pw
        self.patch_w, self.patch_b = h(pwp), f(sd["vision_model.embeddings.patch_embedding.bias"])
        self.cls = f(sd["vision_model.embeddings.class_embedding"].reshape(D))
        self.pos = f(sd["vision_model.embeddings.position_embedding"].reshape(d.tokens, D))
        self.vit: List[Dict[str, torch.Tensor]] = []
        for i in range(d.v_layers):
            p = f"vision_model.encoder.layers.{i}."
            self.vit.append(dict(
                ln1_w=f(sd[p + "layer_norm1.weight"]), ln1_b=f(sd[p + "layer_norm1.bias"]),
                qkv_w=h(sd[p + "self_attn.qkv.weight"]), qkv_b=f(sd[p + "self_attn.qkv.bias"]),
                proj_w=h(sd[p + "self_attn.projection.weight"]), proj_b=f(sd[p + "self_attn.projection.bias"]),
                ln2_w=f(sd[p + "layer_norm2.weight"]), ln2_b=f(sd[p + "layer_norm2.bias"]),
                fc1_w=h(sd[p + "mlp.fc1.weight"]), fc1_b=f(sd[p + "mlp.fc1.bias"]),
                fc2_w=h(sd[p + "mlp.fc2.weight"]), fc2_b=f(sd[p + "mlp.fc2.bias"]),
            ))
        self.post_w, self.post_b = f(sd["vision_model.post_layernorm.weight"]), f(sd["vision_model.post_layernorm.bias"])
        H = d.q_hidden
        self.q_ln_w, self.q_ln_b = f(sd["qformer.layernorm.weight"]), f(sd["qformer.layernorm.bias"])
        self.word_emb, self.pos_emb = f(sd["embeddings.word_embeddings.weight"]), f(sd["embeddings.position_embeddings.weight"])
        self.qf: List[Dict[str, torch.Tensor]] = []
        kv_w, kv_b = [], []
        for i in range(d.q_layers):
            p = f"qformer.encoder.layer.{i}."
            a = p + "attention."
            L = dict(
                qkv_w=h(torch.cat([sd[a + "attention.query.weight"], sd[a + "attention.key.weight"], sd[a + "attention.value.weight"]], 0)),
                qkv_b=f(torch.cat([sd[a + "attention.query.bias"], sd[a + "attention.key.bias"], sd[a + "attention.value.bias"]], 0)),
                so_w=h(sd[a + "output.dense.weight"]), so_b=f(sd[a + "output.dense.bias"]),
                sln_w=f(sd[a + "output.LayerNorm.weight"]), sln_b=f(sd[a + "output.LayerNorm.bias"]),
                iq_w=h(sd[p + "intermediate_query.dense.weight"]), iq_b=f(sd[p + "intermediate_query.dense.bias"]),
                oq_w=h(sd[p + "output_query.dense.weight"]), oq_b=f(sd[p + "output_query.dense.bias"]),
                oqln_w=f(sd[p + "output_query.LayerNorm.weight"]), oqln_b=f(sd[p + "output_query.LayerNorm.bias"]),
                it_w=h(sd[p + "intermediate.dense.weight"]), it_b=f(sd[p + "intermediate.dense.bias"]),
                ot_w=h(sd[p + "output.dense.weight"]), ot_b=f(sd[p + "output.dense.bias"]),
                otln_w=f(sd[p + "output.LayerNorm.weight"]), otln_b=f(sd[p + "output.LayerNorm.bias"]),
                cross=-1,
            )
            if i % d.cross_freq == 0:
                c = p + "crossattention."
                L["cross"] = len(kv_w)
                L["cq_w"], L["cq_b"] = h(sd[c + "attention.query.weight"]), f(sd[c + "attention.query.bias"])
                L["co_w"], L["co_b"] = h(sd[c + "output.dense.weight"]), f(sd[c + "output.dense.bias"])
                L["cln_w"], L["cln_b"] = f(sd[c + "output.LayerNorm.weight"]), f(sd[c + "output.LayerNorm.bias"])
                kv_w.append(torch.cat([sd[c + "attention.key.weight"], sd[c + "attention.value.weight"]], 0))
                kv_b.append(torch.cat([sd[c + "attention.key.bias"], sd[c + "attention.value.bias"]], 0))
            srcs = {"qkv_w": torch.cat([sd[a + "attention.query.weight"], sd[a + "attention.key.weight"], sd[a + "attention.value.weight"]], 0),
                    "so_w": sd[a + "output.dense.weight"], "iq_w": sd[p + "intermediate_query.dense.weight"],
                    "oq_w": sd[p + "output_query.dense.weight"], "it_w": sd[p + "intermediate.dense.weight"], "ot_w": sd[p + "output.dense.weight"]}
            if L["cross"] >= 0:
                srcs["cq_w"], srcs["co_w"] = sd[c + "attention.query.weight"], sd[c + "output.dense.weight"]
            for k_, w_ in srcs.items():
                L[k_ + "l"] = lo(w_)
            self.qf.append(L)
        self.ncross = len(kv_w)
        self.kv_w, self.kv_b = h(torch.cat(kv_w, 0)), f(torch.cat(kv_b, 0))  # one GEMM feeds every cross layer
        self.vp_w, self.vp_b = h(sd["vision_projection.weight"]), f(sd["vision_projection.bias"])
        self.tp_w, self.tp_b = h(sd["text_projection.weight"]), f(sd["text_projection.bias"])
        self.kv_wl, self.vp_wl, self.tp_wl = lo(torch.cat(kv_w, 0)), lo(sd["vision_projection.weight"]), lo(sd["text_projection.weight"])
        self.query_tokens = f(sd["query_tokens"].reshape(d.queries, H))

    # ------------------------------------------------------------------ buffers ----
    def _alloc(self, B: int) -> None:
        d, dev = self.d, self.dev
        T, D, Fv, Q, H, I = d.tokens, d.v_hidden, d.v_inter, d.queries, d.q_hidden, d.q_inter
        e = lambda *s, dt=F16: torch.empty(*s, dtype=dt, device=dev)
        self.b_col = torch.zeros(B * (T - 1), d.patch_k_padded, dtype=F16, device=dev)  # zero K padding stays zero
        self.b_patch = e(B * (T - 1), D, dt=F32)
        self.b_x = e(B * T, D, dt=F32)
        self.b_xn = e(B * T, D)
        self.b_qkv = e(B * T, 3 * D)
        self.b_ao = e(B * T, D)
        self.b_h = e(B * T, Fv)
        self.b_img = e(B * T, D)
        self.b_img32 = e(B * T, D, dt=F32)
        self.b_img_lo = e(B * T, D)
        self.b_kv32 = e(B * T, self.ncross * 2 * H, dt=F32)
        # the Q-Former's activations: x2 operand pairs (hi, lo) and fp32 q / k / v
        self.q_h32 = e(B * Q, H, dt=F32)
        self.q_h16 = e(B * Q, H)
        self.q_h_lo = e(B * Q, H)
        self.q_qkv32 = e(B * Q, 3 * H, dt=F32)
        self.q_q32 = e(B * Q, H, dt=F32)
        self.q_ao = e(B * Q, H)
        self.q_ao_lo = e(B * Q, H)
        self.q_f = e(B * Q, I)
        self.q_f_lo = e(B * Q, I)
        self.q_proj = e(B * Q, d.proj, dt=F32)
        self.out = torch.zeros(B, dtype=F32, device=dev)

    # ---------------------------------------------------------------- primitives ----
    # _gemm / _gemm_x2 stay methods: bench.py's GEMM replay swaps them for recording wrappers (with fuse_ln off, every GEMM of the
    # forward goes through them)
    def _gemm(self, a, w, bias, epi, out):
        dense.gemm_f16(a, w, bias, epi, out)

    def _gemm_x2(self, a, al, w, wl, bias, epi, out, out_lo=None):
        dense.gemm_f16x2(a, al, w, wl, bias, epi, out, out_lo)

    def _gemm_resid_ln(self, a, w, bias, x, g, b, out16, out32, eps):
        """x += a @ w^T + bias ; LayerNorm(x) -> out16 / out32 (GEMM launch + reduce/LayerNorm launch, bitwise reproducible)."""
        if not self.fuse_ln:
            self._gemm(a, w, bias, _lib.EPI_BIAS_RESID_F32, x)
            dense.layernorm(x, g, b, eps, out16, out32)
            return
        dense.gemm_f16_resid_ln(a, w, bias, x, g, b, eps, out16, out32, partials=self._partials)

    def _gemm_x2_resid_ln(self, a, al, w, wl, bias, x, g, b, out_hi, out_lo, out32, eps):
        if not self.fuse_ln:
            self._gemm_x2(a, al, w, wl, bias, _lib.EPI_BIAS_RESID_F32, x)
            dense.layernorm_x2(x, g, b, eps, out_hi, out_lo, out32)
            return
        dense.gemm_f16x2_resid_ln(a, al, w, wl, bias, x, g, b, eps, out_hi, out_lo, out32, partials=self._partials)

    def _resize_tables(self, h: int, w: int):
        key = (h, w)
        if key not in self._tables:
            hb, hk, hks = bicubic_tables(w, self.d.image)
            vb, vk, vks = bicubic_tables(h, self.d.image)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
            self._tables[key] = (t(hb), t(hk), hks, t(vb), t(vk), vks)
        return self._tables[key]

    # ------------------------------------------------------------------ forward ----
    def _forward_impl(self, img: torch.Tensor, mid: torch.Tensor) -> None:
        """img [B,H,W,3] uint8 (device) -> self.out[:B] cosines.  Pure launch sequence."""
        d = self.d
        B, Hh, Ww, _ = img.shape
        T, D, Q, H = d.tokens, d.v_hidden, d.queries, d.q_hidden
        n, nq = B * T, B * Q
        hb, hk, hks, vb, vk, vks = self._resize_tables(Hh, Ww)
        rc = self.lib.vlfm_preprocess_im2col(img.data_ptr(), mid.data_ptr(), self.b_col.data_ptr(), B, Hh, Ww, d.image, d.image,
                                             d.patch, d.patch_k_padded, hb.data_ptr(), hk.data_ptr(), hks, vb.data_ptr(),
                                             vk.data_ptr(), vks, self._mean, self._std, _lib.stream_ptr())
        _lib.check(rc, "vlfm_preprocess_im2col")
        self._gemm(self.b_col[: B * (T - 1)], self.patch_w, self.patch_b, _lib.EPI_BIAS_F32, self.b_patch[: B * (T - 1)])
        rc = self.lib.vlfm_assemble_tokens(self.b_patch.data_ptr(), self.cls.data_ptr(), self.pos.data_ptr(), self.b_x.data_ptr(),
                                           B, T, D, _lib.stream_ptr())
        _lib.check(rc, "vlfm_assemble_tokens")
        x, xn, qkv, ao, hb_ = self.b_x[:n], self.b_xn[:n], self.b_qkv[:n], self.b_ao[:n], self.b_h[:n]
        hd = D // d.v_heads
        img16, img32 = self.b_img[:n], self.b_img32[:n]
        dense.layernorm(x, self.vit[0]["ln1_w"], self.vit[0]["ln1_b"], d.v_eps, xn)
        for i, L in enumerate(self.vit):
            self._gemm(xn, L["qkv_w"], L["qkv_b"], _lib.EPI_BIAS_F16, qkv)
            dense.attention_f16(qkv[:, 0:D], qkv[:, D : 2 * D], qkv[:, 2 * D : 3 * D], B, d.v_heads, T, T, hd, hd**-0.5, ao)
            self._gemm_resid_ln(ao, L["proj_w"], L["proj_b"], x, L["ln2_w"], L["ln2_b"], xn, None, d.v_eps)
            self._gemm(xn, L["fc1_w"], L["fc1_b"], _lib.EPI_BIAS_GELU_F16, hb_)
            if i + 1 < len(self.vit):   # the next block's pre-norm rides on this block's residual GEMM
                nx = self.vit[i + 1]
                self._gemm_resid_ln(hb_, L["fc2_w"], L["fc2_b"], x, nx["ln1_w"], nx["ln1_b"], xn, None, d.v_eps)
            else:                       # ... and the post-LayerNorm on the last one
                self._gemm_resid_ln(hb_, L["fc2_w"], L["fc2_b"], x, self.post_w, self.post_b, img16, img32, d.v_eps)
        # image embeds as x2 operands: hi is the fp16 LayerNorm output itself, lo its residual against the fp32 one
        img_lo = self.b_img_lo[:n]
        dense.split_x2(img32, img_lo)
        kv = self.b_kv32[:n]
        self._gemm_x2(img16, img_lo, self.kv_w, self.kv_wl, self.kv_b, _lib.EPI_BIAS_F32, kv)
        # layer 0's self-attention block is folded (_fold_layer0): only the residual stream needs its start value, the x2 operands
        # are rewritten by layer 0's cross block
        h32, hhi, hlo = self.q_h32[:nq], self.q_h16[:nq], self.q_h_lo[:nq]
        h32.copy_(self.f0_32x[:nq])
        self._qformer_layers(h32, hhi, hlo, B, Q, kv, T, text=False)
        self._gemm_x2(hhi, hlo, self.vp_w, self.vp_wl, self.vp_b, _lib.EPI_BIAS_F32, self.q_proj[:nq])
        rc = self.lib.vlfm_itc_head(self.q_proj.data_ptr(), self.text_feat.data_ptr(), self.out.data_ptr(), B, Q, d.proj,
                                    _lib.stream_ptr())
        _lib.check(rc, "vlfm_itc_head")

    def _fold_layer0(self) -> None:
        """Layer 0's self-attention block sees only LayerNorm(query_tokens) (modeling: qformer.layernorm on query_embeds): it (and
        the query projection of layer 0's cross-attention that follows it) is the same for every image -- computed once here with
        the step's own kernels."""
        d = self.d
        Q, H = d.queries, d.q_hidden
        hd = H // d.q_heads
        L = self.qf[0]                  # a cross-attention layer: i % cross_freq == 0
        with torch.cuda.device(self.dev):
            h32 = torch.empty(Q, H, dtype=F32, device=self.dev)
            hhi, hlo = torch.empty(Q, H, dtype=F16, device=self.dev), torch.empty(Q, H, dtype=F16, device=self.dev)
            dense.layernorm_x2(self.query_tokens, self.q_ln_w, self.q_ln_b, d.q_eps, hhi, hlo, h32)
            qkv, ahi, alo = self.q_qkv32[:Q], self.q_ao[:Q], self.q_ao_lo[:Q]
            self._gemm_x2(hhi, hlo, L["qkv_w"], L["qkv_wl"], L["qkv_b"], _lib.EPI_BIAS_F32, qkv)
            dense.attention_f32(qkv[:, 0:H], qkv[:, H : 2 * H], qkv[:, 2 * H : 3 * H], 1, d.q_heads, Q, Q, hd, 1.0 / math.sqrt(hd), ahi, alo)
            self._gemm_x2_resid_ln(ahi, alo, L["so_w"], L["so_wl"], L["so_b"], h32, L["sln_w"], L["sln_b"], hhi, hlo, h32, d.q_eps)
            f0_q = torch.empty(Q, H, dtype=F32, device=self.dev)
            self._gemm_x2(hhi, hlo, L["cq_w"], L["cq_wl"], L["cq_b"], _lib.EPI_BIAS_F32, f0_q)
            torch.cuda.synchronize()
        self.f0_32x = h32.repeat(self.max_batch, 1)
        self.f0_qx = f0_q.repeat(self.max_batch, 1)

    def _qformer_layers(self, h32, hhi, hlo, B, S, kv, T, text: bool) -> None:
        """The Q-Former layers (modeling: Blip2QFormerLayer; float32 in the reference) with x2 operands everywhere and float32
        attention.  The image path (text=False) starts after layer 0's self-attention block, which _fold_layer0 computed: h32 holds
        its output; the text path (query_length=0: no cross-attention) runs every layer."""
        d = self.d
        H = d.q_hidden
        hd = H // d.q_heads
        n = B * S
        qkv, qq, ahi, alo, fhi, flo = self.q_qkv32[:n], self.q_q32[:n], self.q_ao[:n], self.q_ao_lo[:n], self.q_f[:n], self.q_f_lo[:n]
        sc = 1.0 / math.sqrt(hd)
        for li, L in enumerate(self.qf):
            folded = not text and li == 0
            if not folded:
                self._gemm_x2(hhi, hlo, L["qkv_w"], L["qkv_wl"], L["qkv_b"], _lib.EPI_BIAS_F32, qkv)
                dense.attention_f32(qkv[:, 0:H], qkv[:, H : 2 * H], qkv[:, 2 * H : 3 * H], B, d.q_heads, S, S, hd, sc, ahi, alo)
                self._gemm_x2_resid_ln(ahi, alo, L["so_w"], L["so_wl"], L["so_b"], h32, L["sln_w"], L["sln_b"], hhi, hlo, h32, d.q_eps)
            if not text and L["cross"] >= 0:
                j = L["cross"]
                if folded:
                    cq = self.f0_qx[:n]                  # constant: never written
                else:
                    cq = qq
                    self._gemm_x2(hhi, hlo, L["cq_w"], L["cq_wl"], L["cq_b"], _lib.EPI_BIAS_F32, qq)
                dense.attention_f32(cq, kv[:, j * 2 * H : j * 2 * H + H], kv[:, j * 2 * H + H : (j + 1) * 2 * H], B, d.q_heads, S, T, hd, sc,
                                    ahi, alo)
                self._gemm_x2_resid_ln(ahi, alo, L["co_w"], L["co_wl"], L["co_b"], h32, L["cln_w"], L["cln_b"], hhi, hlo, h32, d.q_eps)
            k1, k2, kl = ("it", "ot", "otln") if text else ("iq", "oq", "oqln")
            self._gemm_x2(hhi, hlo, L[k1 + "_w"], L[k1 + "_wl"], L[k1 + "_b"], _lib.EPI_BIAS_GELU_F16X2, fhi, flo)
            self._gemm_x2_resid_ln(fhi, flo, L[k2 + "_w"], L[k2 + "_wl"], L[k2 + "_b"], h32, L[kl + "_w"], L[kl + "_b"], hhi, hlo, h32, d.q_eps)

    # ------------------------------------------------------------------- public ----
    @torch.inference_mode()
    def encode_text(self, token_ids: Sequence[int]) -> torch.Tensor:
        """Q-Former text branch (query_length=0) -> normalised text feature [proj]; run once per prompt."""
        d = self.d
        self.generation += 1
        ids = torch.tensor(list(token_ids), dtype=torch.long, device=self.dev)
        S = len(ids)
        assert 1 <= S <= self.d.queries * self.max_batch and S <= 272
        emb = (self.word_emb[ids] + self.pos_emb[:S]).contiguous()
        h32, hhi, hlo = self.q_h32[:S], self.q_h16[:S], self.q_h_lo[:S]
        with torch.cuda.device(self.dev):
            tp = torch.empty(1, d.proj, dtype=F32, device=self.dev)
            dense.layernorm_x2(emb, self.q_ln_w, self.q_ln_b, d.q_eps, hhi, hlo, h32)
            self._qformer_layers(h32, hhi, hlo, 1, S, None, 0, text=True)
            self._gemm_x2(hhi[:1], hlo[:1], self.tp_w, self.tp_wl, self.tp_b, _lib.EPI_BIAS_F32, tp)
        return torch.nn.functional.normalize(tp[0], dim=-1)

    def set_text(self, feat: torch.Tensor) -> None:
        self.text_feat.copy_(feat)

    @torch.inference_mode()
    def forward(self, images: torch.Tensor) -> torch.Tensor:
        """images [B,H,W,3] uint8 on the device -> cosine [B] (device, fp32) against the
        text feature last given to set_text()."""
        B, Hh, Ww, _ = images.shape
        assert B <= self.max_batch and images.dtype == torch.uint8 and images.is_contiguous()
        key = (B, Hh, Ww)
        self.generation += 1
        with torch.cuda.device(self.dev):
            if not self.use_graph:
                mid = torch.empty(B, Hh, self.d.image, 3, dtype=torch.uint8, device=self.dev)
                self._forward_impl(images, mid)
                return self.out[:B]
            if key not in self._graphs:
                static_in = torch.empty_like(images)
                mid = torch.empty(B, Hh, self.d.image, 3, dtype=torch.uint8, device=self.dev)
                static_in.copy_(images)
                self._forward_impl(static_in, mid)  # warm-up: function attributes, table upload
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._forward_impl(static_in, mid)
                self._graphs[key] = (g, static_in, mid)
            g, static_in, _ = self._graphs[key]
            static_in.copy_(images, non_blocking=True)
            g.replay()
        return self.out[:B]

    @torch.inference_mode()
    def forward_many(self, images: torch.Tensor, text_feats: torch.Tensor) -> torch.Tensor:
        """images [B,H,W,3] uint8 on the device, text_feats [P, proj] fp32 normalised (encode_text rows) -> cosines [B, P]
        (device, fp32): one image forward and one head launch for all P prompts.  Column p is bitwise equal to forward()
        after set_text(text_feats[p]).  The result is a view of a buffer kept per P, rewritten by the next call."""
        self.forward(images)
        return self.head(text_feats, images.shape[0])

    @torch.inference_mode()
    def head(self, text_feats: torch.Tensor, B: int) -> torch.Tensor:
        """Scores the image features the last forward left in q_proj (its first B images) against text_feats [P, proj]
        -> [B, P] (device, fp32, same buffer as forward_many's).  Runs no forward."""
        P = text_feats.shape[0]
        assert 1 <= B <= self.max_batch and text_feats.shape == (P, self.d.proj) and text_feats.dtype == F32
        assert text_feats.is_contiguous() and text_feats.is_cuda
        out = self._many_out.get(P)
        if out is None:
            out = self._many_out[P] = torch.empty(self.max_batch, P, dtype=F32, device=self.dev)
        with torch.cuda.device(self.dev):
            rc = self.lib.vlfm_itc_head_multi(self.q_proj.data_ptr(), text_feats.data_ptr(), out.data_ptr(), B, P, self.d.queries,
                                              self.d.proj, P, _lib.stream_ptr())
        _lib.check(rc, "vlfm_itc_head_multi")
        return out[:B]
