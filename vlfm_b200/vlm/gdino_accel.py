"""Hand-written kernels under the GroundingDINO feature enhancer / decoder (SURVEY.md 8f rank 1).

``accelerate`` swaps the layers of HF's ``GroundingDinoForObjectDetection`` in place for classes that run on the library's
own kernels; ``gdino_forward.GdinoForward`` then sequences them:

* ``GroundingDinoDeformableLayer`` -> ``TcDeformableLayer``, ``GroundingDinoFusionLayer`` -> ``TcFusionLayer``,
  ``GroundingDinoDecoderLayer`` -> ``TcDecoderLayer``: GEMMs, fused multi-scale deformable sampling (``vlfm_msda_fused``,
  replacing groundingdino's ms_deform_attn_cuda.cu) and bi-attention (``vlfm_biattn_f16``), csrc/gdino_ops.cu;
* every other ``nn.Linear`` whose shape the GEMM takes -> ``TcLinear``: fp16 operands on the wgmma GEMM (csrc/gemm_wgmma.cu),
  fp32 accumulate, bias fused, fp32 out (the reference runs these in fp32 SIMT GEMMs: groundingdino ... nn.Linear).
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib
from .dense import cast_addpos_f16, cast_f16, gemm_f16, layernorm

F16 = torch.float16


def _f16(x: torch.Tensor) -> torch.Tensor:
    return torch.empty(x.shape, dtype=F16, device=x.device)


class TcLinear(torch.nn.Module):
    def __init__(self, lin: torch.nn.Linear):
        super().__init__()
        self.in_features, self.out_features = lin.in_features, lin.out_features
        self.weight, self.bias = lin.weight, lin.bias                      # state_dict keys stay those of nn.Linear
        self.register_buffer("w16", lin.weight.detach().to(torch.float16).contiguous(), persistent=False)
        self.register_buffer("b32", None if lin.bias is None else lin.bias.detach().float().contiguous(), persistent=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shp = x.shape
        x2 = x.reshape(-1, self.in_features)
        if x2.dtype != torch.float16:
            x2 = cast_f16(x2.float().contiguous())
        elif not x2.is_contiguous():
            x2 = x2.contiguous()
        out = torch.empty((x2.shape[0], self.out_features), dtype=torch.float32, device=x.device)
        if x2.shape[0]:                 # the GEMM refuses M = 0
            gemm_f16(x2, self.w16, self.b32, _lib.EPI_BIAS_F32, out)
        return out.view(*shp[:-1], self.out_features)


def _w16(lin: torch.nn.Linear):
    return lin.weight.detach().to(torch.float16).contiguous(), lin.bias.detach().float().contiguous()


def _shapes(spatial_shapes_list):
    flat = [int(v) for hw in spatial_shapes_list for v in hw]
    return (ctypes.c_int32 * len(flat))(*flat)


class TcDeformAttn(torch.nn.Module):
    """``GroundingDinoMultiscaleDeformableAttention`` (groundingdino MSDeformAttn.forward) on the library's kernels:
    cast(+pos) -> value GEMM (fp16 out) -> offsets|logits GEMM (one launch, fp32 out) -> fused softmax + sampling
    locations + bilinear gather (``vlfm_msda_fused``) -> output GEMM.  Padding masks are not supported on this path
    (the detector is always fed unpadded, equally sized frames: grounding_dino.py:52-54 passes one native-size image)."""

    def __init__(self, m):
        super().__init__()
        self.heads, self.levels, self.points, self.d = m.n_heads, m.n_levels, m.n_points, m.d_model
        assert self.d // self.heads == 32 and self.levels * self.points <= 16
        wv, bv = _w16(m.value_proj); wo, bo = _w16(m.output_proj)
        ws, bs = _w16(m.sampling_offsets); wa, ba = _w16(m.attention_weights)
        for n, t in (("wv", wv), ("bv", bv), ("wo", wo), ("bo", bo), ("wc", torch.cat([ws, wa]).contiguous()), ("bc", torch.cat([bs, ba]).contiguous())):
            self.register_buffer(n, t, persistent=False)
        self.logit_col = ws.shape[0]
        self.orig = [m]                                    # keeps the parameters reachable without registering them twice

    def sample(self, hidden: torch.Tensor, pos, enc, ref: torch.Tensor, shapes_list) -> torch.Tensor:
        """-> fp16 [B*Q, d] attention output before the output projection."""
        b, q, d = hidden.shape
        same = enc is None or enc is hidden
        x = hidden.contiguous()
        p = None if pos is None else pos.expand_as(x).contiguous()
        x = x.view(b * q, d)
        x16 = _f16(x) if same else None
        xp16 = cast_addpos_f16(x, p, x16)
        if not same:
            s = enc.shape[1]
            x16 = getattr(enc, "_vlfm_f16", None)      # the six decoder layers read the same encoder output
            if x16 is None:
                x16 = cast_f16(enc.contiguous()).view(b * s, d)
                enc._vlfm_f16 = x16
        else:
            s = q
        value16 = gemm_f16(x16, self.wv, self.bv, _lib.EPI_BIAS_F16)
        offlog = gemm_f16(xp16, self.wc, self.bc, _lib.EPI_BIAS_F32)
        ref = ref.float().contiguous()
        out16 = torch.empty((b * q, d), dtype=torch.float16, device=x.device)
        rc = _lib.load().vlfm_msda_fused(value16.data_ptr(), offlog.data_ptr(), offlog.stride(0), self.logit_col, ref.data_ptr(),
                                          ref.shape[-1], out16.data_ptr(), b, s, q, self.heads, self.levels, self.points,
                                          ctypes.cast(_shapes(shapes_list), ctypes.c_void_p), _lib.stream_ptr())
        _lib.check(rc, "vlfm_msda_fused")
        return out16

    def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None, encoder_attention_mask=None, position_embeddings=None,
                reference_points=None, spatial_shapes=None, spatial_shapes_list=None, level_start_index=None, output_attentions=False):
        b, q, d = hidden_states.shape
        out16 = self.sample(hidden_states, position_embeddings, encoder_hidden_states, reference_points, spatial_shapes_list)
        return gemm_f16(out16, self.wo, self.bo, _lib.EPI_BIAS_F32).view(b, q, d), None


class TcDeformableLayer(torch.nn.Module):
    """``GroundingDinoDeformableLayer.forward`` (deformable self-attention + FFN, post-LN) entirely on the library's
    kernels: residual adds fused into the GEMM epilogues (fp32 stream), ReLU fused into fc1, LayerNorms on
    ``vlfm_layernorm``."""

    def __init__(self, m):
        super().__init__()
        self.attn = TcDeformAttn(m.self_attn)
        w1, b1 = _w16(m.fc1); w2, b2 = _w16(m.fc2)
        for n, t in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2),
                     ("g1", m.self_attn_layer_norm.weight.detach().float().contiguous()), ("be1", m.self_attn_layer_norm.bias.detach().float().contiguous()),
                     ("g2", m.final_layer_norm.weight.detach().float().contiguous()), ("be2", m.final_layer_norm.bias.detach().float().contiguous())):
            self.register_buffer(n, t, persistent=False)
        self.eps1, self.eps2 = m.self_attn_layer_norm.eps, m.final_layer_norm.eps
        self.orig = [m]

    def forward(self, hidden_states, attention_mask=None, position_embeddings=None, reference_points=None, spatial_shapes=None,
                spatial_shapes_list=None, level_start_index=None, output_attentions=False):
        b, s, d = hidden_states.shape
        x = hidden_states.reshape(b * s, d).clone()                                   # fp32 residual stream
        out16 = self.attn.sample(hidden_states, position_embeddings, None, reference_points, spatial_shapes_list)
        gemm_f16(out16, self.attn.wo, self.attn.bo, _lib.EPI_BIAS_RESID_F32, out=x)   # x += out_proj(attn)
        x16, x32 = layernorm(x, self.g1, self.be1, self.eps1, True, True)
        h16 = gemm_f16(x16, self.w1, self.b1, _lib.EPI_BIAS_RELU_F16)
        gemm_f16(h16, self.w2, self.b2, _lib.EPI_BIAS_RESID_F32, out=x32)             # x32 += fc2(relu(fc1(x)))
        _, y = layernorm(x32, self.g2, self.be2, self.eps2, out32=True)
        return y.view(b, s, d), None


def biattn_f16(q, k, v, b: int, heads: int, nq: int, nk: int, scale: float, key_chunk: int = 0, head_dim: int = 256) -> torch.Tensor:
    """softmax(scale q k^T) v per (batch, head), head_dim 256 or 32; q/k/v are fp16 2-D (strided column views allowed)."""
    if key_chunk == 0:
        key_chunk = 128 if head_dim == 256 else 1024
    out = torch.empty((b * nq, heads * head_dim), dtype=torch.float16, device=q.device)
    part = None
    if nk > key_chunk:
        chunks = (nk + key_chunk - 1) // key_chunk
        rpb = 64 if head_dim == 256 else 128
        part = torch.empty(b * heads * chunks * ((nq + rpb - 1) // rpb * rpb) * (head_dim + 2), dtype=torch.float32, device=q.device)
    rc = _lib.load().vlfm_biattn_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), _lib.ptr(part), 0 if part is None else part.numel(),
                                    b, heads, head_dim, nq, nk, q.stride(0), k.stride(0), v.stride(0), out.stride(0), key_chunk, float(scale),
                                    _lib.stream_ptr())
    _lib.check(rc, "vlfm_biattn_f16")
    return out


class TcFusionLayer(torch.nn.Module):
    """``GroundingDinoFusionLayer.forward`` (groundingdino BiAttentionBlock: pre-LN, bi-directional image<->text attention,
    layer-scaled residuals) on the library's kernels: ``vlfm_layernorm`` -> ONE GEMM per modality for (query|value) resp.
    (key|value) projections with fp16 out -> ``vlfm_biattn_f16`` in both directions -> output GEMMs with the layer scale
    folded into the weights and the residual add in the epilogue.  The reference's global-max subtraction and +-50000 clamp
    are softmax-invariant for finite logits and are not reproduced.  No padding masks (see TcDeformAttn); captions longer
    than 128 tokens fall back to the original module."""

    MAX_TEXT = 128

    def __init__(self, m):
        super().__init__()
        at = m.attn
        assert at.head_dim == 256
        self.heads, self.scale = at.num_heads, at.scale
        wq, bq = _w16(at.vision_proj); wvv, bvv = _w16(at.values_vision_proj)
        wk, bk = _w16(at.text_proj); wvt, bvt = _w16(at.values_text_proj)
        gv, gt = m.vision_param.detach().float(), m.text_param.detach().float()
        wov = (at.out_vision_proj.weight.detach().float() * gv[:, None]).to(torch.float16).contiguous()
        wot = (at.out_text_proj.weight.detach().float() * gt[:, None]).to(torch.float16).contiguous()
        bufs = {"wv": torch.cat([wq, wvv]).contiguous(), "bv": torch.cat([bq, bvv]).contiguous(),
                "wt": torch.cat([wk, wvt]).contiguous(), "bt": torch.cat([bk, bvt]).contiguous(),
                "wov": wov, "bov": (at.out_vision_proj.bias.detach().float() * gv).contiguous(),
                "wot": wot, "bot": (at.out_text_proj.bias.detach().float() * gt).contiguous(),
                "gv": m.layer_norm_vision.weight.detach().float().contiguous(), "bev": m.layer_norm_vision.bias.detach().float().contiguous(),
                "gt": m.layer_norm_text.weight.detach().float().contiguous(), "bet": m.layer_norm_text.bias.detach().float().contiguous()}
        for n, t in bufs.items():
            self.register_buffer(n, t, persistent=False)
        self.epsv, self.epst = m.layer_norm_vision.eps, m.layer_norm_text.eps
        self.e = self.heads * 256
        self.orig = [m]

    def forward(self, vision_features, text_features, attention_mask_vision=None, attention_mask_text=None):
        b, nv, d = vision_features.shape
        t = text_features.shape[1]
        if t > self.MAX_TEXT:
            return self.orig[0](vision_features, text_features, attention_mask_vision, attention_mask_text)
        v16, v32 = layernorm(vision_features.reshape(b * nv, d).contiguous(), self.gv, self.bev, self.epsv, True, True)
        t16, t32 = layernorm(text_features.reshape(b * t, d).contiguous(), self.gt, self.bet, self.epst, True, True)
        qv = gemm_f16(v16, self.wv, self.bv, _lib.EPI_BIAS_F16)            # [b*nv, 2e]: image queries | image values
        kt = gemm_f16(t16, self.wt, self.bt, _lib.EPI_BIAS_F16)            # [b*t, 2e]: text keys | text values
        e = self.e
        ov = biattn_f16(qv[:, :e], kt[:, :e], kt[:, e:], b, self.heads, nv, t, self.scale)      # image <- text
        ot = biattn_f16(kt[:, :e], qv[:, :e], qv[:, e:], b, self.heads, t, nv, self.scale)      # text <- image
        gemm_f16(ov, self.wov, self.bov, _lib.EPI_BIAS_RESID_F32, out=v32)  # LN(x) + gamma * out_proj(attn)
        gemm_f16(ot, self.wot, self.bot, _lib.EPI_BIAS_RESID_F32, out=t32)
        return (v32.view(b, nv, d), None), (t32.view(b, t, d), None)


class TcDecoderLayer(torch.nn.Module):
    """``GroundingDinoDecoderLayer.forward`` (self-attention over the 900 queries, text cross-attention, deformable image
    cross-attention, FFN; post-LN) on the library's kernels.  Attention masks are not supported (``self_attn_mask`` is None
    at inference and captions are never padded on this path); neither are attention outputs."""

    def __init__(self, m):
        super().__init__()
        sa, ta = m.self_attn, m.encoder_attn_text
        assert sa.attention_head_size == 32 and ta.attention_head_size == 32
        self.heads = sa.num_attention_heads
        self.deform = TcDeformAttn(m.encoder_attn)
        wq, bq = _w16(sa.query); wk, bk = _w16(sa.key); wv, bv = _w16(sa.value); wo, bo = _w16(sa.out_proj)
        tq, tbq = _w16(ta.query); tk, tbk = _w16(ta.key); tv, tbv = _w16(ta.value); to, tbo = _w16(ta.out_proj)
        w1, b1 = _w16(m.fc1); w2, b2 = _w16(m.fc2)
        bufs = {"wqk": torch.cat([wq, wk]).contiguous(), "bqk": torch.cat([bq, bk]).contiguous(), "wv": wv, "bv": bv, "wo": wo, "bo": bo,
                "xq": tq, "xbq": tbq, "xkv": torch.cat([tk, tv]).contiguous(), "xbkv": torch.cat([tbk, tbv]).contiguous(), "xo": to, "xbo": tbo,
                "w1": w1, "b1": b1, "w2": w2, "b2": b2}
        self.eps = []
        for i, ln in enumerate((m.self_attn_layer_norm, m.encoder_attn_text_layer_norm, m.encoder_attn_layer_norm, m.final_layer_norm)):
            bufs[f"g{i}"] = ln.weight.detach().float().contiguous(); bufs[f"be{i}"] = ln.bias.detach().float().contiguous()
            self.eps.append(ln.eps)
        for n, t in bufs.items():
            self.register_buffer(n, t, persistent=False)

    def forward(self, hidden_states, position_embeddings=None, reference_points=None, spatial_shapes=None, spatial_shapes_list=None,
                level_start_index=None, vision_encoder_hidden_states=None, vision_encoder_attention_mask=None,
                text_encoder_hidden_states=None, text_encoder_attention_mask=None, self_attn_mask=None, output_attentions=False):
        assert self_attn_mask is None and not output_attentions
        b, nq, d = hidden_states.shape
        t = text_encoder_hidden_states.shape[1]
        scale = 32 ** -0.5
        x = hidden_states.reshape(b * nq, d).clone()                              # fp32 residual stream
        pos = None if position_embeddings is None else position_embeddings.expand(b, nq, d).reshape(b * nq, d).contiguous()
        # ---- self-attention: q = k = x + pos, v = x
        x16 = _f16(x)
        xp16 = cast_addpos_f16(x, pos, x16)
        qk = gemm_f16(xp16, self.wqk, self.bqk, _lib.EPI_BIAS_F16)
        v = gemm_f16(x16, self.wv, self.bv, _lib.EPI_BIAS_F16)
        a = biattn_f16(qk[:, :d], qk[:, d:], v, b, self.heads, nq, nq, scale, head_dim=32)
        gemm_f16(a, self.wo, self.bo, _lib.EPI_BIAS_RESID_F32, out=x)
        _, x = layernorm(x, self.g0, self.be0, self.eps[0], out32=True)
        # ---- text cross-attention: q = x + pos, k = v = text
        xp16 = cast_addpos_f16(x, pos)
        q = gemm_f16(xp16, self.xq, self.xbq, _lib.EPI_BIAS_F16)
        txt = text_encoder_hidden_states
        t16 = getattr(txt, "_vlfm_f16", None)
        if t16 is None:
            t16 = cast_f16(txt.reshape(b * t, d).float().contiguous())
            txt._vlfm_f16 = t16
        kv = gemm_f16(t16, self.xkv, self.xbkv, _lib.EPI_BIAS_F16)
        a = biattn_f16(q, kv[:, :d], kv[:, d:], b, self.heads, nq, t, scale, head_dim=32)
        gemm_f16(a, self.xo, self.xbo, _lib.EPI_BIAS_RESID_F32, out=x)
        _, x = layernorm(x, self.g1, self.be1, self.eps[1], out32=True)
        # ---- deformable cross-attention over the image features
        out16 = self.deform.sample(x.view(b, nq, d), position_embeddings, vision_encoder_hidden_states, reference_points, spatial_shapes_list)
        gemm_f16(out16, self.deform.wo, self.deform.bo, _lib.EPI_BIAS_RESID_F32, out=x)
        x16, x = layernorm(x, self.g2, self.be2, self.eps[2], True, True)
        # ---- FFN
        h16 = gemm_f16(x16, self.w1, self.b1, _lib.EPI_BIAS_RELU_F16)
        gemm_f16(h16, self.w2, self.b2, _lib.EPI_BIAS_RESID_F32, out=x)
        _, y = layernorm(x, self.g3, self.be3, self.eps[3], out32=True)
        return (y.view(b, nq, d),)


def accelerate(model: torch.nn.Module, min_out: int = 16) -> dict:
    """Swap the layers and linears in place (model already on the GPU).  Returns counts for the log / tests."""
    from transformers.models.grounding_dino.modeling_grounding_dino import (GroundingDinoDecoderLayer, GroundingDinoDeformableLayer,
                                                                           GroundingDinoFusionLayer)

    n_lin = n_skip = n_layer = n_fuse = n_dec = 0
    assert getattr(model.config, "activation_function", "relu") == "relu"
    for parent in list(model.modules()):
        for name, child in list(parent.named_children()):
            if isinstance(child, GroundingDinoDeformableLayer):
                setattr(parent, name, TcDeformableLayer(child)); n_layer += 1
            elif isinstance(child, GroundingDinoFusionLayer) and child.attn.head_dim == 256:
                setattr(parent, name, TcFusionLayer(child)); n_fuse += 1
            elif isinstance(child, GroundingDinoDecoderLayer) and child.self_attn.attention_head_size == 32:
                setattr(parent, name, TcDecoderLayer(child)); n_dec += 1
    for parent in list(model.modules()):
        for name, child in list(parent.named_children()):
            if isinstance(child, torch.nn.Linear):
                if child.in_features % 8 == 0 and child.in_features >= 16 and child.out_features >= min_out and child.out_features % 4 == 0:
                    setattr(parent, name, TcLinear(child)); n_lin += 1
                else:
                    n_skip += 1
    return {"linear": n_lin, "linear_kept": n_skip, "deformable_layers": n_layer, "fusion_layers": n_fuse, "decoder_layers": n_dec}
