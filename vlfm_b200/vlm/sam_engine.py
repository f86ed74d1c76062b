"""MobileSAM on hand-written sm_90a kernels (through the C-ABI): TinyViT-5M image encoder and the box-prompted mask decoder.

Reference: ``SamPredictor.set_image`` + ``predict(box=..., multimask_output=False)`` as called by MobileSAM.segment_bbox
(vlfm/vlm/sam.py:40-57).  GEMMs (every 1x1 conv, Linear, the im2col'd 3x3 convs and the transposed convs) run on the wgmma
GEMM, LayerNorms on the shared LayerNorm kernel, the 7-key attentions on ``vlfm_attention_f16``; the rest is csrc/sam_ops.cu.

Precision: fp16 GEMM / attention operands with fp32 accumulation; the encoder's residual stream, the decoder's tokens and
per-box image keys stay fp32.  Every launch is deterministic (no atomics, no K split that depends on the batch), and the
decoder runs its token GEMMs on row counts padded to whole 128-row tiles and its 7 x 7 self-attention in groups of at most 64
boxes, so a box's result does not depend on which other boxes share the launch.

The IoU head is not computed: ``segment_bbox`` discards it.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Tuple

import numpy as np
import torch

from .. import _lib
from .dense import attention_f16, gemm_f16, gemm_f16_resid_ln, im2col, layernorm
from .preprocess import bilinear_tables, pillow_vertical_first
from .sam_config import SamDims

F16, F32 = torch.float16, torch.float32
PIXEL_MEAN = (123.675, 116.28, 103.53)
PIXEL_STD = (58.395, 57.12, 57.375)
ROWS = 128          # GEMM row tile: token GEMMs run on whole tiles (no CUDA-core tail rows that would depend on M)
SELF_ATTN_GROUP = 64


def preshape(h: int, w: int, long_side: int) -> Tuple[int, int]:
    """ResizeLongestSide.get_preprocess_shape"""
    scale = long_side * 1.0 / max(h, w)
    return int(h * scale + 0.5), int(w * scale + 0.5)


class MobileSamEngine:
    def __init__(self, d: SamDims, w: Dict[str, torch.Tensor], device="cuda", max_batch: int = 1) -> None:
        if not torch.cuda.is_available():
            raise _lib.VlfmError("vlfm_b200 needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.d, self.dev, self.max_batch = d, torch.device(device), max_batch
        self.generation = 0          # encoder passes so far
        self.frames = 0              # frame slots holding an embedding (the last encode's batch)
        self._mean = (ctypes.c_float * 3)(*PIXEL_MEAN)
        self._std = (ctypes.c_float * 3)(*PIXEL_STD)
        h = lambda t: t.to(self.dev, F16).contiguous()
        f = lambda t: t.to(self.dev, F32).contiguous()
        self.w: Dict[str, torch.Tensor] = {}
        for k, v in w.items():
            # GEMM weights in fp16; biases, LayerNorm parameters, depthwise taps and tables in fp32
            part = k.split(".")[-2] if "." in k else ""
            gemm_w = k.endswith(".w") and part not in ("ln1", "ln2", "neck1", "neck3", "up_ln", "conv2", "local") and "norm" not in part
            self.w[k] = h(v) if gemm_w else f(v)
        # padded window tokens: LayerNorm(0) = beta, so their q/k/v row is W_qkv @ fp16(beta) + b_qkv (fp16 operands as the GEMM)
        for s in range(1, len(d.embed_dims)):
            for b in range(d.depths[s]):
                p = f"l{s}.b{b}."
                beta = w[p + "ln1.b"].half().double()
                row = w[p + "qkv.w"].half().double() @ beta + w[p + "qkv.b"].double()
                self.w[p + "pad_qkv"] = h(row.float())
        n = d.emb_side
        grid = torch.ones((n, n))
        y = (grid.cumsum(0) - 0.5) / n
        x = (grid.cumsum(1) - 0.5) / n
        c = (2 * torch.stack([x, y], -1) - 1) @ w["pe.gauss"].float()
        c = 2 * np.pi * c
        self.dense_pe = f(torch.cat([torch.sin(c), torch.cos(c)], -1).reshape(n * n, -1))
        self.emb = torch.empty(max_batch, n * n, d.prompt_dim, dtype=F32, device=self.dev)
        self._enc: Dict[int, Dict[str, torch.Tensor]] = {}
        self._pre: Dict[Tuple[int, int, int], Tuple] = {}
        self._dec: Dict[int, Dict[str, torch.Tensor]] = {}

    # ---------------------------------------------------------------------------------------------------- primitives
    def _wb(self, name):    # (weight, bias or None) of a GEMM; (gamma, beta) of a LayerNorm
        return self.w[name + ".w"], self.w.get(name + ".b")

    def _dw(self, x, x_f32, name, out, out_f32, B, H, W, C, stride, gelu):
        rc = self.lib.vlfm_sam_dwconv3x3(x.data_ptr(), x_f32, self.w[name + ".w"].data_ptr(), self.w[name + ".b"].data_ptr(), out.data_ptr(),
                                         out_f32, B, H, W, C, stride, gelu, _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_dwconv3x3")

    def _add_act(self, a, b, out32, out16, n, gelu):
        rc = self.lib.vlfm_sam_add_act(a.data_ptr(), _lib.ptr(b), _lib.ptr(out32), _lib.ptr(out16), n, gelu, _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_add_act")

    # ------------------------------------------------------------------------------------------------------- encoder
    def _tables(self, H: int, W: int):
        S = self.d.img_size
        key = (H, W, S)
        if key not in self._pre:
            newh, neww = preshape(H, W, S)
            hb, hk, hks = bilinear_tables(W, neww)
            vb, vk, vks = bilinear_tables(H, newh)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
            self._pre[key] = (newh, neww, t(hb), t(hk), hks, t(vb), t(vk), vks, int(pillow_vertical_first(H, W, newh)))
        return self._pre[key]

    def _enc_buffers(self, B: int) -> Dict[str, torch.Tensor]:
        if B not in self._enc:
            d, S = self.d, self.d.img_size
            E, r = d.embed_dims, d.resolutions
            n0 = B * r[0] * r[0]
            big = max(B * r[s] * r[s] * max(4 * E[s], 3 * E[s]) for s in range(len(E)))
            big = max(big, n0 * d.mbconv_ratio * E[0], B * (S // 2) ** 2 * 32, n0 * ((9 * d.stem_mid + 7) // 8 * 8),
                      B * r[-1] * r[-1] * 9 * d.prompt_dim)
            self._enc[B] = dict(
                img=torch.empty(B, S, S, 3, dtype=F16, device=self.dev),
                a=torch.empty(big, dtype=F16, device=self.dev), b=torch.empty(big, dtype=F16, device=self.dev),
                x32=torch.empty(n0 * E[0], dtype=F32, device=self.dev), y32=torch.empty(n0 * E[0], dtype=F32, device=self.dev),
                z32=torch.empty(n0 * E[0], dtype=F32, device=self.dev), x16=torch.empty(n0 * E[0], dtype=F16, device=self.dev))
        return self._enc[B]

    def preprocess(self, images: torch.Tensor) -> torch.Tensor:
        """[B,H,W,3] uint8 (device) -> [B,S,S,3] fp16: ResizeLongestSide, normalise, zero pad"""
        B, H, W, _ = images.shape
        newh, neww, hb, hk, hks, vb, vk, vks, v_first = self._tables(H, W)
        buf = self._enc_buffers(B)
        mid = torch.empty(B * (newh * W if v_first else H * neww) * 3, dtype=torch.uint8, device=self.dev)
        rc = self.lib.vlfm_sam_preprocess(images.data_ptr(), mid.data_ptr(), buf["img"].data_ptr(), B, H, W, newh, neww, self.d.img_size,
                                          hb.data_ptr(), hk.data_ptr(), hks, vb.data_ptr(), vk.data_ptr(), vks, v_first, self._mean,
                                          self._std, _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_preprocess")
        return buf["img"]

    @torch.inference_mode()
    def encode(self, images: torch.Tensor) -> torch.Tensor:
        """images [B,H,W,3] uint8 (device), B <= max_batch -> image embeddings in frame slots 0..B-1: [B, e*e, P] fp32."""
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3 or not images.is_cuda:
            raise ValueError("MobileSamEngine.encode: images must be a [B,H,W,3] uint8 CUDA tensor")
        B = images.shape[0]
        if not 1 <= B <= self.max_batch:
            raise ValueError(f"MobileSamEngine.encode: batch {B} outside 1..max_batch={self.max_batch}")
        images = images.contiguous()
        d, S = self.d, self.d.img_size
        E, r = d.embed_dims, d.resolutions
        bf = self._enc_buffers(B)
        x0 = self.preprocess(images)
        A, Bb = bf["a"], bf["b"]
        v = lambda t, n, c: t[: n * c].view(n, c)
        # stem: conv3x3 s2 (3 -> E0/2) + GELU, conv3x3 s2 (E0/2 -> E0)
        h1 = S // 2
        col = v(A, B * h1 * h1, self.w["stem0.w"].shape[1])
        im2col(x0.view(-1, 3), B, S, S, 3, 2, col)
        s0 = v(Bb, B * h1 * h1, d.stem_mid)
        gemm_f16(col, *self._wb("stem0"), _lib.EPI_BIAS_GELU_F16, s0)
        n0 = B * r[0] * r[0]
        col = v(A, n0, self.w["stem1.w"].shape[1])
        im2col(s0, B, h1, h1, 3, 2, col)
        x32, y32, z32, x16 = v(bf["x32"], n0, E[0]), v(bf["y32"], n0, E[0]), v(bf["z32"], n0, E[0]), v(bf["x16"], n0, E[0])
        gemm_f16(col, *self._wb("stem1"), _lib.EPI_BIAS_F32, x32)
        self._add_act(x32, None, None, x16, x32.numel(), 0)
        for s in range(len(E)):
            C, R = E[s], r[s]
            n = B * R * R
            x32, y32, z32, x16 = v(bf["x32"], n, C), v(bf["y32"], n, C), v(bf["z32"], n, C), v(bf["x16"], n, C)
            for b in range(d.depths[s]):
                p = f"l{s}.b{b}."
                if s == 0:      # MBConv: 1x1 + GELU, dw3x3 + GELU, 1x1, + shortcut, GELU
                    hid = C * d.mbconv_ratio
                    t1, t2 = v(A, n, hid), v(Bb, n, hid)
                    gemm_f16(x16, *self._wb(p + "conv1"), _lib.EPI_BIAS_GELU_F16, t1)
                    self._dw(t1, 0, p + "conv2", t2, 0, B, R, R, hid, 1, 1)
                    gemm_f16(t2, *self._wb(p + "conv3"), _lib.EPI_BIAS_F32, y32)
                    self._add_act(y32, x32, x32, x16, n * C, 1)
                    continue
                heads, ws = d.heads[s], d.windows[s]
                xn, qkv, ao, hh = v(A, n, C), v(Bb, n, 3 * C), v(A[n * C:], n, C), v(Bb, n, 4 * C)
                layernorm(x32, *self._wb(p + "ln1"), 1e-5, xn)
                gemm_f16(xn, *self._wb(p + "qkv"), _lib.EPI_BIAS_F16, qkv)
                rc = self.lib.vlfm_sam_window_attention(qkv.data_ptr(), self.w[p + "pad_qkv"].data_ptr(), self.w[p + "bias"].data_ptr(),
                                                        ao.data_ptr(), B, R, R, C, heads, ws, float((C // heads) ** -0.5), _lib.stream_ptr())
                _lib.check(rc, "vlfm_sam_window_attention")
                gemm_f16(ao, *self._wb(p + "proj"), _lib.EPI_BIAS_RESID_F32, x32)      # K = C <= 320: one K split, no atomics
                self._dw(x32, 1, p + "local", z32, 1, B, R, R, C, 1, 0)
                layernorm(z32, *self._wb(p + "ln2"), 1e-5, xn)
                gemm_f16(xn, *self._wb(p + "fc1"), _lib.EPI_BIAS_GELU_F16, hh)
                gemm_f16(hh, *self._wb(p + "fc2"), _lib.EPI_BIAS_F32, y32)
                self._add_act(y32, z32, x32, x16, n * C, 0)
            if s + 1 < len(E):   # PatchMerging: 1x1 + GELU, dw3x3 (stride) + GELU, 1x1
                Co, st = E[s + 1], d.merge_stride(s)
                Ro = r[s + 1]
                no = B * Ro * Ro
                t1, t2 = v(A, n, Co), v(Bb, no, Co)
                gemm_f16(x16, *self._wb(f"l{s}.down.conv1"), _lib.EPI_BIAS_GELU_F16, t1)
                self._dw(t1, 0, f"l{s}.down.conv2", t2, 0, B, R, R, Co, st, 1)
                x32n = v(bf["x32"], no, Co)
                gemm_f16(t2, *self._wb(f"l{s}.down.conv3"), _lib.EPI_BIAS_F32, x32n)
        # neck: 1x1 (no bias) -> LayerNorm2d -> 3x3 (no bias) -> LayerNorm2d
        R, P = r[-1], d.prompt_dim
        n = B * R * R
        x16 = v(bf["x16"], n, E[-1])
        t32 = v(bf["y32"], n, P)
        gemm_f16(x16, *self._wb("neck0"), _lib.EPI_BIAS_F32, t32)
        t16 = v(Bb, n, P)
        layernorm(t32, *self._wb("neck1"), 1e-6, t16)
        col = v(A, n, self.w["neck2.w"].shape[1])
        im2col(t16, B, R, R, 3, 1, col)
        gemm_f16(col, *self._wb("neck2"), _lib.EPI_BIAS_F32, t32)
        out = self.emb[:B].view(n, P)
        layernorm(t32, *self._wb("neck3"), 1e-6, out32=out)
        self.frames = B
        self.generation += 1
        return self.emb[:B]

    # ------------------------------------------------------------------------------------------------------- decoder
    def _dec_buffers(self, M: int) -> Dict[str, torch.Tensor]:
        cap = max(1, 1 << (M - 1).bit_length())
        for c, buf in self._dec.items():
            if c >= M:
                return buf
        d, P = self.d, self.d.prompt_dim
        HW = d.emb_side ** 2
        Mp = (cap + ROWS - 1) // ROWS * ROWS
        T = 7 * Mp + ROWS           # token rows: whole tiles for 7*Mp rows, plus room for the hypernetwork's strided view
        e = lambda n, c, dt=F16: torch.zeros(n, c, dtype=dt, device=self.dev)
        buf = dict(
            tok0=e(T, P, F32), qs=e(T, P, F32), q16=e(T, P), qp16=e(T, P), tq=e(T, P), tk=e(T, P), tv=e(T, P), to=e(T, P),
            h16=e(T, d.dec_mlp), keys=e(cap * HW, P, F32), k16=e(cap * HW, P), kp16=e(cap * HW, P), iq=e(cap * HW, P // 2),
            iv=e(cap * HW, P // 2), u1=e(cap * HW, P, F32), u1s=e(4 * cap * HW, P // 4, F32),
            u1n=e(4 * cap * HW, P // 4, F32), u16=e(4 * cap * HW, P // 4), u2=e(4 * cap * HW, P // 2, F32),
            hy1=e(Mp, P), hy2=e(Mp, P), hyper=e(Mp, P // 8, F32), low=e(cap, 16 * HW, F32),
            part=torch.empty(cap * d.dec_heads * ((HW + 255) // 256) * 8 * 18, dtype=F32, device=self.dev))
        buf["Mp"] = Mp
        self._dec = {cap: buf}
        return buf

    def _add_pe(self, x, pe, out16, outp16, rows, pe_rows):
        rc = self.lib.vlfm_sam_add_pe_f16(x.data_ptr(), _lib.ptr(pe), _lib.ptr(out16), _lib.ptr(outp16), rows, pe_rows, x.shape[1],
                                          _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_add_pe_f16")

    def _t2i(self, p, bf, M, HW, qsrc, ksrc, vsrc, T):
        """token -> image attention of block `p`: q from qsrc [T rows], k / v from ksrc / vsrc [M*HW rows] -> bf['to']"""
        d, P = self.d, self.d.prompt_dim
        tq, to = bf["tq"][:, : P // 2], bf["to"][:, : P // 2]
        tk, tv = bf["iq"][: M * HW], bf["iv"][: M * HW]
        gemm_f16(qsrc, *self._wb(p + ".q"), _lib.EPI_BIAS_F16, tq, rows=T)
        gemm_f16(ksrc, *self._wb(p + ".k"), _lib.EPI_BIAS_F16, tk)
        gemm_f16(vsrc, *self._wb(p + ".v"), _lib.EPI_BIAS_F16, tv)
        rc = self.lib.vlfm_sam_t2i_attention(tq.data_ptr(), tk.data_ptr(), tv.data_ptr(), to.data_ptr(), M, d.dec_heads, 7, HW, tq.stride(0),
                                             tk.stride(0), tv.stride(0), to.stride(0), float((P // 2 // d.dec_heads) ** -0.5),
                                             bf["part"].data_ptr(), bf["part"].numel(), _lib.stream_ptr())
        _lib.check(rc, "vlfm_sam_t2i_attention")
        return to

    @torch.inference_mode()
    def decode(self, boxes: torch.Tensor, frame_idx: torch.Tensor, hw: Tuple[int, int], out: torch.Tensor = None,
               low_out: bool = False):
        """boxes [M,4] float64 (device, frame pixels), frame_idx [M] int32 (device, slots of the last encode) -> masks
        [M,H,W] uint8 (device); with low_out=True also the low-res mask-0 logits [M, 4e, 4e] (a view, rewritten next call).
        A frame index outside the last encode's batch gives NaN logits and an all-False mask for that box."""
        d, P = self.d, self.d.prompt_dim
        M = boxes.shape[0]
        if M < 1:
            raise ValueError("MobileSamEngine.decode: at least one box is needed")
        H, W = hw
        S, e = d.img_size, d.emb_side
        HW = e * e
        newh, neww = preshape(H, W, S)
        bf = self._dec_buffers(M)
        Mp = bf["Mp"]
        T = 7 * Mp
        boxes = boxes.to(self.dev, torch.float64).contiguous()
        frame_idx = frame_idx.to(self.dev, torch.int32).contiguous()
        st = _lib.stream_ptr()
        tok0, qs, q16, qp16 = bf["tok0"], bf["qs"], bf["q16"], bf["qp16"]
        rc = self.lib.vlfm_sam_box_tokens(boxes.data_ptr(), M, H, W, newh, neww, S, self.w["pe.gauss"].data_ptr(), self.w["fixed"].data_ptr(),
                                          tok0.data_ptr(), P, st)
        _lib.check(rc, "vlfm_sam_box_tokens")
        qs[: 7 * M].copy_(tok0[: 7 * M])
        keys = bf["keys"][: M * HW]
        rc = self.lib.vlfm_sam_decoder_init(self.emb.data_ptr(), frame_idx.data_ptr(), self.w["no_mask"].data_ptr(), keys.data_ptr(), M,
                                            max(self.frames, 1), HW, P, st)
        _lib.check(rc, "vlfm_sam_decoder_init")
        k16, kp16 = bf["k16"][: M * HW], bf["kp16"][: M * HW]
        hd_s = P // d.dec_heads
        for i in range(d.dec_depth):
            p = f"dec{i}"
            # self-attention (layer 0: no position embedding, no residual)
            if i == 0:
                self._add_pe(qs, None, q16, None, T, 1)
                src_qk = q16
            else:
                self._add_pe(qs, tok0, q16, qp16, T, T)
                src_qk = qp16
            gemm_f16(src_qk, *self._wb(p + ".self.q"), _lib.EPI_BIAS_F16, bf["tq"], rows=T)
            gemm_f16(src_qk, *self._wb(p + ".self.k"), _lib.EPI_BIAS_F16, bf["tk"], rows=T)
            gemm_f16(q16, *self._wb(p + ".self.v"), _lib.EPI_BIAS_F16, bf["tv"], rows=T)
            for g0 in range(0, M, SELF_ATTN_GROUP):
                gb = min(SELF_ATTN_GROUP, M - g0)
                r0 = 7 * g0
                attention_f16(bf["tq"][r0:], bf["tk"][r0:], bf["tv"][r0:], gb, d.dec_heads, 7, 7, hd_s, float(hd_s ** -0.5), bf["to"][r0:])
            if i == 0:
                qs.zero_()
            gemm_f16_resid_ln(bf["to"], *self._wb(p + ".self.o"), qs, *self._wb(f"{p}.norm1"), 1e-5, out32=qs, rows=T)
            # token -> image
            self._add_pe(qs, tok0, None, qp16, T, T)
            self._add_pe(keys, self.dense_pe, k16, kp16, M * HW, HW)
            to = self._t2i(p + ".t2i", bf, M, HW, qp16, kp16, k16, T)
            gemm_f16_resid_ln(to, *self._wb(p + ".t2i.o"), qs, *self._wb(f"{p}.norm2"), 1e-5, q16, qs, rows=T)
            # MLP
            gemm_f16(q16, *self._wb(p + ".mlp1"), _lib.EPI_BIAS_RELU_F16, bf["h16"], rows=T)
            gemm_f16_resid_ln(bf["h16"], *self._wb(p + ".mlp2"), qs, *self._wb(f"{p}.norm3"), 1e-5, out32=qs, rows=T)
            # image -> token (keys unchanged since the token -> image step: kp16 still holds keys + pe)
            self._add_pe(qs, tok0, q16, qp16, T, T)
            iq, ik, iv, io = bf["iq"][: M * HW], bf["tk"][:, : P // 2], bf["tv"][:, : P // 2], bf["iv"][: M * HW]
            gemm_f16(kp16, *self._wb(p + ".i2t.q"), _lib.EPI_BIAS_F16, iq)
            gemm_f16(qp16, *self._wb(p + ".i2t.k"), _lib.EPI_BIAS_F16, ik, rows=T)
            gemm_f16(q16, *self._wb(p + ".i2t.v"), _lib.EPI_BIAS_F16, iv, rows=T)
            hd_c = P // 2 // d.dec_heads
            attention_f16(iq, ik, iv, M, d.dec_heads, HW, 7, hd_c, float(hd_c ** -0.5), io)
            gemm_f16_resid_ln(io, *self._wb(p + ".i2t.o"), keys, *self._wb(f"{p}.norm4"), 1e-5, out32=keys, rows=M * HW)
        # final token -> image attention
        self._add_pe(qs, tok0, None, qp16, T, T)
        self._add_pe(keys, self.dense_pe, k16, kp16, M * HW, HW)
        to = self._t2i("final", bf, M, HW, qp16, kp16, k16, T)
        gemm_f16_resid_ln(to, *self._wb("final.o"), qs, *self._wb("norm_final"), 1e-5, q16, qs, rows=T)
        # upscaling: ConvT 2x2 s2 -> LayerNorm2d -> GELU -> ConvT 2x2 s2 -> GELU, then the mask-0 hypernetwork dot product
        u1 = bf["u1"][: M * HW]
        gemm_f16(k16, *self._wb("up1"), _lib.EPI_BIAS_F32, u1)
        u1s, u1n, u16, u2 = bf["u1s"][: 4 * M * HW], bf["u1n"][: 4 * M * HW], bf["u16"][: 4 * M * HW], bf["u2"][: 4 * M * HW]
        rc = self.lib.vlfm_sam_pixel_shuffle2(u1.data_ptr(), u1s.data_ptr(), M, e, e, P // 4, st)
        _lib.check(rc, "vlfm_sam_pixel_shuffle2")
        layernorm(u1s, *self._wb("up_ln"), 1e-6, out32=u1n)
        self._add_act(u1n, None, None, u16, u1n.numel(), 1)
        gemm_f16(u16, *self._wb("up2"), _lib.EPI_BIAS_F32, u2)
        tok1 = q16[1:].as_strided((Mp, P), (7 * P, 1))
        gemm_f16(tok1, *self._wb("hyper0"), _lib.EPI_BIAS_RELU_F16, bf["hy1"])
        gemm_f16(bf["hy1"], *self._wb("hyper1"), _lib.EPI_BIAS_RELU_F16, bf["hy2"])
        gemm_f16(bf["hy2"], *self._wb("hyper2"), _lib.EPI_BIAS_F32, bf["hyper"])
        L = 4 * e
        low = bf["low"][:M]
        rc = self.lib.vlfm_sam_mask_logits(u2.data_ptr(), bf["hyper"].data_ptr(), low.data_ptr(), M, 2 * e, 2 * e, P // 8, st)
        _lib.check(rc, "vlfm_sam_mask_logits")
        if out is None:
            out = torch.empty(M, H, W, dtype=torch.uint8, device=self.dev)
        rc = self.lib.vlfm_sam_mask_finish(low.data_ptr(), out.data_ptr(), M, L, S, newh, neww, H, W, st)
        _lib.check(rc, "vlfm_sam_mask_finish")
        if low_out:
            return out, low.view(M, L, L)
        return out
