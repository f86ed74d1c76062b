"""Spec of MobileSAM's ``segment_bbox`` (vlfm/vlm/sam.py:40-57: ``SamPredictor.set_image`` + ``predict(box=...,
multimask_output=False)`` with ``sam_model_registry["vit_t"]``), in fp32 on the CPU.

The mobile_sam package is not available, so parity with it is unpinned; this restates the published architecture:
- preprocess: ``ResizeLongestSide`` = torchvision ``resize(to_pil_image(img), (newh, neww))`` (Pillow BILINEAR, antialiased),
  ``(x - mean) / std`` in fp32, zero pad to S x S;
- TinyViT-5M as plain torch ops with every BatchNorm left unfolded (eval mode, eps 1e-5);
- prompt encoder and mask decoder: transformers' ``SamPromptEncoder`` / ``SamMaskDecoder`` (an independent implementation of
  the decoder math) loaded through a mobile_sam -> HF name map.  Two choices differ from segment_anything and are overridden
  here: HF builds the two-way blocks' norm1..norm4 with ``layer_norm_eps`` (1e-6) where segment_anything's ``nn.LayerNorm``
  uses 1e-5 (the upscaling LayerNorm2d keeps 1e-6, as in segment_anything); HF's ``multimask_output=False`` slice (mask 0)
  matches segment_anything's;
- postprocess: ``F.interpolate`` (bilinear, align_corners=False) to S x S, crop, ``F.interpolate`` to (H, W), ``> 0``.

``fp16_operands=True`` rounds every GEMM / conv operand (inputs and weights of each conv / linear layer, and the q, k, v the
attentions multiply) to fp16 while computing in fp32: the drift of that run from the fp32 run sets the GPU tests' bar.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from vlfm_b200.vlm.sam_config import SamDims
from vlfm_b200.vlm.sam_weights import offset_index

PIXEL_MEAN = (123.675, 116.28, 103.53)
PIXEL_STD = (58.395, 57.12, 57.375)


def preshape(h: int, w: int, long_side: int) -> Tuple[int, int]:
    """ResizeLongestSide.get_preprocess_shape"""
    scale = long_side * 1.0 / max(h, w)
    return int(h * scale + 0.5), int(w * scale + 0.5)


def preprocess(image: np.ndarray, S: int) -> Tuple[torch.Tensor, Tuple[int, int]]:
    """uint8 [H,W,3] -> fp32 [1,3,S,S] (normalised, zero-padded), (newh, neww)"""
    from torchvision.transforms.functional import resize, to_pil_image

    newh, neww = preshape(image.shape[0], image.shape[1], S)
    img = np.array(resize(to_pil_image(image), [newh, neww]))
    x = torch.as_tensor(img).permute(2, 0, 1).contiguous()[None].float()
    x = (x - torch.tensor(PIXEL_MEAN).view(1, 3, 1, 1)) / torch.tensor(PIXEL_STD).view(1, 3, 1, 1)
    return F.pad(x, (0, S - neww, 0, S - newh)), (newh, neww)


def apply_box(box, hw: Tuple[int, int], S: int) -> torch.Tensor:
    """ResizeLongestSide.apply_boxes in float64, then the predictor's cast to float32 -> [1, 4]"""
    newh, neww = preshape(hw[0], hw[1], S)
    b = np.asarray(box, dtype=np.float64).reshape(2, 2).copy()
    b[:, 0] *= neww / hw[1]
    b[:, 1] *= newh / hw[0]
    return torch.as_tensor(b.reshape(1, 4), dtype=torch.float32)


class SamOracle:
    def __init__(self, d: SamDims, sd: Dict[str, torch.Tensor], fp16_operands: bool = False) -> None:
        self.d = d
        self.sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
        self.f16 = fp16_operands
        self._build_decoder()

    def q(self, t: torch.Tensor) -> torch.Tensor:
        return t.half().float() if self.f16 else t

    # ------------------------------------------------------------------------------------------------- TinyViT
    def conv_bn(self, x: torch.Tensor, name: str, stride: int = 1, groups: int = 1) -> torch.Tensor:
        w = self.sd[name + ".c.weight"]
        y = F.conv2d(self.q(x), self.q(w), None, stride, w.shape[-1] // 2, 1, groups)
        return F.batch_norm(y, self.sd[name + ".bn.running_mean"], self.sd[name + ".bn.running_var"], self.sd[name + ".bn.weight"],
                            self.sd[name + ".bn.bias"], False, 0.0, 1e-5)

    def lin(self, x: torch.Tensor, name: str) -> torch.Tensor:
        return F.linear(self.q(x), self.q(self.sd[name + ".weight"]), self.sd[name + ".bias"])

    def ln(self, x: torch.Tensor, name: str, eps: float = 1e-5) -> torch.Tensor:
        return F.layer_norm(x, (x.shape[-1],), self.sd[name + ".weight"], self.sd[name + ".bias"], eps)

    def window_attention(self, x: torch.Tensor, name: str, heads: int, ws: int) -> torch.Tensor:
        """TinyViT Attention over windows x [nW, N, C] (N = ws*ws), LayerNorm and qkv inside"""
        nW, N, C = x.shape
        hd = C // heads
        x = self.ln(x, name + ".norm")
        qkv = self.lin(x, name + ".qkv").view(nW, N, heads, 3 * hd)
        q, k, v = [self.q(t).permute(0, 2, 1, 3) for t in qkv.split([hd, hd, hd], dim=3)]
        idx = offset_index(ws)
        pts = [(i, j) for i in range(ws) for j in range(ws)]
        idxs = torch.tensor([[idx[(abs(a[0] - b[0]), abs(a[1] - b[1]))] for b in pts] for a in pts])
        attn = (q @ k.transpose(-2, -1)) * hd ** -0.5 + self.sd[name + ".attention_biases"][:, idxs]
        o = (attn.softmax(-1) @ v).transpose(1, 2).reshape(nW, N, C)
        return self.lin(o, name + ".proj")

    def tinyvit_block(self, x: torch.Tensor, name: str, heads: int, ws: int) -> torch.Tensor:
        """x [B, H, W, C] -> same; the map is zero-padded to a window multiple BEFORE the attention's LayerNorm"""
        B, H, W, C = x.shape
        res = x
        if H == ws and W == ws:
            a = self.window_attention(x.reshape(B, ws * ws, C), name + ".attn", heads, ws).view(B, H, W, C)
        else:
            pb, pr = (ws - H % ws) % ws, (ws - W % ws) % ws
            xp = F.pad(x, (0, 0, 0, pr, 0, pb))
            pH, pW = H + pb, W + pr
            nH, nW = pH // ws, pW // ws
            t = xp.view(B, nH, ws, nW, ws, C).transpose(2, 3).reshape(B * nH * nW, ws * ws, C)
            t = self.window_attention(t, name + ".attn", heads, ws)
            a = t.view(B, nH, nW, ws, ws, C).transpose(2, 3).reshape(B, pH, pW, C)[:, :H, :W]
        x = res + a
        x = self.conv_bn(x.permute(0, 3, 1, 2), name + ".local_conv", 1, C).permute(0, 2, 3, 1)
        m = self.lin(F.gelu(self.lin(self.ln(x, name + ".mlp.norm"), name + ".mlp.fc1")), name + ".mlp.fc2")
        return x + m

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        """[B,3,S,S] -> image embedding [B, P, S/16, S/16]"""
        d, e = self.d, "image_encoder."
        x = F.gelu(self.conv_bn(x, e + "patch_embed.seq.0", 2))
        x = self.conv_bn(x, e + "patch_embed.seq.2", 2)
        for s in range(len(d.embed_dims)):
            p = f"{e}layers.{s}."
            for b in range(d.depths[s]):
                q = f"{p}blocks.{b}."
                if s == 0:
                    y = F.gelu(self.conv_bn(x, q + "conv1"))
                    y = F.gelu(self.conv_bn(y, q + "conv2", 1, y.shape[1]))
                    x = F.gelu(self.conv_bn(y, q + "conv3") + x)
                else:
                    x = self.tinyvit_block(x.permute(0, 2, 3, 1), q[:-1], d.heads[s], d.windows[s]).permute(0, 3, 1, 2)
            if s + 1 < len(d.embed_dims):
                y = F.gelu(self.conv_bn(x, p + "downsample.conv1"))
                y = F.gelu(self.conv_bn(y, p + "downsample.conv2", d.merge_stride(s), y.shape[1]))
                x = self.conv_bn(y, p + "downsample.conv3")
        x = F.conv2d(self.q(x), self.q(self.sd[e + "neck.0.weight"]))
        x = self.ln(x.permute(0, 2, 3, 1), e + "neck.1", 1e-6).permute(0, 3, 1, 2)
        x = F.conv2d(self.q(x), self.q(self.sd[e + "neck.2.weight"]), padding=1)
        return self.ln(x.permute(0, 2, 3, 1), e + "neck.3", 1e-6).permute(0, 3, 1, 2)

    # ------------------------------------------------------------------------------------------------- decoder (HF)
    def _build_decoder(self) -> None:
        from transformers import SamConfig, SamMaskDecoderConfig, SamPromptEncoderConfig, SamVisionConfig
        from transformers.models.sam.modeling_sam import SamMaskDecoder, SamPromptEncoder

        d, P = self.d, self.d.prompt_dim
        vc = SamVisionConfig(output_channels=P, num_pos_feats=P // 2)
        pc = SamPromptEncoderConfig(hidden_size=P, image_size=d.img_size, image_embedding_size=d.emb_side)
        mc = SamMaskDecoderConfig(hidden_size=P, mlp_dim=d.dec_mlp, num_hidden_layers=d.dec_depth, num_attention_heads=d.dec_heads)
        cfg = SamConfig(vision_config=vc.to_dict(), prompt_encoder_config=pc.to_dict(), mask_decoder_config=mc.to_dict())
        cfg.mask_decoder_config._attn_implementation = "eager"
        self.pe = SamPromptEncoder(cfg).eval()
        self.dec = SamMaskDecoder(cfg.mask_decoder_config).eval()
        for layer in self.dec.transformer.layers:     # segment_anything: nn.LayerNorm(embedding_dim), eps 1e-5
            for n in (layer.layer_norm1, layer.layer_norm2, layer.layer_norm3, layer.layer_norm4):
                n.eps = 1e-5
        sd, pe, md = self.sd, "prompt_encoder.", "mask_decoder."
        pe_sd = {"shared_embedding.positional_embedding": sd[pe + "pe_layer.positional_encoding_gaussian_matrix"],
                 "no_mask_embed.weight": sd[pe + "no_mask_embed.weight"], "not_a_point_embed.weight": sd[pe + "not_a_point_embed.weight"]}
        for i in range(4):
            pe_sd[f"point_embed.{i}.weight"] = sd[f"{pe}point_embeddings.{i}.weight"]
        for a, b in (("conv1", "0"), ("layer_norm1", "1"), ("conv2", "3"), ("layer_norm2", "4"), ("conv3", "6")):
            for t in ("weight", "bias"):
                pe_sd[f"mask_embed.{a}.{t}"] = sd[f"{pe}mask_downscaling.{b}.{t}"]
        self.pe.load_state_dict(pe_sd)
        dec_sd = {}
        for k, v in sd.items():
            if not k.startswith(md):
                continue
            h = k[len(md):]
            h = h.replace("norm_final_attn", "layer_norm_final_attn")
            for n in range(1, 5):
                h = h.replace(f".norm{n}.", f".layer_norm{n}.")
            h = h.replace("output_upscaling.0.", "upscale_conv1.").replace("output_upscaling.1.", "upscale_layer_norm.")
            h = h.replace("output_upscaling.3.", "upscale_conv2.")
            if "output_hypernetworks_mlps" in h or "iou_prediction_head" in h:
                h = h.replace("layers.0.", "proj_in.").replace("layers.2.", "proj_out.").replace("layers.1.", "layers.0.")
            dec_sd[h] = v
        self.dec.load_state_dict(dec_sd)
        if self.f16:
            with torch.no_grad():
                for m in self.dec.modules():
                    if isinstance(m, (torch.nn.Linear, torch.nn.ConvTranspose2d)):
                        m.weight.copy_(m.weight.half().float())
                        m.register_forward_pre_hook(lambda mod, args: tuple(a.half().float() for a in args))
                for m in self.dec.modules():
                    if hasattr(m, "q_proj"):
                        for p in (m.q_proj, m.k_proj, m.v_proj):
                            p.register_forward_hook(lambda mod, args, out: out.half().float())

    def dense_pe(self) -> torch.Tensor:
        n = self.d.emb_side
        grid = torch.ones((n, n))
        y = (grid.cumsum(0) - 0.5) / n
        x = (grid.cumsum(1) - 0.5) / n
        return self.pe.shared_embedding(torch.stack([x, y], -1)).permute(2, 0, 1)[None]

    def low_res_logits(self, emb: torch.Tensor, box, hw: Tuple[int, int]) -> torch.Tensor:
        """emb [1, P, e, e], box [x1,y1,x2,y2] in frame pixels -> mask-0 logits [4e, 4e]"""
        b = apply_box(box, hw, self.d.img_size)
        sparse, dense = self.pe(None, None, b[None], None)
        masks, _ = self.dec(emb, self.dense_pe(), sparse, dense, multimask_output=False)
        return masks[0, 0, 0]

    def postprocess(self, low: torch.Tensor, hw: Tuple[int, int]) -> torch.Tensor:
        S = self.d.img_size
        newh, neww = preshape(hw[0], hw[1], S)
        m = F.interpolate(low[None, None], (S, S), mode="bilinear", align_corners=False)[..., :newh, :neww]
        return F.interpolate(m, hw, mode="bilinear", align_corners=False)[0, 0]

    @torch.no_grad()
    def segment(self, image: np.ndarray, box):
        """-> (bool mask [H,W], full-resolution logits [H,W], low-res logits, image embedding)"""
        x, _ = preprocess(image, self.d.img_size)
        emb = self.encode(x)
        low = self.low_res_logits(emb, box, image.shape[:2])
        full = self.postprocess(low, image.shape[:2])
        return (full > 0).numpy(), full, low, emb
