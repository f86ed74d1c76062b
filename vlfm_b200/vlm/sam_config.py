"""MobileSAM (``sam_model_registry["vit_t"]``: TinyViT-5M encoder, box-prompted two-way mask decoder) dimensions and seeded
synthetic weights.

``random_state_dict`` returns a state dict under the mobile_sam checkpoint's own names (``image_encoder.*``,
``prompt_encoder.*``, ``mask_decoder.*``), BatchNorm running statistics, the TinyViT classification head and the unused
prompt / IoU modules included, so that it goes through the same key map (``sam_weights.convert_state_dict``) as a real
checkpoint.  No checkpoint is available offline: tests and benchmarks use these weights.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Tuple

import torch


@dataclass(frozen=True)
class SamDims:
    embed_dims: Tuple[int, ...] = (64, 128, 160, 320)
    depths: Tuple[int, ...] = (2, 2, 6, 2)
    heads: Tuple[int, ...] = (2, 4, 5, 10)
    windows: Tuple[int, ...] = (7, 7, 14, 7)
    mlp_ratio: int = 4
    mbconv_ratio: int = 4
    img_size: int = 1024          # ResizeLongestSide target and the encoder's input side
    prompt_dim: int = 256         # neck output channels = decoder width
    dec_depth: int = 2
    dec_heads: int = 8
    dec_mlp: int = 2048
    num_mask_tokens: int = 4      # multimask (3) + 1
    classes: int = 1000           # TinyViT classification head (dropped at load)

    @property
    def stem_mid(self) -> int:
        return self.embed_dims[0] // 2

    @property
    def emb_side(self) -> int:
        return self.img_size // 16

    @property
    def resolutions(self) -> Tuple[int, ...]:
        """Side of the map each stage runs on: S/4, S/8, S/16, S/16 (the merge into the last stage has stride 1)."""
        r0 = self.img_size // 4
        return (r0, r0 // 2, r0 // 4, r0 // 4)

    def merge_stride(self, s: int) -> int:
        """stride of the PatchMerging after stage s.  mobile_sam uses stride 1 into out dims 320 / 448 / 576, which for vit_t is
        the merge into the last stage; TINY keeps that geometry."""
        return 1 if s + 1 == len(self.embed_dims) - 1 else 2


VIT_T = SamDims()
# head dim 32 (window attention) and 16 (decoder cross attention) as at full size; 256-pixel input, embedding 16 x 16
TINY = SamDims(embed_dims=(32, 64, 64, 96), depths=(1, 1, 2, 1), heads=(1, 2, 2, 3), img_size=256, prompt_dim=128, dec_heads=4,
               dec_mlp=256, classes=10)


def random_state_dict(d: SamDims, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded mobile_sam-named weights.  Weights ~ N(0, 1/fan_in), BatchNorm statistics and affine parameters around
    identity, attention biases ~ N(0, 0.5): every term of the forward contributes.  The mask tokens and the hypernetwork
    output layer are scaled so that the low-res logits change sign across the image (non-degenerate masks)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    rn = lambda *s, std=1.0: torch.randn(*s, generator=g) * std
    ru = lambda *s, lo=0.5, hi=1.5: lo + (hi - lo) * torch.rand(*s, generator=g)

    def lin(name: str, o: int, i: int, bias: bool = True, gain: float = 1.0) -> None:
        sd[name + ".weight"] = rn(o, i, std=gain / math.sqrt(i))
        if bias:
            sd[name + ".bias"] = rn(o, std=0.05)

    def ln(name: str, n: int) -> None:
        sd[name + ".weight"] = ru(n, lo=0.7, hi=1.3)
        sd[name + ".bias"] = rn(n, std=0.1)

    def conv_bn(name: str, o: int, i: int, k: int, groups: int = 1) -> None:
        sd[name + ".c.weight"] = rn(o, i // groups, k, k, std=1.0 / math.sqrt(i // groups * k * k))
        sd[name + ".bn.weight"] = ru(o)
        sd[name + ".bn.bias"] = rn(o, std=0.1)
        sd[name + ".bn.running_mean"] = rn(o, std=0.1)
        sd[name + ".bn.running_var"] = ru(o)
        sd[name + ".bn.num_batches_tracked"] = torch.tensor(1000)

    e = "image_encoder."
    E = d.embed_dims
    conv_bn(e + "patch_embed.seq.0", d.stem_mid, 3, 3)
    conv_bn(e + "patch_embed.seq.2", E[0], d.stem_mid, 3)
    for s in range(len(E)):
        p = f"{e}layers.{s}."
        for b in range(d.depths[s]):
            q = f"{p}blocks.{b}."
            if s == 0:
                hid = E[0] * d.mbconv_ratio
                conv_bn(q + "conv1", hid, E[0], 1)
                conv_bn(q + "conv2", hid, hid, 3, groups=hid)
                conv_bn(q + "conv3", E[0], hid, 1)
            else:
                C, ws = E[s], d.windows[s]
                ln(q + "attn.norm", C)
                lin(q + "attn.qkv", 3 * C, C)
                lin(q + "attn.proj", C, C)
                sd[q + "attn.attention_biases"] = rn(d.heads[s], ws * ws, std=0.5)
                conv_bn(q + "local_conv", C, C, 3, groups=C)
                ln(q + "mlp.norm", C)
                lin(q + "mlp.fc1", d.mlp_ratio * C, C)
                lin(q + "mlp.fc2", C, d.mlp_ratio * C)
        if s + 1 < len(E):
            conv_bn(p + "downsample.conv1", E[s + 1], E[s], 1)
            conv_bn(p + "downsample.conv2", E[s + 1], E[s + 1], 3, groups=E[s + 1])
            conv_bn(p + "downsample.conv3", E[s + 1], E[s + 1], 1)
    ln(e + "norm_head", E[-1])
    lin(e + "head", d.classes, E[-1])
    P = d.prompt_dim
    sd[e + "neck.0.weight"] = rn(P, E[-1], 1, 1, std=1.0 / math.sqrt(E[-1]))
    ln(e + "neck.1", P)
    sd[e + "neck.2.weight"] = rn(P, P, 3, 3, std=1.0 / math.sqrt(9 * P))
    ln(e + "neck.3", P)

    pe = "prompt_encoder."
    sd[pe + "pe_layer.positional_encoding_gaussian_matrix"] = rn(2, P // 2)
    for i in range(4):
        sd[f"{pe}point_embeddings.{i}.weight"] = rn(1, P)
    sd[pe + "not_a_point_embed.weight"] = rn(1, P)
    sd[pe + "no_mask_embed.weight"] = rn(1, P)
    mi = 16
    sd[pe + "mask_downscaling.0.weight"] = rn(mi // 4, 1, 2, 2, std=0.5)
    sd[pe + "mask_downscaling.0.bias"] = rn(mi // 4, std=0.05)
    ln(pe + "mask_downscaling.1", mi // 4)
    sd[pe + "mask_downscaling.3.weight"] = rn(mi, mi // 4, 2, 2, std=0.25)
    sd[pe + "mask_downscaling.3.bias"] = rn(mi, std=0.05)
    ln(pe + "mask_downscaling.4", mi)
    sd[pe + "mask_downscaling.6.weight"] = rn(P, mi, 1, 1, std=0.25)
    sd[pe + "mask_downscaling.6.bias"] = rn(P, std=0.05)

    md = "mask_decoder."
    t = md + "transformer."

    def attn(name: str, inner: int) -> None:
        lin(name + ".q_proj", inner, P)
        lin(name + ".k_proj", inner, P)
        lin(name + ".v_proj", inner, P)
        lin(name + ".out_proj", P, inner)

    for i in range(d.dec_depth):
        q = f"{t}layers.{i}."
        attn(q + "self_attn", P)
        ln(q + "norm1", P)
        attn(q + "cross_attn_token_to_image", P // 2)
        ln(q + "norm2", P)
        lin(q + "mlp.lin1", d.dec_mlp, P)
        lin(q + "mlp.lin2", P, d.dec_mlp)
        ln(q + "norm3", P)
        ln(q + "norm4", P)
        attn(q + "cross_attn_image_to_token", P // 2)
    attn(t + "final_attn_token_to_image", P // 2)
    ln(t + "norm_final_attn", P)
    sd[md + "iou_token.weight"] = rn(1, P)
    sd[md + "mask_tokens.weight"] = rn(d.num_mask_tokens, P)
    sd[md + "output_upscaling.0.weight"] = rn(P, P // 4, 2, 2, std=1.0 / math.sqrt(P))
    sd[md + "output_upscaling.0.bias"] = rn(P // 4, std=0.05)
    ln(md + "output_upscaling.1", P // 4)
    sd[md + "output_upscaling.3.weight"] = rn(P // 4, P // 8, 2, 2, std=1.0 / math.sqrt(P // 4))
    sd[md + "output_upscaling.3.bias"] = rn(P // 8, std=0.05)
    for m in range(d.num_mask_tokens):
        h = f"{md}output_hypernetworks_mlps.{m}.layers."
        lin(h + "0", P, P)
        lin(h + "1", P, P)
        lin(h + "2", P // 8, P, gain=2.0)
    lin(md + "iou_prediction_head.layers.0", 256, P)
    lin(md + "iou_prediction_head.layers.1", 256, 256)
    lin(md + "iou_prediction_head.layers.2", d.num_mask_tokens, 256)
    return sd
