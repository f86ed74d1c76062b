"""mobile_sam checkpoint names -> the layout of ``sam_engine.MobileSamEngine``.

- Every ``Conv2d_BN`` (conv + eval-mode BatchNorm, eps 1e-5) is folded into one weight and bias.
- Convolutions become GEMM operands: 1x1 -> [O, C]; 3x3 -> [O, ldk] with columns (ky, kx, c), K zero-padded to a multiple of 8
  (the stem's 27 -> 32); depthwise 3x3 -> [9, C] (tap-major) for ``vlfm_sam_dwconv3x3``.
- The TinyViT qkv rows, interleaved per head (q_h, k_h, v_h), are permuted to [q | k | v] with head h at h*32 inside each, and
  ``attention_biases[h, idx]`` is re-indexed by |dy|*ws + |dx|.
- The 2x2 stride-2 transposed convs become GEMMs with rows (dy, dx, o).
- Accepted and dropped: the TinyViT classification head (``norm_head``, ``head``), BatchNorm ``num_batches_tracked``, the
  buffers the architecture recomputes (``attention_bias_idxs``, ``pixel_mean`` / ``pixel_std``) and the modules a box prompt
  with ``multimask_output=False`` never runs (point / mask prompt embeddings, the IoU head, hypernetworks 1..3).  Any other
  unknown key raises, and so does a missing one.
"""
from __future__ import annotations

import itertools
import re
from typing import Dict

import torch

from .sam_config import SamDims

BN_EPS = 1e-5

_DROP = [
    r"image_encoder\.norm_head\..*", r"image_encoder\.head\..*", r".*\.num_batches_tracked", r".*\.attention_bias_idxs",
    r"pixel_mean", r"pixel_std",
    r"prompt_encoder\.point_embeddings\.[01]\.weight", r"prompt_encoder\.not_a_point_embed\.weight",
    r"prompt_encoder\.mask_downscaling\..*", r"mask_decoder\.iou_prediction_head\..*",
    r"mask_decoder\.output_hypernetworks_mlps\.[1-9]\d*\..*",
]
_DROP_RE = re.compile("|".join(f"(?:{p})" for p in _DROP))


def offset_index(ws: int) -> Dict[tuple, int]:
    """TinyViT's Attention: (|dy|, |dx|) -> column of ``attention_biases``, numbered in order of first appearance."""
    points = list(itertools.product(range(ws), range(ws)))
    offsets: Dict[tuple, int] = {}
    for p1 in points:
        for p2 in points:
            off = (abs(p1[0] - p2[0]), abs(p1[1] - p2[1]))
            if off not in offsets:
                offsets[off] = len(offsets)
    return offsets


def fold_conv_bn(sd: Dict[str, torch.Tensor], name: str):
    """Conv2d_BN -> (weight [O, Cg, k, k], bias [O]) of the equivalent conv, in float64 then float32."""
    w = sd[name + ".c.weight"].double()
    g, b = sd[name + ".bn.weight"].double(), sd[name + ".bn.bias"].double()
    mu, var = sd[name + ".bn.running_mean"].double(), sd[name + ".bn.running_var"].double()
    s = g / torch.sqrt(var + BN_EPS)
    return (w * s[:, None, None, None]).float(), (b - mu * s).float()


def conv3x3_rows(w: torch.Tensor) -> torch.Tensor:
    """[O, C, 3, 3] -> [O, ldk] GEMM rows with columns (ky, kx, c), ldk = 9C rounded up to a multiple of 8."""
    O, C = w.shape[:2]
    r = w.permute(0, 2, 3, 1).reshape(O, 9 * C)
    ldk = (9 * C + 7) // 8 * 8
    return torch.nn.functional.pad(r, (0, ldk - 9 * C)).contiguous()


def convT_rows(w: torch.Tensor, b: torch.Tensor):
    """ConvTranspose2d(k=2, s=2) weight [C, O, 2, 2] -> GEMM rows [4*O, C] ordered (dy, dx, o), bias [4*O]."""
    C, O = w.shape[:2]
    return w.permute(2, 3, 1, 0).reshape(4 * O, C).contiguous(), b.repeat(4).contiguous()


def convert_state_dict(sd: Dict[str, torch.Tensor], d: SamDims) -> Dict[str, torch.Tensor]:
    used = set()

    def g(k: str) -> torch.Tensor:
        if k not in sd:
            raise KeyError(f"mobile_sam checkpoint: missing {k}")
        used.add(k)
        return sd[k].float()

    def cbn(name: str):
        for s in (".c.weight", ".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"):
            g(name + s)
        return fold_conv_bn(sd, name)

    out: Dict[str, torch.Tensor] = {}

    def put_1x1(dst: str, name: str) -> None:
        w, b = cbn(name)
        out[dst + ".w"], out[dst + ".b"] = w.reshape(w.shape[0], -1).contiguous(), b

    def put_dw(dst: str, name: str) -> None:
        w, b = cbn(name)
        out[dst + ".w"], out[dst + ".b"] = w.reshape(w.shape[0], 9).t().contiguous(), b

    def put_lin(dst: str, name: str) -> None:
        out[dst + ".w"], out[dst + ".b"] = g(name + ".weight"), g(name + ".bias")

    def put_ln(dst: str, name: str) -> None:
        out[dst + ".w"], out[dst + ".b"] = g(name + ".weight"), g(name + ".bias")

    e = "image_encoder."
    E = d.embed_dims
    for i, name in enumerate(("patch_embed.seq.0", "patch_embed.seq.2")):
        w, b = cbn(e + name)
        out[f"stem{i}.w"], out[f"stem{i}.b"] = conv3x3_rows(w), b
    for s in range(len(E)):
        p = f"{e}layers.{s}."
        for bi in range(d.depths[s]):
            q, o = f"{p}blocks.{bi}.", f"l{s}.b{bi}."
            if s == 0:
                put_1x1(o + "conv1", q + "conv1")
                put_dw(o + "conv2", q + "conv2")
                put_1x1(o + "conv3", q + "conv3")
                continue
            C, H, ws = E[s], d.heads[s], d.windows[s]
            hd = C // H
            put_ln(o + "ln1", q + "attn.norm")
            w, b = g(q + "attn.qkv.weight"), g(q + "attn.qkv.bias")
            # rows (head, [q k v], dim) -> ([q k v], head, dim)
            out[o + "qkv.w"] = w.reshape(H, 3, hd, C).transpose(0, 1).reshape(3 * C, C).contiguous()
            out[o + "qkv.b"] = b.reshape(H, 3, hd).transpose(0, 1).reshape(3 * C).contiguous()
            ab = g(q + "attn.attention_biases")
            idx = offset_index(ws)
            cols = torch.tensor([idx[(dy, dx)] for dy in range(ws) for dx in range(ws)])
            out[o + "bias"] = ab[:, cols].contiguous()
            put_lin(o + "proj", q + "attn.proj")
            put_dw(o + "local", q + "local_conv")
            put_ln(o + "ln2", q + "mlp.norm")
            put_lin(o + "fc1", q + "mlp.fc1")
            put_lin(o + "fc2", q + "mlp.fc2")
        if s + 1 < len(E):
            put_1x1(f"l{s}.down.conv1", p + "downsample.conv1")
            put_dw(f"l{s}.down.conv2", p + "downsample.conv2")
            put_1x1(f"l{s}.down.conv3", p + "downsample.conv3")
    out["neck0.w"] = g(e + "neck.0.weight").reshape(d.prompt_dim, E[-1]).contiguous()
    put_ln("neck1", e + "neck.1")
    out["neck2.w"] = conv3x3_rows(g(e + "neck.2.weight"))
    put_ln("neck3", e + "neck.3")

    pe = "prompt_encoder."
    out["pe.gauss"] = g(pe + "pe_layer.positional_encoding_gaussian_matrix").contiguous()
    out["no_mask"] = g(pe + "no_mask_embed.weight").reshape(-1).contiguous()
    md = "mask_decoder."
    out["fixed"] = torch.cat([g(md + "iou_token.weight"), g(md + "mask_tokens.weight"),
                              g(pe + "point_embeddings.2.weight"), g(pe + "point_embeddings.3.weight")], 0).contiguous()
    t = md + "transformer."

    def put_attn(dst: str, name: str) -> None:
        for a, b in (("q", "q_proj"), ("k", "k_proj"), ("v", "v_proj"), ("o", "out_proj")):
            put_lin(f"{dst}.{a}", f"{name}.{b}")

    for i in range(d.dec_depth):
        q, o = f"{t}layers.{i}.", f"dec{i}."
        put_attn(o + "self", q + "self_attn")
        put_attn(o + "t2i", q + "cross_attn_token_to_image")
        put_attn(o + "i2t", q + "cross_attn_image_to_token")
        for n in range(1, 5):
            put_ln(f"{o}norm{n}", f"{q}norm{n}")
        put_lin(o + "mlp1", q + "mlp.lin1")
        put_lin(o + "mlp2", q + "mlp.lin2")
    put_attn("final", t + "final_attn_token_to_image")
    put_ln("norm_final", t + "norm_final_attn")
    out["up1.w"], out["up1.b"] = convT_rows(g(md + "output_upscaling.0.weight"), g(md + "output_upscaling.0.bias"))
    put_ln("up_ln", md + "output_upscaling.1")
    out["up2.w"], out["up2.b"] = convT_rows(g(md + "output_upscaling.3.weight"), g(md + "output_upscaling.3.bias"))
    for j in range(3):
        put_lin(f"hyper{j}", f"{md}output_hypernetworks_mlps.0.layers.{j}")

    unknown = sorted(k for k in sd if k not in used and not _DROP_RE.fullmatch(k))
    if unknown:
        raise KeyError(f"mobile_sam checkpoint: unknown keys {unknown[:8]}{' ...' if len(unknown) > 8 else ''}")
    return out


def load_checkpoint(path: str, d: SamDims) -> Dict[str, torch.Tensor]:
    """mobile_sam.pt (a plain state dict, or {'model': ...}) -> engine layout."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "model" in sd and isinstance(sd["model"], dict):
        sd = sd["model"]
    return convert_state_dict(sd, d)
