"""GroundingDINO model-level forward on the library: everything between the Swin backbone and the (boxes, logits) pair that is not
inside an encoder / decoder layer -- neck (1x1 / 3x3 conv + GroupNorm), position embeddings, flattening, two-stage proposal
scoring, language-guided top-900 query selection, and the final box / class heads.

Reference: ``groundingdino.util.inference.predict`` -> ``model(image, captions=[caption])`` (vlfm/vlm/grounding_dino.py:61-67);
the architecture-equivalent module graph is HF's ``GroundingDinoModel.forward`` + ``GroundingDinoForObjectDetection.forward``,
which this class restates for inference on fully valid images (pixel_mask all ones -- the reference never pads):

  * the neck is a GEMM over the backbone's NHWC rows (a 1x1 conv IS a row GEMM; the 3x3 stride-2 conv of the fourth level is an
    im2col + GEMM) followed by ``groupnorm_rows`` writing straight into the flattened [B, S, 256] encoder input -- no NCHW round
    trip, no cat;
  * position embeddings (+ level embeddings), padding masks, valid ratios, proposal anchors and their validity mask depend on the
    shapes only: built once per (batch, image size) with the reference's own arithmetic and cached;
  * the text tower output, its projection and the text masks depend on the caption only: cached per caption;
  * two-stage selection scores = max over valid tokens of <proposal feature, text feature> (``proposal_scores``), top-900 per image
    (``topk_rows``), and the 3-layer box head runs on the 900 SELECTED rows only (it is row-wise: same values as selecting after
    running it on all 6380 proposals, which is what the module graph does);
  * the heads run for the LAST decoder layer only (the other five are training-time auxiliary outputs).

The encoder and decoder LAYERS are the HF layer objects whose sublayers ``gdino_accel`` replaced (wgmma GEMMs, fused deformable
sampling, bi-attention); the stacks are sequenced here: the encoder loop feeds every layer the cached deformable reference points
and the cached sine embedding of the text position ids (the module code rebuilds both per call / per layer), the decoder loop
computes each layer's query position embedding with one kernel + the reference_points_head GEMMs and refines the reference points
with the per-layer box head + ``box_finish`` (no auxiliary outputs).  Every array operation here goes through ``ops`` (C-ABI kernels, ``gdino_ops.LibOps``); tests substitute a
torch implementation of the same interface to check the orchestration against HF on the CPU (tests/test_gdino_forward_cpu.py).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from .dense import conv_rows


class GdinoForward:
    def __init__(self, model, ops, backbone=None) -> None:
        """model: HF GroundingDinoForObjectDetection (eval, layers already accelerated); ops: kernel interface; backbone:
        SwinBackboneEngine (None in the CPU test, where feature rows are supplied directly)."""
        self.m = model
        self.core = model.model
        self.cfg = model.config
        self.ops = ops
        self.backbone = backbone
        self.d = self.cfg.d_model
        self.nq = self.cfg.num_queries
        self._shape_cache: Dict[Tuple[int, int, int], Dict[str, Any]] = {}
        self._text_cache: Dict[Tuple[Tuple[int, ...], int], Dict[str, Any]] = {}
        core = self.core
        assert self.cfg.two_stage and self.cfg.num_feature_levels == 4 and len(core.input_proj_vision) == 4
        # neck weights as row-GEMM operands
        self.neck: List[Dict[str, torch.Tensor]] = []
        for lvl, seq in enumerate(core.input_proj_vision):
            conv, gn = seq[0], seq[1]
            self.neck.append(dict(w=ops.weight(conv_rows(conv.weight.detach())), b=conv.bias.detach().float().contiguous(),
                                  g=gn.weight.detach().float().contiguous(), be=gn.bias.detach().float().contiguous(), groups=gn.num_groups, eps=gn.eps, k=conv.kernel_size[0]))
        self.enc_out_w = ops.weight(core.enc_output.weight.detach())
        self.enc_out_b = core.enc_output.bias.detach().float().contiguous()
        self.enc_norm = (core.enc_output_norm.weight.detach().float().contiguous(), core.enc_output_norm.bias.detach().float().contiguous(),
                         core.enc_output_norm.eps)
        self.text_proj_w = ops.weight(core.text_projection.weight.detach())
        self.text_proj_b = core.text_projection.bias.detach().float().contiguous()

        def mlp(head):
            """3-layer box head as GEMM operands; the 4-wide last layer is zero-padded to 8 outputs (the GEMM's store granularity),
            the caller keeps the first four columns."""
            out = []
            for l in head.layers:
                w, b = l.weight.detach().float(), l.bias.detach().float()
                if w.shape[0] % 8:
                    pad = 8 - w.shape[0] % 8
                    w = torch.cat([w, w.new_zeros(pad, w.shape[1])], 0)
                    b = torch.cat([b, b.new_zeros(pad)], 0)
                out.append((ops.weight(w), b.contiguous()))
            return out

        self.enc_bbox = mlp(core.encoder_output_bbox_embed)
        self.layer_bbox = [mlp(model.bbox_embed[i]) for i in range(self.cfg.decoder_layers)]     # iterative box refinement, one head per layer
        self.last_bbox = self.layer_bbox[-1]
        self.ref_head = mlp(core.decoder.reference_points_head)
        ln = core.decoder.layer_norm
        self.dec_norm = (ln.weight.detach().float().contiguous(), ln.bias.detach().float().contiguous(), ln.eps)
        # get_sine_pos_embed's frequency table, by the reference's own expression (float32)
        P = self.d // 2
        dim_t = torch.arange(P, dtype=torch.float32, device=core.level_embed.device)
        self.dim_t = (10000 ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / P)).contiguous()
        self.last_reference_points: Optional[torch.Tensor] = None

    # ------------------------------------------------------------------------------ caches ----
    def _shape_constants(self, B: int, H: int, W: int, shapes: Sequence[Tuple[int, int]], device) -> Dict[str, Any]:
        key = (B, H, W)
        c = self._shape_cache.get(key)
        if c is not None:
            return c
        core, d = self.core, self.d
        pixel_mask = torch.ones((B, H, W), dtype=torch.long, device=device)
        pos_list, masks = [], []
        for (h, w) in shapes:
            mask = torch.nn.functional.interpolate(pixel_mask[None].float(), size=(h, w)).to(torch.bool)[0]
            pos = core.backbone.position_embedding(torch.empty(0, device=device), mask).float()         # [B, 256, h, w]
            pos_list.append(pos.flatten(2).transpose(1, 2) + core.level_embed[len(pos_list)].detach().view(1, 1, -1))
            masks.append(mask)
        S = sum(h * w for h, w in shapes)
        spatial_shapes = torch.as_tensor(list(shapes), dtype=torch.long, device=device)
        level_start = torch.cat((spatial_shapes.new_zeros((1,)), spatial_shapes.prod(1).cumsum(0)[:-1]))
        mask_flatten = torch.cat([m.flatten(1) for m in masks], 1)                                   # True = valid pixel
        valid_ratios = torch.stack([core.get_valid_ratio(m) for m in masks], 1).float()
        # two-stage anchors (generate_encoder_output_proposals with an all-valid padding mask)
        _, proposals = self._anchors(B, shapes, device)
        valid = ((proposals > 0.01) & (proposals < 0.99)).all(-1, keepdim=True)
        logits = torch.log(proposals / (1 - proposals)).masked_fill(~valid, float("inf"))
        c = dict(pos=torch.cat(pos_list, 1).contiguous(), S=S, spatial_shapes=spatial_shapes, shapes=[tuple(s) for s in shapes],
                 level_start=level_start, mask_flatten=mask_flatten, valid_ratios=valid_ratios, anchor_logits=logits.contiguous(),
                 anchor_valid=valid.to(torch.uint8).contiguous(), offsets=[int(v) for v in level_start.tolist()])
        if len(self._shape_cache) >= 4:
            self._shape_cache.pop(next(iter(self._shape_cache)))
        self._shape_cache[key] = c
        return c

    @staticmethod
    def _anchors(B: int, shapes, device):
        props = []
        for level, (h, w) in enumerate(shapes):
            gy, gx = torch.meshgrid(torch.linspace(0, h - 1, h, dtype=torch.float32, device=device),
                                    torch.linspace(0, w - 1, w, dtype=torch.float32, device=device), indexing="ij")
            grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
            scale = torch.tensor([w, h], dtype=torch.float32, device=device).view(1, 1, 1, 2)
            grid = (grid.unsqueeze(0).expand(B, -1, -1, -1) + 0.5) / scale
            wh = torch.ones_like(grid) * 0.05 * (2.0 ** level)
            props.append(torch.cat((grid, wh), -1).view(B, -1, 4))
        return None, torch.cat(props, 1)

    def _text(self, input_ids: Sequence[int], B: int, device) -> Dict[str, Any]:
        key = (tuple(int(i) for i in input_ids), B)
        t = self._text_cache.get(key)
        if t is not None:
            return t
        from transformers.models.grounding_dino.modeling_grounding_dino import generate_masks_with_special_tokens_and_transfer_map

        core = self.core
        ids = torch.tensor([list(key[0])], dtype=torch.long, device=device).expand(B, -1).contiguous()
        self_masks, position_ids = generate_masks_with_special_tokens_and_transfer_map(ids)
        tt = torch.zeros_like(ids)
        token_mask = torch.ones_like(ids).bool()
        out = core.text_backbone(ids, self_masks[:, None, :, :], tt, position_ids, return_dict=True)
        feats = out.last_hidden_state.float()
        T = feats.shape[1]
        proj = self.ops.linear(feats.reshape(B * T, -1), self.text_proj_w, self.text_proj_b).view(B, T, self.d)
        t = dict(features=proj.contiguous(), token_mask=token_mask, self_masks=self_masks, position_ids=position_ids, T=T)
        if len(self._text_cache) >= 8:
            self._text_cache.pop(next(iter(self._text_cache)))
        self._text_cache[key] = t
        return t

    # ----------------------------------------------------------------------------- forward ----
    @torch.inference_mode()
    def forward_features(self, feats: List[Tuple[torch.Tensor, int, int]], B: int, H: int, W: int, input_ids: Sequence[int]):
        """feats: three (rows [B*h*w, C] fp32, h, w) backbone stages (NHWC rows).  -> (sigmoid logits [B, nq, max_text_len],
        boxes [B, nq, 4] cxcywh)."""
        ops, core, d = self.ops, self.core, self.d
        dev = feats[0][0].device
        h4, w4 = feats[-1][1], feats[-1][2]
        shapes = [(h, w) for _, h, w in feats] + [((h4 + 2 - 3) // 2 + 1, (w4 + 2 - 3) // 2 + 1)]
        sc = self._shape_constants(B, H, W, shapes, dev)
        tx = self._text(input_ids, B, dev)
        self.last = (sc, tx)
        S = sc["S"]
        # ---- neck -> flattened encoder input
        src = torch.empty((B, S, d), dtype=torch.float32, device=dev)
        for lvl in range(4):
            nk = self.neck[lvl]
            h, w = shapes[lvl]
            if nk["k"] == 1:
                a = last16 = ops.to_operand(feats[lvl][0])
            else:   # the 3x3 stride-2 conv reads the last backbone stage, whose fp16 operand level 2 has just made
                _, hh, ww = feats[-1]
                a = ops.im2col3x3s2(last16, B, hh, ww)
            y = ops.linear_operand(a, nk["w"], nk["b"])                                     # [B*h*w, 256] fp32
            ops.groupnorm_rows(y, B, h * w, d, nk["groups"], nk["g"], nk["be"], nk["eps"], src, sc["offsets"][lvl], S)
        # ---- encoder: GroundingDinoEncoder.forward is a loop over its layers; the per-call constants it rebuilds -- the deformable
        # reference points (shapes only) and, inside EVERY layer, the sine embedding of the text position ids (caption only) -- come
        # from the caches instead (~80 elementwise launches per image batch)
        if "enc_ref" not in sc:
            sc["enc_ref"] = core.encoder.get_reference_points(sc["shapes"], sc["valid_ratios"], device=dev)
        if "pos_embed" not in tx:
            from transformers.models.grounding_dino.modeling_grounding_dino import get_sine_pos_embed

            tx["pos_embed"] = get_sine_pos_embed(tx["position_ids"][..., None], num_pos_feats=d, exchange_xy=False)
            tx["not_token_mask"], tx["not_self_masks"] = ~tx["token_mask"], ~tx["self_masks"]
        if "not_mask_flatten" not in sc:
            sc["not_mask_flatten"] = ~sc["mask_flatten"]
        memory, text_mem = src, tx["features"]
        for layer in core.encoder.layers:
            (memory, text_mem), _ = layer(vision_features=memory, vision_position_embedding=sc["pos"], spatial_shapes=sc["spatial_shapes"],
                                          spatial_shapes_list=sc["shapes"], level_start_index=sc["level_start"],
                                          key_padding_mask=sc["not_mask_flatten"], reference_points=sc["enc_ref"], text_features=text_mem,
                                          text_attention_mask=tx["not_token_mask"], text_position_embedding=tx["pos_embed"],
                                          text_self_attention_masks=tx["not_self_masks"], text_position_ids=None)
        # ---- two-stage proposals: object queries, scores, top-k, box head on the selected rows
        oq = ops.mask_rows(memory.reshape(B * S, d), sc["anchor_valid"].reshape(B * S))                # invalid anchors -> 0
        oq = ops.linear(oq, self.enc_out_w, self.enc_out_b)
        oq = ops.layernorm(oq, *self.enc_norm)                                                         # [B*S, 256]
        scores = ops.proposal_scores(oq, text_mem.reshape(B * tx["T"], d).contiguous(), B, S, tx["T"])   # [B, S]: max over tokens
        topk = ops.topk_rows(scores, self.nq)                                                          # [B, nq] int64, descending score
        sel = ops.gather_rows(oq.view(B, S, d), topk)                                                  # [B, nq, 256]
        x = sel.reshape(B * self.nq, d)
        for i, (w_, b_) in enumerate(self.enc_bbox):
            x = ops.linear(x, w_, b_, relu=i < len(self.enc_bbox) - 1)
        anchors = ops.gather_rows(sc["anchor_logits"], topk)                                           # [B, nq, 4]
        reference_points = (x[:, :4].reshape(B, self.nq, 4) + anchors).sigmoid()
        target = core.query_position_embeddings.weight.detach().unsqueeze(0).repeat(B, 1, 1)
        self.last_reference_points = reference_points
        hs, ref_last = self._decoder(target, memory, text_mem, reference_points, sc, tx, B)
        # ---- heads of the last layer
        x = hs.reshape(B * self.nq, d)
        for i, (w_, b_) in enumerate(self.last_bbox):
            x = ops.linear(x, w_, b_, relu=i < len(self.last_bbox) - 1)
        boxes = ops.box_finish(x[:, :4].reshape(B, self.nq, 4).contiguous(), ref_last.contiguous())    # sigmoid(delta + logit(ref, eps=1e-5))
        logits = ops.contrastive_sigmoid(hs.contiguous(), text_mem.contiguous(), self.cfg.max_text_len)   # [B, nq, max_text_len]
        return logits, boxes

    def _decoder(self, hidden, memory, text_mem, ref, sc, tx, B):
        """GroundingDinoDecoder.forward restated for inference (no auxiliary outputs): per layer the query position embedding
        (one kernel + the two-layer reference_points_head on the GEMM), the decoder layer (HF module, accelerated), and -- between
        layers -- the iterative box refinement ref <- sigmoid(bbox_embed[i](h) + logit(ref)).  Returns the post-norm hidden state of the
        last layer and the reference points that layer received (what the final box head refines)."""
        ops, core, d, nq = self.ops, self.core, self.d, self.nq
        dec = core.decoder
        tmask = tx.get("dec_text_mask")
        if tmask is None:       # as the module builds it (additive, all zeros for the never-padded captions of this path)
            m = (~tx["token_mask"])[:, None, None, :].repeat(1, self.cfg.decoder_attention_heads, nq, 1).to(text_mem.dtype)
            tmask = tx["dec_text_mask"] = m * torch.finfo(text_mem.dtype).min
        n_layers = len(dec.layers)
        for idx, layer in enumerate(dec.layers):
            ref_in, emb = ops.decoder_query_pos(ref, sc["valid_ratios"], self.dim_t)
            x = emb
            for i, (w_, b_) in enumerate(self.ref_head):
                x = ops.linear(x, w_, b_, relu=i < len(self.ref_head) - 1)
            query_pos = x.view(B, nq, d)
            hidden = layer(hidden_states=hidden, position_embeddings=query_pos, reference_points=ref_in, spatial_shapes=sc["spatial_shapes"],
                           spatial_shapes_list=sc["shapes"], level_start_index=sc["level_start"], vision_encoder_hidden_states=memory,
                           vision_encoder_attention_mask=sc["mask_flatten"], text_encoder_hidden_states=text_mem,
                           text_encoder_attention_mask=tmask, self_attn_mask=None, output_attentions=False)[0]
            if idx + 1 < n_layers:
                x = hidden.reshape(B * nq, d)
                for i, (w_, b_) in enumerate(self.layer_bbox[idx]):
                    x = ops.linear(x, w_, b_, relu=i < len(self.layer_bbox[idx]) - 1)
                ref = ops.box_finish(x[:, :4].reshape(B, nq, 4).contiguous(), ref.contiguous())
        hs = ops.layernorm(hidden.reshape(B * nq, d).contiguous(), *self.dec_norm).view(B, nq, d)
        return hs, ref

    @torch.inference_mode()
    def forward(self, images: torch.Tensor, input_ids: Sequence[int]):
        """images [B, H, W, 3] uint8 on the device."""
        B, H, W = int(images.shape[0]), int(images.shape[1]), int(images.shape[2])
        feats = self.backbone.forward_rows(images)
        return self.forward_features(feats, B, H, W, input_ids)
