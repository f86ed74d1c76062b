"""GroundingDINO behind the reference's class surface (vlfm/vlm/grounding_dino.py:23-85).

The Swin-T backbone -- the dense contraction north_star names -- runs on the hand-written sm_90a kernels
(``SwinBackboneEngine``); every nn.Linear, the deformable encoder layers, the image<->text fusion layers and the decoder layers
run on the library too (``gdino_accel``: wgmma GEMM, fused multi-scale deformable sampling, bi-attention).  ``GdinoForward``
(``gdino_forward``) sequences them -- neck, encoder loop, proposal selection, decoder loop, heads -- over the weights of HF's
``GroundingDinoForObjectDetection`` (architecture-equivalent to groundingdino@eeba084); what is still PyTorch glue is listed in
DESIGN.md section 7.  Post-processing restates groundingdino.util.inference.predict.
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from ..utils.cuda_graph import GraphCache, default_use_graph
from .detections import ObjectDetections
from .gdino_accel import accelerate
from .gdino_forward import GdinoForward
from .gdino_ops import LibOps
from .swin_engine import SwinBackboneEngine

GROUNDING_DINO_CONFIG = "GroundingDINO/groundingdino/config/GroundingDINO_SwinT_OGC.py"
GROUNDING_DINO_WEIGHTS = "data/groundingdino_swint_ogc.pth"
CLASSES = "chair . person . dog ."  # grounding_dino.py:20
BACKBONE_PREFIX = "model.backbone.conv_encoder.model."
GRAPH_MAX_BATCH = 4


class SimpleCaptionTokenizer:
    """SYNTHETIC stand-in for bert-base-uncased (no vocab offline): [CLS]=101, '.'=1012, [SEP]=102,
    words -> stable ids in [2000, vocab).  decode() inverts it for the words it has seen."""

    def __init__(self, vocab: int = 30522):
        self.vocab = vocab
        self.words: Dict[int, str] = {}

    def encode(self, caption: str) -> List[int]:
        import zlib

        ids = [101]
        for tok in caption.replace(".", " . ").split():
            if tok == ".":
                ids.append(1012)
            else:
                i = 2000 + zlib.crc32(tok.encode()) % (self.vocab - 2000)
                self.words[i] = tok
                ids.append(i)
        return ids + [102]

    def decode(self, ids: List[int]) -> str:
        return " ".join("." if i == 1012 else self.words.get(i, "[UNK]") for i in ids if i not in (101, 102))


class GroundingDINO:
    def __init__(self, config_path: str = GROUNDING_DINO_CONFIG, weights_path: str = GROUNDING_DINO_WEIGHTS,
                 caption: str = CLASSES, box_threshold: float = 0.35, text_threshold: float = 0.25,
                 device: torch.device = torch.device("cuda"), state_dict: Optional[Dict[str, torch.Tensor]] = None,
                 tokenizer: Optional[Any] = None, seed: int = 0, synthetic: bool = False):
        """``weights_path`` (grounding_dino.py:33 ``load_model(config_path, weights_path)``) is honoured: a groundingdino
        ``.pth`` (original key names, converted by ``gdino_weights.convert_groundingdino_state_dict``) or an HF-layout
        state dict; ``VLFM_GDINO_WEIGHTS`` overrides it.  ``config_path`` selects nothing here: the only architecture built
        is GroundingDINO_SwinT_OGC (the reference's default and the one its weights file is for).  Without a checkpoint
        the constructor RAISES unless ``synthetic=True`` (seeded random weights: tests / benchmarks only) -- a detector
        that silently runs on random weights returns meaningless boxes."""
        from transformers import GroundingDinoConfig, GroundingDinoForObjectDetection

        from .gdino_weights import load_checkpoint

        cfg = GroundingDinoConfig()
        real = False          # weights read from a checkpoint file (then the real vocabulary is mandatory)
        if state_dict is None:
            path = os.environ.get("VLFM_GDINO_WEIGHTS", "") or (weights_path if weights_path and os.path.exists(weights_path) else "")
            if path:
                state_dict = load_checkpoint(path)
                real = True
            elif not synthetic:
                raise FileNotFoundError(
                    f"GroundingDINO: no checkpoint at weights_path={weights_path!r} and VLFM_GDINO_WEIGHTS is unset. "
                    "Pass synthetic=True to run on seeded random weights (tests / benchmarks only).")
        torch.manual_seed(seed)
        model = GroundingDinoForObjectDetection(cfg)
        if state_dict is not None:
            missing, unexpected = model.load_state_dict(state_dict, strict=False)
            missing = [k for k in missing if "position_ids" not in k]
            if missing or unexpected:      # a checkpoint that does not cover the model is an error, never a silent partial load
                raise KeyError(f"GroundingDINO checkpoint does not match the model: {len(missing)} missing keys (e.g. {missing[:4]}), "
                               f"{len(unexpected)} unexpected keys (e.g. {list(unexpected)[:4]})")
        sd = model.state_dict()
        self.device = device
        self.backbone = SwinBackboneEngine(sd, prefix=BACKBONE_PREFIX, embed_dim=cfg.backbone_config.embed_dim,
                                           depths=cfg.backbone_config.depths, heads=cfg.backbone_config.num_heads,
                                           out_stages=tuple(cfg.backbone_config.out_indices), eps=cfg.backbone_config.layer_norm_eps,
                                           device=device)
        # the engine above holds the Swin weights; HF's copy would only occupy the device twice (GdinoForward reads just the
        # backbone's position embedding)
        model.model.backbone.conv_encoder.model = torch.nn.Identity()
        self.model = model.to(device).eval()
        # encoder / decoder layers and every nn.Linear on the library's kernels
        self.accel = accelerate(self.model)
        # model-level sequencing (neck, encoder loop, proposal selection, decoder loop, heads)
        self.fwd = GdinoForward(self.model, LibOps(), self.backbone)
        self.caption = caption
        self.box_threshold = box_threshold
        self.text_threshold = text_threshold
        if tokenizer is None:
            vocab = os.environ.get("VLFM_BERT_VOCAB", "")
            if vocab:
                from .blip2itm import WordPieceCaptionTokenizer

                tokenizer = WordPieceCaptionTokenizer(vocab)
            elif real and not synthetic:
                raise FileNotFoundError("GroundingDINO: real weights need the bert-base-uncased vocabulary: set VLFM_BERT_VOCAB=<vocab.txt> "
                                        "or pass tokenizer= (the crc32 stand-in only makes sense with synthetic weights)")
            else:
                if not synthetic:
                    import warnings

                    warnings.warn("GroundingDINO: in-memory state_dict without tokenizer= / VLFM_BERT_VOCAB: using the crc32 stand-in "
                                  "tokenizer, which is only meaningful with synthetic weights")
                tokenizer = SimpleCaptionTokenizer(cfg.text_config.vocab_size)
        self.tokenizer = tokenizer
        self._pin: Optional[torch.Tensor] = None
        self._dev: Optional[torch.Tensor] = None
        self._pin_ev: Optional[torch.cuda.Event] = None
        self.use_graph = default_use_graph()
        self.graphs = GraphCache(max_keys=4)

    @torch.inference_mode()
    def raw_outputs_device(self, images: torch.Tensor, input_ids: List[int]):
        """images [B,H,W,3] uint8 on the device -> (sigmoid logits [B,900,256], boxes [B,900,4] cxcywh).

        Batches up to GRAPH_MAX_BATCH (the per-step policy call is batch 1) replay a CUDA graph of the whole detector per
        (batch, image size, caption) from their second call: the forward is launch-bound otherwise."""
        ids = [int(i) for i in input_ids]

        def run(img: torch.Tensor):
            logits, boxes = self.fwd.forward(img, ids)
            # a captured graph reads the cached shape / caption constants by address: returning them keeps them alive
            return logits, boxes, self.fwd.last

        b, h, w = images.shape[:3]
        logits, boxes, _ = self.graphs((int(b), int(h), int(w), tuple(ids)), self.use_graph and b <= GRAPH_MAX_BATCH, run, images)
        return logits, boxes

    def raw_outputs(self, image: np.ndarray, input_ids: List[int]):
        """-> (sigmoid logits [900,256], boxes [900,4] cxcywh) on the device."""
        image = np.ascontiguousarray(image, dtype=np.uint8)
        if self._pin_ev is not None:
            # the last call's copy out of the page-locked buffer is asynchronous: overwriting the buffer before it has executed
            # would hand that call this call's frame
            self._pin_ev.synchronize()
        if self._pin is None or self._pin.shape[1:] != image.shape:
            self._pin = torch.empty((1,) + image.shape, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty((1,) + image.shape, dtype=torch.uint8, device=self.device)
        self._pin[0].numpy()[...] = image
        self._dev.copy_(self._pin, non_blocking=True)
        self._pin_ev = torch.cuda.Event()
        self._pin_ev.record()
        logits, boxes = self.raw_outputs_device(self._dev, input_ids)
        return logits[0], boxes[0]

    def predict(self, image: np.ndarray, caption: Optional[str] = None) -> ObjectDetections:
        """grounding_dino.py:38-74."""
        caption_to_use = self.caption if caption is None else caption
        text = caption_to_use.lower().strip()
        if not text.endswith("."):
            text = text + "."
        ids = self.tokenizer.encode(text)
        logits, boxes = self.raw_outputs(image, ids)
        logits, boxes = logits.cpu(), boxes.cpu()
        keep = logits.max(dim=1)[0] > self.box_threshold
        logits, boxes = logits[keep], boxes[keep]
        phrases = []
        for row in logits:
            pos = row > self.text_threshold
            pos[0] = False
            pos[len(ids) - 1 :] = False
            phrases.append(self.tokenizer.decode([ids[i] for i in pos.nonzero(as_tuple=True)[0].tolist()]).replace(".", "").strip())
        det = ObjectDetections(boxes, logits.max(dim=1)[0], phrases, image_source=image)
        classes = caption_to_use[: -len(" .")].split(" . ")
        det.filter_by_class(classes)
        return det


_SHARED: Dict[str, GroundingDINO] = {}


class GroundingDINOClient:
    """Same signature as the HTTP client (grounding_dino.py:77-85); in-process."""

    def __init__(self, port: int = 12181, model: Optional[GroundingDINO] = None):
        if model is None:
            if "default" not in _SHARED:
                _SHARED["default"] = GroundingDINO(synthetic=os.environ.get("VLFM_SYNTHETIC_WEIGHTS", "") == "1")
            model = _SHARED["default"]
        self.model = model

    def predict(self, image_numpy: np.ndarray, caption: Optional[str] = "") -> ObjectDetections:
        return self.model.predict(image_numpy, caption=caption if caption else None)
