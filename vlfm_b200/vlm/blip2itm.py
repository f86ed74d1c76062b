"""In-process GPU BLIP-2 image-text matching behind the reference's class surface.

Reference: vlfm/vlm/blip2itm.py -- ``BLIP2ITM.__init__`` :20-35, ``cosine`` :37-54,
``BLIP2ITMClient`` :57-64.  The client twin keeps the constructor/method signature the
policies use (itm_policy.py:48, frontier_map.py:20) but calls the engine directly: no
Flask, no JPEG, no lock files (server_wrapper.py is transport only and is not rebuilt).
"""
from __future__ import annotations

import os
import re
import zlib
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import torch

from .blip2_config import Blip2Dims, random_state_dict
from .blip2_engine import Blip2ITCEngine


def pre_caption(caption: str, max_words: int = 50) -> str:
    """lavis BlipCaptionProcessor (text_processors["eval"], blip2itm.py:50)."""
    caption = re.sub(r"([.!\"()*#:;~])", " ", caption.lower())
    caption = re.sub(r"\s{2,}", " ", caption).rstrip("\n").strip(" ")
    words = caption.split(" ")
    return " ".join(words[:max_words]) if len(words) > max_words else caption


class WordPieceTokenizer:
    """bert-base-uncased WordPiece (greedy longest-match-first) from a vocab.txt."""

    def __init__(self, vocab_path: str, max_len: int = 32):
        with open(vocab_path, encoding="utf-8") as fh:
            self.vocab = {tok.rstrip("\n"): i for i, tok in enumerate(fh)}
        self.max_len = max_len

    def __call__(self, text: str) -> List[int]:
        ids = [self.vocab["[CLS]"]]
        for word in re.findall(r"\w+|[^\w\s]", text.lower()):
            start, pieces = 0, []
            while start < len(word):
                end = len(word)
                cur = None
                while start < end:
                    sub = ("##" if start > 0 else "") + word[start:end]
                    if sub in self.vocab:
                        cur = sub
                        break
                    end -= 1
                if cur is None:
                    pieces = ["[UNK]"]
                    break
                pieces.append(cur)
                start = end
            ids.extend(self.vocab[p] for p in pieces)
        ids = ids[: self.max_len - 1]
        return ids + [self.vocab["[SEP]"]]


class WordPieceCaptionTokenizer(WordPieceTokenizer):
    """encode / decode pair GroundingDINO.predict needs (bert-base-uncased ids <-> words)."""

    def __init__(self, vocab_path: str, max_len: int = 256):
        super().__init__(vocab_path, max_len)
        self.inv = {i: t for t, i in self.vocab.items()}

    def encode(self, caption: str) -> List[int]:
        return self(caption)

    def decode(self, ids: Sequence[int]) -> str:
        out = ""
        for i in ids:
            t = self.inv.get(int(i), "[UNK]")
            if t in ("[CLS]", "[SEP]", "[PAD]"):
                continue
            out = out + t[2:] if t.startswith("##") else (out + " " + t if out else t)
        return out


class HashTokenizer:
    """SYNTHETIC stand-in used when no bert-base-uncased vocab is on disk (there is none
    offline): [CLS]=101, one crc32-hashed id per word, [SEP]=102.  Scores are then only
    meaningful for synthetic weights."""

    def __init__(self, vocab: int, max_len: int = 32):
        self.vocab, self.max_len = vocab, max_len

    def __call__(self, text: str) -> List[int]:
        lo = min(1000, self.vocab // 2)
        ids = [101 % self.vocab] + [lo + zlib.crc32(w.encode()) % (self.vocab - lo) for w in text.split(" ") if w]
        return ids[: self.max_len - 1] + [102 % self.vocab]


class BLIP2ITM:
    """BLIP 2 Image-Text Matching model (ITC head), hand-written sm_90a forward."""

    def __init__(self, name: str = "blip2_image_text_matching", model_type: str = "pretrain", device: Optional[Any] = None,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, dims: Optional[Blip2Dims] = None,
                 tokenizer: Optional[Any] = None, max_batch: int = 1, seed: int = 0, synthetic: bool = False) -> None:
        """``name`` / ``model_type`` are lavis registry keys (blip2itm.py:29-34); the only pair this engine implements is the
        reference's default ("blip2_image_text_matching", "pretrain") = ViT-g/14 + 12-layer Q-Former, anything else raises.
        Weights: ``state_dict`` (HF ``Blip2ForImageTextRetrieval`` names or lavis names -- converted by
        ``blip2_weights.convert_lavis_state_dict``) or the file ``VLFM_BLIP2_WEIGHTS``.  Without either the constructor
        RAISES unless ``synthetic=True`` (seeded random weights: tests / benchmarks only)."""
        if (name, model_type) != ("blip2_image_text_matching", "pretrain"):
            raise ValueError(f"BLIP2ITM: only ('blip2_image_text_matching', 'pretrain') is implemented, got ({name!r}, {model_type!r})")
        if device is None:
            device = torch.device("cuda")
        self.device = device
        self.dims = dims or Blip2Dims()
        from .blip2_weights import load_checkpoint

        real = False
        if state_dict is None:
            path = os.environ.get("VLFM_BLIP2_WEIGHTS", "")
            if path:
                state_dict = load_checkpoint(path, self.dims)
                real = True
            elif synthetic:   # no checkpoint offline: seeded synthetic weights of the right architecture
                state_dict = random_state_dict(self.dims, seed)
            else:
                raise FileNotFoundError("BLIP2ITM: no checkpoint configured (VLFM_BLIP2_WEIGHTS unset, no state_dict). "
                                        "Pass synthetic=True to run on seeded random weights (tests / benchmarks only).")
        if tokenizer is None:
            vocab = os.environ.get("VLFM_BERT_VOCAB", "")
            if vocab:
                tokenizer = WordPieceTokenizer(vocab)
            elif real:
                raise FileNotFoundError("BLIP2ITM: real weights need the bert-base-uncased vocabulary: set VLFM_BERT_VOCAB=<vocab.txt> "
                                        "or pass tokenizer=")
            else:
                tokenizer = HashTokenizer(self.dims.vocab)
        self.tokenizer = tokenizer
        self.engine = Blip2ITCEngine(self.dims, state_dict, device=device, max_batch=max_batch)
        self._text_cache: Dict[str, torch.Tensor] = {}
        self._cur_text: Optional[str] = None
        self._pin: Optional[torch.Tensor] = None
        self._dev_img: Optional[torch.Tensor] = None

    def _use_text(self, txt: str) -> None:
        if txt != self._cur_text:
            if txt not in self._text_cache:
                self._text_cache[txt] = self.engine.encode_text(self.tokenizer(pre_caption(txt)))
            self.engine.set_text(self._text_cache[txt])
            self._cur_text = txt

    def cosine_device(self, images: torch.Tensor, txt: str) -> torch.Tensor:
        """images [B,H,W,3] uint8 already in HBM -> cosines [B] (device)."""
        self._use_text(txt)
        return self.engine.forward(images)

    def cosine(self, image: np.ndarray, txt: str) -> float:
        """blip2itm.py:37-54: host uint8 RGB frame + prompt -> Python float."""
        self._use_text(txt)
        image = np.ascontiguousarray(image, dtype=np.uint8)
        if self._pin is None or self._pin.shape[1:] != image.shape:
            self._pin = torch.empty((1,) + image.shape, dtype=torch.uint8).pin_memory()
            self._dev_img = torch.empty((1,) + image.shape, dtype=torch.uint8, device=self.device)
        src = torch.from_numpy(image)
        if src.is_pinned():          # caller's frame already lives in page-locked memory: DMA straight from it (the call syncs below)
            self._dev_img.copy_(src[None], non_blocking=True)
        else:
            self._pin[0].numpy()[...] = image
            self._dev_img.copy_(self._pin, non_blocking=True)
        return float(self.engine.forward(self._dev_img)[0].item())  # .item(): D2H sync, as in the reference


_SHARED: Dict[str, BLIP2ITM] = {}


class BLIP2ITMClient:
    """Same call signature as the HTTP client (blip2itm.py:57-64); ``port`` is accepted and
    ignored -- the model lives in this process."""

    def __init__(self, port: int = 12182, model: Optional[BLIP2ITM] = None):
        if model is None:
            if "default" not in _SHARED:
                _SHARED["default"] = BLIP2ITM(synthetic=os.environ.get("VLFM_SYNTHETIC_WEIGHTS", "") == "1")
            model = _SHARED["default"]
        self.model = model

    def cosine(self, image: np.ndarray, txt: str) -> float:
        return self.model.cosine(image, txt)
