"""In-process GPU MobileSAM behind the reference's class surface (vlfm/vlm/sam.py).

``MobileSAM.segment_bbox`` in the reference runs ``predictor.set_image`` on every call, so the policy's per-detection loop
(``BaseObjectNavPolicy._update_object_map``) pays one 1024 x 1024 encoder pass per detection.  Here the image embedding of the
last host frame is kept: a call on the same unchanged frame object runs the decoder only, and ``segment_bboxes`` serves N boxes
from one encoder pass and one decoder launch sequence.
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .sam_config import VIT_T, SamDims, random_state_dict
from .sam_engine import MobileSamEngine
from .sam_weights import convert_state_dict, load_checkpoint


class MobileSAM:
    def __init__(self, sam_checkpoint: Optional[str] = None, model_type: str = "vit_t", device: Optional[Any] = None, *,
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, dims: Optional[SamDims] = None, max_batch: int = 1,
                 seed: int = 0, synthetic: bool = False) -> None:
        """Weights: ``state_dict`` (mobile_sam names), else the file ``sam_checkpoint`` or ``MOBILE_SAM_CHECKPOINT``.  Without
        any the constructor RAISES unless ``synthetic=True`` (seeded random weights: tests / benchmarks only).  Only
        ``model_type="vit_t"`` (TinyViT-5M) is implemented."""
        if model_type != "vit_t":
            raise ValueError(f"MobileSAM: only model_type='vit_t' is implemented, got {model_type!r}")
        if device is None:
            device = torch.device("cuda")
        self.device = torch.device(device)
        self.dims = dims or VIT_T
        if state_dict is not None:
            w = convert_state_dict(state_dict, self.dims)
        else:
            path = sam_checkpoint or os.environ.get("MOBILE_SAM_CHECKPOINT", "")
            if path:
                w = load_checkpoint(path, self.dims)
            elif synthetic:
                w = convert_state_dict(random_state_dict(self.dims, seed), self.dims)
            else:
                raise FileNotFoundError("MobileSAM: no checkpoint configured (sam_checkpoint / MOBILE_SAM_CHECKPOINT unset, no "
                                        "state_dict).  Pass synthetic=True to run on seeded random weights (tests / benchmarks only).")
        self.engine = MobileSamEngine(self.dims, w, device=self.device, max_batch=max_batch)
        self._pin: Optional[torch.Tensor] = None
        self._dev_img: Optional[torch.Tensor] = None
        # the host frame of the last host-side encode: (caller's object, shape, dtype, engine generation, the bytes it saw)
        self._frame: Optional[Tuple[np.ndarray, Tuple[int, ...], np.dtype, int, np.ndarray]] = None

    def _cached(self, image: Any) -> bool:
        """True when the engine still holds the embedding of ``image``: the same object as the last host-side encode's frame,
        same shape and dtype, the same bytes (callers may refill one buffer in place) and no encode since (BLIP2ITM's rule)."""
        f = self._frame
        if f is None or image is not f[0] or image.shape != f[1] or image.dtype != f[2] or self.engine.generation != f[3]:
            return False
        a, b = np.ascontiguousarray(image, dtype=np.uint8), f[4]
        if a.nbytes % 8 == 0:
            a, b = a.reshape(-1).view(np.uint64), b.reshape(-1).view(np.uint64)
        return bool(np.array_equal(a, b))

    def _encode_host(self, image: np.ndarray) -> None:
        """One H2D of a host frame and one encoder pass into frame slot 0; records the frame for ``_cached``."""
        arg, self._frame = image, None
        image = np.ascontiguousarray(image, dtype=np.uint8)
        if image.ndim != 3 or image.shape[2] != 3:
            raise ValueError(f"MobileSAM: expected an RGB uint8 frame [H, W, 3], got shape {image.shape}")
        if self._pin is None or self._pin.shape[1:] != image.shape:
            self._pin = torch.empty((1,) + image.shape, dtype=torch.uint8).pin_memory()
            self._dev_img = torch.empty((1,) + image.shape, dtype=torch.uint8, device=self.device)
        self._pin[0].numpy()[...] = image
        self._dev_img.copy_(self._pin, non_blocking=True)
        self.engine.encode(self._dev_img)
        if isinstance(arg, np.ndarray):
            self._frame = (arg, arg.shape, arg.dtype, self.engine.generation, self._pin[0].numpy())

    @staticmethod
    def _boxes(bboxes) -> np.ndarray:
        b = np.asarray(bboxes, dtype=np.float64)
        if b.ndim == 1:
            b = b[None]
        if b.ndim != 2 or b.shape[1] != 4:
            raise ValueError(f"MobileSAM: boxes must be [x1, y1, x2, y2] rows, got shape {b.shape}")
        return b

    def segment_bboxes(self, image: np.ndarray, bboxes: Sequence[Sequence[float]]) -> np.ndarray:
        """Host uint8 RGB frame + N boxes [x1, y1, x2, y2] (frame pixels, int or float) -> bool [N, H, W]: one encoder pass
        (none when ``image`` is the cached frame), one decoder launch sequence, one D2H.  Row i is bitwise equal to
        ``segment_bbox(image, bboxes[i])``."""
        b = self._boxes(bboxes)
        if not self._cached(image):
            self._encode_host(image)
        H, W = image.shape[:2]
        boxes = torch.from_numpy(b).to(self.device, non_blocking=False)
        frames = torch.zeros(b.shape[0], dtype=torch.int32, device=self.device)
        masks = self.engine.decode(boxes, frames, (H, W))
        return masks.cpu().numpy().astype(bool)

    def segment_bbox(self, image: np.ndarray, bbox: List[int]) -> np.ndarray:
        """sam.py:40-57: the object in ``bbox`` [x1, y1, x2, y2] as a bool mask [H, W] of the whole frame.  When ``image`` is
        the frame of the last host-side call (same object, unchanged bytes, no encode since), only the decoder runs."""
        return self.segment_bboxes(image, [bbox])[0]

    def segment_bboxes_device(self, images: torch.Tensor, boxes: torch.Tensor, frame_idx: torch.Tensor) -> torch.Tensor:
        """images [B,H,W,3] uint8 (device, B <= max_batch), boxes [M,4] (frame pixels), frame_idx [M] (index into images)
        -> uint8 [M,H,W] masks (device).  One encoder pass over the B frames, one decoder launch sequence for the M boxes.
        A frame index outside [0, B) gives an all-zero mask."""
        self._frame = None
        self.engine.encode(images)
        return self.engine.decode(boxes.to(self.device, torch.float64), frame_idx.to(self.device, torch.int32),
                                  (images.shape[1], images.shape[2]))


_SHARED: Dict[str, MobileSAM] = {}


class MobileSAMClient:
    """Same call signature as the HTTP client (sam.py:60-70); ``port`` is accepted and ignored -- the model lives in this
    process, shared by every client (seeded synthetic weights when ``VLFM_SYNTHETIC_WEIGHTS=1``)."""

    def __init__(self, port: int = 12183, model: Optional[MobileSAM] = None):
        if model is None:
            if "default" not in _SHARED:
                _SHARED["default"] = MobileSAM(synthetic=os.environ.get("VLFM_SYNTHETIC_WEIGHTS", "") == "1")
            model = _SHARED["default"]
        self.model = model

    def segment_bbox(self, image: np.ndarray, bbox: List[int]) -> np.ndarray:
        return self.model.segment_bbox(image, bbox)
