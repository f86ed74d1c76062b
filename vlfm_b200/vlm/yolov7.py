"""In-process GPU YOLOv7-E6E behind the reference's class surface (vlfm/vlm/yolov7.py).

``YOLOv7.predict`` runs the reference's whole pipeline on the device as one CUDA graph per (batch, frame size): cv2's
INTER_AREA resize to 640 x 448, the letterbox (the identity at 640 x 448: both sides are multiples of the stride 64 and the
long side is already 640, so it is not built), /255 in fp16, the fp16 network with the BatchNorms and implicit layers folded,
the decode, yolov7's ``non_max_suppression`` (class-offset greedy NMS, at most 300 kept) and ``scale_coords``.  The boxes keep
the reference's ``scale_coords`` quirk: it treats the 448 x 640 input as a letterbox of the frame, so y maps exactly and x is
stretched about the centre (by 7 % for 640 x 480 frames).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .coco_classes import COCO_CLASSES
from .detections import ObjectDetections
from .yolov7_config import synthetic_layers
from .yolov7_engine import YoloEngine
from .yolov7_weights import Layer, load_checkpoint


class YOLOv7:
    def __init__(self, weights: Optional[str] = None, image_size: int = 640, half_precision: bool = True, *,
                 layers: Optional[List[Layer]] = None, synthetic: bool = False, seed: int = 0, device=None) -> None:
        """Weights: ``layers`` (records of ``yolov7_weights``), else the checkpoint ``weights`` or ``VLFM_YOLOV7_WEIGHTS``.  Without
        any the constructor RAISES unless ``synthetic=True`` (seeded random E6E weights: tests / benchmarks only).  Only
        ``image_size=640`` and fp16 (``half_precision=True``) are implemented."""
        if image_size != 640:
            raise NotImplementedError(f"YOLOv7: only image_size=640 is implemented, got {image_size}")
        if not half_precision:
            raise NotImplementedError("YOLOv7: only half_precision=True is implemented (there is no fp32 path)")
        if layers is None:
            path = weights or os.environ.get("VLFM_YOLOV7_WEIGHTS", "")
            if path:
                layers = load_checkpoint(path)
            elif synthetic:
                layers = synthetic_layers(seed)
            else:
                raise FileNotFoundError("YOLOv7: no weights configured (weights / VLFM_YOLOV7_WEIGHTS unset).  Pass synthetic=True to "
                                        "run on seeded random weights (tests / benchmarks only).")
        self.device = torch.device(device or "cuda")
        self.engine = YoloEngine(layers, self.device)
        self._pin: Optional[torch.Tensor] = None
        self._dev: Optional[torch.Tensor] = None

    def _set(self, conf_thres: float, iou_thres: float, classes, agnostic_nms: bool) -> None:
        if classes is not None:
            classes = list(classes) if isinstance(classes, (list, tuple, np.ndarray, torch.Tensor)) else [classes]
            if any(isinstance(c, str) for c in classes):
                raise TypeError("YOLOv7: `classes` are class indices (as in yolov7's non_max_suppression), not names")
            classes = [int(c) for c in classes]
        self.engine.set_params(conf_thres, iou_thres, classes, agnostic_nms)

    def predict_device(self, images: torch.Tensor, conf_thres: float = 0.25, iou_thres: float = 0.45, classes: Optional[Sequence[int]] = None,
                       agnostic_nms: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """images [B,H,W,3] uint8 RGB (device) -> (boxes [B,300,4] normalised xyxy, scores [B,300], classes [B,300] int32,
        counts [B]) on the device; row i of frame b is valid for i < counts[b] (the rest: 0 / class -1)."""
        self._set(conf_thres, iou_thres, classes, agnostic_nms)
        return tuple(t.clone() for t in self.engine.run(images.to(self.device)))

    def predict(self, image: np.ndarray, conf_thres: float = 0.25, iou_thres: float = 0.45, classes: Optional[Sequence[int]] = None,
                agnostic_nms: bool = False) -> ObjectDetections:
        """yolov7.py:50-110 for one RGB uint8 frame [H, W, 3] (H >= 448, W >= 640).  Boxes and logits are float32 CPU tensors."""
        self._set(conf_thres, iou_thres, classes, agnostic_nms)
        img = np.ascontiguousarray(image, dtype=np.uint8)
        if img.ndim != 3 or img.shape[2] != 3:
            raise ValueError(f"YOLOv7: expected an RGB uint8 frame [H, W, 3], got shape {img.shape}")
        if self._pin is None or self._pin.shape[1:] != img.shape:
            self._pin = torch.empty((1,) + img.shape, dtype=torch.uint8).pin_memory()
            self._dev = torch.empty((1,) + img.shape, dtype=torch.uint8, device=self.device)
        self._pin[0].numpy()[...] = img
        self._dev.copy_(self._pin, non_blocking=True)
        boxes, scores, cls, counts = self.engine.run(self._dev)
        n = int(counts[0].item())
        b, s, c = boxes[0, :n].cpu(), scores[0, :n].cpu(), cls[0, :n].cpu().tolist()
        return ObjectDetections(b, s, [COCO_CLASSES[j] for j in c], image_source=image, fmt="xyxy")


_SHARED: Dict[str, YOLOv7] = {}


class YOLOv7Client:
    """Same call signature as the HTTP client (yolov7.py:113-121); ``port`` is accepted and ignored -- the model lives in this
    process, shared by every client (seeded synthetic weights when ``VLFM_SYNTHETIC_WEIGHTS=1``).  Returns float32 CPU tensors,
    as ``ObjectDetections.from_json`` does."""

    def __init__(self, port: int = 12184, model: Optional[YOLOv7] = None):
        if model is None:
            if "default" not in _SHARED:
                _SHARED["default"] = YOLOv7(synthetic=os.environ.get("VLFM_SYNTHETIC_WEIGHTS", "") == "1")
            model = _SHARED["default"]
        self.model = model

    def predict(self, image_numpy: np.ndarray) -> ObjectDetections:
        return self.model.predict(image_numpy)
