"""Torch restatement of the reference's YOLOv7.predict (vlfm/vlm/yolov7.py:50-110 with yolov7's modules, non_max_suppression
and scale_coords), walking the same ``yolov7_weights.Layer`` records as the engine.

``forward(..., fused=False)`` runs every conv, BatchNorm and SiLU separately and applies ImplicitA / ImplicitM, so comparing it
with ``fused=True`` checks the fold.  ``round16=True`` rounds the fused weights and every stored activation to fp16 (what the
engine stores), in float64 otherwise: the difference from the float64 run is the drift that sets the GPU bars.
Suppression uses ``torchvision.ops.nms``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import cv2
import numpy as np
import torch
import torch.nn.functional as Fn
import torchvision

from vlfm_b200.vlm.yolov7_engine import IN_H, IN_W, area_tables
from vlfm_b200.vlm.yolov7_weights import Layer, fold, fold_detect


def area_resize(img: np.ndarray, OH: int = IN_H, OW: int = IN_W) -> np.ndarray:
    """cv2.resize(img, (OW, OH), INTER_AREA) for a downscale, in float32 in cv2's accumulation order (numpy: no FMA)."""
    H, W = img.shape[:2]
    yo, ys, yb = area_tables(H, OH)
    xo, xs, xa = area_tables(W, OW)
    src = img.astype(np.float32)
    out = np.empty((OH, OW, 3), np.uint8)
    # per destination column: the (source column, weight) entries, padded with weight 0 entries that add exact zeros
    kmax = int(np.max(np.diff(xo)))
    idx = np.zeros((OW, kmax), np.int64)
    wts = np.zeros((OW, kmax), np.float32)
    for d in range(OW):
        n = xo[d + 1] - xo[d]
        idx[d, :n], wts[d, :n] = xs[xo[d]:xo[d + 1]], xa[xo[d]:xo[d + 1]]
    for dy in range(OH):
        s = None
        for j in range(yo[dy], yo[dy + 1]):
            row = src[ys[j]]
            buf = np.zeros((OW, 3), np.float32)
            for k in range(kmax):
                buf = buf + row[idx[:, k]] * wts[:, k:k + 1]
            s = yb[j] * buf if s is None else s + yb[j] * buf
        out[dy] = np.clip(np.rint(s), 0, 255).astype(np.uint8)
    return out


def preprocess(image: np.ndarray, use_cv2: bool = True) -> torch.Tensor:
    """[1, 3, 448, 640] float64 of fp16(x / 255) (letterbox: the identity at 448 x 640; no channel swap)."""
    img = cv2.resize(image, (IN_W, IN_H), interpolation=cv2.INTER_AREA) if use_cv2 else area_resize(image)
    t = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).half() / 255.0
    return t.double()[None]


def _silu(x):
    return x / (1 + torch.exp(-x))


_FOLDED: dict = {}        # (id(conv), dtype, device, round16) -> (conv, folded weight, bias); the conv is kept so its id stays its own


def forward(layers: List[Layer], x: torch.Tensor, fused: bool = True, round16: bool = False,
            dtype=torch.float64, taps: Optional[dict] = None) -> List[torch.Tensor]:
    """x [B, 3, 448, 640] -> the head conv outputs per level [B, na*no, ny, nx] (after ImplicitM), NCHW in ``dtype`` (float16:
    the reference's own fp16 model on cuDNN, for timing).  ``taps``, when given, receives every layer's output by index."""
    dt, dev = dtype, x.device
    x = x.to(dt)
    r16 = (lambda t: t.half().to(dt)) if round16 else (lambda t: t)

    def conv(c, t):
        if fused or c.bn is None:
            key = (id(c), dt, str(dev), round16)
            if key not in _FOLDED:
                w, b = fold(c)
                _FOLDED[key] = (c, r16(w.to(dev, dt)), b)
            _, w, b = _FOLDED[key]
            y = Fn.conv2d(t, w, b.to(dev, dt), stride=c.stride, padding=c.k // 2)
        else:
            y = Fn.conv2d(t, c.w.to(dev, dt), None if c.b is None else c.b.to(dev, dt), stride=c.stride, padding=c.k // 2)
            g, beta, mean, var, eps = (v.to(dev, dt).view(1, -1, 1, 1) if isinstance(v, torch.Tensor) else v for v in c.bn)
            y = (y - mean) / torch.sqrt(var + eps) * g + beta
        return r16(_silu(y) if c.act else y)

    y = {-1: x}
    heads = []
    for l in layers:
        ins = [y[j] for j in l.f]
        t = l.type
        if t == "ReOrg":
            a = ins[0]
            out = torch.cat([a[..., ::2, ::2], a[..., 1::2, ::2], a[..., ::2, 1::2], a[..., 1::2, 1::2]], 1)
        elif t == "Conv":
            out = conv(l.convs[""], ins[0])
        elif t == "DownC":
            c = l.convs
            out = torch.cat((conv(c["cv2"], conv(c["cv1"], ins[0])), conv(c["cv3"], Fn.max_pool2d(ins[0], 2, 2))), 1)
        elif t == "SPPCSPC":
            c = l.convs
            x1 = conv(c["cv4"], conv(c["cv3"], conv(c["cv1"], ins[0])))
            pools = [Fn.max_pool2d(x1, k, 1, k // 2) for k in (5, 9, 13)]
            y1 = conv(c["cv6"], conv(c["cv5"], torch.cat([x1] + pools, 1)))
            out = conv(c["cv7"], torch.cat((y1, conv(c["cv2"], ins[0])), 1))
        elif t == "Upsample":
            out = Fn.interpolate(ins[0], scale_factor=2, mode="nearest")
        elif t == "Concat":
            out = torch.cat(ins, 1)
        elif t == "Shortcut":
            out = r16(ins[0] + ins[1])
        else:
            for k, a in enumerate(ins):
                c = l.convs[f"m{k}"]
                ia, im = l.extra["ia"][k].to(dev, dt), l.extra["im"][k].to(dev, dt)
                if fused:
                    w, b = fold_detect(c, l.extra["ia"][k], l.extra["im"][k])
                    h = Fn.conv2d(a, r16(w.to(dev, dt)), b.to(dev, dt))
                else:
                    h = Fn.conv2d(a + ia, c.w.to(dev, dt), c.b.to(dev, dt)) * im
                heads.append(r16(h))
            break
        y[l.i] = out
        if taps is not None:
            taps[l.i] = out
    return heads


def decode(heads: List[torch.Tensor], layers: List[Layer]) -> torch.Tensor:
    """IDetect's inference decode -> [B, rows, no] (x, y, w, h, obj, cls...) in the heads' dtype."""
    det = layers[-1]
    anchors = det.extra["anchors"]
    z = []
    for k, h in enumerate(heads):
        B, _, ny, nx = h.shape
        na = anchors.shape[1]
        v = h.view(B, na, -1, ny, nx).permute(0, 1, 3, 4, 2).sigmoid()
        yv, xv = torch.meshgrid(torch.arange(ny, device=h.device), torch.arange(nx, device=h.device), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).to(h.dtype)
        ag = anchors[k].to(h.device, h.dtype).view(1, na, 1, 1, 2)
        xy = (v[..., 0:2] * 2.0 - 0.5 + grid) * det.extra["strides"][k]
        wh = (v[..., 2:4] * 2) ** 2 * ag
        z.append(torch.cat((xy, wh, v[..., 4:]), -1).view(B, -1, v.shape[-1]))
    return torch.cat(z, 1)


def nms(pred: torch.Tensor, conf_thres: float = 0.25, iou_thres: float = 0.45, classes: Optional[Sequence[int]] = None,
        agnostic: bool = False, max_det: int = 300) -> List[torch.Tensor]:
    """yolov7's non_max_suppression (multi_label off) -> per frame [n, 7] (x1, y1, x2, y2, conf, class, row), float32 boxes
    and scores as the engine computes them; candidate order is row order, ties keep it (a stable descending sort)."""
    out = []
    for x in pred:
        rows = torch.arange(x.shape[0], device=x.device)
        keep = x[:, 4] > conf_thres
        x, rows = x[keep].clone(), rows[keep]
        x[:, 5:] *= x[:, 4:5]
        box = torch.stack((x[:, 0] - x[:, 2] / 2, x[:, 1] - x[:, 3] / 2, x[:, 0] + x[:, 2] / 2, x[:, 1] + x[:, 3] / 2), 1)
        conf, j = x[:, 5:].max(1, keepdim=True)
        d = torch.cat((box, conf, j.to(x.dtype), rows[:, None].to(x.dtype)), 1)[conf.view(-1) > conf_thres]
        if classes is not None:
            d = d[(d[:, 5:6] == torch.tensor(classes, device=d.device, dtype=d.dtype)).any(1)]
        d = d.float()
        order = torch.sort(-d[:, 4], stable=True).indices          # descending score, row order on ties
        d = d[order]
        c = d[:, 5:6] * (0 if agnostic else 4096)
        i = torchvision.ops.nms((d[:, :4] + c).cpu(), d[:, 4].cpu(), iou_thres)[:max_det]
        out.append(d[i.to(d.device)])
    return out


def scale_boxes(det: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """scale_coords((448, 640), boxes, (H, W)) + clip + round + normalise, float64 -> [n, 4]."""
    b = det[:, :4].double().clone()
    gain = min(IN_H / H, IN_W / W)
    pad = (IN_W - W * gain) / 2, (IN_H - H * gain) / 2
    b[:, [0, 2]] -= pad[0]
    b[:, [1, 3]] -= pad[1]
    b /= gain
    b[:, [0, 2]] = b[:, [0, 2]].clamp(0, W)
    b[:, [1, 3]] = b[:, [1, 3]].clamp(0, H)
    b = b.round()
    b[:, [0, 2]] /= W
    b[:, [1, 3]] /= H
    return b


def detect(layers: List[Layer], image: np.ndarray, device="cpu", **kw) -> Tuple[torch.Tensor, torch.Tensor, List[torch.Tensor]]:
    """One frame -> (kept rows [n, 7], normalised boxes [n, 4], heads) in float64."""
    heads = forward(layers, preprocess(image).to(device))
    d = nms(decode(heads, layers), **kw)[0]
    return d, scale_boxes(d, *image.shape[:2]), heads
