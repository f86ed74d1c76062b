"""YOLOv7-E6E's layer table (restating yolov7's public cfg/deploy/yolov7-e6e.yaml, with the training config's IAuxDetect head of
the released checkpoint) and seeded synthetic weights for it.  A real checkpoint's own module tree always overrides this table.

Each row is (from, module, args) as in the yaml; ``synthetic_layers`` turns the table into unfused ``yolov7_weights.Layer`` records.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import numpy as np
import torch

from .yolov7_weights import ConvBN, Layer, prune, resolve

NC = 80
STRIDES = (8, 16, 32, 64)
ANCHORS = (((19, 27), (44, 40), (38, 94)), ((96, 68), (86, 152), (180, 137)), ((140, 301), (303, 264), (238, 542)),
           ((436, 615), (739, 380), (925, 792)))


def _eelan(t: list, c: int, c3: int, cout: int, cat: list) -> None:
    """Two ELAN blocks on the same input (the row before), summed by a Shortcut."""
    for rep in range(2):
        t.append((-1 if rep == 0 else -11, "Conv", (c, 1, 1)))
        t.append((-2 if rep == 0 else -12, "Conv", (c, 1, 1)))
        t.extend([(-1, "Conv", (c3, 3, 1))] * 6)
        t.append((cat, "Concat", ()))
        t.append((-1, "Conv", (cout, 1, 1)))
    t.append(([-1, -11], "Shortcut", ()))


def e6e_table(div: int = 1) -> List[Tuple[object, str, tuple]]:
    """The table; ``div`` > 1 divides every width (rounded up to a multiple of 8), for small test networks."""
    t = _e6e_rows()
    if div == 1:
        return t
    w = lambda c: max(8, -(-(c // div) // 8) * 8)
    return [(f, m, (w(a[0]),) + tuple(a[1:]) if m in ("Conv", "DownC", "SPPCSPC") else a) for f, m, a in t]


def _e6e_rows() -> List[Tuple[object, str, tuple]]:
    back, head = [-1, -3, -5, -7, -8], [-1, -2, -3, -4, -5, -6, -7, -8]
    t: list = [(-1, "ReOrg", ()), (-1, "Conv", (80, 3, 1))]
    for cout, c in ((160, 64), (320, 128), (640, 256), (960, 384), (1280, 512)):      # P2 .. P6
        t.append((-1, "DownC", (cout,)))
        _eelan(t, c, c, cout, back)
    t.append((-1, "SPPCSPC", (640,)))                                                    # 112
    for cu, c, c3, route in ((480, 384, 192, 89), (320, 256, 128, 67), (160, 128, 64, 45)):
        t += [(-1, "Conv", (cu, 1, 1)), (-1, "Upsample", ()), (route, "Conv", (cu, 1, 1)), ([-1, -2], "Concat", ())]
        _eelan(t, c, c3, cu, head)
    for cd, c, c3, route in ((320, 256, 128, 162), (480, 384, 192, 137), (640, 512, 256, 112)):
        t += [(-1, "DownC", (cd,)), ([-1, route], "Concat", ())]
        _eelan(t, c, c3, cd, head)
    for src, c in ((187, 320), (210, 640), (233, 960), (256, 1280), (186, 320), (161, 640), (136, 960), (112, 1280)):
        t.append((src, "Conv", (c, 3, 1)))                                               # 257-260 main, 261-264 aux
    t.append((list(range(257, 265)), "IAuxDetect", (NC,)))                               # 265
    assert len(t) == 266
    return t


def out_channels(table) -> List[int]:
    """Output channels of every row (ReOrg of an RGB input: 12)."""
    ch: List[int] = []
    for i, (f, mod, args) in enumerate(table):
        src = resolve(i, f)
        cin = [ch[j] if j >= 0 else 3 for j in src]
        if mod == "ReOrg":
            ch.append(4 * cin[0])
        elif mod in ("Conv", "DownC", "SPPCSPC"):
            ch.append(args[0])
        elif mod == "Concat":
            ch.append(sum(cin))
        elif mod in ("Shortcut", "Upsample"):
            ch.append(cin[0])
        else:
            ch.append(0)
    return ch


def _conv_shapes(table) -> List[Tuple[int, str, int, int, int, int]]:
    """(layer, name, cout, cin, k, stride) of every conv of the table, head convs last (cout = 3 * 85, k = 1)."""
    ch = out_channels(table)
    out = []
    for i, (f, mod, args) in enumerate(table):
        src = resolve(i, f)
        c1 = ch[src[0]] if src[0] >= 0 else 3
        if mod == "Conv":
            out.append((i, "", args[0], c1, args[1], args[2]))
        elif mod == "DownC":
            out += [(i, "cv1", c1, c1, 1, 1), (i, "cv2", args[0] // 2, c1, 3, 2), (i, "cv3", args[0] // 2, c1, 1, 1)]
        elif mod == "SPPCSPC":
            c_ = args[0]
            out += [(i, "cv1", c_, c1, 1, 1), (i, "cv2", c_, c1, 1, 1), (i, "cv3", c_, c_, 3, 1), (i, "cv4", c_, c_, 1, 1),
                    (i, "cv5", c_, 4 * c_, 1, 1), (i, "cv6", c_, c_, 3, 1), (i, "cv7", args[0], 2 * c_, 1, 1)]
        elif mod == "IAuxDetect":
            out += [(i, f"m{k}", 3 * (NC + 5), ch[j], 1, 1) for k, j in enumerate(src[:4])]
    return out


def cost(H: int = 448, W: int = 640, pruned: bool = True) -> Tuple[int, float]:
    """(parameters, GFLOP of one H x W frame, 2 per multiply-add) of the fused network; ``pruned`` counts only what the engine runs."""
    table = e6e_table()
    keep = {l.i for l in prune(_skeleton(table))} if pruned else set(range(len(table)))
    params, flop = 0, 0.0
    hw = []                                   # output size of every row
    for i, (f, mod, args) in enumerate(table):
        src = resolve(i, f)
        h, w = hw[src[0]] if src[0] >= 0 else (H, W)
        if mod in ("ReOrg", "DownC"):
            h, w = h // 2, w // 2
        elif mod == "Upsample":
            h, w = 2 * h, 2 * w
        hw.append((h, w))
    for i, name, co, ci, k, s in _conv_shapes(table):
        if i not in keep:
            continue
        h, w = hw[i]
        if table[i][1] == "DownC" and name == "cv1":          # runs before the stride-2 conv and the pool
            h, w = hw[resolve(i, table[i][0])[0]]
        params += co * ci * k * k + co
        flop += 2.0 * co * ci * k * k * h * w
    return params, flop / 1e9


def _skeleton(table) -> List[Layer]:
    ls = [Layer(i, resolve(i, f), mod) for i, (f, mod, _) in enumerate(table)]
    ls[-1].type, ls[-1].f = "Detect", ls[-1].f[:4]
    return ls


def synthetic_layers(seed: int = 0, table=None, head_std: float = 4.0) -> List[Layer]:
    """Seeded weights (numpy PCG64) for the table, unfused and rounded to fp16 as in a stripped release.  BatchNorms are near the
    identity; each conv's weights are N(0, 1) scaled, in a float32 calibration pass over one seeded uniform-noise 128 x 192 input,
    so that its pre-BatchNorm output has unit RMS: the post-SiLU RMS of every layer stays O(1) over the ~100 layers of the deepest
    path for area-downscaled frames (a fixed gain either vanishes or overflows fp16 there).  Random weights are far more sensitive
    to their input than trained ones: unfiltered full-band pixel noise at 448 x 640 (no downscale) overflows fp16 in the P6 head.  The head convs are scaled so that their outputs vary with RMS ``head_std``
    around yolov7's _initialize_biases priors (objectness log(8 / (640 / s)^2), classes log(0.6 / (nc - 0.99))): the candidate
    set is sparse, as with a trained model.  ImplicitA ~ N(0, 0.02), ImplicitM ~ N(1, 0.02)."""
    table = table or e6e_table()
    rng = np.random.Generator(np.random.PCG64(seed))
    t16 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32)).half().float()
    layers = _skeleton(table)
    det = layers[-1]
    for i, name, co, ci, k, s in _conv_shapes(table):
        w = torch.from_numpy(rng.standard_normal((co, ci, k, k), dtype=np.float32))
        if layers[i].type == "Detect":
            b = np.zeros((3, NC + 5), np.float32)
            b[:, 4] += math.log(8 / (640 / STRIDES[int(name[1:])]) ** 2)
            b[:, 5:] += math.log(0.6 / (NC - 0.99))
            layers[i].convs[name] = ConvBN(w, t16(b.reshape(-1)), None, 1, act=False)
            continue
        bn = (t16(1.0 + 0.1 * rng.standard_normal(co)), t16(0.1 * rng.standard_normal(co)), t16(0.1 * rng.standard_normal(co)),
              t16(1.0 + 0.1 * np.abs(rng.standard_normal(co))), 1e-3)
        layers[i].convs[name] = ConvBN(w, None, bn, s)
    ch = out_channels(table)
    det.extra = {
        "ia": [t16(0.02 * rng.standard_normal((1, ch[j], 1, 1))) for j in det.f],
        "im": [t16(1.0 + 0.02 * rng.standard_normal((1, 3 * (NC + 5), 1, 1))) for _ in det.f],
        "anchors": torch.tensor(ANCHORS, dtype=torch.float32),
        "strides": [float(s) for s in STRIDES],
        "nc": NC,
    }
    layers = prune(layers)
    _calibrate(layers, torch.from_numpy(rng.random((1, 3, 128, 192), dtype=np.float32)), head_std)
    return layers


@torch.no_grad()
def _calibrate(layers: List[Layer], x: torch.Tensor, head_std: float) -> None:
    """Scale every conv's weights in place (then round them to fp16) from one float32 forward, see synthetic_layers."""
    import torch.nn.functional as Fn

    def conv(c: ConvBN, t: torch.Tensor) -> torch.Tensor:
        z = Fn.conv2d(t, c.w, None, c.stride, c.k // 2)
        r = float(z.pow(2).mean().sqrt())
        c.w = (c.w / r).half().float()
        g, beta, mean, var, eps = c.bn
        z = (Fn.conv2d(t, c.w, None, c.stride, c.k // 2) - mean.view(1, -1, 1, 1)) / torch.sqrt(var.view(1, -1, 1, 1) + eps)
        z = z * g.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)
        return z * torch.sigmoid(z)

    y = {-1: x}
    for l in layers:
        a = [y[j] for j in l.f]
        c = l.convs
        if l.type == "ReOrg":
            t = a[0]
            y[l.i] = torch.cat([t[..., ::2, ::2], t[..., 1::2, ::2], t[..., ::2, 1::2], t[..., 1::2, 1::2]], 1)
        elif l.type == "Conv":
            y[l.i] = conv(c[""], a[0])
        elif l.type == "DownC":
            y[l.i] = torch.cat((conv(c["cv2"], conv(c["cv1"], a[0])), conv(c["cv3"], Fn.max_pool2d(a[0], 2, 2))), 1)
        elif l.type == "SPPCSPC":
            x1 = conv(c["cv4"], conv(c["cv3"], conv(c["cv1"], a[0])))
            y1 = conv(c["cv6"], conv(c["cv5"], torch.cat([x1] + [Fn.max_pool2d(x1, k, 1, k // 2) for k in (5, 9, 13)], 1)))
            y[l.i] = conv(c["cv7"], torch.cat((y1, conv(c["cv2"], a[0])), 1))
        elif l.type == "Upsample":
            y[l.i] = Fn.interpolate(a[0], scale_factor=2, mode="nearest")
        elif l.type == "Concat":
            y[l.i] = torch.cat(a, 1)
        elif l.type == "Shortcut":
            y[l.i] = a[0] + a[1]
        else:
            for k, t in enumerate(a):
                m = c[f"m{k}"]
                r = float(t.pow(2).mean().sqrt())
                m.w = (m.w * (head_std / (math.sqrt(m.w.shape[1]) * r))).half().float()
