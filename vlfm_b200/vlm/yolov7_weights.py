"""YOLOv7 checkpoints -> a list of layer records, unfused, and the fold that the fp16 engine runs.

A yolov7 ``.pt`` file holds a pickled ``models.yolo.Model`` (``attempt_load`` takes ``ckpt["ema"]`` when it is present and truthy,
else ``ckpt["model"]``).  ``load_checkpoint`` unpickles it with ``YoloUnpickler``, the PointNav ``RestrictedUnpickler`` extended
so that classes under ``models.*`` and ``torch.nn.modules.*`` become inert placeholders that keep their ``__dict__``; tensors,
plain containers, ``OrderedDict`` and numpy arrays (training-state fields) are rebuilt, and every other global is refused before
anything runs.  Neither the yolov7 code nor its ``models`` package is needed.

``model.model`` is walked in order: each module's ``f`` (its input layers; -1 is the previous layer, other negatives count back
from its own index ``i``) and type name give a ``Layer``.  Only the E6E vocabulary is supported: ``Conv`` (k 1 or 3, stride 1 or
2, SiLU), ``ReOrg``, ``DownC``, ``Concat``, ``Shortcut``, ``SPPCSPC``, ``Upsample`` (nearest x2), ``IDetect`` and ``IAuxDetect``.
Of ``IAuxDetect`` only the main heads ``m[:nl]`` are evaluated, and layers whose outputs reach only its aux inputs are pruned.
"""
from __future__ import annotations

import pickle
import types
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from ..policy.pointnav_weights import RestrictedUnpickler

SUPPORTED = ("Conv", "ReOrg", "DownC", "Concat", "Shortcut", "SPPCSPC", "Upsample", "IDetect", "IAuxDetect")


@dataclass
class ConvBN:
    """One yolov7 ``Conv``: conv (bias optional) -> BatchNorm (absent once fused) -> SiLU when ``act``.  fp32 CPU tensors."""
    w: torch.Tensor
    b: Optional[torch.Tensor]
    bn: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, float]]   # weight, bias, mean, var, eps
    stride: int = 1
    act: bool = True

    @property
    def k(self) -> int:
        return self.w.shape[2]


@dataclass
class Layer:
    i: int
    f: List[int]                      # absolute input layer indices; -1 = the network input
    type: str                         # one of SUPPORTED, with IDetect / IAuxDetect both as "Detect"
    convs: Dict[str, ConvBN] = field(default_factory=dict)
    # Detect: ia / im [nl] implicit tensors, anchors [nl, na, 2] in pixels, strides [nl], nc
    extra: Dict[str, object] = field(default_factory=dict)


def fold(c: ConvBN) -> Tuple[torch.Tensor, torch.Tensor]:
    """yolov7's fuse_conv_and_bn in fp32: (weight [o, i, k, k], bias [o])."""
    w = c.w.float()
    b = torch.zeros(w.shape[0]) if c.b is None else c.b.float()
    if c.bn is None:
        return w, b
    g, beta, mean, var, eps = (t.float() if isinstance(t, torch.Tensor) else t for t in c.bn)
    scale = g.div(torch.sqrt(eps + var))
    wf = torch.mm(torch.diag(scale), w.reshape(w.shape[0], -1)).view(w.shape)
    bf = torch.mm(torch.diag(scale), b.reshape(-1, 1)).reshape(-1) + (beta - g.mul(mean).div(torch.sqrt(var + eps)))
    return wf, bf


def fold_detect(c: ConvBN, ia: torch.Tensor, im: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """IDetect.fuse for one level in fp32: ImplicitA into the bias, then ImplicitM into bias and weight."""
    w, b = c.w.float().clone(), c.b.float().clone()
    o, i = w.shape[:2]
    b += torch.matmul(w.reshape(o, i), ia.float().reshape(i, 1)).squeeze(1)
    b *= im.float().reshape(o)
    w *= im.float().transpose(0, 1)
    return w, b


def resolve(i: int, f) -> List[int]:
    return [(i - 1 if j == -1 else (i + j if j < 0 else j)) for j in ([f] if isinstance(f, int) else list(f))]


def prune(layers: List[Layer]) -> List[Layer]:
    """The layers whose outputs reach the detection layer's evaluated inputs, in order (the detection layer last)."""
    by_i = {l.i: l for l in layers}
    det = layers[-1]
    need, todo = {det.i}, list(det.f)
    while todo:
        j = todo.pop()
        if j >= 0 and j not in need:
            need.add(j)
            todo.extend(by_i[j].f)
    return [l for l in layers if l.i in need]


# ------------------------------------------------------------------------------------------------------------- unpickling
class _Module:
    """Stands in for a yolov7 or torch.nn module class: keeps the pickled ``__dict__`` and does nothing else."""

    def __new__(cls, *args, **kwargs):
        return object.__new__(cls)

    def __init__(self, *args, **kwargs):
        pass

    def __setstate__(self, state):
        self.__dict__.update(state if isinstance(state, dict) else {"_state": state})


_MODULE_PLACEHOLDERS: Dict[str, type] = {}
_NUMPY = {("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "_reconstruct"), ("numpy", "ndarray"), ("numpy", "dtype"),
          ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar")}


class YoloUnpickler(RestrictedUnpickler):
    """``RestrictedUnpickler`` plus placeholders for ``models.*`` and ``torch.nn.modules.*`` classes and numpy arrays."""

    what = "YOLOv7 checkpoint"

    def placeholder(self, module, name):
        if module == "models" or module.startswith("models.") or module.startswith("torch.nn.modules."):
            key = module + "." + name
            if key not in _MODULE_PLACEHOLDERS:
                _MODULE_PLACEHOLDERS[key] = type(name, (_Module,), {"__module__": "yolo_placeholder." + module})
            return _MODULE_PLACEHOLDERS[key]
        return None

    def find_class(self, module, name):
        if (module, name) in _NUMPY:
            return pickle.Unpickler.find_class(self, module, name)
        return super().find_class(module, name)


def _restricted_load(f, **kwargs):
    return YoloUnpickler(f, **kwargs).load()


restricted_pickle = types.ModuleType("yolov7_restricted_pickle")
restricted_pickle.Unpickler = YoloUnpickler
restricted_pickle.load = _restricted_load
restricted_pickle.__version__ = pickle.format_version


# ----------------------------------------------------------------------------------------------------------- module tree
def _d(m) -> dict:
    return m.__dict__


def _mods(m) -> dict:
    return dict(_d(m).get("_modules") or {})


def _param(m, name) -> Optional[torch.Tensor]:
    d = _d(m)
    for store in ("_parameters", "_buffers"):
        t = (d.get(store) or {}).get(name)
        if t is not None:
            return t.detach().float()
    t = d.get(name)
    return t.detach().float() if isinstance(t, torch.Tensor) else None


def _tname(m) -> str:
    return type(m).__name__


def _conv(m, where: str) -> ConvBN:
    """A yolov7 Conv module (conv [+ bn] + act) -> ConvBN."""
    if _tname(m) != "Conv":
        raise ValueError(f"YOLOv7 checkpoint: {where} is a {_tname(m)}, expected Conv")
    sub = _mods(m)
    conv, bn, act = sub.get("conv"), sub.get("bn"), sub.get("act")
    if conv is None or _tname(conv) != "Conv2d":
        raise ValueError(f"YOLOv7 checkpoint: {where} has no Conv2d")
    c = _conv2d(conv, where)
    if bn is not None:
        if _tname(bn) != "BatchNorm2d":
            raise ValueError(f"YOLOv7 checkpoint: {where}.bn is a {_tname(bn)}")
        c.bn = (_param(bn, "weight"), _param(bn, "bias"), _param(bn, "running_mean"), _param(bn, "running_var"), float(_d(bn)["eps"]))
    if act is None or _tname(act) != "SiLU":
        raise NotImplementedError(f"YOLOv7 checkpoint: {where} activation {_tname(act) if act is not None else None} (only SiLU)")
    return c


def _conv2d(m, where: str, act: bool = True) -> ConvBN:
    d = _d(m)
    w = _param(m, "weight")
    k, s = tuple(d["kernel_size"]), tuple(d["stride"])
    if (d.get("groups", 1) != 1 or tuple(d.get("dilation", (1, 1))) != (1, 1) or k[0] != k[1] or k[0] not in (1, 3) or s[0] != s[1]
            or s[0] not in (1, 2) or tuple(d["padding"]) != (k[0] // 2, k[0] // 2)):
        raise NotImplementedError(f"YOLOv7 checkpoint: {where} conv kernel {k} stride {s} padding {d.get('padding')} unsupported")
    return ConvBN(w, _param(m, "bias"), None, s[0], act)


def layers_from_model(model) -> List[Layer]:
    """Walk ``model.model`` -> pruned ``Layer`` list (see the module docstring)."""
    seq = _mods(model).get("model")
    if seq is None:
        raise ValueError("YOLOv7 checkpoint: the model has no `model` module list")
    layers: List[Layer] = []
    for idx, m in enumerate(_mods(seq).values()):
        d, t = _d(m), _tname(m)
        i = int(d.get("i", idx))
        f = resolve(i, d.get("f", -1))
        where = f"layer {i} ({t})"
        if t not in SUPPORTED:
            raise NotImplementedError(f"YOLOv7 checkpoint: layer {i} is a {t}; supported: {', '.join(SUPPORTED)}")
        sub = _mods(m)
        if t == "Conv":
            layers.append(Layer(i, f, t, {"": _conv(m, where)}))
        elif t == "DownC":
            layers.append(Layer(i, f, t, {n: _conv(sub[n], f"{where}.{n}") for n in ("cv1", "cv2", "cv3")}))
            if _d(sub["mp"]).get("kernel_size") not in (2, (2, 2)) or layers[-1].convs["cv2"].stride != 2:
                raise NotImplementedError(f"YOLOv7 checkpoint: {where} is not a stride-2 DownC")
        elif t == "SPPCSPC":
            ks = [_d(p)["kernel_size"] for p in _mods(sub["m"]).values()]
            if ks != [5, 9, 13]:
                raise NotImplementedError(f"YOLOv7 checkpoint: {where} pools {ks} (only 5, 9, 13)")
            layers.append(Layer(i, f, t, {n: _conv(sub[n], f"{where}.{n}") for n in ("cv1", "cv2", "cv3", "cv4", "cv5", "cv6", "cv7")}))
        elif t == "Upsample":
            if d.get("mode") != "nearest" or float(d.get("scale_factor") or 0) != 2.0:
                raise NotImplementedError(f"YOLOv7 checkpoint: {where} mode {d.get('mode')} scale {d.get('scale_factor')}")
            layers.append(Layer(i, f, t))
        elif t in ("ReOrg", "Concat", "Shortcut"):
            if t == "Concat" and d.get("d", 1) != 1:
                raise NotImplementedError(f"YOLOv7 checkpoint: {where} concatenates along dim {d.get('d')}")
            layers.append(Layer(i, f, t))
        else:                                    # IDetect / IAuxDetect: the main heads m[:nl] only
            nl, na, nc = int(d["nl"]), int(d["na"]), int(d["nc"])
            heads = list(_mods(sub["m"]).values())[:nl]
            convs = {f"m{k}": _conv2d(h, f"{where}.m.{k}", act=False) for k, h in enumerate(heads)}
            ia = [_param(x, "implicit") for x in list(_mods(sub["ia"]).values())[:nl]]
            im = [_param(x, "implicit") for x in list(_mods(sub["im"]).values())[:nl]]
            stride = _param(m, "stride")
            anchors, grid = _param(m, "anchors"), _param(m, "anchor_grid")
            if stride is None or anchors is None or grid is None:
                raise ValueError(f"YOLOv7 checkpoint: {where} lacks stride / anchors / anchor_grid")
            grid = grid.reshape(nl, na, 2)
            if not torch.allclose(grid, anchors.reshape(nl, na, 2) * stride.reshape(nl, 1, 1), rtol=1e-3, atol=1e-2):
                raise ValueError(f"YOLOv7 checkpoint: {where} anchor_grid is not anchors * stride")
            for c in convs.values():
                if c.k != 1 or c.w.shape[0] != na * (nc + 5) or c.b is None:
                    raise ValueError(f"YOLOv7 checkpoint: {where} head conv shape {tuple(c.w.shape)}")
            layers.append(Layer(i, f[:nl], "Detect", convs, {"ia": ia, "im": im, "anchors": grid, "strides": stride.reshape(nl).tolist(),
                                                             "nc": nc}))
            break
    if not layers or layers[-1].type != "Detect":
        raise ValueError("YOLOv7 checkpoint: no IDetect / IAuxDetect layer")
    return prune(layers)


def load_checkpoint(path: str) -> List[Layer]:
    """A yolov7 ``.pt`` -> pruned layer records (``ema`` when present and truthy, else ``model``)."""
    ckpt = torch.load(path, map_location="cpu", pickle_module=restricted_pickle, weights_only=False)
    if not isinstance(ckpt, dict):
        raise ValueError(f"YOLOv7 checkpoint {path}: expected a dict with `model`")
    model = ckpt["ema"] if ckpt.get("ema") else ckpt.get("model")
    if model is None:
        raise ValueError(f"YOLOv7 checkpoint {path}: no `model` / `ema`")
    return layers_from_model(model)
