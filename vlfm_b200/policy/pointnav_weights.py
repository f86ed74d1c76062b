"""PointNav checkpoints -> the state dict of ``pointnav_engine.PointNavEngine``.

Two layouts hold the same network (a ResNet-18 over depth with GroupNorm, a 2-layer LSTM of 512 and an action head):

- a habitat-baselines checkpoint ``{"config", "extra_state", "state_dict"}`` (``data/pointnav_weights.pth``): Discrete(4) actions,
  ``net.prev_action_embedding.weight`` [5, 32] (an embedding of ``prev + 1``, 0 = start), head ``action_distribution.linear``;
- a flat state dict (``data/spot_pointnav_weights.pth``): continuous actions, ``net.prev_action_embedding(_cont).{weight [32, 2],
  bias}`` (a Linear of ``mask * prev``), head ``action_distribution.mu_maybe_std`` [4, 512] (mu | log_std).

Discrete or continuous is decided by the presence of ``action_distribution.mu_maybe_std.weight``.  ``critic.*`` is ignored; any
other missing or unknown key raises.

The habitat checkpoint's ``config`` is a pickled omegaconf ``DictConfig`` of habitat structured-config classes, with a
``collections.defaultdict`` that ``torch.load(weights_only=True)`` refuses.  ``load_checkpoint`` therefore unpickles with
``RestrictedUnpickler``: tensors, plain containers and typing names are rebuilt; classes under omegaconf / habitat /
habitat_baselines / vlfm become inert placeholders (neither package is needed); every other global is refused before anything
runs.
"""
from __future__ import annotations

import math
import pickle
import types
from typing import Dict, Tuple

import numpy as np
import torch

HID, EMB, VIS = 512, 32, 512
NGROUPS = 16
STAGES = ((32, 1), (64, 2), (128, 2), (256, 2))     # (channels, stride of the first block)
BACKBONE = "net.visual_encoder.backbone."
HEAD_DISCRETE = "action_distribution.linear."
HEAD_CONTINUOUS = "action_distribution.mu_maybe_std."


def _conv_gn(shapes, name, o, i, k, conv="0", gn="1"):
    shapes[f"{name}.{conv}.weight"] = (o, i, k, k)
    shapes[f"{name}.{gn}.weight"] = (o,)
    shapes[f"{name}.{gn}.bias"] = (o,)


def shared_shapes() -> Dict[str, tuple]:
    """Name -> shape of every tensor both layouts share (checkpoint names)."""
    s: Dict[str, tuple] = {}
    _conv_gn(s, BACKBONE + "conv1", 32, 1, 7)
    cin = 32
    for li, (c, stride) in enumerate(STAGES, start=1):
        for bi in range(2):
            p = f"{BACKBONE}layer{li}.{bi}"
            _conv_gn(s, p + ".convs", c, cin if bi == 0 else c, 3, "0", "1")
            _conv_gn(s, p + ".convs", c, c, 3, "3", "4")
            if bi == 0 and (stride != 1 or cin != c):
                _conv_gn(s, p + ".downsample", c, cin, 1)
        cin = c
    _conv_gn(s, "net.visual_encoder.compression", 128, 256, 3)
    s["net.visual_fc.1.weight"], s["net.visual_fc.1.bias"] = (VIS, 2048), (VIS,)
    s["net.tgt_embeding.weight"], s["net.tgt_embeding.bias"] = (EMB, 3), (EMB,)
    for l, k in ((0, VIS + 2 * EMB), (1, HID)):
        s[f"net.state_encoder.rnn.weight_ih_l{l}"] = (4 * HID, k)
        s[f"net.state_encoder.rnn.weight_hh_l{l}"] = (4 * HID, HID)
        s[f"net.state_encoder.rnn.bias_ih_l{l}"] = (4 * HID,)
        s[f"net.state_encoder.rnn.bias_hh_l{l}"] = (4 * HID,)
    return s


def engine_shapes(discrete: bool) -> Dict[str, tuple]:
    """The engine's key set: the shared tensors, ``net.prev_action_embedding.*`` and the head under its checkpoint name."""
    s = shared_shapes()
    if discrete:
        s["net.prev_action_embedding.weight"] = (5, EMB)
        s[HEAD_DISCRETE + "weight"], s[HEAD_DISCRETE + "bias"] = (4, HID), (4,)
    else:
        s["net.prev_action_embedding.weight"], s["net.prev_action_embedding.bias"] = (EMB, 2), (EMB,)
        s[HEAD_CONTINUOUS + "weight"], s[HEAD_CONTINUOUS + "bias"] = (4, HID), (4,)
    return s


def convert_state_dict(sd: Dict[str, torch.Tensor]) -> Tuple[Dict[str, torch.Tensor], bool]:
    """A checkpoint's state dict (either layout) -> (engine state dict of float32 CPU tensors, discrete).  Raises on a missing,
    unknown or misshapen key."""
    discrete = HEAD_CONTINUOUS + "weight" not in sd
    out: Dict[str, torch.Tensor] = {}
    unknown = []
    for k, v in sd.items():
        if k.startswith("critic."):
            continue
        name = k
        for alias in ("net.prev_action_embedding_cont.", "net.prev_action_embedding_discrete."):
            if k.startswith(alias):
                name = "net.prev_action_embedding." + k[len(alias):]
        if name in out:
            raise KeyError(f"PointNav checkpoint: {k!r} duplicates another name of {name!r}")
        out[name] = v
    want = engine_shapes(discrete)
    unknown = sorted(set(out) - set(want))
    missing = sorted(set(want) - set(out))
    if unknown or missing:
        raise KeyError(f"PointNav checkpoint ({'discrete' if discrete else 'continuous'} head): missing {missing}, unknown {unknown}")
    for k, shape in want.items():
        if not isinstance(out[k], torch.Tensor) or tuple(out[k].shape) != shape:
            raise ValueError(f"PointNav checkpoint: {k} has shape {tuple(getattr(out[k], 'shape', ()))}, expected {shape}")
        out[k] = out[k].detach().to("cpu", torch.float32).contiguous()
    return out, discrete


# ------------------------------------------------------------------------------------------------------------- unpickling
_PLACEHOLDER_ROOTS = ("omegaconf", "habitat", "habitat_baselines", "vlfm")
_ALLOWED = {
    "torch._utils": {"_rebuild_tensor_v2", "_rebuild_parameter"},
    "collections": {"OrderedDict", "defaultdict"},
    "builtins": {"dict", "list", "tuple", "set", "frozenset", "bool", "int", "float", "str", "bytes", "Ellipsis", "slice"},
    "__builtin__": {"dict", "list", "tuple", "set", "frozenset", "bool", "int", "long", "float", "str", "unicode", "bytes",
                    "Ellipsis", "slice"},
    "typing": {"Any", "Dict", "List", "Tuple", "Optional", "Union"},
    "_operator": {"getitem"},
    "operator": {"getitem"},
}


class _Inert:
    """Stands in for a config class of a package that is not imported: accepts any construction and state, and does nothing."""

    def __new__(cls, *args, **kwargs):
        return object.__new__(cls)

    def __init__(self, *args, **kwargs):
        pass

    def __setstate__(self, state):
        self.__dict__["_state"] = state

    def __setitem__(self, key, value):   # SETITEM(S) on a dict subclass placeholder
        self.__dict__.setdefault("_items", {})[key] = value


_PLACEHOLDERS: Dict[str, type] = {}


def _placeholder(module: str, name: str) -> type:
    key = module + "." + name
    if key not in _PLACEHOLDERS:
        _PLACEHOLDERS[key] = type(name, (_Inert,), {"__module__": "pointnav_placeholder." + module})
    return _PLACEHOLDERS[key]


class RestrictedUnpickler(pickle.Unpickler):
    """Rebuilds tensors, builtins, ``collections.OrderedDict`` / ``defaultdict``, ``typing`` names and ``operator.getitem``;
    classes under omegaconf / habitat / habitat_baselines / vlfm become inert placeholders; any other global raises
    ``pickle.UnpicklingError`` before it is called."""

    def find_class(self, module, name):
        if module.split(".")[0] in _PLACEHOLDER_ROOTS:
            return _placeholder(module, name)
        if name in _ALLOWED.get(module, ()):
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"PointNav checkpoint: refusing to load global {module}.{name}")


def _restricted_load(f, **kwargs):
    return RestrictedUnpickler(f, **kwargs).load()


restricted_pickle = types.ModuleType("pointnav_restricted_pickle")
restricted_pickle.Unpickler = RestrictedUnpickler
restricted_pickle.load = _restricted_load
restricted_pickle.__version__ = pickle.format_version


def load_checkpoint(path: str) -> Tuple[Dict[str, torch.Tensor], bool]:
    """Either checkpoint layout -> (engine state dict, discrete)."""
    obj = torch.load(path, map_location="cpu", pickle_module=restricted_pickle, weights_only=False)
    if isinstance(obj, dict) and "state_dict" in obj and isinstance(obj["state_dict"], dict):
        sd = obj["state_dict"]
    elif isinstance(obj, dict) and all(isinstance(v, torch.Tensor) for v in obj.values()):
        sd = obj
    else:
        raise ValueError(f"PointNav checkpoint {path}: neither a habitat-baselines checkpoint nor a flat state dict")
    return convert_state_dict(sd)


# -------------------------------------------------------------------------------------------------------- synthetic weights
def random_state_dict(seed: int = 0, discrete: bool = True) -> Dict[str, torch.Tensor]:
    """Seeded weights (numpy PCG64) in the checkpoint layout (habitat names for discrete, flat-file names for continuous).  Conv
    weights ~ N(0, 1/fan_in) (each is followed by a GroupNorm), GroupNorm affine around identity, Linear / LSTM weights scaled so
    that gate pre-activations and head outputs are O(1): every term of the step contributes."""
    rng = np.random.Generator(np.random.PCG64(seed))
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    sd: Dict[str, torch.Tensor] = {}
    shapes = engine_shapes(discrete)
    for k, shape in shapes.items():
        if len(shape) == 4:
            fan = shape[1] * shape[2] * shape[3]
            sd[k] = t(rng.standard_normal(shape) / math.sqrt(fan))
        elif len(shape) == 1 and (".convs." in k or "conv1.1" in k or "downsample.1" in k or "compression.1" in k):
            sd[k] = t(1.0 + 0.2 * rng.standard_normal(shape)) if k.endswith("weight") else t(0.2 * rng.standard_normal(shape))
        elif k.startswith("net.state_encoder.rnn.weight"):
            sd[k] = t(rng.standard_normal(shape) * 1.5 / math.sqrt(shape[1]))
        elif k.startswith("net.state_encoder.rnn.bias"):
            sd[k] = t(0.1 * rng.standard_normal(shape))
        elif k == "net.visual_fc.1.weight":
            sd[k] = t(rng.standard_normal(shape) * 2.0 / math.sqrt(shape[1]))
        elif k == "net.tgt_embeding.weight":
            sd[k] = t(rng.standard_normal(shape))
        elif k == "net.prev_action_embedding.weight" and discrete:
            sd[k] = t(rng.standard_normal(shape))
        elif k.endswith(".weight") and k.startswith("action_distribution."):
            sd[k] = t(rng.standard_normal(shape) * 4.0 / math.sqrt(shape[1]))
        elif k.endswith(".weight"):
            sd[k] = t(rng.standard_normal(shape) / math.sqrt(shape[1]))
        else:
            sd[k] = t(0.1 * rng.standard_normal(shape))
    sd["critic.fc.weight"], sd["critic.fc.bias"] = t(rng.standard_normal((1, HID)) / math.sqrt(HID)), t(np.zeros(1))
    return sd
