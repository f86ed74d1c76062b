"""PointNav checkpoint loading (vlfm_b200/policy/pointnav_weights.py) on synthetic files with the exact layout of the two real
checkpoints (tests/golden/pointnav_layout.json): the habitat-baselines file, whose pickled config names omegaconf / habitat
classes, and the flat state dict.  Also: the restricted unpickler refuses other globals before they run, the key rules, and that
the synthetic weights give non-degenerate actions."""
import collections
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import pointnav_oracle as po
from vlfm_b200.policy.pointnav_weights import convert_state_dict, engine_shapes, load_checkpoint, random_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LAYOUT = json.load(open(os.path.join(GOLDEN, "pointnav_layout.json")))


def _layout_state_dict(name, seed):
    """An OrderedDict with the real file's names, shapes and dtypes, values from random_state_dict."""
    entries = LAYOUT[name]["tensors"]
    discrete = any(k.startswith("action_distribution.linear.") for k, _, _ in entries)
    src = random_state_dict(seed, discrete)
    sd = collections.OrderedDict()
    for k, shape, dtype in entries:
        assert tuple(src[k].shape) == tuple(shape), k
        sd[k] = src[k].to(getattr(torch, dtype))
    return sd, discrete


def _stub_config_modules():
    """Modules named like the classes the real config pickles (a habitat config dataclass inside an omegaconf DictConfig)."""
    mods = {}
    for name in ("omegaconf", "omegaconf.dictconfig", "habitat", "habitat.config", "habitat.config.default_structured_configs"):
        mods[name] = types.ModuleType(name)

    class DictConfig:
        def __init__(self, content):
            self.content = content

    class HabitatConfig:
        def __init__(self):
            self.seed = 100

    DictConfig.__module__, DictConfig.__qualname__ = "omegaconf.dictconfig", "DictConfig"
    HabitatConfig.__module__, HabitatConfig.__qualname__ = "habitat.config.default_structured_configs", "HabitatConfig"
    mods["omegaconf.dictconfig"].DictConfig = DictConfig
    mods["habitat.config.default_structured_configs"].HabitatConfig = HabitatConfig
    return mods, DictConfig, HabitatConfig


def test_layout_fixture_matches_engine_keys():
    for name, discrete in (("pointnav_weights.pth", True), ("spot_pointnav_weights.pth", False)):
        names = {k for k, _, _ in LAYOUT[name]["tensors"] if not k.startswith("critic.")}
        assert names == set(engine_shapes(discrete)), name
    assert LAYOUT["pointnav_weights.pth"]["top_level"] == ["config", "extra_state", "state_dict"]
    assert "collections.defaultdict" in LAYOUT["pointnav_weights.pth"]["pickle_globals"]


def test_habitat_checkpoint_loads_without_omegaconf_or_habitat(tmp_path):
    sd, discrete = _layout_state_dict("pointnav_weights.pth", 3)
    mods, DictConfig, HabitatConfig = _stub_config_modules()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        extra = collections.defaultdict(list)
        extra["step"].append(1)
        cfg = DictConfig({"habitat": HabitatConfig(), "types": __import__("typing").Any, "extra": extra})
        path = str(tmp_path / "ckpt.pth")
        torch.save({"config": cfg, "extra_state": {"step": 7}, "state_dict": sd}, path, _use_new_zipfile_serialization=True)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    assert "omegaconf" not in sys.modules or sys.modules["omegaconf"] is saved["omegaconf"]
    w, d = load_checkpoint(path)
    want, _ = convert_state_dict(sd)
    assert d is True and discrete
    assert set(w) == set(want)
    for k in w:
        assert torch.equal(w[k].view(torch.int32), want[k].view(torch.int32)), k


def test_flat_checkpoint_loads(tmp_path):
    sd, discrete = _layout_state_dict("spot_pointnav_weights.pth", 4)
    path = str(tmp_path / "flat.pth")
    torch.save(sd, path)
    w, d = load_checkpoint(path)
    assert d is False and not discrete
    want, _ = convert_state_dict(sd)
    assert all(torch.equal(w[k], want[k]) for k in want)


class _Evil:
    def __init__(self, fn, arg):
        self.fn, self.arg = fn, arg

    def __reduce__(self):
        return (self.fn, (self.arg,))


@pytest.mark.parametrize("which", ["os.system", "builtins.eval"])
def test_restricted_unpickler_refuses_other_globals(tmp_path, which):
    marker = tmp_path / "ran"
    if which == "os.system":
        payload = _Evil(os.system, f"touch {marker}")
    else:
        payload = _Evil(eval, f"open({str(marker)!r}, 'w').close()")
    path = str(tmp_path / "evil.pth")
    torch.save({"state_dict": {"x": torch.zeros(1)}, "config": payload}, path)
    with pytest.raises(Exception, match="refusing to load global"):
        load_checkpoint(path)
    assert not marker.exists()


def test_key_rules():
    sd = random_state_dict(0, False)
    w, d = convert_state_dict(sd)
    assert d is False
    cont = {k.replace("net.prev_action_embedding.", "net.prev_action_embedding_cont."): v for k, v in sd.items()}
    w2, _ = convert_state_dict(cont)
    assert all(torch.equal(w[k], w2[k]) for k in w)
    missing = dict(sd)
    del missing["net.visual_fc.1.bias"]
    with pytest.raises(KeyError, match="missing"):
        convert_state_dict(missing)
    unknown = dict(sd, **{"net.extra.weight": torch.zeros(1)})
    with pytest.raises(KeyError, match="unknown"):
        convert_state_dict(unknown)
    bad = dict(sd, **{"net.tgt_embeding.weight": torch.zeros(32, 4)})
    with pytest.raises(ValueError):
        convert_state_dict(bad)
    no_critic = {k: v for k, v in sd.items() if not k.startswith("critic.")}
    convert_state_dict(no_critic)


def test_synthetic_weights_are_not_degenerate():
    """On the fixture episodes (the reference's own outputs): every discrete episode takes at least 3 distinct actions, the
    median top-2 logit gap is at least 10x the GPU head bar (so the action check decides most steps), and fewer than half the
    continuous mu values saturate tanh."""
    live = np.load(os.path.join(GOLDEN, "live_pointnav.npz"))
    for ci, (layout, _, _, _, _) in enumerate(po.LIVE_CASES):
        head = torch.from_numpy(live[f"c{ci}_head"]).reshape(-1, 4)
        if layout == "discrete":
            assert np.unique(live[f"c{ci}_action"]).size >= 3
            assert po.top2_gap(head).median().item() >= 10 * po.GPU_BARS["head"]
        else:
            assert (torch.tanh(head[:, :2]).abs() > 0.99).double().mean().item() < 0.5
