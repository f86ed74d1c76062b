"""YOLOv7 checkpoints: a yolov7-shaped pickle (stub classes registered as models.common / models.yolo, fp16 tensors as in a
stripped release, an IAuxDetect head) loads without the yolov7 code, folds as yolov7 fuses, prunes the aux-only layers, and
refuses unknown modules and malicious globals (no GPU)."""
import os
import pickle
import sys
import types

import pytest
import torch
import torch.nn as nn

from vlfm_b200.vlm import yolov7_config as cfg
from vlfm_b200.vlm import yolov7_weights as yw


def _stub_modules():
    common, yolo = types.ModuleType("models.common"), types.ModuleType("models.yolo")
    pkg = types.ModuleType("models")
    pkg.common, pkg.yolo = common, yolo

    def cls(mod, name):
        c = type(name, (nn.Module,), {"__module__": mod.__name__, "forward": lambda self, x: x})
        setattr(mod, name, c)
        return c

    names = {n: cls(common, n) for n in ("Conv", "ReOrg", "DownC", "Concat", "Shortcut", "SPPCSPC", "ImplicitA", "ImplicitM", "RepConv")}
    names.update({n: cls(yolo, n) for n in ("IAuxDetect", "Model")})
    return {"models": pkg, "models.common": common, "models.yolo": yolo}, names


def _conv_module(S, c: yw.ConvBN):
    m = S["Conv"]()
    o, i, k, _ = c.w.shape
    m.conv = nn.Conv2d(i, o, k, c.stride, k // 2, bias=False)
    m.conv.weight.data = c.w.half()
    m.bn = nn.BatchNorm2d(o, eps=c.bn[4])
    m.bn.weight.data, m.bn.bias.data, m.bn.running_mean, m.bn.running_var = (t.half() for t in c.bn[:4])
    m.act = nn.SiLU()
    return m


def build_model(S, table, layers, extra_layer=None):
    """An nn.Module tree shaped like yolov7's Model from the table and the (unpruned-table) records."""
    by_i = {l.i: l for l in layers}
    mods = []
    for i, (f, mod, args) in enumerate(table):
        l = by_i.get(i)
        if mod == "Conv":
            m = _conv_module(S, l.convs[""]) if l else _conv_module(S, yw.ConvBN(torch.zeros(args[0], 8, args[1], args[1]), None,
                                                                            (torch.ones(args[0]), torch.zeros(args[0]), torch.zeros(args[0]),
                                                                             torch.ones(args[0]), 1e-3), args[2]))
        elif mod == "DownC":
            m = S["DownC"]()
            for n in ("cv1", "cv2", "cv3"):
                setattr(m, n, _conv_module(S, l.convs[n]))
            m.mp = nn.MaxPool2d(2, 2)
        elif mod == "SPPCSPC":
            m = S["SPPCSPC"]()
            for n in ("cv1", "cv2", "cv3", "cv4", "cv5", "cv6", "cv7"):
                setattr(m, n, _conv_module(S, l.convs[n]))
            m.m = nn.ModuleList([nn.MaxPool2d(k, 1, k // 2) for k in (5, 9, 13)])
        elif mod == "Upsample":
            m = nn.Upsample(None, 2, "nearest")
        elif mod == "IAuxDetect":
            m = S["IAuxDetect"]()
            m.nl, m.na, m.nc, m.no = 4, 3, 80, 85
            heads = [l.convs[f"m{k}"] for k in range(4)]
            m.m = nn.ModuleList()
            for c in heads:
                conv = nn.Conv2d(c.w.shape[1], c.w.shape[0], 1)
                conv.weight.data, conv.bias.data = c.w.half(), c.b.half()
                m.m.append(conv)
            m.m2 = nn.ModuleList([nn.Conv2d(8, 255, 1) for _ in range(4)])
            m.ia, m.im = nn.ModuleList(), nn.ModuleList()
            for a, b in zip(l.extra["ia"], l.extra["im"]):
                ia, im = S["ImplicitA"](), S["ImplicitM"]()
                ia.implicit, im.implicit = nn.Parameter(a.half()), nn.Parameter(b.half())
                m.ia.append(ia)
                m.im.append(im)
            m.stride = torch.tensor(cfg.STRIDES, dtype=torch.float32)
            m.register_buffer("anchors", (l.extra["anchors"] / m.stride.view(-1, 1, 1)).half())
            m.register_buffer("anchor_grid", l.extra["anchors"].view(4, 1, 3, 1, 1, 2).half())
        else:
            m = S[mod]()
            if mod == "Concat":
                m.d = 1
        m.i, m.f, m.type = i, f, mod
        mods.append(m)
    if extra_layer is not None:
        mods.insert(extra_layer[0], extra_layer[1])
    model = S["Model"]()
    model.model = nn.Sequential(*mods)
    model.save = sorted({j % i for i, (f, _, _) in enumerate(table) for j in ([f] if isinstance(f, int) else f) if j != -1})
    return model


def save_checkpoint(path, model, sysmods, ema=True):
    saved = {k: sys.modules.get(k) for k in sysmods}
    sys.modules.update(sysmods)
    try:
        torch.save({"epoch": -1, "model": None if ema else model, "ema": model if ema else None, "updates": 10, "optimizer": None}, path)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def full_records(div, seed=1):
    """Records of every table row (aux layers included, as a checkpoint has them) -> (table, records, pruned)."""
    table = cfg.e6e_table(div)
    pruned = cfg.synthetic_layers(seed, table=table)
    return table, pruned


@pytest.mark.parametrize("div", [8, 1])
def test_checkpoint_loads_folds_and_prunes(tmp_path, div):
    sysmods, S = _stub_modules()
    table, layers = full_records(div)
    path = str(tmp_path / "yolov7.pt")
    save_checkpoint(path, build_model(S, table, layers), sysmods)
    with pytest.raises(ImportError):
        import models  # noqa: F401  (the yolov7 package is not importable here)
    got = yw.load_checkpoint(path)
    assert [l.i for l in got] == [l.i for l in layers]
    aux_only = {261, 262, 263, 264}
    assert not aux_only & {l.i for l in got}
    assert got[-1].type == "Detect" and got[-1].f == [257, 258, 259, 260]
    for a, b in zip(got, layers):
        assert a.type == b.type and a.f == b.f
        for n, c in b.convs.items():
            if a.type == "Detect":
                k = int(n[1:])
                w, bias = yw.fold_detect(a.convs[n], a.extra["ia"][k], a.extra["im"][k])
                # IDetect.fuse: b' = (b + W ia) * im, W' = W * im
                W = c.w.half().float().reshape(c.w.shape[0], -1)
                ia = b.extra["ia"][k].half().float().reshape(-1)
                im = b.extra["im"][k].half().float().reshape(-1)
                assert torch.allclose(bias, (c.b.half().float() + W @ ia) * im, rtol=1e-6, atol=1e-6)
                assert torch.allclose(w.reshape(W.shape), W * im[:, None], rtol=1e-6, atol=0)
            else:
                w, bias = yw.fold(a.convs[n])
                g, beta, mean, var, eps = (t.half().float() if isinstance(t, torch.Tensor) else t for t in c.bn)
                s = g / torch.sqrt(var + eps)
                assert torch.allclose(w, c.w.half().float() * s.view(-1, 1, 1, 1), rtol=1e-6, atol=1e-7)
                assert torch.allclose(bias, beta - g * mean / torch.sqrt(var + eps), rtol=1e-6, atol=1e-6)


def test_model_taken_when_ema_is_absent(tmp_path):
    sysmods, S = _stub_modules()
    table, layers = full_records(8)
    path = str(tmp_path / "m.pt")
    save_checkpoint(path, build_model(S, table, layers), sysmods, ema=False)
    assert len(yw.load_checkpoint(path)) == len(layers)


def test_unknown_module_raises_with_its_index(tmp_path):
    sysmods, S = _stub_modules()
    table, layers = full_records(8)
    rep = S["RepConv"]()
    rep.i, rep.f = 5, -1
    model = build_model(S, table, layers)
    model.model[5] = rep
    path = str(tmp_path / "rep.pt")
    save_checkpoint(path, model, sysmods)
    with pytest.raises(NotImplementedError, match="layer 5 is a RepConv"):
        yw.load_checkpoint(path)


class _Evil:
    def __init__(self, fn, arg):
        self.fn, self.arg = fn, arg

    def __reduce__(self):
        return (self.fn, (self.arg,))


@pytest.mark.parametrize("fn", ["os.system", "builtins.eval"])
def test_malicious_pickles_are_refused_before_they_run(tmp_path, fn):
    marker = tmp_path / "ran"
    if fn == "os.system":
        payload = _Evil(os.system, f"touch {marker}")
    else:
        payload = _Evil(eval, f"open({str(marker)!r}, 'w').close()")
    path = str(tmp_path / "evil.pt")
    torch.save({"model": payload, "ema": None}, path)
    with pytest.raises(pickle.UnpicklingError, match="refusing to load global"):
        yw.load_checkpoint(path)
    assert not marker.exists()
