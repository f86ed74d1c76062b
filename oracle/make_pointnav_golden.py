"""Generate tests/golden/live_pointnav.npz and tests/golden/pointnav_layout.json by running the REAL reference PointNav modules.

Usage:  VLFM_REFERENCE=<checkout of bdaiinstitute/vlfm> python oracle/make_pointnav_golden.py

live_pointnav.npz: the reference's own modules in float32 on the CPU, on ``random_state_dict`` weights of both layouts, over the
episodes of ``oracle.pointnav_oracle.LIVE_CASES`` (depth from ``depth_frames``: only the seeds are stored), own actions fed back.
  - continuous: ``PointNavResNetPolicy.act(deterministic=True)``, and at batch 1 the real ``WrappedPointNavResNetPolicy`` loaded
    through ``load_pointnav_policy`` from a temporary file;
  - discrete: ``PointNavResNetNet(discrete_actions=True)`` (the reference's construction for a discrete policy) plus a Linear and
    argmax for habitat's ``CategoricalNet``, which is absent from the reference tree (that head is unpinned).
  Recorded: head outputs and actions at every step, features and hidden states at ``RECORD_STEPS``.
pointnav_layout.json: for both real checkpoints under $VLFM_REFERENCE/data, the top-level structure, every state-dict name / shape /
dtype and the set of pickle globals.  Both files are then loaded with the product loader, and the float64 oracle is checked against
the reference module on the real weights; a mismatch stops the script.

``vlfm.policy.utils.pointnav_policy`` imports ``gym``, which is absent: a stub ``gym`` / ``gym.spaces`` is injected (its names are
used only on the habitat branch, which is not taken without habitat).
"""
from __future__ import annotations

import json
import os
import pickletools
import sys
import tempfile
import types
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pointnav_oracle as po  # noqa: E402
from oracle import ref_import  # noqa: E402
from vlfm_b200.policy.pointnav_weights import convert_state_dict, load_checkpoint, random_state_dict  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
WRAPPED_STEPS = 12


def _stub_gym() -> None:
    if "gym" in sys.modules:
        return
    gym = types.ModuleType("gym")
    spaces = types.ModuleType("gym.spaces")

    class _Space:
        def __init__(self, *a, **k):
            pass

    spaces.Box = spaces.Dict = spaces.Discrete = _Space
    gym.spaces = spaces
    sys.modules["gym"] = gym
    sys.modules["gym.spaces"] = spaces


def reference_modules():
    ref_import._ensure_path()
    _stub_gym()
    import vlfm.policy.utils.non_habitat_policy.nh_pointnav_policy as nh  # type: ignore
    import vlfm.policy.utils.pointnav_policy as pp  # type: ignore

    assert not pp.HABITAT_BASELINES_AVAILABLE
    return nh, pp


class DiscreteRef(torch.nn.Module):
    """The reference's PointNavResNetNet(discrete_actions=True) + a Linear head with argmax (habitat's CategoricalNet mode)."""

    def __init__(self, nh, sd):
        super().__init__()
        self.net = nh.PointNavResNetNet(discrete_actions=True)
        self.linear = torch.nn.Linear(512, 4)
        net_sd = {k[4:].replace("prev_action_embedding.", "prev_action_embedding_discrete."): v for k, v in sd.items() if k.startswith("net.")}
        self.net.load_state_dict(net_sd)
        self.linear.load_state_dict({"weight": sd["action_distribution.linear.weight"], "bias": sd["action_distribution.linear.bias"]})

    def act(self, obs, hidden, prev, masks):
        feats, hidden, _ = self.net(obs, hidden, prev, masks)
        head = self.linear(feats)
        return head.argmax(1, keepdim=True), hidden, head, feats


class ContinuousRef:
    def __init__(self, nh, sd):
        self.policy = nh.PointNavResNetPolicy()
        self.policy.load_state_dict({k.replace("net.prev_action_embedding.", "net.prev_action_embedding_cont."): v
                                     for k, v in sd.items() if not k.startswith("critic.")})

    def act(self, obs, hidden, prev, masks):
        feats, hidden, _ = self.policy.net(obs, hidden, prev, masks)
        head = self.policy.action_distribution.mu_maybe_std(feats)
        return torch.tanh(head[:, :2]), hidden, head, feats


def reference_episode(model, frames, goals, masks, discrete):
    steps, B = frames.shape[:2]
    hidden = torch.zeros(B, 4, 512)
    prev = torch.zeros(B, 1, dtype=torch.long) if discrete else torch.zeros(B, 2)
    rec = {"head": [], "action": [], "features": [], "hidden": []}
    with torch.no_grad():
        for t in range(steps):
            obs = {"depth": torch.from_numpy(frames[t])[..., None], "pointgoal_with_gps_compass": torch.from_numpy(goals[t])}
            m = torch.from_numpy(masks[t])[:, None]
            action, hidden, head, feats = model.act(obs, hidden, prev, m)
            prev = action.clone()
            rec["head"].append(head.numpy().copy())
            rec["action"].append(action.numpy().copy())
            rec["features"].append(feats.numpy().copy())
            rec["hidden"].append(hidden.numpy().copy())
    return {k: np.stack(v) for k, v in rec.items()}


def live_cases(nh, pp):
    out = {}
    for ci, (layout, hw, B, steps, seed) in enumerate(po.LIVE_CASES):
        discrete = layout == "discrete"
        sd = random_state_dict(po.WEIGHT_SEEDS[layout], discrete)
        model = DiscreteRef(nh, sd) if discrete else ContinuousRef(nh, sd)
        frames = po.depth_frames(seed, steps, B, *hw)
        goals, masks = po.episode_script(seed, steps, B)
        if not discrete:
            # the policy's own act() must agree with the head + tanh restated above
            with torch.no_grad():
                obs = {"depth": torch.from_numpy(frames[0])[..., None], "pointgoal_with_gps_compass": torch.from_numpy(goals[0])}
                a, _ = model.policy.act(obs, torch.zeros(B, 4, 512), torch.zeros(B, 2), torch.from_numpy(masks[0])[:, None], deterministic=True)
                a2 = model.act(obs, torch.zeros(B, 4, 512), torch.zeros(B, 2), torch.from_numpy(masks[0])[:, None])[0]
                assert torch.equal(a, a2)
        rec = reference_episode(model, frames, goals, masks, discrete)
        p = f"c{ci}_"
        out[p + "head"] = rec["head"]
        out[p + "action"] = rec["action"]
        out[p + "features"] = rec["features"][list(po.RECORD_STEPS)]
        out[p + "hidden"] = rec["hidden"][list(po.RECORD_STEPS)]
        print(f"case {ci} {layout} {hw} B={B}: actions {np.unique(rec['action'].round(3)).size} distinct")
    # the real WrappedPointNavResNetPolicy at batch 1 (continuous: the only layout its non-habitat loader reads)
    sd = random_state_dict(po.WEIGHT_SEEDS["continuous"], False)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "pointnav.pth")
        torch.save(sd, path)
        wrapped = pp.WrappedPointNavResNetPolicy(path, device="cpu")
    layout, hw, _, _, seed = po.LIVE_CASES[2]
    frames = po.depth_frames(seed, WRAPPED_STEPS, 1, *hw)
    goals, masks = po.episode_script(seed, WRAPPED_STEPS, 1)
    masks[7, 0] = False
    acts = []
    with torch.no_grad():
        for t in range(WRAPPED_STEPS):
            obs = {"depth": frames[t][..., None].copy(), "pointgoal_with_gps_compass": goals[t].copy()}
            acts.append(wrapped.act(obs, torch.from_numpy(masks[t])[:, None], deterministic=True).numpy().copy())
    out["wrapped_action"] = np.stack(acts)
    out["wrapped_hidden"] = wrapped.pointnav_test_recurrent_hidden_states.numpy().copy()
    out["wrapped_masks"] = masks
    return out


def pickle_globals(path):
    z = zipfile.ZipFile(path)
    pk = [n for n in z.namelist() if n.endswith("data.pkl")][0]
    names, strings = set(), []
    for op, arg, _ in pickletools.genops(z.read(pk)):
        if op.name == "GLOBAL":
            names.add(arg.replace(" ", "."))
        elif op.name == "STACK_GLOBAL":
            names.add(strings[-2] + "." + strings[-1])
        elif op.name in ("SHORT_BINUNICODE", "BINUNICODE", "UNICODE"):
            strings.append(arg)
    return sorted(names)


def layout(nh):
    res = {}
    from vlfm_b200.policy.pointnav_weights import restricted_pickle

    for name in ("pointnav_weights.pth", "spot_pointnav_weights.pth"):
        path = os.path.join(ref_import.REFERENCE_ROOT, "data", name)
        obj = torch.load(path, map_location="cpu", pickle_module=restricted_pickle, weights_only=False)
        top = sorted(obj.keys()) if "state_dict" in obj else None
        sd = obj["state_dict"] if top else obj
        res[name] = {"top_level": top or "state_dict", "container": type(sd).__name__,
                     "tensors": [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()],
                     "pickle_globals": pickle_globals(path)}
        w, discrete = load_checkpoint(path)
        check_real(nh, w, discrete, name)
    return res


def check_real(nh, w, discrete, name):
    """The float64 oracle against the reference module (float64 as well) on the real weights: 8 steps, batch 2, 224 x 224.  The
    oracle forms cos / sin of the goal angle in float32, as the reference does on its float32 observations; the module here gets
    float64 goals, so the two differ by that rounding (~1e-8), not more."""
    B, steps = 2, 8
    frames = po.depth_frames(77, steps, B, 224, 224)
    goals, masks = po.episode_script(77, steps, B)
    model = DiscreteRef(nh, w) if discrete else ContinuousRef(nh, w)
    mods = [model] if discrete else [model.policy]
    for m in mods:
        m.double()
    if not discrete:
        # the reference embeds `masks * prev_actions.float()`: give the float64 Linear a float64 input (prev rounded to fp32)
        model.policy.net.prev_action_embedding_cont.register_forward_pre_hook(lambda mod, args: (args[0].double(),))
    orc = po.PointNavOracle(w, discrete)
    hidden = torch.zeros(B, 4, 512, dtype=torch.float64)
    prev = torch.zeros(B, 1, dtype=torch.long) if discrete else torch.zeros(B, 2, dtype=torch.float64)
    worst = 0.0
    with torch.no_grad():
        for t in range(steps):
            obs = {"depth": torch.from_numpy(frames[t]).double()[..., None], "pointgoal_with_gps_compass": torch.from_numpy(goals[t]).double()}
            m = torch.from_numpy(masks[t])[:, None]
            action, h_ref, head, _ = model.act(obs, hidden, prev, m)
            r = orc.step(torch.from_numpy(frames[t]), torch.from_numpy(goals[t]), torch.from_numpy(masks[t]), hidden, prev)
            d = max((r["head"] - head).abs().max().item(), (r["hidden"] - h_ref).abs().max().item())
            worst = max(worst, d)
            if d > 1e-6 or (discrete and not torch.equal(r["action"], action)):
                raise SystemExit(f"{name}: oracle differs from the reference module at step {t}: {d:.3e}")
            hidden, prev = h_ref, action
    print(f"{name}: {'discrete' if discrete else 'continuous'}, float64 oracle vs reference module max |diff| {worst:.3e} over {steps} steps")


def main():
    if not ref_import.available():
        raise SystemExit("set VLFM_REFERENCE to a checkout of bdaiinstitute/vlfm")
    nh, pp = reference_modules()
    lay = layout(nh)
    with open(os.path.join(OUT, "pointnav_layout.json"), "w") as f:
        json.dump(lay, f, indent=1, sort_keys=True)
    out = live_cases(nh, pp)
    np.savez_compressed(os.path.join(OUT, "live_pointnav.npz"), **out)
    print("wrote", os.path.join(OUT, "live_pointnav.npz"), sum(v.nbytes for v in out.values()), "bytes raw")


if __name__ == "__main__":
    main()
