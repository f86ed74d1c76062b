"""The float64 PointNav oracle (oracle/pointnav_oracle.py) against what the reference's own modules computed in float32 on the CPU
(tests/golden/live_pointnav.npz, oracle/make_pointnav_golden.py): both checkpoint layouts, 224 x 224 and 212 x 240 input, batch
3 with mid-episode resets, and the real WrappedPointNavResNetPolicy at batch 1.

Bars: the reference runs in float32 through ~20 conv / GroupNorm layers and an LSTM whose cell state reaches |c| ~ 20; the
differences seen are 5e-6 (head, features) and 4e-5 (hidden).  The bars are ~10x that: float32 rounding, not a formula error
(a wrong gate order, flatten order or mask rule moves these by 1e-2 or more)."""
import numpy as np
import pytest
import torch

from oracle import pointnav_oracle as po
from vlfm_b200.policy.pointnav_weights import convert_state_dict, random_state_dict

BARS = {"head": 5e-5, "features": 5e-5, "hidden": 3e-4}


@pytest.fixture(scope="module")
def live():
    return dict(np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "live_pointnav.npz")))


def _oracle(layout):
    d = layout == "discrete"
    w, discrete = convert_state_dict(random_state_dict(po.WEIGHT_SEEDS[layout], d))
    assert discrete == d
    return po.PointNavOracle(w, d)


@pytest.mark.parametrize("ci", range(len(po.LIVE_CASES)))
def test_oracle_matches_reference_modules(live, ci):
    layout, hw, B, steps, seed = po.LIVE_CASES[ci]
    d = layout == "discrete"
    orc = _oracle(layout)
    frames = po.depth_frames(seed, steps, B, *hw)
    goals, masks = po.episode_script(seed, steps, B)
    acts = live[f"c{ci}_action"]
    # the reference's previous actions are fed to the oracle, so a continuous action's rounding cannot carry over
    zero = torch.zeros(B, 1, dtype=torch.long) if d else torch.zeros(B, 2, dtype=torch.float64)
    res = po.run_episode(orc, frames, goals, masks, prev_feed=[zero] + [torch.from_numpy(a) for a in acts[:-1]])
    head = np.stack([r["head"].numpy() for r in res])
    assert np.abs(head - live[f"c{ci}_head"]).max() < BARS["head"]
    ours = np.stack([r["action"].numpy() for r in res])
    if d:
        assert np.array_equal(ours, acts)
    else:
        assert np.abs(ours - acts).max() < BARS["head"]
    for k in ("features", "hidden"):
        got = np.stack([res[s][k].numpy() for s in po.RECORD_STEPS])
        assert np.abs(got - live[f"c{ci}_{k}"]).max() < BARS[k], k


def test_oracle_matches_wrapped_policy(live):
    """The reference's WrappedPointNavResNetPolicy (continuous, batch 1; mask False at steps 0 and 7), own actions fed back."""
    layout, hw, _, _, seed = po.LIVE_CASES[2]
    masks = live["wrapped_masks"]
    steps = masks.shape[0]
    frames = po.depth_frames(seed, steps, 1, *hw)
    goals, _ = po.episode_script(seed, steps, 1)
    res = po.run_episode(_oracle(layout), frames, goals, masks)
    acts = np.stack([r["action"].numpy() for r in res])
    assert np.abs(acts - live["wrapped_action"]).max() < BARS["head"]
    assert np.abs(res[-1]["hidden"].numpy() - live["wrapped_hidden"]).max() < BARS["hidden"]


def test_area_resize_identity_and_scaling():
    rng = np.random.default_rng(0)
    d = rng.random((2, 30, 41)).astype(np.float32)
    assert torch.equal(po.area_resize(d, (30, 41)), torch.from_numpy(d))
    r = po.area_resize(d, (10, 41))
    ref = d.astype(np.float64).reshape(2, 10, 3, 41).mean(2)
    assert np.abs(r.numpy() - ref).max() < 1e-7
