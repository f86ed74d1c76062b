"""The PointNav policy on the GPU (vlfm_b200/policy) against the float64 oracle over whole episodes, on seeded weights of both
checkpoint layouts: 64 steps at batch 1, 16 steps at batches 3 and 32; 224 x 224 and 212 x 240 input, and frames of another
size area-resized to it; mid-episode resets by mask and by reset(env_ids); permuted env_ids.

Bars: oracle.pointnav_oracle.GPU_BARS, derived before the first GPU run from the oracle alone (2x the drift that fp16 conv
operands cause over such episodes).  The oracle's previous actions are fed to the engine, so one flipped discrete action cannot
fork the rest of an episode; a discrete action must equal the oracle's wherever the oracle's top-2 logit gap exceeds the head
bar."""
import numpy as np
import pytest
import torch

from oracle import pointnav_oracle as po
from vlfm_b200.policy.pointnav_policy import PointNavBatch, WrappedPointNavResNetPolicy
from vlfm_b200.policy.pointnav_weights import convert_state_dict, random_state_dict

pytestmark = pytest.mark.gpu
BARS = po.GPU_BARS


def _weights(layout):
    return random_state_dict(po.WEIGHT_SEEDS[layout], layout == "discrete")


def _episode(layout, hw, B, steps, seed, frame_hw=None, env_perm=None, reset_env=None):
    """Engine vs oracle over one episode; returns the worst |diff| per quantity."""
    d = layout == "discrete"
    sd = _weights(layout)
    w, _ = convert_state_dict(sd)
    orc = po.PointNavOracle(w, d)
    E = B + 2
    pol = PointNavBatch(sd, max_batch=B, input_hw=hw, num_envs=E)
    src = frame_hw or hw
    frames = po.depth_frames(seed, steps, B, *src)
    goals, masks = po.episode_script(seed, steps, B)
    ids = torch.arange(B) if env_perm is None else torch.as_tensor(env_perm)
    hidden = torch.zeros(B, 4, 512, dtype=torch.float64)
    prev = torch.zeros(B, 1, dtype=torch.long) if d else torch.zeros(B, 2, dtype=torch.float64)
    worst = {k: 0.0 for k in BARS}
    decided = 0
    for t in range(steps):
        if reset_env is not None and t == steps // 2:
            # reset(env_ids) on the engine == a zero state and previous action on the oracle's side
            pol.reset([int(ids[reset_env])])
            hidden[reset_env] = 0
            prev[reset_env] = 0
        # the oracle's previous action goes to the engine as well
        pol.prev_actions[ids.long()] = prev.to(pol.prev_actions.dtype).cuda()
        x = po.area_resize(frames[t], hw)
        r = orc.step(x, torch.from_numpy(goals[t]), torch.from_numpy(masks[t]), hidden, prev)
        a = pol.act(torch.from_numpy(frames[t]), goals[t], masks[t], env_ids=ids.tolist())
        eng = pol.engine
        got = {"visual": None, "features": eng.features[:B], "head": eng.head[:B], "hidden": pol.hidden_states[ids.long()]}
        vis_ref = r["visual"]
        got["visual"] = torch.relu(eng.visual[:B].double() @ eng.w["net.visual_fc.1.weight"].double().T + eng.w["net.visual_fc.1.bias"].double())
        for k in BARS:
            ref = vis_ref if k == "visual" else r[k]
            worst[k] = max(worst[k], (got[k].double().cpu() - ref).abs().max().item())
        if d:
            gap = po.top2_gap(r["head"])
            sure = gap > BARS["head"]
            assert torch.equal(a.cpu()[sure], r["action"][sure]), f"step {t}: {a.cpu().tolist()} vs {r['action'].tolist()}"
            decided += int(sure.sum())
        else:
            assert (a.cpu().double() - r["action"]).abs().max() < BARS["head"]
        hidden, prev = r["hidden"], r["action"]
    for k in BARS:
        assert worst[k] < BARS[k], f"{k}: {worst[k]:.3e} >= {BARS[k]:.3e}"
    if d:
        assert decided >= steps * B // 2
    return worst


@pytest.mark.parametrize("layout", ["discrete", "continuous"])
def test_episode_batch1_64_steps(layout):
    hw = (224, 224) if layout == "discrete" else (212, 240)
    _episode(layout, hw, 1, 64, 51)


@pytest.mark.parametrize("layout,hw", [("discrete", (224, 224)), ("continuous", (212, 240)), ("continuous", (224, 224)),
                                       ("discrete", (212, 240))])
def test_episode_batch3_resets_and_permuted_ids(layout, hw):
    _episode(layout, hw, 3, 16, 52, env_perm=[4, 0, 2], reset_env=0)


@pytest.mark.parametrize("layout", ["discrete", "continuous"])
def test_episode_batch32_resized_frames(layout):
    _episode(layout, (224, 224), 32, 16, 53, frame_hw=(240, 320))


def test_graph_replay_equals_eager_and_repeats():
    sd = _weights("discrete")
    B = 3
    frames = po.depth_frames(60, 4, B, 224, 224)
    goals, masks = po.episode_script(60, 4, B)
    runs = []
    for graph in (True, False, True):
        pol = PointNavBatch(sd, max_batch=B)
        pol.engine.use_graph = graph
        outs = []
        for t in range(4):
            pol.engine.step(torch.from_numpy(frames[t]).cuda(), torch.from_numpy(goals[t]).cuda(), torch.from_numpy(masks[t]).cuda(),
                            torch.arange(B).cuda())
            outs.append((pol.engine.head[:B].clone(), pol.hidden_states.clone(), pol.engine.action[:B].clone()))
        assert ((B, 224, 224) in pol.engine.graphs.captured) == graph
        runs.append(outs)
    for a, b in zip(runs[0], runs[1]):
        for x, y in zip(a, b):
            assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x, y.view(torch.int32) if y.dtype == torch.float32 else y)
    for a, b in zip(runs[0], runs[2]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


@pytest.mark.parametrize("layout", ["discrete", "continuous"])
def test_wrapped_policy_surface(layout):
    d = layout == "discrete"
    pol = WrappedPointNavResNetPolicy(state_dict=_weights(layout), device="cuda")
    assert pol.pointnav_test_recurrent_hidden_states.shape == (1, 4, 512)
    assert pol.pointnav_prev_actions.shape == ((1, 1) if d else (1, 2))
    assert pol.pointnav_prev_actions.dtype == (torch.long if d else torch.float32)
    frames = po.depth_frames(61, 3, 1, 224, 224)
    goals, _ = po.episode_script(61, 3, 1)
    obs_np = {"depth": frames[0][..., None], "pointgoal_with_gps_compass": goals[0]}
    a0 = pol.act(obs_np, torch.tensor([False], device="cuda"), deterministic=True)
    assert a0.shape == ((1, 1) if d else (1, 2)) and a0.dtype == (torch.long if d else torch.float32) and a0.is_cuda
    assert torch.equal(pol.pointnav_prev_actions, a0)
    h1 = pol.pointnav_test_recurrent_hidden_states.clone()
    assert h1.abs().sum() > 0
    obs_t = {"depth": torch.from_numpy(frames[1][..., None]).cuda(), "pointgoal_with_gps_compass": torch.from_numpy(goals[1]).cuda()}
    a1 = pol.act(obs_t, torch.tensor([[True]], device="cuda"), deterministic=True)
    # the oracle from the carried state and previous action
    w, _ = convert_state_dict(_weights(layout))
    r = po.PointNavOracle(w, d).step(torch.from_numpy(frames[1]), torch.from_numpy(goals[1]), np.array([True]), h1.cpu(), a0.cpu())
    assert (pol.pointnav_test_recurrent_hidden_states.cpu().double() - r["hidden"]).abs().max() < BARS["hidden"]
    assert torch.equal(pol.pointnav_prev_actions, a1)
    pol.reset()
    assert not pol.pointnav_test_recurrent_hidden_states.any() and not pol.pointnav_prev_actions.any()


def test_wrapped_policy_raises_without_checkpoint(monkeypatch):
    monkeypatch.delenv("VLFM_POINTNAV_WEIGHTS", raising=False)
    with pytest.raises(FileNotFoundError):
        WrappedPointNavResNetPolicy()
    with pytest.raises(ValueError):
        PointNavBatch(_weights("discrete"), max_batch=2).act(np.zeros((2, 224, 224), np.float32), np.zeros((2, 2)), [True, True], env_ids=[1, 1])
    with pytest.raises(ValueError):
        PointNavBatch(_weights("discrete"), input_hw=(160, 160))     # a 3 x 3 final map


@pytest.mark.parametrize("layout", ["discrete", "continuous"])
def test_sampling_shapes_and_seed(layout):
    d = layout == "discrete"
    B = 4
    frames = po.depth_frames(62, 2, B, 224, 224)
    goals, masks = po.episode_script(62, 2, B)
    outs = []
    for _ in range(2):
        pol = PointNavBatch(_weights(layout), max_batch=B)
        torch.manual_seed(123)
        acts = [pol.act(frames[t], goals[t], masks[t], deterministic=False) for t in range(2)]
        outs.append(acts)
        for a in acts:
            assert a.shape == ((B, 1) if d else (B, 2)) and a.dtype == (torch.long if d else torch.float32)
        assert torch.equal(pol.prev_actions[:B], acts[-1])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
