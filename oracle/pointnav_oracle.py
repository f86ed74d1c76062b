"""Float64 functional restatement of the PointNav policy step (WrappedPointNavResNetPolicy.act in
vlfm/policy/utils/pointnav_policy.py), written from the architecture: ``F.conv2d``, ``F.group_norm``, ``F.max_pool2d`` and explicit
LSTM gate arithmetic over a dict of tensors keyed by checkpoint names (``vlfm_b200.policy.pointnav_weights.engine_shapes``).

    depth [B,H,W] in [0,1] -> area resize to the input size (rounded to fp32) -> avg_pool2d(2)
    -> conv 7x7 s2 p3 (1 -> 32), GN(16), ReLU, maxpool 3x3 s2 p1
    -> 4 stages x 2 BasicBlocks (32, 64, 128, 256; strides 1, 2, 2, 2): relu(GN(conv(relu(GN(conv x)))) + residual),
       residual = x or GN(conv1x1 s2 x)
    -> conv 3x3 (256 -> 128), GN(1), ReLU -> NCHW flatten (c*16 + y*4 + x) -> Linear(2048 -> 512), ReLU
    -> cat(visual, Linear(3 -> 32)(rho, cos -theta, sin -theta), prev-action embedding) -> 2-layer LSTM (h, c zeroed where
       mask is False; hidden layout [h_l0, h_l1, c_l0, c_l1]) -> head: logits (argmax) or mu | log_std (tanh(mu)).

``f16_convs=True`` rounds every conv operand (input map and weight) to fp16 first, as the engine's GEMMs do: the difference of
the two runs over an episode is the drift the GPU bars are derived from.  Also here: the seeded depth generator and episode
scripts of tests/golden/live_pointnav.npz (oracle/make_pointnav_golden.py), shared by that generator and the tests.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

BB = "net.visual_encoder.backbone."
STAGES = ((32, 1), (64, 2), (128, 2), (256, 2))
f64 = torch.float64


def area_resize(depth: torch.Tensor, hw) -> torch.Tensor:
    """torch's "area" interpolation (adaptive average pooling) of [B,H,W], computed in float64 and rounded to fp32."""
    d = torch.as_tensor(depth, dtype=f64)
    if tuple(d.shape[1:]) == tuple(hw):
        return d.float()
    return F.adaptive_avg_pool2d(d[:, None], tuple(hw))[:, 0].float()


class PointNavOracle:
    def __init__(self, sd: Dict[str, torch.Tensor], discrete: bool, f16_convs: bool = False, dtype=f64, device="cpu") -> None:
        """``dtype`` / ``device``: float64 on the CPU is the oracle; float32 on a GPU is the eager stand-in a benchmark times."""
        self.dt, self.dev = dtype, torch.device(device)
        self.w = {k: v.detach().to(self.dev, dtype) for k, v in sd.items()}
        self.discrete, self.f16 = discrete, f16_convs

    def _conv(self, x, name, stride, pad):
        w = self.w[name]
        if self.f16:
            x, w = x.half().to(self.dt), w.half().to(self.dt)
        return F.conv2d(x, w, stride=stride, padding=pad)

    def _gn(self, x, name, groups):
        return F.group_norm(x, groups, self.w[name + ".weight"], self.w[name + ".bias"], eps=1e-5)

    def encoder(self, depth_in: torch.Tensor) -> torch.Tensor:
        """depth at the network's input size [B,IH,IW] (fp32 values) -> the compression output [B,128,4,4] (float64)."""
        x = F.avg_pool2d(depth_in.to(self.dev, self.dt)[:, None], 2)
        x = F.relu(self._gn(self._conv(x, BB + "conv1.0.weight", 2, 3), BB + "conv1.1", 16))
        x = F.max_pool2d(x, 3, 2, 1)
        cin = 32
        for li, (c, stride) in enumerate(STAGES, start=1):
            for bi in range(2):
                p = f"{BB}layer{li}.{bi}."
                s = stride if bi == 0 else 1
                y = F.relu(self._gn(self._conv(x, p + "convs.0.weight", s, 1), p + "convs.1", 16))
                y = self._gn(self._conv(y, p + "convs.3.weight", 1, 1), p + "convs.4", 16)
                r = x
                if bi == 0 and (s != 1 or cin != c):
                    r = self._gn(self._conv(x, p + "downsample.0.weight", s, 0), p + "downsample.1", 16)
                x = F.relu(y + r)
            cin = c
        x = F.relu(self._gn(self._conv(x, "net.visual_encoder.compression.0.weight", 1, 1), "net.visual_encoder.compression.1", 1))
        return x

    def step(self, depth_in, goal, masks, hidden, prev) -> Dict[str, torch.Tensor]:
        """One act() step.  depth_in [B,IH,IW] at the input size; goal [B,2] (rho, theta); masks [B] bool; hidden [B,4,512];
        prev [B,1] int (discrete) or [B,2] float.  Returns float64 'visual', 'features' (h_l1'), 'head' [B,4], 'hidden'
        [B,4,512] and 'action' ([B,1] int64 or [B,2] float64)."""
        w = self.w
        B = depth_in.shape[0]
        m = torch.as_tensor(masks, dtype=torch.bool).reshape(B).to(self.dev)
        vis = self.encoder(torch.as_tensor(depth_in))
        vis = F.relu(vis.reshape(B, -1) @ w["net.visual_fc.1.weight"].T + w["net.visual_fc.1.bias"])
        g = torch.as_tensor(goal).to(self.dev, torch.float32)
        # the reference forms (rho, cos(-theta), sin(-theta)) in float32
        gf = torch.stack([g[:, 0], torch.cos(-g[:, 1]), torch.sin(-g[:, 1])], -1).to(self.dt)
        goal_f = gf @ w["net.tgt_embeding.weight"].T + w["net.tgt_embeding.bias"]
        if self.discrete:
            idx = torch.where(m, torch.as_tensor(prev).to(self.dev).reshape(B).long() + 1, torch.zeros(B, dtype=torch.long, device=self.dev))
            prev_f = w["net.prev_action_embedding.weight"][idx]
        else:
            p = torch.as_tensor(prev).to(self.dev, self.dt).reshape(B, 2) * m[:, None].to(self.dt)
            prev_f = p @ w["net.prev_action_embedding.weight"].T + w["net.prev_action_embedding.bias"]
        x = torch.cat([vis, goal_f, prev_f], 1)
        hs = torch.as_tensor(hidden).to(self.dev, self.dt).clone()
        hs[~m] = 0
        h_new, c_new = [], []
        for l in range(2):
            h, c = hs[:, l], hs[:, 2 + l]
            gates = (x @ w[f"net.state_encoder.rnn.weight_ih_l{l}"].T + w[f"net.state_encoder.rnn.bias_ih_l{l}"]
                     + h @ w[f"net.state_encoder.rnn.weight_hh_l{l}"].T + w[f"net.state_encoder.rnn.bias_hh_l{l}"])
            i, f, gg, o = gates.chunk(4, 1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            h_new.append(h)
            c_new.append(c)
            x = h
        hk = "action_distribution.linear." if self.discrete else "action_distribution.mu_maybe_std."
        head = x @ w[hk + "weight"].T + w[hk + "bias"]
        if self.discrete:
            action = head.argmax(1, keepdim=True)
        else:
            action = torch.tanh(head[:, :2])
        return {"visual": vis, "features": x, "head": head, "hidden": torch.stack(h_new + c_new, 1), "action": action}


def top2_gap(head: torch.Tensor) -> torch.Tensor:
    """Per row: the largest logit minus the second largest."""
    t = head.topk(2, dim=1).values
    return t[:, 0] - t[:, 1]


# --------------------------------------------------------------------------------------------- episode scripts (fixtures)
# (layout, input (H, W), batch, steps, seed).  Depth frames come from depth_frames(seed, ...); masks and goals from the script.
LIVE_CASES = [("discrete", (224, 224), 3, 20, 31), ("discrete", (212, 240), 3, 16, 32),
              ("continuous", (224, 224), 3, 20, 33), ("continuous", (212, 240), 3, 16, 34)]
WEIGHT_SEEDS = {"discrete": 4, "continuous": 6}
RECORD_STEPS = (0, 5, 11)   # steps at which features and hidden states are stored

# GPU bars (max |engine - float64 oracle| over every step of an episode, per quantity).  Each is 2x the largest drift of the
# float64 oracle with every conv operand rounded to fp16 (``f16_convs=True``) from the exact float64 oracle, previous actions of
# the exact run fed to both, measured before the first GPU run over LIVE_CASES plus 64-step batch-1 episodes (224^2 discrete,
# 212x240 continuous) and 16-step batch-8 episodes of both layouts: visual 1.13e-2, features 4.82e-3, head 5.86e-3, hidden
# 7.56e-2 (the cell states reach |c| ~ 20).
GPU_BARS = {"visual": 2.3e-2, "features": 9.7e-3, "head": 1.2e-2, "hidden": 1.6e-1}


def depth_frames(seed: int, steps: int, B: int, H: int, W: int) -> np.ndarray:
    """[steps, B, H, W] float32 in [0, 1]: smooth depth (a tilted floor plane plus low-frequency blobs that drift per step) with
    zero holes (missing returns) in a few patches."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    out = np.empty((steps, B, H, W), np.float32)
    params = rng.uniform(0, 1, (B, 6, 5))
    for t in range(steps):
        for b in range(B):
            p = params[b]
            d = 0.3 + 0.5 * (1 - yy) * (0.6 + 0.4 * p[0, 0])
            for k in range(6):
                cy, cx = p[k, 1] + 0.03 * t * np.sin(k + b), p[k, 2] + 0.03 * t * np.cos(k - b)
                d += 0.25 * (p[k, 3] - 0.5) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (0.02 + 0.05 * p[k, 4]))
            d = np.clip(d, 0, 1)
            for _ in range(3):
                h0, w0 = rng.integers(0, H - 8), rng.integers(0, W - 8)
                d[h0:h0 + rng.integers(2, 8), w0:w0 + rng.integers(2, 8)] = 0
            out[t, b] = d
    return out


def episode_script(seed: int, steps: int, B: int):
    """(goals [steps,B,2] float32, masks [steps,B] bool): mask False at step 0 for every env, and env 1 at steps//3, env 2 at
    2*steps//3 (mid-episode resets).  Goals drift slowly, theta covers both turn directions."""
    rng = np.random.default_rng(1000 + seed)
    rho0 = rng.uniform(0.5, 5.0, B)
    th0 = rng.uniform(-np.pi, np.pi, B)
    t = np.arange(steps)[:, None]
    goals = np.stack([rho0 + 0.1 * np.sin(0.3 * t + rho0), np.angle(np.exp(1j * (th0 + 0.25 * t)))], -1).astype(np.float32)
    masks = np.ones((steps, B), bool)
    masks[0] = False
    if B > 1:
        masks[steps // 3, 1] = False
    if B > 2:
        masks[2 * steps // 3, 2] = False
    return goals, masks


def run_episode(orc: PointNavOracle, frames, goals, masks, prev_feed: Optional[list] = None):
    """Oracle over an episode with its own actions fed back (or ``prev_feed[t]`` as the previous action of step t).  -> list of
    step dicts."""
    steps, B = frames.shape[:2]
    hidden = torch.zeros(B, 4, 512, dtype=f64)
    prev = torch.zeros(B, 1, dtype=torch.long) if orc.discrete else torch.zeros(B, 2, dtype=f64)
    out = []
    for t in range(steps):
        if prev_feed is not None:
            prev = prev_feed[t]
        r = orc.step(torch.from_numpy(frames[t]), torch.from_numpy(goals[t]), torch.from_numpy(masks[t]), hidden, prev)
        hidden, prev = r["hidden"], r["action"]
        out.append(r)
    return out
