"""The PointNav policy behind the reference's class surface (vlfm/policy/utils/pointnav_policy.py), and a batched form of it.

``PointNavBatch`` keeps a hidden state and previous action per environment and steps any subset of environments in one launch
sequence (a CUDA graph per batch size and frame size).  ``WrappedPointNavResNetPolicy`` is its one-environment instance with the
reference's ``act`` / ``reset`` and its ``pointnav_test_recurrent_hidden_states`` / ``pointnav_prev_actions`` tensors.
"""
from __future__ import annotations

import os
from typing import Any, Dict, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .pointnav_engine import MAX_GEMV_BATCH, PointNavEngine
from .pointnav_weights import convert_state_dict, load_checkpoint, random_state_dict

WeightsArg = Union[None, str, Dict[str, torch.Tensor]]


def resolve_weights(weights: WeightsArg, synthetic: bool = False, seed: int = 0, discrete: bool = True) -> Tuple[Dict[str, torch.Tensor], bool]:
    """A state dict (either checkpoint layout) or a checkpoint path, else ``VLFM_POINTNAV_WEIGHTS``.  Without any, raises unless
    ``synthetic=True`` (seeded random weights: tests / benchmarks only)."""
    if isinstance(weights, dict):
        return convert_state_dict(weights)
    path = weights or os.environ.get("VLFM_POINTNAV_WEIGHTS", "")
    if path:
        return load_checkpoint(path)
    if synthetic:
        return convert_state_dict(random_state_dict(seed, discrete))
    raise FileNotFoundError("PointNav: no checkpoint configured (ckpt_path / VLFM_POINTNAV_WEIGHTS unset, no state dict).  Pass "
                            "synthetic=True to run on seeded random weights (tests / benchmarks only).")


def _to_device(x: Any, device: torch.device, dtype=torch.float32) -> torch.Tensor:
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    return torch.as_tensor(x).to(device=device, dtype=dtype)


class PointNavBatch:
    def __init__(self, weights: WeightsArg = None, max_batch: int = 1, input_hw: Tuple[int, int] = (224, 224), device="cuda", *,
                 num_envs: Optional[int] = None, synthetic: bool = False, seed: int = 0, discrete: bool = True) -> None:
        """``weights``: a state dict or checkpoint path (see ``resolve_weights``); ``max_batch`` <= 64 environments per step;
        ``input_hw`` the network's input size (depth of any size is area-resized to it); ``num_envs`` state slots (default
        ``max_batch``)."""
        w, self.discrete = resolve_weights(weights, synthetic, seed, discrete)
        self.device = torch.device(device)
        self.engine = PointNavEngine(w, self.discrete, max_batch=max_batch, input_hw=input_hw, num_envs=num_envs, device=self.device)
        self.max_batch, self.num_envs = max_batch, self.engine.num_envs

    @property
    def hidden_states(self) -> torch.Tensor:
        """[num_envs, 4, 512] = [h_l0, h_l1, c_l0, c_l1] per environment (the live tensor)."""
        return self.engine.hidden

    @property
    def prev_actions(self) -> torch.Tensor:
        """[num_envs, 1] int64 (discrete) or [num_envs, 2] float32 (the live tensor)."""
        return self.engine.prev

    def _env_ids(self, env_ids, B: int) -> torch.Tensor:
        if env_ids is None:
            ids = torch.arange(B)
        else:
            ids = torch.as_tensor(np.asarray(env_ids) if not isinstance(env_ids, torch.Tensor) else env_ids.cpu()).reshape(-1).long()
        if ids.numel() != B or (ids < 0).any() or (ids >= self.num_envs).any() or ids.unique().numel() != B:
            raise ValueError(f"PointNav: env_ids must be {B} distinct slots in [0, {self.num_envs}), got {ids.tolist()}")
        return ids.to(self.device, torch.int32)

    def act(self, depth, pointgoal, masks, env_ids: Optional[Sequence[int]] = None, deterministic: bool = True) -> torch.Tensor:
        """depth [B,H,W] (or [B,H,W,1]) in [0,1] at any size, pointgoal [B,2] (rho, theta), masks [B] (False: first step of an
        episode) -> action [B,1] int64 (discrete) or [B,2] float32 on the device.  Each environment's hidden state and previous
        action (slot env_ids[b], default b) are updated.  ``deterministic=False`` samples from the head's distribution with torch."""
        depth = _to_device(depth, self.device)
        if depth.dim() == 4 and depth.shape[-1] == 1:
            depth = depth[..., 0]
        B = depth.shape[0]
        if depth.dim() != 3 or not 1 <= B <= self.max_batch:
            raise ValueError(f"PointNav: depth must be [B,H,W] with 1 <= B <= {self.max_batch}, got {tuple(depth.shape)}")
        goal = _to_device(pointgoal, self.device).reshape(B, 2)
        m = _to_device(masks, self.device, torch.bool).reshape(B)
        ids = self._env_ids(env_ids, B)
        eng = self.engine
        eng.step(depth, goal, m, ids)
        if deterministic:
            return eng.action[:B].clone()
        head = eng.head[:B]
        if self.discrete:
            action = torch.distributions.Categorical(logits=head).sample().unsqueeze(1)
        else:
            std = torch.exp(torch.clamp(head[:, 2:], -5.0, 2.0))
            action = torch.normal(torch.tanh(head[:, :2]), std)
        eng.prev[ids.long()] = action
        return action

    def reset(self, env_ids: Optional[Sequence[int]] = None) -> None:
        """Zero the hidden state and previous action of ``env_ids`` (default: every environment)."""
        idx = slice(None) if env_ids is None else torch.as_tensor(list(env_ids), dtype=torch.long, device=self.device)
        self.engine.hidden[idx] = 0
        self.engine.prev[idx] = 0


class WrappedPointNavResNetPolicy:
    """pointnav_policy.py:51-128 for one environment: ``act(observations, masks, deterministic)`` with observations
    {"depth": [1,H,W,1], "pointgoal_with_gps_compass": [1,2]} (numpy or torch), and ``reset()``."""

    def __init__(self, ckpt_path: Optional[str] = None, device: Union[str, torch.device] = "cuda", *, input_hw: Tuple[int, int] = (224, 224),
                 state_dict: Optional[Dict[str, torch.Tensor]] = None, synthetic: bool = False, seed: int = 0, discrete: bool = True) -> None:
        """Weights: ``state_dict``, else the file ``ckpt_path`` or ``VLFM_POINTNAV_WEIGHTS``; raises without any unless
        ``synthetic=True``.  ``input_hw``: the network's input size (``depth_image_shape``; depth of another size is
        area-resized to it)."""
        if isinstance(device, str):
            device = torch.device(device)
        self.device = device
        self.batch = PointNavBatch(state_dict if state_dict is not None else ckpt_path, 1, input_hw, device, synthetic=synthetic,
                                   seed=seed, discrete=discrete)

    @property
    def pointnav_test_recurrent_hidden_states(self) -> torch.Tensor:
        """[1, 4, 512] float32"""
        return self.batch.hidden_states

    @property
    def pointnav_prev_actions(self) -> torch.Tensor:
        """[1, 1] int64 (discrete) or [1, 2] float32"""
        return self.batch.prev_actions

    def act(self, observations: Dict[str, Any], masks, deterministic: bool = False) -> torch.Tensor:
        return self.batch.act(observations["depth"], observations["pointgoal_with_gps_compass"], masks, deterministic=deterministic)

    def reset(self) -> None:
        self.batch.reset()


__all__ = ["PointNavBatch", "WrappedPointNavResNetPolicy", "resolve_weights", "MAX_GEMV_BATCH"]
