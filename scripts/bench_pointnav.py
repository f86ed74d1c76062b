"""PointNav policy step on the GPU: device time per step (CUDA-graph replay, CUDA events) at B = 1, 8 and 32 for 224 x 224 input,
alternated with the float32 torch-eager restatement of the same step (oracle/pointnav_oracle.py) as the stand-in for what the
reference runs; the host latency of WrappedPointNavResNetPolicy.act including the action's D2H; launches per step; algorithmic
FLOPs and weight bytes against the H100 SXM data-sheet bounds; the card's name and power limit, read in the same run.

Usage: python scripts/bench_pointnav.py [--iters N] [--out FILE]    (seeded synthetic weights; prints one JSON object)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import pointnav_oracle as po  # noqa: E402
from vlfm_b200.policy.pointnav_policy import PointNavBatch, WrappedPointNavResNetPolicy  # noqa: E402
from vlfm_b200.policy.pointnav_weights import convert_state_dict, random_state_dict  # noqa: E402

PEAK_F16_TFLOPS, PEAK_F32_TFLOPS, PEAK_TBPS = 989.0, 67.0, 3.35   # H100 SXM data sheet (dense), at up to 700 W


def encoder_flops(hw=(224, 224)) -> float:
    """2 * MACs of every conv of the encoder for one frame, from the shapes."""
    from vlfm_b200.policy.pointnav_engine import spatial_plan

    s = spatial_plan(hw)
    f = 2.0 * s[1][0] * s[1][1] * 32 * 49
    cin = 32
    for (c, stride), (h, w) in zip(po.STAGES, s[2:]):
        f += 2.0 * h * w * c * 9 * cin + 2.0 * h * w * c * 9 * c            # block 0
        if cin != c or stride != 1:
            f += 2.0 * h * w * c * cin                                       # downsample
        f += 2.0 * 2 * h * w * c * 9 * c                                     # block 1
        cin = c
    return f + 2.0 * 16 * 128 * 9 * 256                                      # compression


def recurrent_flops() -> float:
    return 2.0 * (512 * 2048 + 2048 * 1088 + 2048 * 1024 + 4 * 512)


def weight_bytes(w) -> dict:
    conv = sum(v.numel() for v in w.values() if v.dim() == 4) * 2
    fp32 = sum(v.numel() for k, v in w.items() if v.dim() != 4) * 4
    return {"conv_fp16": conv, "recurrent_fp32": fp32}


def time_events(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1e3   # us


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": q.stdout.strip(), "torch_name": torch.cuda.get_device_name(0)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pointnav needs a CUDA device")
    torch.cuda.set_device(0)
    sd = random_state_dict(0, True)
    w, _ = convert_state_dict(sd)
    res = {"card": card(), "input": [224, 224], "encoder_gflop_per_frame": encoder_flops() / 1e9,
           "recurrent_mflop_per_env": recurrent_flops() / 1e6, "weight_bytes": weight_bytes(w), "batches": {}}
    eager = po.PointNavOracle(w, True, dtype=torch.float32, device="cuda")
    for B in (1, 8, 32):
        pol = PointNavBatch(sd, max_batch=B)
        frames = torch.from_numpy(po.depth_frames(1, 1, B, 224, 224)[0]).cuda()
        goal = torch.rand(B, 2, device="cuda")
        masks = torch.ones(B, dtype=torch.bool, device="cuda")
        ids = torch.arange(B, device="cuda")
        eng = pol.engine
        hidden = torch.zeros(B, 4, 512, device="cuda")
        prev = torch.zeros(B, 1, dtype=torch.long, device="cuda")
        with torch.inference_mode():
            g_replay = lambda: eng.step(frames, goal, masks, ids)
            g_eager = lambda: eager.step(frames, goal, masks, hidden, prev)
            for _ in range(10):
                g_replay()
                g_eager()
            torch.cuda.synchronize()
            ours, ref = [], []
            for _ in range(a.rounds):
                ours.append(time_events(g_replay, a.iters))
                ref.append(time_events(g_eager, max(20, a.iters // 10)))
        t = min(ours)
        enc = encoder_flops() * B
        wb = sum(res["weight_bytes"].values())
        res["batches"][B] = {
            "engine_us_per_step": ours, "torch_fp32_eager_us_per_step": ref, "speedup": min(ref) / t,
            "launches_per_step": eng.launches_per_step(B),
            "encoder_tflops_achieved": enc / (t * 1e-6) / 1e12,
            "bound_us_f16_compute": enc / (PEAK_F16_TFLOPS * 1e12) * 1e6 + recurrent_flops() * B / (PEAK_F32_TFLOPS * 1e12) * 1e6,
            "bound_us_weight_bytes": wb / (PEAK_TBPS * 1e12) * 1e6,
        }
    wrapped = WrappedPointNavResNetPolicy(state_dict=sd)
    obs = {"depth": po.depth_frames(2, 1, 1, 224, 224)[0][..., None], "pointgoal_with_gps_compass": torch.rand(1, 2).numpy()}
    m = torch.ones(1, dtype=torch.bool, device="cuda")
    for _ in range(20):
        wrapped.act(dict(obs), m, deterministic=True).cpu()
    lat = []
    for _ in range(200):
        t0 = time.perf_counter()
        wrapped.act(dict(obs), m, deterministic=True).cpu()
        lat.append((time.perf_counter() - t0) * 1e6)
    lat.sort()
    res["wrapped_act_host_us"] = {"median": lat[len(lat) // 2], "p90": lat[int(len(lat) * 0.9)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
