"""BASELINE.json configs[2]: the FULL policy step for a batch of environments on one H100 (vlfm_b200/utils/full_step.py:
GroundingDINO detect + BLIP-2 ITC + batched ObstacleMap update + ValueMap fuse + frontier scoring) with per-component
CUDA-event times.  bench.py runs the same harness for its `extra` block; this script is for one-off sweeps.

    python scripts/bench_full_step.py --batch 32 --steps 6 --warmup 3 [--no-gdino] [--grid 1000] [--ppm 20] [--hw 480 640]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vlfm_b200.utils.full_step import FullStep  # noqa: E402
from vlfm_b200.utils.peaks import peaks  # noqa: E402
from vlfm_b200.vlm.blip2_config import Blip2Dims, random_state_dict  # noqa: E402
from vlfm_b200.vlm.blip2itm import BLIP2ITM  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--grid", type=int, default=1000)
    ap.add_argument("--ppm", type=int, default=20)
    ap.add_argument("--hw", type=int, nargs=2, default=[480, 640])
    ap.add_argument("--hole-thresh", type=int, default=100000)
    ap.add_argument("--no-gdino", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    dims = Blip2Dims()
    itm = BLIP2ITM(state_dict=random_state_dict(dims, 0), dims=dims, max_batch=a.batch, device=dev)
    gd = None
    if not a.no_gdino:
        from vlfm_b200.vlm.grounding_dino import GroundingDINO

        gd = GroundingDINO(device=dev, synthetic=True)
    fs = FullStep(dev, a.batch, a.hw[0], a.hw[1], a.grid, a.ppm, itm, gd, frames_per_env=a.steps + a.warmup, hole_thresh=a.hole_thresh,
                  bound_m=0.015 * a.grid)
    r = fs.run(a.steps, a.warmup)
    pk, src = peaks()
    r["grid_rooflines"] = fs.grid_rooflines(float(pk["hbm_gbs"]))
    r["peak_hbm_gbs"], r["peak_source"] = float(pk["hbm_gbs"]), src
    r["config"] = {"workload": f"full step, batch={a.batch} envs, {a.hw[1]}x{a.hw[0]} RGB-D, {a.grid}^2 grid at {a.ppm} px/m, 1xH100", "data": "synthetic"}
    print(json.dumps(r))


if __name__ == "__main__":
    main()
