"""Per-kernel device-time table of graph-replayed configs[1] steps (ITM cosine + value-map update, batch 1).

torch.profiler with CUDA activities records `--steps` steps after warm-up (the step's CUDA graph is captured during warm-up,
so the profiled window is what bench.py times).  Writes OUT/kernels.md (one row per kernel name: launches per step, total us
per step, share of device time) and OUT/kernels.json, and prints the table.

  python scripts/kernel_table.py --out DIR [--steps 10] [--batch 1]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from bench import FOV, G, MAX_D, MIN_D, NFRAMES, PROMPT, make_frames
from vlfm_b200.mapping.value_map import ValueMapBatch
from vlfm_b200.vlm.blip2_config import Blip2Dims, random_state_dict
from vlfm_b200.vlm.blip2itm import BLIP2ITM


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=1)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    dims, B = Blip2Dims(), a.batch
    itm = BLIP2ITM(state_dict=random_state_dict(dims, 0), dims=dims, max_batch=B, device=dev)
    eng = ValueMapBatch(B, 1, size=G, use_max_confidence=False, device=dev)
    fr = make_frames(0)
    rgb = torch.from_numpy(np.stack([np.stack([f.rgb] * B) for f in fr])).to(dev)
    dep = torch.from_numpy(np.stack([np.stack([f.depth] * B) for f in fr])).to(dev)
    tfs = torch.from_numpy(np.stack([np.stack([f.tf] * B) for f in fr])).to(dev)

    def step(i):
        j = i % NFRAMES
        c = itm.cosine_device(rgb[j], PROMPT)
        eng.update(c.double().view(B, 1), dep[j], tfs[j], MIN_D, MAX_D, FOV)

    for i in range(5):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            step(5 + i)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith(("Memcpy", "Memset")):
            per[ev.name][0] += 1
            per[ev.name][1] += ev.time_range.elapsed_us()
    total = sum(v[1] for v in per.values())
    rows = sorted(((n, c / a.steps, t / a.steps, t / total) for n, (c, t) in per.items()), key=lambda r: -r[2])
    props = torch.cuda.get_device_properties(dev)
    head = (f"# Kernels of one graph-replayed configs[1] step (batch {B}), mean of {a.steps} steps\n\n"
            f"{props.name}, {props.multi_processor_count} SMs.  Device time summed over kernels: {total / a.steps:.1f} us per step.\n\n"
            "| kernel | launches/step | us/step | share |\n|---|---|---|---|\n")
    md = head + "".join(f"| `{n[:110]}` | {c:g} | {t:.1f} | {s * 100:.1f} % |\n" for n, c, t, s in rows)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "kernels.md"), "w") as f:
        f.write(md)
    with open(os.path.join(a.out, "kernels.json"), "w") as f:
        json.dump({"device": props.name, "sms": props.multi_processor_count, "steps": a.steps, "batch": B, "us_per_step": total / a.steps,
                   "kernels": [{"name": n, "launches_per_step": c, "us_per_step": t, "share": s} for n, c, t, s in rows]}, f, indent=1)
    print(md)


if __name__ == "__main__":
    main()
