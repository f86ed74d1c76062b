"""Cost of scoring one frame against P prompts: the per-frame feature cache behind BLIP2ITM.cosine and cosine_device_many.

Full-size ViT-g/14 + Q-Former with seeded synthetic weights, 16 cycling 640x480 frames (bench.py's trajectory).

1. Batch 1, ValueMap(value_channels=P) fed the way ITMPolicy._update_value_map feeds it, P in {1, 2, 4}:
   (a) ``[itm.cosine(rgb, p) for p in prompts]`` on the same frame object: one forward, then the head alone;
   (b) the same loop with ``rgb.copy()`` per prompt: one forward per prompt.
   (a) and (b) alternate, three times each.  Host clock around K steps ending in a device synchronise.
2. ``cosine_device_many`` at B in {1, 32} and P in {1, 2} against P ``cosine_device`` calls, CUDA events, every shape warmed.

The card's name, power limit and SM clock are read in the same run.  Writes OUT/itm_prompts.json and prints it.

  python scripts/bench_itm_prompts.py --out DIR [--steps 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import FOV, G, MAX_D, MIN_D, NFRAMES, make_frames
from vlfm_b200.mapping.value_map import ValueMap
from vlfm_b200.vlm.blip2_config import Blip2Dims, random_state_dict
from vlfm_b200.vlm.blip2itm import BLIP2ITM

PROMPTS = ["Seems like there is a chair ahead.", "There is a lot of area to explore ahead.",
           "Seems like there is a potted plant ahead.", "Seems like there is a toilet ahead."]


def card():
    """name, power limit and clocks (read-only query)"""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        return dict(zip(q.split(","), (c.strip() for c in out.split(","))))
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "error": f"nvidia-smi: {e}"}


def host_loop(itm, vm, frames, prompts, copy, steps, start):
    """steps value-map steps; returns seconds (host clock, ends in a device synchronise)"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        f = frames[(start + i) % NFRAMES]
        vals = [itm.cosine(f.rgb.copy() if copy else f.rgb, p) for p in prompts]
        vm.update_map(np.array(vals), f.depth, f.tf, MIN_D, MAX_D, FOV)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def device_time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--device-iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_itm_prompts: needs a CUDA device")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dims = Blip2Dims()
    sd = random_state_dict(dims, 0)
    frames = make_frames(0)
    res = {"card_before": card(), "host_batch1": {}, "device": {}}

    # ---- 1. batch 1, host frames, ValueMap(value_channels=P)
    itm = BLIP2ITM(state_dict=sd, dims=dims, max_batch=1, device=dev)
    for P in (1, 2, 4):
        prompts = PROMPTS[:P]
        vm = ValueMap(P, size=G, use_max_confidence=False, device=dev)
        host_loop(itm, vm, frames, prompts, False, a.warmup, 0)
        host_loop(itm, vm, frames, prompts, True, a.warmup, 0)
        runs = {"cached": [], "copy": []}
        for rep in range(3):
            for mode, copy in (("cached", False), ("copy", True)):
                s = host_loop(itm, vm, frames, prompts, copy, a.steps, rep * a.steps)
                runs[mode].append(a.steps / s)
        med = {k: float(np.median(v)) for k, v in runs.items()}
        res["host_batch1"][f"P{P}"] = {"steps_per_s": runs, "median": med, "speedup": med["cached"] / med["copy"]}
        print(f"batch 1, P={P}: cached {med['cached']:.1f} steps/s, copy per prompt {med['copy']:.1f} steps/s "
              f"(x{med['cached'] / med['copy']:.2f}); runs {runs}", flush=True)
    del itm
    torch.cuda.empty_cache()

    # ---- 2. device path: cosine_device_many vs P cosine_device calls
    itm32 = BLIP2ITM(state_dict=sd, dims=dims, max_batch=32, device=dev)
    itm1 = BLIP2ITM(state_dict=sd, dims=dims, max_batch=1, device=dev)
    rgb = torch.from_numpy(np.stack([f.rgb for f in frames])).to(dev)                    # [16, H, W, 3]
    rgb32 = torch.from_numpy(np.stack([np.stack([frames[(i + k) % NFRAMES].rgb for k in range(32)]) for i in range(NFRAMES)])).to(dev)
    for B, m, src in ((1, itm1, lambda i: rgb[i % NFRAMES][None]), (32, itm32, lambda i: rgb32[i % NFRAMES])):
        for P in (1, 2):
            prompts = PROMPTS[:P]
            many = lambda i: m.cosine_device_many(src(i), prompts)                            # noqa: E731
            sep = lambda i: [m.cosine_device(src(i), p) for p in prompts]                     # noqa: E731
            for i in range(3):
                many(i); sep(i)
            t = {"many": [], "separate": []}
            for rep in range(3):
                t["many"].append(device_time(many, a.device_iters))
                t["separate"].append(device_time(sep, a.device_iters))
            med = {k: float(np.median(v)) for k, v in t.items()}
            res["device"][f"B{B}_P{P}"] = {"ms_per_call": t, "median_ms": med, "speedup": med["separate"] / med["many"]}
            print(f"device B={B}, P={P}: cosine_device_many {med['many']:.3f} ms, {P} x cosine_device {med['separate']:.3f} ms "
                  f"(x{med['separate'] / med['many']:.2f})", flush=True)
    res["card_after"] = card()
    res["config"] = {"model": "ViT-g/14 + 12-layer Q-Former, synthetic weights", "frames": f"{NFRAMES} cycling 480x640",
                     "grid": G, "steps": a.steps, "warmup": a.warmup, "device_iters": a.device_iters,
                     "host_timing": "host clock around K steps ending in torch.cuda.synchronize, pageable numpy frames",
                     "device_timing": "CUDA events around device_iters calls"}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "itm_prompts.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
