"""YOLOv7-E6E device time per frame (CUDA events over graph replay) at batch 1, 8 and 32 on synthetic weights, its split into
im2col, GEMM and the rest (torch.profiler over one replay, a separate run), predict() host latency, and the same network as
yolov7 runs it (the oracle in fp16 on cuDNN, eager) timed alternately on the same card.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import yolov7_oracle as O  # noqa: E402
from vlfm_b200.vlm.yolov7 import YOLOv7  # noqa: E402
from vlfm_b200.vlm.yolov7_config import cost  # noqa: E402

PEAK_TFLOPS = 989.0     # H100 SXM data sheet, dense fp16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", default="1,8,32")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    model = YOLOv7(synthetic=True)
    e = model.engine
    rng = np.random.default_rng(0)
    _, gflop = cost(448, 640)
    out = {"card": card(), "gflop_per_frame": round(gflop, 2), "batches": {}}
    for B in [int(b) for b in args.batches.split(",")]:
        imgs = torch.from_numpy(rng.integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)).cuda()
        e.run(imgs)
        e.run(imgs)
        g = e.graphs.captured[(B, 480, 640)].graph
        x = O.preprocess(imgs[0].cpu().numpy()).cuda().half().repeat(B, 1, 1, 1)
        fp16 = lambda: O.forward(e.layers, x, dtype=torch.float16)
        with torch.inference_mode():
            fp16()
            ours, ref = [], []
            for _ in range(args.rounds):                       # alternate the two
                ours.append(timed(g.replay, args.iters))
                ref.append(timed(fp16, max(2, args.iters // 4)))
        ms = min(ours) / B
        out["batches"][B] = {"ms_per_frame": round(ms, 4), "ms_per_call": [round(t, 3) for t in ours],
                             "tflops": round(gflop / ms, 1), "share_of_989": round(gflop / ms / PEAK_TFLOPS, 3),
                             "fp16_cudnn_eager_network_only_ms_per_frame": round(min(ref) / B, 4),
                             "peak_MiB": round(e.peak_bytes(B) / 2 ** 20, 1)}
    # split of one batch-1 replay by kernel name (profiler run of its own)
    from torch.profiler import ProfilerActivity, profile

    g = e.graphs.captured[(1, 480, 640)].graph
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    split = {"im2col": 0.0, "gemm": 0.0, "rest": 0.0}
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        k = "im2col" if "im2col" in ev.key else ("gemm" if "wgmma" in ev.key else "rest")
        split[k] += t / 5 / 1000.0
    out["split_ms_b1"] = {k: round(v, 3) for k, v in split.items()}
    # predict() host latency: host frame in, ObjectDetections out
    img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
    model.predict(img)
    t0 = time.perf_counter()
    for _ in range(args.iters):
        model.predict(img)
    out["predict_ms"] = round((time.perf_counter() - t0) / args.iters * 1000, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
