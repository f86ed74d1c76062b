"""MobileSAM timings on the GPU (seeded synthetic vit_t weights; the timings do not depend on the weight values).

Reports, with the card name and power limit read in the same run:
- encoder device time at 640x480 for B = 1 and B = 8 frames (CUDA events, warm-up, repeats alternated between the shapes);
- decoder device time for M = 1, 4 and 16 boxes;
- segment_bbox host latency including the D2H, for a fresh frame object (encoder + decoder) and for the cached frame;
- the reference's pattern (one encoder pass per detection) against segment_bboxes (one pass for all detections), per detection;
- encoder FLOPs and weight bytes computed from the shapes, and the least time the H100 data-sheet rates allow for them.

Usage: python scripts/bench_sam.py [--reps 20] [--out /tmp/bench_sam.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vlfm_b200.utils.synthetic import make_rgb  # noqa: E402
from vlfm_b200.vlm.sam import MobileSAM  # noqa: E402
from vlfm_b200.vlm.sam_config import VIT_T, SamDims  # noqa: E402

H100_FP16_FLOPS = 989e12     # dense fp16 tensor core, H100 SXM data sheet (700 W)
H100_HBM_BYTES = 3.35e12


def encoder_cost(d: SamDims, B: int):
    """(FLOPs, weight bytes) of one encoder pass over B frames: 2 per multiply-add of every conv / linear / attention product."""
    S, E, r = d.img_size, d.embed_dims, d.resolutions
    fl = 0.0
    wbytes = 0
    h1 = S // 2
    fl += 2 * B * h1 * h1 * d.stem_mid * 27 + 2 * B * r[0] ** 2 * E[0] * 9 * d.stem_mid
    wbytes += 2 * (d.stem_mid * 32 + E[0] * 9 * d.stem_mid)
    for s in range(len(E)):
        C, R = E[s], r[s]
        n = B * R * R
        for _ in range(d.depths[s]):
            if s == 0:
                hid = C * d.mbconv_ratio
                fl += 2 * n * (2 * C * hid + 9 * hid)
                wbytes += 2 * 2 * C * hid
            else:
                ws = d.windows[s]
                Rp = (R + ws - 1) // ws * ws
                fl += 2 * n * (3 * C * C + C * C + 8 * C * C) + 2 * n * 9 * C + 2 * 2 * B * Rp * Rp * ws * ws * C
                wbytes += 2 * 12 * C * C
        if s + 1 < len(E):
            Co = E[s + 1]
            Ro = r[s + 1]
            fl += 2 * n * C * Co + 2 * B * Ro * Ro * (9 * Co + Co * Co)
            wbytes += 2 * (C * Co + Co * Co)
    P, n = d.prompt_dim, B * r[-1] ** 2
    fl += 2 * n * (E[-1] * P + 9 * P * P)
    wbytes += 2 * (E[-1] * P + 9 * P * P)
    return fl, wbytes


def device_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sam.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    sam = MobileSAM(synthetic=True, max_batch=8, device="cuda:0")
    eng = sam.engine
    rng = np.random.default_rng(0)
    H, W = 480, 640
    frames = torch.from_numpy(np.stack([make_rgb(rng, H, W) for _ in range(8)])).cuda()
    boxes = torch.tensor([[40 + 30 * i, 30 + 20 * i, 300 + 15 * i, 400 - 10 * i] for i in range(16)], dtype=torch.float64).cuda()
    fidx = torch.zeros(16, dtype=torch.int32).cuda()
    enc = {B: (lambda B=B: eng.encode(frames[:B])) for B in (1, 8)}
    dec = {M: (lambda M=M: eng.decode(boxes[:M], fidx[:M], (H, W))) for M in (1, 4, 16)}
    for f in list(enc.values()) + list(dec.values()):   # warm-up every shape
        f(); f()
    torch.cuda.synchronize()
    res = {k: [] for k in ["enc1", "enc8", "dec1", "dec4", "dec16"]}
    for _ in range(args.rounds):            # alternate the shapes within each round
        res["enc1"].append(device_ms(enc[1], args.reps))
        res["enc8"].append(device_ms(enc[8], args.reps))
        eng.encode(frames[:1])
        for M in (1, 4, 16):
            res[f"dec{M}"].append(device_ms(dec[M], args.reps))
    img = frames[0].cpu().numpy()
    box = [60, 40, 400, 420]
    for _ in range(3):
        sam.segment_bbox(img.copy(), box)
        sam.segment_bbox(img, box)
    fresh, cached = [], []
    for _ in range(args.reps):
        c = img.copy()
        t = time.perf_counter(); sam.segment_bbox(c, box); fresh.append(time.perf_counter() - t)
        t = time.perf_counter(); sam.segment_bbox(c, box); cached.append(time.perf_counter() - t)
    dets = boxes[:4].cpu().numpy().tolist()
    per_box, batched = [], []
    for _ in range(args.reps):
        t = time.perf_counter()
        for b in dets:                       # reference pattern: set_image on every call
            sam.segment_bbox(img.copy(), b)
        per_box.append(time.perf_counter() - t)
        t = time.perf_counter(); sam.segment_bboxes(img.copy(), dets); batched.append(time.perf_counter() - t)
    fl1, wb = encoder_cost(VIT_T, 1)
    med = lambda v: float(np.median(v))
    out = {
        "card": card,
        "encoder_ms": {"B1": med(res["enc1"]), "B8": med(res["enc8"]), "B8_per_frame": med(res["enc8"]) / 8,
                       "rounds_B1": res["enc1"], "rounds_B8": res["enc8"]},
        "decoder_ms": {f"M{M}": med(res[f"dec{M}"]) for M in (1, 4, 16)},
        "segment_bbox_host_ms": {"fresh_frame": 1e3 * med(fresh), "cached_frame": 1e3 * med(cached)},
        "per_detection_ms_4_boxes": {"reencode_per_box": 1e3 * med(per_box) / 4, "segment_bboxes": 1e3 * med(batched) / 4},
        "encoder_cost": {"gflop_per_frame": fl1 / 1e9, "weight_mb": wb / 1e6,
                         "flop_bound_ms_per_frame": 1e3 * fl1 / H100_FP16_FLOPS, "weight_bound_ms": 1e3 * wb / H100_HBM_BYTES,
                         "achieved_tflops_B8": fl1 * 8 / (med(res["enc8"]) * 1e-3) / 1e12},
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
