"""Time the map frames for video: device render (CUDA events), render + device-to-host copy, and the former host rendering.

Conditions: G = 1000, C = 1 and 2, a 400-point trajectory and 20 markers, batch 1 and 32.  The former host rendering (numpy +
cv2 on a device-to-host copy of the value grid, no trajectory) is restated here and alternated with the new path in the same
process.  Prints the card name and power limit with the numbers.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vlfm_b200.mapping import render
from vlfm_b200.mapping.value_map import ValueMap, ValueMapBatch


def former_host_visualize(vm: ValueMap) -> np.ndarray:
    import cv2

    reduced = np.max(vm._value_map, axis=-1).copy()
    img = np.flipud(reduced)
    zero = img == 0
    img = img.copy()
    img[zero] = np.max(img)
    lo, hi = float(img.min()), float(img.max())
    norm = ((img - lo) / (hi - lo) * 255).astype(np.uint8) if hi > lo else np.zeros_like(img, np.uint8)
    rgb = cv2.applyColorMap(norm, cv2.COLORMAP_INFERNO)
    rgb[zero] = (255, 255, 255)
    return rgb


def scene(rng, g, ch, npts=400, nmark=20):
    v = np.zeros((g, g, ch), np.float32)
    m = rng.random((g, g)) < 0.3
    v[m] = rng.uniform(0, 1, (int(m.sum()), ch)).astype(np.float32)
    xy = np.cumsum(rng.normal(0, 0.15, (npts, 2)), axis=0)
    markers = [(xy[-1] + rng.normal(0, 3, 2), {"radius": 5, "thickness": 2, "color": (0, 0, 255)}) for _ in range(nmark)]
    return v, xy, markers


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip())
    rng = np.random.default_rng(0)
    g = a.size
    for ch in (1, 2):
        v, xy, markers = scene(rng, g, ch)
        origin = np.array([g // 2, g // 2])
        recs = render.trajectory_records(list(xy), 0.3, 20, origin) + render.marker_records(markers, 20, origin)
        for b in (1, 32):
            vb = ValueMapBatch(b, ch, g, use_max_confidence=False)
            vb.value.copy_(torch.from_numpy(v)[None].expand(b, -1, -1, -1))
            lists = [recs] * b
            for _ in range(3):
                vb.render(draw_lists=lists)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                vb.render(draw_lists=lists)
            e1.record()
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / a.reps
            t0 = time.perf_counter()
            for _ in range(a.reps):
                vb.render(draw_lists=lists).cpu().numpy()
            host_ms = (time.perf_counter() - t0) * 1e3 / a.reps
            print(f"C={ch} B={b}: device {dev_ms:.3f} ms/call = {dev_ms / b * 1e3:.1f} us/frame; render + D2H {host_ms:.3f} ms/call = "
                  f"{host_ms / b:.3f} ms/frame")
        # batch 1 through the class, alternated with the former host rendering on the same state
        vm = ValueMap(ch, size=g, use_max_confidence=False)
        vm._eng.value[0].copy_(torch.from_numpy(v))
        for p in xy:
            vm.update_agent_traj(p, 0.3)
        # ITMPolicy passes its own reducer (itm_policy.py:36-37, 275-287): that callable runs on the host, on the grid
        # copied to the host (float64 for a weighted map), and its result is uploaded
        def itm_reduce(arr):
            return np.where(arr[:, :, 0] > 0.3, arr[:, :, 0], np.max(arr, axis=2))

        new, host_fn, old = [], [], []
        for r in range(a.reps):
            t0 = time.perf_counter(); vm.visualize(markers); new.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); vm.visualize(markers, reduce_fn=itm_reduce); host_fn.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); former_host_visualize(vm); old.append(time.perf_counter() - t0)
        print(f"C={ch} B=1 ValueMap.visualize (trajectory + markers): device reducer median {np.median(new) * 1e3:.2f} ms, "
              f"host reducer (ITMPolicyV3-style) median {np.median(host_fn) * 1e3:.2f} ms; former host visualize "
              f"(no trajectory): median {np.median(old) * 1e3:.2f} ms")


if __name__ == "__main__":
    main()
