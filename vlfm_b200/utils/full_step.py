"""The FULL policy step for a batch of environments on one GPU -- GroundingDINO detect + BLIP-2 ITC + ObstacleMap (hole fill,
scatter, dilate, fog-of-war, frontiers) + ValueMap fuse + frontier scoring -- with per-component CUDA-event times and the
grid kernels' achieved HBM bandwidth.  Shared by bench.py (BASELINE.json configs[2], [3], [4] slices) and
scripts/bench_full_step.py.  Reference call sites: base_objectnav_policy.py:153-241 (_cache_observations /
_get_object_detections), itm_policy.py:191-211, 263-294 (_update_value_map / _sort_frontiers_by_value)."""
from __future__ import annotations

import os
import time
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from ..mapping.value_map import frontier_values

MIN_D, MAX_D, FOV = 0.5, 5.0, float(np.deg2rad(79))
PROMPT = "Seems like there is a chair ahead."
CAPTION = "chair . couch . potted plant . bed . toilet . tv ."


def grid_bytes(h: int, w: int, g: int, ppm: int, channels: int = 1, max_depth: float = MAX_D) -> Dict[str, float]:
    """Algorithmic bytes per env-step of the grid path (SURVEY.md section 8d)."""
    r = 2 * int(max_depth * ppm) + 1
    return {"value": 4.0 * h * w + (12 + 8 * channels) * r * r, "obstacle": 4.0 * h * w + 7.0 * g * g, "R": r}


class FullStep:
    def __init__(self, dev: torch.device, batch: int, h: int, w: int, grid: int, ppm: int, itm, gdino, frames_per_env: int,
                 seed0: int = 0, streams: int = 8, hole_thresh: int = 100000, bound_m: float = 15.0) -> None:
        from ..mapping.obstacle_batch import ObstacleMapBatch
        from ..mapping.value_map import ValueMapBatch
        from .synthetic import focal_from_hfov, trajectory

        self.dev, self.B, self.H, self.W, self.G, self.ppm = dev, batch, h, w, grid, ppm
        self.itm, self.gd = itm, gdino
        self.ids = gdino.tokenizer.encode(CAPTION) if gdino is not None else None
        self.vmb = ValueMapBatch(batch, 1, size=grid, pixels_per_meter=ppm, use_max_confidence=False, device=dev)
        self.omb = ObstacleMapBatch(batch, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=hole_thresh, size=grid, pixels_per_meter=ppm, device=dev)
        self.fx = focal_from_hfov(w)
        nf = frames_per_env
        self.frames = [trajectory(seed0 + e, nf, h=h, w=w, bound_m=bound_m, with_rgb=True) for e in range(batch)]
        # every step's frames wait in page-locked host memory, batched per step (as a vectorised simulator bridge leaves them)
        self.rgb_pin = torch.empty((nf, batch, h, w, 3), dtype=torch.uint8).pin_memory()
        self.depth_pin = torch.empty((nf, batch, h, w), dtype=torch.float32).pin_memory()
        self.tf_pin = torch.empty((nf, batch, 16), dtype=torch.float64).pin_memory()
        for i in range(nf):
            for e in range(batch):
                f = self.frames[e][i]
                self.rgb_pin[i, e].numpy()[...] = f.rgb
                self.depth_pin[i, e].numpy()[...] = f.depth
                self.tf_pin[i, e].numpy()[...] = f.tf.reshape(16)
                f.depth = None
                f.rgb = None
        self.tf_host = [np.stack([self.frames[e][i].tf for e in range(batch)]) for i in range(nf)]
        self.rgb_dev, self.depth_dev, self.tf_dev = (torch.empty_like(t[0], device=dev) for t in (self.rgb_pin, self.depth_pin, self.tf_pin))
        self.names = ["h2d", "gdino", "itc", "obstacle+explore", "value_fuse", "frontier_scoring"]
        self.acc = {k: 0.0 for k in self.names}
        self.n_front = 0
        self.nf = nf
        # Three streams (detector | ITC | map update) are opt-in: VLFM_FULLSTEP_STREAMS=1.  Full bench.py runs with them have stopped
        # making progress (never reproduced in scripts/bench_full_step.py; not root-caused) -- the default is the one-stream sequence.
        self.serial = os.environ.get("VLFM_FULLSTEP_STREAMS", "0") != "1"
        self.sync_each = os.environ.get("VLFM_FULLSTEP_SERIAL", "0") == "1"   # diagnostic: device sync after every component
        self._streams = None

    def step(self, i: int, timed: bool) -> None:
        """One policy step.  The detector, the ITC model and the obstacle / explore update consume the same uploaded frame and do not
        depend on each other (base_objectnav_policy.py:153-241 calls them one after the other because each call is a blocking HTTP /
        numpy round trip): with VLFM_FULLSTEP_STREAMS=1 they are issued on three streams and joined before the value-map fuse (needs the
        cosine) and the frontier scoring (needs both maps); by default they are issued back to back on one stream."""
        i %= self.nf
        B = self.B
        main = torch.cuda.current_stream()
        E = lambda: torch.cuda.Event(enable_timing=True)
        e_in0, e_in1 = E(), E()
        e_in0.record()
        self.rgb_dev.copy_(self.rgb_pin[i], non_blocking=True)
        self.depth_dev.copy_(self.depth_pin[i], non_blocking=True)
        self.tf_dev.copy_(self.tf_pin[i], non_blocking=True)
        e_in1.record()
        conc = not self.serial
        if conc and self._streams is None:
            # the detector is the longest of the three: its stream gets the higher priority, the other two fill the gaps
            prio = os.environ.get("VLFM_FULLSTEP_PRIO", "0") == "1"     # measured: no effect on graph replays (B=1), within noise at B=32
            self._streams = [torch.cuda.Stream(device=self.dev, priority=-1 if (prio and k == 0) else 0) for k in range(3)]
        s_det, s_itc, s_map = self._streams if conc else (main, main, main)
        spans = {}

        def on(stream, name, fn):
            with torch.cuda.stream(stream):
                if conc:
                    stream.wait_event(e_in1)
                a, b = E(), E()
                a.record()
                out = fn()
                b.record()
                spans[name] = (a, b)
                if self.sync_each:
                    torch.cuda.synchronize()
            return out

        def detect():
            if self.gd is None:
                return None
            logits, boxes = self.gd.raw_outputs_device(self.rgb_dev, self.ids)
            keep = logits.max(dim=2)[0] > self.gd.box_threshold        # compaction mask stays on the device
            return keep.sum()

        det = on(s_det, "gdino", detect)
        cos = on(s_itc, "itc", lambda: self.itm.cosine_device(self.rgb_dev, PROMPT))
        # all environments' obstacle + explore update: ONE launch sequence (hole fill, scatter, dilate, fog-of-war, frontiers)
        on(s_map, "obstacle+explore", lambda: self.omb.update(self.depth_dev, self.tf_host[i], self.tf_dev, MIN_D, MAX_D, self.fx, self.fx, FOV))
        if conc:
            main.wait_event(spans["itc"][1])
        on(main, "value_fuse", lambda: self.vmb.update(cos.double().view(B, 1), self.depth_dev, self.tf_dev.view(B, 4, 4), MIN_D, MAX_D, FOV))
        if conc:
            main.wait_event(spans["obstacle+explore"][1])

        def score():
            # ITMPolicy._sort_frontiers_by_value for every environment: one D2H of the frontier lists, one disc-median launch, one D2H
            for fr, _ in frontier_values(self.omb, self.vmb, B, 0.5):
                self.n_front += len(fr)

        on(main, "frontier_scoring", score)
        if conc:
            main.wait_event(spans["gdino"][1])
        torch.cuda.synchronize()
        _ = det
        if timed:
            self.acc["h2d"] += e_in0.elapsed_time(e_in1)
            for nme, (a, b) in spans.items():
                self.acc[nme] += a.elapsed_time(b)

    def run(self, steps: int, warmup: int) -> Dict[str, Any]:
        for i in range(warmup):
            self.step(i, False)
        # the map update is captured into a CUDA graph on its second call with the same buffers (third call overall): keep the
        # capture (tens to hundreds of ms) out of the timed region whatever `warmup` is
        extra = 0
        while self.omb.use_graph and not self.omb.graphs.captured and extra < 3:
            self.step(warmup + extra, False)
            extra += 1
        torch.cuda.synchronize()
        self.n_front = 0
        self.acc = {k: 0.0 for k in self.names}
        t0 = time.perf_counter()
        for i in range(steps):
            self.step(warmup + i, True)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        comp = {k: v / steps for k, v in self.acc.items()}
        gb = grid_bytes(self.H, self.W, self.G, self.ppm)
        return {"env_steps_per_s": self.B * steps / wall, "ms_per_step": 1e3 * wall / steps, "wall_s": wall, "steps": steps, "warmup": warmup,
                "batch": self.B, "component_ms_per_step": comp,
                "component_note": "CUDA-event spans; gdino / itc / obstacle+explore run on three streams and OVERLAP (their sum exceeds the step)" if not self.serial else "serial: one stream", "frontiers_per_env_step": self.n_front / (self.B * steps),
                "grid_bytes_per_env_step": gb}

    def grid_rooflines(self, hbm_gbs: float, reps: int = 6) -> Dict[str, Any]:
        """Achieved algorithmic-bytes/s of the grid kernels alone (CUDA events on the launching stream, inputs resident in HBM)."""
        B = self.B
        gb = grid_bytes(self.H, self.W, self.G, self.ppm)
        out: Dict[str, Any] = {}
        cos = torch.full((B, 1), 0.5, dtype=torch.float64, device=self.dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(2):
            self.vmb.update(cos, self.depth_dev, self.tf_dev.view(B, 4, 4), MIN_D, MAX_D, FOV)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            self.vmb.update(cos, self.depth_dev, self.tf_dev.view(B, 4, 4), MIN_D, MAX_D, FOV)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        ach = gb["value"] * B / (ms * 1e-3) / 1e9
        out["value_update"] = {"kernels": "value_depth_geom_kernel + value_cone_fuse_kernel", "ms": ms, "envs": B, "bytes_per_env": gb["value"],
                               "achieved_gbs": ach, "peak_gbs": hbm_gbs, "frac": ach / hbm_gbs, "bound": "hbm"}
        # obstacle + explore: the batched launch sequence of step(), depth already in HBM
        def obst():
            self.omb.update(self.depth_dev, self.tf_host[0], self.tf_dev, MIN_D, MAX_D, self.fx, self.fx, FOV)

        obst()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            obst()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        ach = gb["obstacle"] * B / (ms * 1e-3) / 1e9
        out["obstacle_explore"] = {"kernels": "fill_small_holes + obstacle_scatter/dilate + explore (fog-of-war, component, frontiers), one launch sequence for all envs",
                                   "ms": ms, "envs": B, "bytes_per_env": gb["obstacle"], "achieved_gbs": ach, "peak_gbs": hbm_gbs,
                                   "frac": ach / hbm_gbs, "bound": "hbm (latency-bound border following in practice)"}
        return out
