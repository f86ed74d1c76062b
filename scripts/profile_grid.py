"""Grid-path workload for ncu / timing (round 2): ValueMapBatch.update and ObstacleMapBatch.update (hole fill + scatter + dilate +
explore half + frontiers, one launch sequence for the batch) on 640x480 depth.

    python scripts/profile_grid.py --batch 32 --grid 1000 --time          # CUDA-event timings
    ncu --profile-from-start off --set full --clock-control none -o /tmp/grid python scripts/profile_grid.py --batch 32
"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
from vlfm_b200.mapping.value_map import ValueMapBatch
from vlfm_b200.utils.full_step import grid_bytes
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--grid", type=int, default=1000)
ap.add_argument("--ppm", type=int, default=20)
ap.add_argument("--hw", type=int, nargs=2, default=[480, 640])
ap.add_argument("--warm", type=int, default=6)
ap.add_argument("--time", action="store_true")
ap.add_argument("--hole", type=int, default=100000)
a = ap.parse_args()
B, G, (H, W) = a.batch, a.grid, a.hw
FOV = float(np.deg2rad(79.0))
fx = focal_from_hfov(W)
nf = a.warm + 2
frames = [trajectory(s, nf, h=H, w=W, bound_m=0.012 * G) for s in range(B)]
vm = ValueMapBatch(B, 1, size=G, pixels_per_meter=a.ppm, use_max_confidence=False)
om = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=a.hole, size=G, pixels_per_meter=a.ppm)
vals = torch.full((B, 1), 0.5, dtype=torch.float64, device="cuda")


def load(i):
    d = torch.from_numpy(np.stack([frames[b][i].depth for b in range(B)])).cuda()
    tfh = np.stack([frames[b][i].tf for b in range(B)])
    return d, tfh, torch.from_numpy(tfh.reshape(B, 16)).cuda()


def step(d, tfh, tfd):
    vm.update(vals, d, tfd.view(B, 4, 4), 0.5, 5.0, FOV)
    om.update(d, tfh, tfd, 0.5, 5.0, fx, fx, FOV)


for i in range(a.warm):
    step(*load(i))
torch.cuda.synchronize()
d, tfh, tfd = load(a.warm)
gb = grid_bytes(H, W, G, a.ppm)
if a.time:
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 20

    def loop(fn):          # back-to-back launches, one pair of events around the loop (no host sync inside)
        fn(); torch.cuda.synchronize()
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record(); torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / reps

    tv = loop(lambda: vm.update(vals, d, tfd.view(B, 4, 4), 0.5, 5.0, FOV))
    to = loop(lambda: om.update(d, tfh, tfd, 0.5, 5.0, fx, fx, FOV))
    fr = om._frame(0)
    print(f"B={B} G={G} ppm={a.ppm} {W}x{H}: value update {tv*1e3:.1f} us ({gb['value']*B/tv/1e6:.0f} GB/s algorithmic), "
          f"obstacle+explore {to*1e3:.1f} us ({gb['obstacle']*B/to/1e6:.0f} GB/s algorithmic); S frame of env 0: {fr[2]-fr[0]}x{fr[3]-fr[1]}; "
          f"frontiers/env {float(om.count[:B].float().mean()):.1f}")
else:
    torch.cuda.profiler.start(); step(d, tfh, tfd); torch.cuda.synchronize(); torch.cuda.profiler.stop()
print("done")
