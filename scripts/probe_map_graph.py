"""Per-step device time of ObstacleMapBatch.update along a trajectory with STATIC input buffers (the FullStep / policy-loop
situation: graph replay from step 3), with and without the CUDA graph.  python scripts/probe_map_graph.py --batch 32 [--profile-step 8]"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--grid", type=int, default=1000)
ap.add_argument("--ppm", type=int, default=20)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--bound", type=float, default=15.0)
ap.add_argument("--profile-step", type=int, default=-1)
ap.add_argument("--seed0", type=int, default=0)
a = ap.parse_args()
B, G, H, W = a.batch, a.grid, 480, 640
FOV = float(np.deg2rad(79.0))
fx = focal_from_hfov(W)
frames = [trajectory(a.seed0 + s, a.steps, h=H, w=W, bound_m=a.bound) for s in range(B)]
om = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=100000, size=G, pixels_per_meter=a.ppm)
depth = torch.empty((B, H, W), dtype=torch.float32, device="cuda")
tfd = torch.empty((B, 16), dtype=torch.float64, device="cuda")
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for i in range(a.steps):
    depth.copy_(torch.from_numpy(np.stack([frames[b][i].depth for b in range(B)])))
    tfh = np.stack([frames[b][i].tf for b in range(B)])
    tfd.copy_(torch.from_numpy(tfh.reshape(B, 16)))
    torch.cuda.synchronize()
    if i == a.profile_step:
        torch.cuda.profiler.start()
    ev[0].record()
    om.update(depth, tfh, tfd, 0.5, 5.0, fx, fx, FOV)
    ev[1].record()
    torch.cuda.synchronize()
    if i == a.profile_step:
        torch.cuda.profiler.stop()
    fr = om._frame(0)
    print(f"step {i}: {ev[0].elapsed_time(ev[1])*1e3:.0f} us  graph={'yes' if om.graphs.captured else 'no'}  S frame env0 {fr[2]-fr[0]}x{fr[3]-fr[1]}  frontiers {om.count[:B].tolist()[:6]}  status {int(om.ex_status.max())}", flush=True)
