"""Small invocations of the round-2 kernels for compute-sanitizer (memcheck / racecheck): batched explore (border clipping, slots,
one-pass trace, warp-parallel rays), value K2, x2 GEMM / fp32 attention / LayerNorm x2 (TINY BLIP-2 forward), radix-select top-k, object cloud."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("VLFM_NO_GRAPH", "1")
import numpy as np, torch
from vlfm_b200.mapping.obstacle_batch import ObstacleMapBatch
from vlfm_b200.mapping.value_map import ValueMapBatch
from vlfm_b200.utils.synthetic import focal_from_hfov, make_rgb, trajectory
from vlfm_b200.vlm.blip2_config import TINY, random_state_dict
from vlfm_b200.vlm.blip2itm import BLIP2ITM
from vlfm_b200.vlm.gdino_ops import LibOps

B, G, H, W = 3, 400, 120, 160
FOV = float(np.deg2rad(79.0))
fx = focal_from_hfov(W)
om = ObstacleMapBatch(B, 0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=100000, size=G, pixels_per_meter=20)
vm = ValueMapBatch(B, 1, size=G, pixels_per_meter=20, use_max_confidence=False)
frames = [trajectory(s, 4, h=H, w=W, bound_m=3.0) for s in range(B)]
vals = torch.full((B, 1), 0.5, dtype=torch.float64, device="cuda")
for i in range(4):
    d = torch.from_numpy(np.stack([frames[b][i].depth for b in range(B)])).cuda()
    tfh = np.stack([frames[b][i].tf for b in range(B)])
    tfd = torch.from_numpy(tfh.reshape(B, 16)).cuda()
    vm.update(vals, d, tfd.view(B, 4, 4), 0.5, 5.0, FOV)
    om.update(d, tfh, tfd, 0.5, 5.0, fx, fx, FOV)
torch.cuda.synchronize()
print("explored", int(om.explored.sum()), "frontiers", om.count[:B].tolist(), "conf", float(vm.conf.sum()))
itm = BLIP2ITM(state_dict=random_state_dict(TINY, 0), dims=TINY)
itm.tokenizer = lambda s: [3, 14, 15, 9, 2]
c = itm.cosine(make_rgb(np.random.default_rng(0), 120, 160), "a chair")
print("cosine", c)
ops = LibOps()
big = (torch.randn(2, 21760) * 4).round().div(4).cuda()
idx = ops.topk_rows(big, 900)
torch.cuda.synchronize()
print("topk", int(idx.sum()))
