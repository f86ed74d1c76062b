"""Small invocations of the round-1 late additions for compute-sanitizer (memcheck / racecheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from vlfm_b200.mapping.obstacle_map import ObstacleMap
from vlfm_b200.mapping.value_map import build_cone_template
from vlfm_b200.utils.synthetic import focal_from_hfov, trajectory
from vlfm_b200.vlm.dense import cast_f16
from vlfm_b200 import _lib
import ctypes

fx = focal_from_hfov(160)
g = ObstacleMap(0.61, 0.88, 0.18, area_thresh=1.5, hole_area_thresh=100000, size=400)
for f in trajectory(3, 4, h=120, w=160, bound_m=3.0):
    g.update_map(f.depth, f.tf, 0.5, 5.0, fx, fx, np.deg2rad(79))
print("explored", int(g.explored_area.sum()), "frontiers", len(g._frontiers_px))
t = build_cone_template(float(np.deg2rad(79)), 5.0, 20, torch.device("cuda"))
print("template", float(t.sum()))
torch.manual_seed(0)
shapes = [(15, 20), (8, 10), (4, 5), (2, 3)]
b, heads, hd, q, pts = 2, 8, 32, 77, 4
s = sum(h * w for h, w in shapes)
value = torch.randn(b, s, heads, hd, device="cuda")
# fused deformable attention
offlog = torch.randn(b * q, 384, device="cuda")
ref = torch.rand(b, q, 4, 2, device="cuda")
out16 = torch.empty(b * q, 256, dtype=torch.float16, device="cuda")
flat = [v for hw in shapes for v in hw]
arr = (ctypes.c_int32 * 8)(*flat)
rc = _lib.load().vlfm_msda_fused(value.half().data_ptr(), offlog.data_ptr(), 384, 256, ref.data_ptr(), 2, out16.data_ptr(), b, s, q, heads, 4, 4,
                                ctypes.cast(arr, ctypes.c_void_p), _lib.stream_ptr())
_lib.check(rc, "msda_fused")
ref4 = torch.rand(b, q, 4, 4, device="cuda")
rc = _lib.load().vlfm_msda_fused(value.half().data_ptr(), offlog.data_ptr(), 384, 256, ref4.data_ptr(), 4, out16.data_ptr(), b, s, q, heads, 4, 4,
                                ctypes.cast(arr, ctypes.c_void_p), _lib.stream_ptr())
_lib.check(rc, "msda_fused4")
x = torch.randn(1003, device="cuda")
h = cast_f16(x)
torch.cuda.synchronize()
print("ok", float(out16.float().abs().sum()), float(h.float().sum()))
