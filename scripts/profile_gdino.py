"""Where does GroundingDINO.predict spend its time at batch B?  torch.profiler table + per-module CUDA-event times."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from vlfm_b200.vlm.grounding_dino import GroundingDINO

B = int(os.environ.get("B", "32"))
dev = torch.device("cuda", 0)
gd = GroundingDINO(device=dev, synthetic=True)
ids = gd.tokenizer.encode("chair . couch . potted plant . bed . toilet . tv .")
rng = np.random.default_rng(0)
img = torch.from_numpy(rng.integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)).to(dev)
for _ in range(2):
    gd.raw_outputs_device(img, ids)
torch.cuda.synchronize()

# module-level timing
times = {}
def hook(name):
    def pre(m, a, k=None):
        e = torch.cuda.Event(enable_timing=True); e.record(); times.setdefault(name, []).append([e, None])
    def post(m, a, o):
        e = torch.cuda.Event(enable_timing=True); e.record(); times[name][-1][1] = e
    return pre, post
# GdinoForward sequences the encoder / decoder stacks itself: the per-layer modules are what is called.  Hooks fire on eager
# forwards only (B above GRAPH_MAX_BATCH, or VLFM_NO_GRAPH=1).
mods = []
for l in gd.model.model.encoder.layers:
    mods += [("enc.fusion", l.fusion_layer), ("enc.text_enh", l.text_enhancer_layer), ("enc.deform", l.deformable_layer)]
mods += [("dec.layer", l) for l in gd.model.model.decoder.layers]
hs = []
for n, m in mods:
    pre, post = hook(n)
    hs.append(m.register_forward_pre_hook(pre)); hs.append(m.register_forward_hook(post))
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True); e2 = torch.cuda.Event(enable_timing=True)
e0.record(); maps = gd.backbone.forward(img); e1.record()
gd.raw_outputs_device(img, ids); e2.record()
torch.cuda.synchronize()
print(f"B={B}  swin engine alone {e0.elapsed_time(e1):.2f} ms ; whole raw_outputs {e1.elapsed_time(e2):.2f} ms")
for n, v in times.items():
    print(f"  {n:28s} {sum(a.elapsed_time(b) for a, b in v):9.2f} ms  ({len(v)} calls)")
for h in hs: h.remove()
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    gd.raw_outputs_device(img, ids); torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=45, max_name_column_width=70))
