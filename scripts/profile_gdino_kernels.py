"""One eager GroundingDINO forward (batch from $B) between cudaProfilerStart/Stop, for ncu kernel filters."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["VLFM_NO_GRAPH"] = "1"
import numpy as np, torch
from vlfm_b200.vlm.grounding_dino import GroundingDINO
B = int(os.environ.get("B", "8"))
gd = GroundingDINO(device=torch.device("cuda", 0), synthetic=True)
ids = gd.tokenizer.encode("chair . couch . potted plant . bed . toilet . tv .")
img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)).cuda()
for _ in range(2): gd.raw_outputs_device(img, ids)
torch.cuda.synchronize(); torch.cuda.profiler.start()
gd.raw_outputs_device(img, ids)
torch.cuda.synchronize(); torch.cuda.profiler.stop()
