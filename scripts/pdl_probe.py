# NOTE: needs a development build of the library (NVCC flag -DVLFM_DEV_PROBES): the probe entry points are not in the shipped C-ABI.
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vlfm_b200 import _lib
lib = _lib.load()
sink = torch.zeros(1, dtype=torch.int32, device="cuda")
def run(n, blocks, smem):
    for _ in range(n): lib.vlfm_pdl_probe(blocks, smem, 10000, 10000, sink.data_ptr(), _lib.stream_ptr())
def timeit(fn, it=5):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(it): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / it
print("PDL", os.environ.get("VLFM_PDL", "1"), "(each kernel: 10us pre-wait + 10us post-wait; 20us = no overlap, 10us = full overlap)")
for blocks, smem in [(132, 0), (132, 100 * 1024), (132, 200 * 1024), (100, 200 * 1024)]:
    t_s = timeit(lambda: run(50, blocks, smem)) * 1e3 / 50
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        run(50, blocks, smem); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g): run(50, blocks, smem)
        t_g = timeit(g.replay) * 1e3 / 50
    print(f"blocks={blocks} smem={smem//1024}KB: stream {t_s:.1f} us/kernel, graph {t_g:.1f} us/kernel")
