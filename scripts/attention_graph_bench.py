"""Per-call time of the ViT-g self-attention at batch 1 (16 heads, 257 queries and keys, hd 88): 200 vlfm_attention_f16 calls
captured in a CUDA graph (no CPU launch bound), on the strided q / k / v column views of a [257, 4224] qkv buffer as the BLIP-2
engine passes them, cycling through 8 such buffers.  The batch-1 variant (attention_kernel<96, 4, true>: 64-row blocks, 80 CTAs) and
VLFM_ATT_IMPL=legacy (attention_kernel<96, 4>: 32-row blocks, 144 CTAs) are alternated, ROUNDS times each; each line gives every round and the median.

  python scripts/attention_graph_bench.py
"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vlfm_b200.vlm.dense import attention_f16

B, HEADS, T, HD = 1, 16, 257, 88
D = HEADS * HD
N, RING, ROUNDS = 200, 8, 3


def bench(impl):
    os.environ["VLFM_ATT_IMPL"] = impl
    try:
        bufs = [torch.randn(B * T, 3 * D, device="cuda").half() for _ in range(RING)]
        out = torch.empty(B * T, D + 64, device="cuda", dtype=torch.float16)[:, :D]   # output stride != input stride

        def seq():
            for i in range(N):
                q = bufs[i % RING]
                attention_f16(q[:, 0:D], q[:, D : 2 * D], q[:, 2 * D :], B, HEADS, T, T, HD, HD ** -0.5, out)

        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            seq()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                seq()
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (5 * N)
    finally:
        os.environ.pop("VLFM_ATT_IMPL", None)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the timings stand without it; say that the card was not read
        q = f"nvidia-smi not readable ({e})"
    return f"{torch.cuda.get_device_name(0)} | power limit, SM clock, max SM clock: {q}"


def main():
    print(f"PDL {'on' if os.environ.get('VLFM_PDL', '1') != '0' else 'off'}", flush=True)
    times = {"legacy": [], "b1": []}
    for _ in range(ROUNDS):
        for impl in times:
            times[impl].append(bench(impl))
    flops = 4.0 * B * HEADS * T * T * HD
    for impl, ts in times.items():
        med = sorted(ts)[ROUNDS // 2]
        print(f"{impl:6s}: {' '.join(f'{t:.2f}' for t in ts)} us per call, median {med:.2f} us "
              f"({flops / med / 1e6:.1f} TFLOP/s; x39 layers = {39 * med / 1e3:.3f} ms per forward)", flush=True)
    print(card(), flush=True)


if __name__ == "__main__":
    main()
