"""Per-shape GEMM timing at full clocks: 200 back-to-back launches captured in a CUDA graph
(no CPU launch bound), optional sweep of the tile plan via VLFM_GEMM_FORCE=bn:splits.

The four ViT-g layer GEMMs at batch 1 run as the forward runs them: qkv and fc1 through vlfm_gemm_f16, proj and fc2 through
vlfm_gemm_f16_resid_ln with the engine's split-K workspace, and qkv and fc1 with the EPI_CLUSTER_SPLIT flag the engine sets.
Those four are timed under both batch-1 plans, alternated: the cluster split (one 256-row tile per column block, K split over a
thread-block cluster) and VLFM_GEMM_CSPLIT=0 (128-row tiles, sub-wave tile widths, stream-K + LayerNorm reduction)."""
import ctypes, os, sys, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vlfm_b200 import _lib
from vlfm_b200.vlm.dense import gemm_f16, gemm_f16_resid_ln

SHAPES = [(257, 4224, 1408, 0), (257, 1408, 1408, 2), (257, 6144, 1408, 1), (257, 1408, 6144, 2),
          (32, 2304, 768, 0), (32, 768, 768, 2), (32, 3072, 768, 1), (32, 768, 3072, 2), (257, 9216, 1408, 0)]
N = 200
PARTIAL_FLOATS = 8 * 257 * 1408      # the BLIP-2 engine's workspace at batch 1 (partials_floats in vlm/blip2_engine.py)

def bench(M, Nn, K, epi, resid_ln=False):
    # distinct weights per launch (ring of 8) so that weights stream from HBM like in the real forward
    a = torch.randn(M, K, device="cuda").half()
    ws = [torch.randn(Nn, K, device="cuda").half() for _ in range(8)]
    b = torch.zeros(Nn, device="cuda")
    o = torch.zeros(M, Nn, device="cuda", dtype=torch.float32 if epi >= 2 else torch.float16)
    if resid_ln:
        gamma, beta = torch.ones(Nn, device="cuda"), torch.zeros(Nn, device="cuda")
        y16 = torch.empty(M, Nn, device="cuda", dtype=torch.float16)
        partials = torch.empty(PARTIAL_FLOATS, device="cuda")
    def seq():
        for i in range(N):
            if resid_ln:
                gemm_f16_resid_ln(a, ws[i % 8], b, o, gamma, beta, 1e-6, out16=y16, partials=partials)
            else:
                gemm_f16(a, ws[i % 8], b, epi | _lib.EPI_CLUSTER_SPLIT, o)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        seq(); torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g): seq()
        for _ in range(3): g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): g.replay()
        e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (5 * N)

def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the timings stand without it; say that the card was not read
        q = f"nvidia-smi not readable ({e})"
    return f"{torch.cuda.get_device_name(0)} | power limit, SM clock, max SM clock: {q}"

def csplit_plan(M, Nn, K):
    """(BN, cluster size, bytes the busiest CTA loads, bytes all CTAs load) of the cluster-split plan, or None."""
    bn, sp, cta = ctypes.c_int(), ctypes.c_int(), ctypes.c_double()
    _lib.load().vlfm_gemm_csplit_plan(M, Nn, K, ctypes.addressof(bn), ctypes.addressof(sp), ctypes.addressof(cta))
    if not bn.value:
        return None
    nk = (K + 63) // 64
    return bn.value, sp.value, cta.value, (Nn + bn.value - 1) // bn.value * nk * (256 + bn.value) * 64 * 2

def with_plan(csplit, fn, *args, **kw):
    os.environ["VLFM_GEMM_CSPLIT"] = "1" if csplit else "0"
    try:
        return fn(*args, **kw)
    finally:
        os.environ.pop("VLFM_GEMM_CSPLIT", None)

ROUNDS = 3
sweep = len(sys.argv) > 1 and sys.argv[1] == "sweep"
vit = 0.0
vit_old = 0.0
for i, (M, Nn, K, epi) in enumerate(SHAPES):
    os.environ.pop("VLFM_GEMM_FORCE", None)
    ln = i < 4 and epi == 2
    if i < 4:
        # old and new plan alternated, ROUNDS times each; the median of each
        old, new = [], []
        for _ in range(ROUNDS):
            old.append(with_plan(False, bench, M, Nn, K, epi, resid_ln=ln))
            new.append(with_plan(True, bench, M, Nn, K, epi, resid_ln=ln))
        old_m, base = sorted(old)[ROUNDS // 2], sorted(new)[ROUNDS // 2]
        vit_old += old_m
        p = csplit_plan(M, Nn, K)
        plan = "no cluster-split plan" if p is None else f"BN {p[0]}, cluster {p[1]}: busiest CTA {p[2] / 1e3:.0f} KB, all CTAs {p[3] / 1e6:.1f} MB"
        print(f"{M}x{Nn}x{K} epi{epi}{' +LN' if ln else ''}: VLFM_GEMM_CSPLIT=0 {' '.join(f'{t:.2f}' for t in old)} us | "
              f"cluster split {' '.join(f'{t:.2f}' for t in new)} us ({plan})", flush=True)
    else:
        base = bench(M, Nn, K, epi, resid_ln=ln)
    vit += base if i < 4 else 0.0
    line = f"{M}x{Nn}x{K} epi{epi}{' +LN' if ln else ''}: model-plan {base:6.2f} us ({2*M*Nn*K/base/1e6:6.1f} TF)"
    if sweep:
        for bn in (128, 64, 32):
            for sp in ((1, 2, 3, 4, 6, 8) if epi == 2 else (1,)):
                os.environ["VLFM_GEMM_FORCE"] = f"{bn}:{sp}"
                line += f" | {bn}:{sp}={bench(M, Nn, K, epi):.2f}"
    print(line, flush=True)
# the four ViT-g layer GEMMs at batch 1 (qkv, proj + LayerNorm, fc1, fc2 + LayerNorm) x 39 layers
print(f"ViT-g batch-1 GEMMs x 39 layers (medians): cluster split {vit * 39 / 1e3:.3f} ms, VLFM_GEMM_CSPLIT=0 {vit_old * 39 / 1e3:.3f} ms",
      flush=True)
print(card(), flush=True)
