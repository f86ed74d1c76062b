"""The full-size BLIP-2 ITC forward (ViT-g/14 + 12-layer Q-Former) above batch 1, and the reduction of its residual GEMMs.

Each batch size runs different code: the fp16 attention variant (KH 4 at B = 1, KH 2 at B = 2-3, KH 1 from B = 4), the plan of
the residual GEMMs (stream-K up to B = 5, partial-sum splits at B = 6-9 and for fc2 at 12-14, unsplit above) and the row groups
of the fp32 Q-Former attention (z = 4 up to B = 5, 3 at B = 6-7, 1 from B = 12).  Every batch is held to the bar of batch 1: the
fp32 oracle within 1e-4 on the cosine."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import blip2_oracle
from vlfm_b200.utils.synthetic import make_rgb
from vlfm_b200.vlm.blip2_config import Blip2Dims, random_state_dict

pytestmark = pytest.mark.gpu

PROMPTS = ["Seems like there is a chair ahead.", "Seems like there is a potted plant ahead.", "Seems like there is a toilet ahead."]
BATCHES = (2, 3, 4, 6, 12, 32)
# largest |cos_B - cos_1| over the frames and prompts of BATCHES: 1.40e-5 (at B = 32) measured on an H100 80GB HBM3 at 700 W;
# pinned with a margin of about 3.5x.  The batches reorder sums (other GEMM plans and attention variants), so they are not bitwise
# equal to batch 1.
BATCH_VS_B1_PIN = 5e-5


def _oracle_text(orc, dims):
    from vlfm_b200.vlm.blip2itm import HashTokenizer, pre_caption

    tok = HashTokenizer(dims.vocab)
    return [orc.text_feature(tok(pre_caption(p))) for p in PROMPTS]


def _setup(outliers, frames, max_batch):
    from vlfm_b200.vlm.blip2itm import BLIP2ITM

    dims = Blip2Dims()
    sd = random_state_dict(dims, 0, outliers=outliers)
    orc = blip2_oracle.Blip2Oracle(dims, sd)
    m = BLIP2ITM(state_dict=sd, dims=dims, max_batch=max_batch)
    txt = _oracle_text(orc, dims)
    rng = np.random.default_rng(2)
    imgs = np.stack([make_rgb(rng, 480, 640) for _ in range(frames)])
    ref = np.array([[orc.cosine_from(f, t) for t in txt] for f in (orc.image_features(i) for i in imgs)])
    dev = torch.from_numpy(imgs).cuda()
    return SimpleNamespace(dims=dims, orc=orc, m=m, imgs=imgs, dev=dev, ref=ref)


@pytest.fixture(scope="module")
def full():
    """The seeded weights of test_full_size_vitg_vs_oracle, one engine for up to 32 frames of 480 x 640, the oracle cosines of
    every (frame, prompt) and every frame's batch-1 cosines."""
    s = _setup(False, 32, 32)
    s.cos1 = np.stack([s.m.cosine_device_many(s.dev[i : i + 1], PROMPTS).cpu().numpy()[0] for i in range(32)])
    return s


def test_batches_vs_oracle(full):
    m, ref = full.m, full.ref
    e1 = float(np.abs(full.cos1 - ref).max())
    print(f"B = 1: max |cos - oracle| {e1:.3e}")
    assert e1 <= 1e-4
    worst = 0.0
    for B in BATCHES:
        got = m.cosine_device_many(full.dev[:B], PROMPTS).cpu().numpy()
        err, d1 = float(np.abs(got - ref[:B]).max()), float(np.abs(got - full.cos1[:B]).max())
        print(f"B = {B}: max |cos - oracle| {err:.3e}, max |cos_B - cos_1| {d1:.3e}")
        assert err <= 1e-4, (B, err)
        worst = max(worst, d1)
    assert worst <= BATCH_VS_B1_PIN, worst


def test_outlier_weights_batch8_vs_oracle():
    """trained-checkpoint-like LayerNorm outlier channels at B = 8, the batch of the configs[4] slice (8 envs per GPU)"""
    s = _setup(True, 8, 8)
    got = s.m.cosine_device_many(s.dev, PROMPTS).cpu().numpy()
    err = float(np.abs(got - s.ref).max())
    print(f"outliers, B = 8: max |cos - oracle| {err:.3e}")
    assert err <= 1e-4


@pytest.mark.parametrize("B", [3, 4, 32])
def test_rows_independent_bitwise(full, B):
    """A row's arithmetic depends on its position and on B, never on the other frames' data: replacing every frame but those at
    {0, 13 mod B, B - 1} leaves their q_proj rows and cosines unchanged to the bit."""
    m, Q = full.m, full.dims.queries
    keep = sorted({0, 13 % B, B - 1})
    a = full.dev[:B].clone()
    b = a.clone()
    rng = np.random.default_rng(100 + B)
    for i in range(B):
        if i not in keep:
            b[i] = torch.from_numpy(make_rgb(rng, 480, 640)).cuda()
    ca = m.cosine_device_many(a, PROMPTS).clone()
    qa = m.engine.q_proj[: B * Q].clone()
    cb = m.cosine_device_many(b, PROMPTS).clone()
    qb = m.engine.q_proj[: B * Q].clone()
    for i in keep:
        assert torch.equal(ca[i], cb[i]), (B, i)
        assert torch.equal(qa[i * Q : (i + 1) * Q], qb[i * Q : (i + 1) * Q]), (B, i)
    if len(keep) < B:
        assert not torch.equal(ca, cb)


@pytest.mark.parametrize("B", [3, 32])
def test_graph_replays_and_eager_bitwise(full, B):
    """three graph replays on distinct copies of one batch agree to the bit, and so does the eager (uncaptured) forward"""
    m, Q = full.m, full.dims.queries
    m.cosine_device_many(full.dev[:B].clone(), PROMPTS)          # warm-up: the first call of a shape runs eagerly
    outs = []
    for _ in range(3):
        c = m.cosine_device_many(full.dev[:B].clone(), PROMPTS).clone()
        outs.append((c, m.engine.q_proj[: B * Q].clone()))
    assert (B, *full.dev.shape[1:3]) in m.engine.graphs.captured
    m.engine.use_graph = False
    try:
        c = m.cosine_device_many(full.dev[:B].clone(), PROMPTS).clone()
        outs.append((c, m.engine.q_proj[: B * Q].clone()))
    finally:
        m.engine.use_graph = True
    for c, q in outs[1:]:
        assert torch.equal(c, outs[0][0]) and torch.equal(q, outs[0][1])


def test_preprocess_and_image_tokens_at_batch32(full):
    """After a 32-frame forward: the im2col bytes of frames 0, 17 and 31 equal PIL's (up to the fp16 store), and the post-LN
    image tokens of frames 0 and 31 are as close to the oracle as the same frame's at batch 1 (mean within 1.25x, max 1.5x)."""
    m, d, orc = full.m, full.dims, full.orc
    e = m.engine
    T, D, G = d.tokens, d.v_hidden, d.image // d.patch
    m.cosine_device_many(full.dev, PROMPTS)
    torch.cuda.synchronize()
    col = e.b_col[: 32 * (T - 1)].float().cpu().numpy().reshape(32, G, G, -1)[..., : d.patch_k]
    col = col.reshape(32, G, G, 3, d.patch, d.patch).transpose(0, 3, 1, 4, 2, 5).reshape(32, 3, d.image, d.image)
    for b in (0, 17, 31):
        assert np.array_equal(col[b], blip2_oracle.preprocess(full.imgs[b], d.image).half().float().numpy()), b
    tok32 = e.b_img[: 32 * T].float().cpu().numpy().reshape(32, T, D)
    for b in (0, 31):
        tref = orc.image_tokens(full.imgs[b]).numpy()
        m.cosine_device_many(full.dev[b : b + 1], PROMPTS)
        torch.cuda.synchronize()
        tok1 = e.b_img[:T].float().cpu().numpy()
        e32, e1 = np.abs(tok32[b] - tref), np.abs(tok1 - tref)
        print(f"frame {b}: image-token error at B = 32 mean {e32.mean():.3e} max {e32.max():.3e}; at B = 1 mean {e1.mean():.3e} max {e1.max():.3e}")
        assert e32.mean() <= 1.25 * e1.mean() and e32.max() <= 1.5 * e1.max()


def test_resid_ln_never_reduces_with_atomics():
    """vlfm_gemm_f16_resid_ln reduces a split K only through its workspace, in K order; a split that does not fit runs unsplit.

    Probe: x = 2^24, bias 0, A = 1 in K-columns 0 and K - 1 (0 elsewhere), W = 0.75 there.  Unsplit, the GEMM adds 1.5 once:
    x = 2^24 + 2.  Any split (uniform or stream-K) has the first and last K-blocks in different splits, added one at a time:
    2^24 + 0.75 rounds back to 2^24.  So at M = 257 B for B = 1..64, for the ViT's proj (K = 1408) and fc2 (K = 6144), with the
    engine's workspace and with a smaller one (8 slabs of at most 1024 rows), each prefilled with NaN:
      - x is 2^24 or 2^24 + 2 everywhere, and the LayerNorm output is finite;
      - x = 2^24 (a split) implies the workspace was written: the splits were not added into x with red.global.add;
      - when the workspace holds fewer than 2 M N floats and the 128 x 128 tiles fill the SMs (no stream-K), x = 2^24 + 2."""
    from vlfm_b200 import _lib as L
    from vlfm_b200.vlm.blip2_engine import partials_floats

    lib = L.load()
    dims = Blip2Dims()
    N, sms = dims.v_hidden, torch.cuda.get_device_properties(0).multi_processor_count
    big, one = 2.0 ** 24, 2.0 ** 24 + 2
    bias, gam, bet = torch.zeros(N, device="cuda"), torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    plans = {}
    for name, K in (("proj", dims.v_hidden), ("fc2", dims.v_inter)):
        A = torch.zeros(dims.tokens * 64, K, dtype=torch.float16, device="cuda")
        A[:, 0] = A[:, K - 1] = 1.0
        W = torch.zeros(N, K, dtype=torch.float16, device="cuda")
        W[:, 0] = W[:, K - 1] = 0.75
        split = []
        for B, nf in ((B, nf) for B in range(1, 65) for nf in {partials_floats(dims, B), 8 * min(dims.tokens * B, 1024) * N}):
            M = dims.tokens * B
            part = torch.full((nf,), float("nan"), device="cuda")
            x = torch.full((M, N), big, device="cuda")
            o16 = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
            L.check(lib.vlfm_gemm_f16_resid_ln(A.data_ptr(), W.data_ptr(), bias.data_ptr(), x.data_ptr(), M, N, K, K, K, N, gam.data_ptr(),
                                               bet.data_ptr(), o16.data_ptr(), N, None, 0, 1e-6, part.data_ptr(), nf * 4, L.stream_ptr()),
                    "vlfm_gemm_f16_resid_ln")
            torch.cuda.synchronize()
            vals = set(torch.unique(x).tolist())
            assert vals <= {big, one}, (name, B, sorted(vals)[:4])
            assert bool(torch.isfinite(o16).all()), (name, B)
            if big in vals:
                split.append((B, nf // (M * N)))
                assert not bool(torch.isnan(part).all()), f"{name} B = {B}: split K reduced without the workspace (atomics)"
            if nf < 2 * M * N and (M // 128) * math.ceil(N / 128) >= sms:
                assert vals == {one}, (name, B)
        plans[name] = split
    print("(batch, workspace / (M N)) whose residual GEMM split K:", plans)
