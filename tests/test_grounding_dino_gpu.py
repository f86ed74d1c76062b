"""GroundingDINO: Swin-T backbone on the hand-written kernels vs the fp32 HF oracle, and the
predict() surface.  Tolerances stated per check (fp16 tensor-core operands, fp32 accumulate)."""
import numpy as np
import pytest
import torch

from oracle.gdino_oracle import GdinoOracle
from vlfm_b200.utils.synthetic import make_rgb

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pair():
    from vlfm_b200.vlm.grounding_dino import GroundingDINO

    orc = GdinoOracle(0)
    g = GroundingDINO(state_dict={k: v.clone() for k, v in orc.state_dict().items()}, seed=0, synthetic=True)
    return orc, g


@pytest.mark.parametrize("hw", [(480, 640), (225, 318)])   # second: not a multiple of 4 / 7 / 2 anywhere
def test_swin_backbone_feature_maps(pair, hw):
    orc, g = pair
    img = make_rgb(np.random.default_rng(hw[0]), *hw)
    ref = orc.backbone_features(img)
    got = g.backbone.forward(torch.from_numpy(img[None]).cuda())
    torch.cuda.synchronize()
    assert len(ref) == len(got) == 3
    for r, o in zip(ref, got):
        o = o[0].cpu()
        assert o.shape == r.shape
        err = (o - r).abs()
        print("stage", tuple(r.shape), "max", float(err.max()), "mean", float(err.mean()))
        assert float(err.mean()) <= 5e-3 and float(err.max()) <= 1e-1


def test_predict_surface_and_outputs(pair):
    orc, g = pair
    img = make_rgb(np.random.default_rng(5), 480, 640)
    ids = g.tokenizer.encode("chair . person . dog .")
    ref_l, ref_b = orc.raw_outputs(img, ids)
    got_l, got_b = g.raw_outputs(img, ids)
    got_l, got_b = got_l.cpu(), got_b.cpu()
    assert got_l.shape == ref_l.shape == (900, 256) and got_b.shape == (900, 4)
    print("logit mean abs err", float((got_l - ref_l).abs().mean()), "box mean abs err", float((got_b - ref_b).abs().mean()))
    # the 900 queries come from a top-k over near-tied random-weight scores, so rows can permute between the
    # two runs: compare logits per row loosely and boxes as sets (nearest-neighbour distance)
    assert float((got_l - ref_l).abs().mean()) <= 1e-2
    d = (got_b[:, None, :] - ref_b[None, :, :]).abs().sum(-1).min(dim=1)[0]
    print("box set distance mean", float(d.mean()))
    assert float(d.mean()) <= 2e-2
    det = g.predict(img)                       # default caption (grounding_dino.py:20)
    assert det.boxes.shape[1] == 4 and len(det.phrases) == det.boxes.shape[0] == det.logits.shape[0]
    assert all(p in ("chair", "person", "dog") for p in det.phrases)     # filter_by_class
    assert (det.boxes[:, 2] >= det.boxes[:, 0]).all()                    # xyxy
    j = det.to_json()
    from vlfm_b200.vlm.detections import ObjectDetections

    back = ObjectDetections.from_json(j, image_source=img)
    assert back.num_detections == det.num_detections


def test_tc_linear_and_cast_vs_torch():
    from vlfm_b200.vlm.dense import cast_f16
    from vlfm_b200.vlm.gdino_accel import TcLinear

    torch.manual_seed(1)
    x = torch.randn(3, 1001, 256, device="cuda")
    assert torch.equal(cast_f16(x.reshape(-1)[:1001 * 3 + 2].contiguous()), x.reshape(-1)[:1001 * 3 + 2].half())   # tail path
    for n_out in (384, 2048, 128):
        lin = torch.nn.Linear(256, n_out).cuda()
        ref = lin(x)
        got = TcLinear(lin)(x)
        torch.cuda.synchronize()
        # fp16 operands (11-bit mantissa), fp32 accumulate over K=256: |err| <~ 2^-11 * sum|x_k w_k|
        err = float((got - ref).abs().max())
        print("TcLinear", n_out, "max abs err", err)
        assert got.shape == ref.shape and err <= 5e-3


def test_accelerated_primitives_are_installed(pair):
    _, g = pair
    # 6 encoder deformable layers rewritten whole, 6 decoder cross-attentions, every other nn.Linear on the wgmma GEMM
    assert g.accel["deformable_layers"] == 6 and g.accel["decoder_layers"] == 6 and g.accel["fusion_layers"] == 6, g.accel
    assert g.accel["linear"] > 60, g.accel


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_fused_deformable_attention_vs_hf_module(ref_dim):
    """TcDeformAttn (cast+pos, value / offsets|logits GEMMs, fused softmax+locations+gather, output GEMM) against the HF
    fp32 module it replaces.  fp16 GEMM operands and fp16 values: |err| <= 2e-2 absolute on O(1) outputs, mean <= 2e-3."""
    from transformers import GroundingDinoConfig
    from transformers.models.grounding_dino.modeling_grounding_dino import GroundingDinoMultiscaleDeformableAttention
    from vlfm_b200.vlm.gdino_accel import TcDeformAttn

    torch.manual_seed(2)
    cfg = GroundingDinoConfig()
    m = GroundingDinoMultiscaleDeformableAttention(cfg, num_heads=8, n_points=4).cuda().eval()
    with torch.no_grad():
        m.sampling_offsets.weight.normal_(0, 0.05); m.sampling_offsets.bias.normal_(0, 1.0)
        m.attention_weights.weight.normal_(0, 0.05); m.attention_weights.bias.normal_(0, 0.5)
    shapes = [(60, 80), (30, 40), (15, 20), (8, 10)]
    s = sum(h * w for h, w in shapes)
    b = 2
    q = s if ref_dim == 2 else 900
    enc = torch.randn(b, s, 256, device="cuda")
    hid = enc if ref_dim == 2 else torch.randn(b, q, 256, device="cuda")
    pos = torch.randn(b, q, 256, device="cuda") * 0.5
    ref = torch.rand(b, q, 4, ref_dim, device="cuda")
    if ref_dim == 4:
        ref[..., 2:] *= 0.3
    sp = torch.tensor(shapes, device="cuda")
    start = torch.cat([sp.new_zeros(1), (sp[:, 0] * sp[:, 1]).cumsum(0)[:-1]])
    with torch.no_grad():
        want, _ = m(hid, attention_mask=None, encoder_hidden_states=enc, position_embeddings=pos, reference_points=ref, spatial_shapes=sp,
                    spatial_shapes_list=shapes, level_start_index=start)
        got, _ = TcDeformAttn(m)(hid, attention_mask=None, encoder_hidden_states=enc, position_embeddings=pos, reference_points=ref,
                                 spatial_shapes=sp, spatial_shapes_list=shapes, level_start_index=start)
    torch.cuda.synchronize()
    err = (got - want).abs()
    print("deform attn ref_dim", ref_dim, "max", float(err.max()), "mean", float(err.mean()), "ref scale", float(want.abs().mean()))
    assert float(err.max()) <= 2e-2 and float(err.mean()) <= 2e-3


@pytest.mark.parametrize("nq,nk", [(777, 10), (10, 777), (64, 130), (3, 6380), (130, 48)])
def test_biattn_kernel_vs_torch(nq, nk):
    """vlfm_biattn_f16 (head_dim 256; key chunks merged by log-sum-exp) against fp32 torch attention on the same fp16
    inputs.  Tolerance 3e-3 (fp16 probabilities and outputs)."""
    from vlfm_b200.vlm.gdino_accel import biattn_f16

    torch.manual_seed(nq * 1000 + nk)
    b, heads = 2, 4
    q = (torch.randn(b * nq, heads * 256, device="cuda") * 0.5).half()
    kv = (torch.randn(b * nk, 2 * heads * 256, device="cuda") * 0.5).half()       # keys | values interleaved like the fused projection
    k, v = kv[:, : heads * 256], kv[:, heads * 256 :]
    scale = 256 ** -0.5
    got = biattn_f16(q, k, v, b, heads, nq, nk, scale)
    qf = q.float().view(b, nq, heads, 256).transpose(1, 2)
    kf = k.float().reshape(b, nk, heads, 256).transpose(1, 2)
    vf = v.float().reshape(b, nk, heads, 256).transpose(1, 2)
    want = (torch.softmax(qf @ kf.transpose(-1, -2) * scale, -1) @ vf).transpose(1, 2).reshape(b * nq, heads * 256)
    torch.cuda.synchronize()
    err = float((got.float() - want).abs().max())
    print("biattn", nq, nk, "max abs err", err)
    assert err <= 3e-3


def test_fusion_layer_vs_hf_module():
    """TcFusionLayer against the HF fp32 GroundingDinoFusionLayer it replaces (layer scale set to O(1) so that the attention
    path is visible in the output).  fp16 operands: max |err| <= 3e-2, mean <= 3e-3 on O(1) outputs."""
    from transformers import GroundingDinoConfig
    from transformers.models.grounding_dino.modeling_grounding_dino import GroundingDinoFusionLayer
    from vlfm_b200.vlm.gdino_accel import TcFusionLayer

    torch.manual_seed(3)
    m = GroundingDinoFusionLayer(GroundingDinoConfig()).cuda().eval()
    with torch.no_grad():
        m.vision_param.fill_(0.7); m.text_param.fill_(0.9)
    b, nv, t = 2, 1500, 12
    vis = torch.randn(b, nv, 256, device="cuda")
    txt = torch.randn(b, t, 256, device="cuda")
    with torch.no_grad():
        (wv, _), (wt, _) = m(vis, txt, attention_mask_vision=None, attention_mask_text=None)
        (gv, _), (gt, _) = TcFusionLayer(m)(vis, txt)
    torch.cuda.synchronize()
    ev, et = (gv - wv).abs(), (gt - wt).abs()
    print("fusion vision max", float(ev.max()), "mean", float(ev.mean()), "text max", float(et.max()), "mean", float(et.mean()))
    assert float(ev.max()) <= 3e-2 and float(ev.mean()) <= 3e-3 and float(et.max()) <= 3e-2 and float(et.mean()) <= 3e-3


@pytest.mark.parametrize("nq,nk,kc", [(900, 900, 0), (900, 12, 0), (130, 2000, 512), (7, 33, 0)])
def test_biattn_head_dim_32_vs_torch(nq, nk, kc):
    """Decoder-shaped attention (8 heads x 32) on vlfm_biattn_f16 against fp32 torch attention; tolerance 3e-3."""
    from vlfm_b200.vlm.gdino_accel import biattn_f16

    torch.manual_seed(nq + nk)
    b, heads = 3, 8
    qk = (torch.randn(b * nq, 2 * heads * 32, device="cuda")).half()
    q = qk[:, : heads * 32]
    kv = (torch.randn(b * nk, 2 * heads * 32, device="cuda")).half()
    k, v = kv[:, : heads * 32], kv[:, heads * 32 :]
    scale = 32 ** -0.5
    got = biattn_f16(q, k, v, b, heads, nq, nk, scale, key_chunk=kc, head_dim=32)
    qf = q.float().reshape(b, nq, heads, 32).transpose(1, 2)
    kf = k.float().reshape(b, nk, heads, 32).transpose(1, 2)
    vf = v.float().reshape(b, nk, heads, 32).transpose(1, 2)
    want = (torch.softmax(qf @ kf.transpose(-1, -2) * scale, -1) @ vf).transpose(1, 2).reshape(b * nq, heads * 32)
    torch.cuda.synchronize()
    err = float((got.float() - want).abs().max())
    print("biattn32", nq, nk, "max abs err", err)
    assert err <= 3e-3


def test_decoder_layer_vs_hf_module():
    """TcDecoderLayer against the HF fp32 GroundingDinoDecoderLayer it replaces; fp16 operands: max <= 5e-2, mean <= 5e-3 on
    LayerNorm-scaled (O(1)) outputs."""
    from transformers import GroundingDinoConfig
    from transformers.models.grounding_dino.modeling_grounding_dino import GroundingDinoDecoderLayer
    from vlfm_b200.vlm.gdino_accel import TcDecoderLayer

    torch.manual_seed(4)
    m = GroundingDinoDecoderLayer(GroundingDinoConfig()).cuda().eval()
    with torch.no_grad():
        m.encoder_attn.sampling_offsets.weight.normal_(0, 0.05); m.encoder_attn.sampling_offsets.bias.normal_(0, 1.0)
        m.encoder_attn.attention_weights.weight.normal_(0, 0.05); m.encoder_attn.attention_weights.bias.normal_(0, 0.5)
    shapes = [(30, 40), (15, 20), (8, 10), (4, 5)]
    s = sum(h * w for h, w in shapes)
    b, nq, t = 2, 900, 11
    hid = torch.randn(b, nq, 256, device="cuda")
    pos = torch.randn(b, nq, 256, device="cuda") * 0.5
    enc = torch.randn(b, s, 256, device="cuda")
    txt = torch.randn(b, t, 256, device="cuda")
    ref = torch.rand(b, nq, 4, 4, device="cuda"); ref[..., 2:] *= 0.3
    sp = torch.tensor(shapes, device="cuda")
    start = torch.cat([sp.new_zeros(1), (sp[:, 0] * sp[:, 1]).cumsum(0)[:-1]])
    kw = dict(position_embeddings=pos, reference_points=ref, spatial_shapes=sp, spatial_shapes_list=shapes, level_start_index=start,
              vision_encoder_hidden_states=enc, vision_encoder_attention_mask=None, text_encoder_hidden_states=txt,
              text_encoder_attention_mask=None, self_attn_mask=None)
    with torch.no_grad():
        want = m(hid, **kw)[0]
        got = TcDecoderLayer(m)(hid, **kw)[0]
    torch.cuda.synchronize()
    err = (got - want).abs()
    print("decoder layer max", float(err.max()), "mean", float(err.mean()))
    assert float(err.max()) <= 5e-2 and float(err.mean()) <= 5e-3


def test_batch1_cuda_graph_replay_matches_eager(pair):
    """The per-step policy call (batch 1) replays a CUDA graph of the whole detector from the second call on; its outputs must
    be those of the eager forward.  With random weights the 900-of-6380 query selection is a top-k over near-tied scores,
    so even two EAGER runs differ (fp32 atomics order in the split-K GEMMs flips selections): the graph-vs-eager difference is
    held to the same level as eager-vs-eager, measured here on the spot (sorted confidences, boxes as sets)."""
    import time

    _, g = pair
    ids = g.tokenizer.encode("chair . couch . tv .")
    rng = np.random.default_rng(11)
    img1, img2 = make_rgb(rng, 480, 640), make_rgb(rng, 480, 640)

    def metrics(la, ba, lb, bb):
        ca, cb = la.max(dim=1)[0].sort()[0], lb.max(dim=1)[0].sort()[0]
        dist = (bb[:, None, :] - ba[None, :, :]).abs().sum(-1).min(dim=1)[0]
        return float((ca - cb).abs().mean()), float(dist.mean())

    g.use_graph = False                                               # eager baseline: same image twice
    e0 = [t.clone() for t in g.raw_outputs(img1, ids)]
    e1 = [t.clone() for t in g.raw_outputs(img1, ids)]
    g.use_graph = True
    g.raw_outputs(img2, ids)                                          # capture + first replay (this key already ran eagerly)
    assert g.graphs.error is None, g.graphs.error
    assert (1, 480, 640, tuple(ids)) in g.graphs.captured
    r = [t.clone() for t in g.raw_outputs(img1, ids)]                 # replay
    ee, ge = metrics(e0[0], e0[1], e1[0], e1[1]), metrics(e0[0], e0[1], r[0], r[1])
    print("eager vs eager (confidence, box-set):", ee, " graph vs eager:", ge)
    # run-to-run differences are a few 1e-4 .. 1e-3 of mean confidence (a broken replay is off by > 1e-1)
    assert ge[0] <= max(5e-3, 3 * ee[0]) and ge[1] <= max(1e-3, 3 * ee[1])
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(10):
        g.raw_outputs(img1, ids)
    torch.cuda.synchronize()
    print(f"batch-1 GroundingDINO forward (graph replay incl. H2D): {(time.perf_counter() - t0) * 100:.2f} ms")


@pytest.fixture(scope="module")
def pair_calibrated():
    """Same seeded weights with the decoder's output LayerNorm scaled by 0.1: with plain random weights the contrastive
    logits (dot products of two un-normalised 256-d vectors) saturate the sigmoid at 0 / 1 and every decision is trivial."""
    from vlfm_b200.vlm.grounding_dino import GroundingDINO

    orc = GdinoOracle(0)
    sd = orc.model.state_dict()
    for k in ("model.decoder.layer_norm.weight", "model.decoder.layer_norm.bias"):
        sd[k].mul_(0.1)
    g = GroundingDINO(state_dict={k: v.clone() for k, v in orc.state_dict().items()}, seed=0, synthetic=True)
    return orc, g


def test_detection_decisions_match_the_fp32_twin(pair_calibrated):
    """Decision level: which queries pass box_threshold, which tokens pass text_threshold (the phrase) and where the box is.
    A random-weight GroundingDINO is badly conditioned: the fp32 twin moves ITS OWN class scores by ~0.03 on average (p99 0.2)
    when its input pixels are perturbed by 2^-11 relative -- one half-precision rounding (measured below, every run).  A fixed
    tolerance would therefore test the weights, not the kernels; the bar is the twin's own conditioning:
      * rows are paired by PROPOSAL IDENTITY (the initial reference point the decoder receives; the 900 rows permute between two
        computations because the query selection is a top-k over near-tied scores);
      * decision = (kept: score > box_thr, phrase: tokens > text_thr), thresholds at quantiles of the twin's score distribution
        (synthetic scores have no natural gap at 0.35 / 0.25);
      * the fraction of paired decisions that differ between OUR forward and the twin, the mean |score difference| and the mean box
        L1 distance must not exceed 2x (+ a small floor; measured 1.6-1.7x) what the twin shows against its own perturbed run, and at most 5 % of
        the proposals may be unpaired."""
    orc, g = pair_calibrated
    EPS16 = 2.0 ** -11
    cap = {}
    h1 = orc.model.model.decoder.register_forward_hook(lambda m_, a_, kw, o_: cap.__setitem__("ref", kw["reference_points"][0].detach().float().cpu()), with_kwargs=True)
    use_graph, g.use_graph = g.use_graph, False                                 # eager: every call sets g.fwd.last_reference_points
    stats = {"ours": [0, 0, 0, [], []], "twin": [0, 0, 0, [], []]}              # paired, unpaired, flipped, |dscore|, box L1
    try:
        for seed, caption in ((21, "chair . person . dog ."), (22, "couch . potted plant . tv .")):
            img = make_rgb(np.random.default_rng(seed), 480, 640)
            ids = g.tokenizer.encode(caption)
            ref_l, ref_b = (t.cpu().float() for t in orc.raw_outputs(img, ids))
            ref_p = cap["ref"]
            got_l, got_b = (t.cpu().float() for t in g.raw_outputs(img, ids))
            got_p = g.fwd.last_reference_points[0].detach().float().cpu()
            per_l, per_b = (t.cpu().float() for t in orc.raw_outputs(img, ids, input_noise=EPS16, noise_seed=seed))
            per_p = cap["ref"]
            box_thr = float(ref_l.max(dim=1)[0].quantile(0.5))
            text_thr = box_thr * 0.25 / 0.35

            def decision(row):
                pos = row > text_thr
                pos[0] = False
                pos[len(ids) - 1:] = False
                return bool(row.max() > box_thr), tuple(pos.nonzero(as_tuple=True)[0].tolist())

            for name, (dl, db, dp) in (("ours", (got_l, got_b, got_p)), ("twin", (per_l, per_b, per_p))):
                st = stats[name]
                dist, j = (ref_p[:, None, :] - dp[None, :, :]).abs().sum(-1).min(dim=1)
                for i in range(ref_l.shape[0]):
                    if float(dist[i]) > 4e-3:
                        st[1] += 1
                        continue
                    k = int(j[i])
                    st[0] += 1
                    da, dbb = decision(ref_l[i].clone()), decision(dl[k].clone())
                    st[2] += int(da[0] != dbb[0] or (da[0] and da[1] != dbb[1]))
                    st[3].append(abs(float(ref_l[i].max()) - float(dl[k].max())))
                    st[4].append(float((ref_b[i] - db[k]).abs().sum()))
    finally:
        h1.remove(); g.use_graph = use_graph
    rep = {}
    for name, st in stats.items():
        rep[name] = {"paired": st[0], "unpaired": st[1], "flipped": st[2] / max(st[0], 1), "dscore": float(np.mean(st[3])), "dbox": float(np.mean(st[4]))}
    print("decision test (fp16-operand forward vs fp32 twin | twin vs twin with 2^-11 relative input noise):", rep)
    o, t = rep["ours"], rep["twin"]
    assert o["paired"] >= 1700 and o["unpaired"] <= 0.05 * (o["paired"] + o["unpaired"])
    assert o["flipped"] <= 2.0 * t["flipped"] + 0.01, rep
    assert o["dscore"] <= 2.0 * t["dscore"] + 2e-3, rep
    assert o["dbox"] <= 2.0 * t["dbox"] + 2e-3, rep


def test_head_kernels_vs_torch():
    """csrc/gdino_head.cu through vlm/gdino_ops.py::LibOps against torch fp32: GroupNorm on NHWC rows, im2col of the 3x3 stride-2
    conv, masked cast, proposal scores, top-k, gather, box / class heads."""
    from vlfm_b200.vlm.gdino_ops import LibOps

    ops = LibOps()
    g = torch.Generator(device="cpu").manual_seed(5)
    B, h, w, C = 3, 15, 20, 768
    # GroupNorm into a flattened buffer at an offset
    y = torch.randn(B * h * w, 256, generator=g).cuda() * 3 + 0.5
    gam, bet = torch.randn(256, generator=g).cuda(), torch.randn(256, generator=g).cuda()
    S = h * w + 37
    out = torch.zeros(B, S, 256, device="cuda")
    ops.groupnorm_rows(y, B, h * w, 256, 32, gam, bet, 1e-5, out, 37, S)
    ref = torch.nn.functional.group_norm(y.view(B, h * w, 256).permute(0, 2, 1), 32, gam, bet, 1e-5).permute(0, 2, 1)
    assert float((out[:, 37:] - ref).abs().max()) <= 2e-5 and float(out[:, :37].abs().max()) == 0.0
    # im2col (ky, kx, c) order == conv2d with the permuted weight
    x = torch.randn(B * h * w, C, generator=g).cuda()
    col = ops.im2col3x3s2(x, B, h, w).float()
    wt = torch.randn(64, C, 3, 3, generator=g).cuda() * 0.02
    ref = torch.nn.functional.conv2d(x.view(B, h, w, C).permute(0, 3, 1, 2), wt, stride=2, padding=1)
    got = (col @ wt.permute(0, 2, 3, 1).reshape(64, -1).t()).view(B, ref.shape[2], ref.shape[3], 64).permute(0, 3, 1, 2)
    assert float((got - ref).abs().max()) <= 2e-2 * float(ref.abs().max())          # fp16 operand rounding of x
    # masked cast
    valid = (torch.rand(B * h * w, generator=g) > 0.3).to(torch.uint8).cuda()
    m = ops.mask_rows(x, valid).float()
    assert torch.equal(m, (x * valid[:, None]).half().float())
    # proposal scores / top-k / gather
    Sq, T = 1234, 9
    q = torch.randn(B * Sq, 256, generator=g).cuda()
    text = torch.randn(B * T, 256, generator=g).cuda()
    sc = ops.proposal_scores(q, text, B, Sq, T)
    ref = (q.view(B, Sq, 256) @ text.view(B, T, 256).transpose(1, 2)).max(-1)[0]
    assert float((sc - ref).abs().max()) <= 1e-3
    idx = ops.topk_rows(sc, 900)
    tv, ti = torch.topk(sc, 900, dim=1)
    assert torch.equal(torch.gather(sc, 1, idx), tv)                                    # same scores in the same (descending) order
    assert all(len(set(r.tolist())) == 900 for r in idx)
    # 1024 x 1024 frames: 21760 proposals -> radix-select path; quantised scores force ties at the cut (lower index wins, as torch.topk
    # does not promise -- so compare the score sequence and the tie rule separately)
    big = (torch.randn(B, 21760, generator=g) * 4).round().div(4).cuda()
    bi = ops.topk_rows(big, 900)
    bv, _ = torch.topk(big, 900, dim=1)
    assert torch.equal(torch.gather(big, 1, bi), bv)
    for r in range(B):
        ks = (-big[r].double()) * 1e6 + torch.arange(21760, device="cuda").double()      # descending score, then ascending index
        assert torch.equal(bi[r], torch.argsort(ks)[:900])
    gat = ops.gather_rows(q.view(B, Sq, 256), idx)
    assert torch.equal(gat, torch.gather(q.view(B, Sq, 256), 1, idx.unsqueeze(-1).repeat(1, 1, 256)))
    # decoder query positions: reference_points_input and the sine embedding operand, against the module code's expressions
    from transformers.models.grounding_dino.modeling_grounding_dino import get_sine_pos_embed

    rp = torch.rand(B, 900, 4, generator=g).cuda()
    vr = (0.7 + 0.3 * torch.rand(B, 4, 2, generator=g)).cuda()
    dim_t = (10000 ** (2 * torch.div(torch.arange(128, dtype=torch.float32), 2, rounding_mode="floor") / 128)).cuda()
    rin, emb = ops.decoder_query_pos(rp, vr, dim_t)
    rin_ref = rp[:, :, None] * torch.cat([vr, vr], -1)[:, None]
    assert torch.equal(rin, rin_ref)
    emb_ref = get_sine_pos_embed(rin_ref[:, :, 0, :], num_pos_feats=128).reshape(B * 900, 512)
    assert float((emb.float() - emb_ref.half().float()).abs().max()) <= 1e-3          # sinf / cosf of the same float32 argument, then fp16
    assert float((emb.float() - emb_ref).abs().max()) <= 1e-3
    # heads
    delta, refp = torch.randn(B, 900, 4, generator=g).cuda(), torch.rand(B, 900, 4, generator=g).cuda()
    refp[0, 0] = torch.tensor([0.0, 1.0, 0.5, 1e-7])
    bx = ops.box_finish(delta, refp)
    assert float((bx - (delta + torch.special.logit(refp, eps=1e-5)).sigmoid()).abs().max()) <= 1e-6
    hs = torch.randn(B, 900, 256, generator=g).cuda() * 0.2
    tx = text.view(B, T, 256)
    lg = ops.contrastive_sigmoid(hs, tx, 256)
    assert lg.shape == (B, 900, 256) and float(lg[..., T:].abs().max()) == 0.0
    assert float((lg[..., :T] - (hs @ tx.transpose(1, 2)).sigmoid()).abs().max()) <= 1e-5

