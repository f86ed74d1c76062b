"""MobileSAM on the GPU against the fp32 oracle (oracle/sam_oracle.py), plus batching, determinism, the frame cache and the
class surface.

Bars are set from the oracle alone, before any GPU run: the same oracle with every GEMM / conv operand rounded to fp16
(``fp16_operands=True``) drifts from the fp32 oracle by some amount; the engine, which rounds the same operands, must stay
within twice that drift (max abs).  For the final masks the bar on the low-res logits, tau, also bounds the error of the
full-resolution logits (both bilinear resizes are convex combinations), so every pixel with |oracle logit| > tau must agree.
"""
import numpy as np
import pytest
import torch

from oracle.sam_oracle import SamOracle, apply_box, preprocess
from vlfm_b200.utils.synthetic import make_rgb
from vlfm_b200.vlm.sam import MobileSAM, MobileSAMClient
from vlfm_b200.vlm.sam_config import TINY, VIT_T, random_state_dict

pytestmark = pytest.mark.gpu

SIZES = [(480, 640), (640, 480), (1024, 1024), (120, 160)]


def boxes_for(H, W):
    return {
        "inside": [W * 0.2, H * 0.25, W * 0.7, H * 0.8],
        "edges": [0, 0, W - 1, H * 0.6],
        "off_frame": [-W * 0.1, H * 0.5, W * 0.5, H * 1.2],
        "degenerate": [W * 0.4, H * 0.2, W * 0.4, H * 0.7],
        "fractional": [W * 0.13 + 0.37, H * 0.31 + 0.61, W * 0.58 + 0.29, H * 0.77 + 0.13],
    }


def frame(H, W, seed):
    rng = np.random.default_rng(seed)
    return make_rgb(rng, H, W)


@pytest.fixture(scope="module")
def models():
    out = {}
    for name, d in (("vit_t", VIT_T), ("tiny", TINY)):
        sd = random_state_dict(d, 0)
        out[name] = (d, sd, SamOracle(d, sd), SamOracle(d, sd, fp16_operands=True),
                     MobileSAM(state_dict=sd, dims=d, max_batch=3, device="cuda:0"))
    return out


def engine_low(sam, image, box):
    """engine low-res logits of one box on one frame (device encode + decode)"""
    img = torch.from_numpy(image).cuda()[None]
    sam.engine.encode(img)
    _, low = sam.engine.decode(torch.tensor([box], dtype=torch.float64), torch.zeros(1, dtype=torch.int32), image.shape[:2], low_out=True)
    return low[0].float().cpu()


@pytest.mark.parametrize("hw", SIZES)
def test_preprocess_matches_oracle(models, hw):
    d, _, orc, _, sam = models["vit_t"]
    img = frame(*hw, seed=hw[0])
    ref, _ = preprocess(img, d.img_size)
    got = sam.engine.preprocess(torch.from_numpy(img).cuda()[None]).cpu()
    assert torch.equal(got[0].permute(2, 0, 1), ref[0].half())


@pytest.mark.parametrize("name", ["vit_t", "tiny"])
def test_encoder_and_low_res_logits(models, name):
    d, _, orc, orc16, sam = models[name]
    img = frame(480, 640, seed=5)
    box = boxes_for(480, 640)["inside"]
    x, _ = preprocess(img, d.img_size)
    with torch.no_grad():
        e32, e16 = orc.encode(x), orc16.encode(x)
        l32, l16 = orc.low_res_logits(e32, box, img.shape[:2]), orc16.low_res_logits(e16, box, img.shape[:2])
    low = engine_low(sam, img, box)
    emb = sam.engine.emb[0].cpu().view(d.emb_side, d.emb_side, d.prompt_dim).permute(2, 0, 1)
    e_drift, l_drift = (e16 - e32).abs().max().item(), (l16 - l32).abs().max().item()
    e_err, l_err = (emb - e32[0]).abs().max().item(), (low - l32).abs().max().item()
    print(f"\n{name}: embedding err {e_err:.3e} (fp16-operand drift {e_drift:.3e}); low-res err {l_err:.3e} (drift {l_drift:.3e})")
    assert e_err <= 2 * e_drift
    assert l_err <= 2 * l_drift


@pytest.mark.parametrize("hw", SIZES)
def test_final_masks(models, hw):
    d, _, orc, orc16, sam = models["vit_t"]
    H, W = hw
    img = frame(H, W, seed=H + W)
    x, _ = preprocess(img, d.img_size)
    with torch.no_grad():
        e32, e16 = orc.encode(x), orc16.encode(x)
    names, boxes = zip(*boxes_for(H, W).items())
    got = sam.segment_bboxes(img, list(boxes))
    for i, (name, box) in enumerate(zip(names, boxes)):
        with torch.no_grad():
            l32, l16 = orc.low_res_logits(e32, box, hw), orc16.low_res_logits(e16, box, hw)
            full = orc.postprocess(l32, hw).numpy()
        tau = 2 * (l16 - l32).abs().max().item()
        low = engine_low(sam, img, box)
        assert (low - l32).abs().max().item() <= tau, name
        ref = full > 0
        x0, x1 = sorted((int(np.clip(box[0], 0, W - 1)), int(np.clip(box[2], 0, W - 1))))
        y0, y1 = sorted((int(np.clip(box[1], 0, H - 1)), int(np.clip(box[3], 0, H - 1))))
        inside = ref[y0:y1 + 1, x0:x1 + 1] if (x1 - x0 + 1) * (y1 - y0 + 1) >= 64 else ref
        assert 0.05 <= inside.mean() <= 0.95, f"{name}: oracle mask is {inside.mean():.3f} positive inside the box"
        sure = np.abs(full) > tau
        assert np.array_equal(got[i][sure], ref[sure]), name
        print(f"\n{hw} {name}: tau {tau:.3e}, pixels compared {sure.mean():.4f}, disagreeing {(got[i] != ref).mean():.2e}")


@pytest.mark.parametrize("n", [1, 2, 5, 17])
def test_segment_bboxes_rows_equal_single_calls(models, n):
    _, _, _, _, sam = models["vit_t"]
    img = frame(480, 640, seed=11)
    rng = np.random.default_rng(n)
    xy = rng.uniform(-40, 680, (n, 2)), rng.uniform(-40, 520, (n, 2))
    boxes = [[min(a), min(b), max(a), max(b)] for a, b in zip(xy[0], xy[1])]
    many = sam.segment_bboxes(img, boxes)
    assert many.shape == (n, 480, 640) and many.dtype == bool
    for i, b in enumerate(boxes):
        assert np.array_equal(sam.segment_bbox(img, b), many[i])


def test_device_batch_with_shuffled_frames(models):
    _, _, _, _, sam = models["vit_t"]
    imgs = torch.from_numpy(np.stack([frame(480, 640, seed=20 + i) for i in range(3)])).cuda()
    boxes = torch.tensor([[100, 80, 400, 300], [10, 20, 600, 470], [250.5, 100.25, 251.5, 400], [0, 0, 639, 479],
                          [300, 200, 500, 460], [-20, 50, 200, 520]], dtype=torch.float64)
    fidx = torch.tensor([2, 0, 1, 2, 1, 0], dtype=torch.int32)
    batched = sam.segment_bboxes_device(imgs, boxes.cuda(), fidx.cuda()).cpu()
    for f in range(3):
        sel = (fidx == f).nonzero().flatten()
        single = sam.segment_bboxes_device(imgs[f:f + 1], boxes[sel].cuda(), torch.zeros(len(sel), dtype=torch.int32).cuda()).cpu()
        assert torch.equal(batched[sel], single)


def test_deterministic(models):
    _, _, _, _, sam = models["vit_t"]
    img = frame(480, 640, seed=3)
    a = engine_low(sam, img, [50, 60, 300, 400])
    emb_a = sam.engine.emb[0].clone()
    b = engine_low(sam, img, [50, 60, 300, 400])
    assert torch.equal(a, b) and torch.equal(emb_a, sam.engine.emb[0])


def test_frame_cache(models):
    _, _, _, _, sam = models["vit_t"]
    img = frame(480, 640, seed=8)
    dets = [[20, 30, 200, 250], [300, 100, 600, 400], [100.5, 200.5, 350.5, 470.5]]
    g0 = sam.engine.generation
    cached = [sam.segment_bbox(img, b) for b in dets]          # the policy's per-detection loop on one frame object
    assert sam.engine.generation == g0 + 1
    img[0, 0, 0] ^= 1                                           # in-place refill: re-encode
    sam.segment_bbox(img, dets[0])
    assert sam.engine.generation == g0 + 2
    img[0, 0, 0] ^= 1
    fresh = [sam.segment_bbox(img.copy(), b) for b in dets]     # a different object every call: re-encode each time
    assert sam.engine.generation == g0 + 5
    assert all(np.array_equal(a, b) for a, b in zip(cached, fresh))
    sam.segment_bbox(img, dets[0])
    g1 = sam.engine.generation
    sam.segment_bboxes_device(torch.from_numpy(img).cuda()[None], torch.tensor([dets[0]]).cuda(), torch.zeros(1, dtype=torch.int32).cuda())
    again = sam.segment_bbox(img, dets[1])                      # an intervening forward: re-encode
    assert sam.engine.generation == g1 + 2
    assert np.array_equal(again, cached[1])


def test_surface(models, monkeypatch):
    d, sd, _, _, sam = models["tiny"]
    img = frame(120, 160, seed=1)
    m = MobileSAMClient(model=sam).segment_bbox(img, [10, 20, 90, 100])
    assert isinstance(m, np.ndarray) and m.dtype == bool and m.shape == (120, 160)
    assert np.array_equal(m, sam.segment_bbox(img, [10.0, 20.0, 90.0, 100.0]))
    monkeypatch.delenv("MOBILE_SAM_CHECKPOINT", raising=False)
    with pytest.raises(FileNotFoundError):
        MobileSAM(dims=d)
    with pytest.raises(ValueError):
        MobileSAM(model_type="vit_h", state_dict=sd, dims=d)
    # the box goes through apply_boxes exactly as the oracle's
    assert torch.equal(apply_box([10, 20, 90, 100], (120, 160), d.img_size), torch.tensor([[16.0, 32.0, 144.0, 160.0]]))
