"""Each YOLOv7 entry point (csrc/yolo_ops.cu) alone, against cv2, torch, torchvision and float64: NaN-prefilled outputs, bitwise
repeat launches and a bad-argument table."""
import ctypes as C

import numpy as np
import pytest
import torch
import torchvision

cv2 = pytest.importorskip("cv2")

from vlfm_b200 import _lib
from vlfm_b200.vlm.yolov7_engine import IN_H, IN_W, MAX_DET, area_tables, scale_coords_params

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F16 = torch.float16


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return _lib.load()


def st():
    return _lib.stream_ptr()


def params(conf=0.25, iou=0.45, agnostic=False, classes=None):
    p = _lib.YoloParams()
    p.conf_thres, p.iou_thres, p.agnostic = conf, iou, int(agnostic)
    mask = [0] * 4
    for j in (range(80) if classes is None else classes):
        mask[j >> 5] |= 1 << (j & 31)
    for k in range(4):
        p.class_mask[k] = mask[k]
    return torch.frombuffer(bytearray(C.string_at(C.addressof(p), C.sizeof(p))), dtype=torch.int32).to(dev)


def nan16(*shape):
    return torch.full(shape, float("nan"), dtype=F16, device=dev)


@pytest.mark.parametrize("hw", [(480, 640), (720, 1280), (448, 640), (481, 1001)])
def test_preprocess_equals_cv2_then_torch(lib, hw):
    H, W = hw
    B = 2
    imgs = np.random.default_rng(H + W).integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    yo, ys, yb = (torch.from_numpy(a).to(dev) for a in area_tables(H, IN_H))
    xo, xs, xa = (torch.from_numpy(a).to(dev) for a in area_tables(W, IN_W))
    d_img = torch.from_numpy(imgs).to(dev)
    outs = []
    for _ in range(2):
        out = nan16(B, IN_H // 2, IN_W // 2, 16)
        _lib.check(lib.vlfm_yolo_preprocess(d_img.data_ptr(), out.data_ptr(), B, H, W, IN_H, IN_W, yo.data_ptr(), ys.data_ptr(), yb.data_ptr(),
                                            xo.data_ptr(), xs.data_ptr(), xa.data_ptr(), st()), "preprocess")
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    for b in range(B):
        ref = torch.from_numpy(cv2.resize(imgs[b], (IN_W, IN_H), interpolation=cv2.INTER_AREA)).to(dev).permute(2, 0, 1).half() / 255.0
        reorg = torch.cat([ref[:, ::2, ::2], ref[:, 1::2, ::2], ref[:, ::2, 1::2], ref[:, 1::2, 1::2]], 0).permute(1, 2, 0)
        assert torch.equal(outs[0][b, ..., :12].view(torch.int16), reorg.contiguous().view(torch.int16))
        assert torch.equal(outs[0][b, ..., 12:], torch.zeros_like(outs[0][b, ..., 12:]))


def test_pools_upsample_add_bit_exact(lib):
    B, H, W, C = 2, 14, 20, 64
    ld = 3 * C                                  # inputs and outputs are slices of wider rows
    x = torch.randn(B, H, W, ld, device=dev).half()
    xs = x[..., C:2 * C]
    # maxpool 2x2
    out = nan16(B, H // 2, W // 2, ld)
    _lib.check(lib.vlfm_yolo_maxpool2(xs.data_ptr(), ld, out[..., 8:].data_ptr(), ld, B, H, W, C, st()), "maxpool2")
    ref = torch.nn.functional.max_pool2d(xs.permute(0, 3, 1, 2).float(), 2, 2).permute(0, 2, 3, 1).half()
    assert torch.equal(out[..., 8:8 + C], ref)
    # SPP pools 5 / 9 / 13
    out = nan16(B, H, W, 4 * C)
    _lib.check(lib.vlfm_yolo_spp_pools(xs.data_ptr(), ld, out[..., C:].data_ptr(), 4 * C, B, H, W, C, st()), "spp")
    for j, k in enumerate((5, 9, 13)):
        ref = torch.nn.functional.max_pool2d(xs.permute(0, 3, 1, 2).float(), k, 1, k // 2).permute(0, 2, 3, 1).half()
        assert torch.equal(out[..., (j + 1) * C:(j + 2) * C], ref)
    # nearest x2
    out = nan16(B, 2 * H, 2 * W, ld)
    _lib.check(lib.vlfm_yolo_upsample2(xs.data_ptr(), ld, out[..., 2 * C:].data_ptr(), ld, B, H, W, C, st()), "upsample2")
    ref = torch.nn.functional.interpolate(xs.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(out[..., 2 * C:], ref)
    # shortcut add
    y = torch.randn(B * H * W, C, device=dev).half()
    out = nan16(B * H * W, C)
    rows = x.reshape(B * H * W, ld)[:, C:2 * C]
    _lib.check(lib.vlfm_yolo_add(rows.data_ptr(), ld, y.data_ptr(), C, out.data_ptr(), C, B * H * W, C, st()), "add")
    assert torch.equal(out, rows + y)


def decode_ref(head, nc, anchors, stride, conf):
    """float64 decode of one level [B, ny, nx, na*no] -> per frame {row: (x1, y1, x2, y2, conf, cls)}"""
    B, ny, nx, _ = head.shape
    na = anchors.shape[0]
    v = head.double().view(B, ny, nx, na, nc + 5).permute(0, 3, 1, 2, 4).sigmoid()
    yv, xv = torch.meshgrid(torch.arange(ny, device=dev), torch.arange(nx, device=dev), indexing="ij")
    cx = (v[..., 0] * 2 - 0.5 + xv) * stride
    cy = (v[..., 1] * 2 - 0.5 + yv) * stride
    w = (v[..., 2] * 2) ** 2 * anchors[:, 0].view(1, na, 1, 1)
    h = (v[..., 3] * 2) ** 2 * anchors[:, 1].view(1, na, 1, 1)
    cls = v[..., 5:] * v[..., 4:5]
    c, j = cls.max(-1)
    ok = (v[..., 4] > conf) & (c > conf)
    out = []
    for b in range(B):
        idx = ok[b].flatten().nonzero().flatten()
        box = torch.stack((cx[b] - w[b] / 2, cy[b] - h[b] / 2, cx[b] + w[b] / 2, cy[b] + h[b] / 2, c[b], j[b].double()), -1).view(-1, 6)
        out.append({int(i): box[i] for i in idx})
    return out


def test_decode_against_float64(lib):
    B, ny, nx, na, nc = 3, 28, 40, 3, 80
    ld = 256
    head = torch.randn(B, ny, nx, ld, device=dev) * 2
    head[..., 4:na * 85:85] += 1.0
    head = head.half()
    anchors = torch.tensor([[96, 68], [86, 152], [180, 137]], dtype=torch.float32, device=dev)
    R = 5000
    cand = torch.full((B * R * 8,), float("nan"), device=dev)
    count = torch.zeros(B, dtype=torch.int32, device=dev)
    p = params(0.25)
    _lib.check(lib.vlfm_yolo_decode(head.data_ptr(), ld, B, ny, nx, na, nc, anchors.data_ptr(), 16.0, 100, R, p.data_ptr(), cand.data_ptr(),
                                    count.data_ptr(), st()), "decode")
    ref = decode_ref(head[..., :na * 85], nc, anchors.double(), 16.0, 0.25)
    c = cand.view(B, R, 8)
    for b in range(B):
        n = int(count[b])
        got = {int(c[b, i, 6]) - 100: c[b, i] for i in range(n)}
        near = {r for r, v in ref[b].items() if abs(float(v[4]) - 0.25) < 1e-5}
        assert set(got) ^ set(ref[b]) <= near
        for r in set(got) & set(ref[b]):
            assert torch.allclose(got[r][:5].double(), ref[b][r][:5], rtol=1e-5, atol=1e-3)
            assert int(got[r][5]) == int(ref[b][r][5])
    # class filter: only classes 3 and 62 survive
    count.zero_()
    _lib.check(lib.vlfm_yolo_decode(head.data_ptr(), ld, B, ny, nx, na, nc, anchors.data_ptr(), 16.0, 0, R, params(0.25, classes=[3, 62]).data_ptr(),
                                    cand.data_ptr(), count.data_ptr(), st()), "decode")
    for b in range(B):
        assert set(c[b, :int(count[b]), 5].long().tolist()) <= {3, 62}


def run_nms(lib, boxes, scores, classes, iou, agnostic, R=None):
    """Candidates of one or more frames [B, n, ...] through sort + NMS -> per-frame keep lists (candidate slots) and order."""
    B, n = scores.shape
    R = R or max(n, 1)
    cand = torch.zeros(B, R, 8, device=dev)
    cand[:, :n, :4], cand[:, :n, 4], cand[:, :n, 5] = boxes, scores, classes.float()
    cand[:, :n, 6] = torch.arange(n, device=dev).float()
    count = torch.full((B,), n, dtype=torch.int32, device=dev)
    order = torch.full((B * R,), -7, dtype=torch.int32, device=dev)
    keep = torch.full((B * MAX_DET,), -7, dtype=torch.int32, device=dev)
    nkeep = torch.full((B,), -7, dtype=torch.int32, device=dev)
    p = params(0.25, iou, agnostic)
    _lib.check(lib.vlfm_yolo_sort(cand.data_ptr(), count.data_ptr(), R, B, order.data_ptr(), st()), "sort")
    _lib.check(lib.vlfm_yolo_nms(cand.data_ptr(), order.data_ptr(), count.data_ptr(), R, B, p.data_ptr(), MAX_DET, keep.data_ptr(),
                                 nkeep.data_ptr(), st()), "nms")
    keep = keep.view(B, MAX_DET)
    return [keep[b, :int(nkeep[b])].tolist() for b in range(B)], order.view(B, R), cand


def random_boxes(n, seed, nclass=80):
    g = torch.Generator(device="cpu").manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * 600
    wh = 10 + torch.rand(n, 2, generator=g) * 120
    boxes = torch.cat((xy, xy + wh), 1)
    scores = 0.26 + 0.7 * (torch.randperm(n, generator=g).float() / n)       # distinct: no ties
    cls = torch.randint(0, nclass, (n,), generator=g)
    return boxes, scores, cls


@pytest.mark.parametrize("n,nclass,agnostic", [(50, 80, False), (2000, 80, False), (2000, 3, True), (17850, 80, False), (17850, 80, True),
                                               (4000, 1, True)])
def test_nms_keep_lists_equal_torchvision(lib, n, nclass, agnostic):
    boxes, scores, cls = random_boxes(n, n + nclass, nclass)
    assert scores.unique().numel() == n
    keeps, _, _ = run_nms(lib, boxes[None].to(dev), scores[None].to(dev), cls[None].to(dev), 0.45, agnostic)
    off = boxes + (0 if agnostic else 4096) * cls[:, None].float()
    ref = torchvision.ops.nms(off, scores, 0.45)[:MAX_DET].tolist()
    assert keeps[0] == ref
    if n >= 4000:
        assert len(ref) == MAX_DET                 # the cap is reached


def test_nms_ties_keep_candidate_order(lib):
    n = 64
    boxes = torch.tensor([[i * 50.0, 0, i * 50.0 + 40, 40] for i in range(n)])
    scores = torch.full((n,), 0.5)
    scores[10:20] = 0.7
    cls = torch.zeros(n, dtype=torch.long)
    keeps, order, _ = run_nms(lib, boxes[None].to(dev), scores[None].to(dev), cls[None].to(dev), 0.45, False)
    assert order[0, :n].tolist() == list(range(10, 20)) + list(range(10)) + list(range(20, n))
    assert keeps[0] == order[0, :n].tolist()


def test_nms_batch_and_repeat(lib):
    b1, s1, c1 = random_boxes(3000, 1)
    b2, s2, c2 = random_boxes(3000, 2)
    k1, _, _ = run_nms(lib, b1[None].to(dev), s1[None].to(dev), c1[None].to(dev), 0.5, False)
    kb, _, _ = run_nms(lib, torch.stack((b2, b1)).to(dev), torch.stack((s2, s1)).to(dev), torch.stack((c2, c1)).to(dev), 0.5, False)
    kb2, _, _ = run_nms(lib, torch.stack((b2, b1)).to(dev), torch.stack((s2, s1)).to(dev), torch.stack((c2, c1)).to(dev), 0.5, False)
    assert kb[1] == k1[0] and kb == kb2


@pytest.mark.parametrize("hw", [(480, 640), (720, 1280), (448, 640)])
def test_boxes_against_float64(lib, hw):
    H, W = hw
    B, R, n = 2, 1000, 350
    g = torch.Generator(device="cpu").manual_seed(H)
    cand = torch.zeros(B, R, 8)
    cand[:, :, :2] = torch.rand(B, R, 2, generator=g) * 700 - 30
    cand[:, :, 2:4] = cand[:, :, :2] + torch.rand(B, R, 2, generator=g) * 200
    cand[:, :, 4] = torch.rand(B, R, generator=g)
    cand[:, :, 5] = torch.randint(0, 80, (B, R), generator=g).float()
    keep = torch.stack([torch.randperm(R, generator=g)[:MAX_DET] for _ in range(B)]).int()
    nkeep = torch.tensor([MAX_DET, 17], dtype=torch.int32)
    cand, keep, nkeep = cand.to(dev), keep.to(dev), nkeep.to(dev)
    boxes = torch.full((B, MAX_DET, 4), float("nan"), device=dev)
    scores = torch.full((B, MAX_DET), float("nan"), device=dev)
    classes = torch.full((B, MAX_DET), -7, dtype=torch.int32, device=dev)
    counts = torch.full((B,), -7, dtype=torch.int32, device=dev)
    gain, px, py = scale_coords_params(H, W)
    _lib.check(lib.vlfm_yolo_boxes(cand.data_ptr(), keep.data_ptr(), nkeep.data_ptr(), R, B, MAX_DET, gain, px, py, H, W, boxes.data_ptr(),
                                   scores.data_ptr(), classes.data_ptr(), counts.data_ptr(), st()), "boxes")
    assert counts.tolist() == nkeep.tolist()
    for b in range(B):
        k = int(nkeep[b])
        sel = cand[b, keep[b, :k].long()].double()
        v = sel[:, :4].clone()
        v[:, [0, 2]] = ((v[:, [0, 2]] - px) / gain).clamp(0, W)
        v[:, [1, 3]] = ((v[:, [1, 3]] - py) / gain).clamp(0, H)
        raw = v.clone()
        v = v.round()
        v[:, [0, 2]] /= W
        v[:, [1, 3]] /= H
        frac = (raw - raw.floor() - 0.5).abs()
        ok = (frac > 1e-3)                       # a value within float32 rounding of .5 may round either way
        got = boxes[b, :k].double()
        assert torch.allclose(got[ok], v[ok], rtol=0, atol=1e-6)
        assert torch.equal(scores[b, :k], sel[:, 4].float()) and torch.equal(classes[b, :k], sel[:, 5].int())
        assert torch.all(boxes[b, k:] == 0) and torch.all(scores[b, k:] == 0) and torch.all(classes[b, k:] == -1)


def test_bad_arguments_are_refused(lib):
    x = torch.zeros(4096, dtype=F16, device=dev)
    f = torch.zeros(4096, device=dev)
    i = torch.zeros(4096, dtype=torch.int32, device=dev)
    p = params()
    P = x.data_ptr()
    cases = [
        lambda: lib.vlfm_yolo_preprocess(None, P, 1, 480, 640, 448, 640, i.data_ptr(), i.data_ptr(), f.data_ptr(), i.data_ptr(), i.data_ptr(), f.data_ptr(), None),
        lambda: lib.vlfm_yolo_preprocess(P, P, 1, 400, 640, 448, 640, i.data_ptr(), i.data_ptr(), f.data_ptr(), i.data_ptr(), i.data_ptr(), f.data_ptr(), None),
        lambda: lib.vlfm_yolo_maxpool2(P, 4, P, 8, 1, 4, 4, 8, None),
        lambda: lib.vlfm_yolo_spp_pools(P, 8, P, 16, 1, 4, 4, 8, None),
        lambda: lib.vlfm_yolo_upsample2(P, 8, P, 8, 1, 4, 4, 4, None),
        lambda: lib.vlfm_yolo_add(P, 8, P, 8, P, 8, 0, 8, None),
        lambda: lib.vlfm_yolo_decode(P, 200, 1, 2, 2, 3, 80, f.data_ptr(), 8.0, 0, 12, p.data_ptr(), f.data_ptr(), i.data_ptr(), None),
        lambda: lib.vlfm_yolo_decode(P, 256, 1, 2, 2, 3, 80, f.data_ptr(), 8.0, 1, 12, p.data_ptr(), f.data_ptr(), i.data_ptr(), None),
        lambda: lib.vlfm_yolo_sort(f.data_ptr(), i.data_ptr(), 0, 1, i.data_ptr(), None),
        lambda: lib.vlfm_yolo_nms(f.data_ptr(), i.data_ptr(), i.data_ptr(), 100000, 1, p.data_ptr(), 300, i.data_ptr(), i.data_ptr(), None),
        lambda: lib.vlfm_yolo_boxes(f.data_ptr(), i.data_ptr(), i.data_ptr(), 10, 1, 300, 0.0, 0.0, 0.0, 480, 640, f.data_ptr(), f.data_ptr(),
                                    i.data_ptr(), i.data_ptr(), None),
    ]
    n0 = _lib.launch_count()
    for k, c in enumerate(cases):
        assert c() == 1, f"case {k} accepted"
    assert _lib.launch_count() == n0
