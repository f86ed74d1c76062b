"""The YOLOv7 oracle (oracle/yolov7_oracle.py) against cv2, torchvision and hand-computed values (no GPU)."""
import numpy as np
import pytest
import torch
import torchvision

cv2 = pytest.importorskip("cv2")

from oracle import ref_import
from oracle import yolov7_oracle as O
from vlfm_b200.vlm import yolov7_config as cfg
from vlfm_b200.vlm.coco_classes import COCO_CLASSES
from vlfm_b200.vlm.yolov7_engine import check_frame


@pytest.mark.parametrize("hw", [(480, 640), (720, 1280), (449, 641), (600, 800), (1080, 1920), (500, 1000), (448, 640)])
def test_area_resize_matches_cv2(hw):
    img = np.random.default_rng(hw[0] * 7 + hw[1]).integers(0, 256, hw + (3,), dtype=np.uint8)
    ref = cv2.resize(img, (640, 448), interpolation=cv2.INTER_AREA)
    np.testing.assert_array_equal(O.area_resize(img), ref)
    assert torch.equal(O.preprocess(img, use_cv2=False), O.preprocess(img))


def test_frames_outside_the_restatement_raise():
    with pytest.raises(ValueError):
        check_frame(447, 640)
    with pytest.raises(ValueError):
        check_frame(480, 639)
    with pytest.raises(NotImplementedError):        # 2 x 2 integer downscale: cv2's resizeAreaFast rounds differently
        check_frame(896, 1280)
    check_frame(448, 640)


def tiny_layers():
    return cfg.synthetic_layers(3, table=cfg.e6e_table(div=8))


def test_unfused_and_fused_oracles_agree():
    layers = tiny_layers()
    x = O.preprocess(np.random.default_rng(0).integers(0, 256, (480, 640, 3), dtype=np.uint8))
    a, b = O.forward(layers, x, fused=True), O.forward(layers, x, fused=False)
    for u, v in zip(a, b):        # the fold runs in fp32, as yolov7's does
        assert (u - v).abs().max() <= 1e-4 * u.abs().max(), (u - v).abs().max()


def _greedy(boxes, scores, thr):
    order = sorted(range(len(scores)), key=lambda i: (-float(scores[i]), i))
    keep, removed = [], set()
    for i in order:
        if i in removed:
            continue
        keep.append(i)
        for j in order:
            if j not in removed and j != i and float(torchvision.ops.box_iou(boxes[i:i + 1], boxes[j:j + 1])[0, 0]) > thr:
                removed.add(j)
    return keep


@pytest.mark.parametrize("agnostic", [False, True])
def test_nms_restatement_is_class_offset_torchvision(agnostic):
    g = torch.Generator().manual_seed(5)
    n = 400
    xy = torch.rand(n, 2, generator=g) * 600
    pred = torch.zeros(1, n, 85, dtype=torch.float64)
    pred[0, :, :2] = xy
    pred[0, :, 2:4] = 20 + torch.rand(n, 2, generator=g) * 100
    pred[0, :, 4] = 0.3 + 0.7 * torch.rand(n, generator=g)
    pred[0, :, 5:] = torch.rand(n, 80, generator=g) * 0.5
    pred[0, torch.arange(n), 5 + torch.randint(0, 5, (n,), generator=g)] = 0.5 + 0.5 * torch.rand(n, generator=g, dtype=torch.float64)
    d = O.nms(pred, 0.25, 0.45, agnostic=agnostic)[0]
    # the same rows from a plain restatement: filter, score, class offset, torchvision's greedy order
    x = pred[0].clone()
    x = x[x[:, 4] > 0.25]
    x[:, 5:] *= x[:, 4:5]
    conf, j = x[:, 5:].max(1)
    box = torch.stack((x[:, 0] - x[:, 2] / 2, x[:, 1] - x[:, 3] / 2, x[:, 0] + x[:, 2] / 2, x[:, 1] + x[:, 3] / 2), 1).float()
    m = conf > 0.25
    box, conf, j = box[m], conf[m].float(), j[m]
    off = box + (0 if agnostic else 4096) * j[:, None].float()
    keep = torchvision.ops.nms(off, conf, 0.45)[:300]     # per-class NMS keeps more than max_det here
    assert torch.equal(d[:, 4], conf[keep]) and torch.equal(d[:, 5].long(), j[keep])
    small = _greedy(off[:60], conf[:60], 0.45)
    assert small == torchvision.ops.nms(off[:60], conf[:60], 0.45).tolist()


def test_scale_coords_hand_computed():
    # a 640 x 480 frame: gain = min(448 / 480, 640 / 640) = 14/15, pad = ((640 - 640 * 14/15) / 2, 0) = (21.33, 0)
    det = torch.tensor([[100.0, 56.0, 400.0, 392.0, 0.9, 0.0, 0.0]])
    b = O.scale_boxes(det, 480, 640)[0].tolist()
    # x: (100 - 21.33) * 15/14 = 84.29 -> 84;  (400 - 21.33) * 15/14 = 405.71 -> 406 (stretched about the centre)
    # y: 56 * 15/14 = 60, 392 * 15/14 = 420 (exact)
    assert b == [84 / 640, 60 / 480, 406 / 640, 420 / 480]
    clip = O.scale_boxes(torch.tensor([[0.0, -5.0, 640.0, 460.0, 0.5, 1.0, 0.0]]), 480, 640)[0].tolist()
    assert clip == [0.0, 0.0, 1.0, 1.0]


def test_coco_classes():
    assert len(COCO_CLASSES) == 80 and len(set(COCO_CLASSES)) == 80
    assert [COCO_CLASSES.index(n) for n in ("chair", "bed", "potted plant", "toilet", "tv", "couch")] == [56, 59, 58, 61, 62, 57]
    if not ref_import.available():
        pytest.skip("reference checkout not configured (VLFM_REFERENCE)")
    ref_import._ensure_path()
    from vlfm.vlm.coco_classes import COCO_CLASSES as REF  # type: ignore

    assert list(REF) == COCO_CLASSES


def test_e6e_table_size():
    params, gflop = cfg.cost(448, 640)
    assert params == 151_687_420                   # yolov7 publishes 151.7 M for E6E
    assert 150 < gflop < 157
