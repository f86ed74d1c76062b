"""YOLOv7-E6E end to end on the GPU (synthetic full-size weights) against the float64 oracle (oracle/yolov7_oracle.py).

GPU_BARS were fixed from an oracle-only run before the first GPU run: over the test frames (uniform pixel noise at 640 x 480 and
1280 x 720, seeds 1 and 2), the float64 oracle with the fused weights and every stored activation rounded to fp16 differed from
the pure float64 oracle by at most 0.0081 / 0.0045 / 0.0047 / 0.0200 on the four levels' head outputs (head RMS ~5, 45-52 rows
over the objectness threshold, 29-39 kept).  The head bar is 2x the largest; the conf and IoU bars follow from it (sigmoid slopes
are at most 1/4).  Boxes are paired within 3 px plus 3 % of the box size: wh = (2 sigmoid)^2 * anchor moves up to 2 anchors per
unit of logit, and the P6 anchors are up to 925 px.

The 448 x 640 frame (the identity resize) is itself an area-downscaled noise frame: random weights amplify unfiltered full-band
pixel noise into fp16 overflow in the P6 head, which no camera frame carries.
"""
import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import yolov7_oracle as O
from vlfm_b200.vlm.detections import ObjectDetections

pytestmark = pytest.mark.gpu
GPU_BARS = {"head": 0.04, "conf": 0.01, "iou": 0.01, "box_px": 3.0}
FRAMES = [(480, 640), (720, 1280), (448, 640)]


@pytest.fixture(scope="module")
def model():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from vlfm_b200.vlm.yolov7 import YOLOv7

    return YOLOv7(synthetic=True, seed=0)


@pytest.fixture(scope="module")
def layers(model):
    return model.engine.layers


def frame(hw, seed=1):
    if hw == (448, 640):
        noise = np.random.default_rng(seed).integers(0, 256, (480, 640, 3), dtype=np.uint8)
        return cv2.resize(noise, (640, 448), interpolation=cv2.INTER_AREA)
    return np.random.default_rng(seed).integers(0, 256, hw + (3,), dtype=np.uint8)


def engine_heads(model, B):
    e = model.engine
    bufs = e._bufs[B]
    out = []
    for k, (_, h, w, _) in enumerate(e.levels):
        t = bufs["head"][k].view(B, h, w, e.head_ld)[..., :e.na * e.no]
        out.append(t.permute(0, 3, 1, 2).double())
    return out


@pytest.fixture(scope="module")
def oracle_runs(layers):
    res = {}
    for hw in FRAMES:
        img = frame(hw)
        heads = O.forward(layers, O.preprocess(img).cuda())
        res[hw] = (img, heads)
    return res


@pytest.mark.parametrize("hw", FRAMES)
def test_head_within_bars_of_float64(model, oracle_runs, hw):
    img, ref = oracle_runs[hw]
    model.engine.run(torch.from_numpy(img[None]).cuda())
    for g, r in zip(engine_heads(model, 1), ref):
        assert (g - r).abs().max().item() <= GPU_BARS["head"], (g - r).abs().max().item()


@pytest.mark.parametrize("hw", FRAMES)
@pytest.mark.parametrize("agnostic", [False, True])
def test_postprocess_on_oracle_heads_equals_oracle(model, layers, oracle_runs, hw, agnostic):
    img, ref = oracle_runs[hw]
    H, W = hw
    e = model.engine
    e.run(torch.from_numpy(img[None]).cuda())          # allocates B = 1 buffers and the frame's tables
    e.set_params(0.25, 0.45, None, agnostic)
    bufs = e._bufs[1]
    h16 = []
    with torch.inference_mode():                       # the engine's buffers are inference tensors
        for k, (t, (_, h, w, _)) in enumerate(zip(ref, e.levels)):
            v = t.half()
            h16.append(v.double())
            bufs["head"][k].view(1, h, w, e.head_ld)[..., :e.na * e.no].copy_(v.permute(0, 2, 3, 1))
        e.postprocess(1, H, W, bufs)
    d = O.nms(O.decode([t.float() for t in h16], layers), agnostic=agnostic)[0]
    n = int(bufs["counts"][0])
    assert n == d.shape[0] and n > 0
    assert bufs["classes"][0, :n].tolist() == d[:, 5].long().tolist()
    assert torch.allclose(bufs["scores"][0, :n], d[:, 4].to(bufs["scores"].device), rtol=1e-5, atol=1e-6)
    ob = O.scale_boxes(d, H, W).to(bufs["boxes"].device)
    assert (bufs["boxes"][0, :n].double() - ob).abs().max() <= 1.01 / min(H, W)      # a .5 may round either way
    e.set_params(0.25, 0.45, None, False)


def pair(det_g, det_o, hw):
    """Pair GPU rows with oracle rows by class and box; oracle rows near conf_thres may be missing."""
    H, W = hw
    unmatched = []
    used = set()
    for i in range(det_o[0].shape[0]):
        c, s, b = int(det_o[0][i, 5]), float(det_o[0][i, 4]), det_o[1][i]
        size = torch.stack((b[2] - b[0], b[3] - b[1])).repeat(2)
        tol = torch.tensor([GPU_BARS["box_px"] / W, GPU_BARS["box_px"] / H] * 2, dtype=torch.float64) + 0.03 * size
        hit = [j for j in range(len(det_g[2])) if j not in used and det_g[2][j] == c and torch.all((det_g[0][j].double() - b).abs() <= tol)
               and abs(float(det_g[1][j]) - s) <= GPU_BARS["conf"]]
        if hit:
            used.add(hit[0])
        else:
            unmatched.append(i)
    return unmatched, [j for j in range(len(det_g[2])) if j not in used]


@pytest.mark.parametrize("hw", FRAMES)
def test_end_to_end_detections_pair_with_oracle(model, layers, oracle_runs, hw, capsys):
    img, ref = oracle_runs[hw]
    boxes, scores, classes, counts = model.predict_device(torch.from_numpy(img[None]).cuda())
    n = int(counts[0])
    g = (boxes[0, :n].cpu(), scores[0, :n].cpu(), classes[0, :n].cpu().tolist())
    d = O.nms(O.decode(ref, layers))[0].cpu()
    o = (d, O.scale_boxes(d, *hw))
    miss_o, miss_g = pair(g, o, hw)
    # excluded: rows whose conf is within the bar of conf_thres, or that overlap a kept box of the same class within the bar of
    # iou_thres (their suppression may go either way)
    def borderline(conf, box, cls, others):
        if abs(conf - 0.25) <= GPU_BARS["conf"]:
            return True
        import torchvision
        for ob, oc in others:
            if oc == cls and abs(float(torchvision.ops.box_iou(box[None], ob[None])[0, 0]) - 0.45) <= GPU_BARS["iou"]:
                return True
        return False
    allrows = O.nms(O.decode(ref, layers), iou_thres=1.0)[0].cpu()     # every candidate, unsuppressed
    others = [(allrows[k, :4].double(), int(allrows[k, 5])) for k in range(allrows.shape[0])]
    bad = [i for i in miss_o if not borderline(float(d[i, 4]), d[i, :4].double(), int(d[i, 5]), others)]
    assert not bad, f"oracle rows {bad} have no GPU match"
    assert len(miss_g) <= len(miss_o) + 2
    with capsys.disabled():
        print(f"\n[yolov7 {hw[1]}x{hw[0]}] oracle rows {d.shape[0]}, GPU rows {n}, excluded {len(miss_o)} oracle / {len(miss_g)} GPU")
    assert n > 0


def test_predict_device_batches_match_single_frames(model):
    imgs = [frame((480, 640), s) for s in range(8)]
    single = []
    for im in imgs:
        b, s, c, n = model.predict_device(torch.from_numpy(im[None]).cuda())
        single.append((b[0], s[0], c[0], int(n[0])))
    for B in (1, 2, 5, 8):
        perm = np.random.default_rng(B).permutation(8)[:B]
        b, s, c, n = model.predict_device(torch.from_numpy(np.stack([imgs[p] for p in perm])).cuda())
        for k, p in enumerate(perm):
            assert int(n[k]) == single[p][3]
            m = single[p][3]
            assert torch.equal(c[k, :m], single[p][2][:m])
            assert torch.allclose(s[k, :m], single[p][1][:m], atol=GPU_BARS["conf"])
            assert torch.allclose(b[k, :m], single[p][0][:m], atol=GPU_BARS["box_px"] / 640)


def test_graph_replay_equals_eager_and_repeats(model):
    img = torch.from_numpy(np.stack([frame((720, 1280), 3), frame((720, 1280), 4)])).cuda()
    e = model.engine
    e.use_graph = False
    try:
        eager = [t.clone() for t in e.run(img)]
    finally:
        e.use_graph = True
    heads_eager = [t.clone() for t in e._bufs[2]["head"]]
    for _ in range(3):
        got = e.run(img)
        assert (2, 720, 1280) in e.graphs.captured
        for a, b in zip(got, eager):
            assert torch.equal(a.view(torch.int32) if a.is_floating_point() else a, b.view(torch.int32) if b.is_floating_point() else b)
        for a, b in zip(e._bufs[2]["head"], heads_eager):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_predict_and_client_surface(model, monkeypatch):
    from vlfm_b200.vlm import yolov7 as Y

    img = frame((480, 640))
    det = model.predict(img)
    assert isinstance(det, ObjectDetections) and det.num_detections > 0
    assert det.boxes.dtype == torch.float32 and det.boxes.device.type == "cpu" and det.logits.dtype == torch.float32
    assert torch.all((det.boxes >= 0) & (det.boxes <= 1))
    b, s, c, n = model.predict_device(torch.from_numpy(img[None]).cuda())
    assert torch.equal(det.boxes, b[0, :int(n[0])].cpu())
    client = Y.YOLOv7Client(port=12184, model=model)
    det2 = client.predict(img)
    assert det2.phrases == det.phrases and torch.equal(det2.boxes, det.boxes)
    # the way BaseObjectNavPolicy._get_object_detections uses them
    target = det.phrases[0]
    det2.filter_by_class([target])
    assert set(det2.phrases) == {target}
    det2.filter_by_conf(0.3)
    assert torch.all(det2.logits >= 0.3)
    # thresholds and classes change without re-capturing
    assert (1, 480, 640) in model.engine.graphs.captured
    ngraph = len(model.engine.graphs.captured)
    strict = model.predict(img, conf_thres=0.6)
    assert strict.num_detections <= det.num_detections and torch.all(strict.logits > 0.6)
    only = model.predict(img, classes=[56, 57])
    assert set(only.phrases) <= {"chair", "couch"}
    assert len(model.engine.graphs.captured) == ngraph
    monkeypatch.setenv("VLFM_SYNTHETIC_WEIGHTS", "1")
    monkeypatch.setattr(Y, "_SHARED", {"default": model})
    assert Y.YOLOv7Client().model is model


def test_argument_errors(model, monkeypatch):
    from vlfm_b200.vlm.yolov7 import YOLOv7

    with pytest.raises(ValueError):
        model.predict(frame((400, 640)))
    with pytest.raises(ValueError):
        model.predict(np.zeros((480, 640), np.uint8))
    with pytest.raises(NotImplementedError):
        model.predict(frame((896, 1280)))
    with pytest.raises(TypeError):
        model.predict(frame((480, 640)), classes=["chair"])
    with pytest.raises(NotImplementedError):
        YOLOv7(synthetic=True, image_size=1280)
    with pytest.raises(NotImplementedError):
        YOLOv7(synthetic=True, half_precision=False)
    monkeypatch.delenv("VLFM_YOLOV7_WEIGHTS", raising=False)
    with pytest.raises(FileNotFoundError):
        YOLOv7()
