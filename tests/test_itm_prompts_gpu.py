"""Scoring one frame against many prompts: the multi-prompt ITC head, BLIP2ITM.cosine_many / cosine_device_many and the
per-frame feature cache behind BLIP2ITM.cosine.

Every multi-prompt score must be bitwise equal to a single-prompt score from a fresh forward, and within the existing
tolerances of the fp32 oracle."""
import numpy as np
import pytest
import torch

from oracle import blip2_oracle
from vlfm_b200 import _lib
from vlfm_b200.utils.synthetic import make_rgb, trajectory
from vlfm_b200.vlm.blip2_config import SMALL, TINY, Blip2Dims, random_state_dict

pytestmark = pytest.mark.gpu

# short prompts: TINY's text branch holds at most queries * max_batch tokens
PROMPTS33 = [f"thing {k} ahead" for k in range(33)]
FULL_PROMPTS = ["Seems like there is a chair ahead.", "Seems like there is a potted plant ahead.", "Seems like there is a toilet ahead."]


def _model(dims, seed=3, max_batch=3):
    from vlfm_b200.vlm.blip2itm import BLIP2ITM

    return BLIP2ITM(state_dict=random_state_dict(dims, seed), dims=dims, max_batch=max_batch)


def _oracle_text(orc, dims, prompts):
    from vlfm_b200.vlm.blip2itm import HashTokenizer, pre_caption

    tok = HashTokenizer(dims.vocab)
    return [orc.text_feature(tok(pre_caption(p))) for p in prompts]


@pytest.mark.parametrize("dims", [TINY, SMALL], ids=["tiny", "small"])
def test_cosine_many_equals_single_prompt_and_oracle(dims):
    sd = random_state_dict(dims, 3)
    orc = blip2_oracle.Blip2Oracle(dims, sd)
    from vlfm_b200.vlm.blip2itm import BLIP2ITM

    m = BLIP2ITM(state_dict=sd, dims=dims, max_batch=3)
    txt = _oracle_text(orc, dims, PROMPTS33)
    rng = np.random.default_rng(1)
    for P in (1, 2, 3, 8, 33):
        img = make_rgb(rng, 480, 640)
        feat = orc.image_features(img)
        many = m.cosine_many(img, PROMPTS33[:P])
        assert len(many) == P and all(isinstance(v, float) for v in many)
        gen = m.engine.generation
        cached = [m.cosine(img, p) for p in PROMPTS33[:P]]   # the same frame object: the head alone runs
        assert m.engine.generation == gen
        single = [m.cosine(img.copy(), p) for p in PROMPTS33[:P]]
        assert many == single, (P, np.max(np.abs(np.array(many) - np.array(single))))
        assert cached == single
        for p in range(P):
            assert abs(many[p] - orc.cosine_from(feat, txt[p])) <= 2e-3


def test_cosine_device_many_equals_cosine_device():
    dims = SMALL
    sd = random_state_dict(dims, 3)
    orc = blip2_oracle.Blip2Oracle(dims, sd)
    from vlfm_b200.vlm.blip2itm import BLIP2ITM

    m = BLIP2ITM(state_dict=sd, dims=dims, max_batch=3)
    prompts = PROMPTS33[:5]
    txt = _oracle_text(orc, dims, prompts)
    rng = np.random.default_rng(4)
    imgs = np.stack([make_rgb(rng, 480, 640) for _ in range(3)])
    dev = torch.from_numpy(imgs).cuda()
    many = m.cosine_device_many(dev, prompts)
    assert many.shape == (3, 5) and many.dtype == torch.float32 and many.is_cuda
    many = many.cpu().numpy()
    for p, prompt in enumerate(prompts):
        one = m.cosine_device(dev, prompt).cpu().numpy()
        assert np.array_equal(many[:, p], one), (p, many[:, p], one)
    for b in range(3):
        feat = orc.image_features(imgs[b])
        for p in range(5):
            assert abs(many[b, p] - orc.cosine_from(feat, txt[p])) <= 2e-3
    # a sub-batch after a larger one, and the result feeds ValueMapBatch.update as float64
    sub = m.cosine_device_many(dev[:2], prompts[:2]).double()
    assert sub.shape == (2, 2) and sub.is_contiguous()


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "page_locked"])
def test_frame_cache(pinned):
    dims = SMALL
    m, ref = _model(dims), _model(dims)
    rng = np.random.default_rng(5)
    a, b = make_rgb(rng, 480, 640), make_rgb(rng, 480, 640)
    if pinned:
        frame = torch.empty((480, 640, 3), dtype=torch.uint8).pin_memory().numpy()
        assert torch.from_numpy(frame).is_pinned()
    else:
        frame = np.empty((480, 640, 3), dtype=np.uint8)
    frame[...] = a
    p0, p1, p2 = PROMPTS33[:3]
    for p in (p0, p1, p2):   # encode every prompt up front: encode_text also invalidates the cache
        m._text(p)

    def fresh(img, p):
        return ref.cosine(img.copy(), p)

    v0 = m.cosine(frame, p0)
    assert v0 == fresh(a, p0)
    gen = m.engine.generation
    # same object, other prompts: the head alone runs
    assert m.cosine(frame, p1) == fresh(a, p1)
    assert m.cosine(frame, p0) == v0
    assert m.cosine_many(frame, [p2, p0]) == [fresh(a, p2), v0]
    assert m.engine.generation == gen
    # the same buffer refilled in place with another frame: recomputed
    frame[...] = b
    assert m.cosine(frame, p1) == fresh(b, p1)
    assert m.engine.generation == gen + 1
    assert m.cosine(frame, p0) == fresh(b, p0)
    assert m.engine.generation == gen + 1
    # another forward in between (a device batch): recomputed
    m.cosine_device(torch.from_numpy(np.stack([a, a])).cuda(), p2)
    assert m.cosine(frame, p0) == fresh(b, p0)
    # a new prompt is encoded in between: still correct
    assert m.cosine(frame, "a brand new prompt") == fresh(b, "a brand new prompt")
    assert m.cosine(frame, p1) == fresh(b, p1)
    # a one-byte change is seen
    gen = m.engine.generation
    frame[100, 200, 1] ^= 1
    assert m.cosine(frame, p1) == fresh(frame, p1)
    assert m.engine.generation == gen + 1
    # the same object reshaped in place (same bytes, another frame shape): recomputed
    gen = m.engine.generation
    frame.shape = (640, 480, 3)
    assert m.cosine(frame, p2) == fresh(frame, p2)
    assert m.engine.generation == gen + 1
    frame.shape = (480, 640, 3)
    assert m.cosine(frame, p2) == fresh(frame, p2)
    # a different object with equal bytes always runs the forward
    gen = m.engine.generation
    m.cosine(frame.copy(), p2)
    assert m.engine.generation == gen + 1


def test_full_size_vitg_cosine_many_vs_oracle():
    """ViT-g/14 + 12-layer Q-Former at full size: cosine_many within 1e-4 of the fp32 oracle for 8 frames x 3 prompts, and the
    forward is bitwise reproducible over distinct frame objects (each one runs the forward)."""
    from vlfm_b200.vlm.blip2itm import BLIP2ITM

    dims = Blip2Dims()
    sd = random_state_dict(dims, 0)
    orc = blip2_oracle.Blip2Oracle(dims, sd)
    m = BLIP2ITM(state_dict=sd, dims=dims, max_batch=1)
    txt = _oracle_text(orc, dims, FULL_PROMPTS)
    rng = np.random.default_rng(2)
    errs, spread = [], 0.0
    for k in range(8):
        img = make_rgb(rng, 480, 640)
        feat = orc.image_features(img)
        got = m.cosine_many(img, FULL_PROMPTS)
        errs += [abs(g - orc.cosine_from(feat, t)) for g, t in zip(got, txt)]
        if k < 3:
            gen = m.engine.generation
            rep = [m.cosine(img.copy(), FULL_PROMPTS[0]) for _ in range(6)]
            assert m.engine.generation == gen + 6
            spread = max(spread, max(rep) - min(rep))
            assert rep[0] == got[0]
    errs = np.array(errs)
    print(f"{len(errs)} cosines, max |err| {errs.max():.3e}, mean {errs.mean():.3e}, run-to-run spread {spread:.3e}")
    assert errs.max() <= 1e-4
    assert spread == 0.0


def test_value_map_fed_from_cosine_many():
    """ValueMap(value_channels=2) fed from cosine_many is bitwise the map fed from one cosine per prompt on frame copies."""
    from vlfm_b200.mapping.value_map import ValueMap

    m, ref = _model(SMALL), _model(SMALL)
    prompts = ["Seems like there is a chair ahead.", "There is a lot of area to explore ahead."]
    fov = float(np.deg2rad(79.0))
    vm_many = ValueMap(2, size=400, use_max_confidence=False, device="cuda:0")
    vm_one = ValueMap(2, size=400, use_max_confidence=False, device="cuda:0")
    frames = trajectory(0, 16, h=120, w=160, bound_m=3.0, with_rgb=True)
    for f in frames:
        a = np.array(m.cosine_many(f.rgb, prompts))
        b = np.array([ref.cosine(f.rgb.copy(), p) for p in prompts])
        assert np.array_equal(a, b)
        vm_many.update_map(a, f.depth, f.tf, 0.5, 5.0, fov)
        vm_one.update_map(b, f.depth, f.tf, 0.5, 5.0, fov)
    assert np.array_equal(vm_many._map, vm_one._map)
    assert np.array_equal(vm_many._value_map, vm_one._value_map)
    assert vm_many._value_map.max() > 0
    waypoints = np.array([f.xy for f in frames[::3]])
    reduce_fn = lambda vals: [max(v) for v in vals]   # noqa: E731
    w1, v1 = vm_many.sort_waypoints(waypoints, 0.5, reduce_fn=reduce_fn)
    w2, v2 = vm_one.sort_waypoints(waypoints, 0.5, reduce_fn=reduce_fn)
    assert np.array_equal(w1, w2) and v1 == v2


def test_argument_errors():
    m = _model(TINY, max_batch=1)
    img = make_rgb(np.random.default_rng(0), 120, 160)
    with pytest.raises(ValueError):
        m.cosine_many(img, [])
    with pytest.raises(ValueError):
        m.cosine_device_many(torch.from_numpy(img[None]).cuda(), [])
    lib = _lib.load()
    e = m.engine
    text = torch.zeros(4, TINY.proj, dtype=torch.float32, device="cuda")
    out = torch.zeros(1, 4, dtype=torch.float32, device="cuda")
    q, t, o = e.q_proj.data_ptr(), text.data_ptr(), out.data_ptr()
    s = _lib.stream_ptr()
    assert lib.vlfm_itc_head_multi(q, t, o, 1, 0, TINY.queries, TINY.proj, 4, s) == 1      # VLFM_E_INVALID: P = 0
    assert lib.vlfm_itc_head_multi(q, t, o, 1, 4, TINY.queries, TINY.proj, 3, s) == 1      # ldo < P
    assert lib.vlfm_itc_head_multi(q, t, o, 0, 4, TINY.queries, TINY.proj, 4, s) == 1      # B = 0
    assert lib.vlfm_itc_head_multi(None, t, o, 1, 4, TINY.queries, TINY.proj, 4, s) == 1   # NULL
    with pytest.raises(_lib.VlfmError):
        _lib.check(lib.vlfm_itc_head_multi(q, t, o, 1, 0, TINY.queries, TINY.proj, 4, s), "vlfm_itc_head_multi")
    with pytest.raises(_lib.VlfmError):
        e.head(text[:0], 1)
    assert lib.vlfm_itc_head_multi(q, t, o, 1, 4, TINY.queries, TINY.proj, 4, s) == 0
    torch.cuda.synchronize()
