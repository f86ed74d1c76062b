"""Every launch plan of the wgmma GEMM (csrc/gemm_wgmma.cu), bit for bit against float64.

The operands are small multiples of powers of two: A = k / 4, W = k / 8 (|k| <= 3, fp16), bias = k / 32 (|bias| <= 20) and the
residual k / 32 (|r| <= 64).  Every product is a multiple of 2^-5, and for K <= 6152 every partial sum, bias and residual
included, stays below 2^11: at most 16 significant bits.  fp32 holds each of them exactly in any order of summation (tensor-core
K steps, the CUDA-core tail rows, split-K with red.add, stream-K slabs, the cluster reduction in shared memory), so the float64
product is the exact value and the checks are bitwise: fp32 outputs equal it, fp16 outputs equal its round-to-nearest-even, and
GELU / SiLU outputs lie within one fp16 ulp of the float64 activation of it.

Each case runs in two layouts.  "contiguous": A [M, K], W [N, K], the output [M, N] in rows of ceil8(N).  "embedded", as the
engines use it: A a column window of a wider NaN buffer (NaN past K inside lda, a NaN row past M that the call is told to skip
with ``rows``), W [:, :K] of a NaN buffer [N + 1, K + 8], the output a window at row 1, column 8 of a buffer with spare rows and
columns.  Output buffers start as payload NaN (finite values for the residual epilogue): every element outside the window must
keep its bits, every element inside must be written, and no NaN may reach the result (nothing is read past K or M).

Plans are reached on purpose: VLFM_GEMM_FORCE="bn:s" (read on every call) pins the grid tile width and, for the residual
epilogue, the red.add split count; the default plan runs the sub-wave tile width choice and the cost model; VLFM_GEMM_CSPLIT=2
with VLFM_EPI_CLUSTER_SPLIT runs the 256-row cluster split at 257 / 258 rows; vlfm_gemm_f16_resid_ln runs stream-K and the
deterministic uniform split from workspace sizes derived from the SM count; the x2 GEMMs run with lo = 0 (exact) and lo != 0.
"""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN16 = 0x7E5A            # fp16 NaN with a payload: an untouched element still holds exactly this bit pattern
NAN32 = 0x7FC05A5A        # the same for fp32
FLAG = 256                # VLFM_EPI_CLUSTER_SPLIT
EPS = 1e-6


@pytest.fixture(autouse=True)
def plan_env(monkeypatch):
    """No plan override unless a case sets one."""
    monkeypatch.delenv("VLFM_GEMM_FORCE", raising=False)
    monkeypatch.delenv("VLFM_GEMM_CSPLIT", raising=False)
    return monkeypatch


def _lib():
    from vlfm_b200 import _lib

    return _lib, _lib.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ceil8(n):
    return (n + 7) // 8 * 8


# ---------------------------------------------------------------------------------------------------------------- inputs ----
def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _grid(shape, k, den, g, dtype):
    """Integers in [-k, k] over den, exactly representable in fp16 / fp32."""
    return (torch.randint(-k, k + 1, shape, generator=g).to(torch.float64) / den).to(dtype).cuda()


def _operands(M, N, K, seed):
    g = _gen(seed)
    a = _grid((M, K), 3, 4, g, torch.float16)
    w = _grid((N, K), 3, 8, g, torch.float16)
    bias = _grid((N,), 640, 32, g, torch.float32)
    return a, w, bias, g


def _sentinel(shape, dtype, g=None):
    """Payload-NaN buffer, or (g given) a buffer of finite residual-grid values."""
    if g is not None:
        return _grid(shape, 2048, 32, g, dtype)
    if dtype == torch.float16:
        return torch.full(shape, NAN16, dtype=torch.int16, device="cuda").view(torch.float16)
    return torch.full(shape, NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _nan_buffer(shape, window, src):
    """A NaN fp16 buffer with `src` written into buf[window]."""
    buf = torch.full(shape, float("nan"), dtype=src.dtype, device="cuda")
    buf[window] = src
    return buf


def _outside_kept(after, before, window, what):
    keep = torch.ones(after.shape, dtype=torch.bool, device=after.device)
    keep[window] = False
    bad = (_bits(after) != _bits(before)) & keep
    n = int(bad.sum())
    assert n == 0, f"{what}: {n} elements outside the output window were written, first at {bad.nonzero()[:4].tolist()}"


# ---------------------------------------------------------------------------------------------------------------- checks ----
def _assert_equal(got, exp, what):
    bad = ~(got == exp)          # NaN compares unequal: an unwritten or poisoned element fails here
    n = int(bad.sum())
    if n:
        i = bad.nonzero()[:4].tolist()
        pairs = [(got[tuple(j)].item(), exp[tuple(j)].item()) for j in i]
        raise AssertionError(f"{what}: {n} of {got.numel()} elements differ, first at {i}: (got, exact) {pairs}")


def _ulp16(x):
    """The fp16 ulp at |x| (float64 in), 2^-24 in the subnormal range."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -24)))
    return torch.exp2(e.clamp_min(-14.0) - 10.0)


def _assert_within_ulp16(got, ref, what, slack=0.0):
    g = got.double()
    err = (g - ref).abs()
    bad = ~(err <= _ulp16(torch.maximum(g.abs(), ref.abs())) + slack)
    n = int(bad.sum())
    if n:
        i = bad.nonzero()[:4].tolist()
        pairs = [(g[tuple(j)].item(), ref[tuple(j)].item()) for j in i]
        raise AssertionError(f"{what}: {n} elements further than one fp16 ulp, first at {i}: (got, float64) {pairs}")


def _activation(pre, epi):
    if epi == 1:
        return torch.nn.functional.gelu(pre)
    if epi == 7:
        return torch.nn.functional.silu(pre)
    if epi == 4:
        return torch.relu(pre)
    return pre


def _check_epilogue(got, pre, epi, what):
    """got: the output window; pre: the exact pre-activation (float64, residual included)."""
    if epi in (2, 3):
        _assert_equal(got, pre.float(), what)
    elif epi in (0, 4):
        _assert_equal(got, _activation(pre, epi).half(), what)
    elif epi == 7:
        _assert_within_ulp16(got, _activation(pre, epi), what)
    else:
        # GELU below x = -2 is x / 2 times 1 + erff(x / sqrt 2), a cancellation: erff's result near -1 is off by a few multiples
        # of 2^-24 (its ulp there), so the fp32 value carries up to about |x| 2^-22 of absolute error, several fp16 ulps where
        # GELU is small (-1.4e-6 at x = -5)
        _assert_within_ulp16(got, _activation(pre, epi), what, slack=pre.abs() * 2.0 ** -22)


# ----------------------------------------------------------------------------------------------------------------- cases ----
# Edge values: M = 1, 31, 32, 33 (32-row A box), 64, 65 (64-row box), 127, 128, 129 / 130 (tail rows), 131 (no tail), 257, 258,
# 300, 386 (tail at three row tiles), 8194 (many waves with a tail); N = 1, 8, 255, 520, 1000, 1408, 4224; K = 8, 56, 64, 72, 1000,
# 6144 (the last K with tail rows), 6152 (tail rows off: M = 258 then runs three row tiles, the last one partial).
SHAPES = [(1, 1000, 1000), (31, 255, 56), (32, 4224, 64), (33, 1, 72), (64, 1408, 8), (65, 520, 6144), (127, 8, 1000),
          (128, 255, 6152), (129, 1000, 72), (130, 520, 6144), (131, 1408, 56), (257, 4224, 6144), (258, 255, 6152),
          (300, 8, 8), (386, 1000, 64), (8194, 520, 1000)]
FORCE_EPIS = (0, 1, 3, 4, 7)
# every grid tile width meets every shape; the epilogue rotates so that each (width, epilogue) pair sees three or four shapes
FORCE_CASES = [(M, N, K, FORCE_EPIS[(i + b) % 5], f"{bn}:1", (i + 2 * b) % 4 != 3)
               for b, bn in enumerate((128, 96, 64, 32)) for i, (M, N, K) in enumerate(SHAPES)]
# the residual epilogue of vlfm_gemm_f16 splits K with red.add; the split count is capped at the K-block count (K = 72: 2)
SPLIT_SHAPES = [(1, 520, 6144), (33, 255, 1000), (130, 1000, 6144), (257, 1408, 1000), (300, 8, 72), (8194, 255, 1000),
                (131, 4224, 6152)]
SPLIT_CASES = [(*SPLIT_SHAPES[(3 * j + k) % 7], 2, plan, k != 1)
               for j, plan in enumerate(("128:1", "128:2", "128:3", "128:8", "32:8")) for k in range(3)]
# no override: below one wave the tile width of the busiest SM's columns, above it the cost model (8194 rows: 65 row tiles)
DEFAULT_EPIS = (0, 1, 2, 3, 4, 7)
DEFAULT_CASES = [(M, N, K, DEFAULT_EPIS[i % 6], "default", i % 5 != 4) for i, (M, N, K) in enumerate(SHAPES + [(8194, 4224, 72)])]
# the cluster split (VLFM_GEMM_CSPLIT=2): tile width and cluster size come from the device's cluster occupancy.  On an H100 SXM
# (132 SMs) the (BN, s) are, in this order: (96, 8), (96, 1), (128, 1) (BN 96 would need 171 clusters), (64, 8), (64, 1)
CS_SHAPES = [(257, 1000, 1000), (258, 9216, 64), (257, 16384, 64), (258, 520, 6144), (257, 255, 8)]
CS_CASES = [(M, N, K, DEFAULT_EPIS[(3 * i + k) % 6], "csplit", k != 2) for i, (M, N, K) in enumerate(CS_SHAPES) for k in range(3)]
CASES = FORCE_CASES + SPLIT_CASES + DEFAULT_CASES + CS_CASES


def _case_id(c):
    M, N, K, epi, plan, bias = c
    return f"{M}x{N}x{K}-e{epi}-{plan}" + ("" if bias else "-nobias")


def test_case_list_covers_every_edge():
    assert len(CASES) == len({_case_id(c) for c in CASES}) and 80 <= len(CASES) <= 120
    for plan in ("128:1", "96:1", "64:1", "32:1"):
        sel = [c for c in FORCE_CASES if c[4] == plan]
        assert {c[0] for c in sel} == {c[0] for c in SHAPES} and {c[3] for c in sel} == set(FORCE_EPIS)
    for M in (1, 31, 32, 33, 64, 65, 127, 128, 129, 130, 131, 257, 258, 300, 386, 8194):
        assert any(c[0] == M for c in SHAPES)
    for N in (1, 8, 255, 520, 1000, 1408, 4224):
        assert any(c[1] == N for c in SHAPES) and any(c[1] == N for c in DEFAULT_CASES)
    for K in (8, 56, 64, 72, 1000, 6144, 6152):
        assert any(c[2] == K for c in SHAPES)
    assert {c[3] for c in CS_CASES} == set(DEFAULT_EPIS) and {c[3] for c in DEFAULT_CASES} == set(DEFAULT_EPIS)
    assert not all(c[5] for c in FORCE_CASES + DEFAULT_CASES + CS_CASES + SPLIT_CASES)


@pytest.mark.parametrize("layout", ["contiguous", "embedded"])
@pytest.mark.parametrize("M,N,K,epi,plan,with_bias", CASES, ids=[_case_id(c) for c in CASES])
def test_gemm_is_exact(M, N, K, epi, plan, with_bias, layout, plan_env):
    from vlfm_b200.vlm.dense import gemm_f16

    if plan == "csplit":
        plan_env.setenv("VLFM_GEMM_CSPLIT", "2")
    elif plan != "default":
        plan_env.setenv("VLFM_GEMM_FORCE", plan)
    a, w, bias, g = _operands(M, N, K, M * 7919 + N * 31 + K * 3 + epi)
    if not with_bias:
        bias = None
    out_dtype = torch.float32 if epi in (2, 3) else torch.float16
    if layout == "contiguous":
        buf = _sentinel((M, _ceil8(N)), out_dtype, g if epi == 2 else None)
        window = (slice(0, M), slice(0, N))
        a_op, w_op, rows = a, w, None
    else:
        buf = _sentinel((M + 2, _ceil8(N + 16)), out_dtype, g if epi == 2 else None)
        window = (slice(1, M + 1), slice(8, 8 + N))
        a_op = _nan_buffer((M + 3, K + 16), (slice(1, M + 1), slice(8, 8 + K)), a)[1:M + 2, 8:8 + K]   # one NaN row past M
        w_op = _nan_buffer((N + 1, K + 8), (slice(0, N), slice(0, K)), w)[:N, :K]
        rows = M
    before = buf.clone()
    pre = a.double() @ w.double().t()
    if bias is not None:
        pre = pre + bias.double()
    if epi == 2:
        pre = pre + before[window].double()
    gemm_f16(a_op, w_op, bias, epi | (FLAG if plan == "csplit" else 0), buf[window], rows=rows)
    torch.cuda.synchronize()
    _check_epilogue(buf[window], pre, epi, "output")
    _outside_kept(buf, before, window, "output")


def test_cluster_split_plans_cover_every_width_and_split(plan_env):
    """The (BN, s) the cluster split takes for CS_SHAPES: BN 128, 96 and 64, unsplit and split, all occur."""
    _, lib = _lib()
    plan_env.setenv("VLFM_GEMM_CSPLIT", "2")
    plans = {}
    for M, N, K in CS_SHAPES:
        bn, s, nbytes = ctypes.c_int(), ctypes.c_int(), ctypes.c_double()
        assert lib.vlfm_gemm_csplit_plan(M, N, K, ctypes.addressof(bn), ctypes.addressof(s), ctypes.addressof(nbytes)) == 0
        plans[(M, N, K)] = (bn.value, s.value)
    print("cluster-split plans:", plans)
    assert {p[0] for p in plans.values()} == {128, 96, 64}, plans
    assert any(p[1] == 1 for p in plans.values()) and any(p[1] > 1 for p in plans.values()), plans


# ----------------------------------------------------------------------------------------------------- resid + LayerNorm ----
SLAB_FLOATS = 130 * 128       # SK_SLAB in common.cuh: one 128 x 128 tile and two tail rows


def _tiles128(M, N, K):
    tail = M > 128 and 1 <= M % 128 <= 2 and (K + 63) // 64 * 64 <= 6144
    return (M // 128 if tail else (M + 127) // 128) * ((N + 127) // 128)


def _ln_params(N, seed):
    g = _gen(seed)
    gamma = (1 + 0.1 * torch.randn(N, generator=g)).float().cuda()
    beta = (0.1 * torch.randn(N, generator=g)).float().cuda()
    return gamma, beta


def _ln_ref(x, gamma, beta):
    return torch.nn.functional.layer_norm(x.double(), (x.shape[1],), gamma.double(), beta.double(), EPS)


def _check_ln(y32, y16, ref):
    scale = max(1.0, float(ref.abs().max()))
    assert float((y32.double() - ref).abs().max()) <= 2e-5 * scale
    if y16 is not None:
        assert float((y16.double() - ref).abs().max()) <= 4e-3 * scale


class _ResidLN:
    """Embedded operands of one resid-LN call: A, W as in test_gemm_is_exact, x a window of a buffer of finite values, y16 / y32
    windows of payload-NaN buffers, and a workspace of `floats` declared floats followed by 1024 spare ones, all payload NaN."""

    def __init__(self, M, N, K, seed, x2=False):
        self.M, self.N, self.K = M, N, K
        self.a, self.w, self.bias, g = _operands(M, N, K, seed)
        self.a_op = _nan_buffer((M + 3, K + 16), (slice(1, M + 1), slice(8, 8 + K)), self.a)[1:M + 1, 8:8 + K]
        self.w_op = _nan_buffer((N + 1, K + 8), (slice(0, N), slice(0, K)), self.w)[:N, :K]
        self.win = (slice(1, M + 1), slice(8, 8 + N))
        self.xbuf = _sentinel((M + 2, N + 16), torch.float32, g)
        self.x0 = self.xbuf.clone()
        self.gamma, self.beta = _ln_params(N, seed)
        self.bufs = {"y32": _sentinel((M + 2, N + 16), torch.float32), "y16": _sentinel((M + 2, N + 16), torch.float16)}
        if x2:
            self.bufs["ylo"] = _sentinel((M + 2, N + 16), torch.float16)
        self.before = {k: v.clone() for k, v in self.bufs.items()}
        self.exact_x = (self.x0[self.win].double() + self.a.double() @ self.w.double().t() + self.bias.double())

    def workspace(self, floats):
        if floats is None:
            return None, None
        ws = _sentinel((floats + 1024,), torch.float32)
        return ws, floats * 4

    def check(self, what):
        _assert_equal(self.xbuf[self.win], self.exact_x.float(), f"{what}: x")
        _outside_kept(self.xbuf, self.x0, self.win, f"{what}: x")
        for k, buf in self.bufs.items():
            _outside_kept(buf, self.before[k], self.win, f"{what}: {k}")
        ref = _ln_ref(self.exact_x.float(), self.gamma, self.beta)
        y16 = self.bufs["y16"][self.win].double()
        if "ylo" in self.bufs:
            y16 = y16 + self.bufs["ylo"][self.win].double() / 2048.0
            assert float((y16 - self.bufs["y32"][self.win].double()).abs().max()) <= 2e-6 * max(1.0, float(ref.abs().max()))
        _check_ln(self.bufs["y32"][self.win], y16, ref)


def _resid_ln(c, ws, nbytes):
    L, lib = _lib()
    x, y16, y32 = c.xbuf[c.win], c.bufs["y16"][c.win], c.bufs["y32"][c.win]
    return lib.vlfm_gemm_f16_resid_ln(c.a_op.data_ptr(), c.w_op.data_ptr(), c.bias.data_ptr(), x.data_ptr(), c.M, c.N, c.K,
                                      c.a_op.stride(0), c.w_op.stride(0), x.stride(0), c.gamma.data_ptr(), c.beta.data_ptr(),
                                      y16.data_ptr(), y16.stride(0), y32.data_ptr(), y32.stride(0), EPS, L.ptr(ws), nbytes or 0,
                                      L.stream_ptr())


def _slabs_written(ws, floats, unit):
    """Indices of the `unit`-float chunks of the declared workspace that hold anything but the NaN sentinel."""
    used = (_bits(ws[:floats]) != NAN32).view(-1)
    n = floats // unit
    return [i for i in range(n) if bool(used[i * unit:(i + 1) * unit].any())]


# stream-K below one wave: P CTAs need P + tiles - 1 slabs.  P = SMs (the full plan), P = tiles + 1 (the least that splits), and
# P = tiles (which runs unsplit: the workspace stays untouched)
@pytest.mark.parametrize("M,N,K", [(257, 1408, 1408), (300, 1000, 520), (130, 1536, 6144)])
@pytest.mark.parametrize("variant", ["sms", "tiles+1", "tiles"])
def test_resid_ln_stream_k_is_exact(M, N, K, variant):
    c = _ResidLN(M, N, K, M + N + K)
    tiles = _tiles128(M, N, K)
    assert tiles < _sms()
    P = {"sms": _sms(), "tiles+1": tiles + 1, "tiles": tiles}[variant]
    floats = (P + tiles - 1) * SLAB_FLOATS
    ws, nbytes = c.workspace(floats)
    L, _ = _lib()
    L.check(_resid_ln(c, ws, nbytes), "vlfm_gemm_f16_resid_ln")
    torch.cuda.synchronize()
    c.check(variant)
    assert bool((_bits(ws[floats:]) == NAN32).all()), "written past the declared workspace"
    written = _slabs_written(ws, floats, SLAB_FLOATS)
    if variant == "tiles":
        assert not written, "P = tiles must run unsplit"
    else:
        assert written, "stream-K wrote no slab"


def test_resid_ln_uniform_split_is_exact():
    """Above one wave of 128 x 128 tiles the split is uniform, one M x N slab per split.  With room for 8, the plan takes s > 1
    of them; exactly s slabs give the same plan; 4 bytes less cap it at s - 1; no workspace runs unsplit.  x is exact every time
    and nothing past the declared workspace is written."""
    sms = _sms()
    M, N, K = 128 * math.ceil(sms / 12) + 64, 1536, 6144
    assert _tiles128(M, N, K) >= sms
    L, _ = _lib()
    unit = M * N
    c = _ResidLN(M, N, K, 11)
    ws, nbytes = c.workspace(8 * unit)
    L.check(_resid_ln(c, ws, nbytes), "vlfm_gemm_f16_resid_ln")
    torch.cuda.synchronize()
    c.check("8 slabs")
    s = len(_slabs_written(ws, 8 * unit, unit))
    assert s > 1, "the uniform split did not split"
    for label, floats, nbytes_less, most in (("exactly s slabs", s * unit, 0, s), ("s slabs - 4 bytes", s * unit, 4, s - 1),
                                               ("no workspace", None, 0, 0)):
        c = _ResidLN(M, N, K, 11)
        ws, nbytes = c.workspace(floats)
        L.check(_resid_ln(c, ws, None if nbytes is None else nbytes - nbytes_less), "vlfm_gemm_f16_resid_ln")
        torch.cuda.synchronize()
        c.check(label)
        if ws is not None:
            written = _slabs_written(ws, floats, unit)
            assert len(written) <= most and written == list(range(len(written))), (label, written)
            if nbytes_less == 0:
                assert len(written) == s, (label, written)
            assert bool((_bits(ws[floats:]) == NAN32).all()), f"{label}: written past the workspace"


# --------------------------------------------------------------------------------------------------------------- x2 GEMM ----
# M > 128 with M % 128 <= 32 runs its last rows as a launch of their own for the fp32 and GELU-x2 epilogues (129, 160, 257; not
# 161); M > 128 with N >= 4096 takes BN 128, 33 x 6144 BN 64, the others BN 32
X2_SHAPES = [(1, 1000, 1000), (32, 520, 72), (33, 6144, 1408), (129, 4224, 8), (160, 1000, 520), (161, 4224, 6152), (257, 4224, 64)]
X2_EPIS = {"f32": 3, "resid": 2, "gelu_x2": 6}
X2_CASES = ([(M, N, K, e, False) for (M, N, K) in X2_SHAPES for e in X2_EPIS]
            + [(M, N, K, list(X2_EPIS)[i % 3], True) for i, (M, N, K) in enumerate(X2_SHAPES)])


def _x2_operands(M, N, K, seed, lo):
    a, w, bias, g = _operands(M, N, K, seed)
    if lo:
        a_lo, w_lo = _grid((M, K), 3, 4, g, torch.float16), _grid((N, K), 3, 8, g, torch.float16)
    else:
        a_lo, w_lo = torch.zeros_like(a), torch.zeros_like(w)
    emb_a = lambda t: _nan_buffer((M + 3, K + 16), (slice(1, M + 1), slice(8, 8 + K)), t)[1:M + 1, 8:8 + K]
    emb_w = lambda t: _nan_buffer((N + 1, K + 8), (slice(0, N), slice(0, K)), t)[:N, :K]
    ops = (emb_a(a), emb_a(a_lo), emb_w(w), emb_w(w_lo))
    exact = (a.double() + a_lo.double() / 2048) @ (w.double() + w_lo.double() / 2048).t() + bias.double()
    return ops, bias, exact, g


@pytest.mark.parametrize("M,N,K,epi,lo", X2_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}" + ("-lo" if c[4] else "") for c in X2_CASES])
def test_gemm_x2_is_exact(M, N, K, epi, lo):
    L, lib = _lib()
    (ahi, alo, whi, wlo), bias, exact, g = _x2_operands(M, N, K, 7 * M + N + K, lo)
    win = (slice(1, M + 1), slice(8, 8 + N))
    shape = (M + 2, _ceil8(N + 16))
    if epi == "gelu_x2":
        out, out_lo = _sentinel(shape, torch.float16), _sentinel(shape, torch.float16)
    else:
        out, out_lo = _sentinel(shape, torch.float32, g if epi == "resid" else None), None
    before, before_lo = out.clone(), None if out_lo is None else out_lo.clone()
    if epi == "resid":
        exact = exact + before[win].double()
    L.check(lib.vlfm_gemm_f16x2(ahi.data_ptr(), alo.data_ptr(), whi.data_ptr(), wlo.data_ptr(), bias.data_ptr(), out[win].data_ptr(),
                                None if out_lo is None else out_lo[win].data_ptr(), M, N, K, ahi.stride(0), whi.stride(0), out.stride(0),
                                X2_EPIS[epi], L.stream_ptr()), "vlfm_gemm_f16x2")
    torch.cuda.synchronize()
    _outside_kept(out, before, win, "out")
    if epi == "gelu_x2":
        _outside_kept(out_lo, before_lo, win, "out_lo")
        got = out[win].double() + out_lo[win].double() / 2048.0
        ref = torch.nn.functional.gelu(exact)
    else:
        got, ref = out[win].double(), exact
    assert bool(torch.isfinite(got).all()), "an output element was not written"
    if lo:
        scale = float(ref.abs().max())
        assert float((got - ref).abs().max()) <= 5e-6 * scale
    elif epi == "gelu_x2":
        # the pre-activation is exact; what is left is erff in fp32 (its cancellation in 1 + erf below -3) and the pair's rounding
        err = (got - ref).abs()
        assert bool((err <= 2.0 ** -18 * ref.abs() + 1e-6).all()), float(err.max())
    else:
        _assert_equal(out[win], exact.float(), "out")


@pytest.mark.parametrize("M,N,K,split", [(1, 768, 1000, True), (33, 1408, 3072, True), (160, 768, 520, True), (257, 1408, 1408, True),
                                         (257, 1408, 1408, False)])
def test_gemm_x2_resid_ln_is_exact(M, N, K, split):
    """lo = 0: x is the exact value, split (deterministic partial sums in the workspace) or not; the x2 LayerNorm output pair
    and the fp32 output are within the LayerNorm bars of float64, and nothing is written outside the windows."""
    L, lib = _lib()
    c = _ResidLN(M, N, K, 3 * M + N + K, x2=True)
    zeros_a = _nan_buffer((M + 3, K + 16), (slice(1, M + 1), slice(8, 8 + K)), torch.zeros_like(c.a))[1:M + 1, 8:8 + K]
    zeros_w = _nan_buffer((N + 1, K + 8), (slice(0, N), slice(0, K)), torch.zeros_like(c.w))[:N, :K]
    ws, nbytes = c.workspace(8 * M * N if split else None)
    x, hi, lo, y32 = c.xbuf[c.win], c.bufs["y16"][c.win], c.bufs["ylo"][c.win], c.bufs["y32"][c.win]
    L.check(lib.vlfm_gemm_f16x2_resid_ln(c.a_op.data_ptr(), zeros_a.data_ptr(), c.w_op.data_ptr(), zeros_w.data_ptr(), c.bias.data_ptr(),
                                         x.data_ptr(), M, N, K, c.a_op.stride(0), c.w_op.stride(0), x.stride(0), c.gamma.data_ptr(),
                                         c.beta.data_ptr(), hi.data_ptr(), lo.data_ptr(), hi.stride(0), y32.data_ptr(), y32.stride(0), EPS,
                                         L.ptr(ws), nbytes or 0, L.stream_ptr()), "vlfm_gemm_f16x2_resid_ln")
    torch.cuda.synchronize()
    c.check("x2 resid ln")
    if ws is not None:
        assert bool((_bits(ws[8 * M * N:]) == NAN32).all())


# ---------------------------------------------------------------------------------------------------------------- refusals ----
def test_gemm_f16_refusals():
    """Each bad call returns VLFM_E_INVALID, launches nothing and leaves the output alone; then one valid call launches."""
    L, lib = _lib()
    M, N, K = 64, 64, 64
    a = torch.ones(M, K + 16, dtype=torch.float16, device="cuda")
    w = torch.ones(N, K + 16, dtype=torch.float16, device="cuda")
    bias = torch.zeros(N + 8, device="cuda")
    out = _sentinel((M, N + 16), torch.float16)
    before = out.clone()

    def call(A=a.data_ptr(), W=w.data_ptr(), O=out.data_ptr(), m=M, n=N, k=K, lda=K + 16, ldw=K + 16, ldo=N + 16, epi=0):
        return lib.vlfm_gemm_f16(A, W, bias.data_ptr(), O, m, n, k, lda, ldw, ldo, epi, L.stream_ptr())

    bad = [dict(k=60), dict(lda=K + 12), dict(ldw=K + 4), dict(ldo=N + 12), dict(A=a.data_ptr() + 8), dict(W=w.data_ptr() + 8),
           dict(O=out.data_ptr() + 8), dict(epi=-1), dict(epi=5), dict(epi=6), dict(epi=8), dict(m=0), dict(n=0), dict(k=0),
           dict(A=None), dict(W=None), dict(O=None)]
    n0 = L.launch_count()
    for kw in bad:
        assert call(**kw) == 1, kw
    torch.cuda.synchronize()
    assert L.launch_count() == n0
    assert torch.equal(_bits(out), _bits(before))
    assert call() == 0
    torch.cuda.synchronize()
    assert L.launch_count() == n0 + 1
    _assert_equal(out[:, :N], torch.full((M, N), float(K), dtype=torch.float16, device="cuda"), "valid call")


class _LNFamily:
    """Buffers for the six LayerNorm entry points at D up to 2048 (a refused D must not be launched, so nothing overruns):
    x of finite values, payload-NaN outputs and workspace.  call(fn, ...) returns the code; every buffer is checked afterwards."""
    ROWS, DMAX, K = 4, 2048, 64

    def __init__(self):
        R, D = self.ROWS, self.DMAX
        g = _gen(5)
        self.ld = D + 16
        self.x = _grid((R, self.ld), 2048, 32, g, torch.float32)
        self.gamma = torch.ones(D + 16, device="cuda")
        self.beta = torch.zeros(D + 16, device="cuda")
        self.y32, self.y16, self.ylo = (_sentinel((R, self.ld), t) for t in (torch.float32, torch.float16, torch.float16))
        self.ws = _sentinel((8 * R * self.ld,), torch.float32)
        self.a = _grid((R, self.K), 3, 4, g, torch.float16)
        self.w = _grid((D, self.K), 3, 8, g, torch.float16)
        self.bufs = (self.x, self.y32, self.y16, self.ylo, self.ws)
        self.before = [b.clone() for b in self.bufs]

    def call(self, fn, D, gamma_off=0, beta_off=0, y32_off=0, y16_off=0, ylo_off=0):
        L, lib = _lib()
        R, ld, K = self.ROWS, self.ld, self.K
        x, ws = self.x.data_ptr(), self.ws.data_ptr()
        gm, bt = self.gamma.data_ptr() + gamma_off, self.beta.data_ptr() + beta_off
        y32, y16, ylo = self.y32.data_ptr() + y32_off, self.y16.data_ptr() + y16_off, self.ylo.data_ptr() + ylo_off
        st, a, w = L.stream_ptr(), self.a.data_ptr(), self.w.data_ptr()
        eps = ctypes.c_float(EPS)
        if fn == "layernorm":
            return lib.vlfm_layernorm(x, gm, bt, y16, y32, R, D, ld, ld, ld, eps, st)
        if fn == "layernorm_x2":
            return lib.vlfm_layernorm_x2(x, gm, bt, y16, ylo, y32, R, D, ld, ld, ld, eps, st)
        if fn == "layernorm_reduce":
            return lib.vlfm_layernorm_reduce(x, ws, 2, R * ld, gm, bt, y16, y32, R, D, ld, ld, ld, eps, st)
        if fn == "layernorm_reduce_x2":
            return lib.vlfm_layernorm_reduce_x2(x, ws, 2, R * ld, gm, bt, y16, ylo, y32, R, D, ld, ld, ld, eps, st)
        if fn == "resid_ln":
            return lib.vlfm_gemm_f16_resid_ln(a, w, None, x, R, D, K, K, K, ld, gm, bt, y16, ld, y32, ld, EPS, ws, self.ws.numel() * 4, st)
        assert fn == "resid_ln_x2"
        return lib.vlfm_gemm_f16x2_resid_ln(a, a, w, w, None, x, R, D, K, K, K, ld, gm, bt, y16, ylo, ld, y32, ld, EPS, ws,
                                            self.ws.numel() * 4, st)

    def untouched(self):
        torch.cuda.synchronize()
        return all(torch.equal(_bits(b), _bits(c)) for b, c in zip(self.bufs, self.before))


LN_FNS = ["layernorm", "layernorm_x2", "layernorm_reduce", "layernorm_reduce_x2", "resid_ln", "resid_ln_x2"]


def _refusals(cases):
    L, _ = _lib()
    f = _LNFamily()
    n0 = L.launch_count()
    for fn, kw, code in cases:
        rc = f.call(fn, **kw)
        assert rc == code, (fn, kw, rc)
        assert L.launch_count() == n0, f"{fn} {kw}: refused but launched"
        assert f.untouched(), f"{fn} {kw}: refused but changed x, an output or the workspace"
    for fn in LN_FNS:
        assert f.call(fn, 1408) == 0, fn
        torch.cuda.synchronize()
        assert L.launch_count() > n0, fn
        n0 = L.launch_count()


def test_layernorm_family_refuses_wide_and_ragged_rows():
    """D (the GEMM's N) above 1536, the LayerNorm's limit, or not a multiple of 4: refused before anything runs.  The resid-LN
    GEMMs check it before their GEMM, so x and the workspace keep their values."""
    cases = []
    for fn in LN_FNS:
        resid = fn.startswith("resid")
        cases += [(fn, dict(D=1540), 3), (fn, dict(D=2048), 3), (fn, dict(D=1406), 1 if resid else 3)]
    _refusals(cases)


def test_layernorm_family_refuses_misaligned_pointers():
    """gamma, beta, out32 are read / written as float4 and the fp16 outputs as 4 halves: an offset of one element is refused with
    VLFM_E_INVALID instead of reaching the kernel."""
    cases = []
    for fn in LN_FNS:
        cases += [(fn, dict(D=1408, gamma_off=4), 1), (fn, dict(D=1408, beta_off=4), 1), (fn, dict(D=1408, y32_off=4), 1),
                  (fn, dict(D=1408, y16_off=2), 1)]
        if fn.endswith("x2"):
            cases.append((fn, dict(D=1408, ylo_off=2), 1))
    _refusals(cases)
