"""CPU checks of two algorithm restatements the kernels rely on (the kernels themselves are checked on the GPU):

* `ppt_distance_warp` (csrc/explore.cu) evaluates cv2.pointPolygonTest in 32 contiguous chunks and combines the chunk results in
  order with the sequential "first strictly smaller" comparison -- here the same chunked scan in numpy against the oracle's
  sequential one;
* the x2 operand arithmetic of `gemm_f16x2_wgmma_kernel` (csrc/gemm_wgmma.cu): v = hi + lo/2048 with fp16 pairs and the
  three-product expansion hi.hi + (lo.hi + hi.lo)/2048 -- here in numpy against float64."""
import numpy as np

from oracle import contours as C


def _chunked_ppt(c, pt, nl=32):
    p = c.reshape(-1, 2)
    n = len(p)
    px, py = np.float32(pt[0]), np.float32(pt[1])
    chunk = (n + nl - 1) // nl
    res, counter = [], 0
    for lane in range(nl):
        c0 = min(n, lane * chunk)
        c1 = min(n, c0 + chunk)
        mn, md = float(np.finfo(np.float32).max), 1.0
        if c0 < c1:
            v = p[(c0 - 1) % n].astype(np.float32)
            for i in range(c0, c1):
                v0, v = v, p[i].astype(np.float32)
                dx, dy = float(v[0] - v0[0]), float(v[1] - v0[1])
                dx1, dy1 = float(px - v0[0]), float(py - v0[1])
                dx2, dy2 = float(px - v[0]), float(py - v[1])
                den = 1.0
                if dx1 * dx + dy1 * dy <= 0:
                    num = dx1 * dx1 + dy1 * dy1
                elif dx2 * dx + dy2 * dy >= 0:
                    num = dx2 * dx2 + dy2 * dy2
                else:
                    num = dy1 * dx - dx1 * dy
                    num *= num
                    den = dx * dx + dy * dy
                if num * md < mn * den:
                    mn, md = num, den
                    if mn == 0:
                        return 0.0
                if (v0[1] <= py and v[1] <= py) or (v0[1] > py and v[1] > py):
                    continue
                cr = dy1 * dx - dx1 * dy
                if dy < 0:
                    cr = -cr
                counter += cr > 0
        res.append((mn, md))
    bn, bd = res[0]
    for mn, md in res[1:]:
        if mn * bd < bn * md:
            bn, bd = mn, md
    r = float(np.sqrt(bn / bd))
    return r if counter % 2 else -r


def test_chunked_point_polygon_test_equals_the_sequential_scan():
    rng = np.random.default_rng(0)
    n = 0
    for _ in range(25):
        img = (rng.random((40, 50)) < 0.55).astype(np.uint8)
        img = ((np.roll(img, 1, 0) + np.roll(img, -1, 0) + np.roll(img, 1, 1) + np.roll(img, -1, 1) + img) >= 3).astype(np.uint8)
        for c in C.find_external_contours(img):
            s = C.approx_simple(c)
            for _ in range(3):
                pt = (int(rng.integers(-5, 55)), int(rng.integers(-5, 45)))
                a, b = C.point_polygon_distance(s, pt), _chunked_ppt(s, pt)
                assert a == b or (a == 0 and b == 0), (a, b, len(s))
                n += 1
    assert n > 300


def test_x2_operands_carry_float32_values_and_three_products_suffice():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal((32, 768)) * 0.7).astype(np.float32)
    w = (rng.standard_normal((96, 768)) * 0.04).astype(np.float32)
    a[0, :4] = [40.0, -25.0, 1e-4, 3e-6]

    def split(t):
        hi = t.astype(np.float16)
        lo = ((t - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
        return hi, lo

    ahi, alo = split(a)
    whi, wlo = split(w)
    # the pair reconstructs the float32 value to ~2^-22 relative (the residual keeps 11 more bits)
    rec = ahi.astype(np.float64) + alo.astype(np.float64) / 2048.0
    assert np.abs(rec - a.astype(np.float64)).max() <= 2.0 ** -21 * np.abs(a).max()
    assert np.isfinite(alo.astype(np.float32)).all() and np.abs(alo.astype(np.float32)).max() <= np.abs(a).max()   # no overflow, no tiny subnormals
    ref = a.astype(np.float64) @ w.astype(np.float64).T
    main = ahi.astype(np.float64) @ whi.astype(np.float64).T
    corr = alo.astype(np.float64) @ whi.astype(np.float64).T + ahi.astype(np.float64) @ wlo.astype(np.float64).T
    x2 = main + corr / 2048.0
    scale = np.abs(ref).max()
    assert np.abs(x2 - ref).max() <= 1e-6 * scale                      # dropped lo.lo term + residual rounding
    assert np.abs(main - ref).max() >= 1e-4 * scale                    # ... where plain fp16 operands are three orders worse
