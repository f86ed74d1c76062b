"""Host-side configuration tables for the GPU image preprocessor.

The reference preprocesses with lavis' ``BlipImageEvalProcessor`` (called at
vlfm/vlm/blip2itm.py:48-49): PIL ``Resize((224,224), BICUBIC)`` -> ToTensor ->
Normalize(CLIP mean/std).  PIL's resize is an antialiased separable convolution on
uint8 with 22-bit fixed-point coefficients; the tables built here restate Pillow's
``precompute_coeffs`` / ``normalize_coeffs_8bpc`` (libImaging/Resample.c) so that the
CUDA kernels (csrc/vit_ops.cu) reproduce PIL's bytes exactly.  They depend only on
(in_size, out_size) and are computed once.
"""
from __future__ import annotations

import math
from functools import lru_cache
from typing import Tuple

import numpy as np

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
PRECISION_BITS = 32 - 8 - 2


def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


@lru_cache(maxsize=None)
def bicubic_tables(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray, int]:
    """-> bounds [out,2] int32 (first index, count), kk [out,ksize] int32, ksize."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        xmin = max(xmin, 0)
        xmax = int(center + support + 0.5)
        xmax = min(xmax, in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = sum(w)
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk, ksize


def _bilinear(x: float) -> float:
    x = abs(x)
    return 1.0 - x if x < 1.0 else 0.0


@lru_cache(maxsize=None)
def bilinear_tables(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray, int]:
    """Pillow's BILINEAR (support 1) tables in the layout of ``bicubic_tables`` (MobileSAM's ResizeLongestSide)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bilinear((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = sum(w)
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk, ksize


def resize_numpy(img: np.ndarray, out_h: int, out_w: int, tables=bicubic_tables) -> np.ndarray:
    """Reference emulation of the two GPU passes (used by CPU tests to pin the tables to PIL)."""
    h, w, _ = img.shape
    hb, hk, _ = tables(w, out_w)
    vb, vk, _ = tables(h, out_h)
    src = img.astype(np.int64)
    mid = np.zeros((h, out_w, 3), np.int64)
    for xo in range(out_w):
        x0, n = hb[xo]
        acc = (src[:, x0 : x0 + n, :] * hk[xo, :n][None, :, None].astype(np.int64)).sum(1) + (1 << (PRECISION_BITS - 1))
        mid[:, xo, :] = np.clip(acc >> PRECISION_BITS, 0, 255)
    out = np.zeros((out_h, out_w, 3), np.int64)
    for yo in range(out_h):
        y0, n = vb[yo]
        acc = (mid[y0 : y0 + n] * vk[yo, :n][:, None, None].astype(np.int64)).sum(0) + (1 << (PRECISION_BITS - 1))
        out[yo] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return out.astype(np.uint8)
