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


def pillow_vertical_first(in_h: int, in_w: int, out_h: int) -> bool:
    """Pillow's pass order: ``Image.resize`` (Pillow 12.2, Image.py) resizes a frame more than 100x taller than wide that
    shrinks vertically as a vertical resize to (in_w, out_h) followed by a horizontal one; every other frame goes through one
    ``ImagingResample`` call, horizontal pass first.  The passes round to uint8 in between, so the order changes bytes."""
    return in_h > in_w * 100 and out_h < in_h


def _resize_pass(src: np.ndarray, out_n: int, tables, axis: int) -> np.ndarray:
    """One fixed-point pass of [h, w, 3] int64 along axis 1 (horizontal) or 0 (vertical), clipped to 0..255."""
    b, k, _ = tables(src.shape[axis], out_n)
    t = np.moveaxis(src, axis, 1)
    out = np.zeros((t.shape[0], out_n, 3), np.int64)
    for o in range(out_n):
        s0, n = b[o]
        acc = (t[:, s0 : s0 + n, :] * k[o, :n][None, :, None].astype(np.int64)).sum(1) + (1 << (PRECISION_BITS - 1))
        out[:, o, :] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 1, axis)


def resize_numpy(img: np.ndarray, out_h: int, out_w: int, tables=bicubic_tables) -> np.ndarray:
    """Reference emulation of the two GPU passes in Pillow's order (used by CPU tests to pin the tables to PIL)."""
    src = img.astype(np.int64)
    if pillow_vertical_first(img.shape[0], img.shape[1], out_h):
        out = _resize_pass(_resize_pass(src, out_h, tables, 0), out_w, tables, 1)
    else:
        out = _resize_pass(_resize_pass(src, out_w, tables, 1), out_h, tables, 0)
    return out.astype(np.uint8)
