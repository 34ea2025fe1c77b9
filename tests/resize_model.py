"""Executable model of the resize stage (DESIGN §13): Pillow's convolution resampler (Image.resize with box=None and
reducing_gap=None) on uint8 images, one channel at a time.

The coefficients are computed with Python's math module, which evaluates in C doubles in the order DESIGN §13 gives, so the
tables equal the library's b200jpg_resample_coefficients bit for bit. The two passes run in int64 with the clamp."""
import math

import numpy as np

BOX, BILINEAR, HAMMING, BICUBIC, LANCZOS = 4, 2, 5, 3, 1  # PIL's enum values, B200JPG_RESAMPLE_*
NAMES = {"box": BOX, "bilinear": BILINEAR, "hamming": HAMMING, "bicubic": BICUBIC, "lanczos": LANCZOS}
PRECISION_BITS = 22


def _box(x):
    return 1.0 if -0.5 < x <= 0.5 else 0.0


def _bilinear(x):
    x = -x if x < 0.0 else x
    return 1.0 - x if x < 1.0 else 0.0


def _hamming(x):
    x = -x if x < 0.0 else x
    if x == 0.0:
        return 1.0
    if x >= 1.0:
        return 0.0
    x = x * math.pi
    return math.sin(x) / x * (0.54 + 0.46 * math.cos(x))


def _bicubic(x):
    a = -0.5
    x = -x if x < 0.0 else x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


FILTERS = {BOX: (_box, 0.5), BILINEAR: (_bilinear, 1.0), HAMMING: (_hamming, 1.0), BICUBIC: (_bicubic, 2.0), LANCZOS: (_lanczos, 3.0)}


def coefficients(in_size, out_size, resample):
    """(bounds [out_size, 2] int64 of (xmin, n), table [out_size, ksize] int64 of fixed-point coefficients, ksize)"""
    f, s = FILTERS[resample]
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = s * fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int64)
    table = np.zeros((out_size, ksize), dtype=np.int64)
    for j in range(out_size):
        center = (j + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [f((t + xmin - center + 0.5) / fs) for t in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        for t, v in enumerate(w):
            table[j, t] = int(v * (1 << PRECISION_BITS) - 0.5) if v < 0 else int(v * (1 << PRECISION_BITS) + 0.5)
        bounds[j] = (xmin, n)
    return bounds, table, ksize


def _pass(src, bounds, table, axis):
    """one pass along `axis` of a 2-D int64 array: out[j] = clamp((2^21 + sum_t k_t v[xmin + t]) >> 22, 0, 255)"""
    src = np.moveaxis(src, axis, 0)
    out = np.empty((len(bounds),) + src.shape[1:], dtype=np.int64)
    for j, (xmin, n) in enumerate(bounds):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
        for t in range(n):
            acc += table[j, t] * src[xmin + t]
        out[j] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def resize_channel(img, width, height, resample):
    """R of DESIGN §13 on one [h, w] uint8 channel: horizontal pass over the rows the vertical table touches, then vertical;
    an axis whose size does not change is not resampled"""
    h, w = img.shape
    a = img.astype(np.int64)
    vb, vt, _ = coefficients(h, height, resample)
    if width != w:
        y0, y1 = int(vb[0, 0]), int(vb[-1, 0] + vb[-1, 1])
        hb, ht, _ = coefficients(w, width, resample)
        a = _pass(a[y0:y1], hb, ht, 1)
        vb = vb.copy()
        vb[:, 0] -= y0
    if height != h:
        a = _pass(a, vb, vt, 0)
    return a.astype(np.uint8)


def resize(img, width, height, resample):
    """R on an [h, w] or [h, w, C] uint8 image, every channel on its own"""
    if img.ndim == 2:
        return resize_channel(img, width, height, resample)
    return np.stack([resize_channel(img[..., c], width, height, resample) for c in range(img.shape[2])], axis=-1)


def int32_bound_ok(table):
    """every row's positive coefficients keep 2^21 + 255 * sum(k > 0) inside int32"""
    pos = np.where(table > 0, table, 0).sum(axis=1)
    return bool(((1 << 21) + 255 * pos.max(initial=0) < 2 ** 31))
