"""Executable model of b200jpg_batch_create_resample (DESIGN §19): Pillow 12.2's Image.resize with a source box and a reducing_gap,
then a window of the result, on uint8 images, one channel at a time. TEST-ONLY.

Built on tests/resize_model.py (filters, fixed point, passes). The box reaches the resampler as Pillow's C floats (float32), the
reduce step is computed in doubles as Pillow's Python does, and Image.reduce is ((s + n / 2) * (2^24 // n)) >> 24 over each block
of n real pixels. tests/test_resize_box_cpu.py pins it on Pillow byte for byte."""
import math

import numpy as np

from tests import resize_model as rm

SUPPORT = {rm.BOX: 0.5, rm.BILINEAR: 1.0, rm.HAMMING: 1.0, rm.BICUBIC: 2.0, rm.LANCZOS: 3.0}  # Pillow's _filters_support


def coefficients_box(in_size, in0, in1, out_size, resample, box_dtype=np.float32):
    """precompute_coeffs with the box [in0, in1) as C floats: scale = (double)(in1 - in0) / out_size with the difference in float,
    center = in0 + (j + 0.5) * scale. Returns (bounds, table, ksize) as resize_model.coefficients."""
    f, s = rm.FILTERS[resample]
    in0, in1 = box_dtype(in0), box_dtype(in1)
    scale = float(box_dtype(in1 - in0)) / out_size
    fs = max(scale, 1.0)
    support = s * fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int64)
    table = np.zeros((out_size, ksize), dtype=np.int64)
    for j in range(out_size):
        center = float(in0) + (j + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [f((t + xmin - center + 0.5) / fs) for t in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        for t, v in enumerate(w):
            table[j, t] = int(v * (1 << rm.PRECISION_BITS) - 0.5) if v < 0 else int(v * (1 << rm.PRECISION_BITS) + 0.5)
        bounds[j] = (xmin, max(n, 0))
    return bounds, table, ksize


def reduce_channel(img, fx, fy, rbox=None):
    """Image.reduce((fx, fy), box=rbox) of one [h, w] uint8 channel: blocks of fx x fy from the box's origin, the last ones partial"""
    h, w = img.shape
    x0, y0, x1, y1 = rbox if rbox is not None else (0, 0, w, h)
    a = img[y0:y1, x0:x1].astype(np.int64)
    bh, bw = a.shape
    oh, ow = -(-bh // fy), -(-bw // fx)
    out = np.empty((oh, ow), dtype=np.uint8)
    for y in range(oh):
        for x in range(ow):
            blk = a[y * fy:(y + 1) * fy, x * fx:(x + 1) * fx]
            n = blk.size
            out[y, x] = (((int(blk.sum()) + n // 2) * ((1 << 24) // n)) & 0xFFFFFFFF) >> 24
    return out


def reduce_plan(w, h, width, height, resample, box, gap):
    """(fx, fy, reduce box or None, box after the reduce) of Image.resize on a w x h image, Pillow's Python in doubles"""
    box = (0, 0, w, h) if box is None else tuple(box)
    if gap is None:
        return 1, 1, None, box
    fx = int((box[2] - box[0]) / width / gap) or 1
    fy = int((box[3] - box[1]) / height / gap) or 1
    if fx == 1 and fy == 1:
        return 1, 1, None, box
    support = SUPPORT[resample] - 0.5
    sx = support * ((box[2] - box[0]) / width)
    sy = support * ((box[3] - box[1]) / height)
    rb = (max(0, int(box[0] - sx)), max(0, int(box[1] - sy)), min(w, math.ceil(box[2] + sx)), min(h, math.ceil(box[3] + sy)))
    nb = ((box[0] - rb[0]) / fx, (box[1] - rb[1]) / fy, (box[2] - rb[0]) / fx, (box[3] - rb[1]) / fy)
    return fx, fy, rb, nb


def resize_channel(img, width, height, resample, box=None, gap=None, window=None, box_dtype=np.float32):
    """One [h, w] uint8 channel: reduce step, Pillow's passes where need_horizontal / need_vertical say so, then the window
    (x, y, width, height) of the width x height result. box_dtype=np.float64 gives what a double box would (tests only)."""
    h, w = img.shape
    fx, fy, rb, box = reduce_plan(w, h, width, height, resample, box, gap)
    src = img if rb is None else reduce_channel(img, fx, fy, rb)
    sh, sw = src.shape
    fb = np.asarray(box, dtype=box_dtype)
    need_h = width != sw or fb[0] != 0 or fb[2] != width
    need_v = height != sh or fb[1] != 0 or fb[3] != height
    a = src.astype(np.int64)
    if need_v:
        vb, vt, _ = coefficients_box(sh, fb[1], fb[3], height, resample, box_dtype)
    if need_h:
        y0, y1 = (int(vb[0, 0]), int(vb[-1, 0] + vb[-1, 1])) if need_v else (0, sh)
        hb, ht, _ = coefficients_box(sw, fb[0], fb[2], width, resample, box_dtype)
        a = rm._pass(a[y0:y1], hb, ht, 1)
        if need_v:
            vb = vb.copy()
            vb[:, 0] -= y0
    if need_v:
        a = rm._pass(a, vb, vt, 0)
    out = a.astype(np.uint8)
    if window is not None:
        x, y, ww, wh = window
        out = out[y:y + wh, x:x + ww]
    return out


def resize(img, width, height, resample, box=None, gap=None, window=None, box_dtype=np.float32):
    """on an [h, w] or [h, w, C] uint8 image, every channel on its own"""
    if img.ndim == 2:
        return resize_channel(img, width, height, resample, box, gap, window, box_dtype)
    return np.stack([resize_channel(img[..., c], width, height, resample, box, gap, window, box_dtype) for c in range(img.shape[2])],
                    axis=-1)
