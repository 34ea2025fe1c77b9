"""Crop rectangles: a restatement of the planner's rectangle algebra (abi.cpp: crop_to_decoded, translate_plane, DESIGN §12) and
a byte-addressed store model that follows it, for the CPU tests; rectangle helpers for the GPU tests."""
import numpy as np

from tests import orientation_model as om


def crop_to_decoded(o, rect, w, h):
    """the output rectangle (x, y, width, height) of orientation o as [x0, x1) x [y0, y1) of the decoded image of extent w x h"""
    x, y, rw, rh = rect
    u0, u1, v0, v1 = x, x + rw, y, y + rh
    return {
        1: (u0, v0, u1, v1),
        2: (w - u1, v0, w - u0, v1),
        3: (w - u1, h - v1, w - u0, h - v0),
        4: (u0, h - v1, u1, h - v0),
        5: (v0, u0, v1, u1),
        6: (v0, h - u1, v1, h - u0),
        7: (w - v1, h - u1, w - v0, h - u0),
        8: (w - v1, u0, w - v0, u1),
    }[o]


def translate(data, p, r, rect):
    """a destination of the cropped image as a destination of the uncropped output"""
    return data - rect[0] * p - rect[1] * r, p, r


def store(decoded, o, rect, p, r, origin, size):
    """The kernels' store, modelled: every sample of `decoded` ([h, w] uint8) inside the clip rectangle goes through the caller's
    descriptor (origin, p, r) of the cropped image, translated and then oriented, into a byte buffer of `size`. Returns the
    buffer (0xA5 where nothing was written); an address outside it raises IndexError."""
    h, w = decoded.shape
    x0, y0, x1, y1 = crop_to_decoded(o, rect, w, h)
    d, pp, rr = om.orient_plane(*translate(origin, p, r, rect), o, w, h)
    buf = np.full(size, 0xA5, dtype=np.uint8)
    for y in range(y0, y1):
        for x in range(x0, x1):
            a = d + x * pp + y * rr
            if not 0 <= a < size:
                raise IndexError("store at %d outside the destination" % a)
            buf[a] = decoded[y, x]
    return buf


def rectangles(ow, oh, rng, n_random=4, sub=(1, 1)):
    """rectangles (x, y, width, height) of an oh x ow output: the full frame, 1x1 at each corner, one row, one column, one inside
    an 8x8 block, origins and ends at the tile seams +-1 (x = 255 / 256 / 257, y around multiples of 32 and 8), an origin in
    the middle of an MCU of `sub` and seeded random ones; each clipped to the frame and deduplicated"""
    cand = [(0, 0, ow, oh), (0, 0, 1, 1), (ow - 1, 0, 1, 1), (0, oh - 1, 1, 1), (ow - 1, oh - 1, 1, 1),
            (0, oh // 2, ow, 1), (ow // 2, 0, 1, oh), (min(9, ow - 1), min(10, oh - 1), 5, 4)]
    for sx in (255, 256, 257):
        cand.append((sx, 0, ow - sx, oh))
        cand.append((0, 0, sx, oh))
    for sy in (7, 8, 9, 31, 32, 33, 63, 64, 65):
        cand.append((0, sy, ow, oh - sy))
        cand.append((3, 0, ow - 3, sy))
    mx, my = 8 * sub[0], 8 * sub[1]
    cand.append((mx // 2 + 1, my // 2 + 1, ow - mx // 2 - 1, oh - my // 2 - 1))
    for _ in range(n_random):
        x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
        cand.append((x, y, int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))))
    out = []
    for x, y, w, h in cand:
        if 0 <= x < ow and 0 <= y < oh and w >= 1 and h >= 1 and x + w <= ow and y + h <= oh and (x, y, w, h) not in out:
            out.append((x, y, w, h))
    return out
