"""CPU: crop rectangles without a device. The composition model (translate into the uncropped output, then orient_plane, store only
inside crop_to_decoded's clip) against numpy slicing of the oriented image; b200jpg_output_size against b200jpg_parse plus
b200jpg_exif_orientation; and the argument checks of BatchDecoder(crop=...) that run before any device is touched."""
import ctypes
import glob
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("o", list(om.ORIENTATIONS))
@pytest.mark.parametrize("shape", [(1, 1), (5, 9), (13, 6), (33, 40)])
@pytest.mark.parametrize("layout", ["packed", "planar_padded", "nhwc_bgr"])
def test_composition(o, shape, layout):
    """every rectangle of the oriented image: the stores through the rewritten descriptor are exactly its slice, inside the caller's
    bitmap, and nothing else is written"""
    h, w = shape
    rng = np.random.default_rng(h * 100 + w + o)
    d = rng.integers(0, 256, size=(h, w), dtype=np.uint8)
    want_full = om.orient(d, o)
    oh, ow = want_full.shape
    for rect in cm.rectangles(ow, oh, rng, n_random=6):
        x, y, rw, rh = rect
        want = want_full[y:y + rh, x:x + rw]
        if layout == "packed":  # one component of an interleaved 3-byte pixel, tight rows
            p, r, off = 3, 3 * rw, 1
            size = 3 * rw * rh
        elif layout == "planar_padded":
            p, r, off = 1, rw + 5, 2 * (rw + 5) + 3
            size = off + rh * r
        else:  # BGR NHWC with the pixel stride 4 and rows walked bottom-up
            p, r, off = 4, -(4 * rw + 8), (rh - 1) * (4 * rw + 8) + 2
            size = off + 4 * rw + 1
        buf = cm.store(d, o, rect, p, r, off, size)
        got = np.array([[buf[off + i * p + j * r] for i in range(rw)] for j in range(rh)], dtype=np.uint8)
        assert np.array_equal(got, want), (o, shape, rect)
        touched = np.zeros(size, dtype=bool)
        for j in range(rh):
            for i in range(rw):
                touched[off + i * p + j * r] = True
        assert (buf[~touched] == 0xA5).all(), (o, shape, rect)


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_composition_downscaled_extents(k):
    """the clip rectangle stays inside the decoded extent ceil(W / k) x ceil(H / k) for every orientation and rectangle"""
    rng = np.random.default_rng(k)
    for W, H in [(1, 1), (17, 9), (127, 255), (1920, 1080), (4000, 3000)]:
        w, h = -(-W // k), -(-H // k)
        for o in om.ORIENTATIONS:
            ow, oh = (h, w) if o >= 5 else (w, h)
            for rect in cm.rectangles(ow, oh, rng):
                x0, y0, x1, y1 = cm.crop_to_decoded(o, rect, w, h)
                assert 0 <= x0 < x1 <= w and 0 <= y0 < y1 <= h
                assert (x1 - x0) * (y1 - y0) == rect[2] * rect[3]


def _vectors():
    paths = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg")) + glob.glob(os.path.join(GOLDEN, "*", "*.jpg")))
    return [p for p in paths if "__nimpl" not in p]


def test_output_size(built):
    """b200jpg_output_size for every golden vector and for copies tagged with each Exif orientation, under every downscale, with
    and without the orientation flag: the parse's size, reduced, swapped for 5..8 when the flag applies"""
    from libjpeg_b200 import decoder, native
    checked = 0
    for path in _vectors():
        base = open(path, "rb").read()
        for data in [base] + [om.tag(base, o) for o in (2, 5, 6, 8)]:
            info = native.FrameInfoStruct()
            rc = native.lib.b200jpg_parse(data, len(data), ctypes.byref(info))
            o = native.lib.b200jpg_exif_orientation(data, len(data))
            for k in (1, 2, 4, 8):
                for flag in (False, True):
                    if rc != 0:
                        with pytest.raises(native.NativeError):
                            decoder.output_size(data, downscale=k, exif_orientation=flag)
                        continue
                    hw = (-(-info.height // k), -(-info.width // k))
                    want = hw[::-1] if flag and o >= 5 else hw
                    assert decoder.output_size(data, downscale=k, exif_orientation=flag) == want, (path, k, flag)
                    checked += 1
    assert checked > 0


def test_output_size_arguments(built):
    from libjpeg_b200 import decoder, native
    data = open(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"), "rb").read()
    for bad in (3, 0, True, 2.0):
        with pytest.raises(ValueError):
            decoder.output_size(data, downscale=bad)
    w = ctypes.c_uint32()
    assert native.lib.b200jpg_output_size(data, len(data), 0, ctypes.byref(w), None) == -1024


@pytest.mark.parametrize("crop", [
    [None],                              # one rectangle for two frames
    [None, None, None],
    [None, (0, 0, 1)],                   # three values
    [None, (0, 0, 1, 1, 1)],
    [None, (-1, 0, 4, 4)],               # negative
    [None, (0, 0, 4, -4)],
    [None, (0, 0, 4.0, 4)],              # not an integer
    [None, (0, 0, True, 4)],
    [None, (0, 0, 2 ** 32, 4)],          # does not fit b200jpg_rect
    [None, "abcd"],
])
def test_python_arguments(built, crop, monkeypatch):
    """wrong crop arguments raise ValueError before a context (a device) is created"""
    from libjpeg_b200 import decoder

    def no_device(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(decoder, "Context", no_device)
    data = open(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"), "rb").read()
    with pytest.raises(ValueError):
        decoder.BatchDecoder([data, data], crop=crop)


def test_rect_table(built):
    from libjpeg_b200 import decoder, native
    t = decoder.crop_table([None, (1, 2, 3, 4), np.array([5, 6, 7, 8])], 3)
    assert ctypes.sizeof(native.RectStruct) == 16
    assert [(r.x, r.y, r.width, r.height) for r in t] == [(0, 0, 0, 0), (1, 2, 3, 4), (5, 6, 7, 8)]
