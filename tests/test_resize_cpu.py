"""No device: the resize model (tests/resize_model.py) against Pillow's Image.resize byte for byte, the library's host tables
(b200jpg_resample_coefficients) against the model, and the argument checks of BatchDecoder(resize=..., resample=...)."""
import ctypes

import numpy as np
import pytest

from tests import resize_model as rm

FILTERS = [rm.BOX, rm.BILINEAR, rm.HAMMING, rm.BICUBIC, rm.LANCZOS]


def _cases():
    """(w, h, W_t, H_t, binary) over seeded sizes: shrinking, growing, one axis unchanged, target = source, 1 x 1 <-> N"""
    rng = np.random.default_rng(13)
    cases = []
    for k in range(60):
        w, h = int(rng.integers(1, 121)), int(rng.integers(1, 121))
        tw, th = int(rng.integers(1, 121)), int(rng.integers(1, 121))
        if k % 6 == 1:
            tw = w
        elif k % 6 == 2:
            th = h
        elif k % 6 == 3:
            tw, th = w, h
        cases.append((w, h, tw, th, k % 4 == 0))
    cases += [(1, 1, 57, 33, False), (57, 33, 1, 1, False), (1, 1, 1, 1, False), (1, 90, 7, 1, True), (90, 1, 1, 7, True),
              (300, 2000, 224, 37, False)]
    return cases


def _image(rng, h, w, binary, channels=None):
    shape = (h, w) if channels is None else (h, w, channels)
    if binary:  # 0 / 255 edges: the negative lobes push the sums past both ends of the clamp
        return (rng.integers(0, 2, shape) * 255).astype(np.uint8)
    return rng.integers(0, 256, shape, dtype=np.uint8)


@pytest.mark.parametrize("resample", FILTERS)
def test_model_equals_pillow(resample):
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(resample)
    for w, h, tw, th, binary in _cases():
        img = _image(rng, h, w, binary)
        want = np.asarray(Image.fromarray(img, "L").resize((tw, th), resample))
        assert np.array_equal(rm.resize(img, tw, th, resample), want), (w, h, tw, th, binary)


@pytest.mark.parametrize("resample", FILTERS)
def test_model_equals_pillow_4k_to_224(resample):
    Image = pytest.importorskip("PIL.Image")
    img = _image(np.random.default_rng(40 + resample), 2160, 3840, False)
    want = np.asarray(Image.fromarray(img, "L").resize((224, 224), resample))
    assert np.array_equal(rm.resize(img, 224, 224, resample), want)


@pytest.mark.parametrize("mode,channels", [("L", None), ("RGB", 3), ("CMYK", 4)])
def test_modes_are_the_per_channel_model(mode, channels):
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(7)
    for resample in FILTERS:
        for w, h, tw, th, binary in [(97, 41, 31, 60, False), (40, 90, 123, 17, True), (64, 48, 64, 11, False)]:
            img = _image(rng, h, w, binary, channels)
            want = np.asarray(Image.fromarray(img, mode).resize((tw, th), resample))
            got = rm.resize(img, tw, th, resample)
            assert np.array_equal(got, want), (mode, resample, w, h, tw, th)
            if channels:
                for c in range(channels):
                    assert np.array_equal(got[..., c], rm.resize_channel(img[..., c], tw, th, resample))


def test_tall_image_deviation():
    """Pillow's Image.resize runs the vertical pass first when the source is taller than 100 x its width and the height shrinks;
    R always runs horizontal then vertical, which is what Pillow's resampler itself does in one call"""
    Image = pytest.importorskip("PIL.Image")
    img = _image(np.random.default_rng(3), 400, 3, False)
    im = Image.fromarray(img, "L")
    for resample in FILTERS:
        got = rm.resize(img, 2, 37, resample)
        one_call = np.asarray(im._new(im.im.resize((2, 37), resample, (0, 0, 3, 400))))
        assert np.array_equal(got, one_call), resample
    differs = [not np.array_equal(rm.resize(img, 2, 37, f), np.asarray(im.resize((2, 37), f))) for f in FILTERS]
    assert any(differs)


def _library_tables(built, in_size, out_size, resample):
    lib = built.native.lib
    ks = ctypes.c_uint32()
    assert lib.b200jpg_resample_coefficients(in_size, out_size, resample, None, None, 0, ctypes.byref(ks)) == 0
    bounds = np.zeros(2 * out_size, dtype=np.int32)
    table = np.zeros(out_size * ks.value, dtype=np.int32)
    assert lib.b200jpg_resample_coefficients(in_size, out_size, resample, bounds.ctypes.data, table.ctypes.data, table.size,
                                             ctypes.byref(ks)) == 0
    return bounds.reshape(out_size, 2), table.reshape(out_size, ks.value), ks.value


@pytest.mark.parametrize("resample", FILTERS)
def test_library_tables_equal_the_model(built, resample):
    sizes = set()
    for w, h, tw, th, _ in _cases():
        sizes |= {(w, tw), (h, th)}
    sizes |= {(3840, 224), (2160, 224), (2000, 1), (1, 2000), (65535, 1), (1, 65535), (300, 17)}
    for in_size, out_size in sorted(sizes):
        bounds, table, ks = _library_tables(built, in_size, out_size, resample)
        want_b, want_t, want_ks = rm.coefficients(in_size, out_size, resample)
        assert ks == want_ks, (in_size, out_size)
        assert np.array_equal(bounds, want_b), (in_size, out_size)
        assert np.array_equal(table, want_t), (in_size, out_size)
        assert rm.int32_bound_ok(table), (in_size, out_size)


def test_library_tables_refused(built):
    lib = built.native.lib
    ks = ctypes.c_uint32()
    for args in [(0, 5, rm.BILINEAR), (5, 0, rm.BILINEAR), (5, 5, 0), (5, 5, 6)]:
        assert lib.b200jpg_resample_coefficients(*args, None, None, 0, ctypes.byref(ks)) == -1024, args
    assert lib.b200jpg_resample_coefficients(9, 4, rm.BILINEAR, None, None, 0, None) == -1024
    b, t = np.zeros(8, dtype=np.int32), np.zeros(100, dtype=np.int32)
    assert lib.b200jpg_resample_coefficients(9, 4, rm.BILINEAR, b.ctypes.data, t.ctypes.data, 4, ctypes.byref(ks)) == -1024


def test_python_arguments(built):
    """ValueError before any device is touched"""
    from libjpeg_b200.decoder import BatchDecoder
    frames = [b"\xff\xd8", b"\xff\xd8"]
    bad = [dict(resize=[(1, 1)]), dict(resize=[(1, 1)] * 3), dict(resize=(1.0, 2)), dict(resize=[(1, 2), (3, "4")]),
           dict(resize=[(1, 2), (3,)]), dict(resize=[(1, 2), 5]), dict(resize=(-1, 2)), dict(resize=[None, (2, -3)]),
           dict(resize=(0, 5)), dict(resize=[(5, 0), None]), dict(resize=(2 ** 32, 1)), dict(resize=(True, 2)),
           dict(resize=(4, 4), resample="nearest"), dict(resample="Bilinear"), dict(resample=2)]
    for kw in bad:
        with pytest.raises(ValueError):
            BatchDecoder(frames, **kw)
    from libjpeg_b200 import decoder
    t = decoder.resize_table((224, 300), 2)
    assert [(t[i].width, t[i].height) for i in range(2)] == [(300, 224)] * 2
    t = decoder.resize_table([None, (0, 0)], 2)
    assert [(t[i].width, t[i].height) for i in range(2)] == [(0, 0)] * 2
    assert [decoder.resample_filter(n) for n in ("lanczos", "bilinear", "bicubic", "box", "hamming")] == [1, 2, 3, 4, 5]
