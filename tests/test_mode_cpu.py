"""No device: the output modes' definitions (DESIGN §14) against Pillow -- the L formula on every RGB triple, grey replication,
resizing that commutes with replication -- and the host side of BatchDecoder(mode=...) and b200jpg_output_size."""
import ctypes
import glob
import os

import numpy as np
import pytest

from tests import resize_model as rm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FLAG_OUTPUT_RGB, FLAG_OUTPUT_L = 0x20, 0x40


def luma(rgb):
    """B200JPG_FLAG_OUTPUT_L of clamped R, G, B samples (last axis), in int64: PIL's L24, libjpeg's rgb_gray_convert"""
    rgb = rgb.astype(np.int64)
    return (19595 * rgb[..., 0] + 38470 * rgb[..., 1] + 7471 * rgb[..., 2] + 32768) >> 16


def test_luma_equals_pillow_on_every_triple():
    Image = pytest.importorskip("PIL.Image")
    i = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    want = np.asarray(Image.fromarray(rgb, "RGB").convert("L"))
    assert np.array_equal(luma(rgb), want)


def test_luma_fits_int32_for_12_bit_samples():
    top = luma(np.array([4095, 4095, 4095]))
    assert top == 4095 and 19595 * 4095 + 38470 * 4095 + 7471 * 4095 + 32768 < 2 ** 31


def test_replication_equals_pillow():
    Image = pytest.importorskip("PIL.Image")
    g = np.random.default_rng(3).integers(0, 256, (37, 53), dtype=np.uint8)
    want = np.asarray(Image.fromarray(g, "L").convert("RGB"))
    assert np.array_equal(np.repeat(g[..., None], 3, axis=-1), want)


@pytest.mark.parametrize("resample", [rm.BOX, rm.BILINEAR, rm.HAMMING, rm.BICUBIC, rm.LANCZOS])
def test_resize_commutes_with_replication(resample):
    """mode -> resize (the batch's order) equals resize -> replication: Pillow resizes every channel on its own"""
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(resample)
    for h, w, th, tw in [(40, 24, 17, 33), (97, 53, 224, 224), (5, 300, 5, 17), (224, 224, 224, 224)]:
        g = rng.integers(0, 256, (h, w), dtype=np.uint8)
        rgb = np.repeat(g[..., None], 3, axis=-1)
        resized = rm.resize(rgb, tw, th, resample)
        assert np.array_equal(resized, np.repeat(rm.resize(g, tw, th, resample)[..., None], 3, axis=-1))
        assert np.array_equal(resized, np.asarray(Image.fromarray(rgb, "RGB").resize((tw, th), resample)))


def test_python_arguments(built):
    """ValueError before any device is touched"""
    from libjpeg_b200.decoder import BatchDecoder
    for mode in ["rgb", "l", "LA", "CMYK", "YCbCr", 1, True, b"RGB", ("RGB",)]:
        with pytest.raises(ValueError):
            BatchDecoder([b"\xff\xd8"], mode=mode)
    assert built.native.MODE_FLAGS == {None: 0, "RGB": FLAG_OUTPUT_RGB, "L": FLAG_OUTPUT_L}


def test_output_size_ignores_the_mode(built):
    """b200jpg_output_size with a mode bit gives the (h, w) it gives without it, for every golden vector"""
    lib = built.native.lib
    paths = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg")) + glob.glob(os.path.join(GOLDEN, "*", "*.jpg")))
    assert len(paths) > 40
    checked = 0
    for path in paths:
        data = open(path, "rb").read()
        for base in (0, 0x4, 0x8, 0xC, 0x10, 0x14):
            got = []
            for mode in (0, FLAG_OUTPUT_RGB, FLAG_OUTPUT_L):
                w, h = ctypes.c_uint32(), ctypes.c_uint32()
                rc = lib.b200jpg_output_size(data, len(data), base | mode, ctypes.byref(w), ctypes.byref(h))
                got.append((rc, w.value, h.value))
            assert got[1] == got[0] and got[2] == got[0], (path, base, got)
            checked += got[0][0] == 0
    assert checked > 200
