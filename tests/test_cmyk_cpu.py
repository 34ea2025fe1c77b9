"""No device: the CMYK and YCCK conversions of the output modes (DESIGN §15) against Pillow, and the Adobe rules of
b200jpg_colorspace / decoder.colorspace() on spliced segments."""
import io

import numpy as np
import pytest

from tests import cmyk_model as km

GREY, YCBCR, RGB, CMYK, YCCK = "L", "YCbCr", "RGB", "CMYK", "YCCK"


def test_rgb_equals_pillow_on_every_pair():
    """each output channel depends on (s_c, s3) only: a 256 x 256 image holds every pair for each of the three channels"""
    Image = pytest.importorskip("PIL.Image")
    i = np.arange(256)
    sc, s3 = np.meshgrid(i, i, indexing="ij")
    s = np.stack([sc, (sc + 85) % 256, 255 - sc, s3], axis=-1)  # every channel meets every s3
    want = np.asarray(Image.fromarray((255 - s).astype(np.uint8), "CMYK").convert("RGB"))
    assert np.array_equal(km.to_rgb(s, km.CMYK), want)


def test_luma_equals_pillow():
    """2^24 random quadruples and a grid of the edges"""
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(15)
    edges = np.array([0, 1, 2, 127, 128, 129, 253, 254, 255])
    grid = np.stack(np.meshgrid(edges, edges, edges, edges, indexing="ij"), axis=-1).reshape(-1, 4)
    for s in (rng.integers(0, 256, (4096, 4096, 4)), grid.reshape(1, -1, 4)):
        want = np.asarray(Image.fromarray((255 - s).astype(np.uint8), "CMYK").convert("L"))
        assert np.array_equal(km.luma(km.to_rgb(s, km.CMYK)), want)


def _pillow_cmyk(pixels, **kw):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(pixels, "CMYK").save(buf, "JPEG", **kw)
    return buf.getvalue()


def _with_transform(data, t):
    """the transform byte of the file's Adobe segment (Pillow writes it behind SOI) set to t"""
    at = data.find(b"\xff\xee")
    assert at >= 0 and data[at + 4:at + 9] == b"Adobe" and data[at + 4 + 11] == 0
    return data[:at + 4 + 11] + bytes([t]) + data[at + 4 + 12:]


@pytest.mark.parametrize("w,h,quality,subsampling,rows", [(64, 48, 90, 0, 0), (97, 61, 75, 2, 0), (123, 45, 80, 0, 1),
                                                          (40, 72, 85, 2, 2), (301, 17, 95, 0, 0), (16, 16, 50, 2, 1)])
def test_ycck_step_on_libjpeg(w, h, quality, subsampling, rows):
    """libjpeg decodes a YCCK file as the model's YCC step applied to the CMYK decode of the same coefficients, exactly: Pillow's
    decode of the file with the transform byte patched equals the model on 255 - Pillow's decode of the original"""
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(w * h)
    px = np.clip(rng.normal(128, 70, (h, w, 4)), 0, 255).astype(np.uint8)
    kw = dict(quality=quality, subsampling=subsampling)
    if rows:
        kw["restart_marker_rows"] = rows
    data = _pillow_cmyk(px, **kw)
    assert (b"\xff\xdd" in data) == bool(rows)
    s = 255 - np.asarray(Image.open(io.BytesIO(data))).astype(np.int64)  # the samples as libjpeg decodes them
    rgb = km.ycc_to_rgb(s[..., 0], s[..., 1], s[..., 2])
    want = np.stack(rgb + [255 - s[..., 3]], axis=-1)  # libjpeg's C = 255 - R, inverted again by Pillow; K untouched
    for t in (1, 2, 255):
        got = np.asarray(Image.open(io.BytesIO(_with_transform(data, t))))
        assert np.array_equal(got, want), t
        # and so Pillow's RGB of the YCCK file is the model's, from the same samples
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(_with_transform(data, t))).convert("RGB")), km.to_rgb(s, km.YCCK))


def _colorspace(data):
    from libjpeg_b200 import decoder
    return decoder.colorspace(data)


def _info(data):
    from libjpeg_b200 import decoder
    return decoder.parse(data)


def test_adobe_rules(built):
    four = km.four_component(64, 48, 1)
    assert _info(four).ncomp == 4 and _colorspace(four) is None
    cases = [
        (km.after_soi(four, km.adobe(0)), CMYK),                          # in front of the frame header
        (km.after_soi(four, km.adobe(2)), YCCK),
        (km.before_sos(four, km.adobe(0)), CMYK),                         # between the frame header and the first scan
        (km.before_sos(four, km.adobe(1)), YCCK),
        (km.before_sos(four, km.adobe(255)), YCCK),
        (km.before_sos(four, km.adobe(0), k=1), None),                    # behind the first scan: ignored
        (km.before_sos(km.after_soi(four, km.adobe(2)), km.adobe(0), k=2), YCCK),
        (km.after_soi(four, km.adobe(0, payload=11)), None),              # a payload too short
        (km.after_soi(four, km.adobe(0, payload=40)), CMYK),              # longer is fine
        (km.after_soi(four, km.adobe(0, tag=b"Adobf")), None),            # not the tag
        (km.after_soi(four, km.adobe(0, tag=b"adobe")), None),
        (km.before_sos(km.after_soi(four, km.adobe(0)), km.adobe(2)), YCCK),  # the last one in front of the first scan counts
        (km.before_sos(km.after_soi(four, km.adobe(2)), km.adobe(0)), CMYK),
        (km.after_soi(km.after_soi(four, km.adobe(0, payload=11)), km.adobe(2)), YCCK),  # a short one behind a valid one: no effect
        (km.after_soi(km.deep12_four(), km.adobe(0)), None),             # 12-bit four-component frames
        (km.after_soi(km.deep12_four(), km.adobe(2)), None),
    ]
    deep = km.deep12_four()
    for k, (data, want) in enumerate(cases):
        assert _colorspace(data) == want, k
        info = _info(data)  # parses as before, with the same frame info
        assert info == _info(four if info.precision == 8 else deep), k


@pytest.mark.parametrize("sub", [(1, 1), (2, 2), (2, 1), (1, 2)])
def test_adobe_rules_per_sampling(built, sub):
    four = km.four_component(97, 61, 2, sub, restart=3)
    for t, want in ((0, CMYK), (2, YCCK)):
        assert _colorspace(km.after_soi(four, km.adobe(t))) == want
        assert _colorspace(km.before_sos(four, km.adobe(t), k=1)) is None


def test_one_and_three_components_follow_ycbcr(built):
    """grey frames are "L"; three-component frames are "YCbCr" exactly where the parser sets ycbcr, Adobe segments or not"""
    import glob
    import os
    from tests.test_mode_cpu import GOLDEN
    paths = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg")) + glob.glob(os.path.join(GOLDEN, "*", "*.jpg")))
    checked = 0
    for path in paths:
        data = open(path, "rb").read()
        for d in (data, km.after_soi(data, km.adobe(0)), km.after_soi(data, km.adobe(1)), km.before_sos(data, km.adobe(0), k=0)):
            try:
                fi = _info(d)
            except Exception:
                continue
            cs = _colorspace(d)
            if fi.ncomp == 1:
                assert cs == GREY, path
            elif fi.ncomp == 3:
                assert cs == (YCBCR if fi.ycbcr else RGB), path
            else:
                continue
            checked += 1
    assert checked > 100


def test_fixtures_are_pillow_cmyk(built):
    """the files of tests/golden/cmyk: Pillow's CMYK files are "CMYK", their twins "YCCK"; the stored conversions are Pillow's"""
    import glob
    import os
    from tests.test_mode_cpu import GOLDEN
    paths = sorted(glob.glob(os.path.join(GOLDEN, "cmyk", "*.jpg")))
    assert len(paths) == 8
    expected = np.load(os.path.join(GOLDEN, "cmyk", "expected.npz"))
    Image = pytest.importorskip("PIL.Image")
    for path in paths:
        name = os.path.basename(path)[:-4]
        data = open(path, "rb").read()
        assert _colorspace(data) == (CMYK if name.startswith("cmyk") else YCCK)
        im = Image.open(io.BytesIO(data))
        assert np.array_equal(np.asarray(im.convert("RGB")), expected[name + "_RGB"])
        assert np.array_equal(np.asarray(im.convert("L")), expected[name + "_L"])


def test_colorspace_errors(built):
    from libjpeg_b200 import decoder
    with pytest.raises(built.native.NativeError):
        decoder.colorspace(b"\xff\xd8\xff\xd9")
    assert built.native.COLORSPACES == [None, GREY, YCBCR, RGB, CMYK, YCCK]
