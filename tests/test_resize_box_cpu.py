"""CPU: tests/resize_box_model.py (DESIGN §19) against Pillow 12.2 byte for byte -- boxes as Pillow's C floats, Image.reduce,
reducing_gap, windows -- the table entry point b200jpg_resample_coefficients_box against the model, the host helpers thumbnail_args /
fit_args / resize_center_crop_args against Pillow and torchvision, the stored digests, and BatchDecoder's argument checks."""
import ctypes
import hashlib
import io
import json
import math
import os

import numpy as np
import pytest
from PIL import Image, ImageOps

from tests import resize_box_model as bm
from tests import resize_model as rm

FILTERS = [rm.BOX, rm.BILINEAR, rm.HAMMING, rm.BICUBIC, rm.LANCZOS]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_box")
MODES = {1: "L", 3: "RGB", 4: "CMYK"}

# boxes where rounding to float32 instead of keeping double changes Pillow's output: (w, h, out_w, out_h, filter, box); found by
# searching random boxes whose double and float32 tables differ (test_float_box_vectors checks that they still do)
FLOAT_VECTORS = [
    (49, 8, 32, 4, rm.LANCZOS, (15.629586351596117, 0.0, 36.75323830524287, 8.0)),
    (55, 9, 18, 9, rm.BICUBIC, (32.08653858180356, 0.0, 45.623612120174315, 9.0)),
    (35, 4, 31, 8, rm.HAMMING, (20.53852163861825, 0.0, 32.54347349606651, 4.0)),
    (46, 4, 29, 4, rm.LANCZOS, (7.30237167721243, 0.0, 35.04565260890589, 4.0)),
    (48, 11, 10, 8, rm.LANCZOS, (3.6505239584762545, 0.0, 26.07795787865452, 11.0)),
    (56, 10, 20, 6, rm.HAMMING, (20.010892218199253, 0.0, 24.329977856538136, 10.0)),
]


def _img(h, w, c, seed):
    a = np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
    return a[..., 0] if c == 1 else a


def _pil(a):
    return Image.fromarray(a, MODES[1 if a.ndim == 2 else a.shape[2]])


def _np(im):
    return np.asarray(im)


@pytest.mark.parametrize("resample", FILTERS)
def test_boxes_against_pillow(resample):
    """integer, dyadic and arbitrary double boxes, zero-width boxes, modes L / RGB / CMYK, shrinking and growing"""
    rng = np.random.default_rng(resample)
    for case in range(36):
        c = [1, 3, 4][case % 3]
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        a = _img(h, w, c, 1000 * resample + case)
        kind = case % 4
        if kind == 0:
            x0, x1 = sorted(int(v) for v in rng.integers(0, w + 1, 2))
            y0, y1 = sorted(int(v) for v in rng.integers(0, h + 1, 2))
        elif kind == 1:
            x0, x1 = sorted(float(v) / 8 for v in rng.integers(0, 8 * w + 1, 2))
            y0, y1 = sorted(float(v) / 8 for v in rng.integers(0, 8 * h + 1, 2))
        else:
            x0, x1 = sorted(float(v) for v in rng.uniform(0, w, 2))
            y0, y1 = sorted(float(v) for v in rng.uniform(0, h, 2))
        if case % 9 == 0:
            x1 = x0  # zero width
        box = (x0, y0, x1, y1)
        tw, th = int(rng.integers(1, 2 * w + 3)), int(rng.integers(1, 2 * h + 3))
        want = _np(_pil(a).resize((tw, th), resample, box=box))
        got = bm.resize(a, tw, th, resample, box=box)
        assert np.array_equal(got, want), (case, a.shape, box, tw, th)


def test_float_box_vectors():
    """the stored vectors: float32 boxes give Pillow's bytes, double boxes would not"""
    for w, h, tw, th, resample, box in FLOAT_VECTORS:
        a = _img(h, w, 1, w * h)
        want = _np(_pil(a).resize((tw, th), resample, box=box))
        assert np.array_equal(bm.resize(a, tw, th, resample, box=box), want)
        assert not np.array_equal(bm.resize(a, tw, th, resample, box=box, box_dtype=np.float64), want)


def test_reduce_against_pillow():
    """Image.reduce for every (fx, fy) in 1..8 squared, large and asymmetric factors, partial edges, constant 255 and rounding-edge
    images, with and without a box"""
    rng = np.random.default_rng(5)
    cases = [(fx, fy) for fx in range(1, 9) for fy in range(1, 9)] + [(13, 1), (1, 17), (31, 7), (64, 3), (100, 100), (45, 2)]
    for k, (fx, fy) in enumerate(cases):
        if (fx, fy) == (1, 1):
            continue
        c = [1, 3, 4][k % 3]
        h, w = int(rng.integers(fy, 3 * fy + 5)), int(rng.integers(fx, 3 * fx + 5))
        for a in (_img(h, w, c, k), np.full((h, w, c) if c > 1 else (h, w), 255, np.uint8),
                  np.where(_img(h, w, c, k + 1) > 127, 128, 127).astype(np.uint8)):
            box = None
            if k % 2:
                bx0, by0 = int(rng.integers(0, w // 2 + 1)), int(rng.integers(0, h // 2 + 1))
                box = (bx0, by0, int(rng.integers(bx0 + 1, w + 1)), int(rng.integers(by0 + 1, h + 1)))
            want = _np(_pil(a).reduce((fx, fy), box=box))
            chans = [a] if a.ndim == 2 else [a[..., i] for i in range(c)]
            got = [bm.reduce_channel(ch, fx, fy, box) for ch in chans]
            got = got[0] if a.ndim == 2 else np.stack(got, -1)
            assert np.array_equal(got, want), (fx, fy, a.shape, box)


def test_reduce_multiplier():
    """Pillow's float32 multiplier (2^32 / (256 n), truncated) is floor(2^24 / n) for every block size the batch reduces with"""
    n = np.arange(1, 1 << 24, dtype=np.uint64)
    f = (np.float32(4294967296.0) / (n * 256).astype(np.float32)).astype(np.uint64)
    assert np.array_equal(f, (1 << 24) // n)


@pytest.mark.parametrize("gap", [1.0, 1.5, 2.0, 3.0])
def test_reducing_gap_against_pillow(gap):
    """Image.resize(..., reducing_gap=g) over sizes where the factors are 1, 2 or more, with and without boxes"""
    rng = np.random.default_rng(int(gap * 10))
    for case in range(30):
        c = [1, 3, 4][case % 3]
        resample = FILTERS[case % 5]
        h, w = int(rng.integers(8, 120)), int(rng.integers(8, 120))
        a = _img(h, w, c, case)
        tw, th = max(1, w // int(rng.integers(1, 12))), max(1, h // int(rng.integers(1, 12)))
        box = None
        if case % 2:
            x0, y0 = float(rng.uniform(0, w / 3)), float(rng.uniform(0, h / 3))
            box = (x0, y0, float(rng.uniform(x0 + 1, w)), float(rng.uniform(y0 + 1, h)))
        want = _np(_pil(a).resize((tw, th), resample, box=box, reducing_gap=gap))
        assert np.array_equal(bm.resize(a, tw, th, resample, box=box, gap=gap), want), (case, a.shape, box, tw, th)


def test_window_is_a_crop():
    rng = np.random.default_rng(9)
    for case in range(20):
        a = _img(30, 41, 3, case)
        tw, th = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        x, y = int(rng.integers(0, tw)), int(rng.integers(0, th))
        win = (x, y, int(rng.integers(1, tw - x + 1)), int(rng.integers(1, th - y + 1)))
        box = (1.25, 0.5, 39.75, 29.0)
        want = _np(_pil(a).resize((tw, th), rm.BICUBIC, box=box, reducing_gap=2.0).crop((x, y, x + win[2], y + win[3])))
        assert np.array_equal(bm.resize(a, tw, th, rm.BICUBIC, box=box, gap=2.0, window=win), want)


def test_coefficients_box_entry(built):
    """b200jpg_resample_coefficients_box equals the model's tables; the default box equals b200jpg_resample_coefficients"""
    from libjpeg_b200.native import lib
    rng = np.random.default_rng(3)
    for case in range(60):
        resample = FILTERS[case % 5]
        n_in, n_out = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        in0, in1 = sorted(float(v) for v in rng.uniform(0, n_in, 2))
        if case % 7 == 0:
            in0, in1 = 0.0, float(n_in)
        f0, f1 = float(np.float32(in0)), float(np.float32(in1))
        if f1 > n_in:
            continue
        ks = ctypes.c_uint32()
        assert lib.b200jpg_resample_coefficients_box(n_in, f0, f1, n_out, resample, None, None, 0, ctypes.byref(ks)) == 0
        b = np.zeros(2 * n_out, np.int32)
        k = np.zeros(n_out * ks.value, np.int32)
        assert lib.b200jpg_resample_coefficients_box(n_in, f0, f1, n_out, resample, b.ctypes.data, k.ctypes.data, k.size,
                                                     ctypes.byref(ks)) == 0
        mb, mt, mk = bm.coefficients_box(n_in, f0, f1, n_out, resample)
        assert mk == ks.value
        assert np.array_equal(b.reshape(-1, 2), mb) and np.array_equal(k.reshape(n_out, -1), mt), (n_in, n_out, in0, in1)
        if (in0, in1) == (0.0, float(n_in)):
            b2, k2 = np.zeros_like(b), np.zeros_like(k)
            assert lib.b200jpg_resample_coefficients(n_in, n_out, resample, b2.ctypes.data, k2.ctypes.data, k2.size, ctypes.byref(ks)) == 0
            assert np.array_equal(b, b2) and np.array_equal(k, k2)
    ks = ctypes.c_uint32()
    for in0, in1 in ((-1.0, 2.0), (3.0, 2.0), (0.0, 11.0), (float("nan"), 1.0)):
        assert lib.b200jpg_resample_coefficients_box(10, in0, in1, 4, rm.BILINEAR, None, None, 0, ctypes.byref(ks)) == -1024  # B200JPG_ERR_INVALID_PARAMETER


def _jpeg(w, h, seed, mode="RGB", sub=2, q=80):
    a = _img(h, w, 3 if mode == "RGB" else 1, seed)
    a = np.clip(a.astype(np.int32) // 4 + np.linspace(0, 180, w, dtype=np.int32)[None, :, None] if mode == "RGB" else
                a.astype(np.int32) // 4 + np.linspace(0, 180, w, dtype=np.int32)[None, :], 0, 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(a, mode).save(buf, "JPEG", quality=q, subsampling=sub)
    return buf.getvalue()


def _thumb_model(data, args, gap, exif):
    """the batch's pixels for thumbnail_args: Pillow's own (drafted) decode as C -- the turbo path's pixels, pinned elsewhere --
    then the model"""
    im = Image.open(io.BytesIO(data))
    if args["draft"] is not None:
        dh, dw = args["draft"]
        im.draft(None, (dw, dh))
    if exif:
        im = ImageOps.exif_transpose(im)
    c = np.asarray(im)
    if args["resize"] is None:
        return c
    h, w = args["resize"]
    return bm.resize(c, w, h, rm.BICUBIC, box=args["box"], gap=gap)


@pytest.mark.parametrize("exif", [False, True])
def test_thumbnail_args(exif):
    """thumbnail_args + the model against im.thumbnail() on Pillow-written JPEGs: W mod k != 0, reduce() after a k = 8 draft,
    images already within the size, the drafted size equal to the thumbnail's, grey frames"""
    from libjpeg_b200.decoder import thumbnail_args
    files = [_jpeg(517, 389, 1), _jpeg(1001, 333, 2, sub=0), _jpeg(240, 400, 3, "L", 0), _jpeg(64, 48, 4), _jpeg(800, 600, 5)]
    sizes = [(128, 128), (16, 16), (37, 100), (600, 800), (75, 100), (3, 5), (2000, 2000)]  # (h, w)
    for gap in (2.0, 3.0, None):
        for data in files:
            for h, w in sizes:
                im = Image.open(io.BytesIO(data))
                if exif:
                    im = ImageOps.exif_transpose(im)
                im.thumbnail((w, h), reducing_gap=gap)
                args = thumbnail_args(data, (h, w), reducing_gap=gap, exif_orientation=exif)
                got = _thumb_model(data, args, gap, exif)
                assert np.array_equal(got, np.asarray(im)), (len(data), (h, w), gap, args)


def test_fit_args():
    from libjpeg_b200.decoder import fit_args
    rng = np.random.default_rng(11)
    files = [_jpeg(517, 389, 1), _jpeg(240, 400, 3, "L", 0), _jpeg(333, 90, 6, sub=1)]
    for case in range(24):
        data = files[case % 3]
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        bleed = [0.0, 0.1, 0.37, 0.6, -0.2][case % 5]
        cen = [(0.5, 0.5), (0.0, 1.0), (0.3, 0.8), (1.5, -0.1)][case % 4]
        want = np.asarray(ImageOps.fit(Image.open(io.BytesIO(data)), (w, h), bleed=bleed, centering=cen))
        args = fit_args(data, (h, w), bleed=bleed, centering=cen)
        c = np.asarray(Image.open(io.BytesIO(data)))
        got = bm.resize(c, w, h, rm.BICUBIC, box=args["box"])
        assert args["resize"] == (h, w) and np.array_equal(got, want), (case, args)


def test_resize_center_crop_args():
    import torchvision.transforms as T
    from libjpeg_b200.decoder import resize_center_crop_args
    files = [_jpeg(517, 389, 1), _jpeg(240, 400, 3, "L", 0), _jpeg(333, 90, 6, sub=1), _jpeg(300, 300, 7)]
    for data in files:
        c = np.asarray(Image.open(io.BytesIO(data)))
        for resize, crop in ((256, 224), (100, 77), ((120, 90), (61, 90)), (90, 90), ((50, 333), 50)):
            try:
                args = resize_center_crop_args(data, resize, crop)
            except ValueError:
                with pytest.raises(Exception):  # torchvision pads here; the helper refuses
                    r = T.Resize(resize)(Image.open(io.BytesIO(data)))
                    cc = (crop, crop) if isinstance(crop, int) else crop
                    assert r.size[0] >= cc[1] and r.size[1] >= cc[0]
                continue
            want = np.asarray(T.Compose([T.Resize(resize), T.CenterCrop(crop)])(Image.open(io.BytesIO(data))))
            h, w = args["resize"]
            got = bm.resize(c, w, h, rm.BILINEAR, window=args["window"])
            assert np.array_equal(got, want), (resize, crop, args)


def test_stored_digests():
    """the fixtures' digests are what Pillow and torchvision make of them here, and the helpers + the model give the same"""
    from libjpeg_b200.decoder import fit_args, resize_center_crop_args, thumbnail_args
    with open(os.path.join(GOLDEN, "digests.json")) as f:
        digests = json.load(f)
    for name, chains in digests.items():
        data = open(os.path.join(GOLDEN, name + ".jpg"), "rb").read()
        c = np.asarray(Image.open(io.BytesIO(data)))
        for chain, dig in chains.items():
            parts = chain.split("_")
            if parts[0] == "thumbnail":
                w, h = (int(v) for v in parts[1].split("x"))
                got = _thumb_model(data, thumbnail_args(data, (h, w)), 2.0, False)
            elif parts[0] == "fit":
                w, h = (int(v) for v in parts[1].split("x"))
                args = fit_args(data, (h, w), bleed=float(parts[2]), centering=(float(parts[3]), float(parts[4])))
                got = bm.resize(c, w, h, rm.BICUBIC, box=args["box"])
            else:
                args = resize_center_crop_args(data, 256, 224)
                h, w = args["resize"]
                got = bm.resize(c, w, h, rm.BILINEAR, window=args["window"])
                if got.ndim == 2:
                    got = np.repeat(got[..., None], 3, -1)  # (the chain converts to RGB)
            got = got[..., None] if got.ndim == 2 else got
            assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() + ":%dx%dx%d" % got.shape == dig, (name, chain)


def test_argument_checks(built):
    """BatchDecoder raises ValueError before any device is touched"""
    from libjpeg_b200.decoder import BatchDecoder, box_table, reducing_gap_value
    frames = [b"\xff\xd8", b"\xff\xd8"]
    bad = [dict(box=[(0, 0, 1, 1)]), dict(box=[(0, 0, 1), None]), dict(box=[(0, 0, float("nan"), 1), None]),
           dict(box=[(0, 0, float("inf"), 1), None]), dict(box=[(-1, 0, 1, 1), None]), dict(box=[(2, 0, 1, 1), None]),
           dict(box=[(0, 3, 1, 1), None]), dict(box=[(True, 0, 1, 1), None]), dict(box=["abcd", None]),
           dict(reducing_gap=0.5), dict(reducing_gap=float("nan")), dict(reducing_gap=True), dict(reducing_gap="2"),
           dict(window=[(0, 0, 1, 1)]), dict(window=[(0, 0, 1.5, 1), None]), dict(window=[(-1, 0, 1, 1), None])]
    for kw in bad:
        with pytest.raises(ValueError):
            BatchDecoder(frames, resize=(4, 4), **kw)
    assert reducing_gap_value(None) == 0.0 and reducing_gap_value(1) == 1.0
    t = box_table([None, (0, 0.5, 2, 3.25)], 2)
    assert (t[0].x0, t[0].x1, t[1].y0, t[1].y1) == (0.0, 0.0, 0.5, 3.25)


def test_helper_checks():
    from libjpeg_b200.decoder import fit_args, resize_center_crop_args, thumbnail_args
    data = _jpeg(64, 48, 1)
    for call in (lambda: thumbnail_args(data, (0, 4)), lambda: thumbnail_args(data, (4, 4), reducing_gap=0.5),
                 lambda: fit_args(data, (4,)), lambda: resize_center_crop_args(data, 0, 4),
                 lambda: resize_center_crop_args(data, 32, 40)):
        with pytest.raises(ValueError):
            call()
    assert math.isclose(fit_args(data, (48, 64))["box"][2], 64.0)
