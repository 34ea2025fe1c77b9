"""GPU: BatchDecoder(hflip=..., vflip=...) / b200jpg_batch_create_flip (DESIGN §21). The oracle is the same batch without the
flips, flipped by numpy (tests/flip_model.py), byte for byte; statuses, shapes and Exif orientations are those of the unflipped
batch, and nothing outside a frame's slot or destination is written. The end-to-end test holds the batch to Pillow and
torchvision's hflip of the training crop."""
import ctypes
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import flip_model as fm
from tests import orientation_model as om
from tests.test_crop import CROP_SETS
from tests.test_decode_into import GOLDEN, SETS, _read
from tests.test_orientation import _batch, _decode, _images, _synth, _view_as_int

pytestmark = pytest.mark.gpu

SENT = 0xA5
FLIPS = range(4)
TURBO = "libjpeg-turbo"
PIL_FILTERS = ["box", "bilinear", "hamming", "bicubic", "lanczos"]
CV_FILTERS = ["cv2-linear", "cv2-area"]
CMYK_DIR = os.path.join(GOLDEN, "cmyk")


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _flip_args(flips):
    return {"hflip": [bool(f & fm.H) for f in flips], "vflip": [bool(f & fm.V) for f in flips]}


def _slots_untouched(dec, out):
    mask = np.ones(out.numel(), dtype=bool)
    for j in range(dec.n):
        mask[dec.out_offset(j):dec.out_offset(j) + dec.frame_bytes(j)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"


def _check(built, ctx, frames, per_frame=None, **kw):
    """every frame four times, under each flip (per_frame: lists of per-frame arguments, repeated with the frames): decode() of the
    flipped batch is decode() of the unflipped one flipped"""
    batch = [f for f in frames for _ in FLIPS]
    flips = [f for _ in frames for f in FLIPS]
    rep = {k: [v for v in vals for _ in FLIPS] for k, vals in (per_frame or {}).items()}
    plain = _batch(built, ctx, batch, **kw, **rep)
    ref = _images(plain, _decode(plain))
    dec = _batch(built, ctx, batch, **_flip_args(flips), **kw, **rep)
    out = _decode(dec)
    got = _images(dec, out)
    live = 0
    for j, f in enumerate(flips):
        assert dec.status(j) == plain.status(j), "frame %d" % j
        assert dec.orientation(j) == plain.orientation(j)
        want = fm.flip(ref[j], f)
        if want is None:
            assert got[j] is None
            continue
        if isinstance(want, list):
            for c, (g, w) in enumerate(zip(got[j], want)):
                assert np.array_equal(g, w), "frame %d (flip %d) component %d" % (j, f, c)
        else:
            assert dec.output_shape(j, 0) == plain.output_shape(j, 0)
            assert np.array_equal(got[j], want), "frame %d (flip %d)" % (j, f)
        assert dec.frame_bytes(j) == plain.frame_bytes(j)
        live += 1
    assert live > 0
    _slots_untouched(dec, out)
    return plain, dec


# (every 12-bit frame is B200JPG_ERR_NOT_IMPLEMENTED under libjpeg-turbo's reconstruction: that batch has no live frame)
@pytest.mark.parametrize("name,reconstruction", [(n, r) for n in CROP_SETS for r in ("reference", TURBO) if (n, r) != ("deep12", TURBO)])
def test_sets(built, ctx, name, reconstruction):
    """every frame set (golden, progressive, 3x / 4x factors, restart-less, 12-bit, damaged, JPEG XT, hand-built, synthetic)"""
    _check(built, ctx, CROP_SETS[name](), reconstruction=reconstruction)


@pytest.mark.parametrize("exif", [False, True])
def test_orientations(built, ctx, exif):
    """all eight Exif orientations under every flip, applied or not: the flip composes with the orientation"""
    frames = [_synth(97, 61, 1), _synth(64, 40, 2, (1, 1)), _synth(50, 70, 3, (2, 1))] + SETS["baseline"]()[:2] + SETS["deep12"]()[:1]
    _check(built, ctx, [om.tag(f, o) for f in frames for o in om.ORIENTATIONS], exif_orientation=exif)


@pytest.mark.parametrize("reconstruction", ["reference", TURBO])
def test_crops(built, ctx, reconstruction):
    """seeded rectangles (tile seams, corners, single rows and columns) of oriented frames: the rectangle is mirrored in the plan"""
    from libjpeg_b200.decoder import output_size
    rng = np.random.default_rng(5)
    src = [om.tag(_synth(600, 301, 11), 6), om.tag(_synth(333, 517, 12, (1, 1)), 2), _synth(300, 200, 13, (2, 1))] + SETS["baseline"]()[:3]
    frames, rects = [], []
    for f in src:
        oh, ow = output_size(f, exif_orientation=True)
        for r in cm.rectangles(ow, oh, rng, n_random=3):
            frames.append(f), rects.append(r)
    _check(built, ctx, frames, {"crop": rects}, exif_orientation=True, reconstruction=reconstruction)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_downscale(built, ctx, k):
    frames = SETS["baseline"]() + SETS["deep12"]() + SETS["subsampling"]() + [_synth(1000, 333, 7), _synth(333, 1000, 8, (1, 1))]
    _check(built, ctx, [om.tag(f, 5) for f in frames[:3]] + frames, downscale=k, exif_orientation=True)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_draft(built, ctx, k):
    frames = [_synth(800, 600, 14), _synth(517, 300, 15, (2, 1)), _synth(300, 517, 16, (1, 1))] + SETS["baseline"]()[:3]
    drafts = [(-(-600 // k), -(-800 // k)), (-(-300 // k), -(-517 // k)), (-(-517 // k), -(-300 // k))] + [(8, 8)] * 3
    _check(built, ctx, frames, {"draft": drafts}, reconstruction=TURBO, mode="RGB")


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("reconstruction", ["reference", TURBO])
def test_modes(built, ctx, mode, reconstruction):
    """grey frames replicated, luma alone, RGB-coded and CMYK / YCCK frames under the output modes"""
    cmyk = [_read(os.path.join(CMYK_DIR, f)) for f in sorted(os.listdir(CMYK_DIR)) if f.endswith(".jpg")][:6]
    frames = SETS["baseline"]() + [om.tag(_synth(120, 70, 17), 7)] + cmyk
    _check(built, ctx, frames, mode=mode, reconstruction=reconstruction, exif_orientation=True)


@pytest.mark.parametrize("mode", ["no_color", "no_upsample", "no_upsample_k2"])
def test_flags(built, ctx, mode):
    """upsample=False: every plane flipped at its own extent"""
    frames = SETS["baseline"]() + SETS["subsampling"]() + SETS["deep12"]() + [om.tag(_synth(97, 61, 18), 8)]
    kw = {"no_color": {"color_transform": False}, "no_upsample": {"upsample": False},
          "no_upsample_k2": {"upsample": False, "downscale": 2}}[mode]
    _check(built, ctx, frames, exif_orientation=True, **kw)


def _resize_cases(frames, resample, rng, exif):
    """per frame a size, and with Pillow's filters a box; a window on every other frame"""
    from libjpeg_b200.decoder import output_size
    sizes, boxes, wins = [], [], []
    for j, f in enumerate(frames):
        h, w = output_size(f, exif_orientation=exif)
        th, tw = int(rng.integers(1, 2 * h + 2)), int(rng.integers(1, 2 * w + 2))
        if j % 3 == 0:
            th, tw = max(1, h // 3), max(1, w // 4)
        sizes.append((th, tw))
        box = None
        if resample in PIL_FILTERS and j % 2 == 1:
            x0, y0 = float(rng.uniform(0, w / 3)), float(rng.uniform(0, h / 3))
            box = (x0, y0, float(rng.uniform(x0, w)), float(rng.uniform(y0, h)))
        boxes.append(box)
        win = None
        if j % 2 == 0:
            x, y = int(rng.integers(0, tw)), int(rng.integers(0, th))
            win = (x, y, int(rng.integers(1, tw - x + 1)), int(rng.integers(1, th - y + 1)))
        wins.append(win)
    return sizes, boxes, wins


@pytest.mark.parametrize("reconstruction", ["reference", TURBO])
@pytest.mark.parametrize("resample", PIL_FILTERS + CV_FILTERS)
def test_resize(built, ctx, resample, reconstruction):
    """resized frames (sizes, boxes, windows, a reducing_gap with Pillow's filters, oriented frames): the resample pass stores
    mirrored, behind the resize"""
    rng = np.random.default_rng(PIL_FILTERS.index(resample) if resample in PIL_FILTERS else 9 + CV_FILTERS.index(resample))
    frames = [_synth(700, 301, 19), om.tag(_synth(301, 700, 20, (1, 1)), 6), _synth(500, 260, 21, (2, 1)), om.tag(_synth(99, 45, 22), 3)]
    frames += SETS["baseline"]()[:4] + SETS["subsampling"]()[:2]
    sizes, boxes, wins = _resize_cases(frames, resample, rng, True)
    per_frame = {"resize": sizes, "window": wins}
    kw = {"exif_orientation": True, "reconstruction": reconstruction, "resample": resample}
    if resample in PIL_FILTERS:
        per_frame["box"] = boxes
        kw["reducing_gap"] = 2.0 if resample in ("bilinear", "lanczos") else None
    _check(built, ctx, frames, per_frame, **kw)


def test_resize_modes_and_crops(built, ctx):
    """grey frames replicated by the resample pass, CMYK frames and a crop in front of the resize"""
    cmyk = [_read(os.path.join(CMYK_DIR, f)) for f in sorted(os.listdir(CMYK_DIR)) if f.endswith(".jpg")][:4]
    frames = SETS["baseline"]() + cmyk
    from libjpeg_b200.decoder import output_size
    rects = []
    for f in frames:
        h, w = output_size(f)
        rects.append((w // 5, h // 7, max(1, w - w // 5 - 1), max(1, h - h // 7 - 2)))
    for resample in ("bicubic", "cv2-area"):
        _check(built, ctx, frames, {"crop": rects}, resize=(37, 53), resample=resample, mode="RGB", reconstruction=TURBO)


def test_tolerant_mixed_batch(built, ctx):
    """flipped and unflipped, damaged, unparseable and 12-bit frames, resized and not, in one tolerant batch"""
    frames = [b"\xff\xd8\xff\xd9", _synth(300, 200, 23), _read(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"))]
    frames += SETS["damaged"]()[:4] + SETS["deep12"]()[:1] + [_synth(64, 48, 24, (1, 1))]
    _check(built, ctx, frames)
    sizes = [None if j % 2 else (21, 33) for j in range(len(frames))]
    _check(built, ctx, frames, {"resize": sizes})


def _launches(dec):
    out = _decode(dec)
    return dec.launches, out.cpu().numpy()


def test_launches(built, ctx):
    """no flip, hflip=None and all-False flips are the batch without flips: same launches and bytes; a flipped resized batch
    issues the launches of the unflipped one"""
    frames = [_synth(300, 200, 25), _synth(97, 61, 26, (1, 1)), om.tag(_synth(120, 70, 27), 6)] + SETS["baseline"]()[:3]
    n = len(frames)
    for kw in ({}, {"resize": (64, 48)}, {"exif_orientation": True, "crop": [(1, 2, 20, 10)] * n}):
        n0, b0 = _launches(_batch(built, ctx, frames, **kw))
        for flips in ({"hflip": None, "vflip": None}, {"hflip": False}, {"hflip": [False] * n, "vflip": False}):
            n1, b1 = _launches(_batch(built, ctx, frames, **flips, **kw))
            assert n1 == n0 and np.array_equal(b1, b0), (kw, flips)
    n0, _ = _launches(_batch(built, ctx, frames, resize=(64, 48)))
    for flips in ({"hflip": True}, {"vflip": [j % 2 == 0 for j in range(n)]}, {"hflip": True, "vflip": True}):
        n1, _ = _launches(_batch(built, ctx, frames, resize=(64, 48), **flips))
        assert n1 == n0, flips


def test_exif_mirror_undone_keeps_the_upright_group(built, ctx):
    """Exif 2 with hflip (and 4 with vflip) is orientation 1: those frames launch as the upright batch does"""
    src = [_synth(300, 200, 28), _synth(97, 61, 29, (1, 1))]
    up = _batch(built, ctx, src, exif_orientation=True)
    n0, b0 = _launches(up)
    dec = _batch(built, ctx, [om.tag(src[0], 2), om.tag(src[1], 4)], exif_orientation=True, hflip=[True, False], vflip=[False, True])
    n1, b1 = _launches(dec)
    assert n1 == n0 and np.array_equal(b1, b0)
    assert [dec.orientation(i) for i in range(2)] == [2, 4]


def _dst(n, oh, ow, dtype, layout):
    import torch
    esz = torch.empty(0, dtype=dtype).element_size()
    if layout == "nchw":
        full = torch.full((n * 3 * oh * ow * esz,), SENT, dtype=torch.uint8, device="cuda").view(dtype).view(n, 3, oh, ow)
        region = (slice(None),) * 4
        return full, region, full
    if layout == "padded":
        full = torch.full((n * 3 * (oh + 2) * (ow + 3) * esz,), SENT, dtype=torch.uint8, device="cuda").view(dtype).view(n, 3, oh + 2, ow + 3)
        region = (slice(None), slice(None), slice(1, oh + 1), slice(1, ow + 1))
        return full, region, full[region]
    full = torch.full((n * (oh + 1) * (ow + 2) * 4 * esz,), SENT, dtype=torch.uint8, device="cuda").view(dtype).view(n, oh + 1, ow + 2, 4)
    region = (slice(None), slice(0, oh), slice(1, ow + 1), slice(0, 3))
    return full, region, full[region].permute(0, 3, 1, 2)


@pytest.mark.parametrize("path", ["resized", "cropped"])
def test_destinations(built, ctx, path):
    """decode_into uint8 NCHW / NHWC / padded and float16 with a map: the flipped batch writes the unflipped batch's tensor
    flipped, and nothing outside the samples"""
    import torch
    src = [_synth(333, 201, 30, (2, 2)), _synth(333, 201, 31, (1, 1)), om.tag(_synth(201, 333, 32, (2, 1)), 6)]
    frames = [f for f in src for _ in FLIPS]
    flips = [f for _ in src for f in FLIPS]
    oh, ow = 45, 77
    kw = {"exif_orientation": True}
    if path == "resized":
        kw.update(resize=(61, 90), window=[(3, 5, ow, oh)] * len(frames), resample="bicubic")
    else:
        kw.update(crop=[(7, 9, ow, oh)] * len(frames))
    plain = _batch(built, ctx, frames, **kw)
    dec = _batch(built, ctx, frames, **_flip_args(flips), **kw)
    n = len(frames)
    ref = torch.empty((n, 3, oh, ow), dtype=torch.uint8, device="cuda")
    plain.decode_into(ref)
    torch.cuda.synchronize()
    want_u8 = torch.stack([torch.flip(ref[j], [d for d, b in ((2, fm.H), (1, fm.V)) if f & b]) for j, f in enumerate(flips)])
    scale, bias = [1 / 58.4, 1 / 57.1, 1 / 57.4], [-2.1, -2.0, -1.8]
    for dtype, layout in [(torch.uint8, "nchw"), (torch.uint8, "padded"), (torch.uint8, "nhwc"), (torch.float16, "nchw"),
                          (torch.float16, "nhwc")]:
        full, region, dst = _dst(n, oh, ow, dtype, layout)
        if dtype == torch.uint8:
            dec.decode_into(dst)
            want = want_u8
        else:
            dec.decode_into(dst, scale=scale, bias=bias)
            want = (want_u8.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) +
                    torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
        torch.cuda.synchronize()
        assert torch.equal(_view_as_int(dst), _view_as_int(want)), (dtype, layout)
        mask = torch.ones(full.shape, dtype=torch.bool, device="cuda")
        mask[region] = False
        esz = full.element_size()
        sent = int(np.frombuffer(bytes([SENT] * esz), dtype={1: np.uint8, 2: np.int16}[esz])[0])
        assert bool((_view_as_int(full)[mask] == sent).all()), (dtype, layout)


def _create(ctx, frames, flips, tolerate=0):
    from libjpeg_b200 import native
    n = len(frames)
    ptrs = (ctypes.c_void_p * n)(*[ctypes.cast(ctypes.c_char_p(f), ctypes.c_void_p).value for f in frames])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    ft = None if flips is None else (ctypes.c_uint8 * n)(*flips)
    handle = ctypes.c_void_p()
    rc = native.lib.b200jpg_batch_create_flip(ctx.handle, ptrs, lens, n, tolerate, 0, None, None, None, None, None, 0, 0.0, ft,
                                              ctypes.byref(handle))
    msg = native.last_error(ctx.handle)[1]
    if rc == 0:
        native.lib.b200jpg_batch_destroy(handle)
    return rc, msg


def test_refused(built, ctx):
    """a flip entry with another bit fails the call with INVALID_PARAMETER naming the frame, tolerate_bad or not; the flip of a
    frame that fails to parse is ignored"""
    frames = [_synth(64, 48, 33), _synth(64, 48, 34)]
    for tolerate in (0, 1):
        for bad in (4, 8, 0x80, 0xFF):
            rc, msg = _create(ctx, frames, [1, bad], tolerate)
            assert rc == -1024 and "frame 1" in msg, (rc, msg)
    assert _create(ctx, frames, None)[0] == 0
    assert _create(ctx, frames, [3, 0])[0] == 0
    assert _create(ctx, [b"\xff\xd8\xff\xd9"] + frames, [3, 1, 2], 1)[0] == 0


def test_pillow_training_crop(built, ctx):
    """RandomResizedCrop + RandomHorizontalFlip / RandomVerticalFlip of the golden 8-bit vectors as Pillow computes them:
    flip(Image.open(f).convert("RGB").crop(box).resize((224, 224), BILINEAR)), byte for byte in one [N, 3, 224, 224] tensor"""
    import io

    import torch
    from PIL import Image
    frames = []
    for f in SETS["baseline"]():
        with Image.open(io.BytesIO(f)) as im:
            if im.mode in ("L", "RGB") and im.info.get("progression") is None:
                frames.append(f)
    rng = np.random.default_rng(42)
    rects, flips = [], []
    for f in frames:
        with Image.open(io.BytesIO(f)) as im:
            w, h = im.size
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        rects.append((x, y, int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))))
        flips.append(int(rng.integers(0, 4)))
    dec = _batch(built, ctx, frames, crop=rects, resize=(224, 224), resample="bilinear", reconstruction=TURBO, mode="RGB",
                 **_flip_args(flips))
    dst = torch.zeros((len(frames), 3, 224, 224), dtype=torch.uint8, device="cuda")
    dec.decode_into(dst)
    torch.cuda.synchronize()
    got = dst.cpu().numpy()
    ops = {fm.H: [Image.Transpose.FLIP_LEFT_RIGHT], fm.V: [Image.Transpose.FLIP_TOP_BOTTOM],
           fm.H | fm.V: [Image.Transpose.FLIP_LEFT_RIGHT, Image.Transpose.FLIP_TOP_BOTTOM], 0: []}
    assert len(frames) >= 5
    for j, (f, (x, y, w, h), fl) in enumerate(zip(frames, rects, flips)):
        assert dec.status(j) == 0
        with Image.open(io.BytesIO(f)) as im:
            out = im.convert("RGB").crop((x, y, x + w, y + h)).resize((224, 224), Image.Resampling.BILINEAR)
        for op in ops[fl]:
            out = out.transpose(op)
        assert np.array_equal(got[j], np.asarray(out).transpose(2, 0, 1)), "frame %d (flip %d)" % (j, fl)
