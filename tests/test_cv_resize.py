"""GPU: BatchDecoder(resample="cv2-linear" | "cv2-area") / B200JPG_RESAMPLE_CV_LINEAR, _CV_AREA (DESIGN §20). The oracle is
tests/cv_resize_model.py (pinned to OpenCV by test_cv_resize_cpu.py) applied to the decode of the same batch without sizes, byte
for byte; turbo batches of the stored fixtures are also checked against the digests OpenCV gave for them
(tests/golden/cv_resize), so this test needs no cv2."""
import ctypes
import hashlib
import json
import math
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import cv_resize_model as cvm
from tests import orientation_model as om
from tests.test_crop import CROP_SETS
from tests.test_decode_into import SETS
from tests.test_orientation import _batch, _decode, _images, _synth, _view_as_int

pytestmark = pytest.mark.gpu

FILTERS = ["cv2-linear", "cv2-area"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SYNTH = [(1920, 1080, 71, (2, 2)), (1000, 333, 72, (2, 1)), (333, 1000, 73, (1, 2)), (640, 480, 74, (1, 1)), (517, 300, 75, (2, 2))]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _divisor(n):
    return next((d for d in (2, 3, 4, 5, 7) if n % d == 0 and n > d), 1)


def _cases(h, w, rng, n):
    """(size (h_t, w_t), window) for a C of h x w: integer shrinks (2 x 2 and others), a fractional shrink, ultralytics' long side
    640, 224 x 224, a growth with a window, one axis up and one down, the same size, and a seeded mix"""
    def window(th, tw):
        x, y = int(rng.integers(0, tw)), int(rng.integers(0, th))
        return (x, y, int(rng.integers(1, tw - x + 1)), int(rng.integers(1, th - y + 1)))

    r = 640 / max(w, h)
    dy, dx = _divisor(h), _divisor(w)
    out = [((h // dy, w // dx), None),
           ((max(1, h // 2), max(1, w // 2)), None),
           ((max(1, h * 2 // 3), max(1, w * 3 // 5)), window(max(1, h * 2 // 3), max(1, w * 3 // 5))),
           ((min(math.ceil(h * r), 640), min(math.ceil(w * r), 640)), None),
           ((224, 224), None),
           ((h + 5, w * 3 // 2 + 1), window(h + 5, w * 3 // 2 + 1)),
           ((2 * h, max(1, w // 3)), None),
           ((h, w), window(h, w)),
           ((max(1, h // 7), max(1, w // 9)), None)]
    th, tw = int(rng.integers(1, 2 * h + 2)), int(rng.integers(1, 2 * w + 2))
    out.append(((th, tw), window(th, tw)))
    return out[:n]


def _check(built, ctx, frames, resample, seed=0, per_frame=10, crop=False, **kw):
    """every live 8-bit frame under _cases (after a seeded rectangle when `crop`): decode() equals the model on the decode without
    sizes, shapes and statuses agree, nothing outside the slots is written"""
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(seed)
    batch, rects, sizes, wins, src = [], [], [], [], []
    for i, f in enumerate(frames):
        if ref[i] is None or ref[i].dtype != np.uint8:
            batch.append(f), rects.append(None), sizes.append(None), wins.append(None), src.append(i)
            continue
        oh, ow = ref[i].shape[:2]
        rect = cm.rectangles(ow, oh, rng, n_random=1)[-1] if crop else None
        ch, cw = (oh, ow) if rect is None else (rect[3], rect[2])
        for s, win in [(None, None)] + _cases(ch, cw, rng, per_frame):
            batch.append(f), rects.append(rect), sizes.append(s), wins.append(win), src.append(i)
    dec = _batch(built, ctx, batch, crop=rects if crop else None, resize=sizes, window=wins, resample=resample, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    for j, (i, r, s, win) in enumerate(zip(src, rects, sizes, wins)):
        assert dec.status(j) == plain.status(i), "frame %d (source %d)" % (j, i)
        if ref[i] is None:
            assert got[j] is None
            continue
        c = ref[i] if r is None else ref[i][r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        want = c if s is None else cvm.resize_window(c, s[1], s[0], resample, win)
        assert dec.output_shape(j, 0) == want.shape[:2]
        assert np.array_equal(got[j], want), "frame %d (source %d, rect %s, size %s, window %s)" % (j, i, r, s, win)
    mask = np.ones(out.numel(), dtype=bool)
    for j in range(len(batch)):
        mask[dec.out_offset(j):dec.out_offset(j) + dec.frame_bytes(j)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


@pytest.mark.parametrize("name", list(CROP_SETS))
def test_sets(built, ctx, name):
    """every frame set of test_resize.py, both filters, with and without a crop before"""
    k = list(CROP_SETS).index(name)
    _check(built, ctx, CROP_SETS[name](), FILTERS[k % 2], seed=k, crop=k % 4 < 2)


@pytest.mark.parametrize("resample", FILTERS)
@pytest.mark.parametrize("reconstruction", ["reference", "libjpeg-turbo"])
def test_filters(built, ctx, resample, reconstruction):
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH] + SETS["baseline"]()[:3] + SETS["subsampling"]()[:2]
    _check(built, ctx, frames, resample, seed=FILTERS.index(resample), crop=True, reconstruction=reconstruction)


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_orientations_drafts_modes(built, ctx, k):
    """all eight orientations on the turbo path, drafted to 1/k (k = 1: undrafted), modes RGB and L (grey frames under RGB)"""
    src = [_synth(700, 301, 12), _synth(301, 700, 13, (1, 1)), _synth(500, 260, 14, (2, 1)), SETS["baseline"]()[0],
           open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read()]
    frames = [om.tag(f, o) for f in src for o in om.ORIENTATIONS]
    draft = None if k == 1 else (700 // k, 700 // k)
    _check(built, ctx, frames, FILTERS[k % 2], seed=30 + k, per_frame=3, exif_orientation=True, reconstruction="libjpeg-turbo", draft=draft,
           mode="RGB" if k < 4 else "L")


@pytest.mark.parametrize("mode", [None, "RGB", "L"])
def test_cmyk(built, ctx, mode):
    """CMYK / YCCK frames: Pillow's conversion under a mode (DESIGN §15 / §18), four channels without one"""
    import glob
    frames = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLDEN, "cmyk", "*.jpg")))]
    for resample in FILTERS:
        _check(built, ctx, frames, resample, seed=40, per_frame=5, mode=mode,
               reconstruction="reference" if mode is None else "libjpeg-turbo")


def _digest(a):
    a = a[..., None] if a.ndim == 2 else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":%dx%dx%d" % a.shape


def _fixtures():
    with open(os.path.join(GOLDEN, "cv_resize", "digests.json")) as f:
        digests = json.load(f)["frames"]
    return [(name, open(os.path.join(GOLDEN, name), "rb").read(), d) for name, d in sorted(digests.items())]


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_opencv_digests(built, ctx, mode):
    """the turbo reconstruction of every stored fixture, resized to every stored size with both filters: equal to OpenCV's stored
    cv2.resize(cv2.imdecode(...)) digests (IMREAD_COLOR, BGR, under "RGB"; IMREAD_GRAYSCALE under "L")"""
    key = "color" if mode == "RGB" else "gray"
    for resample, iname in (("cv2-linear", "linear"), ("cv2-area", "area")):
        frames, sizes, want = [], [], []
        for name, data, d in _fixtures():
            for k, v in d.items():
                m, i, wh = k.split("_")
                if m == key and i == iname:
                    tw, th = (int(x) for x in wh.split("x"))
                    frames.append(data), sizes.append((th, tw)), want.append((name, k, v))
        dec = _batch(built, ctx, frames, resize=sizes, resample=resample, mode=mode, reconstruction="libjpeg-turbo")
        got = _images(dec, _decode(dec))
        for g, (name, k, v) in zip(got, want):
            assert _digest(g[..., ::-1] if mode == "RGB" else g) == v, (name, k)


def test_destinations(built, ctx):
    """uint8 NCHW / NHWC / BGR-ordered planes and fp32 / fp16 / bf16 maps of a 224 x 224 batch: the packed result, mapped by
    PyTorch for the float kinds; padding sentinels untouched"""
    import torch
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH] + [open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read()]
    for resample in FILTERS:
        dec = _batch(built, ctx, frames, resize=(224, 224), resample=resample, mode="RGB", reconstruction="libjpeg-turbo")
        n = len(frames)
        ref = torch.from_numpy(np.stack(_images(dec, _decode(dec)))).cuda().permute(0, 3, 1, 2)
        scale, bias = [1 / 255.0, 1 / 200.0, 1 / 100.0], [-0.5, 0.25, -1.0]
        for dt in (torch.uint8, torch.float32, torch.float16, torch.bfloat16):
            for layout in ("nchw", "nhwc", "bgr", "padded"):
                if layout == "nhwc":
                    base = torch.full((n, 224, 224, 3), 7, dtype=dt, device="cuda")
                    view = dst = base.permute(0, 3, 1, 2)
                elif layout == "bgr":  # output component c into channel 2 - c of an NHWC tensor
                    base = torch.full((n, 224, 224, 3), 7, dtype=dt, device="cuda")
                    view = base.permute(0, 3, 1, 2)[:, [2, 1, 0]]
                    dst = [[base[i, ..., 2], base[i, ..., 1], base[i, ..., 0]] for i in range(n)]
                elif layout == "padded":
                    base = torch.full((n, 3, 224, 240), 7, dtype=dt, device="cuda")
                    view = dst = base[..., 5:229]
                else:
                    base = torch.full((n, 3, 224, 224), 7, dtype=dt, device="cuda")
                    view = dst = base
                if dt == torch.uint8:
                    dec.decode_into(dst)
                    want = ref
                else:
                    dec.decode_into(dst, scale=scale, bias=bias)
                    s = torch.tensor(scale, device="cuda").view(1, 3, 1, 1)
                    b = torch.tensor(bias, device="cuda").view(1, 3, 1, 1)
                    want = (ref.float() * s + b).to(dt)
                torch.cuda.synchronize()
                if layout == "bgr":
                    view = base.permute(0, 3, 1, 2)[:, [2, 1, 0]]
                assert torch.equal(_view_as_int(view.contiguous()), _view_as_int(want.contiguous())), (resample, dt, layout)
                if layout == "padded":
                    seven = _view_as_int(torch.full((1,), 7, dtype=dt, device="cuda"))
                    assert (_view_as_int(base[..., :5]) == seven).all() and (_view_as_int(base[..., 229:]) == seven).all()


def test_letterbox(built, ctx):
    """a YOLO-style letterbox: [N, 3, 640, 640] fp16 filled with 114 / 255, each frame resized to long side 640 (ceil(w r)) and
    described at its centred offset in BGR order; equal to the model inside, the border untouched"""
    import torch
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH] + [_synth(3840, 2160, 76)]
    shapes = [(h, w) for w, h, _, _ in SYNTH] + [(2160, 3840)]
    for resample in FILTERS:
        sizes = []
        for h, w in shapes:
            r = 640 / max(w, h)
            sizes.append((min(math.ceil(h * r), 640), min(math.ceil(w * r), 640)))
        dec = _batch(built, ctx, frames, resize=sizes, resample=resample, mode="RGB", reconstruction="libjpeg-turbo")
        plain = _batch(built, ctx, frames, mode="RGB", reconstruction="libjpeg-turbo")
        ref = _images(plain, _decode(plain))
        n = len(frames)
        fill = torch.tensor(114 / 255, dtype=torch.float16)
        base = torch.full((n, 3, 640, 640), float(fill), dtype=torch.float16, device="cuda")
        dst = []
        for i, (th, tw) in enumerate(sizes):
            y, x = (640 - th) // 2, (640 - tw) // 2
            dst.append([base[i, 2 - c, y:y + th, x:x + tw] for c in range(3)])  # BGR: output component c to plane 2 - c
        dec.decode_into(dst, scale=1 / 255)
        torch.cuda.synchronize()
        got = base.cpu()
        for i, (th, tw) in enumerate(sizes):
            y, x = (640 - th) // 2, (640 - tw) // 2
            want = torch.from_numpy(cvm.resize(ref[i], tw, th, resample)[..., ::-1].copy()).permute(2, 0, 1).float()
            want = (want * torch.tensor(1 / 255, dtype=torch.float32)).half()
            assert torch.equal(got[i, :, y:y + th, x:x + tw].view(torch.int16), want.view(torch.int16)), (resample, i)
            border = torch.ones((3, 640, 640), dtype=torch.bool)
            border[:, y:y + th, x:x + tw] = False
            assert (got[i][border].view(torch.int16) == fill.view(torch.int16)).all(), (resample, i)


def test_tolerant_mixed_batch(built, ctx):
    """a bad codestream, a 12-bit frame, grey and colour frames, resized and not, in one tolerant batch"""
    frames = [b"\xff\xd8\xff\xd9", _synth(300, 200, 5), open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read()]
    frames += [open(os.path.join(GOLDEN, "deep12", "d12_420_50x38_q60.jpg"), "rb").read(), _synth(64, 48, 6, (1, 1))]
    for resample in FILTERS:
        _check(built, ctx, frames, resample, seed=50, per_frame=10)


def test_pillow_and_cv_batches(built, ctx):
    """the same frames through a Pillow-filter batch and a cv batch, as separate calls: each equals its own model, and the
    Pillow batch is unchanged by the cv one before it"""
    from tests import resize_model as rm
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH]
    sizes = [(h // 3 + 1, w // 2 + 1) for w, h, _, _ in SYNTH]
    plain = _batch(built, ctx, frames)
    ref = _images(plain, _decode(plain))
    pil1 = _images(*(lambda d: (d, _decode(d)))(_batch(built, ctx, frames, resize=sizes, resample="bilinear")))
    cv = _images(*(lambda d: (d, _decode(d)))(_batch(built, ctx, frames, resize=sizes, resample="cv2-linear")))
    pil2 = _images(*(lambda d: (d, _decode(d)))(_batch(built, ctx, frames, resize=sizes, resample="bilinear")))
    for i, (th, tw) in enumerate(sizes):
        assert np.array_equal(cv[i], cvm.resize(ref[i], tw, th, "cv2-linear"))
        assert np.array_equal(pil1[i], rm.resize(ref[i], tw, th, rm.BILINEAR))
        assert np.array_equal(pil2[i], pil1[i])


def test_launches(built, ctx):
    """a cv batch launches the same batch without sizes plus its resize kernels: two per table kind (linear rules 1 / 4, area
    rule 3) and one for integer-factor area blocks and copies; two decodes give identical output"""
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH]
    base = _batch(built, ctx, frames, crop=[(0, 0, w, h) for w, h, _, _ in SYNTH])
    _decode(base)
    cases = [("cv2-linear", [(h // 3 + 1, w // 2 + 1) for w, h, _, _ in SYNTH], 2),
             ("cv2-area", [(h // 3 + 1, w // 2 + 1) for w, h, _, _ in SYNTH], 2),  # rule 3 only
             ("cv2-area", [(h, w) for w, h, _, _ in SYNTH], 1),  # copies
             ("cv2-area", [(2 * h, w) for w, h, _, _ in SYNTH], 2),  # rule 4 only
             ("cv2-area", [[(h, w), (h // 3 + 1, w // 2 + 1), (2 * h, w)][min(i, 2) if i < 3 else 0]
                           for i, (w, h, _, _) in enumerate(SYNTH)], 5)]  # copies, rule 3 and rule 4
    for resample, sizes, extra in cases:
        dec = _batch(built, ctx, frames, resize=sizes, resample=resample)
        a, b = _decode(dec), _decode(dec)
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())
        assert dec.launches == base.launches + extra, (resample, sizes, dec.launches, base.launches)


def _create(ctx, frames, sizes, boxes=None, gap=0.0, tolerate=0, resample=cvm.LINEAR):
    from libjpeg_b200 import native
    n = len(frames)
    ptrs = (ctypes.c_void_p * n)(*[ctypes.cast(ctypes.c_char_p(f), ctypes.c_void_p).value for f in frames])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    st = (native.SizeStruct * n)(*[native.SizeStruct(*(s[::-1] if s else (0, 0))) for s in sizes])
    bt = None if boxes is None else (native.BoxStruct * n)(*[native.BoxStruct(*(b or (0, 0, 0, 0))) for b in boxes])
    handle = ctypes.c_void_p()
    rc = native.lib.b200jpg_batch_create_resample(ctx.handle, ptrs, lens, n, tolerate, 0, None, None, st, bt, None, resample, gap,
                                                  ctypes.byref(handle))
    msg = native.last_error(ctx.handle)[1]
    if rc == 0:
        native.lib.b200jpg_batch_destroy(handle)
    return rc, msg


def test_refused(built, ctx):
    """a box or a reducing_gap with a cv filter fails the call with INVALID_PARAMETER naming the frame, tolerate_bad or not; the
    open-batch count is unchanged"""
    from libjpeg_b200 import NativeError
    data = _synth(64, 48, 1)
    inv = -1024
    for resample in (cvm.LINEAR, cvm.AREA):
        for tol in (0, 1):
            rc, msg = _create(ctx, [data, data], [None, (8, 8)], boxes=[None, (0, 0, 32, 24)], tolerate=tol, resample=resample)
            assert rc == inv and "frame 1" in msg and "box" in msg, msg
            rc, msg = _create(ctx, [data, data], [None, (8, 8)], gap=2.0, tolerate=tol, resample=resample)
            assert rc == inv and "frame 1" in msg and "reducing_gap" in msg, msg
            assert _create(ctx, [data, data], [None, (8, 8)], tolerate=tol, resample=resample)[0] == 0
    before = ctx._batches
    for kw in (dict(box=[None, (0, 0, 32, 24)]), dict(reducing_gap=2.0)):
        with pytest.raises(NativeError):
            built.BatchDecoder([data, data], ctx=ctx, resize=[None, (8, 8)], resample="cv2-area", **kw)
    with pytest.raises(ValueError):
        built.BatchDecoder([data], ctx=ctx, resize=(8, 8), resample="cv2-cubic")
    assert ctx._batches == before
