"""GPU: BatchDecoder(box=..., reducing_gap=..., window=...) / b200jpg_batch_create_resample (DESIGN §19). The oracle is
tests/resize_box_model.py (pinned to Pillow by test_resize_box_cpu.py) applied to the decode of the same batch configuration without
sizes, bit for bit, as tests/test_resize.py does; the Resize + CenterCrop and thumbnail batches are also checked against the digests
Pillow and torchvision gave for the fixtures under tests/golden/resize_box."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om
from tests import resize_box_model as bm
from tests import resize_model as rm
from tests.test_crop import CROP_SETS
from tests.test_decode_into import SETS
from tests.test_orientation import _batch, _decode, _images, _synth, _view_as_int

pytestmark = pytest.mark.gpu

FILTERS = ["box", "bilinear", "hamming", "bicubic", "lanczos"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize_box")
SYNTH = [(1920, 1080, 61, (2, 2)), (1000, 333, 62, (2, 1)), (333, 1000, 63, (1, 2)), (640, 480, 64, (1, 1)), (517, 300, 65, (2, 2))]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _cases(h, w, rng, gap, n):
    """(size (h_t, w_t), box, window) for a C of h x w: a fractional box, an integer one, a zero-width one, a window of the resize,
    a strong shrink that reduces under a gap, a growth, and a seeded mix"""
    def box():
        x0, x1 = sorted(float(v) for v in rng.uniform(0, w, 2))
        y0, y1 = sorted(float(v) for v in rng.uniform(0, h, 2))
        return (x0, y0, x1, y1)

    def window(th, tw):
        x, y = int(rng.integers(0, tw)), int(rng.integers(0, th))
        return (x, y, int(rng.integers(1, tw - x + 1)), int(rng.integers(1, th - y + 1)))

    small = (max(1, h // 7), max(1, w // 9))
    out = [((max(1, h // 2), max(1, w // 3)), box(), None),
           ((max(1, h // 3), max(1, w // 2)), (0.0, 1.0, float(w), float(max(h - 1, 1))) if h > 1 else None, None),
           ((5, 4), (w / 2, 0.0, w / 2, float(h)) if gap is None else None, None),  # zero width (its reduce box would be empty)
           ((h + 5, w * 3 // 2 + 1), None, window(h + 5, w * 3 // 2 + 1)),
           (small, None if gap is None else box(), window(*small)),
           ((max(1, h // 17), max(1, w // 19)), None, None),
           ((h, w), (0.5, 0.5, w - 0.5, h - 0.5) if w > 1 and h > 1 else None, window(h, w))]
    th, tw = int(rng.integers(1, 2 * h + 2)), int(rng.integers(1, 2 * w + 2))
    out.append(((th, tw), box(), window(th, tw)))
    return out[:n]


def _check(built, ctx, frames, resample, seed=0, gap=None, per_frame=8, crop=False, **kw):
    """every live 8-bit frame under _cases (after a seeded rectangle when `crop`): decode() equals the model on the decode without
    sizes, shapes and statuses agree, nothing outside the slots is written"""
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(seed)
    batch, rects, sizes, boxes, wins, src = [], [], [], [], [], []
    for i, f in enumerate(frames):
        if ref[i] is None or ref[i].dtype != np.uint8:
            batch.append(f), rects.append(None), sizes.append(None), boxes.append(None), wins.append(None), src.append(i)
            continue
        oh, ow = ref[i].shape[:2]
        rect = cm.rectangles(ow, oh, rng, n_random=1)[-1] if crop else None
        ch, cw = (oh, ow) if rect is None else (rect[3], rect[2])
        for s, b, win in [(None, None, None)] + _cases(ch, cw, rng, gap, per_frame):
            batch.append(f), rects.append(rect), sizes.append(s), boxes.append(b), wins.append(win), src.append(i)
    dec = _batch(built, ctx, batch, crop=rects if crop else None, resize=sizes, box=boxes, window=wins, reducing_gap=gap,
                 resample=resample, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    for j, (i, r, s, b, win) in enumerate(zip(src, rects, sizes, boxes, wins)):
        assert dec.status(j) == plain.status(i), "frame %d (source %d)" % (j, i)
        if ref[i] is None:
            assert got[j] is None
            continue
        c = ref[i] if r is None else ref[i][r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        want = c if s is None else bm.resize(c, s[1], s[0], rm.NAMES[resample], box=b, gap=gap, window=win)
        assert dec.output_shape(j, 0) == want.shape[:2]
        assert np.array_equal(got[j], want), "frame %d (source %d, rect %s, size %s, box %s, window %s)" % (j, i, r, s, b, win)
    mask = np.ones(out.numel(), dtype=bool)
    for j in range(len(batch)):
        mask[dec.out_offset(j):dec.out_offset(j) + dec.frame_bytes(j)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


@pytest.mark.parametrize("name", list(CROP_SETS))
def test_sets(built, ctx, name):
    """boxes, windows and reduce on every frame set of test_resize.py"""
    k = list(CROP_SETS).index(name)
    _check(built, ctx, CROP_SETS[name](), FILTERS[k % 5], seed=k, gap=[None, 2.0, 1.0][k % 3], crop=k % 2 == 0)


@pytest.mark.parametrize("resample", FILTERS)
@pytest.mark.parametrize("gap", [None, 2.0])
def test_filters(built, ctx, resample, gap):
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH] + SETS["baseline"]()[:3] + SETS["subsampling"]()[:2]
    _check(built, ctx, frames, resample, seed=FILTERS.index(resample), gap=gap, crop=True)


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_orientations_and_drafts(built, ctx, k):
    """all eight orientations on the turbo path, drafted to 1/k (k = 1: undrafted), modes RGB and L"""
    src = [_synth(700, 301, 12), _synth(301, 700, 13, (1, 1)), _synth(500, 260, 14, (2, 1)), SETS["baseline"]()[0]]
    frames = [om.tag(f, o) for f in src for o in om.ORIENTATIONS]
    draft = None if k == 1 else (700 // k, 700 // k)
    _check(built, ctx, frames, FILTERS[k % 5], seed=30 + k, gap=2.0 if k % 4 else None, per_frame=3, exif_orientation=True,
           reconstruction="libjpeg-turbo", draft=draft, mode="RGB" if k < 4 else "L")


def _digest(a):
    a = a[..., None] if a.ndim == 2 else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":%dx%dx%d" % a.shape


def _fixtures():
    with open(os.path.join(GOLDEN, "digests.json")) as f:
        digests = json.load(f)
    return [(name, open(os.path.join(GOLDEN, name + ".jpg"), "rb").read(), d) for name, d in sorted(digests.items())]


def test_resize_center_crop_destinations(built, ctx):
    """Resize(256) + CenterCrop(224) of mixed sizes into one [N, 3, 224, 224] tensor: uint8 equal to torchvision's stored digests,
    float32 / float16 / bfloat16 with the ImageNet map equal to the uint8 result mapped by PyTorch, NCHW, NHWC and padded
    destinations, sentinels untouched"""
    import torch
    from libjpeg_b200.decoder import resize_center_crop_args
    fx = _fixtures()
    frames = [d for _, d, _ in fx]
    args = [resize_center_crop_args(d, 256, 224) for d in frames]
    dec = built.BatchDecoder(frames, ctx=ctx, mode="RGB", reconstruction="libjpeg-turbo", resize=[a["resize"] for a in args],
                             window=[a["window"] for a in args], resample="bilinear")
    dec.upload()
    n = len(frames)
    dst = torch.full((n, 3, 224, 224), 0xA5, dtype=torch.uint8, device="cuda")
    dec.decode_into(dst)
    torch.cuda.synchronize()
    u8 = dst.permute(0, 2, 3, 1).cpu().numpy()
    for i, (name, _, d) in enumerate(fx):
        assert _digest(u8[i]) == d["resize256_crop224"], name
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    scale, bias = [1 / (255 * s) for s in std], [-m / s for m, s in zip(mean, std)]
    ref = torch.from_numpy(u8).cuda().permute(0, 3, 1, 2)
    for dt in (torch.uint8, torch.float32, torch.float16, torch.bfloat16):
        for layout in ("nchw", "nhwc", "padded"):
            if layout == "nhwc":
                base = torch.full((n, 224, 224, 3), 7, dtype=dt, device="cuda")
                view = base.permute(0, 3, 1, 2)
            elif layout == "padded":
                base = torch.full((n, 3, 224, 240), 7, dtype=dt, device="cuda")
                view = base[..., 5:229]
            else:
                base = torch.full((n, 3, 224, 224), 7, dtype=dt, device="cuda")
                view = base
            if dt == torch.uint8:
                dec.decode_into(view)
                want = ref
            else:
                dec.decode_into(view, scale=scale, bias=bias)
                s = torch.tensor(scale, device="cuda").view(1, 3, 1, 1)
                b = torch.tensor(bias, device="cuda").view(1, 3, 1, 1)
                want = (ref.float() * s + b).to(dt)
            torch.cuda.synchronize()
            assert torch.equal(_view_as_int(view), _view_as_int(want.contiguous())), (dt, layout)
            if layout == "padded":
                assert (_view_as_int(base[..., :5]) == _view_as_int(torch.full((1,), 7, dtype=dt, device="cuda"))).all()
                assert (_view_as_int(base[..., 229:]) == _view_as_int(torch.full((1,), 7, dtype=dt, device="cuda"))).all()


def test_thumbnail_batch(built, ctx):
    """thumbnail((128, 128)), ((64, 64)), ((100, 37)) and an untouched one, drafted and reduced as Pillow's thumbnail() does, in one
    batch: every frame equal to Pillow's stored digest"""
    from libjpeg_b200.decoder import thumbnail_args
    frames, keys, args = [], [], []
    for name, data, d in _fixtures():
        for w, h in ((128, 128), (64, 64), (100, 37), (2000, 2000)):
            frames.append(data), keys.append((name, d["thumbnail_%dx%d" % (w, h)]))
            args.append(thumbnail_args(data, (h, w)))
    dec = built.BatchDecoder(frames, ctx=ctx, reconstruction="libjpeg-turbo", draft=[a["draft"] for a in args],
                             resize=[a["resize"] for a in args], box=[a["box"] for a in args], reducing_gap=2.0, resample="bicubic")
    dec.upload()
    got = _images(dec, _decode(dec))
    assert any(a["draft"] is not None and a["resize"] is not None for a in args)
    for g, (name, want) in zip(got, keys):
        assert _digest(g) == want, name


def test_decode_twice_and_launches(built, ctx):
    """two decodes give identical output; a batch whose frames reduce issues the launches of the same batch without the gap plus
    one; boxes and windows add none"""
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH]
    sizes = [(h // 9, w // 7) for w, h, _, _ in SYNTH]
    plain = _batch(built, ctx, frames, resize=sizes)
    _decode(plain)
    red = _batch(built, ctx, frames, resize=sizes, reducing_gap=2.0)
    a, b = _decode(red), _decode(red)
    assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())
    assert red.launches == plain.launches + 1
    boxed = _batch(built, ctx, frames, resize=sizes, box=[(1.5, 2.5, w - 3.0, h - 1.0) for w, h, _, _ in SYNTH],
                   window=[(1, 1, max(1, w // 7 - 2), max(1, h // 9 - 2)) for w, h, _, _ in SYNTH])
    _decode(boxed)
    assert boxed.launches == plain.launches


def _create(built, ctx, frames, sizes, boxes=None, windows=None, gap=0.0, tolerate=0, resample=2):
    from libjpeg_b200 import native
    n = len(frames)
    ptrs = (ctypes.c_void_p * n)(*[ctypes.cast(ctypes.c_char_p(f), ctypes.c_void_p).value for f in frames])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    st = (native.SizeStruct * n)(*[native.SizeStruct(*(s[::-1] if s else (0, 0))) for s in sizes])
    bt = None if boxes is None else (native.BoxStruct * n)(*[native.BoxStruct(*(b or (0, 0, 0, 0))) for b in boxes])
    wt = None if windows is None else (native.RectStruct * n)(*[native.RectStruct(*(w or (0, 0, 0, 0))) for w in windows])
    handle = ctypes.c_void_p()
    rc = native.lib.b200jpg_batch_create_resample(ctx.handle, ptrs, lens, n, tolerate, 0, None, None, st, bt, wt, resample, gap,
                                                  ctypes.byref(handle))
    msg = native.last_error(ctx.handle)[1]
    if rc == 0:
        native.lib.b200jpg_batch_destroy(handle)
    return rc, msg, handle


def test_unchanged_without_new_arguments(built, ctx):
    """create_resample with NULL / all-zero boxes and windows and no gap: the bytes and launches of create_resize"""
    import torch
    from libjpeg_b200 import native
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH]
    sizes = [(h // 3, w // 2) for w, h, _, _ in SYNTH]
    ref = _batch(built, ctx, frames, resize=sizes)
    want = _decode(ref).cpu().numpy()
    for boxes, windows in ((None, None), ([None] * len(frames), [None] * len(frames))):
        n = len(frames)
        ptrs = (ctypes.c_void_p * n)(*[ctypes.cast(ctypes.c_char_p(f), ctypes.c_void_p).value for f in frames])
        lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
        st = (native.SizeStruct * n)(*[native.SizeStruct(s[1], s[0]) for s in sizes])
        bt = None if boxes is None else (native.BoxStruct * n)()
        wt = None if windows is None else (native.RectStruct * n)()
        handle = ctypes.c_void_p()
        assert native.lib.b200jpg_batch_create_resample(ctx.handle, ptrs, lens, n, 0, 0, None, None, st, bt, wt, 2, 0.0,
                                                        ctypes.byref(handle)) == 0
        try:
            assert native.lib.b200jpg_batch_upload(handle, None) == 0
            out = torch.full((native.lib.b200jpg_batch_out_bytes(handle, -1),), 0x5A, dtype=torch.uint8, device="cuda")
            assert native.lib.b200jpg_batch_decode(handle, out.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy(), want)
            assert native.lib.b200jpg_batch_last_launch_count(handle) == ref.launches
        finally:
            native.lib.b200jpg_batch_destroy(handle)


def test_refused(built, ctx):
    """each refusal fails the call with INVALID_PARAMETER (NOT_IMPLEMENTED for a reduce block of 2^24 pixels) naming the frame,
    tolerate_bad or not, and leaves the context's open-batch count unchanged"""
    from libjpeg_b200 import NativeError
    data = _synth(64, 48, 1)
    inv, nimp = -1024, -1034
    cases = [([None, None], [None, (0, 0, 1, 1)], None, 0.0, inv),  # a box on a frame without a size
             ([None, None], None, [None, (0, 0, 1, 1)], 0.0, inv),  # a window on a frame without a size
             ([None, (8, 8)], [None, (-1, 0, 4, 4)], None, 0.0, inv),
             ([None, (8, 8)], [None, (0, 0, 64.5, 4)], None, 0.0, inv),
             ([None, (8, 8)], [None, (5, 0, 4, 4)], None, 0.0, inv),
             ([None, (8, 8)], [None, (0, 0, float("nan"), 4)], None, 0.0, inv),
             ([None, (8, 8)], [None, (0, 0, float("inf"), 4)], None, 0.0, inv),
             ([None, (8, 8)], None, [None, (4, 0, 5, 1)], 0.0, inv),
             ([None, (8, 8)], None, [None, (0, 0, 0, 3)], 0.0, inv),
             ([None, (8, 8)], None, None, 0.5, inv),
             ([None, (8, 8)], None, None, float("nan"), inv),
             ([None, (8, 8)], [None, (5, 0, 5, 48)], None, 1.0, inv)]  # a zero-width reduce box: Pillow raises
    for tol in (0, 1):
        for sizes, boxes, windows, gap, code in cases:
            rc, msg, _ = _create(built, ctx, [data, data], sizes, boxes, windows, gap, tol)
            assert rc == code, (sizes, boxes, windows, gap, msg)
            assert ("frame 1" in msg) or "reducing_gap" in msg, msg
    before = ctx._batches
    for kw in (dict(resize=[None, (8, 8)], box=[None, (0, 0, 65, 4)]), dict(resize=[None, (8, 8)], window=[None, (0, 0, 9, 1)])):
        with pytest.raises(NativeError):
            built.BatchDecoder([data, data], ctx=ctx, **kw)
    assert ctx._batches == before
    # a failed frame's box and window are ignored
    dec = built.BatchDecoder([b"\xff\xd8\xff\xd9", data], ctx=ctx, tolerate_bad=True, resize=[None, (3, 4)],
                             box=[(0, 0, 1e9, 1), None], window=[(5, 5, 5, 5), None])
    assert dec.status(0) != 0 and dec.output_shape(1, 0) == (3, 4)
    dec.close()
    big = _synth(4096, 4096, 3)
    rc, msg, _ = _create(built, ctx, [big], [(1, 1)], gap=1.0)
    assert rc == nimp, msg
