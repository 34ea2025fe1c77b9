"""GPU: BatchDecoder(resize=..., resample=...) / b200jpg_batch_create_resize. The oracle is tests/resize_model.py (pinned to Pillow
by test_resize_cpu.py) applied to the crop decode of the same batch configuration without sizes (pinned by test_crop.py), bit
for bit; every frame's status is that of the batch without sizes, and nothing outside a frame's destination is written."""
import ctypes
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om
from tests import resize_model as rm
from tests.test_crop import CROP_SETS
from tests.test_decode_into import GOLDEN, SETS
from tests.test_orientation import _batch, _decode, _images, _synth, _view_as_int

pytestmark = pytest.mark.gpu

SENT = 0xA5
FILTERS = ["box", "bilinear", "hamming", "bicubic", "lanczos"]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _targets(h, w, rng):
    """(h_t, w_t) for a C of h x w: shrinking, growing, identity, one axis unchanged, 1 x 1, ratios of at least 17 both ways,
    and a seeded one"""
    t = [(max(1, h * 2 // 5), max(1, w // 3)), (h + 7, w * 3 // 2 + 1), (h, w), (h, max(1, w // 2 + 1)), (max(1, h - 3), w), (1, 1),
         (max(1, h // 17), max(1, w // 19)), (int(rng.integers(1, 2 * h + 2)), int(rng.integers(1, 2 * w + 2)))]
    if h * w <= 64 * 64:
        t.append((17 * h, 19 * w))
    out = []
    for s in t:
        if s not in out:
            out.append(s)
    return out


def _resized(img, size, resample):
    h, w = size
    return rm.resize(img, w, h, rm.NAMES[resample])


def _check_packed(built, ctx, frames, resample, seed=0, crop=True, per_frame=None, **kw):
    """Every live 8-bit frame under the targets of _targets (with a seeded rectangle when `crop`), and once unresized; failed and
    12-bit frames unresized. decode() equals the model on the crop decode without sizes, statuses agree, and no byte outside the
    slots is written."""
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(seed)
    batch, rects, sizes, src = [], [], [], []
    for i, f in enumerate(frames):
        if ref[i] is None or ref[i].dtype != np.uint8:
            batch.append(f), rects.append(None), sizes.append(None), src.append(i)
            continue
        oh, ow = ref[i].shape[:2]
        rect = None
        if crop:
            rect = cm.rectangles(ow, oh, rng, n_random=1)[-1]
        ch, cw = (oh, ow) if rect is None else (rect[3], rect[2])
        targets = _targets(ch, cw, rng)
        if per_frame:
            targets = targets[:per_frame]
        for s in [None] + targets:
            batch.append(f), rects.append(rect), sizes.append(s), src.append(i)
    dec = _batch(built, ctx, batch, crop=rects, resize=sizes, resample=resample, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    live = 0
    for j, (i, r, s) in enumerate(zip(src, rects, sizes)):
        assert dec.status(j) == plain.status(i), "frame %d (source %d)" % (j, i)
        if ref[i] is None:
            assert got[j] is None
            continue
        c = ref[i] if r is None else ref[i][r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        want = c if s is None else _resized(c, s, resample)
        assert dec.output_shape(j, 0) == want.shape[:2]
        assert np.array_equal(got[j], want), "frame %d (source %d, rectangle %s, size %s)" % (j, i, r, s)
        live += s is not None
    assert live > 0 or not any(r is not None and r.dtype == np.uint8 for r in ref)  # (a set of 12-bit frames: none resized)
    mask = np.ones(out.numel(), dtype=bool)
    for j in range(len(batch)):
        mask[dec.out_offset(j):dec.out_offset(j) + dec.frame_bytes(j)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


@pytest.mark.parametrize("name", list(CROP_SETS))
def test_packed(built, ctx, name):
    k = list(CROP_SETS).index(name)
    _check_packed(built, ctx, CROP_SETS[name](), FILTERS[k % 5], seed=k, crop=k % 2 == 0)


SYNTH = [(1920, 1080, 61, (2, 2)), (1000, 333, 62, (2, 1)), (333, 1000, 63, (1, 2)), (640, 480, 64, (1, 1)), (517, 300, 65, (2, 2))]


@pytest.mark.parametrize("resample", FILTERS)
def test_filters(built, ctx, resample):
    """every filter on synthetic 4:2:0 / 4:2:2 / 4:4:0 / 4:4:4 frames up to 1920 x 1080, grey and generic golden frames, with and
    without rectangles"""
    frames = [_synth(w, h, s, sub) for w, h, s, sub in SYNTH] + SETS["baseline"]()[:4] + SETS["subsampling"]()[:3]
    _check_packed(built, ctx, frames, resample, seed=FILTERS.index(resample), crop=True, per_frame=5)
    _check_packed(built, ctx, frames, resample, seed=10 + FILTERS.index(resample), crop=False, per_frame=4)


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_orientations_and_downscale(built, ctx, k):
    """all eight orientations with rectangles in oriented output coordinates (downscale -> orientation -> crop -> resize)"""
    src = [_synth(700, 301, 12), _synth(301, 700, 13, (1, 1)), _synth(500, 260, 14, (2, 1)), SETS["subsampling"]()[0],
           SETS["baseline"]()[0]]
    frames = [om.tag(f, o) for f in src for o in om.ORIENTATIONS]
    _check_packed(built, ctx, frames, FILTERS[k % 5], seed=30 + k, per_frame=2, exif_orientation=True, downscale=k)


def test_no_color_transform(built, ctx):
    frames = SETS["baseline"]() + SETS["subsampling"]() + [_synth(1000, 333, 10), _synth(300, 200, 11, (1, 2))]
    _check_packed(built, ctx, frames, "bicubic", seed=3, per_frame=3, color_transform=False)


def _fill(shape_bytes, dtype):
    import torch
    return torch.full((shape_bytes,), SENT, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("resample", ["bilinear", "lanczos"])
def test_destinations(built, ctx, resample):
    """decode_into a [N, C, 224, 224] tensor (uint8, float32, float16, bfloat16; contiguous, padded and NHWC, sentinels around) from
    frames and rectangles of different sizes, with oriented frames; the float cases are the model's uint8 result converted by torch"""
    import torch
    src = [_synth(1000, 333, 40, (2, 2)), _synth(640, 480, 41, (1, 1)), _synth(333, 1000, 42, (2, 1)), _synth(97, 61, 43, (1, 2)),
           _synth(1920, 1080, 44)]
    frames = [om.tag(f, o) for f, o in zip(src, (1, 6, 3, 8, 1))]
    plain = _batch(built, ctx, frames, exif_orientation=True)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(7)
    th, tw = 224, 200
    batch, rects, want = [], [], []
    for f, r in zip(frames, ref):
        oh, ow = r.shape[:2]
        for rect in [None, (0, 0, ow, oh)] + cm.rectangles(ow, oh, rng, n_random=3)[-3:]:
            c = r if rect is None else r[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2]]
            batch.append(f), rects.append(rect), want.append(_resized(c, (th, tw), resample))
    dec = _batch(built, ctx, batch, crop=rects, resize=(th, tw), resample=resample, exif_orientation=True)
    n = len(batch)
    assert [dec.output_shape(i, 0) for i in range(n)] == [(th, tw)] * n
    want_u8 = torch.from_numpy(np.stack(want)).permute(0, 3, 1, 2).contiguous().cuda()
    scale, bias = [1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225)], [-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225]
    cases = [(dt, lay) for dt in (torch.uint8, torch.float32, torch.float16, torch.bfloat16) for lay in ("nchw", "nhwc", "padded")]
    for dtype, layout in cases:
        esz = torch.empty(0, dtype=dtype).element_size()
        if layout == "nchw":
            full_t = _fill(n * 3 * th * tw * esz, dtype).view(dtype).view(n, 3, th, tw)
            region = (slice(None),) * 4
            dst = full_t
        elif layout == "padded":
            full_t = _fill(n * 3 * (th + 2) * (tw + 3) * esz, dtype).view(dtype).view(n, 3, th + 2, tw + 3)
            region = (slice(None), slice(None), slice(1, th + 1), slice(1, tw + 1))
            dst = full_t[region]
        else:
            full_t = _fill(n * (th + 1) * (tw + 2) * 4 * esz, dtype).view(dtype).view(n, th + 1, tw + 2, 4)
            region = (slice(None), slice(0, th), slice(1, tw + 1), slice(0, 3))
            dst = full_t[region].permute(0, 3, 1, 2)
        if dtype == torch.uint8:
            dec.decode_into(dst)
            want_t = want_u8
        else:
            dec.decode_into(dst, scale=scale, bias=bias)
            want_t = (want_u8.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) +
                      torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
        torch.cuda.synchronize()
        assert torch.equal(_view_as_int(dst), _view_as_int(want_t)), (dtype, layout)
        mask = torch.ones(full_t.shape, dtype=torch.bool, device="cuda")
        mask[region] = False
        sent = int(np.frombuffer(bytes([SENT] * esz), dtype={1: np.uint8, 2: np.int16, 4: np.int32}[esz])[0])
        assert bool((_view_as_int(full_t)[mask] == sent).all()), (dtype, layout)
    for i in range(n):
        assert dec.status(i) == 0


def test_mixed_tolerant_batch(built, ctx):
    """resized, cropped-only, untouched, damaged and unparseable frames with 12-bit frames with and without a size, decode() and
    decode_into() per-frame tensors: statuses as defined; a 12-bit frame with a size is NOT_IMPLEMENTED and never written"""
    import torch
    base = SETS["baseline"]()[:3] + SETS["damaged"]()
    deep = SETS["deep12"]()[:2]
    frames, rects, sizes = [], [], []
    for k, f in enumerate(base):
        for rect, size in [(None, (31, 45)), ((1, 1, 5, 6), None), (None, None), ((0, 0, 6, 5), (64, 3))]:
            frames.append(f), rects.append(rect), sizes.append(size)
    for f in deep:
        frames += [f, f]
        rects += [None, None]
        sizes += [(20, 20), None]
    plain = _batch(built, ctx, frames, crop=rects)
    ref = _images(plain, _decode(plain))
    dec = _batch(built, ctx, frames, crop=rects, resize=sizes, resample="hamming")
    out = _decode(dec)
    got = _images(dec, out)
    for j, (r, s) in enumerate(zip(ref, sizes)):
        if r is not None and r.dtype != np.uint8 and s is not None:
            assert dec.status(j) == -1034
            assert got[j] is None and dec.frame_bytes(j) == 0
            continue
        assert dec.status(j) == plain.status(j), j
        if r is None:
            assert got[j] is None
            continue
        want = r if s is None else _resized(r, s, "hamming")
        assert np.array_equal(got[j], want), j
    # decode_into per-frame tensors: the same samples
    dst, live = [], []
    for j, geo in enumerate(dec.geometry()):
        if geo is None:
            dst.append(None)
            continue
        shapes, deep12 = geo
        t = torch.full((len(shapes),) + tuple(shapes[0]), 0x5A5A if deep12 else SENT, dtype=torch.int16 if deep12 else torch.uint8,
                       device="cuda")
        dst.append([t[c] for c in range(len(shapes))])
        live.append(j)
    dec.decode_into(dst)
    torch.cuda.synchronize()
    for j in live:
        a = torch.stack(dst[j]).cpu().numpy().transpose(1, 2, 0)
        assert np.array_equal(a.view(np.uint16) if a.dtype == np.int16 else a, got[j]), j
    # without tolerate_bad a 12-bit frame with a size fails the call
    from libjpeg_b200.decoder import BatchDecoder
    from libjpeg_b200.native import NativeError
    with pytest.raises(NativeError) as e:
        BatchDecoder([deep[0]], ctx=ctx, resize=(8, 8))
    assert e.value.code == -1034
    BatchDecoder([deep[0]], ctx=ctx, resize=[None]).close()


def test_decode_twice(built, ctx):
    import torch
    frames = [_synth(1000, 333, 70), _synth(640, 480, 71, (1, 1))] + SETS["baseline"]()[:3]
    dec = _batch(built, ctx, frames, resize=(57, 83), resample="lanczos")
    a = _decode(dec)
    b = _decode(dec)
    assert torch.equal(a, b)


def test_unchanged_plans_and_launches(built, ctx):
    """resize=None, all None and all (0, 0): the launches and every byte of the crop batch; with resized frames, the launches of
    the equivalent crop batch (whole-output rectangles where a resized frame has none) plus two"""
    import torch
    frames = SETS["baseline"]() + SETS["damaged"]() + SETS["progressive"]() + [_synth(1000, 333, 50), _synth(333, 1000, 51, (1, 1))]
    probe = _batch(built, ctx, frames)
    geo = probe.geometry()
    rects = [(1, 2, 3, 4) if i % 2 and g is not None and min(g[0][0]) >= 6 else None for i, g in enumerate(geo)]
    plain = _batch(built, ctx, frames, crop=rects)
    want = _decode(plain)
    for resize in (None, [None] * len(frames), [(0, 0)] * len(frames)):
        dec = _batch(built, ctx, frames, crop=rects, resize=resize)
        assert dec.out_bytes == plain.out_bytes
        got = _decode(dec)
        assert dec.launches == plain.launches
        assert torch.equal(got, want)
        assert [dec.status(i) for i in range(len(frames))] == [plain.status(i) for i in range(len(frames))]
    whole = []
    for r, g in zip(rects, geo):
        if r is None and g is not None:
            h, w = g[0][0]
            r = (0, 0, w, h)
        whole.append(r)
    crop_all = _batch(built, ctx, frames, crop=whole)
    _decode(crop_all)
    dec = _batch(built, ctx, frames, crop=rects, resize=(40, 30))
    _decode(dec)
    assert dec.launches == crop_all.launches + 2


def _create(built, ctx, frames, sizes, resample, flags=0, tolerate=0):
    from libjpeg_b200 import native
    n = len(frames)
    bufs = [ctypes.create_string_buffer(f, len(f)) for f in frames]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    table = (native.SizeStruct * n)()
    for i, (w, h) in enumerate(sizes):
        table[i].width, table[i].height = w, h
    handle = ctypes.c_void_p()
    rc = native.lib.b200jpg_batch_create_resize(ctx.handle, ptrs, lens, n, tolerate, flags, None, table, resample, ctypes.byref(handle))
    if rc == 0:
        native.lib.b200jpg_batch_destroy(handle)
    return rc, native.last_error(ctx.handle)[1]


def test_refused(built, ctx):
    """a half-zero size or an unknown filter fails the call with INVALID_PARAMETER naming the frame, tolerate_bad or not; a size with
    upsample=False is NOT_IMPLEMENTED; a size too large to allocate is OUT_OF_MEMORY; a failed frame's size is ignored"""
    from libjpeg_b200.decoder import BatchDecoder
    from libjpeg_b200.native import NativeError
    data = open(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"), "rb").read()
    for tol in (0, 1):
        for size in [(0, 5), (5, 0)]:
            rc, msg = _create(built, ctx, [data, data], [(0, 0), size], 2, tolerate=tol)
            assert rc == -1024 and "frame 1" in msg, (size, msg)
        for filt in (0, 6, -1):
            rc, msg = _create(built, ctx, [data, data], [(0, 0), (3, 3)], filt, tolerate=tol)
            assert rc == -1024 and "frame 1" in msg, (filt, msg)
    assert _create(built, ctx, [data], [(0, 0)], 0)[0] == 0  # no size: the filter is not looked at
    with pytest.raises(NativeError) as e:
        BatchDecoder([data], ctx=ctx, upsample=False, resize=(4, 4))
    assert e.value.code == -1034
    with pytest.raises(NativeError) as e:
        BatchDecoder([data], ctx=ctx, resize=(2 ** 24 + 1, 4))
    assert e.value.code == -2048
    dec = BatchDecoder([b"\xff\xd8\xff\xd9", data], ctx=ctx, tolerate_bad=True, resize=[(9, 9), (3, 4)])
    assert dec.output_shape(1, 0) == (3, 4) and dec.status(0) != 0
