"""GPU: BatchDecoder(crop=...) / b200jpg_batch_create_crop. The oracle is the uncropped decode of the same batch configuration
(itself pinned to the reference by the other suites), sliced by numpy, bit for bit; every frame's status is that of the uncropped
batch, and nothing outside a rectangle's destination is written."""
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om
from tests.test_decode_into import GOLDEN, SETS
from tests.test_orientation import ORIENT_SETS, _batch, _decode, _images, _synth, _view_as_int

pytestmark = pytest.mark.gpu

SENT = 0xA5
CROP_SETS = dict(ORIENT_SETS)
CROP_SETS["synth_formats"] = lambda: [_synth(1920, 1080, 31), _synth(1000, 333, 32, (2, 1)), _synth(333, 1000, 33, (1, 2)),
                                      _synth(1000, 333, 34, (1, 1)), _synth(777, 301, 35, (2, 2), restart=3)]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _sub(info):
    return max(info.subx), max(info.suby)


def _check_packed(built, ctx, frames, seed=0, n_random=4, **kw):
    """Every live frame under the rectangles of crop_model.rectangles and once uncropped (None), failed frames with a rectangle
    that is ignored, all in one batch: decode() equals the uncropped batch's output sliced, statuses agree, and no byte outside
    the slots is written."""
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(seed)
    batch, rects, src = [], [], []
    for i, f in enumerate(frames):
        if ref[i] is None:
            batch.append(f), rects.append((1, 1, 1, 1)), src.append(i)
            continue
        oh, ow = ref[i].shape[:2]
        for r in [None] + cm.rectangles(ow, oh, rng, n_random=n_random, sub=_sub(plain.info(i))):
            batch.append(f), rects.append(r), src.append(i)
    dec = _batch(built, ctx, batch, crop=rects, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    live = 0
    for j, (i, r) in enumerate(zip(src, rects)):
        assert dec.status(j) == plain.status(i), "frame %d (source %d, rectangle %s)" % (j, i, r)
        if ref[i] is None:
            assert got[j] is None
            continue
        want = ref[i] if r is None else ref[i][r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        assert dec.output_shape(j, 0) == want.shape[:2]
        assert np.array_equal(got[j], want), "frame %d (source %d, rectangle %s)" % (j, i, r)
        live += 1
    assert live > 0
    mask = np.ones(out.numel(), dtype=bool)
    for j in range(len(batch)):
        mask[dec.out_offset(j):dec.out_offset(j) + dec.frame_bytes(j)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"


@pytest.mark.parametrize("name", list(CROP_SETS))
def test_packed(built, ctx, name):
    _check_packed(built, ctx, CROP_SETS[name]())


@pytest.mark.parametrize("k", [2, 4, 8])
def test_downscale(built, ctx, k):
    frames = SETS["baseline"]() + SETS["deep12"]() + SETS["subsampling"]() + [_synth(1920, 1080, 7), _synth(333, 1000, 8, (1, 1)),
                                                                              _synth(1000, 333, 9, (2, 1))]
    _check_packed(built, ctx, frames, seed=k, downscale=k)


def test_no_color_transform(built, ctx):
    frames = SETS["baseline"]() + SETS["subsampling"]() + SETS["deep12"]() + [_synth(1000, 333, 10), _synth(300, 200, 11, (1, 2))]
    _check_packed(built, ctx, frames, seed=3, color_transform=False)


@pytest.mark.parametrize("k", [1, 2])
def test_orientations(built, ctx, k):
    """all eight orientations, the rectangle given in oriented output coordinates (downscale -> orientation -> crop)"""
    src = [_synth(700, 301, 12), _synth(301, 700, 13, (1, 1)), _synth(500, 260, 14, (2, 1)), _synth(260, 500, 15, (1, 2))]
    src += SETS["deep12"]()[:2] + SETS["subsampling"]()[:2] + [SETS["baseline"]()[0]]
    frames = [om.tag(f, o) for f in src for o in om.ORIENTATIONS]
    _check_packed(built, ctx, frames, seed=20 + k, n_random=2, exif_orientation=True, downscale=k)


@pytest.mark.parametrize("orient", [1, 3, 6])
def test_destinations(built, ctx, orient):
    """decode_into: uint8 into [N, C, h, w] (contiguous, and with padded rows at an odd offset), an NHWC view, and float32 /
    float16 / bfloat16 into [N, C, h, w] and NHWC with a per-component map; one rectangle size at many origins (the data loader's
    random crop) over the Fused420, Tiled 4:4:4 / 4:2:2 / 4:4:0 and grey paths; nothing outside the rectangles is written"""
    import torch
    src = [_synth(1000, 333, 40, (2, 2)), _synth(1000, 333, 41, (1, 1)), _synth(1000, 333, 42, (2, 1)), _synth(1000, 333, 43, (1, 2))]
    frames = [om.tag(f, orient) for f in src]
    plain = _batch(built, ctx, frames, exif_orientation=True)
    ref = _images(plain, _decode(plain))
    oh, ow = ref[0].shape[:2]
    rw, rh = 97, 61
    origins = [(0, 0), (ow - rw, oh - rh), (255, 7), (256, 31), (257, 33), (5, oh - rh - 1), (ow - rw - 9, 64)]
    origins = [(min(x, ow - rw), min(y, oh - rh)) for x, y in origins]  # (orientation 6: a 333-wide output)
    batch, rects, want = [], [], []
    for f, r in zip(frames, ref):
        for x, y in origins:
            batch.append(f), rects.append((x, y, rw, rh)), want.append(r[y:y + rh, x:x + rw])
    want_u8 = torch.from_numpy(np.stack(want)).permute(0, 3, 1, 2).contiguous().cuda()
    dec = _batch(built, ctx, batch, crop=rects, exif_orientation=True)
    n = len(batch)
    assert [dec.output_shape(i, 0) for i in range(n)] == [(rh, rw)] * n
    scale, bias = [1 / 58.4, 1 / 57.1, 1 / 57.4], [-2.1, -2.0, -1.8]
    cases = [(torch.uint8, "nchw"), (torch.uint8, "padded"), (torch.uint8, "nhwc")]
    cases += [(dt, lay) for dt in (torch.float32, torch.float16, torch.bfloat16) for lay in ("nchw", "nhwc", "padded")]
    for dtype, layout in cases:
        esz = torch.empty(0, dtype=dtype).element_size()
        if layout == "nchw":
            buf = torch.full((n * 3 * rh * rw * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, 3, rh, rw)
            dst, region = full_t, (slice(None),) * 4
        elif layout == "padded":
            buf = torch.full((n * 3 * (rh + 2) * (rw + 3) * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, 3, rh + 2, rw + 3)
            region = (slice(None), slice(None), slice(1, rh + 1), slice(1, rw + 1))
            dst = full_t[region]
        else:
            buf = torch.full((n * (rh + 1) * (rw + 2) * 4 * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, rh + 1, rw + 2, 4)
            region = (slice(None), slice(0, rh), slice(1, rw + 1), slice(0, 3))
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
            assert dec.status(i) == plain.status(i // len(origins))


def test_generic_and_deep_into_planes(built, ctx):
    """12-bit (generic kernels, int16 samples) and generic-format frames into per-frame [C, h, w] tensors inside sentinel-filled
    padded buffers"""
    import torch
    frames = SETS["deep12"]() + SETS["subsampling"]() + SETS["xt"]()
    plain = _batch(built, ctx, frames)
    ref = _images(plain, _decode(plain))
    rng = np.random.default_rng(5)
    batch, rects, src = [], [], []
    for i, (f, r) in enumerate(zip(frames, ref)):
        if r is None:
            continue
        for rect in cm.rectangles(r.shape[1], r.shape[0], rng, n_random=2)[::3]:
            batch.append(f), rects.append(rect), src.append(i)
    dec = _batch(built, ctx, batch, crop=rects)
    bufs, dst = [], []
    for j, geo in enumerate(dec.geometry()):
        shapes, deep = geo
        h, w = shapes[0]
        dt = torch.int16 if deep else torch.uint8
        full = torch.full((len(shapes), h + 2, w + 3), SENT if not deep else 0x5A5A, dtype=dt, device="cuda")
        bufs.append(full)
        dst.append([full[c, 1:h + 1, 2:w + 2] for c in range(len(shapes))])
    dec.decode_into(dst)
    torch.cuda.synchronize()
    for j, (i, (x, y, w, h)) in enumerate(zip(src, rects)):
        want = ref[i][y:y + h, x:x + w]
        full = bufs[j].cpu().numpy()
        if want.dtype == np.uint16:
            full = full.view(np.uint16)
        got = full[:, 1:h + 1, 2:w + 2].transpose(1, 2, 0)
        assert np.array_equal(got, want), (j, rects[j])
        outside = np.ones(full.shape, dtype=bool)
        outside[:, 1:h + 1, 2:w + 2] = False
        assert (full[outside] == (0x5A5A if want.dtype == np.uint16 else SENT)).all()
        assert dec.status(j) == plain.status(i)


def test_unchanged_plans(built, ctx):
    """rects == NULL, all {0, 0, 0, 0} and all None: the launches and every output byte of b200jpg_batch_create_ex"""
    import torch
    frames = SETS["baseline"]() + SETS["damaged"]() + SETS["progressive"]() + [_synth(1000, 333, 50), _synth(333, 1000, 51, (1, 1))]
    plain = _batch(built, ctx, frames)
    want = _decode(plain)
    for crop in (None, [None] * len(frames), [(0, 0, 0, 0)] * len(frames)):
        dec = _batch(built, ctx, frames, crop=crop)
        assert dec.out_bytes == plain.out_bytes
        got = _decode(dec)
        assert dec.launches == plain.launches
        assert torch.equal(got, want)
        assert [dec.status(i) for i in range(len(frames))] == [plain.status(i) for i in range(len(frames))]


def test_refused(built, ctx):
    """empty, out-of-range and overflowing rectangles fail the call with B200JPG_ERR_INVALID_PARAMETER naming the frame, tolerate_bad
    or not; a rectangle with upsample=False is B200JPG_ERR_NOT_IMPLEMENTED; a failed frame's rectangle is ignored"""
    from libjpeg_b200.decoder import BatchDecoder
    from libjpeg_b200.native import NativeError
    data = open(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"), "rb").read()
    bad = [(0, 0, 0, 1), (0, 0, 1, 0), (5, 5, 0, 0), (96, 0, 1, 1), (0, 80, 1, 1), (90, 0, 7, 1), (0, 0, 97, 80), (0, 0, 96, 81),
           (2 ** 32 - 1, 0, 2, 1), (0, 2 ** 32 - 1, 1, 2), (1, 1, 2 ** 32 - 1, 1)]
    for rect in bad:
        for tol in (False, True):
            with pytest.raises(NativeError) as e:
                BatchDecoder([data, data], ctx=ctx, tolerate_bad=tol, crop=[None, rect])
            assert e.value.code == -1024 and "frame 1" in e.value.message, (rect, e.value.message)
    with pytest.raises(NativeError) as e:
        BatchDecoder([data], ctx=ctx, upsample=False, crop=[(0, 0, 1, 1)])
    assert e.value.code == -1034
    BatchDecoder([data], ctx=ctx, upsample=False, crop=[(0, 0, 0, 0)]).close()  # no rectangle: allowed
    # the bounds are those of the oriented, downscaled output
    t6 = om.tag(data, 6)
    BatchDecoder([t6], ctx=ctx, exif_orientation=True, crop=[(0, 0, 80, 96)]).close()
    with pytest.raises(NativeError):
        BatchDecoder([t6], ctx=ctx, exif_orientation=True, crop=[(0, 0, 96, 80)])
    BatchDecoder([data], ctx=ctx, downscale=8, crop=[(11, 9, 1, 1)]).close()
    with pytest.raises(NativeError):
        BatchDecoder([data], ctx=ctx, downscale=8, crop=[(12, 0, 1, 1)])
    # a frame that fails to parse: its rectangle is ignored
    dec = BatchDecoder([b"\xff\xd8\xff\xd9", data], ctx=ctx, tolerate_bad=True, crop=[(500, 500, 9, 9), (1, 2, 3, 4)])
    assert dec.output_shape(1, 0) == (4, 3)
    assert dec.status(0) != 0
