"""GPU: BatchDecoder(mode="RGB" | "L") / B200JPG_FLAG_OUTPUT_RGB and B200JPG_FLAG_OUTPUT_L (DESIGN §14). The oracle is always the
same library without the mode: "L" of a YCbCr frame is component 0 of the color_transform=False decode of the same batch
configuration, "L" of an RGB-coded or JPEG XT frame the L formula applied by numpy to the decode without the mode, "RGB" of a grey
frame its decode without the mode three times, and every other frame is byte-identical to the decode without the mode."""
import ctypes

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om
from tests import resize_model as rm
from tests.test_crop import CROP_SETS
from tests.test_decode_into import GOLDEN, SETS
from tests.test_orientation import _batch, _decode, _images, _synth

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED, INVALID = -1034, -1024
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def luma(rgb):
    """the L formula on clamped samples (tests/test_mode_cpu.py pins it to PIL's convert("L") on every triple)"""
    rgb = rgb.astype(np.int64)
    return (19595 * rgb[..., 0] + 38470 * rgb[..., 1] + 7471 * rgb[..., 2] + 32768) >> 16


def adobe_rgb(data):
    """the codestream with an Adobe APP14 segment of transform 0 behind SOI: its three components are R, G, B"""
    return data[:2] + b"\xff\xee\x00\x0e" + b"Adobe" + bytes([0, 100, 0, 0, 0, 0, 0]) + data[2:]


def _grey(w, h, seed, restart=0):
    from libjpeg_b200 import synth
    return synth.encode(synth.source_image(w, h, seed)[..., 0], 85, (1, 1), restart).tobytes()


def _expected(built, ctx, frames, mode, xt=False, **kw):
    """per frame the image the batch with `mode` must write, from decodes of the same configuration without it; and the statuses"""
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    nct = None
    want, status = [], []
    for i, r in enumerate(ref):
        st = plain.status(i)
        if r is None:
            want.append(None), status.append(st)
            continue
        nc = r.shape[2]
        if nc not in (1, 3):
            want.append(None), status.append(NOT_IMPLEMENTED)
            continue
        status.append(st)
        if mode == "RGB":
            want.append(np.repeat(r, 3, axis=2) if nc == 1 else r)
        elif nc == 1:
            want.append(r)
        elif plain.info(i).ycbcr and not xt:
            if nct is None:
                d = _batch(built, ctx, frames, color_transform=False, **kw)
                nct = _images(d, _decode(d))
            want.append(nct[i][..., :1])
        else:
            want.append(luma(r)[..., None].astype(r.dtype))
    return want, status


def _check(built, ctx, frames, mode, xt=False, **kw):
    want, status = _expected(built, ctx, frames, mode, xt, **kw)
    dec = _batch(built, ctx, frames, mode=mode, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    for i, w in enumerate(want):
        assert dec.status(i) == status[i], "frame %d" % i
        if w is None:
            assert got[i] is None or status[i] != 0 or dec.status(i) != 0
            continue
        assert dec.output_components(i) == w.shape[2]
        assert np.array_equal(got[i], w), "frame %d" % i
    mask = np.ones(out.numel(), dtype=bool)
    for i in range(len(frames)):
        mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


MODE_SETS = dict(CROP_SETS)
MODE_SETS["grey"] = lambda: [_read(GOLDEN + "/g_40x24_z2_q75.jpg"), _read(GOLDEN + "/progressive/pg_40x24_z2_q75.jpg"),
                             _read(GOLDEN + "/xt/xt_g_40x24_q75_Q90.jpg"), _grey(1920, 1080, 1), _grey(517, 300, 2, restart=3), _grey(33, 257, 3)]
MODE_SETS["rgb_coded"] = lambda: [adobe_rgb(_synth(300, 200, 5, (1, 1))), adobe_rgb(_synth(517, 301, 6, (2, 2))),
                                  adobe_rgb(_read(GOLDEN + "/deep12/d12_444_64x64_z4_q95.jpg")),
                                  adobe_rgb(_read(GOLDEN + "/deep12/d12_420_96x80_z3_q80.jpg"))]


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("name", list(MODE_SETS))
def test_sets(built, ctx, name, mode):
    _check(built, ctx, MODE_SETS[name](), mode, xt=name == "xt")


MIXED = lambda: ([_grey(640, 480, 11), _synth(700, 301, 12), _synth(301, 700, 13, (1, 1)), _synth(500, 260, 14, (2, 1)),
                  adobe_rgb(_synth(200, 120, 15, (1, 1)))] + SETS["subsampling"]()[:2] + SETS["baseline"]()[:2])


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_downscale_and_orientations(built, ctx, k, mode):
    frames = [om.tag(f, o) for f in MIXED() for o in om.ORIENTATIONS]
    _check(built, ctx, frames, mode, downscale=k, exif_orientation=True)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_crops(built, ctx, mode):
    frames, rects = [], []
    rng = np.random.default_rng(5)
    for f in MIXED():
        for o in (1, 6):
            tagged = om.tag(f, o)
            from libjpeg_b200 import decoder
            h, w = decoder.output_size(tagged, exif_orientation=True)
            for r in cm.rectangles(w, h, rng, n_random=2)[-3:]:
                frames.append(tagged), rects.append(r)
    _check(built, ctx, frames, mode, crop=rects, exif_orientation=True)


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("resample", ["bilinear", "bicubic", "lanczos"])
def test_resize(built, ctx, mode, resample):
    """the mode before the resize: the model applied to the mode's image of the crop decode"""
    frames = MIXED()
    rng = np.random.default_rng(len(resample))
    want, _ = _expected(built, ctx, frames, mode)
    rects = [cm.rectangles(w.shape[1], w.shape[0], rng, n_random=1)[-1] for w in want]
    sizes = [(int(rng.integers(1, 300)), int(rng.integers(1, 300))) for _ in frames]
    dec = _batch(built, ctx, frames, mode=mode, crop=rects, resize=sizes, resample=resample)
    got = _images(dec, _decode(dec))
    for i, (w, r, s) in enumerate(zip(want, rects, sizes)):
        c = w[r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        assert np.array_equal(got[i], rm.resize(c, s[1], s[0], rm.NAMES[resample])), "frame %d" % i


def test_four_components_refused_per_frame(built, ctx):
    from tests import recon_cases
    four = [recon_cases.case(n)[1] for n in recon_cases.NAMES if recon_cases.case(n)[1] and _ncomp(built, recon_cases.case(n)[1]) in (2, 4)]
    assert four
    frames = four + [_grey(64, 48, 1), _synth(64, 48, 2)]
    for mode in ("L", "RGB"):
        dec = _batch(built, ctx, frames, mode=mode)
        assert [dec.status(i) for i in range(len(four))] == [NOT_IMPLEMENTED] * len(four)
        assert _refused(built, frames, ctx=ctx, mode=mode) == NOT_IMPLEMENTED
    _check(built, ctx, frames, "L")


def _refused(built, frames, **kw):
    """the error code of a batch that must not be created. (No exception info is kept: a traceback held by a test's frame ties
    the context into a reference cycle, and the garbage collector may then finalise it before batches that still use it.)"""
    try:
        built.BatchDecoder(frames, **kw).close()
    except built.native.NativeError as err:
        return err.code
    return None


def _ncomp(built, data):
    from libjpeg_b200 import decoder
    return decoder.parse(data).ncomp


def test_refused_requests(built, ctx):
    frames = [_synth(64, 48, 1)]
    for kw, code in [(dict(mode="L", color_transform=False), INVALID), (dict(mode="RGB", color_transform=False), INVALID),
                     (dict(mode="L", upsample=False), NOT_IMPLEMENTED), (dict(mode="RGB", upsample=False), NOT_IMPLEMENTED)]:
        assert _refused(built, frames, ctx=ctx, **kw) == code, kw
    lib, h = built.native.lib, ctypes.c_void_p()
    ptrs, lens = (ctypes.c_void_p * 1)(), (ctypes.c_size_t * 1)(len(frames[0]))
    buf = ctypes.create_string_buffer(frames[0], len(frames[0]))
    ptrs[0] = ctypes.addressof(buf)
    assert lib.b200jpg_batch_create_ex(ctx.handle, ptrs, lens, 1, 0, 0x60, ctypes.byref(h)) == INVALID
    assert not h.value


def test_modeless_plans_unchanged(built, ctx):
    """a mode that changes no frame plans the batch without it: launches, bytes, offsets"""
    for frames, mode in [([_synth(700, 301, 1), _synth(300, 200, 2, (1, 1)), _synth(300, 200, 3, (2, 1))], "RGB"),
                         ([_grey(700, 301, 4), _read(GOLDEN + "/g_40x24_z2_q75.jpg")], "L")]:
        a, b = _batch(built, ctx, frames), _batch(built, ctx, frames, mode=mode)
        oa, ob = _decode(a), _decode(b)
        assert a.launches == b.launches and a.h2d_bytes == b.h2d_bytes and a.out_bytes == b.out_bytes
        assert [a.out_offset(i) for i in range(len(frames))] == [b.out_offset(i) for i in range(len(frames))]
        assert bool((oa == ob).all())


def test_luma_skips_the_fused_420_kernel(built, ctx):
    """an L batch of 4:2:0 frames reconstructs like a batch of grey frames: one launch (no reconstruct420_kernel, no exact pass)"""
    c420 = [_synth(1920, 1080, 1), _synth(640, 480, 2), _synth(257, 33, 3)]
    grey = [_grey(1920, 1080, 1), _grey(640, 480, 2), _grey(257, 33, 3)]
    counts = []
    for frames, kw in [(c420, {}), (c420, dict(mode="L")), (grey, {})]:
        dec = _batch(built, ctx, frames, **kw)
        out = dec.new_output()
        dec.decode_entropy()
        dec.reconstruct(out)
        counts.append(dec.launches)
    assert counts[1] == counts[2] == 1 and counts[0] == 3, counts


def test_range_edge_frames(built, ctx):
    """the hand-built 4:2:0 frames, some of whose chroma forces the int32 exact pass, with tiled ones in one batch: their L decode
    is still component 0"""
    from tests import recon420_cases as r4
    _check(built, ctx, [r4.case(n)[1] for n in r4.NAMES] + CROP_SETS["recon"]()[:20], "L")


def test_decode_into_mixed_batch(built, ctx):
    """one [N, 3, 224, 224] tensor from a tolerant batch of grey, colour, RGB-coded, damaged and unparseable frames with per-frame
    crops and resizes: uint8, and fp16 / bf16 / fp32 with the ImageNet map equal to the uint8 result converted by torch; NHWC and
    padded destinations with sentinels"""
    import torch
    frames = MIXED() + SETS["damaged"]()[:3] + [b"\xff\xd8\xff\xd9", _read(GOLDEN + "/g_40x24_z2_q75.jpg")]
    rng = np.random.default_rng(9)
    from libjpeg_b200 import decoder
    rects = []
    for f in frames:
        try:
            h, w = decoder.output_size(f)
            rects.append(cm.rectangles(w, h, rng, n_random=1)[-1])
        except Exception:
            rects.append(None)
    dec = _batch(built, ctx, frames, mode="RGB", crop=rects, resize=(224, 224))
    n, live = len(frames), [i for i in range(len(frames)) if dec.geometry()[i] is not None]
    assert len(live) < n and all(dec.output_components(i) == 3 for i in live)
    packed = _images(dec, _decode(dec))
    u8 = torch.full((n, 3, 224, 224), 0x5A, dtype=torch.uint8, device="cuda")
    dec.decode_into([list(u8[i]) if i in live else None for i in range(n)])
    torch.cuda.synchronize()
    for i in live:
        assert np.array_equal(u8[i].permute(1, 2, 0).cpu().numpy(), packed[i]), i
    scale = [1.0 / (255.0 * s) for s in STD]
    bias = [-m / s for m, s in zip(MEAN, STD)]
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        t = torch.full((n, 3, 224, 224), 7.0, dtype=dtype, device="cuda")
        dec.decode_into([list(t[i]) if i in live else None for i in range(n)], scale=scale, bias=bias)
        ref = (u8.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) + torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
        for i in range(n):
            if i in live:
                assert torch.equal(t[i], ref[i]), (dtype, i)
            else:
                assert bool((t[i] == 7.0).all()), (dtype, i)
    nhwc = torch.full((n, 224, 224, 3), 0x5A, dtype=torch.uint8, device="cuda")
    dec.decode_into([list(nhwc[i].permute(2, 0, 1)) if i in live else None for i in range(n)])
    padded = torch.full((n, 3, 230, 240), 0x5A, dtype=torch.uint8, device="cuda")
    dec.decode_into([list(padded[i, :, 3:227, 5:229]) if i in live else None for i in range(n)])
    torch.cuda.synchronize()
    for i in live:
        assert np.array_equal(nhwc[i].cpu().numpy(), packed[i]), i
        assert np.array_equal(padded[i, :, 3:227, 5:229].permute(1, 2, 0).cpu().numpy(), packed[i]), i
    inner = torch.zeros_like(padded, dtype=torch.bool)
    inner[:, :, 3:227, 5:229] = True
    assert bool((padded[~inner] == 0x5A).all())
    for i in set(range(n)) - set(live):
        assert bool((nhwc[i] == 0x5A).all()) and bool((padded[i] == 0x5A).all())


def test_batch_tensor(built, ctx):
    """mode="RGB" fills one [N, 3, H, W] tensor from grey and colour frames of one size; mode="L" one [N, 1, H, W]"""
    import torch
    frames = [_grey(320, 240, 1), _synth(320, 240, 2), _synth(320, 240, 3, (1, 1)), adobe_rgb(_synth(320, 240, 4, (2, 1)))]
    for mode, c in (("RGB", 3), ("L", 1)):
        want, _ = _expected(built, ctx, frames, mode)
        dec = _batch(built, ctx, frames, mode=mode)
        t = torch.zeros((4, c, 240, 320), dtype=torch.uint8, device="cuda")
        dec.decode_into(t)
        torch.cuda.synchronize()
        for i in range(4):
            assert np.array_equal(t[i].permute(1, 2, 0).cpu().numpy(), want[i]), (mode, i)
