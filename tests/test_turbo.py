"""GPU: BatchDecoder(reconstruction="libjpeg-turbo") / B200JPG_FLAG_LIBJPEG_TURBO (DESIGN §16). The oracle is the numpy model of
libjpeg-turbo's reconstruction (tests/turbo_model.py) on the oracle's coefficients, and for the stored vectors Pillow's own pixels
through tests/golden/turbo/pil_digests.json; every stage after the reconstruction through its existing model (orientation, crop,
resize, float map)."""
import hashlib
import itertools
import json
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import orientation_model as om
from tests import recon420_cases as r4c
from tests import recon_cases as rc
from tests import resize_model as rm
from tests import turbo_model as tm
from tests.test_decode_into import GOLDEN
from tests.test_orientation import _batch, _decode, _images, _synth

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED = -1034
TURBO = "libjpeg-turbo"
SENT = 0xA5
DIGESTS = json.load(open(os.path.join(GOLDEN, "turbo", "pil_digests.json")))


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


@pytest.fixture(scope="module")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()


def _files(d):
    base = os.path.join(GOLDEN, d)
    return [os.path.join(d, f) if d else f for f in sorted(os.listdir(base)) if f.endswith(".jpg")]


def _model(oracle, data, mode=None, color_transform=True):
    from libjpeg_b200 import decoder
    return tm.decode(oracle, data, decoder.colorspace(data), mode, color_transform)


def _check(built, ctx, oracle, frames, names=None, mode=None, color_transform=True):
    """packed decode with sentinels: every frame equals the model (and Pillow's digest where one is stored)"""
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode=mode, color_transform=color_transform)
    out = _decode(dec)
    got = _images(dec, out)
    for i, f in enumerate(frames):
        assert dec.status(i) == 0, i
        want = _model(oracle, f, mode, color_transform)
        assert np.array_equal(got[i], want), (names[i] if names else i)
        if names and names[i] in DIGESTS and mode is None and color_transform:
            g = got[i][..., 0] if got[i].shape[2] == 1 else got[i]
            assert list(g.shape) == DIGESTS[names[i]]["shape"]
            assert hashlib.sha256(np.ascontiguousarray(g).tobytes()).hexdigest() == DIGESTS[names[i]]["sha256"], names[i]
    mask = np.ones(out.numel(), dtype=bool)
    for i in range(len(frames)):
        mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


STORED = {"baseline": "", "progressive": "progressive", "subsampling": "subsampling", "reference": "reference", "xt": "xt",
          "dnl": "dnl"}


@pytest.mark.parametrize("name", list(STORED))
def test_stored_vectors(built, ctx, oracle, name):
    """every intact 8-bit vector of the set: Pillow's digest where Pillow reads it, the model everywhere (3x / 4x factors, more than
    10 blocks per MCU, DNL frames); a JPEG XT frame as its base codestream alone"""
    from libjpeg_b200 import decoder
    names = []
    for n in _files(STORED[name]):
        data = open(os.path.join(GOLDEN, n), "rb").read()
        try:
            if decoder.colorspace(data) in ("L", "YCbCr", "RGB"):
                names.append(n)
        except Exception:  # a JPEG XT profile the parser refuses keeps its status
            continue
    assert names
    _check(built, ctx, oracle, [open(os.path.join(GOLDEN, n), "rb").read() for n in names], names)
    if name in ("baseline", "progressive", "reference", "xt"):
        assert sum(n in DIGESTS for n in names) >= {"baseline": 14, "progressive": 7, "reference": 4, "xt": 11}[name]


@pytest.mark.parametrize("sub", [(2, 2), (2, 1), (1, 2), (1, 1), None])
def test_synthetic(built, ctx, oracle, sub):
    """every sampling the synthetic encoder writes, up to 1080p, with and without restart markers, w = 1, 2, 3 and odd sizes (the
    3x / 4x factors: the stored subsampling and reference vectors)"""
    from libjpeg_b200 import synth
    frames = []
    for k, (w, h) in enumerate([(1920, 1080), (1, 1), (2, 7), (3, 5), (33, 17), (517, 33), (35, 258), (256, 144)]):
        img = synth.source_image(w, h, 10 + k)
        frames.append(synth.encode(img[..., 0] if sub is None else img, 80, sub or (1, 1), k % 3).tobytes())
    _check(built, ctx, oracle, frames)


def _recon_names():
    return [n for n in rc.NAMES if rc.case(n)[0].precision == 8 and len(rc.case(n)[0].components) in (1, 3)]


def test_recon_cases(built, ctx, oracle):
    """the hand-built frames of tests/recon_cases.py and tests/recon420_cases.py: tile seams, saturated and wrapping samples,
    coefficients at the int16 edges"""
    names = _recon_names()
    _check(built, ctx, oracle, [rc.case(n)[1] for n in names], names)
    names4 = [n for n in r4c.NAMES if r4c.case(n)[0].precision == 8]
    _check(built, ctx, oracle, [r4c.case(n)[1] for n in names4], names4)


def _bound_frame(m):
    """a grey frame whose block (0, 1) has pass-1 results of magnitude m in every row, in the sign pattern that gives a pass-2 sum
    of L1 norm 61214 -- past int32 for m > 35079 -- and whose block (0, 2) has them at the int16 coefficient limit"""
    worst = None
    for signs in itertools.product((-1, 1), repeat=8):
        rec = []
        tm.idct1d(list(signs), tm.PASS2_SHIFT, rec)
        if max(abs(v) for v in rec) == 61214:
            worst = np.array(signs)
    w, h = 64, 16
    _, (y,) = rc.base(w, h, 91, rc.TILED["grey"])
    y[0, 1] = 0
    y[0, 1, 0, :] = worst * (m // 4)  # row 0 of the coefficients only: every pass-1 row is 4 x that row
    y[0, 2] = 0
    y[0, 2, 0, :] = worst * 32767
    return rc.frame(w, h, [y], rc.TILED["grey"])


def test_int32_bounds(built, ctx, oracle):
    """pass-1 results at the bound (int32 pass 2) and just past it (64-bit pass 2, where int32 would wrap): equal to the model.
    Whether Pillow agrees on these blocks (its SIMD islow keeps pass-1 results in 16 bits) is recorded, not asserted."""
    from tests import streamwriter as sw
    frames = [sw.encode(_bound_frame(m)) for m in (35076, 35080)]
    dec = _check(built, ctx, oracle, frames)
    try:
        import io
        from PIL import Image
        got = _images(dec, _decode(dec))
        agree = [bool(np.array_equal(np.asarray(Image.open(io.BytesIO(f))), g[..., 0])) for f, g in zip(frames, got)]
        print("Pillow agrees on the bound blocks:", agree)
    except ImportError:
        pass


def test_modes_and_no_color_transform(built, ctx, oracle):
    """mode "RGB" (grey replicated), mode "L" (YCbCr: component 0 upsampled, Pillow's draft("L"); RGB-coded: the L formula) and
    color_transform=False"""
    from tests.test_mode import adobe_rgb
    frames = [open(os.path.join(GOLDEN, n), "rb").read() for n in _files("")]
    frames += [adobe_rgb(_synth(97, 61, 3, (1, 1))), adobe_rgb(_synth(64, 40, 4, (2, 2))), _synth(35, 258, 5, (1, 2)),
               open(os.path.join(GOLDEN, "subsampling", "c410_97x53_z3_q75.jpg"), "rb").read()]
    for mode in ("RGB", "L"):
        _check(built, ctx, oracle, frames, mode=mode)
    _check(built, ctx, oracle, frames, color_transform=False)


def test_orientations_crops_resize(built, ctx, oracle):
    """all eight orientations, seam / edge / random crops and all five filters, packed: the model -> orient -> crop -> resize"""
    from libjpeg_b200 import synth
    src = [_synth(1000, 333, 21, (2, 2)), _synth(333, 517, 22, (2, 1)), _synth(97, 61, 23, (1, 2)), _synth(130, 70, 24, (1, 1)),
           synth.encode(synth.source_image(75, 61, 25)[..., 0], 85, (1, 1), 0).tobytes()]
    rng = np.random.default_rng(5)
    batch, rects, sizes, want = [], [], [], []
    for k, f in enumerate(src):
        for o in om.ORIENTATIONS:
            data = om.tag(f, o)
            img = om.orient(_model(oracle, data), o)
            oh, ow = img.shape[:2]
            for j, rect in enumerate([None] + cm.rectangles(ow, oh, rng, n_random=1)[-3:]):
                filt = sorted(rm.NAMES)[(k + o + j) % 5]
                size = None if j % 2 == 0 else (int(rng.integers(1, 80)), int(rng.integers(1, 80)))
                c = img if rect is None else img[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2]]
                batch.append(data), rects.append(rect), sizes.append(size)
                want.append((c if size is None else rm.resize(np.ascontiguousarray(c), size[1], size[0], rm.NAMES[filt]), filt))
    for filt in sorted(rm.NAMES):
        idx = [i for i, (_, fl) in enumerate(want) if fl == filt]
        dec = _batch(built, ctx, [batch[i] for i in idx], reconstruction=TURBO, exif_orientation=True, crop=[rects[i] for i in idx],
                     resize=[sizes[i] for i in idx], resample=filt)
        got = _images(dec, _decode(dec))
        for j, i in enumerate(idx):
            assert dec.status(j) == 0
            assert np.array_equal(got[j], want[i][0]), (filt, i)


def _fill(nbytes):
    import torch
    return torch.full((nbytes,), SENT, dtype=torch.uint8, device="cuda")


def _view_as_int(t):
    import torch
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def test_destinations(built, ctx, oracle):
    """decode_into [N, 3, 224, 224] uint8 / float32 / float16 / bfloat16, contiguous, padded and NHWC, sentinels around; the
    user path BatchDecoder(frames, reconstruction="libjpeg-turbo", mode="RGB", exif_orientation=True, crop=..., resize=(224, 224))"""
    import torch
    from libjpeg_b200 import synth
    src = [_synth(1000, 333, 40, (2, 2)), _synth(640, 480, 41, (1, 1)), _synth(333, 1000, 42, (2, 1)), _synth(97, 61, 43, (1, 2)),
           _synth(1920, 1080, 44), synth.encode(synth.source_image(120, 90, 45)[..., 0], 80, (1, 1), 0).tobytes()]
    frames = [om.tag(f, o) for f, o in zip(src, (1, 6, 3, 8, 1, 5))]
    rng = np.random.default_rng(9)
    th, tw = 224, 224
    batch, rects, want = [], [], []
    for f, o in zip(frames, (1, 6, 3, 8, 1, 5)):
        img = om.orient(_model(oracle, f, "RGB"), o)
        oh, ow = img.shape[:2]
        for rect in [None, (0, 0, ow, oh)] + cm.rectangles(ow, oh, rng, n_random=2)[-2:]:
            c = img if rect is None else img[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2]]
            batch.append(f), rects.append(rect), want.append(rm.resize(np.ascontiguousarray(c), tw, th, rm.NAMES["bilinear"]))
    dec = _batch(built, ctx, batch, reconstruction=TURBO, mode="RGB", exif_orientation=True, crop=rects, resize=(th, tw))
    n = len(batch)
    want_u8 = torch.from_numpy(np.stack(want)).permute(0, 3, 1, 2).contiguous().cuda()
    scale, bias = [1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225)], [-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225]
    for dtype in (torch.uint8, torch.float32, torch.float16, torch.bfloat16):
        for layout in ("nchw", "nhwc", "padded"):
            esz = torch.empty(0, dtype=dtype).element_size()
            if layout == "nchw":
                full_t = _fill(n * 3 * th * tw * esz).view(dtype).view(n, 3, th, tw)
                region = (slice(None),) * 4
                dst = full_t
            elif layout == "padded":
                full_t = _fill(n * 3 * (th + 2) * (tw + 3) * esz).view(dtype).view(n, 3, th + 2, tw + 3)
                region = (slice(None), slice(None), slice(1, th + 1), slice(1, tw + 1))
                dst = full_t[region]
            else:
                full_t = _fill(n * (th + 1) * (tw + 2) * 4 * esz).view(dtype).view(n, th + 1, tw + 2, 4)
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
    assert all(dec.status(i) == 0 for i in range(n))


def test_mixed_tolerant_batch(built, ctx, oracle):
    """grey, colour, RGB-coded, JPEG XT, damaged, 12-bit and CMYK frames in one tolerant batch: statuses as without the flag except
    NOT_IMPLEMENTED for the 12-bit and the four-component frames; the intact ones equal the model on the oracle's coefficients, the
    cut-off one the model on the coefficients this library decoded (rule 6)"""
    from tests.test_mode import adobe_rgb
    frames = [open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read(), _synth(130, 70, 61, (2, 2)),
              adobe_rgb(_synth(64, 48, 62, (1, 1))), open(os.path.join(GOLDEN, "xt", "xt_420_96x80_z6_q75_Q90.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "damaged", "trunc_c422_100x60.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "deep12", "d12_420_50x38_q60.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "cmyk", "cmyk_64x48_s0_q90.jpg"), "rb").read()]
    plain = _batch(built, ctx, frames)
    dec = _batch(built, ctx, frames, reconstruction=TURBO)
    got = _images(dec, _decode(dec))
    for i, f in enumerate(frames):
        if i >= 5:
            assert dec.status(i) == NOT_IMPLEMENTED and got[i] is None, i
            continue
        assert dec.status(i) == plain.status(i), i
        if i != 4:
            assert np.array_equal(got[i], _model(oracle, f)), i
        else:
            fi = dec.info(i)
            coef = [dec.coefficients(i, c).astype(np.int64) for c in range(fi.ncomp)]
            want = tm.reconstruct(coef, fi.width, fi.height, list(fi.hs), list(fi.vs), "YCbCr")
            assert np.array_equal(got[i], want), i
    # the same under mode "RGB", skipped frames and all, into one [N, 3, H, W] tensor after a resize
    import torch
    live = [f for i, f in enumerate(frames) if i < 4]
    dec = _batch(built, ctx, live, reconstruction=TURBO, mode="RGB", resize=(32, 48))
    dst = torch.zeros((len(live), 3, 32, 48), dtype=torch.uint8, device="cuda")
    dec.decode_into(dst)
    torch.cuda.synchronize()
    for i, f in enumerate(live):
        want = rm.resize(np.ascontiguousarray(_model(oracle, f, "RGB")), 48, 32, rm.NAMES["bilinear"])
        assert np.array_equal(dst[i].permute(1, 2, 0).cpu().numpy(), want), i


def test_decode_twice(built, ctx):
    frames = [_synth(517, 333, 71, (2, 2)), _synth(97, 61, 72, (2, 1))]
    dec = _batch(built, ctx, frames, reconstruction=TURBO)
    a, b = _decode(dec).cpu().numpy(), _decode(dec).cpu().numpy()
    assert np.array_equal(a, b)


def test_refused(built, ctx):
    """with downscale or upsample=False the call fails with NOT_IMPLEMENTED and creates nothing: the context's open batch count
    stays where it was"""
    from libjpeg_b200 import native
    frames = [_synth(64, 48, 81, (2, 2))]
    opened = ctx._batches
    for kw in ({"downscale": 2}, {"downscale": 8}, {"upsample": False}):
        with pytest.raises(native.NativeError) as e:
            built.BatchDecoder(frames, ctx=ctx, reconstruction=TURBO, **kw)
        assert e.value.code == NOT_IMPLEMENTED
    # a 12-bit frame without tolerate_bad fails the call
    with pytest.raises(native.NativeError) as e:
        built.BatchDecoder([open(os.path.join(GOLDEN, "deep12", "d12_444_64x64_z4_q95.jpg"), "rb").read()], ctx=ctx, reconstruction=TURBO)
    assert e.value.code == NOT_IMPLEMENTED
    assert ctx._batches == opened


@pytest.mark.parametrize("device", [False, True])
def test_one_call_entry_points(built, ctx, device):
    """the flag through b200jpg_decode_to_host_ex / b200jpg_decode_to_device_ex (b200jpg_batch_create_ex inside): the packed bytes of
    BatchDecoder(reconstruction="libjpeg-turbo")"""
    import ctypes
    import torch
    from libjpeg_b200 import native
    frames = [_synth(130, 70, 91, (2, 2)), open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read(), _synth(5, 3, 92, (2, 1))]
    dec = _batch(built, ctx, frames, reconstruction=TURBO)
    want = _decode(dec).cpu().numpy()[:dec.out_bytes]
    n = len(frames)
    bufs = [(ctypes.c_uint8 * len(f)).from_buffer_copy(f) for f in frames]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    flags = native.RECONSTRUCTION_FLAGS[TURBO]
    if not device:
        got = np.zeros(dec.out_bytes, dtype=np.uint8)
        native.check(native.lib.b200jpg_decode_to_host_ex(ctx.handle, ptrs, lens, n, got.ctypes.data, got.size, flags), ctx.handle)
    else:
        p, size = ctypes.c_void_p(), ctypes.c_uint64()
        native.check(native.lib.b200jpg_decode_to_device_ex(ctx.handle, ptrs, lens, n, flags, ctypes.byref(p), ctypes.byref(size)), ctx.handle)
        assert size.value == dec.out_bytes
        t = torch.empty(size.value, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        native.lib.b200jpg_device_copy_rect(ctx.handle, t.data_ptr(), size.value, p.value, size.value, size.value, 1)
        torch.cuda.synchronize()
        got = t.cpu().numpy()
    for i in range(n):
        a, b = dec.out_offset(i), dec.out_offset(i) + dec.frame_bytes(i)
        assert np.array_equal(got[a:b], want[a:b]), i

