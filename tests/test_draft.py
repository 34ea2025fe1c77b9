"""GPU: BatchDecoder(reconstruction="libjpeg-turbo", draft=...) / b200jpg_batch_create_draft (DESIGN §17). The oracle is the numpy
model of libjpeg-turbo's reduced decode (tests/draft_model.py) on the oracle's coefficients, and for the stored vectors Pillow's own
drafted pixels through tests/golden/turbo/draft_digests.json; every stage after the reconstruction through its existing model
(orientation, crop, resize, float map)."""
import hashlib
import itertools
import json
import os

import numpy as np
import pytest

from tests import crop_model as cm
from tests import draft_model as dm
from tests import orientation_model as om
from tests import recon420_cases as r4c
from tests import recon_cases as rc
from tests import resize_model as rm
from tests.test_decode_into import GOLDEN
from tests.test_orientation import _batch, _decode, _images, _synth

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED = -1034
INVALID_PARAMETER = -1024
TURBO = "libjpeg-turbo"
SENT = 0xA5
DIGESTS = json.load(open(os.path.join(GOLDEN, "turbo", "draft_digests.json")))


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


def _request(data, k):
    """the draft (h, w) of make_draft.py's request for 1/k"""
    from libjpeg_b200 import decoder
    fi = decoder.parse(data)
    return max(1, fi.height // k), max(1, fi.width // k)


def _model(oracle, data, req, mode=None, color_transform=True):
    from libjpeg_b200 import decoder
    k = decoder.draft_scale(data, req)
    return dm.decode(oracle, data, decoder.colorspace(data), k, mode, color_transform)


def _check(built, ctx, oracle, frames, drafts, names=None, mode=None, color_transform=True):
    """packed decode with sentinels: every frame equals the model (and Pillow's digest where one is stored)"""
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode=mode, color_transform=color_transform, draft=drafts)
    out = _decode(dec)
    got = _images(dec, out)
    for i, f in enumerate(frames):
        assert dec.status(i) == 0, i
        want = _model(oracle, f, drafts[i], mode, color_transform)
        assert np.array_equal(got[i], want), (names[i] if names else i, drafts[i])
        if names and mode and color_transform:
            from libjpeg_b200 import decoder
            k = decoder.draft_scale(f, drafts[i])
            key = [key for key in ("%s|%s|%d" % (names[i], mode, kk) for kk in (2, 4, 8)) if DIGESTS.get(key, {}).get("scale") == k]
            if key:
                g = got[i][..., 0] if got[i].shape[2] == 1 else got[i]
                assert list(g.shape) == DIGESTS[key[0]]["shape"]
                assert hashlib.sha256(np.ascontiguousarray(g).tobytes()).hexdigest() == DIGESTS[key[0]]["sha256"], key[0]
    mask = np.ones(out.numel(), dtype=bool)
    for i in range(len(frames)):
        mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


STORED = {"baseline": "", "progressive": "progressive", "subsampling": "subsampling", "reference": "reference", "xt": "xt",
          "dnl": "dnl"}


@pytest.mark.parametrize("name", list(STORED))
def test_stored_vectors(built, ctx, oracle, name):
    """every intact 8-bit vector of the set at k = 2, 4 and 8 under modes "RGB" and "L": Pillow's digest where Pillow reads it, the
    model everywhere (3x / 4x factors, more than 10 blocks per MCU, DNL frames, JPEG XT base codestreams)"""
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
    frames = [open(os.path.join(GOLDEN, n), "rb").read() for n in names]
    checked = 0
    for k in (2, 4, 8):
        drafts = [_request(f, k) for f in frames]
        for mode in ("RGB", "L"):
            _check(built, ctx, oracle, frames, drafts, names, mode=mode)
            checked += sum("%s|%s|%d" % (n, mode, k) in DIGESTS for n in names)
    if name in ("baseline", "progressive", "reference", "xt"):
        assert checked >= 6 * {"baseline": 14, "progressive": 7, "reference": 4, "xt": 11}[name]


@pytest.mark.parametrize("sub", [(2, 2), (2, 1), (1, 2), (1, 1), None])
def test_synthetic(built, ctx, oracle, sub):
    """every sampling the synthetic encoder writes, up to 1080p, with and without restart markers, at every scale in one batch"""
    from libjpeg_b200 import synth
    frames, drafts = [], []
    for j, (w, h) in enumerate([(1920, 1080), (1, 1), (2, 7), (3, 5), (33, 17), (517, 33), (35, 258), (256, 144), (131, 67)]):
        img = synth.source_image(w, h, 10 + j)
        f = synth.encode(img[..., 0] if sub is None else img, 80, sub or (1, 1), j % 3).tobytes()
        for k in (2, 4, 8):
            frames.append(f), drafts.append((max(1, h // k), max(1, w // k)))
    _check(built, ctx, oracle, frames, drafts)


def test_recon_cases(built, ctx, oracle):
    """the hand-built frames of tests/recon_cases.py and tests/recon420_cases.py at every scale: saturated and wrapping samples,
    coefficients at the int16 edges, every component layout"""
    names = [n for n in rc.NAMES if rc.case(n)[0].precision == 8 and len(rc.case(n)[0].components) in (1, 3)]
    names4 = [n for n in r4c.NAMES if r4c.case(n)[0].precision == 8]
    frames = [rc.case(n)[1] for n in names] + [r4c.case(n)[1] for n in names4]
    for k in (2, 4, 8):
        _check(built, ctx, oracle, frames, [_request(f, k) for f in frames], names + names4)


def _worst(line, shift, n_in):
    best, arg = -1, None
    for signs in itertools.product((-1, 1), repeat=len(n_in)):
        d = [0] * 8
        for i, s in zip(n_in, signs):
            d[i] = s
        rec = []
        line(d, shift, rec)
        if max(abs(v) for v in rec) > best:
            best, arg = max(abs(v) for v in rec), np.array(d)
    return arg


def _bound_frame(line, n_in, p1, p2, m1, m2):
    """a grey frame: block (0, 1) has column 1 at magnitude m1 in the sign pattern of the largest pass-1 sum (an odd column: a pass-1
    result that wrapped in int32 would change the bytes, tests/test_draft_cpu.py::test_bound_blocks_observable), block (0, 2) pass-1
    results of magnitude m2 in every row in the pattern of the largest pass-2 sum (row 0 only: each pass-1 result is 4 x it), block
    (0, 3) that pattern at the int16 limit. A pass-2 wrap (2^32 >> 19 or >> 20) is a multiple of 1024 and cannot show through the
    range-limit table, so only the pass-1 choice is observable in the output; the pass-2 blocks check the 64-bit pass itself."""
    w, h = 64, 16
    _, (y,) = rc.base(w, h, 93, rc.TILED["grey"])
    y[0, 1:4] = 0
    y[0, 1, :, 1] = _worst(line, p1, n_in) * m1
    y[0, 2, 0, :] = _worst(line, p2, n_in) * (m2 // 4)
    y[0, 3, 0, :] = _worst(line, p2, n_in) * 32767
    return rc.frame(w, h, [y], rc.TILED["grey"])


def test_int32_bounds(built, ctx, oracle):
    """blocks on both sides of the pass-1 and pass-2 bounds of jpeg_idct_4x4 (k = 2) and jpeg_idct_2x2 (k = 4): int32 at the bound,
    64 bits past it, equal to the model either way. Whether Pillow agrees on these blocks (its SIMD reduced IDCTs keep 16-bit
    intermediates) is recorded, not asserted."""
    from tests import streamwriter as sw
    cases = []
    for k, line, n_in, p1, p2, b1, b2 in ((2, dm.red4_line, (0, 1, 2, 3, 5, 6, 7), 12, 19, 27563, 27560),
                                          (4, dm.red2_line, (0, 1, 3, 5, 7), 13, 20, 25040, 25034)):
        for d1, d2 in ((0, 0), (1, 4)):
            cases.append((k, sw.encode(_bound_frame(line, n_in, p1, p2, b1 + d1, b2 + d2))))
    frames = [f for _, f in cases]
    drafts = [_request(f, k) for k, f in cases]
    dec = _check(built, ctx, oracle, frames, drafts)
    try:
        import io
        from PIL import Image
        got = _images(dec, _decode(dec))
        agree = []
        for f, g, d in zip(frames, got, drafts):
            im = Image.open(io.BytesIO(f))
            im.draft("L", (d[1], d[0]))
            agree.append(bool(np.array_equal(np.asarray(im), g[..., 0])))
        print("Pillow agrees on the bound blocks:", agree)
    except ImportError:
        pass


def test_mixed_scales_one_tensor(built, ctx, oracle):
    """one batch mixing k = 1, 2, 4 and 8 (and undrafted frames) resized into a single [N, 3, h, w] tensor"""
    import torch
    from libjpeg_b200 import decoder, synth
    src = [_synth(1000, 333, 31, (2, 2)), _synth(640, 480, 32, (1, 1)), _synth(333, 517, 33, (2, 1)), _synth(97, 61, 34, (1, 2)),
           synth.encode(synth.source_image(120, 90, 35)[..., 0], 80, (1, 1), 0).tobytes()]
    frames, drafts = [], []
    for j, f in enumerate(src):
        for k in (1, 2, 4, 8, None):
            frames.append(f), drafts.append(None if k is None else _request(f, k))
    ks = [1 if d is None else decoder.draft_scale(f, d) for f, d in zip(frames, drafts)]
    assert set(ks) == {1, 2, 4, 8}
    th, tw = 56, 72
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", resize=(th, tw), draft=drafts)
    dst = torch.zeros((len(frames), 3, th, tw), dtype=torch.uint8, device="cuda")
    dec.decode_into(dst)
    torch.cuda.synchronize()
    for i, f in enumerate(frames):
        img = _model(oracle, f, drafts[i] or decoder.output_size(f), "RGB")
        want = rm.resize(np.ascontiguousarray(img), tw, th, rm.NAMES["bilinear"])
        assert np.array_equal(dst[i].permute(1, 2, 0).cpu().numpy(), want), (i, ks[i])


def test_k1_frames_equal_undrafted(built, ctx):
    """a frame whose draft scale is 1 (a request of its own size or larger) is written byte for byte as the undrafted turbo batch"""
    from libjpeg_b200 import synth
    frames = [_synth(517, 333, 41, (2, 2)), _synth(97, 61, 42, (2, 1)), _synth(64, 48, 43, (1, 1)),
              synth.encode(synth.source_image(40, 24, 44)[..., 0], 80, (1, 1), 0).tobytes()]
    plain = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB")
    from libjpeg_b200 import decoder
    drafts = [decoder.output_size(f) for f in frames]
    drafts[1] = (10 ** 6, 10 ** 6)
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", draft=drafts)
    assert dec.out_bytes == plain.out_bytes
    a, b = _decode(plain).cpu().numpy(), _decode(dec).cpu().numpy()
    assert dec.launches == plain.launches
    assert np.array_equal(a, b)


def _fill(nbytes):
    import torch
    return torch.full((nbytes,), SENT, dtype=torch.uint8, device="cuda")


def _view_as_int(t):
    import torch
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def test_destinations(built, ctx, oracle):
    """decode_into [N, 3, H', W'] uint8 and fp16 with the ImageNet map, contiguous, padded and NHWC, sentinels around: drafted frames
    of one reduced size (1920 x 1080 at 1/2 and 3840 x 2160 at 1/4), oriented and not"""
    import torch
    frames = [_synth(1920, 1080, 51, (2, 2)), _synth(3840, 2160, 52, (2, 2)), _synth(1920, 1080, 53, (2, 1)), _synth(1920, 1080, 54, (1, 1))]
    drafts = [(540, 960), (540, 960), (540, 960), (540, 960)]
    n, th, tw = len(frames), 540, 960
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", draft=drafts)
    want_u8 = torch.from_numpy(np.stack([_model(oracle, f, d, "RGB") for f, d in zip(frames, drafts)])).permute(0, 3, 1, 2).contiguous().cuda()
    scale, bias = [1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225)], [-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225]
    for dtype in (torch.uint8, torch.float16):
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
            sent = int(np.frombuffer(bytes([SENT] * esz), dtype={1: np.uint8, 2: np.int16}[esz])[0])
            assert bool((_view_as_int(full_t)[mask] == sent).all()), (dtype, layout)


def test_orientations_crops_resize(built, ctx, oracle):
    """all eight orientations, seam / edge / random crops in the drafted, oriented image and all five filters, packed"""
    from libjpeg_b200 import decoder, synth
    src = [_synth(2000, 666, 21, (2, 2)), _synth(666, 1034, 22, (2, 1)), _synth(194, 122, 23, (1, 2)), _synth(260, 140, 24, (1, 1)),
           synth.encode(synth.source_image(150, 122, 25)[..., 0], 85, (1, 1), 0).tobytes()]
    rng = np.random.default_rng(6)
    batch, drafts, rects, sizes, want = [], [], [], [], []
    for j, f in enumerate(src):
        for o in om.ORIENTATIONS:
            data = om.tag(f, o)
            req = _request(data, (2, 4, 8)[(j + o) % 3])
            k = decoder.draft_scale(data, req)
            img = om.orient(_model(oracle, data, req), o)
            oh, ow = img.shape[:2]
            assert (oh, ow) == decoder.output_size(data, downscale=k, exif_orientation=True)
            for i, rect in enumerate([None] + cm.rectangles(ow, oh, rng, n_random=1)[-3:]):
                filt = sorted(rm.NAMES)[(j + o + i) % 5]
                size = None if i % 2 == 0 else (int(rng.integers(1, 80)), int(rng.integers(1, 80)))
                c = img if rect is None else img[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2]]
                batch.append(data), drafts.append(req), rects.append(rect), sizes.append(size)
                want.append((c if size is None else rm.resize(np.ascontiguousarray(c), size[1], size[0], rm.NAMES[filt]), filt))
    for filt in sorted(rm.NAMES):
        idx = [i for i, (_, fl) in enumerate(want) if fl == filt]
        dec = _batch(built, ctx, [batch[i] for i in idx], reconstruction=TURBO, exif_orientation=True, crop=[rects[i] for i in idx],
                     resize=[sizes[i] for i in idx], resample=filt, draft=[drafts[i] for i in idx])
        got = _images(dec, _decode(dec))
        for j, i in enumerate(idx):
            assert dec.status(j) == 0
            assert np.array_equal(got[j], want[i][0]), (filt, i)


def test_modes_and_no_color_transform(built, ctx, oracle):
    """mode "RGB" (grey replicated), mode "L" (YCbCr: component 0 at its reduced size; RGB-coded: the L formula), no mode and
    color_transform=False, at every scale"""
    from tests.test_mode import adobe_rgb
    frames = [open(os.path.join(GOLDEN, n), "rb").read() for n in _files("")]
    frames += [adobe_rgb(_synth(97, 61, 3, (1, 1))), adobe_rgb(_synth(64, 40, 4, (2, 2))), _synth(35, 258, 5, (1, 2)),
               open(os.path.join(GOLDEN, "subsampling", "c410_97x53_z3_q75.jpg"), "rb").read()]
    for k in (2, 4, 8):
        drafts = [_request(f, k) for f in frames]
        for mode in ("RGB", "L", None):
            _check(built, ctx, oracle, frames, drafts, mode=mode)
        _check(built, ctx, oracle, frames, drafts, color_transform=False)


def test_mixed_tolerant_batch(built, ctx, oracle):
    """grey, colour, RGB-coded, JPEG XT, damaged, 12-bit and CMYK frames drafted in one tolerant batch: statuses as without the draft
    (NOT_IMPLEMENTED for the 12-bit and four-component frames); the intact ones equal the model, the cut-off one the model on the
    coefficients this library decoded"""
    from tests.test_mode import adobe_rgb
    frames = [open(os.path.join(GOLDEN, "g_40x24_z2_q75.jpg"), "rb").read(), _synth(130, 70, 61, (2, 2)),
              adobe_rgb(_synth(64, 48, 62, (1, 1))), open(os.path.join(GOLDEN, "xt", "xt_420_96x80_z6_q75_Q90.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "damaged", "trunc_c422_100x60.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "deep12", "d12_420_50x38_q60.jpg"), "rb").read(),
              open(os.path.join(GOLDEN, "cmyk", "cmyk_64x48_s0_q90.jpg"), "rb").read()]
    drafts = [(h // 2, w // 2) for h, w in [(24, 40), (70, 130), (48, 64), (80, 96), (60, 100), (38, 50), (48, 64)]]
    plain = _batch(built, ctx, frames, reconstruction=TURBO)
    _decode(plain)  # its statuses are those of a decode
    dec = _batch(built, ctx, frames, reconstruction=TURBO, draft=drafts)
    got = _images(dec, _decode(dec))
    for i, f in enumerate(frames):
        if i >= 5:
            assert dec.status(i) == NOT_IMPLEMENTED and got[i] is None, i
            continue
        assert dec.status(i) == plain.status(i), i
        if i != 4:
            assert np.array_equal(got[i], _model(oracle, f, drafts[i])), i
        else:
            fi = dec.info(i)
            coef = [dec.coefficients(i, c).astype(np.int64) for c in range(fi.ncomp)]
            want = dm.reconstruct(coef, fi.width, fi.height, list(fi.hs), list(fi.vs), 2, "YCbCr")
            assert np.array_equal(got[i], want), i


def test_decode_twice(built, ctx):
    frames = [_synth(517, 333, 71, (2, 2)), _synth(97, 61, 72, (2, 1))]
    dec = _batch(built, ctx, frames, reconstruction=TURBO, draft=[(80, 120), (30, 40)])
    a, b = _decode(dec).cpu().numpy(), _decode(dec).cpu().numpy()
    assert np.array_equal(a, b)


def test_refused(built, ctx):
    """a draft without reconstruction="libjpeg-turbo", or with downscale / upsample=False, fails with NOT_IMPLEMENTED; a draft with
    exactly one zero side through the C entry point with INVALID_PARAMETER. None of them opens a batch."""
    import ctypes
    from libjpeg_b200 import native
    frames = [_synth(64, 48, 81, (2, 2))]
    opened = ctx._batches
    for kw in ({"reconstruction": "reference"}, {"reconstruction": TURBO, "downscale": 2}, {"reconstruction": TURBO, "upsample": False}):
        with pytest.raises(native.NativeError) as e:
            built.BatchDecoder(frames, ctx=ctx, draft=(24, 32), **kw)
        assert e.value.code == NOT_IMPLEMENTED, kw
    buf = (ctypes.c_uint8 * len(frames[0])).from_buffer_copy(frames[0])
    ptrs = (ctypes.c_void_p * 1)(ctypes.addressof(buf))
    lens = (ctypes.c_size_t * 1)(len(frames[0]))
    for w, h in ((0, 5), (5, 0)):
        table = (native.SizeStruct * 1)()
        table[0].width, table[0].height = w, h
        handle = ctypes.c_void_p()
        rc = native.lib.b200jpg_batch_create_draft(ctx.handle, ptrs, lens, 1, 0, native.RECONSTRUCTION_FLAGS[TURBO], table, None, None, 0,
                                                   ctypes.byref(handle))
        assert rc == INVALID_PARAMETER and not handle.value
    assert ctx._batches == opened
