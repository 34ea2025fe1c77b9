"""GPU: CMYK and YCCK frames under BatchDecoder(reconstruction="libjpeg-turbo", mode="RGB" | "L"), full size and drafted (DESIGN
§18). The oracle is tests/turbo_cmyk_model.py on the oracle's coefficients (pinned to Pillow by tests/test_turbo_cmyk_cpu.py),
and for the fixtures Pillow's own output: expected.npz at full size, turbo_digests.json drafted. Every stage after the reconstruction
through its existing model (orientation, crop, resize, float map)."""
import hashlib
import itertools
import json
import os

import numpy as np
import pytest

from tests import cmyk_model as km
from tests import crop_model as cm
from tests import draft_model as dm
from tests import orientation_model as om
from tests import recon_cases as rc
from tests import resize_model as rm
from tests import test_mode as tmode
from tests import turbo_cmyk_model as tcm
from tests import turbo_model as tm
from tests.test_decode_into import GOLDEN
from tests.test_orientation import _batch, _decode, _images, _synth

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED = -1034
TURBO = "libjpeg-turbo"
CMYK_DIR = os.path.join(GOLDEN, "cmyk")
FIXTURES = sorted(f[:-4] for f in os.listdir(CMYK_DIR) if f.endswith(".jpg"))
DIGESTS = json.load(open(os.path.join(CMYK_DIR, "turbo_digests.json")))
SAMPLINGS = [(1, 1), (2, 2), (2, 1), (1, 2)]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


@pytest.fixture(scope="module")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()


def _fixture(name):
    with open(os.path.join(CMYK_DIR, name + ".jpg"), "rb") as f:
        return f.read()


def _request(data, k):
    """the draft (h, w) that asks for 1/k; None for k = 1 (undrafted)"""
    from libjpeg_b200 import decoder
    if k == 1:
        return None
    fi = decoder.parse(data)
    return max(1, fi.height // k), max(1, fi.width // k)


def _scale(data, req):
    from libjpeg_b200 import decoder
    return 1 if req is None else decoder.draft_scale(data, req)


def _model(oracle, data, req, mode):
    """what the batch writes for one intact frame: tests/turbo_cmyk_model.py for CMYK / YCCK, tests/draft_model.py for the others"""
    from libjpeg_b200 import decoder
    space, k = decoder.colorspace(data), _scale(data, req)
    if space not in (km.CMYK, km.YCCK):
        return dm.decode(oracle, data, space, k, mode)
    r, info, planes = oracle.coefficients(data)
    assert r == 0, r
    return tcm.reconstruct(tm.dequantised(info, planes), info.width, info.height, list(info.hs), list(info.vs), k, space, mode)


def _check(built, ctx, oracle, frames, drafts, mode, names=None):
    """packed decode with sentinels: every frame equals the model, and the fixtures Pillow's stored output"""
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode=mode, draft=drafts)
    out = _decode(dec)
    got = _images(dec, out)
    expected = np.load(os.path.join(CMYK_DIR, "expected.npz"))
    for i, f in enumerate(frames):
        assert dec.status(i) == 0, i
        assert np.array_equal(got[i], _model(oracle, f, drafts[i], mode)), (names[i] if names else i, drafts[i], mode)
        if names:
            k = _scale(f, drafts[i])
            g = got[i][..., 0] if mode == "L" else got[i]
            if k == 1:
                assert np.array_equal(g, expected[names[i] + "_" + mode]), names[i]
            d = DIGESTS["%s|%s|%d" % (names[i], mode, k)]
            assert d["scale"] == k and list(g.shape) == d["shape"]
            assert hashlib.sha256(np.ascontiguousarray(g).tobytes()).hexdigest() == d["sha256"], (names[i], mode, k)
    mask = np.ones(out.numel(), dtype=bool)
    for i in range(len(frames)):
        mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_fixtures(built, ctx, oracle, mode):
    """Pillow's CMYK files and their YCCK twins: at full size equal to expected.npz (Pillow's convert) exactly, drafted to the
    stored digests, in one batch mixing k = 1, 2, 4 and 8"""
    frames, drafts, names = [], [], []
    for name in FIXTURES:
        for k in (1, 2, 4, 8):
            frames.append(_fixture(name)), drafts.append(_request(_fixture(name), k)), names.append(name)
    _check(built, ctx, oracle, frames, drafts, mode, names)


def _synthetic():
    """four-component frames with an Adobe segment of transform 0 and 2, every luma sampling, with and without restart markers"""
    out = []
    for j, sub in enumerate(SAMPLINGS):
        for rst in (0, 3):
            four = km.four_component(97 + 8 * j, 61 + 5 * j, 20 + j, sub, rst)
            out += [km.after_soi(four, km.adobe(0)), km.before_sos(four, km.adobe(2))]
    return out


def _hand_built():
    """the generic path's four-component cases (every component its own content, dense blocks), as CMYK and as YCCK"""
    four = [rc.case(n)[1] for n in rc.NAMES if n.startswith("generic_four")]
    assert len(four) == 2
    return [km.after_soi(f, km.adobe(t)) for f in four for t in (0, 2)]


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("k", [1, 2, 4, 8])
@pytest.mark.parametrize("name", ["synthetic", "hand_built"])
def test_sets(built, ctx, oracle, name, k, mode):
    frames = {"synthetic": _synthetic, "hand_built": _hand_built}[name]()
    _check(built, ctx, oracle, frames, [_request(f, k) for f in frames], mode)


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


def _bound_frame(past, transform):
    """a 4:4:4 four-component frame with a bound block in each component: C (0) pass-1 results of magnitude 35076 / 35080 in the
    pattern of islow's largest pass-2 sum (DESIGN §16), M (1) and Y (2) column 1 at jpeg_idct_4x4's / jpeg_idct_2x2's pass-1 bound
    or one past it (§17), K (3) the islow pattern at the int16 limit"""
    from tests import streamwriter as sw
    w, h, factors = 64, 16, [(1, 1)] * 4
    _, comps = rc.base(w, h, 95 + past, factors)
    islow = _worst(tm.idct1d, tm.PASS2_SHIFT, range(8))
    for c in comps:
        c[0, 1:3] = 0
    comps[0][0, 1, 0, :] = islow * ((35080 if past else 35076) // 4)
    comps[1][0, 1, :, 1] = _worst(dm.red4_line, 12, (0, 1, 2, 3, 5, 6, 7)) * (27563 + past)
    comps[2][0, 1, :, 1] = _worst(dm.red2_line, 13, (0, 1, 3, 5, 7)) * (25040 + past)
    comps[3][0, 2, 0, :] = islow * 32767
    return km.after_soi(sw.encode(rc.frame(w, h, comps, factors)), km.adobe(transform))


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_int32_bounds(built, ctx, oracle, mode):
    """blocks on both sides of the islow and reduced-IDCT int32 bounds in a four-component frame, at k = 1, 2, 4 and 8"""
    frames = [_bound_frame(p, t) for p in (0, 1) for t in (0, 2)]
    for k in (1, 2, 4, 8):
        _check(built, ctx, oracle, frames, [_request(f, k) for f in frames], mode)


def _fill(shape, dtype, value):
    import torch
    return torch.full(shape, value, dtype=dtype, device="cuda")


def test_destinations(built, ctx, oracle):
    """decode_into [N, 3, H, W] uint8 / fp16 / bf16 / fp32 (the ImageNet map for the float types), contiguous, NHWC and padded,
    sentinels around: CMYK and YCCK frames of one output size, full size and drafted"""
    import torch
    four = [km.four_component(320, 240, 31, (2, 2), 4), km.four_component(640, 480, 32, (1, 1)), km.four_component(1280, 960, 33, (2, 1))]
    frames = [km.after_soi(four[0], km.adobe(0)), km.after_soi(four[1], km.adobe(2)), km.after_soi(four[2], km.adobe(0)),
              km.after_soi(four[0], km.adobe(2))]
    drafts = [None, (240, 320), (240, 320), None]
    n, th, tw = len(frames), 240, 320
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", draft=drafts)
    want = torch.from_numpy(np.stack([_model(oracle, f, d, "RGB") for f, d in zip(frames, drafts)])).permute(0, 3, 1, 2).contiguous().cuda()
    scale, bias = [1.0 / (255.0 * s) for s in tmode.STD], [-m / s for m, s in zip(tmode.MEAN, tmode.STD)]
    for dtype in (torch.uint8, torch.float16, torch.bfloat16, torch.float32):
        sent = 0x5A if dtype == torch.uint8 else 7.0
        if dtype == torch.uint8:
            want_t = want
        else:
            want_t = (want.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) + torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
        kw = {} if dtype == torch.uint8 else dict(scale=scale, bias=bias)
        for layout in ("nchw", "nhwc", "padded"):
            if layout == "nchw":
                full = _fill((n, 3, th, tw), dtype, sent)
                region = (slice(None),) * 4
                dst = full
            elif layout == "padded":
                full = _fill((n, 3, th + 2, tw + 3), dtype, sent)
                region = (slice(None), slice(None), slice(1, th + 1), slice(1, tw + 1))
                dst = full[region]
            else:
                full = _fill((n, th + 1, tw + 2, 4), dtype, sent)
                region = (slice(None), slice(0, th), slice(1, tw + 1), slice(0, 3))
                dst = full[region].permute(0, 3, 1, 2)
            dec.decode_into(dst, **kw)
            torch.cuda.synchronize()
            assert torch.equal(dst, want_t), (dtype, layout)
            mask = torch.ones(full.shape, dtype=torch.bool, device="cuda")
            mask[region] = False
            assert bool((full[mask] == sent).all()), (dtype, layout)


def test_orientations_crops_resize(built, ctx, oracle):
    """all eight orientations, seam / edge / random crops in the drafted, oriented image and all five filters, packed, both modes"""
    from libjpeg_b200 import decoder
    src = [km.after_soi(km.four_component(300, 180, 41, (2, 2), 3), km.adobe(0)), km.before_sos(km.four_component(180, 260, 42, (1, 1)), km.adobe(2)),
           km.after_soi(km.four_component(150, 122, 43, (2, 1)), km.adobe(2)), _fixture(FIXTURES[0]), _fixture(FIXTURES[-1])]
    rng = np.random.default_rng(18)
    batch, drafts, rects, sizes, modes, want = [], [], [], [], [], []
    for j, f in enumerate(src):
        for o in om.ORIENTATIONS:
            data = om.tag(f, o)
            mode = ("RGB", "L")[(j + o) % 2]
            req = _request(data, (1, 2, 4, 8)[(j + o) % 4])
            img = om.orient(_model(oracle, data, req, mode), o)
            oh, ow = img.shape[:2]
            assert (oh, ow) == decoder.output_size(data, downscale=_scale(data, req), exif_orientation=True)
            for i, rect in enumerate([None] + cm.rectangles(ow, oh, rng, n_random=1)[-3:]):
                filt = sorted(rm.NAMES)[(j + o + i) % 5]
                size = None if i % 2 == 0 else (int(rng.integers(1, 80)), int(rng.integers(1, 80)))
                c = img if rect is None else img[rect[1]:rect[1] + rect[3], rect[0]:rect[0] + rect[2]]
                batch.append(data), drafts.append(req), rects.append(rect), sizes.append(size), modes.append(mode)
                want.append((c if size is None else rm.resize(np.ascontiguousarray(c), size[1], size[0], rm.NAMES[filt]), filt))
    for filt in sorted(rm.NAMES):
        for mode in ("RGB", "L"):
            idx = [i for i, (_, fl) in enumerate(want) if fl == filt and modes[i] == mode]
            dec = _batch(built, ctx, [batch[i] for i in idx], reconstruction=TURBO, mode=mode, exif_orientation=True,
                         crop=[rects[i] for i in idx], resize=[sizes[i] for i in idx], resample=filt, draft=[drafts[i] for i in idx])
            got = _images(dec, _decode(dec))
            for j, i in enumerate(idx):
                assert dec.status(j) == 0
                assert np.array_equal(got[j], want[i][0]), (filt, mode, i)


def test_luma_tensor(built, ctx, oracle):
    """mode="L" fills one [N, 1, H, W] tensor from CMYK, YCCK, grey and YCbCr frames of one output size, drafted and not"""
    import torch
    four = km.four_component(320, 240, 5, (2, 2))
    big = km.four_component(640, 480, 6, (1, 2), 2)
    frames = [km.after_soi(four, km.adobe(0)), km.after_soi(four, km.adobe(2)), km.after_soi(big, km.adobe(0)),
              km.after_soi(big, km.adobe(2)), tmode._grey(320, 240, 6), _synth(640, 480, 7)]
    drafts = [None, None, (240, 320), (240, 320), None, (240, 320)]
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="L", draft=drafts)
    t = torch.zeros((len(frames), 1, 240, 320), dtype=torch.uint8, device="cuda")
    dec.decode_into(t)
    torch.cuda.synchronize()
    for i, (f, d) in enumerate(zip(frames, drafts)):
        assert np.array_equal(t[i].permute(1, 2, 0).cpu().numpy(), _model(oracle, f, d, "L")), i


def test_mixed_tolerant_batch(built, ctx, oracle):
    """one tolerant batch of grey, YCbCr, Adobe-RGB, CMYK, YCCK, unmarked and 12-bit four-component, cut-off CMYK and unparseable
    frames, drafts mixing k = 1, 2, 4 and 8, into one [N, 3, 224, 224] fp16 tensor with the ImageNet map: statuses those of the
    reference path under the same mode without drafts, NOT_IMPLEMENTED exactly where colorspace() is None; the intact frames equal
    the model resized, the cut-off one the model on the coefficients this batch decoded"""
    import torch
    from libjpeg_b200 import decoder
    unmarked, deep = km.four_component(64, 48, 9), km.after_soi(km.deep12_four(), km.adobe(0))
    cut = _fixture("cmyk_97x61_s2_q75")  # (no restart markers: a cut into its scan still parses, and decodes as far as it goes)
    cut = cut[:len(cut) * 2 // 3]
    assert decoder.colorspace(cut) == km.CMYK
    frames = ([tmode._grey(120, 90, 1), _synth(300, 200, 2), tmode.adobe_rgb(_synth(200, 120, 4, (1, 1)))] +
              [_fixture(n) for n in FIXTURES] + _synthetic()[:4] + [unmarked, deep, cut, b"\xff\xd8\xff\xd9"])
    n = len(frames)
    ks = [(1, 2, 4, 8)[i % 4] for i in range(n)]
    drafts = []
    for f, k in zip(frames, ks):
        try:
            drafts.append(_request(f, k))
        except Exception:
            drafts.append(None)

    def space(f):
        try:
            return decoder.colorspace(f)
        except Exception:
            return "unparseable"
    spaces = [space(f) for f in frames]
    assert spaces.count(None) == 2 and {km.CMYK, km.YCCK} <= set(spaces)
    ref = _batch(built, ctx, frames, mode="RGB", resize=(224, 224))
    _decode(ref)  # its statuses are those of a decode
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", resize=(224, 224), draft=drafts)
    live = [i for i in range(n) if dec.geometry()[i] is not None]
    scale, bias = [1.0 / (255.0 * s) for s in tmode.STD], [-m / s for m, s in zip(tmode.MEAN, tmode.STD)]
    t = torch.full((n, 3, 224, 224), 7.0, dtype=torch.float16, device="cuda")
    dec.decode_into([list(t[i]) if i in live else None for i in range(n)], scale=scale, bias=bias)
    torch.cuda.synchronize()
    cut_i = frames.index(cut)
    assert set(ks[i] for i in live if spaces[i] in (km.CMYK, km.YCCK)) == {1, 2, 4, 8}
    for i in range(n):
        assert dec.status(i) == ref.status(i), i
        assert (dec.status(i) == NOT_IMPLEMENTED) == (spaces[i] is None), i
        if i not in live:
            assert bool((t[i] == 7.0).all()), i
            continue
        if i == cut_i:
            fi = dec.info(i)
            coef = [dec.coefficients(i, c).astype(np.int64) for c in range(fi.ncomp)]
            img = tcm.reconstruct(coef, fi.width, fi.height, list(fi.hs), list(fi.vs), _scale(frames[i], drafts[i]), spaces[i], "RGB")
        else:
            img = _model(oracle, frames[i], drafts[i], "RGB")
        img = rm.resize(np.ascontiguousarray(img), 224, 224, rm.BILINEAR)
        u8 = torch.from_numpy(img).permute(2, 0, 1).cuda()
        want = (u8.float() * torch.tensor(scale, device="cuda").view(3, 1, 1) + torch.tensor(bias, device="cuda").view(3, 1, 1)).half()
        assert torch.equal(t[i], want), i
    assert cut_i in live


def test_decode_to_host_ex(built, ctx):
    """B200JPG_FLAG_LIBJPEG_TURBO | B200JPG_FLAG_OUTPUT_RGB through b200jpg_decode_to_host_ex: the packed bytes of the batch"""
    import ctypes
    from libjpeg_b200 import native
    frames = [_fixture(FIXTURES[1]), _fixture(FIXTURES[-2]), _synth(130, 70, 91, (2, 2)), _hand_built()[1]]
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB")
    want = _decode(dec).cpu().numpy()[:dec.out_bytes]
    n = len(frames)
    bufs = [(ctypes.c_uint8 * len(f)).from_buffer_copy(f) for f in frames]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    flags = native.RECONSTRUCTION_FLAGS[TURBO] | native.MODE_FLAGS["RGB"]
    got = np.zeros(dec.out_bytes, dtype=np.uint8)
    native.check(native.lib.b200jpg_decode_to_host_ex(ctx.handle, ptrs, lens, n, got.ctypes.data, got.size, flags), ctx.handle)
    for i in range(n):
        a, b = dec.out_offset(i), dec.out_offset(i) + dec.frame_bytes(i)
        assert np.array_equal(got[a:b], want[a:b]), i


def test_decode_twice(built, ctx):
    frames = _synthetic()[:4] + [_fixture(FIXTURES[2])]
    dec = _batch(built, ctx, frames, reconstruction=TURBO, mode="RGB", draft=[None, (30, 50), (15, 25), (8, 12), None])
    a, b = _decode(dec).cpu().numpy(), _decode(dec).cpu().numpy()
    assert np.array_equal(a, b)
