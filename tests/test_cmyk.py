"""GPU: CMYK and YCCK frames under BatchDecoder(mode="RGB" | "L") (DESIGN §15). The oracle is the library's own decode of the same
batch configuration without the mode (pinned to the reference for four-component frames by test_four_component_frames_match_oracle)
with the numpy model of tests/cmyk_model.py applied to it (pinned to Pillow by tests/test_cmyk_cpu.py); every other frame is what
tests/test_mode.py expects of it."""
import os

import numpy as np
import pytest

from tests import cmyk_model as km
from tests import crop_model as cm
from tests import orientation_model as om
from tests import resize_model as rm
from tests import test_mode as tm
from tests.test_decode_into import GOLDEN
from tests.test_orientation import _batch, _decode, _images, _synth

pytestmark = pytest.mark.gpu

NOT_IMPLEMENTED = -1034
CMYK_DIR = os.path.join(GOLDEN, "cmyk")
FIXTURES = sorted(f[:-4] for f in os.listdir(CMYK_DIR) if f.endswith(".jpg"))


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _fixture(name):
    with open(os.path.join(CMYK_DIR, name + ".jpg"), "rb") as f:
        return f.read()


def _synthetic():
    """four-component frames with an Adobe segment of transform 0 and 2, every luma sampling, with and without restart markers"""
    out = []
    for k, sub in enumerate([(1, 1), (2, 2), (2, 1), (1, 2)]):
        for rst in (0, 3):
            four = km.four_component(97 + 8 * k, 61 + 5 * k, 20 + k, sub, rst)
            out += [km.after_soi(four, km.adobe(0)), km.before_sos(four, km.adobe(2))]
    return out


def _hand_built():
    """the generic path's four-component cases (every component its own content, dense blocks), as CMYK and as YCCK"""
    from tests import recon_cases
    four = [recon_cases.case(n)[1] for n in recon_cases.NAMES if n.startswith("generic_four")]
    assert four
    return [km.after_soi(f, km.adobe(t)) for f in four for t in (0, 2)]


def _truncated():
    """CMYK and YCCK files cut short: damaged frames, decoded as far as the data goes (or refused) exactly as without the mode"""
    out = []
    for name in FIXTURES:
        d = _fixture(name)
        out += [d[:len(d) * 2 // 3], d[:len(d) - 40]]
    return out


SETS = {"fixtures": lambda: [_fixture(n) for n in FIXTURES], "synthetic": _synthetic, "hand_built": _hand_built,
        "truncated": _truncated}


def _space(data):
    from libjpeg_b200 import decoder
    try:
        return decoder.colorspace(data)
    except Exception:
        return None


def _expected(built, ctx, frames, mode, **kw):
    """per frame the image the batch with `mode` writes and its status: CMYK / YCCK frames the model on the decode of the same
    configuration without the mode, every other frame as tests/test_mode.py has it"""
    want, status = tm._expected(built, ctx, frames, mode, **kw)
    plain = _batch(built, ctx, frames, **kw)
    ref = _images(plain, _decode(plain))
    for i, f in enumerate(frames):
        space = _space(f)
        if space in (km.CMYK, km.YCCK):
            status[i] = plain.status(i)
            want[i] = None if ref[i] is None else km.convert(ref[i], space, mode)
    return want, status


def _check(built, ctx, frames, mode, **kw):
    want, status = _expected(built, ctx, frames, mode, **kw)
    dec = _batch(built, ctx, frames, mode=mode, **kw)
    out = _decode(dec)
    got = _images(dec, out)
    converted = 0
    for i, w in enumerate(want):
        assert dec.status(i) == status[i], "frame %d" % i
        if w is None:
            assert got[i] is None or status[i] != 0
            continue
        assert dec.output_components(i) == w.shape[2]
        assert np.array_equal(got[i], w), "frame %d" % i
        converted += _space(frames[i]) in (km.CMYK, km.YCCK)
    assert converted > 0
    mask = np.ones(out.numel(), dtype=bool)
    for i in range(len(frames)):
        mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (out.cpu().numpy()[mask] == 0x5A).all(), "bytes outside the slots were written"
    return dec


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("name", list(SETS))
def test_sets(built, ctx, name, mode):
    _check(built, ctx, SETS[name](), mode)


def _mixed():
    return [_fixture(FIXTURES[0]), _fixture(FIXTURES[-1]), _synthetic()[3], _hand_built()[1], _synth(200, 120, 3),
            tm._grey(90, 70, 4)]


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_downscale_and_orientations(built, ctx, k, mode):
    frames = [om.tag(f, o) for f in _mixed() for o in om.ORIENTATIONS]
    _check(built, ctx, frames, mode, downscale=k, exif_orientation=True)


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_crops(built, ctx, mode):
    from libjpeg_b200 import decoder
    frames, rects = [], []
    rng = np.random.default_rng(15)
    for f in _mixed():
        for o in (1, 6):
            tagged = om.tag(f, o)
            h, w = decoder.output_size(tagged, exif_orientation=True)
            for r in cm.rectangles(w, h, rng, n_random=2)[-3:]:
                frames.append(tagged), rects.append(r)
    _check(built, ctx, frames, mode, crop=rects, exif_orientation=True)


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("resample", ["box", "bilinear", "hamming", "bicubic", "lanczos"])
def test_resize(built, ctx, mode, resample):
    """the mode before the resize: the resize model applied to the mode's image of the crop"""
    frames = _mixed() + SETS["fixtures"]()
    rng = np.random.default_rng(len(resample) + len(mode))
    want, _ = _expected(built, ctx, frames, mode)
    rects = [cm.rectangles(w.shape[1], w.shape[0], rng, n_random=1)[-1] for w in want]
    sizes = [(int(rng.integers(1, 300)), int(rng.integers(1, 300))) for _ in frames]
    dec = _batch(built, ctx, frames, mode=mode, crop=rects, resize=sizes, resample=resample)
    got = _images(dec, _decode(dec))
    for i, (w, r, s) in enumerate(zip(want, rects, sizes)):
        c = w[r[1]:r[1] + r[3], r[0]:r[0] + r[2]]
        assert np.array_equal(got[i], rm.resize(c, s[1], s[0], rm.NAMES[resample])), "frame %d" % i


def test_refused_frames(built, ctx):
    """unmarked and 12-bit four-component frames keep NOT_IMPLEMENTED under a mode, next to converted ones"""
    unmarked, deep = km.four_component(64, 48, 9), km.after_soi(km.deep12_four(), km.adobe(0))
    frames = [unmarked, deep, km.after_soi(unmarked, km.adobe(0)), km.after_soi(unmarked, km.adobe(2))]
    plain = _batch(built, ctx, frames)
    _decode(plain)
    assert [plain.status(i) for i in range(4)] == [0] * 4 and plain.output_components(2) == 4
    for mode in ("RGB", "L"):
        dec = _batch(built, ctx, frames, mode=mode)
        _decode(dec)  # (the statuses of live frames are read after a decode)
        assert [dec.status(i) for i in range(4)] == [NOT_IMPLEMENTED, NOT_IMPLEMENTED, 0, 0]
        assert [dec.output_components(i) for i in (2, 3)] == [3 if mode == "RGB" else 1] * 2
        assert tm._refused(built, frames, ctx=ctx, mode=mode) == NOT_IMPLEMENTED
        assert tm._refused(built, frames[2:], ctx=ctx, mode=mode) is None


def test_sanity_against_pillow(built, ctx):
    """the fixtures' output lies within a few levels of Pillow's own convert (libjpeg's IDCT and upsampling differ from the
    reference's by that much: at most 4 levels, 0.27 on average, in these files); an inverted polarity misses by about 255"""
    expected = np.load(os.path.join(CMYK_DIR, "expected.npz"))
    frames = SETS["fixtures"]()
    for mode in ("RGB", "L"):
        dec = _batch(built, ctx, frames, mode=mode)
        got = _images(dec, _decode(dec))
        for name, g in zip(FIXTURES, got):
            w = expected[name + "_" + mode]
            d = np.abs(g.astype(int) - (w if w.ndim == 3 else w[..., None]).astype(int))
            assert d.max() <= 4 and d.mean() < 0.3, (name, mode, d.max(), d.mean())


def test_decode_into_mixed_batch(built, ctx):
    """one [N, 3, 224, 224] tensor from a tolerant batch of grey, YCbCr, Adobe-RGB, CMYK and YCCK frames with unmarked and 12-bit
    four-component frames (skipped) and an unparseable one: uint8 equal to the model, fp16 / bf16 / fp32 with the ImageNet map
    equal to the uint8 result converted by torch; NHWC and padded destinations with sentinels; statuses those of the batch without
    the mode, but for the refused frames"""
    import torch
    from libjpeg_b200 import decoder
    unmarked, deep = km.four_component(64, 48, 9), km.after_soi(km.deep12_four(), km.adobe(0))
    frames = ([tm._grey(120, 90, 1), _synth(300, 200, 2), _synth(150, 100, 3, (1, 1)), tm.adobe_rgb(_synth(200, 120, 4, (1, 1)))] +
              SETS["fixtures"]() + _synthetic()[:4] + [unmarked, deep, b"\xff\xd8\xff\xd9"])
    n = len(frames)
    refused = {n - 3, n - 2}
    rng = np.random.default_rng(21)
    rects = []
    for f in frames:
        try:
            h, w = decoder.output_size(f)
            rects.append(cm.rectangles(w, h, rng, n_random=1)[-1])
        except Exception:
            rects.append(None)
    want, status = _expected(built, ctx, frames, "RGB", crop=rects)
    plain = _batch(built, ctx, frames, crop=rects, resize=(224, 224))
    dec = _batch(built, ctx, frames, mode="RGB", crop=rects, resize=(224, 224))
    live = [i for i in range(n) if dec.geometry()[i] is not None]
    assert set(range(n)) - set(live) == refused | {n - 1}
    u8 = torch.full((n, 3, 224, 224), 0x5A, dtype=torch.uint8, device="cuda")
    dec.decode_into([list(u8[i]) if i in live else None for i in range(n)])
    _decode(plain)
    for i in range(n):
        assert dec.status(i) == (NOT_IMPLEMENTED if i in refused else plain.status(i)), i
    for i in live:
        model = rm.resize(want[i], 224, 224, rm.BILINEAR)
        assert np.array_equal(u8[i].permute(1, 2, 0).cpu().numpy(), model), i
    scale = [1.0 / (255.0 * s) for s in tm.STD]
    bias = [-m / s for m, s in zip(tm.MEAN, tm.STD)]
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
        assert torch.equal(nhwc[i], u8[i].permute(1, 2, 0)), i
        assert torch.equal(padded[i, :, 3:227, 5:229], u8[i]), i
    inner = torch.zeros_like(padded, dtype=torch.bool)
    inner[:, :, 3:227, 5:229] = True
    assert bool((padded[~inner] == 0x5A).all())
    for i in set(range(n)) - set(live):
        assert bool((nhwc[i] == 0x5A).all()) and bool((padded[i] == 0x5A).all())


def test_luma_tensor(built, ctx):
    """mode="L" fills one [N, 1, H, W] tensor from CMYK, YCCK, grey and YCbCr frames of one size"""
    import torch
    four = km.four_component(320, 240, 5, (2, 2))
    frames = [km.after_soi(four, km.adobe(0)), km.after_soi(four, km.adobe(2)), tm._grey(320, 240, 6), _synth(320, 240, 7)]
    want, _ = _expected(built, ctx, frames, "L")
    dec = _batch(built, ctx, frames, mode="L")
    t = torch.zeros((4, 1, 240, 320), dtype=torch.uint8, device="cuda")
    dec.decode_into(t)
    torch.cuda.synchronize()
    for i in range(4):
        assert np.array_equal(t[i].permute(1, 2, 0).cpu().numpy(), want[i]), i
