"""No device: the drafted reconstruction model (tests/draft_model.py, DESIGN §17) against Pillow's Image.draft byte for byte --
stored vectors (3x / 4x factors, progressive, JPEG XT base layers), synthetic streams of every size up to 34 x 34 in every
sampling at every scale, Pillow's progressive streams, 1080p and 4K, draft("L"), and the chain draft -> orientation -> crop ->
resize -- plus draft_scale against Pillow's choice, the int32 bounds of the reduced IDCTs, the argument checks and the stored
digests."""
import importlib.util
import io
import itertools
import json
import os

import numpy as np
import pytest

from tests import draft_model as dm
from tests import orientation_model as om
from tests import resize_model as rm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SAMPLINGS = {"420": (2, 2), "422": (2, 1), "440": (1, 2), "444": (1, 1), "grey": None}


@pytest.fixture(scope="module")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()


def _make_draft():
    spec = importlib.util.spec_from_file_location("make_draft", os.path.join(GOLDEN, "turbo", "make_draft.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _model(oracle, data, k, mode=None):
    from libjpeg_b200 import decoder
    out = dm.decode(oracle, data, decoder.colorspace(data), k, mode)
    return out[..., 0] if out.shape[2] == 1 else out


def _pillow(data, k, mode="RGB"):
    """Pillow's draft(mode, ...) asked for 1/k: (its scale, np.asarray(im.convert(mode)))"""
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    im.draft(mode, _make_draft().request(im.size, k))
    return im.decoderconfig[0], np.asarray(im.convert(mode))


def _synth(w, h, seed, sampling, restart=0):
    from libjpeg_b200 import synth
    img = synth.source_image(w, h, seed)
    return synth.encode(img[..., 0] if sampling is None else img, 80, sampling or (1, 1), restart).tobytes()


def _check(oracle, data, k, mode="RGB"):
    scale, want = _pillow(data, k, mode)
    got = _model(oracle, data, scale, mode)
    assert got.shape == want.shape and np.array_equal(got, want)
    return scale


def test_stored_vectors(oracle):
    """every stored vector Pillow reads (baseline, progressive, 3x / 4x subsampling, the reference's set, JPEG XT base layers) at
    k = 2, 4 and 8 under draft("RGB") and draft("L")"""
    pytest.importorskip("PIL.Image")
    mk = _make_draft()
    n = 0
    for rel in mk._make_turbo().vectors():
        for k in mk.SCALES:
            for mode in mk.MODES:
                r = mk.pillow_draft(rel, mode, k)
                if r is None:
                    continue
                scale, want = r
                data = open(os.path.join(GOLDEN, rel), "rb").read()
                assert np.array_equal(_model(oracle, data, scale, mode), want), (rel, mode, k)
                n += 1
    assert n == 246


def test_digests_match_pillow():
    """draft_digests.json is what Pillow gives here"""
    pytest.importorskip("PIL.Image")
    stored = json.load(open(os.path.join(GOLDEN, "turbo", "draft_digests.json")))
    assert stored == _make_draft().table()


@pytest.mark.parametrize("k", [2, 4, 8])
@pytest.mark.parametrize("name", list(SAMPLINGS))
def test_every_small_size(oracle, name, k):
    """every width 1..34 at two heights and every height 1..34 at two widths, with and without restart markers"""
    pytest.importorskip("PIL.Image")
    sizes = [(w, h) for w in range(1, 35) for h in (1, 17)] + [(w, h) for h in range(1, 35) for w in (2, 19)]
    for j, (w, h) in enumerate(sizes):
        data = _synth(w, h, j, SAMPLINGS[name], restart=1 if j % 3 == 0 else 0)
        scale, want = _pillow(data, k)
        got = _model(oracle, data, scale)
        got = np.repeat(got[..., None], 3, axis=2) if got.ndim == 2 else got
        assert np.array_equal(got, want), (name, w, h, k)


@pytest.mark.parametrize("name", ["420", "422", "444", "grey"])
def test_progressive(oracle, name):
    """Pillow's own progressive (and optimised-table) streams at every scale"""
    Image = pytest.importorskip("PIL.Image")
    from libjpeg_b200 import synth
    for j, (w, h) in enumerate([(9, 9), (33, 17), (97, 61), (130, 70)]):
        img = synth.source_image(w, h, 50 + j)
        im = Image.fromarray(img[..., 0]) if name == "grey" else Image.fromarray(img)
        buf = io.BytesIO()
        kw = {} if name == "grey" else {"subsampling": {"444": 0, "422": 1, "420": 2}[name]}
        im.save(buf, "JPEG", quality=85, progressive=True, optimize=True, **kw)
        for k in (2, 4, 8):
            _check(oracle, buf.getvalue(), k, "L" if name == "grey" else "RGB")


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)])
def test_large(oracle, w, h):
    pytest.importorskip("PIL.Image")
    data = _synth(w, h, 7, (2, 2), restart=8)
    assert [_check(oracle, data, k) for k in (2, 4, 8)] == [2, 4, 8]


def test_draft_luma(oracle):
    """draft("L") of YCbCr frames in every sampling and of 3x / 4x-subsampled vectors at every scale"""
    pytest.importorskip("PIL.Image")
    frames = [_synth(35, 19, 1, (2, 2)), _synth(64, 40, 2, (2, 1)), _synth(41, 66, 3, (1, 2)), _synth(50, 38, 4, (1, 1))]
    frames += [open(os.path.join(GOLDEN, "subsampling", f), "rb").read() for f in sorted(os.listdir(os.path.join(GOLDEN, "subsampling")))
               if f.endswith(".jpg")][:6]
    for data in frames:
        for k in (2, 4, 8):
            try:
                _check(oracle, data, k, "L")
            except OSError:  # more than 10 blocks per MCU: Pillow does not read it
                continue


def _chain_frames():
    from libjpeg_b200 import synth
    out = []
    for j, (w, h, s) in enumerate([(197, 161, (2, 2)), (164, 148, (1, 1)), (200, 170, (2, 1)), (161, 197, (1, 2)), (133, 117, (2, 2)),
                                   (140, 124, None), (230, 170, (2, 2)), (175, 161, (2, 1))]):
        img = synth.source_image(w, h, 80 + j)
        data = synth.encode(img[..., 0] if s is None else img, 85, s or (1, 1), 0).tobytes()
        out.append(om.tag(data, 1 + j % 8))
    return out


@pytest.mark.parametrize("resample", sorted(rm.NAMES))
def test_chain_equals_pillow(oracle, resample):
    """the model at Pillow's scale -> orientation -> crop -> tests/resize_model.py equals im.draft("RGB", (w, h)) followed by
    ImageOps.exif_transpose(im).convert("RGB").crop(box).resize(size, filter), all eight orientations, every scale"""
    pytest.importorskip("PIL.Image")
    from PIL import Image, ImageOps
    rng = np.random.default_rng(4)
    for j, data in enumerate(_chain_frames()):
        k = (2, 4, 8)[j % 3]
        im = Image.open(io.BytesIO(data))
        im.draft("RGB", (im.size[0] // k, im.size[1] // k))
        assert im.decoderconfig[0] == k
        o = im.getexif().get(0x0112, 1)
        oriented = om.orient(_model(oracle, data, k, "RGB"), o)
        oh, ow = oriented.shape[:2]
        x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
        cw, ch = int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))
        tw, th = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        got = rm.resize(np.ascontiguousarray(oriented[y:y + ch, x:x + cw]), tw, th, rm.NAMES[resample])
        pil = ImageOps.exif_transpose(im).convert("RGB").crop((x, y, x + cw, y + ch))
        want = np.asarray(pil.resize((tw, th), rm.NAMES[resample]))
        assert np.array_equal(got, want), (o, k, resample)


def test_draft_scale_equals_pillow(built):
    """decoder.draft_scale against Pillow's decoderconfig[0] over a grid of requests: larger than the frame, 1 pixel, non-square,
    exact multiples and one below them; oriented frames take the request in coded orientation"""
    Image = pytest.importorskip("PIL.Image")
    from libjpeg_b200 import decoder
    frames = [_synth(97, 61, 1, (2, 2)), _synth(640, 480, 2, (2, 1)), _synth(16, 16, 3, None), _synth(1, 1, 4, (1, 1))]
    frames += [om.tag(_synth(300, 77, 5, (2, 2)), o) for o in (6, 8, 3)]
    n = 0
    for data in frames:
        W, H = Image.open(io.BytesIO(data)).size
        reqs = {(1, 1), (W, H), (W + 1, H), (2 * W, 3 * H), (1, H), (W, 1)}
        for k in (2, 4, 8, 16):
            reqs |= {(max(1, W // k), max(1, H // k)), (max(1, W // k + 1), max(1, H // k)), (max(1, W // k), max(1, H // k - 1))}
        for w, h in sorted(reqs):
            im = Image.open(io.BytesIO(data))
            im.draft("RGB", (w, h))
            assert decoder.draft_scale(data, (h, w)) == im.decoderconfig[0] == dm.draft_scale(W, H, w, h), (W, H, w, h)
            n += 1
    assert n > 100


@pytest.mark.parametrize("line,n_in,p1,p2,norm", [(dm.red4_line, (0, 1, 2, 3, 5, 6, 7), 12, 19, 77910),
                                                  (dm.red2_line, (0, 1, 3, 5, 7), 13, 20, 85759)])
def test_int32_bounds(line, n_in, p1, p2, norm):
    """the L1 norm of every sum of jpeg_idct_4x4 / jpeg_idct_2x2, as a linear form of the inputs a line reads, found by brute force
    over their sign patterns; the bounds turbo_sm90.cu uses follow from it, and int16 coefficients exceed the pass-1 bound"""
    found = 0
    for signs in itertools.product((-1, 1), repeat=len(n_in)):
        d = [0] * 8
        for i, s in zip(n_in, signs):
            d[i] = s
        rec = []
        line(d, p1, rec)
        found = max(found, max(abs(v) for v in rec))
    assert found == norm
    pass1, pass2 = (2 ** 31 - 1 - 2 ** (p1 - 1)) // norm, (2 ** 31 - 1 - 2 ** (p2 - 1)) // norm
    assert pass1 < 32768  # unlike islow: a block with larger coefficients runs pass 1 in 64 bits
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "libjpeg_b200", "csrc", "turbo_sm90.cu")).read()
    name = "Red4" if line is dm.red4_line else "Red2"
    assert "k%sPass1Exact = %d, k%sPass2Exact = %d" % (name, pass1, name, pass2) in src
    assert (pass1, pass2) == ((27563, 27560) if name == "Red4" else (25040, 25034))


def _wrapped_pass1_block(F, line, p1, p2, s):
    """the s x s samples of block F with every pass-1 result computed in int32 (wrapped mod 2^32), pass 2 exact"""
    def wrap(v):
        return ((v + 2 ** 31) % 2 ** 32) - 2 ** 31
    ws = np.zeros((s, 8), dtype=np.int64)
    for k in range(8):
        rec = []
        line([int(v) for v in F[:, k]], p1, rec)
        ws[:, k] = [wrap(v + (1 << (p1 - 1))) >> p1 for v in rec[-s:]]
    return dm.tm.range_limit(np.stack(line([ws[:, u] for u in range(8)], p2), axis=-1))


@pytest.mark.parametrize("line,n_in,p1,p2,s,bound", [(dm.red4_line, (0, 1, 2, 3, 5, 6, 7), 12, 19, 4, 27563),
                                                     (dm.red2_line, (0, 1, 3, 5, 7), 13, 20, 2, 25040)])
def test_bound_blocks_observable(line, n_in, p1, p2, s, bound):
    """the pass-1 bound blocks of tests/test_draft.py (the worst sign pattern down column 1): at bound + 1 an int32 pass 1 gives
    other bytes than the exact IDCT, at the bound the same; down column 0 the difference would hide behind the range-limit table"""
    worst, best = None, -1
    for signs in itertools.product((-1, 1), repeat=len(n_in)):
        d = [0] * 8
        for i, sg in zip(n_in, signs):
            d[i] = sg
        rec = []
        line(d, p1, rec)
        if max(abs(v) for v in rec) > best:
            best, worst = max(abs(v) for v in rec), np.array(d)
    for col, m, differs in ((1, bound, False), (1, bound + 1, True), (0, bound + 1, False)):
        F = np.zeros((8, 8), dtype=np.int64)
        F[:, col] = worst * m
        assert (not np.array_equal(dm.idct_blocks(F, s), _wrapped_pass1_block(F, line, p1, p2, s))) == differs, (col, m)


def test_idct_size_rule():
    """s_c for the layouts DESIGN §17 names: 4:2:0 chroma 1:1 with the luma, 4:2:2 / 4:4:0 chroma at the luma's size, 4 x 4 chroma
    at 8 from k = 2, 3x and 4:1:1 factors at m"""
    assert [(dm.idct_size([2, 1, 1], [2, 1, 1], 0, k), dm.idct_size([2, 1, 1], [2, 1, 1], 1, k)) for k in (2, 4, 8)] == [(4, 8), (2, 4), (1, 2)]
    assert [dm.idct_size([2, 1, 1], [1, 1, 1], 1, k) for k in (2, 4, 8)] == [4, 2, 1]
    assert [dm.idct_size([4, 1, 1], [4, 1, 1], 1, k) for k in (2, 4, 8)] == [8, 8, 4]
    assert [dm.idct_size([3, 1, 1], [1, 1, 1], 1, k) for k in (2, 4, 8)] == [4, 2, 1]
    assert [dm.idct_size([4, 1, 1], [1, 1, 1], 1, k) for k in (2, 4, 8)] == [4, 2, 1]


@pytest.mark.parametrize("value", [(0, 5), [3, 0], (1, 2, 3), "ab", (1.0, 2), (True, 3), (-1, 4), [(1, 2)]])
def test_draft_argument(built, value):
    """BatchDecoder(draft=...) is checked like resize: ValueError before a context (or a device) is touched"""
    with pytest.raises(ValueError, match="draft"):
        built.BatchDecoder([b"\xff\xd8\xff\xd9", b"\xff\xd8\xff\xd9"], ctx=object(), reconstruction="libjpeg-turbo", draft=value)


@pytest.mark.parametrize("value", [(0, 5), (5, 0), (0, 0), (1, 2, 3), None, (1.5, 2), (True, 1), (-2, 2)])
def test_draft_scale_argument(built, value):
    from libjpeg_b200 import decoder
    with pytest.raises(ValueError, match="draft"):
        decoder.draft_scale(_synth(16, 16, 1, (2, 2)), value)
