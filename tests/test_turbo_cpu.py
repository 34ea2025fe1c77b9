"""No device: the libjpeg-turbo reconstruction model (tests/turbo_model.py, DESIGN §16) against Pillow byte for byte -- stored
vectors, synthetic streams of every size up to 34 x 34 in every sampling, progressive and restart variants, 1080p and 4K, draft("L"),
and the chain orientation -> crop -> resize -- plus the int32 bounds of turbo_idct_kernel, the Python argument checks and the
stored Pillow digests."""
import importlib.util
import io
import itertools
import json
import os

import numpy as np
import pytest

from tests import orientation_model as om
from tests import resize_model as rm
from tests import turbo_model as tm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SAMPLINGS = {"420": (2, 2), "422": (2, 1), "440": (1, 2), "444": (1, 1), "grey": None}


@pytest.fixture(scope="module")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()


def _make_turbo():
    spec = importlib.util.spec_from_file_location("make_turbo", os.path.join(GOLDEN, "turbo", "make_turbo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _model(oracle, data, mode=None):
    from libjpeg_b200 import decoder
    out = tm.decode(oracle, data, decoder.colorspace(data), mode)
    return out[..., 0] if out.shape[2] == 1 else out


def _pillow(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)))


def _synth(w, h, seed, sampling, restart=0):
    from libjpeg_b200 import synth
    img = synth.source_image(w, h, seed)
    return synth.encode(img[..., 0] if sampling is None else img, 80, sampling or (1, 1), restart).tobytes()


def test_stored_vectors(oracle):
    pytest.importorskip("PIL.Image")
    mk = _make_turbo()
    n = 0
    for rel in mk.vectors():
        want = mk.pillow_pixels(rel)
        if want is None:
            continue
        assert np.array_equal(_model(oracle, open(os.path.join(GOLDEN, rel), "rb").read()), want), rel
        n += 1
    assert n == 41


def test_digests_match_pillow():
    """pil_digests.json is what Pillow gives here"""
    pytest.importorskip("PIL.Image")
    stored = json.load(open(os.path.join(GOLDEN, "turbo", "pil_digests.json")))
    assert stored == _make_turbo().table()


@pytest.mark.parametrize("name", list(SAMPLINGS))
def test_every_small_size(oracle, name):
    """every width 1..34 at two heights and every height 1..34 at two widths: w = 1, 2, 3, odd sizes, MCU padding"""
    pytest.importorskip("PIL.Image")
    sizes = [(w, h) for w in range(1, 35) for h in (1, 17)] + [(w, h) for h in range(1, 35) for w in (2, 19)]
    for k, (w, h) in enumerate(sizes):
        data = _synth(w, h, k, SAMPLINGS[name], restart=1 if k % 3 == 0 else 0)
        assert np.array_equal(_model(oracle, data), _pillow(data)), (name, w, h)


@pytest.mark.parametrize("name", ["420", "422", "444", "grey"])
def test_progressive(oracle, name):
    """Pillow's own progressive (and optimised-table) streams"""
    Image = pytest.importorskip("PIL.Image")
    from libjpeg_b200 import synth
    for k, (w, h) in enumerate([(1, 1), (3, 5), (33, 17), (97, 61), (130, 70)]):
        img = synth.source_image(w, h, 50 + k)
        im = Image.fromarray(img[..., 0]) if name == "grey" else Image.fromarray(img)
        buf = io.BytesIO()
        kw = {} if name == "grey" else {"subsampling": {"444": 0, "422": 1, "420": 2}[name]}
        im.save(buf, "JPEG", quality=85, progressive=True, optimize=True, **kw)
        data = buf.getvalue()
        assert np.array_equal(_model(oracle, data), _pillow(data)), (name, w, h)


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)])
def test_large(oracle, w, h):
    pytest.importorskip("PIL.Image")
    data = _synth(w, h, 7, (2, 2), restart=8)
    assert np.array_equal(_model(oracle, data), _pillow(data))


def test_draft_luma(oracle):
    """mode "L" of a YCbCr frame is Pillow's draft("L") at full size"""
    Image = pytest.importorskip("PIL.Image")
    frames = [open(os.path.join(GOLDEN, f), "rb").read() for f in ("c420_127x255_z7_q30.jpg", "c422_100x60_z5_q80.jpg",
                                                                    "c440_100x61_z3_q80.jpg", "c444_17x9_q95.jpg")]
    frames += [open(os.path.join(GOLDEN, "subsampling", "c410_97x53_z3_q75.jpg"), "rb").read(), _synth(35, 3, 1, (2, 2))]
    for data in frames:
        im = Image.open(io.BytesIO(data))
        im.draft("L", im.size)
        assert im.mode == "L"
        assert np.array_equal(_model(oracle, data, "L"), np.asarray(im))


def _chain_frames():
    from libjpeg_b200 import synth
    out = []
    for k, (w, h, s) in enumerate([(97, 61, (2, 2)), (64, 48, (1, 1)), (100, 70, (2, 1)), (61, 97, (1, 2)), (33, 17, (2, 2)),
                                   (40, 24, None), (130, 70, (2, 2)), (75, 61, (2, 1)), (127, 99, (2, 2)), (50, 38, (1, 1)),
                                   (17, 9, (2, 2)), (96, 80, (2, 1))]):
        img = synth.source_image(w, h, 80 + k)
        data = synth.encode(img[..., 0] if s is None else img, 85, s or (1, 1), 0).tobytes()
        out.append(om.tag(data, 1 + k % 8))
    return out


@pytest.mark.parametrize("resample", sorted(rm.NAMES))
def test_chain_equals_pillow(oracle, resample):
    """the model -> orientation -> crop -> tests/resize_model.py equals ImageOps.exif_transpose(Image.open(f)).convert("RGB")
    .crop(box).resize(size, filter) for a dozen frames, all eight orientations"""
    pytest.importorskip("PIL.Image")
    from PIL import Image, ImageOps
    rng = np.random.default_rng(3)
    for data in _chain_frames():
        img = _model(oracle, data, "RGB")
        o = Image.open(io.BytesIO(data)).getexif().get(0x0112, 1)
        oriented = om.orient(img, o)
        oh, ow = oriented.shape[:2]
        x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
        cw, ch = int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))
        tw, th = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        got = rm.resize(np.ascontiguousarray(oriented[y:y + ch, x:x + cw]), tw, th, rm.NAMES[resample])
        pil = ImageOps.exif_transpose(Image.open(io.BytesIO(data))).convert("RGB").crop((x, y, x + cw, y + ch))
        want = np.asarray(pil.resize((tw, th), rm.NAMES[resample]))
        assert np.array_equal(got, want), (o, resample)


def test_int32_bounds():
    """the L1 norm of every sum of the islow butterfly, as a linear form of its 8 inputs, found by brute force over the 256 sign
    patterns; the bounds turbo_sm90.cu uses follow from it (pass 1 adds 2^10 before its shift, pass 2 2^17)"""
    norm = 0
    for signs in itertools.product((-1, 1), repeat=8):
        rec = []
        tm.idct1d(list(signs), tm.PASS1_SHIFT, rec)
        norm = max(norm, max(abs(v) for v in rec))
    assert norm == 61214
    pass1, pass2 = (2 ** 31 - 1 - 2 ** 10) // norm, (2 ** 31 - 1 - 2 ** 17) // norm
    assert (pass1, pass2) == (35081, 35079)
    assert pass1 >= 32768  # every int16 coefficient of the store runs pass 1 in int32
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "libjpeg_b200", "csrc", "turbo_sm90.cu")).read()
    assert "kPass1Exact = %d, kPass2Exact = %d;" % (pass1, pass2) in src
    # the pass-2 bound is tight: the worst sign pattern at pass2 + 1 leaves int32, at pass2 it does not
    worst = None
    for signs in itertools.product((-1, 1), repeat=8):
        rec = []
        tm.idct1d(list(signs), tm.PASS2_SHIFT, rec)
        if max(abs(v) for v in rec) == norm:
            worst = signs
    for m, leaves in ((pass2, False), (pass2 + 1, True)):
        rec = []
        tm.idct1d([s * m for s in worst], tm.PASS2_SHIFT, rec)
        assert (max(abs(v) for v in rec) + 2 ** 17 > 2 ** 31 - 1) == leaves


def test_range_limit_table():
    v = np.arange(-2048, 2048)
    i = v & 1023
    want = np.where(i < 128, i + 128, np.where(i < 512, 255, np.where(i < 896, 0, i - 896)))
    assert np.array_equal(tm.range_limit(v), want)
    assert np.array_equal(tm.range_limit(np.arange(-128, 128)), np.arange(0, 256))


@pytest.mark.parametrize("value", ["libjpeg", "Reference", "", None, 1, True])
def test_reconstruction_argument(built, value):
    """any other value than "reference" and "libjpeg-turbo" raises ValueError before a context (or a device) is created"""
    with pytest.raises(ValueError, match="reconstruction"):
        built.BatchDecoder([b"\xff\xd8\xff\xd9"], ctx=object(), reconstruction=value)


def test_flag_value(built):
    from libjpeg_b200 import native
    assert native.RECONSTRUCTION_FLAGS == {"reference": 0, "libjpeg-turbo": 0x80}
    hdr = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "b200jpg.h")).read()
    assert "#define B200JPG_FLAG_LIBJPEG_TURBO 0x80u" in hdr
