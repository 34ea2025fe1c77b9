"""No device: CMYK and YCCK frames under reconstruction="libjpeg-turbo" and an output mode (DESIGN §18). The model,
tests/turbo_cmyk_model.py (tests/draft_model.py's reconstruction of the four components, then §15's conversion), against
Pillow's Image.open(f) [.draft(mode, (w, h))] .convert(mode) byte for byte: the fixtures of tests/golden/cmyk at every scale, Pillow-written
CMYK files of every size up to 34 x 34 and their YCCK twins, hand-built four-component layouts, the chain draft -> orientation ->
crop -> resize, the stored expected.npz and the stored digests."""
import importlib.util
import io
import json
import os

import numpy as np
import pytest

from tests import cmyk_model as km
from tests import orientation_model as om
from tests import resize_model as rm
from tests import turbo_cmyk_model as tcm
from tests import turbo_model as tm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CMYK_DIR = os.path.join(GOLDEN, "cmyk")
FIXTURES = sorted(f[:-4] for f in os.listdir(CMYK_DIR) if f.endswith(".jpg"))
# the hand-built layouts: 4:4:4, the first component 2 x 2 (Pillow's subsampling=2), Y and K at 2 x 2 (libjpeg's YCCK default),
# at 2 x 1 and at 1 x 2
LAYOUTS = {"444": [(1, 1)] * 4, "first22": [(2, 2), (1, 1), (1, 1), (1, 1)], "yk22": [(2, 2), (1, 1), (1, 1), (2, 2)],
           "yk21": [(2, 1), (1, 1), (1, 1), (2, 1)], "yk12": [(1, 2), (1, 1), (1, 1), (1, 2)]}


@pytest.fixture(scope="module")
def oracle(built):
    from tests import oracle_binding
    return oracle_binding.load()


def _make():
    spec = importlib.util.spec_from_file_location("make_turbo_cmyk", os.path.join(CMYK_DIR, "make_turbo_cmyk.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _fixture(name):
    with open(os.path.join(CMYK_DIR, name + ".jpg"), "rb") as f:
        return f.read()


def _samples(oracle, data, k):
    """the four components as the turbo path reconstructs them at 1/k, before the conversion ([H', W', 4] uint8)"""
    from tests import draft_model as dm
    rc, info, planes = oracle.coefficients(data)
    assert rc == 0, rc
    return dm.reconstruct(tm.dequantised(info, planes), info.width, info.height, list(info.hs), list(info.vs), k, km.CMYK,
                          color_transform=False)


def _model(oracle, data, k, mode):
    """turbo_cmyk_model.reconstruct on the oracle's coefficients, as Pillow shapes it ([H', W'] for "L")"""
    from libjpeg_b200 import decoder
    rc, info, planes = oracle.coefficients(data)
    assert rc == 0, rc
    out = tcm.reconstruct(tm.dequantised(info, planes), info.width, info.height, list(info.hs), list(info.vs), k, decoder.colorspace(data), mode)
    return out[..., 0] if mode == "L" else out


def _check(oracle, data, k, modes=("RGB", "L")):
    """the model equals Pillow at the scale Pillow picks for a request of 1/k (a smaller one for a frame too small for k);
    returns that scale"""
    from libjpeg_b200 import decoder
    mk = _make()
    space = decoder.colorspace(data)
    assert space in (km.CMYK, km.YCCK)
    scale = None
    for mode in modes:
        s, want = mk.pillow(data, mode, k)
        assert scale in (None, s)
        scale = s
        got = km.convert(_samples(oracle, data, s), space, mode)
        got = got[..., 0] if mode == "L" else got
        assert got.shape == want.shape and np.array_equal(got, want), (mode, k, s)
    return scale


def _pillow_cmyk(w, h, seed, subsampling, rows=0, quality=85):
    from PIL import Image
    rng = np.random.default_rng(seed)
    x = np.linspace(0, 255, w)[None, :, None]
    y = np.linspace(0, 255, h)[:, None, None]
    px = np.clip(np.concatenate([x + 0 * y, y + 0 * x, 255 - (x + y) / 2, 128 + 0 * x * y], axis=-1) + rng.normal(0, 40, (h, w, 4)), 0, 255)
    buf = io.BytesIO()
    kw = dict(quality=quality, subsampling=subsampling)
    if rows:
        kw["restart_marker_rows"] = rows
    Image.fromarray(px.astype(np.uint8), "CMYK").save(buf, "JPEG", **kw)
    return buf.getvalue()


def _with_transform(data, t):
    at = data.find(b"\xff\xee")
    assert at >= 0 and data[at + 4:at + 9] == b"Adobe" and data[at + 4 + 11] == 0
    return data[:at + 4 + 11] + bytes([t]) + data[at + 4 + 12:]


@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures(oracle, name):
    """every fixture at k = 1, 2, 4 and 8 under "RGB" and "L", at the scale asked for"""
    pytest.importorskip("PIL.Image")
    assert [_check(oracle, _fixture(name), k) for k in (1, 2, 4, 8)] == [1, 2, 4, 8]


def test_fixtures_equal_expected(oracle):
    """the model at k = 1 on the oracle's coefficients equals the stored expected.npz (Pillow's convert), no Pillow needed"""
    expected = np.load(os.path.join(CMYK_DIR, "expected.npz"))
    assert len(FIXTURES) == 8
    for name in FIXTURES:
        for mode in ("RGB", "L"):
            assert np.array_equal(_model(oracle, _fixture(name), 1, mode), expected[name + "_" + mode]), (name, mode)


def test_digests_match_pillow():
    """turbo_digests.json is what Pillow gives here"""
    pytest.importorskip("PIL.Image")
    stored = json.load(open(os.path.join(CMYK_DIR, "turbo_digests.json")))
    assert stored == _make().table()
    assert len(stored) == len(FIXTURES) * 4 * 2


def test_model_matches_digests(oracle):
    """the model on the oracle's coefficients gives the stored digests, no Pillow needed"""
    mk = _make()
    stored = json.load(open(os.path.join(CMYK_DIR, "turbo_digests.json")))
    for key, d in stored.items():
        name, mode, _ = key.split("|")
        got = _model(oracle, _fixture(name), d["scale"], mode)
        assert list(got.shape) == d["shape"] and mk.digest(got) == d["sha256"], key


@pytest.mark.parametrize("k", [1, 2, 4, 8])
@pytest.mark.parametrize("subsampling", [0, 2])
def test_every_small_size(oracle, subsampling, k):
    """Pillow's CMYK files of every width 1..34 at two heights and every height 1..34 at two widths, some with restart rows, and
    YCCK twins of each at transform 1, 2 or 255"""
    pytest.importorskip("PIL.Image")
    sizes = [(w, h) for w in range(1, 35) for h in (1, 17)] + [(w, h) for h in range(1, 35) for w in (2, 19)]
    for j, (w, h) in enumerate(sizes):
        data = _pillow_cmyk(w, h, j, subsampling, rows=1 if j % 3 == 0 else 0)
        assert (b"\xff\xdd" in data) == (j % 3 == 0)
        _check(oracle, data, k, ("RGB", "L")[j % 2:j % 2 + 1])
        _check(oracle, _with_transform(data, (1, 2, 255)[j % 3]), k, ("RGB", "L")[(j + 1) % 2:(j + 1) % 2 + 1])


@pytest.mark.parametrize("rows", [0, 2])
def test_larger_files(oracle, rows):
    """larger Pillow-written CMYK files and their YCCK twins at every scale, both modes"""
    pytest.importorskip("PIL.Image")
    for j, (w, h, sub) in enumerate([(301, 97, 0), (256, 200, 2), (517, 67, 2)]):
        data = _pillow_cmyk(w, h, 40 + j, sub, rows)
        for k in (1, 2, 4, 8):
            assert _check(oracle, data, k) == k
            assert _check(oracle, _with_transform(data, 2), k) == k


def _hand_built(layout, w, h, transform, seed):
    from tests import recon_cases as rc
    from tests import streamwriter as sw
    factors = LAYOUTS[layout]
    _, comps = rc.base(w, h, seed, factors)
    return km.after_soi(sw.encode(rc.frame(w, h, comps, factors)), km.adobe(transform))


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_hand_built_layouts(oracle, layout):
    """hand-built four-component frames (quantisers 1, every component its own content) with Adobe transform 0 and 2, at 77 x 45,
    130 x 66 and 5 x 3, at every scale, both modes"""
    pytest.importorskip("PIL.Image")
    for j, (w, h) in enumerate([(77, 45), (130, 66), (5, 3)]):
        for t in (0, 2):
            data = _hand_built(layout, w, h, t, 500 + 7 * j + t)
            scales = [_check(oracle, data, k) for k in (1, 2, 4, 8)]
            assert scales[:2] == [1, 2] and scales == sorted(scales), scales


def _chain_frames():
    out = []
    for j, (w, h, sub) in enumerate([(197, 161, 2), (164, 148, 0), (133, 117, 2), (230, 170, 0)]):
        data = _pillow_cmyk(w, h, 80 + j, sub, rows=j % 2)
        for o in (1 + 2 * j, 2 + 2 * j):
            out.append(om.tag(data if o % 2 else _with_transform(data, 2), o))
    return out


@pytest.mark.parametrize("resample", sorted(rm.NAMES))
def test_chain_equals_pillow(oracle, resample):
    """the model at Pillow's scale -> orientation -> crop -> tests/resize_model.py equals im.draft(mode, (w, h)) followed by
    ImageOps.exif_transpose(im).convert(mode).crop(box).resize(size, filter), all eight orientations, every scale, both modes"""
    pytest.importorskip("PIL.Image")
    from PIL import Image, ImageOps
    rng = np.random.default_rng(len(resample))
    for j, data in enumerate(_chain_frames()):
        k, mode = (1, 2, 4, 8)[j % 4], ("RGB", "L")[(j // 4) % 2]
        im = Image.open(io.BytesIO(data))
        if k > 1:
            im.draft(mode, (im.size[0] // k, im.size[1] // k))
        assert (im.decoderconfig[0] if im.decoderconfig else 1) == k
        o = im.getexif().get(0x0112, 1)
        assert o == j + 1
        oriented = om.orient(_model(oracle, data, k, mode), o)
        oh, ow = oriented.shape[:2]
        x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
        cw, ch = int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))
        tw, th = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        got = rm.resize(np.ascontiguousarray(oriented[y:y + ch, x:x + cw]), tw, th, rm.NAMES[resample])
        pil = ImageOps.exif_transpose(im).convert(mode).crop((x, y, x + cw, y + ch))
        want = np.asarray(pil.resize((tw, th), rm.NAMES[resample]))
        assert np.array_equal(got, want), (o, k, mode, resample)
