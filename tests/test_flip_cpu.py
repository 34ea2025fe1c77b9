"""CPU: the flip model of tests/flip_model.py (DESIGN §21) against numpy, the fact that keeps a resized frame's flip behind its
resize, and the argument checks of BatchDecoder(hflip=..., vflip=...) that run before a device is touched."""
import numpy as np
import pytest

from tests import flip_model as fm
from tests import orientation_model as om

FLIPS = range(4)


@pytest.mark.parametrize("o", om.ORIENTATIONS)
def test_dihedral_product(o):
    """flip(orient(D, o), f) is orient(D, ORIENTATION[o - 1][f]) for every orientation and flip"""
    d = np.random.default_rng(o).integers(0, 256, (5, 7, 3), dtype=np.uint8)
    for f in FLIPS:
        want = fm.flip(om.orient(d, o), f)
        got = om.orient(d, fm.ORIENTATION[o - 1][f])
        assert got.shape == want.shape and np.array_equal(got, want), (o, f)


def test_product_is_a_group_action():
    """flipping twice by f is the identity, and H then V is H | V"""
    for o in om.ORIENTATIONS:
        for f in FLIPS:
            assert fm.ORIENTATION[fm.ORIENTATION[o - 1][f] - 1][f] == o
        assert fm.ORIENTATION[fm.ORIENTATION[o - 1][fm.H] - 1][fm.V] == fm.ORIENTATION[o - 1][fm.H | fm.V]


def test_mirrored_rectangle():
    """flip(O[y:y + h, x:x + w]) is flip(O)[y':y' + h, x':x' + w] of the mirrored rectangle, for random rectangles"""
    rng = np.random.default_rng(7)
    for _ in range(300):
        H, W = (int(v) for v in rng.integers(1, 40, 2))
        o = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
        x, y = int(rng.integers(0, W)), int(rng.integers(0, H))
        w, h = int(rng.integers(1, W - x + 1)), int(rng.integers(1, H - y + 1))
        for f in FLIPS:
            mx, my, mw, mh = fm.flip_rect((x, y, w, h), f, W, H)
            assert np.array_equal(fm.flip(o, f)[my:my + mh, mx:mx + mw], fm.flip(o[y:y + h, x:x + w], f))


def _non_commuting(resize, seed):
    """of 200 seeded cases (sizes 5..300 -> 3..260, grey or RGB), how many give flip(resize(x)) != resize(flip(x)) for H"""
    rng = np.random.default_rng(seed)
    count = 0
    for _ in range(200):
        h, w = (int(v) for v in rng.integers(5, 301, 2))
        th, tw = (int(v) for v in rng.integers(3, 261, 2))
        x = rng.integers(0, 256, (h, w) if rng.integers(0, 2) else (h, w, 3), dtype=np.uint8)
        a = fm.flip(resize(x, tw, th), fm.H)
        b = resize(fm.flip(x, fm.H), tw, th)
        count += not np.array_equal(a, b)
    return count


def _pil_box(x, tw, th):
    from PIL import Image
    return np.asarray(Image.fromarray(x).resize((tw, th), Image.Resampling.BOX))


def _cv(interpolation):
    def run(x, tw, th):
        import cv2
        return cv2.resize(x, (tw, th), interpolation=getattr(cv2, interpolation))
    return run


@pytest.mark.parametrize("name,resize,count", [("pil-box", _pil_box, 53), ("cv2-linear", _cv("INTER_LINEAR"), 56),
                                               ("cv2-area", _cv("INTER_AREA"), 66)])
def test_flip_does_not_commute_with_resize(name, resize, count):
    """the reason a resized frame's flip is applied to the resampled image, never folded into the orientation before it: the
    resamplers are not mirror-symmetric (Pillow 12.2, OpenCV 4.13)"""
    if name.startswith("cv2"):
        pytest.importorskip("cv2")
    assert _non_commuting(resize, 11) == count


@pytest.mark.parametrize("kw", [{"hflip": [True]}, {"vflip": [True, False, True]}, {"hflip": 1}, {"hflip": [1, 0]},
                                {"vflip": [True, None]}, {"hflip": "yes"}, {"vflip": np.array([1, 0])}])
def test_flip_arguments(kw):
    """a wrong length or a value that is not a bool raises ValueError before a device is touched"""
    from libjpeg_b200 import BatchDecoder
    with pytest.raises(ValueError):
        BatchDecoder([b"\xff\xd8\xff\xd9"] * 2, **kw)


def test_flip_table():
    from libjpeg_b200 import native
    from libjpeg_b200.decoder import flip_table
    assert flip_table(None, None, 3) is None
    assert flip_table(False, [False, False, False], 3) is None
    t = flip_table([True, False, np.bool_(True)], True, 3)
    assert list(t) == [native.FLIP_H | native.FLIP_V, native.FLIP_V, native.FLIP_H | native.FLIP_V]
