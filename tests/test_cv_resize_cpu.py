"""CPU: pins tests/cv_resize_model.py (DESIGN §20) on the installed OpenCV -- cv2.resize with INTER_LINEAR and INTER_AREA, one
thread and the default thread count, IPP on and off -- and checks b200jpg_resample_coefficients' cv tables, the stored OpenCV
digests of tests/golden/cv_resize against the model on tests/turbo_model.py's decode, and the Python argument checks."""
import ctypes
import hashlib
import itertools
import json
import math
import os

import numpy as np
import pytest

from tests import cv_resize_model as cvm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def cv2():
    cv2 = pytest.importorskip("cv2")
    threads, ipp = cv2.getNumThreads(), cv2.ipp.useIPP()
    yield cv2
    cv2.setNumThreads(threads)
    cv2.ipp.setUseIPP(ipp)


SETTINGS = [(1, True), (1, False), (None, True), (None, False)]  # (threads: None = the default count, IPP)


def _settings(cv2, threads, ipp, default):
    cv2.setNumThreads(default if threads is None else threads)
    cv2.ipp.setUseIPP(ipp)


def _cv(cv2, img, w, h, name):
    out = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR if name == "cv2-linear" else cv2.INTER_AREA)
    return out.reshape(out.shape[:2] + (img.shape[2],)) if img.ndim == 3 else out


@pytest.mark.parametrize("name", list(cvm.NAMES))
@pytest.mark.parametrize("threads,ipp", SETTINGS)
def test_every_small_pair(cv2, name, threads, ipp):
    """every (w, W_t) x (h, H_t) up to 24 per axis: integer factors, up, down and mixed axes; 1 and 3 channels"""
    default = cv2.getNumThreads()
    _settings(cv2, threads, ipp, default)
    rng = np.random.default_rng(7)
    rules = set()
    for k, (w, W) in enumerate(itertools.product(range(1, 25), repeat=2)):
        c = 3 if k % 2 else 1
        for h in (1 + k % 24, 1 + (k * 7) % 24):
            img = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
            for H in range(1, 25):
                rules.add(cvm.rule(w, h, W, H, cvm.NAMES[name]))
                assert np.array_equal(cvm.resize(img, W, H, name), _cv(cv2, img, W, H, name)), (w, h, W, H, c)
    assert rules == ({"copy", 1} if name == "cv2-linear" else {"copy", 2, 3, 4})


@pytest.mark.parametrize("name", list(cvm.NAMES))
@pytest.mark.parametrize("threads,ipp", SETTINGS)
def test_random_sizes(cv2, name, threads, ipp):
    """seeded random sizes up to 2000, 1, 3 and 4 channels"""
    default = cv2.getNumThreads()
    _settings(cv2, threads, ipp, default)
    rng = np.random.default_rng(11 + list(cvm.NAMES).index(name))
    for k in range(60):
        top = 2000 if k % 3 == 0 else 300
        w, h, W, H = (int(v) for v in rng.integers(1, top + 1, 4))
        if k % 5 == 0:  # integer factors
            W, H = max(1, w // int(rng.integers(1, 9))), max(1, h // int(rng.integers(1, 9)))
            w, h = W * max(1, w // W), H * max(1, h // H)
        c = (1, 3, 4)[k % 3]
        img = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        assert np.array_equal(cvm.resize(img, W, H, name), _cv(cv2, img, W, H, name)), (w, h, W, H, c)


def _smooth(w, h, seed):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    rng = np.random.default_rng(seed)
    planes = [127.5 + 100 * np.sin(a * x + b * y) + rng.normal(0, 8, (h, w)) for a, b in rng.uniform(0.001, 0.05, (3, 2))]
    return np.clip(np.stack(planes, -1), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)])
def test_large_frames(cv2, w, h):
    """1080p and 4K to ultralytics' sizes (long side 640, ceil(w r)), to 224 x 224 and to 1138 x 640"""
    img = _smooth(w, h, w)
    r = 640 / max(w, h)
    for W, H in ((min(math.ceil(w * r), 640), min(math.ceil(h * r), 640)), (224, 224), (1138, 640)):
        for name in cvm.NAMES:
            for ipp in (True, False):
                cv2.ipp.setUseIPP(ipp)
                assert np.array_equal(cvm.resize(img, W, H, name), _cv(cv2, img, W, H, name)), (w, h, W, H, name, ipp)
    cv2.ipp.setUseIPP(True)


def _table(built, in_size, out_size, resample):
    from libjpeg_b200 import native
    ks = ctypes.c_uint32()
    assert native.lib.b200jpg_resample_coefficients(in_size, out_size, resample, None, None, 0, ctypes.byref(ks)) == 0
    bounds = np.zeros(2 * out_size, dtype=np.int32)
    coef = np.zeros(out_size * ks.value, dtype=np.int32)
    assert native.lib.b200jpg_resample_coefficients(in_size, out_size, resample, bounds.ctypes.data, coef.ctypes.data, coef.size,
                                                    ctypes.byref(ks)) == 0
    return bounds, coef, ks.value


def test_table_entry_point(built):
    """b200jpg_resample_coefficients for both ids, both axes and rule 4's flag equals the model's tables; the box entry point
    refuses the cv ids"""
    from libjpeg_b200 import native
    ids = [cvm.LINEAR, cvm.LINEAR | cvm.TABLE_VERTICAL, cvm.AREA, cvm.AREA | cvm.TABLE_VERTICAL, cvm.AREA | cvm.TABLE_LINEAR,
           cvm.AREA | cvm.TABLE_LINEAR | cvm.TABLE_VERTICAL]
    pairs = [(i, o) for i in range(1, 34) for o in range(1, 34)] + [(1920, 640), (3840, 1138), (1080, 360), (7, 2000), (2000, 7)]
    for (i, o), r in itertools.product(pairs, ids):
        got, want = _table(built, i, o, r), cvm.coefficients(i, o, r)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2], (i, o, hex(r))
    ks = ctypes.c_uint32()
    for r in (cvm.LINEAR, cvm.AREA):
        assert native.lib.b200jpg_resample_coefficients_box(10, 0.0, 10.0, 5, r, None, None, 0, ctypes.byref(ks)) == -1024
    for r in (0x102, 0x100, cvm.TABLE_VERTICAL | 2, cvm.LINEAR | 0x4000):
        assert native.lib.b200jpg_resample_coefficients(10, 5, r, None, None, 0, ctypes.byref(ks)) == -1024, hex(r)


def _digest(a):
    a = a[..., None] if a.ndim == 2 else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":%dx%dx%d" % a.shape


def test_stored_digests(built):
    """every stored OpenCV digest equals the model on the libjpeg-turbo model's decode of the fixture (mode "RGB" as BGR for
    IMREAD_COLOR, "L" for IMREAD_GRAYSCALE)"""
    from libjpeg_b200 import decoder
    from tests import oracle_binding
    from tests import turbo_model as tm
    oracle = oracle_binding.load()
    with open(os.path.join(GOLDEN, "cv_resize", "digests.json")) as f:
        stored = json.load(f)["frames"]
    assert len(stored) == 20
    for name, d in stored.items():
        data = open(os.path.join(GOLDEN, name), "rb").read()
        imgs = {"color": tm.decode(oracle, data, decoder.colorspace(data), "RGB")[..., ::-1],
                "gray": tm.decode(oracle, data, decoder.colorspace(data), "L")}
        for k, v in d.items():
            mode, interp, wh = k.split("_")
            w, h = (int(x) for x in wh.split("x"))
            assert _digest(cvm.resize(imgs[mode], w, h, "cv2-" + interp)) == v, (name, k)


def test_stored_digests_are_opencvs(cv2):
    """the stored digests are what the installed OpenCV gives (skipped when it is not the 4.13 they were made with)"""
    import importlib.util
    with open(os.path.join(GOLDEN, "cv_resize", "digests.json")) as f:
        stored = json.load(f)
    if cv2.__version__ != stored["opencv"]:
        pytest.skip("OpenCV %s, digests of %s" % (cv2.__version__, stored["opencv"]))
    spec = importlib.util.spec_from_file_location("make_cv_resize", os.path.join(GOLDEN, "cv_resize", "make_cv_resize.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    for name, path in mk.fixtures():
        data = np.fromfile(path, dtype=np.uint8)
        img = cv2.imdecode(data, cv2.IMREAD_COLOR)
        w, h = img.shape[1], img.shape[0]
        for tw, th in mk.sizes(w, h):
            assert mk.digest(cv2.resize(img, (tw, th), interpolation=cv2.INTER_AREA)) == stored["frames"][name]["color_area_%dx%d" % (tw, th)]


def test_python_arguments(built):
    """the filter names map to the C ids; unknown names raise ValueError"""
    from libjpeg_b200 import native
    from libjpeg_b200.decoder import resample_filter
    assert resample_filter("cv2-linear") == 0x101 and resample_filter("cv2-area") == 0x103
    assert native.RESAMPLE["bilinear"] == 2
    for bad in ("cv2-cubic", "CV2-LINEAR", "area", 0x101, None):
        with pytest.raises(ValueError):
            resample_filter(bad)
