"""CPU: the specification of downscaled decoding (tests/downscale_model.py) -- the folding identity, the fixed-point scaled IDCT
against the exact box average, the sample-plane reconstruction against the oracle, the reduced geometry and the Python
argument checks."""
import glob
import os

import numpy as np
import pytest

from tests import downscale_model as dm
from tests import oracle_binding

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# every golden vector the oracle decodes whole (JPEG XT and damaged streams excluded: no residual merge here, and a damaged
# stream has no full decode to compare with)
VECTORS = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg")) + glob.glob(os.path.join(GOLDEN, "progressive", "*.jpg")) +
                 glob.glob(os.path.join(GOLDEN, "subsampling", "*.jpg")) + glob.glob(os.path.join(GOLDEN, "deep12", "*.jpg")) +
                 glob.glob(os.path.join(GOLDEN, "dnl", "*.jpg")) + glob.glob(os.path.join(GOLDEN, "reference", "sub_*.jpg")))
# largest |model - exact box average| in sample levels (1/16 of an output level), per precision
# largest measured: 0.572 (random 8-bit blocks), 0.770 (random 12-bit blocks, every coefficient up to 2^14), 0.539 (golden)
MAX_MODEL_ERROR = {8: 0.6, 12: 0.8}


@pytest.fixture(scope="module")
def oracle():
    return oracle_binding.load()


def _dequantised(oracle, data):
    rc, s, planes = oracle.coefficients(data)
    assert rc == 0
    return s, [planes[c].astype(np.int64) * np.asarray(s.quant[s.tq[c]], dtype=np.int64).reshape(8, 8) for c in range(s.ncomp)]


def _random_blocks(rng, n, big):
    F = np.zeros((n, 8, 8), dtype=np.int64)
    mag = rng.integers(1, big, size=(n, 1, 1))
    F[:] = rng.integers(-1, 2, size=(n, 8, 8)) * rng.integers(0, 1 << 15, size=(n, 8, 8)) % (mag + 1)
    F[:, 0, 0] = rng.integers(-1024 * 8, 1024 * 8, size=n)
    return F


@pytest.mark.parametrize("k", [2, 4])
def test_folding_identity(k):
    """the k x k box average of the exact IDCT is the (8/k)-point IDCT of the folded coefficients, F(8/k... ) dropping out"""
    rng = np.random.default_rng(k)
    F = rng.normal(size=(200, 8)) * 100
    M = dm.idct8_matrix()  # x = M F, C(u)/2 normalisation
    box = (F @ M.T).reshape(200, 8 // k, k).mean(axis=2)
    # fold: G(0) = F(0), G(u) = cos(u pi/16) F(u) - cos((8 - u) pi/16) F(8 - u), u = 1..3; F(4) drops out
    G = np.zeros((200, 4))
    G[:, 0] = F[:, 0]
    for u in range(1, 4):
        G[:, u] = np.cos(u * np.pi / 16) * F[:, u] - np.cos((8 - u) * np.pi / 16) * F[:, 8 - u]
    if k == 4:  # fold once more: H(0) = G(0), H(1) = cos(pi/8) G(1) - cos(3 pi/8) G(3), G(2) drops out
        H = np.zeros((200, 2))
        H[:, 0] = G[:, 0]
        H[:, 1] = np.cos(np.pi / 8) * G[:, 1] - np.cos(3 * np.pi / 8) * G[:, 3]
        G = H
    n = G.shape[1]
    folded = np.zeros((200, n))
    for m in range(n):
        for u in range(n):
            cu = 1 / np.sqrt(2) if u == 0 else 1.0
            folded[:, m] += 0.5 * cu * G[:, u] * np.cos((2 * m + 1) * u * np.pi / (2 * n))
    np.testing.assert_allclose(folded, box, atol=1e-9)
    # and the matrix of the specification is that average
    np.testing.assert_allclose(F @ dm.basis(k).T, box, atol=1e-9)


def test_dc_only_for_k8():
    rng = np.random.default_rng(8)
    F = rng.normal(size=(50, 8, 8)) * 100
    M = dm.idct8_matrix()
    np.testing.assert_allclose(np.einsum("xr,brc,yc->bxy", M, F, M).mean(axis=(1, 2)), F[:, 0, 0] / 8, atol=1e-9)


@pytest.mark.parametrize("k", [2, 4])
def test_basis_table_is_the_rounded_matrix(k):
    assert np.array_equal(dm.BASIS[k], np.floor(dm.basis(k) * (1 << 20) + 0.5).astype(np.int64))


@pytest.mark.parametrize("k", [2, 4, 8])
@pytest.mark.parametrize("precision", [8, 12])
def test_model_against_exact_box_average_random(k, precision):
    rng = np.random.default_rng(100 * k + precision)
    F = _random_blocks(rng, 4000, 2048 if precision == 8 else 16384)
    err = np.abs(dm.scaled_blocks(F, k, precision) - dm.exact_box_average(F, k, precision)).max()
    assert err < MAX_MODEL_ERROR[precision]
    if k == 8:  # exact
        assert err < 1e-9
    # the extremes of the int16 store do not wrap
    ext = np.full((1, 8, 8), -32768, dtype=np.int64) * np.array([[1, -1] * 4] * 8)
    assert np.abs(dm.scaled_blocks(ext, k, precision) - dm.exact_box_average(ext, k, precision)).max() < 1


@pytest.mark.parametrize("path", VECTORS, ids=os.path.basename)
def test_model_against_exact_box_average_golden(oracle, path):
    s, coefs = _dequantised(oracle, open(path, "rb").read())
    for k in (2, 4, 8):
        for F in coefs:
            F = F.reshape(-1, 8, 8)
            assert np.abs(dm.scaled_blocks(F, k, s.precision) - dm.exact_box_average(F, k, s.precision)).max() < MAX_MODEL_ERROR[s.precision]


@pytest.mark.parametrize("path", VECTORS, ids=os.path.basename)
def test_reconstruct_samples_is_the_reference(oracle, path):
    """fed with the reference's full-size IDCT planes, the model's reconstruction is jpgo_decode byte for byte"""
    data = open(path, "rb").read()
    s, coefs = _dequantised(oracle, data)
    planes = [dm.full_planes(oracle, F, s.precision) for F in coefs]
    n = s.ncomp
    got = dm.reconstruct_samples(planes, list(s.subx[:n]), list(s.suby[:n]), s.width, s.height, s.precision, s.ycbcr)
    rc, ref = oracle.decode16(data) if s.precision > 8 else oracle.decode(data)
    assert rc == 0
    assert np.array_equal(got, ref)


def test_scaled_extents():
    for W, H, k, want in [(1, 1, 8, (1, 1)), (17, 9, 2, (9, 5)), (17, 9, 4, (5, 3)), (17, 9, 8, (3, 2)), (127, 255, 4, (32, 64)),
                          (3840, 2160, 8, (480, 270))]:
        assert dm.scaled_extent(W, H, k) == want
    # the planes of the scaled IDCT already cover the reduced components: ceil(ceil(W / sx) / k) == ceil(ceil(W / k) / sx)
    for W in range(1, 80):
        for sx in (1, 2, 3, 4):
            for k in (2, 4, 8):
                assert -(-(-(-W // sx)) // k) == -(-(-(-W // k)) // sx)
                bw = -(-(-(-W // sx)) // 8)  # at least the component's block columns
                assert (8 // k) * bw >= -(-(-(-W // k)) // sx)


def test_downscale_argument_checks():
    pytest.importorskip("torch")
    try:
        from libjpeg_b200.decoder import BatchDecoder
    except ImportError:
        pytest.skip("library not built")
    data = open(os.path.join(GOLDEN, "c420_33x17_q50.jpg"), "rb").read()
    for bad in (0, 3, 16, -2, 2.0, "2", True, None):
        with pytest.raises(ValueError):
            BatchDecoder([data], downscale=bad)


# largest |model - box average of the reference's own planes| in output levels over the k x k groups without a clamped sample,
# measured: 1.0 at k = 2 (53251 groups), 0.75 at k = 4 (12900), 0.625 at k = 8 (3057). The reference's planes are rounded
# samples, so their average already differs from the exact one by up to half a level.
MAX_PLANE_ERROR = {2: 1.0, 4: 0.75, 8: 0.625}


def _reference_planes():
    d = np.load(os.path.join(GOLDEN, "planes.npz"))
    names = sorted({key.rsplit("__", 1)[0] for key in d.keys()})
    return d, names


@pytest.mark.parametrize("k", [2, 4, 8])
def test_model_against_reference_planes(oracle, k):
    """model + planes_out at k against the k x k box average of what the unmodified reference writes without upsampling
    (tests/golden/planes.npz), over every whole group that holds no clamped sample"""
    d, names = _reference_planes()
    worst, groups = 0.0, 0
    for name in names:
        sub, _, rest = name.partition("__")  # keys of vectors in a subdirectory: <dir>__<name>__<component>
        path = os.path.join(GOLDEN, sub, rest + ".jpg") if rest and os.path.isdir(os.path.join(GOLDEN, sub)) else os.path.join(GOLDEN, name + ".jpg")
        s, coefs = _dequantised(oracle, open(path, "rb").read())
        n = s.ncomp
        got = dm.expected(coefs, list(s.subx[:n]), list(s.suby[:n]), s.width, s.height, s.precision, False, k, upsample_=False)
        maxval = (1 << s.precision) - 1
        for c in range(n):
            ref = d["%s__%d" % (name, c)].astype(np.float64)
            gh, gw = ref.shape[0] // k, ref.shape[1] // k
            grp = ref[:gh * k, :gw * k].reshape(gh, k, gw, k)
            ok = ~((grp == 0) | (grp == maxval)).any(axis=(1, 3))
            diff = np.abs(got[c][:gh, :gw].astype(np.float64) - grp.mean(axis=(1, 3)))[ok]
            groups += diff.size
            worst = max(worst, diff.max(initial=0.0))
    assert groups > 1000 // k
    assert worst <= MAX_PLANE_ERROR[k], worst
