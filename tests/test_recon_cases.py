"""CPU: the hand-built cases of tests/recon_cases.py (Tiled and Generic reconstruction, the IDCT's 32-bit limits) have the
property each exists for, and the 64-bit model of tests/downscale_model.py (full-size IDCT planes, then the reference's
upsampling and colour rules) gives the oracle's samples for every one of them."""
import numpy as np
import pytest

from tests import downscale_model as dm
from tests import recon_cases as rc

SENSE = [n for n in rc.NAMES if rc.meta(n).sense]
WIDE = [n for n in rc.NAMES if rc.meta(n).wrap_px]
TWINNED = [n for n in rc.NAMES if rc.meta(n).twin]
ROWMAX = [n for n in rc.NAMES if rc.meta(n).rowmax]
COLWRAP = [n for n in rc.NAMES if rc.meta(n).colwrap]
CHROMA = [n for n in rc.NAMES if len(rc.case(n)[0].components) == 3]


def planes(oracle, f):
    return [dm.full_planes(oracle, c.coef, f.precision) for c in f.components]


def model(oracle, f, color_transform=True):
    subx, suby = rc.subsampling(f)
    ycbcr = color_transform and len(f.components) == 3
    return dm.reconstruct_samples(planes(oracle, f), subx, suby, f.width, f.height, f.precision, ycbcr)


def decode(oracle, data, precision):
    ret, px = oracle.decode16(data) if precision > 8 else oracle.decode(data)
    assert ret == 0
    return px


def _bytes_in(px, rects):
    return np.concatenate([px[y0:y1, x0:x1].ravel() for y0, y1, x0, x1 in rects])


@pytest.mark.parametrize("name", rc.NAMES)
def test_model_matches_oracle(oracle, name):
    f, data = rc.case(name)
    assert np.array_equal(model(oracle, f), decode(oracle, data, f.precision)), name
    if f.precision == 8:
        ret, want = oracle.decode_without_color_transform(data)
        assert ret == 0 and np.array_equal(model(oracle, f, color_transform=False), want), name


@pytest.mark.parametrize("name", rc.NAMES)
def test_oracle_reads_the_written_coefficients(oracle, name):
    f, data = rc.case(name)
    ret, s, got = oracle.coefficients(data)
    assert ret == 0 and s.precision == f.precision
    for c, comp in enumerate(f.components):
        assert np.array_equal(got[c], comp.coef), (name, c)


def test_cases_cover_every_path_and_layout():
    paths = {}
    for n in rc.NAMES:
        f = rc.case(n)[0]
        paths.setdefault(rc.path(f), set()).add((f.precision, tuple((c.h, c.v) for c in f.components)))
    assert {fac for _, fac in paths["Tiled"]} == {tuple(v) for v in rc.TILED.values()}
    generic = {fac for _, fac in paths["Generic"]}
    assert {tuple(v) for v in rc.GENERIC.values()} <= generic
    assert any(p == 12 for p, _ in paths["Generic"]) and "Fused420" in paths
    assert {rc.path(rc.case(n)[0]) for n in COLWRAP} == {"Fused420", "Tiled", "Generic"}
    assert {rc.case(n)[0].precision for n in COLWRAP} == {8, 12}


@pytest.mark.parametrize("name", SENSE)
def test_zeroing_the_targeted_coefficients_changes_the_targeted_pixels(oracle, name):
    f, data = rc.case(name)
    m = rc.meta(name)
    px, px0 = decode(oracle, data, 8), decode(oracle, rc.with_zeroed(f, m.sense), 8)
    changed = int((_bytes_in(px, m.sense_px) != _bytes_in(px0, m.sense_px)).sum())
    assert changed >= m.sense_min, (name, changed)
    for rect in m.sense_px:
        assert (_bytes_in(px, [rect]) != _bytes_in(px0, [rect])).any(), (name, rect)


@pytest.mark.parametrize("name", ["seam_%s" % k for k in rc.TILED])
def test_seam_blocks_are_dense(name):
    f, _ = rc.case(name)
    for c, by, bx, mask in rc.meta(name).sense:
        blk = f.components[c].coef[by, bx]
        assert np.all(blk != 0), (name, c, by, bx)


@pytest.mark.parametrize("name", [n for n in rc.NAMES if n.startswith("sweep_")])
def test_sweep_geometry(name):
    """Every sweep frame has a partial CTA, and its chroma (grey: luma) grid is padded beyond the visible samples or ends in a
    partial block."""
    f, _ = rc.case(name)
    assert f.width % rc.CTA_W or f.height % rc.CTA_H, name
    subx, suby = rc.subsampling(f)
    c = f.components[-1]
    cw, ch = -(-f.width // subx[-1]), -(-f.height // suby[-1])
    assert 8 * c.coef.shape[1] > cw or 8 * c.coef.shape[0] > ch or cw % 8 or ch % 8, name


@pytest.mark.parametrize("name", CHROMA)
def test_chroma_range_is_what_the_case_says(oracle, name):
    """Edges hit their exact extreme in column 0 of their extreme block; `narrow` frames have a visible chroma sample beyond
    int16 (12 bit, whose planes are level shifted by 32768: beyond +-65535, the 32-bit colour range) and no other frame with
    chroma does."""
    f, _ = rc.case(name)
    m = rc.meta(name)
    subx, suby = rc.subsampling(f)
    ps = planes(oracle, f)
    vis = [ps[c][:-(-f.height // suby[c]), :-(-f.width // subx[c])] for c in (1, 2)]
    hi, lo = max(int(p.max()) for p in vis), min(int(p.min()) for p in vis)
    top, bottom = (32767, -32768) if f.precision == 8 else (65535, -65535)
    assert (hi > top or lo < bottom) == m.narrow, (name, lo, hi)
    if m.peak is not None:
        assert (hi if m.peak > 0 else lo) == m.peak, (name, lo, hi)
        c, by, bx = m.extreme
        blk = ps[c][8 * by:8 * by + 8, 8 * bx:8 * bx + 8]
        assert np.array_equal(np.argwhere(blk == m.peak)[:, 1], np.zeros(8)), name


def test_narrow_frames_outnumber_the_exact_pass_slots():
    """More `narrow` Tiled frames of one layout than the exact pass has frame slots (kWideSlots = 4)"""
    for fmt in ("444", "422", "440"):
        n = [x for x in rc.NAMES if rc.meta(x).narrow and rc.path(rc.case(x)[0]) == "Tiled"
             and tuple((c.h, c.v) for c in rc.case(x)[0].components) == tuple(rc.TILED[fmt])]
        assert len(n) > 4, fmt


def _colour32(oracle, f):
    """8-bit YCbCr -> RGB with the sums wrapped to 32 bits: what 32-bit colour arithmetic gives"""
    subx, suby = rc.subsampling(f)
    ps = planes(oracle, f)
    up = [dm.upsample(ps[c], -(-f.width // subx[c]), -(-f.height // suby[c]), subx[c], suby[c], f.width, f.height) for c in range(3)]
    yv, cb, cr = up[0], up[1] - 2048, up[2] - 2048
    sums = [yv * 8192 + cr * 11485 + 65536, yv * 8192 - cb * 2819 - cr * 5850 + 65536, yv * 8192 + cb * 14516 + 65536]
    return np.clip(np.stack([rc._wrap32(s) >> 17 for s in sums], axis=-1), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("name", WIDE)
def test_32bit_colour_differs_from_the_oracle_in_the_targeted_pixels(oracle, name):
    f, data = rc.case(name)
    want = decode(oracle, data, 8)
    rects = rc.meta(name).wrap_px
    assert (_bytes_in(_colour32(oracle, f), rects) != _bytes_in(want, rects)).any(), name
    tf, tdata = rc.case(rc.meta(name).twin)
    assert np.array_equal(_colour32(oracle, tf), decode(oracle, tdata, 8)), name


@pytest.mark.parametrize("name", TWINNED)
def test_twins_differ_only_inside_the_extreme_blocks_reach(oracle, name):
    f, data = rc.case(name)
    m = rc.meta(name)
    tf, tdata = rc.case(m.twin)
    assert rc.meta(m.twin).twin == name and m.extreme == rc.meta(m.twin).extreme
    for c, comp in enumerate(f.components):
        diff = np.argwhere(np.any(comp.coef != tf.components[c].coef, axis=(2, 3)))
        assert [tuple(d) for d in diff] == ([m.extreme[1:]] if c == m.extreme[0] else []), (name, c)
    a, b = decode(oracle, data, f.precision), decode(oracle, tdata, f.precision)
    y0, y1, x0, x1 = rc.reach(f, *m.extreme)
    outside = np.ones(a.shape[:2], dtype=bool)
    outside[y0:y1, x0:x1] = False
    assert np.array_equal(a[outside], b[outside]), name


def test_python_idct_is_the_oracles(oracle):
    rng = np.random.default_rng(5)
    blocks = [rc.wrapping_block(rng, 128) for _ in range(4)] + [rc.dense(rng, True, True) for _ in range(4)]
    one = np.ones(64, dtype=np.uint16)
    for dco in (128, 2048):
        for b in blocks:
            assert np.array_equal(rc.idct(b.reshape(1, 64), dco)[0], oracle.idct(b.reshape(64), one, dco))


@pytest.mark.parametrize("precision", [8, 12])
def test_row_pass_maximum(oracle, precision):
    """The row-pass maximum over coefficients within +-32767, from the weights of idct8t: every output index reaches the same
    bound, just below 2^31, so the row pass never wraps and the kernels' raw-coefficient row pass (unpack_row_raw) is exact."""
    wts = rc.row_weights()
    assert np.array_equal(rc._pass(np.eye(8, dtype=np.int64)), wts.T)
    assert all(int(np.abs(wts[i]).sum()) == 3825 for i in range(8))
    bounds = [rc.row_max_block(i, precision)[1] for i in range(8)]
    assert max(bounds) == rc.ROW_MAX[precision] < 2 ** 31
    int16 = [bounds[i] + 16 * int(np.abs(wts[i][wts[i] < 0]).sum()) for i in range(8)]
    assert max(int16) == int16[1] == rc.INT16_ROW_MAX[precision] < 2 ** 31
    rng = np.random.default_rng(precision)
    dco = 1 << (precision - 1)
    sums = rc.row_pass_sums(rng.integers(-32767, 32768, (2000, 64)), dco)
    assert np.abs(sums).max() < rc.ROW_MAX[precision]
    for i in range(8):
        blk, bound = rc.row_max_block(i, precision)
        assert rc.row_pass_sums(blk.reshape(1, 64), dco)[0, 0, i] == bound
        assert np.array_equal(oracle.idct(blk.reshape(64), np.ones(64, dtype=np.uint16), dco),
                              rc.idct(blk.reshape(1, 64), dco, wrap=False)[0])


@pytest.mark.parametrize("name", ROWMAX)
def test_rowmax_blocks_reach_the_bound(name):
    f, _ = rc.case(name)
    dco = 1 << (f.precision - 1)
    got = set()
    for c, by, bx, i in rc.meta(name).rowmax:
        v = rc.row_pass_sums(f.components[c].coef[by, bx].reshape(1, 64), dco)[0, 0, i]
        assert v == rc.row_max_block(i, f.precision)[1] == rc.ROW_MAX[f.precision], (name, c, by, bx, i)
        got.add((c, i))
    assert got == {(c, i) for c in (0, 1) for i in range(8)}


@pytest.mark.parametrize("name", COLWRAP)
def test_colwrap_blocks_leave_int32_and_wrap(oracle, name):
    """Every component holds blocks whose column pass leaves int32 (idct_peak >= 2^31): the oracle's samples are the 32-bit
    wrap of the IDCT, not its 64-bit value."""
    f, _ = rc.case(name)
    dco = 1 << (f.precision - 1)
    one = np.ones(64, dtype=np.uint16)
    for c in f.components:
        blocks = c.coef.reshape(-1, 64)
        peaks = [rc.ec.idct_peak(b[None], dco) for b in blocks]
        assert max(peaks) >= 2 ** 31, name
        assert np.abs(rc.row_pass_sums(blocks, dco)).max() < 2 ** 31
        wrapped = [k for k, p in enumerate(peaks) if p >= 2 ** 31]
        assert any(not np.array_equal(oracle.idct(blocks[k], one, dco), rc.idct(blocks[k][None], dco, wrap=False)[0])
                   for k in wrapped), name
