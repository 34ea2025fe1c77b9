"""CPU: the hand-built reconstruction cases (tests/recon420_cases.py) have the property each exists for, and the plain 64-bit
model of the upsampling and colour stage gives the oracle's pixels."""
import numpy as np
import pytest

from tests import recon420_cases as rc
from tests.streamwriter import Component, Frame

SENSE = [n for n in rc.NAMES if rc.meta(n).sense]
WIDE = [n for n in rc.NAMES if rc.meta(n).wrap_px]
TWINNED = [n for n in rc.NAMES if rc.meta(n).twin]
SYNTHETIC_420 = [(641, 479, 13, 75), (1000, 300, 0, 30)]


def frame_of(oracle, data):
    """The oracle's reading of a sequential 8-bit stream as a Frame the model takes."""
    ret, s, planes = oracle.coefficients(data)
    assert ret == 0
    comps = [Component(planes[c], s.hs[c], s.vs[c], s.tq[c]) for c in range(s.ncomp)]
    return Frame(s.width, s.height, comps, {c.tq: np.array(s.quant[c.tq], dtype=np.int64) for c in comps}, [])


def _bytes_in(px, rects):
    return np.concatenate([px[y0:y1, x0:x1].ravel() for y0, y1, x0, x1 in rects])


@pytest.mark.parametrize("name", rc.NAMES)
def test_model_matches_oracle(oracle, name):
    f, data = rc.case(name)
    ret, want = oracle.decode(data)
    assert ret == 0
    assert np.array_equal(rc.model(oracle, f), want), name
    ret, want = oracle.decode_without_color_transform(data)
    assert ret == 0 and np.array_equal(rc.model(oracle, f, color_transform=False), want), name


@pytest.mark.parametrize("w,h,z,q", SYNTHETIC_420)
def test_model_matches_oracle_on_synthetic_frames(oracle, built, w, h, z, q):
    from libjpeg_b200 import synth
    data = synth.encode(synth.source_image(w, h, 9), q, (2, 2), z).tobytes()
    ret, want = oracle.decode(data)
    assert ret == 0
    assert np.array_equal(rc.model(oracle, frame_of(oracle, data)), want)


@pytest.mark.parametrize("name", rc.NAMES)
def test_oracle_reads_the_written_coefficients(oracle, name):
    f, data = rc.case(name)
    ret, _, planes = oracle.coefficients(data)
    assert ret == 0
    for c, comp in enumerate(f.components):
        assert np.array_equal(planes[c], comp.coef), (name, c)


@pytest.mark.parametrize("name", ["seam_cols", "seam_rows", "seam_corners"])
def test_seam_blocks_are_dense_and_carry_the_targeted_terms(name):
    """Every block a seam case targets has all 64 coefficients non-zero, with large terms in the coefficients the case zeroes."""
    f, _ = rc.case(name)
    for c, by, bx, mask in rc.meta(name).sense:
        blk = f.components[c].coef[by, bx]
        assert np.all(blk != 0), (name, c, by, bx)
        if name != "seam_corners":
            assert np.abs(blk[mask]).max() >= 300, (name, c, by, bx)


def test_skip_rule_warps_hold_one_high_coefficient():
    """In every warp of skip_rule (one chroma block row of one CTA: 16 Cb + 16 Cr blocks) coefficient rows 6 and 7 are zero,
    except for the one placed coefficient of the warps that have one; the placements cover rows 6 and 7, columns 0 and 7 and
    lanes 0, 15, 16, 31, plus the first and last blocks of a right-edge warp with 5 blocks per component."""
    f, _ = rc.case("skip_rule")
    cb, cr = f.components[1].coef, f.components[2].coef
    bh, bw = cb.shape[:2]
    placed = {(by, bx // rc.CTA_CBX): (c, bx % rc.CTA_CBX, row, col) for c, by, bx, mask in rc.meta("skip_rule").sense
              for row, col in [tuple(np.argwhere(mask)[0])]}
    for by in range(bh):
        for k in range(-(-bw // rc.CTA_CBX)):
            cols = slice(rc.CTA_CBX * k, min(rc.CTA_CBX * (k + 1), bw))
            high = [(c, j, r, col) for c, comp in ((1, cb), (2, cr)) for j, r, col in np.argwhere(comp[by, cols, 6:, :] != 0)]
            want = placed.get((by, k))
            assert [(c, j, r + 6, col) for c, j, r, col in high] == ([want] if want else []), (by, k)
    lanes = {(c - 1) * 16 + j for c, j, _, _ in placed.values() if j in (0, 15)}
    assert lanes == {0, 15, 16, 31}
    assert {(r, col) for _, _, r, col in placed.values()} == {(6, 0), (6, 7), (7, 0), (7, 7)}
    assert bw % rc.CTA_CBX == 5 and {(c, j) for (by, k), (c, j, _, _) in placed.items() if k == bw // rc.CTA_CBX} == {(1, 0), (1, 4), (2, 0), (2, 4)}


@pytest.mark.parametrize("name", SENSE)
def test_zeroing_the_targeted_coefficients_changes_the_targeted_pixels(oracle, name):
    """The coefficients a case targets reach the pixels through the code it targets: without them the oracle's pixels change in
    the stated pixel columns / rows, in at least the stated number of bytes, and in every stated rectangle."""
    f, data = rc.case(name)
    m = rc.meta(name)
    ret, px = oracle.decode(data)
    ret0, px0 = oracle.decode(rc.with_zeroed(f, m.sense))
    assert ret == 0 and ret0 == 0
    changed = int((_bytes_in(px, m.sense_px) != _bytes_in(px0, m.sense_px)).sum())
    assert changed >= m.sense_min, (name, changed)
    for rect in m.sense_px:
        assert (_bytes_in(px, [rect]) != _bytes_in(px0, [rect])).any(), (name, rect)


@pytest.mark.parametrize("name", [n for n in rc.NAMES if rc.meta(n).unsat_px])
def test_targeted_pixels_are_mostly_unsaturated(oracle, name):
    _, px = oracle.decode(rc.case(name)[1])
    v = _bytes_in(px, rc.meta(name).unsat_px)
    assert np.mean((v == 0) | (v == 255)) < 0.25, name


@pytest.mark.parametrize("name", rc.NAMES)
def test_chroma_range_is_what_the_case_says(oracle, name):
    """Narrow edges hit their exact extreme in their extreme block; `narrow` frames leave int16 and no other case does."""
    f, _ = rc.case(name)
    m = rc.meta(name)
    sx, sy = rc.subsampling(f)
    cw, ch = -(-f.width // sx), -(-f.height // sy)
    planes = [p[:ch, :cw] for p in rc.sample_planes(oracle, f)[1:]]
    hi, lo = max(int(p.max()) for p in planes), min(int(p.min()) for p in planes)
    assert (hi > 32767 or lo < -32768) == m.narrow, (name, lo, hi)
    if m.peak is not None:
        assert (hi if m.peak > 0 else lo) == m.peak, (name, lo, hi)
        c, by, bx = m.extreme
        blk = planes[c - 1][8 * by:8 * by + 8, 8 * bx:8 * bx + 8]
        assert np.array_equal(np.argwhere(blk == m.peak)[:, 1], np.zeros(8)), name


def test_edge_coefficients_give_the_exact_extremes(oracle):
    one = np.ones(64, dtype=np.uint16)
    for target, (dc, a) in rc.EDGE.items():
        blk = np.zeros(64, dtype=np.int32)
        blk[0], blk[1] = dc, a
        s = oracle.idct(blk, one)
        assert (s.max() if target > 0 else s.min()) == target
        assert set(np.argwhere(s == target)[:, 1]) == {0}


@pytest.mark.parametrize("name", WIDE)
def test_32bit_colour_differs_from_the_oracle_in_the_targeted_pixels(oracle, name):
    """The wide cases need 64-bit colour where they say: wrapping 32-bit sums give other pixels there; in the twin they do not."""
    f, data = rc.case(name)
    _, want = oracle.decode(data)
    got = rc.model(oracle, f, int32_colour=True)
    rects = rc.meta(name).wrap_px
    assert (_bytes_in(got, rects) != _bytes_in(want, rects)).any(), name
    tf, tdata = rc.case(rc.meta(name).twin)
    assert np.array_equal(rc.model(oracle, tf, int32_colour=True), oracle.decode(tdata)[1]), name


@pytest.mark.parametrize("name", TWINNED)
def test_twins_differ_only_inside_the_extreme_blocks_reach(oracle, name):
    f, data = rc.case(name)
    m = rc.meta(name)
    tf, tdata = rc.case(m.twin)
    assert rc.meta(m.twin).twin == name and m.extreme == rc.meta(m.twin).extreme
    for c, comp in enumerate(f.components):
        diff = np.argwhere(np.any(comp.coef != tf.components[c].coef, axis=(2, 3)))
        assert [tuple(d) for d in diff] == ([m.extreme[1:]] if c == m.extreme[0] else []), (name, c)
    a, b = oracle.decode(data)[1], oracle.decode(tdata)[1]
    y0, y1, x0, x1 = rc.reach(f, *m.extreme)
    outside = np.ones(a.shape[:2], dtype=bool)
    outside[y0:y1, x0:x1] = False
    assert np.array_equal(a[outside], b[outside]), name
