"""The range argument of reconstruct420_kernel's 16-bit luma tile (recon_sm100.cu, tile_rows16), checked with the integer IDCT
model of tests/recon_cases.py: where the row pass of int16 coefficients can reach, that leaving out the level shift and
rounding the column pass with 2048 + (2048 << 12) gives the same samples, and that row-pass outputs inside int16 keep the
column-pass outputs inside int16."""
import numpy as np

from tests import recon_cases as rc

KROUND16 = 2048 + (2048 << 12)   # kRound16
LO, HI = -3916800, 3916757       # the row-pass bound written at tile_rows16


def _row16(v):
    """idct8t<16, 5> on raw int16 coefficients (no level shift), exact"""
    return (rc._pass(np.asarray(v, dtype=np.int64)) + 16) >> 5


def _extreme_rows():
    """per output n: the coefficient rows that give it its largest and its smallest value"""
    w = rc.row_weights()
    hi = np.where(w < 0, -32768, 32767)
    lo = np.where(w < 0, 32767, -32768)
    return hi, lo


def test_weight_sums():
    w = np.abs(rc.row_weights())
    assert (w.sum(axis=1) == 3825).all()
    neg = np.where(rc.row_weights() < 0, -rc.row_weights(), 0).sum(axis=1)
    assert neg.max() == 2434 and int(np.argmax(neg)) == 1


def test_worst_case_row_pass_is_where_the_code_says():
    hi, lo = _extreme_rows()
    top = np.array([_row16(hi[n])[n] for n in range(8)])
    bottom = np.array([_row16(lo[n])[n] for n in range(8)])
    assert top.max() == HI and bottom.min() == LO
    # and nothing beats the sign patterns: random rows and rows of the extreme values stay inside
    rng = np.random.default_rng(5)
    v = rng.integers(-32768, 32768, (20000, 8))
    v[:5000] = np.where(rng.random((5000, 8)) < 0.5, -32768, 32767)
    out = _row16(v)
    assert out.max() <= HI and out.min() >= LO
    assert HI > 32767 * 119 and -LO > 32768 * 119  # far outside int16: the kernel must check


def test_level_shift_moves_to_the_column_rounding():
    """(S + 16384 * 32 + 16) >> 5 == ((S + 16) >> 5) + 16384 for row 0, and the column pass with kRound16 on the centred rows
    equals the reference's column pass with 2048 on the shifted ones: the same samples as oracle.idct"""
    rng = np.random.default_rng(11)
    deq = rng.integers(-600, 601, (400, 64))
    deq[:, 0] = rng.integers(-1024, 1017, 400)
    deq[:100, 0] = 1016                          # flat 255 and beyond
    want = rc.idct(deq, 128, wrap=False)
    rows = _row16(deq.reshape(-1, 8, 8))        # centred, int16 if in range
    cols = (rc._pass(np.swapaxes(rows, 1, 2)) + KROUND16) >> 12
    assert np.array_equal(np.swapaxes(cols, 1, 2), want)
    shifted = rows.copy()
    shifted[:, 0, :] += 16384
    assert np.array_equal(shifted, rc.row_pass_sums(deq, 128) >> 9)


def test_flat_white_block_sits_well_inside_int16():
    blk = np.zeros(64, dtype=np.int64)
    blk[0] = 1016                                # (255 - 128) * 8
    assert _row16(blk.reshape(8, 8))[0, 0] == 16256  # 32640 with the level shift


def test_column_pass_of_int16_rows_fits_int16():
    """rows in [-32768, 32767] -> |out - 2048| <= 30600: the luma of the int16 tile never reaches the 64-bit colour range"""
    hi, lo = _extreme_rows()
    for n in range(8):
        for v in (hi[n], lo[n]):
            col = (rc._pass(v.astype(np.int64)) + KROUND16) >> 12
            assert -30600 + 2048 <= col[n] <= 30600 + 2048
            assert -32768 <= col.min() and col.max() <= 32767
