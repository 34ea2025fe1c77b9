"""GPU: a 4:2:0 frame whose luma row pass leaves int16 (and nothing else does) in a batch of ordinary frames. reconstruct420_kernel
keeps the luma row pass in a 16-bit tile; such a frame must be flagged `narrow` and redone by the int32 instance, bit-exact,
and the frames around it must come out as they would alone. The CPU half shows that the block's 16-bit row pass would wrap and
change the pixels, so exact pixels mean the frame took the exact path."""
import numpy as np
import pytest

from tests import recon420_cases as rc
from tests import recon_cases as rcc
from tests import streamwriter as sw

W, H = 512, 96
AT = (5, 7)  # luma block (row, column): CTA (1, 0), warp 1, lane 7


def _block():
    """row 0: DC 2000 and coefficient 1 at 100 -> row-pass output 0 = (512 * 2000 + 710 * 100 + 16) >> 5 = 34219"""
    b = np.zeros((8, 8), dtype=np.int32)
    b[0, 0], b[0, 1] = 2000, 100
    return b


def _frame(seed, luma_wrap):
    _, (y, cb, cr) = rc.base(W, H, seed)
    if luma_wrap:
        y[AT] = _block()
    return sw.encode(rc.frame(W, H, [y, cb, cr]))


def test_block_wraps_a_16_bit_row_pass():
    """CPU: centred row outputs beyond int16, and the wrapped 16-bit tile would give other samples"""
    b = _block().astype(np.int64)
    rows = (rcc._pass(b) + 16) >> 5
    assert rows.max() == 34219
    wrapped = ((rows + 32768) % 65536) - 32768
    col = lambda r: np.swapaxes((rcc._pass(np.swapaxes(r, 0, 1)) + 2048 + (2048 << 12)) >> 12, 0, 1)
    exact = rcc.idct(b.reshape(1, 64), 128, wrap=False)[0]
    assert np.array_equal(col(rows), exact)
    assert not np.array_equal(col(wrapped), exact)
    assert np.abs(exact).max() < 65535  # no 64-bit colour: only the 16-bit tile is in question


@pytest.mark.gpu
def test_luma_row_pass_beyond_int16_is_redone_exactly(built, oracle):
    import torch
    frames = [_frame(s, luma_wrap=(i % 3 == 1)) for i, s in enumerate(range(401, 410))]
    dec = built.BatchDecoder(frames)
    out = dec.new_output()
    out.fill_(0x5A)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    for i, data in enumerate(frames):
        assert dec.status(i) == 0, i
        rc_, want = oracle.decode(data)
        assert rc_ == 0
        got = dec.frame_view(out, i).cpu().numpy().reshape(want.shape)
        bad = np.argwhere(np.any(got != want, axis=2))
        assert len(bad) == 0, "frame %d: %d pixels differ, first at %s" % (i, len(bad), tuple(bad[0]))
    # the flagged frames' neighbours alone give the same bytes
    for i in (0, 2, 3):
        alone = built.BatchDecoder([frames[i]])
        o = alone.new_output()
        alone.upload()
        alone.decode(o)
        torch.cuda.synchronize()
        assert np.array_equal(alone.frame_view(o, 0).cpu().numpy(), dec.frame_view(out, i).cpu().numpy()), i
