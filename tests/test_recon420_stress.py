"""GPU: the hand-built reconstruction cases (tests/recon420_cases.py) through the CUDA path: the seams of reconstruct420_kernel's
chroma window, its row-6/7 skip, the int16 edge of the window, 64-bit colour reached only through a neighbour's halo, and the
`wide` flag of b1 + b2. Coefficients must equal what the writer coded, pixels the oracle's."""
import glob
import os

import numpy as np
import pytest

from tests import oracle_binding
from tests import recon420_cases as rc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SUB420 = [n for n in rc.NAMES if rc.subsampling(rc.case(n)[0]) == (2, 2)]
NARROW = [n for n in rc.NAMES if rc.meta(n).narrow]
TWINNED = [n for n in rc.NAMES if rc.meta(n).twin]


def gpu_decode(built, frames, **kw):
    import torch
    dec = built.BatchDecoder(frames, **kw)
    out = dec.new_output()
    out.fill_(0x5A)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return dec, out


def check(dec, out, i, name, oracle):
    f, data = rc.case(name)
    assert dec.status(i) == 0, (name, dec.status(i))
    for c, comp in enumerate(f.components):
        got = dec.coefficients(i, c).astype(np.int64)
        assert np.array_equal(got, comp.coef * np.asarray(f.quant[comp.tq]).reshape(8, 8)), (name, c)
    _, want = oracle.decode(data)
    got = dec.frame_view(out, i).cpu().numpy().reshape(want.shape)
    bad = np.argwhere(np.any(got != want, axis=2))
    assert len(bad) == 0, "%s: %d pixels differ, first at (y, x) = %s" % (name, len(bad), tuple(bad[0]))


@pytest.mark.parametrize("name", rc.NAMES)
def test_case_alone(built, oracle, name):
    dec, out = gpu_decode(built, [rc.case(name)[1]])
    check(dec, out, 0, name, oracle)


def test_all_cases_in_one_batch_next_to_golden_frames(built, oracle):
    """One launch per group, its grid sized by the largest frame: the small frames' CTAs beyond their size exit early."""
    px = np.load(os.path.join(GOLDEN, "golden_pixels.npz"))
    golden = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "c420*.jpg")))
    frames, order = [], []
    for i, name in enumerate(rc.NAMES):
        frames.append(rc.case(name)[1])
        order.append(("case", name))
        if i < len(golden):
            frames.append(open(os.path.join(GOLDEN, golden[i] + ".jpg"), "rb").read())
            order.append(("golden", golden[i]))
    dec, out = gpu_decode(built, frames)
    for i, (kind, name) in enumerate(order):
        if kind == "case":
            check(dec, out, i, name, oracle)
        else:
            assert dec.status(i) == 0 and np.array_equal(dec.frame_view(out, i).cpu().numpy(), px[name]), name


def test_narrow_frames_of_different_sizes_interleaved_with_ordinary_ones(built, oracle):
    """More `narrow` frames than the int32 instance has frame slots (kWideSlots = 4), of four sizes, each between two ordinary
    frames: every slot walks the list over frames of different sizes."""
    from libjpeg_b200 import synth
    extra = [oracle_binding.with_dc_quantiser(synth.encode(synth.source_image(w, h, 5), 75, (2, 2), z), 255)
             for w, h, z in [(96, 80, 3), (320, 176, 20)]]
    hot = [rc.case(n)[1] for n in NARROW if n in SUB420] + extra
    assert len(hot) >= 6
    ordinary = [rc.case(n)[1] for n in ("seam_cols", "sweep_513x65", "wide_right_twin", "skip_rule")]
    frames = []
    for i, h in enumerate(hot):
        frames += [ordinary[i % len(ordinary)], h]
    frames.append(ordinary[0])
    dec, out = gpu_decode(built, frames)
    for i, data in enumerate(frames):
        ret, want = oracle.decode(data)
        assert ret == 0 and dec.status(i) == 0, i
        assert np.array_equal(dec.frame_view(out, i).cpu().numpy().reshape(want.shape), want), i


def test_cases_without_colour_transform(built, oracle):
    frames = [rc.case(n)[1] for n in rc.NAMES]
    dec, out = gpu_decode(built, frames, color_transform=False)
    for i, name in enumerate(rc.NAMES):
        ret, want = oracle.decode_without_color_transform(frames[i])
        assert ret == 0 and dec.status(i) == 0, name
        assert np.array_equal(dec.frame_view(out, i).cpu().numpy().reshape(want.shape), want), name


def test_twins_agree_outside_the_extreme_blocks_reach(built):
    """A frame and its twin without the extreme block take different instances and colour modes, yet every pixel the extreme
    block cannot reach (recon420_cases.reach) comes out the same."""
    frames = [rc.case(n)[1] for n in TWINNED]
    dec, out = gpu_decode(built, frames)
    for i, name in enumerate(TWINNED):
        j = TWINNED.index(rc.meta(name).twin)
        a, b = dec.frame_view(out, i).cpu().numpy(), dec.frame_view(out, j).cpu().numpy()
        y0, y1, x0, x1 = rc.reach(rc.case(name)[0], *rc.meta(name).extreme)
        outside = np.ones(a.shape[:2], dtype=bool)
        outside[y0:y1, x0:x1] = False
        assert dec.status(i) == 0 and np.array_equal(a[outside], b[outside]), name
