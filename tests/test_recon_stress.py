"""GPU: the hand-built cases of tests/recon_cases.py through the CUDA path: reconstruct_kernel's tile seams, its `fast` and
per-lane chroma loads, the 4:2:2 neighbour columns and the 4:4:0 rolling lines, the int16 edge of its planes and the exact pass
over more `narrow` frames than it has slots, the generic kernels' layouts, and the IDCT at its 32-bit limits. Coefficients must
equal what the writer coded, samples the oracle's."""
import glob
import os

import numpy as np
import pytest

from tests import downscale_model as dm
from tests import oracle_binding
from tests import recon_cases as rc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NARROW_TILED = [n for n in rc.NAMES if rc.meta(n).narrow and rc.path(rc.case(n)[0]) == "Tiled"]
ORDINARY_TILED = [n for n in rc.NAMES if n.startswith("sweep_") or n.startswith("seam_")]


def gpu_decode(built, frames, **kw):
    import torch
    dec = built.BatchDecoder(frames, **kw)
    out = dec.new_output()
    out.fill_(0x5A)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return dec, out


def _samples(dec, out, i):
    fi = dec.info(i)
    a = dec.frame_view(out, i).cpu().numpy()
    return a.view(np.uint16) if fi.precision > 8 else a


def _want(oracle, data):
    ret, s = oracle.info(data)
    ret, px = oracle.decode16(data) if s.precision > 8 else oracle.decode(data)
    assert ret == 0
    return px


def check(dec, out, i, name, oracle):
    f, data = rc.case(name)
    assert dec.status(i) == 0, (name, dec.status(i))
    for c, comp in enumerate(f.components):
        got = dec.coefficients(i, c).astype(np.int64)
        assert np.array_equal(got, comp.coef), (name, c)
    want = _want(oracle, data)
    got = _samples(dec, out, i).reshape(want.shape)
    bad = np.argwhere(np.any(got != want, axis=2))
    assert len(bad) == 0, "%s: %d pixels differ, first at (y, x) = %s" % (name, len(bad), tuple(bad[0]))


@pytest.mark.parametrize("name", rc.NAMES)
def test_case_alone(built, oracle, name):
    dec, out = gpu_decode(built, [rc.case(name)[1]])
    check(dec, out, 0, name, oracle)


def test_all_cases_in_one_batch_next_to_golden_frames(built, oracle):
    """One launch per group, its grid sized by the largest frame of the group, the cases of every layout between golden frames"""
    golden = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg"))) + sorted(glob.glob(os.path.join(GOLDEN, "subsampling", "*.jpg")))
    frames, order = [], []
    for i, name in enumerate(rc.NAMES):
        frames.append(rc.case(name)[1])
        order.append(name)
        if i < len(golden):
            frames.append(open(golden[i], "rb").read())
            order.append(None)
    dec, out = gpu_decode(built, frames)
    for i, name in enumerate(order):
        if name is not None:
            check(dec, out, i, name, oracle)
        else:
            assert dec.status(i) == 0 and np.array_equal(_samples(dec, out, i), _want(oracle, frames[i])), i


def test_blocks_no_scan_codes_read_as_zeros_in_a_reused_store(built, oracle):
    """Frames coded in one scan per component (an MCU of more than 10 blocks): each scan codes its component's own block grid,
    and the blocks of the MCU-padded grid beyond it must read as zeros, also when the batch's coefficient store comes from the
    context's pool with the coefficients of an earlier batch in it."""
    from libjpeg_b200.decoder import Context
    ctx = Context()
    dec, out = gpu_decode(built, [rc.case(n)[1] for n in rc.NAMES], ctx=ctx)
    assert all(dec.status(i) == 0 for i in range(len(rc.NAMES)))
    del dec, out
    names = [n for n in rc.NAMES if len(rc.case(n)[0].scans) > 1]
    assert names
    for n in names:  # the padded grid is wider or taller than what the scans code
        f = rc.case(n)[0]
        own = rc.sw.geometry(f)[4]
        assert any(c.coef.shape[1] > bw or c.coef.shape[0] > bh for c, (bw, bh) in zip(f.components, own)), n
    dec, out = gpu_decode(built, [rc.case(n)[1] for n in names], ctx=ctx)
    for i, name in enumerate(names):
        check(dec, out, i, name, oracle)


def _narrow_batch():
    """Every `narrow` Tiled case (more than kWideSlots = 4 per layout) plus beyond-range frames of other sizes, each between two
    ordinary frames of the layouts"""
    from libjpeg_b200 import synth
    extra = [oracle_binding.with_dc_quantiser(synth.encode(synth.source_image(w, h, 5), 75, sub, z), 255)
             for w, h, sub, z in [(96, 80, (1, 1), 3), (320, 176, (2, 1), 20), (200, 72, (1, 2), 0), (33, 300, (1, 1), 2)]]
    hot = [rc.case(n)[1] for n in NARROW_TILED] + extra
    ordinary = [rc.case(n)[1] for n in ORDINARY_TILED]
    frames = []
    for i, h in enumerate(hot):
        frames += [ordinary[i % len(ordinary)], h]
    return frames + [ordinary[0]]


def _check_all(oracle, dec, out, frames):
    for i, data in enumerate(frames):
        want = _want(oracle, data)
        assert dec.status(i) == 0, i
        assert np.array_equal(_samples(dec, out, i).reshape(want.shape), want), i


@pytest.mark.parametrize("chunk", [None, 1, 3])
def test_narrow_frames_of_different_sizes_interleaved_with_ordinary_ones(built, oracle, monkeypatch, chunk):
    """More `narrow` frames per Tiled layout than the exact pass has frame slots, of several sizes, each between two ordinary
    frames; B200JPG_RECON_CHUNK = 1 / 3 runs b1 + b2 of the int16 pass a chunk of frames at a time"""
    if chunk is not None:
        monkeypatch.setenv("B200JPG_RECON_CHUNK", str(chunk))
    assert len(NARROW_TILED) > 3 * 4
    frames = _narrow_batch()
    dec, out = gpu_decode(built, frames)
    _check_all(oracle, dec, out, frames)


def test_cases_without_colour_transform(built, oracle):
    frames = [rc.case(n)[1] for n in rc.NAMES if rc.case(n)[0].precision == 8]
    dec, out = gpu_decode(built, frames, color_transform=False)
    for i, data in enumerate(frames):
        ret, want = oracle.decode_without_color_transform(data)
        assert ret == 0 and dec.status(i) == 0, i
        assert np.array_equal(dec.frame_view(out, i).cpu().numpy().reshape(want.shape), want), i


def test_cases_without_upsampling(built, oracle):
    """upsample=False: every component as its own plane, against downscale_model.planes_out on the oracle's IDCT planes"""
    frames = [rc.case(n)[1] for n in rc.NAMES]
    dec, out = gpu_decode(built, frames, upsample=False)
    for i, name in enumerate(rc.NAMES):
        f = rc.case(name)[0]
        subx, suby = rc.subsampling(f)
        want = dm.planes_out([dm.full_planes(oracle, c.coef, f.precision) for c in f.components], subx, suby, f.width, f.height,
                             f.precision)
        assert dec.status(i) == 0, name
        for c, p in enumerate(dec.plane_views(out, i)):
            got = p.cpu().numpy()
            got = got.view(np.uint16) if f.precision > 8 else got
            assert np.array_equal(got, want[c]), (name, c)


def test_twins_agree_outside_the_extreme_blocks_reach(built):
    twinned = [n for n in rc.NAMES if rc.meta(n).twin]
    frames = [rc.case(n)[1] for n in twinned]
    dec, out = gpu_decode(built, frames)
    for i, name in enumerate(twinned):
        j = twinned.index(rc.meta(name).twin)
        a, b = _samples(dec, out, i), _samples(dec, out, j)
        y0, y1, x0, x1 = rc.reach(rc.case(name)[0], *rc.meta(name).extreme)
        outside = np.ones(a.shape[:2], dtype=bool)
        outside[y0:y1, x0:x1] = False
        assert dec.status(i) == 0 and np.array_equal(a[outside], b[outside]), name
