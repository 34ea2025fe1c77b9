"""GPU: hand-built streams at the edges of the Huffman decoders (tests/entropy_cases.py) through the CUDA path. Every frame's
dequantised coefficients must equal what the writer coded times the quantiser, its pixels the oracle's and its status the
oracle's verdict -- except the one frame whose coefficient +32768 leaves the int16 store, which the GPU reports as
MALFORMED_STREAM (DESIGN.md section 7) while the frames around it stay exact. The same cases run again through the host restart
index, the single-work-item path for restart-less scans and the scan-by-scan progressive kernels."""
import glob
import os

import numpy as np
import pytest

from tests import entropy_cases as ec

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEQUENTIAL = [n for n in ec.NAMES if not ec.case(n)[0].progressive]
PROGRESSIVE = [n for n in ec.NAMES if ec.case(n)[0].progressive]


def gpu_decode(built, frames):
    import torch
    dec = built.BatchDecoder(frames, tolerate_bad=True)
    out = dec.new_output()
    out.fill_(0x5A)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return dec, out


def check(dec, out, i, name, oracle):
    frame, data = ec.case(name)
    if name in ec.BEYOND_INT16:
        assert oracle.decode(data)[0] == 0, name  # the reference decodes it: the documented deviation
        assert dec.status(i) == -1038, (name, dec.status(i))
        return
    assert dec.status(i) == 0, (name, dec.status(i))
    for c, want in enumerate(ec.dequantised(frame)):
        got = dec.coefficients(i, c).astype(np.int64)
        assert got.shape == want.shape, (name, c)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, "%s component %d: %d coefficients differ, first at %s: %d != %d" % (
            name, c, len(bad), tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])
    rc, want = (oracle.decode16 if frame.precision > 8 else oracle.decode)(data)
    assert rc == 0, name
    got = dec.frame_view(out, i).cpu().numpy()
    if frame.precision > 8:
        got = got.view(np.uint16)
    assert np.array_equal(got.reshape(want.shape), want), "%s: %d samples differ" % (name, int((got.reshape(want.shape) != want).sum()))


@pytest.mark.parametrize("name", ec.NAMES)
def test_case_decodes_to_the_written_coefficients(built, oracle, name):
    dec, out = gpu_decode(built, [ec.case(name)[1]])
    check(dec, out, 0, name, oracle)


def test_all_cases_in_one_batch_next_to_golden_frames(built, oracle):
    golden = sorted(glob.glob(os.path.join(GOLDEN, "c4*.jpg")))[:4]
    px = np.load(os.path.join(GOLDEN, "golden_pixels.npz"))
    frames, order = [], []
    for i, name in enumerate(ec.NAMES):
        frames.append(ec.case(name)[1])
        order.append(("case", name))
        if i % 4 == 0 and golden:
            g = golden.pop()
            frames.append(open(g, "rb").read())
            order.append(("golden", os.path.basename(g)[:-4]))
    dec, out = gpu_decode(built, frames)
    for i, (kind, name) in enumerate(order):
        if kind == "case":
            check(dec, out, i, name, oracle)
        else:
            assert dec.status(i) == 0 and np.array_equal(dec.frame_view(out, i).cpu().numpy(), px[name]), name


@pytest.mark.parametrize("env,names", [({"B200JPG_HOST_INDEX": "1", "B200JPG_NO_SPEC": "1"}, SEQUENTIAL),
                                       ({"B200JPG_NO_PFUSE": "1"}, PROGRESSIVE)], ids=["host_index_no_spec", "no_pfuse"])
def test_cases_through_the_other_paths(built, oracle, monkeypatch, env, names):
    assert names
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dec, out = gpu_decode(built, [ec.case(n)[1] for n in names])
    for i, name in enumerate(names):
        check(dec, out, i, name, oracle)
