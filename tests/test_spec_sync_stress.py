"""GPU: the hand-built restart-less scans of tests/spec_cases.py through spec_sync_kernel and the indexed entropy decoder.
Every frame's dequantised coefficients must equal what the writer coded times the quantiser (where the stream is whole), its
pixels the oracle's and its status the oracle's verdict: alone, in one batch next to golden and restart-interval frames,
through the single-work-item path, in a batch large enough for the 3-CTAs-per-SM instance of spec_sync_kernel, and on 1080p
and 4K frames whose components all share Huffman table 0."""
import glob
import os

import numpy as np
import pytest

from tests import entropy_cases as ec
from tests import spec_cases as sc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RESTART_CASES = ["long_420", "big_lut_420_rst", "run_edges"]


def gpu_decode(built, frames):
    import torch
    dec = built.BatchDecoder(frames, tolerate_bad=True)
    out = dec.new_output()
    out.fill_(0x5A)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return dec, out


def check(dec, out, i, frame, data, oracle, name, coefficients=True):
    rc, want = (oracle.decode16 if frame is not None and frame.precision > 8 else oracle.decode)(data)
    assert dec.status(i) == rc, (name, dec.status(i), rc)
    if coefficients and frame is not None:
        for c, ref in enumerate(sc.dequantised(frame)):
            got = dec.coefficients(i, c).astype(np.int64)
            bad = np.argwhere(got != ref)
            assert len(bad) == 0, "%s component %d: %d coefficients differ, first at %s" % (name, c, len(bad), tuple(bad[0]))
    if rc == 0:
        got = dec.frame_view(out, i).cpu().numpy()
        if frame is not None and frame.precision > 8:
            got = got.view(np.uint16)
        assert np.array_equal(got.reshape(want.shape), want), "%s: %d samples differ" % (name, int((got.reshape(want.shape) != want).sum()))


def check_case(dec, out, i, name, oracle):
    frame, data = sc.case(name)
    check(dec, out, i, frame, data, oracle, name, coefficients=name not in sc.CUT)


@pytest.mark.parametrize("name", sc.NAMES)
def test_case_alone(built, oracle, name):
    dec, out = gpu_decode(built, [sc.case(name)[1]])
    assert dec.info(0).n_intervals == 1
    check_case(dec, out, 0, name, oracle)


def _mixed():
    golden = sorted(glob.glob(os.path.join(GOLDEN, "c4*.jpg")))[:4]
    rst = list(RESTART_CASES)
    order = []
    for i, name in enumerate(sc.NAMES):
        order.append(("spec", name))
        if i % 4 == 0 and golden:
            order.append(("golden", golden.pop()))
        if i % 4 == 2 and rst:
            order.append(("rst", rst.pop()))
    return order


def _data(kind, name):
    if kind == "spec":
        return sc.case(name)[1]
    if kind == "rst":
        return ec.case(name)[1]
    return open(name, "rb").read()


@pytest.mark.parametrize("no_spec", [False, True], ids=["spec_sync", "no_spec"])
def test_all_cases_in_one_batch_next_to_golden_and_restart_frames(built, oracle, monkeypatch, no_spec):
    if no_spec:
        monkeypatch.setenv("B200JPG_NO_SPEC", "1")
    order = _mixed()
    assert {k for k, _ in order} == {"spec", "golden", "rst"}
    dec, out = gpu_decode(built, [_data(k, n) for k, n in order])
    px = np.load(os.path.join(GOLDEN, "golden_pixels.npz"))
    for i, (kind, name) in enumerate(order):
        if kind == "spec":
            check_case(dec, out, i, name, oracle)
        elif kind == "rst":
            frame, data = ec.case(name)
            check(dec, out, i, frame, data, oracle, name)
        else:
            key = os.path.basename(name)[:-4]
            assert dec.status(i) == 0 and np.array_equal(dec.frame_view(out, i).cpu().numpy(), px[key]), key


def test_batch_for_three_ctas_per_sm(built, oracle):
    """At least 2 x multi_processor_count restart-less scans of one scan class (the launch unit: same tables, same sampling)
    in one batch: launch_spec_sync picks spec_sync_kernel<3>, the 40-register instance, for them. Between them, near-identical,
    periodic and ordinary frames."""
    import torch
    from libjpeg_b200 import synth
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ordinary = synth.encode(synth.source_image(320, 240, 5), 80, (2, 2), 0).tobytes()
    kinds = [("uniform_420", sc.case("uniform_420")[1]), ("near_identical_420", sc.case("near_identical_420")[1]),
             ("periodic_abab", sc.case("periodic_abab")[1]), ("synth", ordinary)]
    frames = [kinds[0] if i % 5 else kinds[(i // 5) % 3 + 1] for i in range(2 * sms * 5 // 4 + 8)]
    dec, out = gpu_decode(built, [d for _, d in frames])
    assert sum(1 for name, _ in frames if name == "uniform_420") >= 2 * sms
    assert all(dec.info(i).n_intervals == 1 and dec.info(i).restart_interval == 0 for i in range(len(frames)))
    assert all(len(d) >= 4096 for _, d in frames)
    first = {}
    for i, (name, data) in enumerate(frames):
        first.setdefault(name, i)
    for name, i in first.items():
        if name == "synth":
            check(dec, out, i, None, frames[i][1], oracle, name)
        else:
            check_case(dec, out, i, name, oracle)
    wants = {name: oracle.decode(data)[1] for name, data in kinds}
    for i, (name, _) in enumerate(frames):
        assert dec.status(i) == 0 and np.array_equal(dec.frame_view(out, i).cpu().numpy().reshape(wants[name].shape), wants[name]), (i, name)


@pytest.mark.parametrize("w,h,sub", [(1920, 1080, (2, 2)), (3840, 2160, (2, 2)), (1920, 1080, (1, 1))])
def test_shared_table_synth_frames_match_oracle(built, oracle, w, h, sub):
    """1080p and 4K frames with every component on Huffman table 0, alone and two in a batch with an ordinary frame."""
    from libjpeg_b200 import synth
    shared = synth.encode(synth.source_image(w, h, 13), 85, sub, 0, synth.SHARED_TABLES).tobytes()
    ordinary = synth.encode(synth.source_image(w, h, 14), 85, sub, 0).tobytes()
    for frames in ([shared], [shared, ordinary, shared]):
        dec, out = gpu_decode(built, frames)
        for i, data in enumerate(frames):
            check(dec, out, i, None, data, oracle, "%dx%d frame %d" % (w, h, i))
