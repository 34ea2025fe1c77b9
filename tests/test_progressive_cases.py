"""GPU: the progressive cases (tests/progressive_cases.py) through both decode paths -- the component-fused kernels and, under
B200JPG_NO_PFUSE, the scan-by-scan kernels. Each frame alone must take the path its case names (the fused path launches fewer
kernels); every frame, alone and in one tolerant batch next to sequential, golden and truncated progressive frames, must have
its dequantised coefficients equal to the model's (tests/progressive_model.py: quantisers latched at each component's first
scan), its pixels equal to the reference decoder's (tests/golden/progressive_cases/reference.json) and leave the bytes outside
its slot alone. A frame with a coefficient beyond int16 is MALFORMED_STREAM (DESIGN.md section 7) although the reference
decodes it; the frames around it stay exact."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import entropy_cases as ec
from tests import progressive_cases as pc
from tests import progressive_model as pm

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = json.load(open(os.path.join(GOLDEN, "progressive_cases", "reference.json")))
SENTINEL = 0x5A
PATHS = [({}, "default"), ({"B200JPG_NO_PFUSE": "1"}, "no_pfuse")]


def gpu_decode(built, frames):
    import torch
    dec = built.BatchDecoder(frames, tolerate_bad=True)
    out = dec.new_output()
    out.fill_(SENTINEL)
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return dec, out


def expected_status(name):
    if name in pc.REFUSED:
        return pc.REFUSED[name]
    return 0 if pm.fits_int16(pc.case(name)[0]) else -1038


def check_case(dec, out, i, name):
    frame, data = pc.case(name)
    want = expected_status(name)
    assert dec.status(i) == want, (name, dec.status(i), want)
    assert FIXTURES[name]["rc"] == 0, name  # the reference decodes every case, those the GPU refuses included
    if want != 0:
        return
    for c, deq in enumerate(pm.dequantised(frame)):
        got = dec.coefficients(i, c).astype(np.int64).reshape(deq.shape)
        bad = np.argwhere(got != deq)
        assert len(bad) == 0, "%s component %d: %d coefficients differ, first at %s: %d != %d" % (
            name, c, len(bad), tuple(bad[0]), got[tuple(bad[0])], deq[tuple(bad[0])])
    px = dec.frame_view(out, i).cpu().numpy()
    if frame.precision > 8:
        px = px.view(np.uint16)
    px = np.ascontiguousarray(px.reshape(FIXTURES[name]["shape"]))
    assert hashlib.sha256(px.tobytes()).hexdigest() == FIXTURES[name]["sha256"], name


def check_outside_slots(dec, out, n):
    """every byte outside the frames' slots (those of failed frames included) still holds the sentinel"""
    rest = out.clone()
    for i in range(n):
        rest[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)].fill_(SENTINEL)
    assert bool((rest == SENTINEL).all()), "bytes outside the frames' slots were written"


@pytest.mark.parametrize("name", pc.NAMES)
@pytest.mark.parametrize("env,label", PATHS, ids=[p[1] for p in PATHS])
def test_each_case_alone(built, monkeypatch, env, label, name):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    if name in pc.REFUSED:  # refused when the batch is made: alone, it leaves nothing to decode
        assert built.BatchDecoder([pc.case(name)[1]], tolerate_bad=True).status(0) == pc.REFUSED[name], name
        return
    dec, out = gpu_decode(built, [pc.case(name)[1]])
    check_case(dec, out, 0, name)
    check_outside_slots(dec, out, 1)


def test_fused_cases_launch_fewer_kernels(built, monkeypatch):
    for name in pc.NAMES:
        if pc.path(name) is None:
            continue
        data = pc.case(name)[1]
        fused = gpu_decode(built, [data])[0].launches
        monkeypatch.setenv("B200JPG_NO_PFUSE", "1")
        scan = gpu_decode(built, [data])[0].launches
        monkeypatch.delenv("B200JPG_NO_PFUSE")
        assert (fused < scan) == (pc.path(name) == "fused") and fused <= scan, (name, fused, scan)


@pytest.mark.parametrize("env,label", PATHS, ids=[p[1] for p in PATHS])
def test_all_cases_in_one_batch_with_other_frames(built, oracle, monkeypatch, env, label):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    prog_px = np.load(os.path.join(GOLDEN, "progressive", "progressive_pixels.npz"))
    noeoi_px = np.load(os.path.join(GOLDEN, "noeoi", "noeoi_pixels.npz"))
    others = [("golden", n, os.path.join(GOLDEN, "progressive", n + ".jpg"), prog_px[n]) for n in sorted(prog_px.keys())]
    others.append(("golden", "cut1_p420_96x80", os.path.join(GOLDEN, "noeoi", "cut1_p420_96x80.jpg"), noeoi_px["cut1_p420_96x80"]))
    frames, order = [], []
    for i, name in enumerate(pc.NAMES):
        frames.append(pc.case(name)[1])
        order.append(("case", name, None))
        if i % 5 == 0 and others:
            kind, n, path, px = others.pop()
            frames.append(open(path, "rb").read())
            order.append((kind, n, px))
        if i % 7 == 3:
            frames.append(ec.case("long_420")[1])
            order.append(("sequential", "long_420", None))
    dec, out = gpu_decode(built, frames)
    for i, (kind, name, px) in enumerate(order):
        if kind == "case":
            check_case(dec, out, i, name)
        elif kind == "golden":
            got = dec.frame_view(out, i).cpu().numpy()
            assert dec.status(i) == 0 and np.array_equal(got.reshape(px.shape), px), name
        else:
            rc, want = oracle.decode(frames[i])
            got = dec.frame_view(out, i).cpu().numpy()
            assert rc == 0 and dec.status(i) == 0 and np.array_equal(got.reshape(want.shape), want), name
    check_outside_slots(dec, out, len(frames))
