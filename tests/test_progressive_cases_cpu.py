"""CPU: the progressive cases (tests/progressive_cases.py) pinned on what the reference decoder made of them
(tests/golden/progressive_cases/reference.json). The writer reproduces every stream the fixtures were taken from; the reference's
pixels are the C oracle's reconstruction of the model's levels (tests/progressive_model.py) under the "component's first scan"
quantiser rule, and under no other rule where the rules differ; the C oracle's own decode matches every fixture."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from tests import progressive_cases as pc
from tests import progressive_model as pm

FIXTURES = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "progressive_cases", "reference.json")))
DECODED = [n for n in pc.NAMES if FIXTURES[n]["rc"] == 0]
REDEFINED = {"dqt_redefined_fused", "dqt_redefined_scan"}


def _digest(px):
    return hashlib.sha256(np.ascontiguousarray(px).tobytes()).hexdigest()


def reconstruct(oracle, data, planes, quantisers):
    """the oracle's reconstruction of the given quantised levels, dequantised with the given per-component tables (component c
    through slot c)"""
    rc, s = oracle.info(data)
    assert rc == 0
    for c, q in enumerate(quantisers):
        s.tq[c] = c
        s.quant_defined[c] = 1
        for i in range(64):
            s.quant[c][i] = int(q[i])
    planes = [np.ascontiguousarray(p, dtype=np.int32) for p in planes]
    ptrs = (ctypes.c_void_p * 4)(*[p.ctypes.data for p in planes] + [None] * (4 - len(planes)))
    wide = s.precision > 8
    out = np.zeros((s.height, s.width, s.ncomp), dtype=np.uint16 if wide else np.uint8)
    fn = oracle.lib.jpgo_reconstruct16 if wide else oracle.lib.jpgo_reconstruct
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.POINTER(type(s)), ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]
    assert fn(ctypes.byref(s), ptrs, out.ctypes.data) == 0
    return out


def test_fixtures_cover_every_case():
    assert sorted(FIXTURES) == sorted(pc.NAMES)


@pytest.mark.parametrize("name", pc.NAMES)
def test_writer_reproduces_the_fixture_stream(name):
    assert hashlib.sha256(pc.case(name)[1]).hexdigest() == FIXTURES[name]["input_sha256"]


@pytest.mark.parametrize("name", DECODED)
def test_reference_follows_the_component_first_scan_rule(oracle, name):
    frame, data = pc.case(name)
    lv = pm.levels(frame)
    matches = {rule for rule in pm.RULES if _digest(reconstruct(oracle, data, lv, pm.quantisers(frame, rule))) == FIXTURES[name]["sha256"]}
    # exactly the rules that give this frame the same tables as the component's first scan
    want = pm.quantisers(frame, "component_first")
    same = {rule for rule in pm.RULES if all(np.array_equal(x, y) for x, y in zip(pm.quantisers(frame, rule), want))}
    assert matches == same, (name, matches)


def test_redefined_cases_tell_the_rules_apart():
    qs = {name: {rule: pm.quantisers(pc.case(name)[0], rule) for rule in pm.RULES} for name in REDEFINED}
    differ = lambda x, y: any(not np.array_equal(a, b) for a, b in zip(x, y))  # noqa: E731
    assert differ(qs["dqt_redefined_fused"]["component_first"], qs["dqt_redefined_fused"]["last"])
    for a in pm.RULES:  # every rule gives the non-interleaved frame other tables
        for b in pm.RULES:
            assert a == b or differ(qs["dqt_redefined_scan"][a], qs["dqt_redefined_scan"][b]), (a, b)
    frame, _ = pc.case("dqt_redefined_scan")  # one slot, two components, two latched tables
    q = pm.quantisers(frame, "component_first")
    assert frame.components[1].tq == frame.components[2].tq and not np.array_equal(q[1], q[2])


def test_int16_edges_sit_where_they_claim():
    for name in pc.NAMES:
        if not name.startswith("i16_"):
            continue
        deq = np.concatenate([d.reshape(-1) for d in pm.dequantised(pc.case(name)[0])])
        if name.endswith("_edge"):
            assert pm.fits_int16(pc.case(name)[0]) and (deq.max() == 32767 or deq.min() == -32768), name
        else:
            assert not pm.fits_int16(pc.case(name)[0]), name
    frame, _ = pc.case("i16_product_over")  # level x (q << Al) = 2^32: an int32 product is 0
    assert (int(np.abs(pm.dequantised(frame)[0]).max()) & 0xFFFFFFFF) == 0


@pytest.mark.parametrize("name", pc.NAMES)
def test_oracle_decode_matches_the_reference(oracle, name):
    frame, data = pc.case(name)
    rc, px = (oracle.decode16 if frame.precision > 8 else oracle.decode)(data)
    assert rc == FIXTURES[name]["rc"], name
    if rc == 0:
        assert _digest(px) == FIXTURES[name]["sha256"], name
