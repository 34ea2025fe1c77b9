"""Host replay of the synchronisation rounds of restart-less scans (specsync.hpp, spec_sync_host_replay) on the hand-built
scans of tests/spec_cases.py. The work items are held against what the writer recorded -- where every block starts and the
DC coefficients in front of it -- not against another walk of the decoder; the rounds against each case's docstring."""
import ctypes
import re

import numpy as np
import pytest

from tests import spec_cases as sc


def replay(built, data):
    from libjpeg_b200 import native
    a = np.frombuffer(data, dtype=np.uint8)
    n, rounds = ctypes.c_uint32(), ctypes.c_uint32()
    rc = native.lib.b200jpg_selftest_restartless_items(a.ctypes.data, a.size, None, 0, ctypes.byref(n), ctypes.byref(rounds))
    assert rc != 0 and n.value >= 1  # nothing to write into: refused, with the count
    items = np.zeros((max(n.value, 1), 7), dtype=np.int32)
    rc = native.lib.b200jpg_selftest_restartless_items(a.ctypes.data, a.size, items.ctypes.data, items.shape[0], ctypes.byref(n), ctypes.byref(rounds))
    assert rc == 0
    return items[:n.value], rounds.value


@pytest.mark.parametrize("name", sc.NAMES)
def test_work_items_match_the_writer(built, name):
    frame, data = sc.case(name)
    items, _ = replay(built, data)
    starts, pred = sc.truth(frame, data if name in sc.CUT else None)
    total = len(sc._units(frame))
    ns = len(frame.scans[0].comps)
    covered = 0
    for bit, first, n, *p in items:
        if n == 0:
            continue
        assert first == covered, (name, "work items must tile the blocks in order")
        if first < len(starts):
            assert bit == starts[first], (name, first, bit, starts[first])
            assert list(p[:ns]) == list(pred[first, :ns]), (name, first, p[:ns], pred[first, :ns])
        covered += n
    assert covered == total, name
    if name not in sc.CUT:
        assert len(starts) == total
    assert len(items) == -(-frame.stats["intervals"][0][0] * 8 // sc.SEQ_BITS) if name not in sc.CUT else len(items) >= 1


@pytest.mark.parametrize("name", sc.NAMES)
def test_rounds_match_the_docstring(built, name):
    _, data = sc.case(name)
    _, rounds = replay(built, data)
    assert rounds == sc.rounds(name), (name, rounds)
    if name in sc.PERIODIC:
        assert rounds <= 12, "self-synchronisation should take a handful of rounds, not one per subsequence"


def test_near_identical_tables_keep_the_rounds_and_the_merge_log_busy(built, capfd, monkeypatch):
    """Paths that stay out of step for thousands of bits: several rounds, later walks that end on logged paths at more than
    one of the seven marks (SpecLog), and no more of the stream walked than those rounds need."""
    monkeypatch.setenv("B200JPG_SPEC_STATS", "1")
    _, data = sc.case("near_identical_420")
    capfd.readouterr()
    _, rounds = replay(built, data)
    line = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("restart-less replay")][-1]
    merges = [int(v) for v in re.search(r"merges at marks((?: \d+)+)", line).group(1).split()]
    assert rounds >= 4 and int(re.search(r"(\d+) rounds", line).group(1)) == rounds
    assert len(merges) == 7 and sum(1 for m in merges if m) >= 2, line
    # a walk whose entry did not change is skipped: re-walking them all every round would take this past 6x the stream
    assert float(re.search(r"([\d.]+) x the stream walked", line).group(1)) < 5.0, line


@pytest.mark.parametrize("w,h,sub", [(1920, 1080, (2, 2)), (1280, 720, (1, 1))])
def test_shared_table_synth_frames_take_a_handful_of_rounds(built, w, h, sub):
    """Frames of the synthetic encoder with every component on table 0 (the reference encoder's layout without colour
    transformation): the replay's work items tile the scan (b200jpg_selftest_restartless) in at most 12 rounds."""
    from libjpeg_b200 import native, synth
    data = np.frombuffer(synth.encode(synth.source_image(w, h, 11), 80, sub, 0, synth.SHARED_TABLES).tobytes(), dtype=np.uint8)
    rounds, nseg = ctypes.c_uint32(), ctypes.c_uint32()
    assert native.lib.b200jpg_selftest_restartless(data.ctypes.data, data.size, ctypes.byref(rounds), ctypes.byref(nseg)) == 0
    assert nseg.value > 100 and 1 <= rounds.value <= 12
