"""CPU: the test stream writer (tests/streamwriter.py) and its case catalogue (tests/entropy_cases.py) pinned on the oracle, the
cases checked for the properties they exist for, and the decoder tables of b200jpg_build_tables checked entry by entry against
a plain restatement of canonical code assignment (T.81 Annex C)."""
import numpy as np
import pytest

from tests import entropy_cases as ec
from tests import streamwriter as sw

TABLE_HEADER_BYTES = 16 + 16 + 4 * 160 * 2 * 4  # magic..flags, lut_off[8], qz[4][160][2] (internal.hpp)
L1 = 11                                          # first-level index bits (internal.hpp kLutL1Bits)
BLOCK_ENDS = 96                                  # zig-zag step of symbols that end the block (kQzBlockEnds)
UNUSED = 0x80000000 | (BLOCK_ENDS << 19) | (31 << 5)


def test_writer_refuses_illegal_tables():
    with pytest.raises(ValueError, match="Kraft|all-ones"):  # an over-full code passes the all-ones word first
        sw.HuffTable([3] + [0] * 15, [0, 1, 2])          # three codes of length 1
    with pytest.raises(ValueError, match="all-ones"):
        sw.HuffTable([2] + [0] * 15, [0, 1])             # '0' and '1': the second is all ones
    with pytest.raises(ValueError, match="all-ones"):
        sw.table_from_lengths({c: 1 + min(c, 15) for c in range(17)})  # lengths 1..15 and two of 16: the last is 1111111111111111
    with pytest.raises(ValueError):
        sw.HuffTable([1] + [0] * 15, [0, 1])             # BITS and HUFFVAL disagree
    with pytest.raises(ValueError):
        sw.HuffTable([2] + [0] * 15, [5, 5])
    t = sw.table_from_lengths({n - 1: n for n in range(1, 17)})  # every length once: legal, the last code is 1111111111111110
    assert t.codes[15] == (0xFFFE, 16) and t.codes[0] == (0, 1)
    frame = ec.degenerate_1bit()
    frame.components[0].coef[0, 0, 0, 1] = 1             # a coefficient the EOB-only table cannot code
    with pytest.raises(ValueError, match="not in the table"):
        sw.encode(frame)


def test_huffman_lengths_from_counts_are_limited_and_canonical():
    counts = {s: 2 ** min(s, 40) for s in range(60)}     # skewed enough that plain Huffman lengths exceed 16
    t = sw.table_from_counts(counts)
    lengths = {s: n for s, (c, n) in t.codes.items()}
    assert max(lengths.values()) == 16 and sum(2.0 ** -n for n in lengths.values()) < 1
    assert all(lengths[a] >= lengths[b] for a in counts for b in counts if counts[a] < counts[b])


@pytest.mark.parametrize("name", ec.NAMES)
def test_oracle_reads_back_what_the_writer_wrote(oracle, name):
    frame, data = ec.case(name)
    rc, s, planes = oracle.coefficients(data)
    assert rc == 0
    assert s.precision == frame.precision and s.ncomp == len(frame.components) and s.frame_type == (2 if frame.progressive else s.frame_type)
    for c, want in enumerate(ec.quantised(frame)):
        assert np.array_equal(planes[c], want), "component %d" % c
        q = np.array(s.quant[s.tq[c]], dtype=np.int64).reshape(8, 8)
        assert np.array_equal(q, np.asarray(frame.quant[frame.components[c].tq]).reshape(8, 8))


def _lut_words(built, data, scan):
    blob = _tables(built, data, scan)
    return int(np.frombuffer(blob[8:12].tobytes(), dtype=np.uint32)[0])


def _tables(built, data, scan):
    from libjpeg_b200 import native
    n = native.lib.b200jpg_build_tables(data, len(data), scan, None, 0)
    assert n > 0, native.last_error()
    blob = np.zeros(n, dtype=np.uint8)
    native.lib.b200jpg_build_tables(data, len(data), scan, blob.ctypes.data, n)
    return blob


def test_cases_reach_what_they_are_for(built):
    # decoder tables beyond shared memory: entropy_decode_kernel<kLutShared = false>, with restart markers and restart-less
    for name in ("big_lut_420_rst", "big_lut_4c_norst"):
        assert _lut_words(built, ec.case(name)[1], 0) > ec.SHARED_LUT_WORDS, name
    # restart-less scans long enough for unstuff_long_kernel + spec_sync_kernel + the indexed decoder (specsync.hpp kSpecMinBytes)
    for name in ("big_lut_4c_norst", "dense_12bit", "stuffing_norst"):
        info = built.parse(ec.case(name)[1])
        assert info.restart_interval == 0 and info.ecs_bytes >= 4096, name
    # dense blocks: more than the 64-byte ring per block, symbols of 26..31 bits at every bit of a 32-bit word
    f8, _ = ec.case("dense_8bit")
    f12, _ = ec.case("dense_12bit")
    assert min(f8.stats["intervals"][0]) > 64  # one block per restart interval
    long_syms = [(b, n) for f in (f8, f12) for b, n in f.stats["symbols"][0] if n >= 26]
    assert {26, 31} <= {n for _, n in long_syms} and len({n for _, n in long_syms}) >= 4
    assert {b % 32 for b, _ in long_syms} == set(range(32))
    assert len({b % 128 for b, _ in long_syms}) > 120   # positions inside the 16-byte chunks of the ring
    # stuffing: mostly FF 00, interval lengths over all residues mod 4 and on both sides of multiples of 16 and 128, a stuffed FF
    # right in front of a restart marker and in front of EOI
    f, data = ec.case("stuffing_rst")
    ecs = data[data.rfind(b"\xff\xda"):]
    assert ecs.count(b"\xff\x00") * 2 > 0.7 * len(ecs)
    lens = f.stats["intervals"][0]
    assert {n % 4 for n in lens} == {0, 1, 2, 3}
    assert {n % 16 for n in lens} >= {15, 0, 1} and any(120 <= n < 128 for n in lens) and any(128 < n <= 136 for n in lens)
    assert any(ecs.find(bytes([0xFF, 0x00, 0xFF, 0xD0 + i])) >= 0 for i in range(8))
    assert data.endswith(b"\xff\x00\xff\xd9")
    # int16 edge: dequantised values exactly at both ends of int16, and one beyond
    for name, lo, hi in (("int16_edge", -32768, 32767), ("int16_over", -32768, 32768)):
        deq = ec.dequantised(ec.case(name)[0])[0]
        assert deq.min() == lo and deq.max() == hi, name
        assert (deq == 32767).sum() >= 2 and (deq == -32768).sum() >= 2 and (deq == -32767).sum() >= 1
    # EOBRUN 32767: EOB14 on a 16-bit code followed by fourteen value bits
    f, _ = ec.case("prog_eobrun_max")
    assert f.scans[1].tables[("ac", 0)].codes[0xE0][1] == 16 and (16 + 14) in {n for _, n in f.stats["symbols"][1]}
    # six distinct AC tables of one component: pf_ac_kernel's shared memory (progfused_sm100.cu launch_pf_ac) near its 227 KB
    f, data = ec.case("prog_big_6scans")
    luts = [_lut_words(built, data, s) for s in range(1, 7)]
    smem = 256 * 144 + 6 * 4 * 256 * 4 + 2 * 6 * 4 + sum((128 + w) * 4 for w in luts)
    assert len(set(luts)) >= 1 and 200 * 1024 < smem <= 227 * 1024, smem
    # the whole catalogue stays in 32-bit IDCT arithmetic (the pixels test the decoders, not wrap-around)
    for name in ec.NAMES:
        fr, _ = ec.case(name)
        for c, deq in enumerate(ec.dequantised(fr)):
            assert ec.idct_peak(deq.reshape(-1, 64), 128 if fr.precision == 8 else 2048) < 2 ** 31, (name, c)


def _expected_entry(sym, length, is_ac, progressive):
    """The decoder-table entry of one code (internal.hpp): [4:0] value bits s, [9:5] code length, sequential [25:19] step of
    the zig-zag index, progressive [13:10] run, [30:26] length + s, [31] decoding it is an error."""
    if is_ac:
        s, r = sym & 15, sym >> 4
        bad = int(s == 0 and r not in (0, 15) and not progressive)
        step = BLOCK_ENDS if bad else (r + 1 if s else (16 if r == 15 else BLOCK_ENDS))
    else:
        bad = int(sym > 15)
        s, r, step = (0 if bad else sym), 0, 0
    if progressive:
        return (bad << 31) | ((length + s) << 26) | (r << 10) | (length << 5) | s
    return (bad << 31) | ((length + s) << 26) | (step << 19) | (length << 5) | s


@pytest.mark.parametrize("name", ec.NAMES)
def test_decoder_tables_follow_canonical_codes(built, name):
    """Every code of every table a scan uses, at both lookup levels: length, value bits, zig-zag step (run), total, error bit;
    every code the table does not assign is marked unused; the LUT holds exactly the first- and second-level tables needed."""
    frame, data = ec.case(name)
    current = dict(frame.tables)
    for si, scan in enumerate(frame.scans):
        current.update(scan.tables)
        blob = _tables(built, data, si)
        lut_off = np.frombuffer(blob[16:32].tobytes(), dtype=np.uint16)
        lut = np.frombuffer(blob[TABLE_HEADER_BYTES:].tobytes(), dtype=np.uint32)
        words = int(np.frombuffer(blob[8:12].tobytes(), dtype=np.uint32)[0])
        need_dc = not frame.progressive or (scan.ss == 0 and scan.ah == 0)
        need_ac = not frame.progressive or scan.se != 0
        ns = len(scan.comps)
        used = {("dc", t) for t in (scan.td or [0] * ns)} if need_dc else set()
        used |= {("ac", t) for t in (scan.ta or [0] * ns)} if need_ac else set()
        expect_words = 0
        for kind, slot in sorted(used):
            table = current[(kind, slot)]
            base = int(lut_off[slot + (4 if kind == "ac" else 0)])
            assert base != 0xFFFF, (si, kind, slot)
            first = lut[base:base + (1 << L1)]
            seen1 = np.zeros(1 << L1, dtype=bool)
            subs = {}
            for sym, (code, length) in table.codes.items():
                e = _expected_entry(sym, length, kind == "ac", frame.progressive)
                if length <= L1:
                    lo, hi = code << (L1 - length), (code + 1) << (L1 - length)
                    assert (first[lo:hi] == e).all(), (si, kind, slot, hex(sym))
                    seen1[lo:hi] = True
                else:
                    for c16 in range(code << (16 - length), (code + 1) << (16 - length)):
                        q = c16 >> (16 - L1)
                        ptr = int(first[q])
                        assert ptr & ~(0xFF << 10) == 0, (si, kind, slot, hex(sym))  # length field 0: pointer, nothing else
                        subs.setdefault(ptr >> 10, set()).add(c16 & 31)
                        seen1[q] = True
                        got = lut[base + (1 << L1) + ((ptr >> 10) << (16 - L1)) + (c16 & 31)]
                        assert got == e, (si, kind, slot, hex(sym), c16)
            assert (first[~seen1] == UNUSED).all(), (si, kind, slot)
            assert sorted(subs) == list(range(len(subs)))
            for sub, filled in subs.items():
                rest = [i for i in range(32) if i not in filled]
                assert (lut[base + (1 << L1) + 32 * sub + np.array(rest, dtype=np.int64)] == UNUSED).all() if rest else True
            expect_words += (1 << L1) + 32 * len(subs)
        assert words == expect_words, (si, words, expect_words)
