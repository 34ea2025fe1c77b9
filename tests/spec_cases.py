"""Hand-built restart-less scans for the synchronisation rounds of spec_sync_kernel (specsync.hpp); tests/streamwriter.py
writes them, seeded and deterministic.

Every block's DC coefficient follows from its index in coding order (a ramp that wraps inside the category range), so a
work item that starts with the wrong block, the wrong position in the MCU or the wrong predictor changes coefficients even
where the AC data repeats. The writer records where every block starts (frame.stats["blocks"]): truth(frame) turns that
and the coefficients into the start bit and the DC predictors of every block, independent of the decoder.

Each case's docstring names what it targets and ends with the rounds the host replay takes on it ("Host replay: N rounds").

case(name) -> (Frame, codestream bytes)."""
import functools
import re

import numpy as np

from tests import entropy_cases as ec
from tests import streamwriter as sw
from tests.streamwriter import Component, Frame, Scan

SEQ_BITS = 8192          # specsync.hpp kSpecSeqBits
AC_SYMS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]


def _ac_counts(bias):
    """Weights of a typical AC table: EOB first, short runs and small sizes next; `bias` tilts them so that two tables
    built from it differ."""
    counts = {0x00: 4000, 0xF0: 12}
    for r in range(16):
        for s in range(1, 11):
            counts[(r << 4) | s] = int(3000 * (0.62 + 0.05 * bias) ** r * (0.55 - 0.04 * bias) ** (s - 1)) + 1
    return counts


def _dc_counts(top=11):
    return {c: int(600 * 0.7 ** abs(c - 4)) + 1 for c in range(top + 1)}


def tables(bias=0, floor=0):
    """(DC table, AC table) of the Annex K.2 construction from typical symbol weights (`floor` added to every AC weight
    shortens the longest codes)."""
    return sw.table_from_counts(_dc_counts()), sw.table_from_counts({s: c + floor for s, c in _ac_counts(bias).items()})


def near_twin(ac, rare):
    """The AC table `ac` plus symbol `rare` on a 16-bit code behind every other code: every symbol of `ac` keeps its code,
    and the new code lies in the code space that `ac` leaves free, so `ac` cannot decode it."""
    lengths = {s: n for s, (_, n) in ac.codes.items()}
    assert rare not in lengths and max(lengths.values()) <= 15
    twin = sw.table_from_lengths({**lengths, rare: 16})
    assert all(twin.codes[s] == ac.codes[s] for s in ac.codes)
    return twin


def ramp(n, precision=8):
    """The DC coefficient of the block with coding-order index n: wraps inside categories 0..9 (0..13 at 12 bits)."""
    span = 401 if precision == 8 else 6001
    return (n * 37) % span - span // 2


def _components(rng, factors, w, h, density, max_size):
    hmax, vmax = max(f[0] for f in factors), max(f[1] for f in factors)
    mcx, mcy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    return [Component(ec.sparse(rng, mcy * v, mcx * hh, density=density, max_size=max_size), hh, v, min(c, 1))
            for c, (hh, v) in enumerate(factors)]


def _units(frame):
    """[(component, block row, block column)] of the scan in coding order."""
    return [(frame.scans[0].comps[k], by, bx) for unit in sw._scan_units(frame, frame.scans[0]) for (k, by, bx) in unit]


def set_ramp(frame):
    for n, (c, by, bx) in enumerate(_units(frame)):
        frame.components[c].coef[by, bx, 0, 0] = ramp(n, frame.precision)
    return frame


def _frame(factors, w, h, slots, tabs, seed, density=0.12, max_size=7, precision=8):
    """A restart-less interleaved frame of the given sampling factors; scan component c on DC / AC slot slots[c]."""
    rng = np.random.default_rng(seed)
    comps = _components(rng, factors, w, h, density, max_size)
    quant = {0: rng.integers(1, 6, 64), 1: rng.integers(1, 6, 64)}
    f = Frame(w, h, comps, quant, [Scan(list(range(len(factors))), list(slots), list(slots))], tabs, precision)
    return set_ramp(f)


def _shared(bias=0):
    dc, ac = tables(bias)
    return {("dc", 0): dc, ("ac", 0): ac}


# ---------------------------------------------------------------------------------------------------------------------
def uniform_444():
    """Three components 4:4:4, all on DC / AC table 0: a block's position in the MCU is knowable modulo 1 only.
    Host replay: 2 rounds."""
    return _frame([(1, 1)] * 3, 256, 256, [0, 0, 0], _shared(), 201)


def uniform_420():
    """4:2:0 (six blocks per MCU) on one table pair. Host replay: 2 rounds."""
    return _frame([(2, 2), (1, 1), (1, 1)], 320, 256, [0, 0, 0], _shared(), 202)


def uniform_4c():
    """Four components 4:4:4 on one table pair. Host replay: 2 rounds."""
    return _frame([(1, 1)] * 4, 224, 224, [0, 0, 0, 0], _shared(), 203)


def uniform_10blk():
    """The largest MCU (kSpecMaxBlocksPerMcu = 10 blocks: factors 2x2, 2x1, 2x2) on one table pair. Host replay: 2 rounds."""
    return _frame([(2, 2), (2, 1), (2, 2)], 256, 224, [0, 0, 0], _shared(), 204)


def periodic_abab():
    """Four components 4:4:4 on tables A, B, A, B: positions are knowable modulo 2 only, so a rule that looks for "every
    table equal" does not see it. Host replay: 2 rounds."""
    dca, aca = tables(0)
    dcb, acb = tables(3)
    return _frame([(1, 1)] * 4, 224, 224, [0, 1, 0, 1], {("dc", 0): dca, ("ac", 0): aca, ("dc", 1): dcb, ("ac", 1): acb}, 205)


NEAR_RARE = 0xFA  # run 15, size 10: never in the luma blocks (sizes up to 7), in one chroma block every few subsequences


def near_identical_420():
    """4:2:0, luma on table A, chroma on table B, and B codes every symbol exactly as A does except the rare AC symbol 0xFA,
    which A cannot decode. A path that stands on the right bit with the wrong block position stays in step with the true
    one until the next chroma 0xFA, about 2000 bits later, and only then gets another chance at the right position: many
    paths cross a subsequence boundary out of step, later rounds re-walk them from corrected entries, and those walks end
    where they meet their logged paths, at several marks. Host replay: 20 rounds."""
    dc, a = tables(0, floor=5)
    del a.codes[NEAR_RARE]
    a = sw.table_from_lengths({s: n for s, (_, n) in a.codes.items()})
    b = near_twin(a, NEAR_RARE)
    f = _frame([(2, 2), (1, 1), (1, 1)], 320, 256, [0, 1, 1], {("dc", 0): dc, ("ac", 0): a, ("dc", 1): dc, ("ac", 1): b}, 206)
    units = _units(f)
    chroma = [i for i, (c, _, _) in enumerate(units) if c != 0]
    for n in chroma[12::23]:  # Cb and Cr in turn, about 70 blocks or 2000 bits apart
        c, by, bx = units[n]
        blk = f.components[c].coef[by, bx]
        blk.reshape(64)[sw.ZIGZAG[1:]] = 0
        blk.reshape(64)[sw.ZIGZAG[16]] = 700  # 15 zeros, then a size-10 value: symbol 0xFA
    return f


def _fill(frame, count, blocks):
    """Puts `count` coefficients +1 at zig-zag 1, 2, .. into the given (component, row, column) blocks, at most 62 each
    (every added coefficient costs the same bits: the block keeps its EOB)."""
    for c, by, bx in blocks:
        n = min(count, 62)
        flat = frame.components[c].coef[by, bx].reshape(64)
        flat[sw.ZIGZAG[1:]] = 0
        flat[sw.ZIGZAG[1:n + 1]] = 1
        count -= n
    assert count == 0, "not enough tuning blocks"
    return frame


def _sized(build, tune, want_bits):
    """build() -> frame with its tuning blocks (tune(frame) -> list) empty; fills them until the unstuffed scan ends in the
    byte that holds bit want_bits - 1, i.e. the scan is ceil(want_bits / 8) bytes long."""
    f = build()
    blocks = tune(f)
    _fill(f, 0, blocks)
    sw.encode(f)
    ac = f.tables[("ac", f.scans[0].ta[0])]
    step = ac.codes[0x01][1] + 1
    assert step <= 8
    bits = f.stats["symbols"][0][-1][0] + f.stats["symbols"][0][-1][1]
    floor_bits = 8 * (-(-want_bits // 8) - 1)  # the scan ends in the byte behind this bit
    need = (floor_bits - bits) // step + 1 if bits <= floor_bits else 0
    f = build()
    _fill(f, need, tune(f))
    sw.encode(f)
    assert f.stats["intervals"][0][0] == -(-want_bits // 8), (f.stats["intervals"][0][0], want_bits)
    return f


def _exact(delta):
    def build():
        return _frame([(1, 1)] * 3, 96, 96, [0, 0, 0], _shared(), 207, density=0.1)

    def tune(f):
        return _units(f)[-140:]

    f = build()
    _fill(f, 0, tune(f))
    sw.encode(f)
    k = -(-f.stats["intervals"][0][0] * 8 // SEQ_BITS)
    return _sized(build, tune, 8 * (k * SEQ_BITS // 8 + delta))


def exact_multiple():
    """Unstuffed scan of exactly a whole number of subsequences (8192 bits each), uniform tables: the last subsequence ends
    on the last bit. Host replay: 2 rounds."""
    return _exact(0)


def exact_plus_byte():
    """One byte more than a whole number of subsequences: the last one holds 8 bits. Host replay: 2 rounds."""
    return _exact(1)


def exact_minus_byte():
    """One byte less than a whole number of subsequences. Host replay: 2 rounds."""
    return _exact(-1)


def dense_tail():
    """The last subsequence has no block boundary of its own: it starts inside the final block, which holds 63 AC
    coefficients of size 10 (about 1300 bits). Host replay: 2 rounds."""
    dense = ec._dense(np.random.default_rng(208), 1, 1, 8)[0, 0]

    def build():
        f = _frame([(1, 1)] * 3, 192, 192, [0, 1, 1], {**_shared(), ("dc", 1): tables(2)[0], ("ac", 1): tables(2)[1]}, 208, density=0.1)
        blk = f.components[2].coef[-1, -1]
        blk[:] = np.clip(dense, -1000, 1000)
        blk[0, 0] = ramp(len(_units(f)) - 1)
        return f

    def tune(f):
        return [u for u in _units(f)[-200:-1] if u[0] == 0]

    f = build()
    _fill(f, 0, tune(f))
    sw.encode(f)
    last = f.stats["blocks"][0][-1]
    length = f.stats["intervals"][0][0] * 8 - last
    k = -(-(last + 300) // SEQ_BITS)
    # move the final block's start to 300 bits in front of a subsequence boundary: the boundary falls inside it
    return _sized(build, tune, k * SEQ_BITS - 300 + length)


def _cut(frame_fn, mcus_short, eoi):
    f = frame_fn()
    data = sw.encode(f)
    hmax, vmax, mcx, mcy, _ = sw.geometry(f)
    bpm = sum(c.h * c.v for c in f.components)
    cut_bit = f.stats["blocks"][0][-mcus_short * bpm]
    sos = data.rfind(b"\xff\xda")
    start = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
    # stuffed position of unstuffed byte cut_bit // 8
    at, seen = start, 0
    while seen < cut_bit // 8:
        at += 2 if data[at] == 0xFF else 1
        seen += 1
    return f, data[:at] + (b"\xff\xd9" if eoi else b"")


def cut_uniform_eoi():
    """uniform_444 cut three MCUs before its end, EOI behind the cut: the padding clip and the last_used top-up; the
    decoder reads zero bits behind the data. Host replay: 2 rounds."""
    return _cut(uniform_444, 3, True)


def cut_uniform_noeoi():
    """The same cut without EOI. Host replay: 2 rounds."""
    return _cut(uniform_444, 3, False)


def cut_separate_eoi():
    """near_identical_420 (luma and chroma on separate tables) cut five MCUs before its end, EOI behind the cut.
    Host replay: 20 rounds."""
    return _cut(near_identical_420, 5, True)


def dc31_12bit():
    """12-bit, one table pair for three components: DC differences of category 15 on a 16-bit code (31-bit symbols), one
    in every block, straddling the subsequence boundaries. Host replay: 2 rounds."""
    rng = np.random.default_rng(210)
    comps = _components(rng, [(1, 1)] * 3, 96, 96, 0.08, 9)
    quant = {0: rng.integers(1, 4, 64), 1: rng.integers(1, 4, 64)}
    quant[0][0] = quant[1][0] = 1  # DC coefficients near +-16000 stay inside the int16 coefficient store
    f = Frame(96, 96, comps, quant, [Scan([0, 1, 2], [0, 0, 0], [0, 0, 0])],
              {("dc", 0): sw.table_from_lengths({c: c + 1 for c in range(15)} | {15: 16}), ("ac", 0): tables()[1]}, precision=12, dqt16=True)
    for n, (c, by, bx) in enumerate(_units(f)):
        f.components[c].coef[by, bx, 0, 0] = (16000 if n % 2 == 0 else -16000) + (n * 7) % 300
    for c in f.components:
        ec.fit_idct(c.coef, f.quant[c.tq], 12)
    return f


CASES = {f.__name__: f for f in [uniform_444, uniform_420, uniform_4c, uniform_10blk, periodic_abab, near_identical_420, exact_multiple,
                                 exact_plus_byte, exact_minus_byte, dense_tail, cut_uniform_eoi, cut_uniform_noeoi, cut_separate_eoi,
                                 dc31_12bit]}
NAMES = list(CASES)
CUT = {"cut_uniform_eoi", "cut_uniform_noeoi", "cut_separate_eoi"}
# every position of the MCU on one table pair, or on a repeating pattern of them: one round per subsequence before the
# synchronisation compared block positions modulo the table period
PERIODIC = {"uniform_444", "uniform_420", "uniform_4c", "uniform_10blk", "periodic_abab"}


def rounds(name):
    """The host-replay rounds the case's docstring states."""
    return int(re.search(r"Host replay: (\d+) rounds?", " ".join(CASES[name].__doc__.split())).group(1))


@functools.lru_cache(maxsize=None)
def case(name):
    made = CASES[name]()
    if isinstance(made, tuple):
        return made
    return made, sw.encode(made)


def truth(frame, data=None):
    """(start bit of every block in the unstuffed scan, [blocks, 4] DC predictors in front of it) from what the writer
    recorded and the coefficients. With `data` (a cut stream) only the blocks whose symbols lie wholly in front of the cut."""
    starts = np.asarray(frame.stats["blocks"][0], dtype=np.int64)
    units = _units(frame)
    pred = np.zeros((len(units), 4), dtype=np.int64)
    last = [0, 0, 0, 0]
    comps = frame.scans[0].comps
    for n, (c, by, bx) in enumerate(units):
        pred[n] = last
        last[comps.index(c)] = int(frame.components[c].coef[by, bx, 0, 0])
    if data is not None:
        end_bit = 8 * _unstuffed_len(data)
        whole = np.searchsorted(starts, end_bit, side="right") - 1  # the block the cut falls into is not whole
        starts, pred = starts[:whole], pred[:whole]
    return starts, pred


def _unstuffed_len(data):
    sos = data.rfind(b"\xff\xda")
    at = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
    n = 0
    while at < len(data):
        if data[at] == 0xFF:
            if at + 1 < len(data) and data[at + 1] == 0:
                at += 2
                n += 1
                continue
            break
        at += 1
        n += 1
    return n


def dequantised(frame):
    return ec.dequantised(frame)
