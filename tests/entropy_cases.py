"""Hand-built streams at the edges of the Huffman decoders (tests/streamwriter.py writes them; seeded, deterministic):
long codes that make the second lookup level the common case, decoder tables too large for shared memory, degenerate tables,
dense blocks of 26- to 31-bit symbols, run-length edges, streams that are mostly FF 00, restart geometries, dequantised
values at the int16 edge and progressive extremes (EOBRUN 32767, six AC scans on distinct large tables).

case(name) -> (Frame, codestream bytes); every frame's coefficients are what oracle.coefficients() must return."""
import functools

import numpy as np

from tests import streamwriter as sw
from tests.streamwriter import Component, Frame, Scan

# symbol sets: every symbol a scan of that kind may need
SEQ_AC = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]
PROG_AC_FIRST = [n << 4 for n in range(15)] + [0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 15)]
PROG_REFINE = [n << 4 for n in range(15)] + [0xF0] + [(r << 4) | 1 for r in range(16)]
DC_ALL = list(range(16))

# entropy_decode_kernel keeps its tables in shared memory up to this many LUT words (huffman_sm100.cu launch_entropy_impl:
# 768 threads x (144 + 64) bytes + 4 x 160 quantiser words next to the LUT must stay within 227 KB)
SHARED_LUT_WORDS = (227 * 1024 - 768 * (144 + 64) - 4 * 160 * 4) // 4


def long_table(syms, rng, lo=12, hi=16, force=None):
    """Every symbol on a code of lo..hi bits (force: {symbol: length} overrides)."""
    lengths = {s: int(rng.integers(lo, hi + 1)) for s in syms}
    lengths.update(force or {})
    return sw.table_from_lengths(lengths)


def wide_table(syms, shift=0):
    """Every symbol on a 12-bit code, one on 13: about one second-level table per two symbols (the most a table can have).
    `shift` picks which symbol gets the 13-bit code, so tables of the same symbols differ."""
    lengths = {s: 12 for s in syms}
    lengths[syms[shift % len(syms)]] = 13
    return sw.table_from_lengths(lengths)


def all_lengths_dc():
    """16 DC categories on codes of lengths 1..16: category 0, the most frequent, on the 16-bit one."""
    return sw.table_from_lengths({c: 16 - c for c in range(16)})


def _set(coef, by, bx, k, v):
    coef[by, bx].reshape(64)[sw.ZIGZAG[k]] = v


def sparse(rng, bh, bw, density=0.25, max_size=7, dc=200):
    coef = np.zeros((bh, bw, 8, 8), dtype=np.int32)
    flat = coef.reshape(bh, bw, 64)
    flat[..., 0] = rng.integers(-dc, dc + 1, size=(bh, bw))
    mask = rng.random((bh, bw, 63)) < density
    size = rng.integers(1, max_size + 1, size=(bh, bw, 63))
    mag = (1 << (size - 1)) + rng.integers(0, 1 << 30, size=size.shape) % (1 << (size - 1))
    sign = np.where(rng.random((bh, bw, 63)) < 0.5, -1, 1)
    flat[..., sw.ZIGZAG[1:]] = np.where(mask, sign * mag, 0)
    return coef


def idct_peak(deq, dcoffset):
    """Largest magnitude any intermediate of the reference's integer IDCT (oracle/jpeg_oracle.c jpgo_idct_block) takes for
    the dequantised raster blocks deq [n, 64]: below 2^31 the 32-bit arithmetic does not wrap."""
    x = deq.astype(np.int64).reshape(-1, 8, 8) * 16
    x[:, 0, 0] += dcoffset << 7
    peak = [0]

    def m(v):
        peak[0] = max(peak[0], int(np.abs(v).max()) if v.size else 0)
        return v

    def one_d(i, rnd, sh):
        z1 = m((i[..., 2] + i[..., 6]) * 277)
        t2, t3 = m(z1 - i[..., 6] * 946), m(z1 + i[..., 2] * 392)
        t0, t1 = m((i[..., 0] + i[..., 4]) << 9), m((i[..., 0] - i[..., 4]) << 9)
        a10, a13, a11, a12 = m(t0 + t3), m(t0 - t3), m(t1 + t2), m(t1 - t2)
        o0, o1, o2, o3 = i[..., 7], i[..., 5], i[..., 3], i[..., 1]
        z1o, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
        z5 = m((z3 + z4) * 602)
        o0, o1, o2, o3 = m(o0 * 153), m(o1 * 1051), m(o2 * 1573), m(o3 * 769)
        z1o, z2 = m(z1o * -461), m(z2 * -1312)
        z3, z4 = m(z3 * -1004 + z5), m(z4 * -200 + z5)
        o0, o1, o2, o3 = m(o0 + z1o + z3), m(o1 + z2 + z4), m(o2 + z2 + z3), m(o3 + z1o + z4)
        out = [a10 + o3, a11 + o2, a12 + o1, a13 + o0, a13 - o0, a12 - o1, a11 - o2, a10 - o3]
        return np.stack([m(v + rnd) >> sh for v in out], axis=-1)

    rows = one_d(x, 256, 9)
    one_d(np.swapaxes(rows, 1, 2), 2048, 12)
    return peak[0]


def fit_idct(coef, q, precision, protect=()):
    """Halves the AC coefficients (zig-zag positions not in `protect`) of blocks whose IDCT would leave 32-bit arithmetic,
    until it does not: the streams test the entropy decoders, not the wrap-around of the reconstruction."""
    flat = coef.reshape(-1, 64)
    qr = np.asarray(q).reshape(64)
    free = np.ones(64, dtype=bool)
    free[0] = False
    for k in protect:
        free[sw.ZIGZAG[k]] = False
    dco = 128 if precision == 8 else 2048
    for b in range(flat.shape[0]):
        while idct_peak((flat[b] * qr)[None], dco) >= 2 ** 31 - 2 ** 20:
            before = flat[b].copy()
            flat[b, free] = np.where(np.abs(flat[b, free]) > 1, flat[b, free] // 2, flat[b, free])
            if np.array_equal(before, flat[b]):
                raise ValueError("block %d cannot be brought into 32-bit IDCT arithmetic" % b)
    return coef


def _grey(coef, w, h, q, tables, dri=0, precision=8, dqt16=False, end_with_zrl=False):
    return Frame(w, h, [Component(coef)], {0: q}, [Scan([0])], tables, precision, dqt16, dri, end_with_zrl=end_with_zrl)


# ---------------------------------------------------------------------------------------------------------------------
def long_420():
    rng = np.random.default_rng(101)
    comps = [Component(sparse(rng, 6, 10), 2, 2, 0), Component(sparse(rng, 3, 5), 1, 1, 1), Component(sparse(rng, 3, 5), 1, 1, 1)]
    tables = {("dc", 0): all_lengths_dc(), ("ac", 0): long_table(SEQ_AC, rng), ("dc", 1): long_table(DC_ALL, rng), ("ac", 1): long_table(SEQ_AC, rng)}
    q = {0: rng.integers(1, 5, 64), 1: rng.integers(1, 5, 64)}
    return Frame(80, 48, comps, q, [Scan([0, 1, 2], [0, 1, 1], [0, 1, 1])], tables, restart_interval=4)


def long_444_12bit():
    rng = np.random.default_rng(102)
    comps = [Component(sparse(rng, 3, 5, max_size=11, dc=1500), 1, 1, 0) for _ in range(3)]
    tables = {("dc", 0): all_lengths_dc(), ("ac", 0): long_table(SEQ_AC, rng, force={0x00: 16, 0xF0: 16})}
    q = {0: rng.integers(1, 9, 64)}
    fit_idct(comps[0].coef, q[0], 12), fit_idct(comps[1].coef, q[0], 12), fit_idct(comps[2].coef, q[0], 12)
    return Frame(40, 24, comps, q, [Scan([0, 1, 2])], tables, precision=12, dqt16=True)


def _big_lut(ncomp, hv, w, h, dri, seed, density):
    rng = np.random.default_rng(seed)
    hmax = max(hv)
    mcx, mcy = -(-w // (8 * hmax)), -(-h // (8 * hmax))
    comps = [Component(sparse(rng, mcy * hv[c], mcx * hv[c], density=density), hv[c], hv[c], c) for c in range(ncomp)]
    tables, q = {}, {}
    for c in range(ncomp):
        tables[("dc", c)] = wide_table(DC_ALL, c)
        tables[("ac", c)] = wide_table(SEQ_AC, 7 * c)
        q[c] = rng.integers(1, 5, 64)
    return Frame(w, h, comps, q, [Scan(list(range(ncomp)), list(range(ncomp)), list(range(ncomp)))], tables, restart_interval=dri)


def big_lut_420_rst():
    return _big_lut(3, [2, 1, 1], 64, 48, 2, 103, 0.3)


def big_lut_4c_norst():
    return _big_lut(4, [1, 1, 1, 1], 64, 64, 0, 104, 0.4)


def degenerate_1bit():
    """DC table: category 0 alone on the code '0'; AC table: EOB alone on '0'."""
    coef = np.zeros((2, 3, 8, 8), dtype=np.int32)
    return _grey(coef, 24, 16, np.full(64, 3), {("dc", 0): sw.table_from_lengths({0: 1}), ("ac", 0): sw.table_from_lengths({0x00: 1})})


def degenerate_16bit():
    """One code of length 16 per table, restart interval 1."""
    coef = np.zeros((2, 2, 8, 8), dtype=np.int32)
    return _grey(coef, 16, 16, np.full(64, 5), {("dc", 0): sw.table_from_lengths({0: 16}), ("ac", 0): sw.table_from_lengths({0x00: 16})}, dri=1)


def _dense(rng, bh, bw, precision):
    """All 63 AC positions non-zero. 8 bit: sizes 1..10 and, at k = 1 and 2, sizes 11..15; 12 bit: sizes up to 14. The DC
    alternates between +-16000: every DC difference is of category 15."""
    top = 10 if precision == 8 else 14
    coef = np.zeros((bh, bw, 8, 8), dtype=np.int32)
    flat = coef.reshape(bh, bw, 64)
    size = rng.integers(1, top + 1, size=(bh, bw, 63))
    if precision == 8:
        size[..., 0:2] = rng.integers(11, 16, size=(bh, bw, 2))
    mag = (1 << (size - 1)) + rng.integers(0, 1 << 30, size=size.shape) % (1 << (size - 1))
    flat[..., sw.ZIGZAG[1:]] = np.where(rng.random(size.shape) < 0.5, -mag, mag)
    flat[..., 0] = np.where((np.arange(bh * bw).reshape(bh, bw) & 1) == 0, 16000, -16000)
    return coef


def dense_8bit():
    rng = np.random.default_rng(105)
    coef = _dense(rng, 5, 9, 8)
    q = np.ones(64, dtype=np.int64)
    q.reshape(64)[sw.ZIGZAG[3:]] = rng.integers(1, 3, 61)
    fit_idct(coef, q, 8, protect=(1, 2))
    tables = {("dc", 0): long_table(DC_ALL, rng, force={15: 16}), ("ac", 0): long_table(SEQ_AC, rng, lo=13)}
    return _grey(coef, 72, 40, q, tables, dri=1)


def dense_12bit():
    rng = np.random.default_rng(106)
    coef = _dense(rng, 4, 8, 12)
    q = np.ones(64, dtype=np.int64)
    fit_idct(coef, q, 12, protect=(1, 2, 3))
    tables = {("dc", 0): long_table(DC_ALL, rng, force={15: 16}), ("ac", 0): long_table(SEQ_AC, rng, lo=13)}
    return _grey(coef, 64, 32, q, tables, precision=12)


def _run_edge_blocks(rng, bh, bw):
    coef = sparse(rng, bh, bw, density=0.1)
    for i in range(bh * bw):
        by, bx = divmod(i, bw)
        kind = i % 5
        if kind < 4:
            coef[by, bx] = 0
            coef[by, bx, 0, 0] = int(rng.integers(-50, 51))
        if kind == 0:
            _set(coef, by, bx, 63, 5)               # run 62: three ZRLs, then run 14 size 3 lands on 63, no EOB
        elif kind == 1:
            _set(coef, by, bx, 1, -1)
            _set(coef, by, bx, 63, 1)               # run 61
        elif kind == 2:
            _set(coef, by, bx, 47, 7)
            _set(coef, by, bx, 63, -9)              # run 15 ends exactly on 63
        elif kind == 3:
            _set(coef, by, bx, 1, 3)
            _set(coef, by, bx, 50, 2)               # ZRL chain of three, then EOB
    return coef


def run_edges():
    rng = np.random.default_rng(107)
    tables = {("dc", 0): long_table(DC_ALL, rng), ("ac", 0): long_table(SEQ_AC, rng)}
    return _grey(_run_edge_blocks(rng, 8, 8), 64, 64, rng.integers(1, 6, 64), tables, dri=7)


def zrl_tail():
    """Blocks end with ZRLs that step over position 63 instead of EOB; one restart interval longer than the scan."""
    rng = np.random.default_rng(108)
    tables = {("dc", 0): long_table(DC_ALL, rng), ("ac", 0): long_table(SEQ_AC, rng)}
    return _grey(_run_edge_blocks(rng, 6, 7), 56, 48, rng.integers(1, 6, 64), tables, dri=1000, end_with_zrl=True)


def _stuffing(nblocks, w, h, dri):
    """Codes and values chosen so that the data is mostly 1-bits: FF 00 every other byte. Block i holds i mod 64 coefficients
    of +31 (value bits 11111, the run-0 size-5 symbol on the 16-bit code 1111111111111110), DC difference 0 on the 16-bit code
    of the DC table: interval lengths sweep every residue mod 4 and both sides of multiples of 16 and 128. The last block holds
    63 coefficients: no EOB, so the byte in front of EOI is a stuffed FF."""
    bh, bw = h // 8, w // 8
    coef = np.zeros((bh, bw, 8, 8), dtype=np.int32)
    for i in range(nblocks):
        n = 63 if i == nblocks - 1 else i % 64
        for k in range(1, n + 1):
            _set(coef, i // bw, i % bw, k, 31)
    ac = {0x00: 1, 0xF0: 2, 0x01: 3, 0x02: 4, 0x03: 5, 0x04: 6, 0x06: 7, 0x11: 8, 0x12: 9, 0x13: 10, 0x21: 11, 0x22: 12, 0x31: 13,
          0x41: 14, 0x51: 15, 0x05: 16}
    dc = {c: 16 - c for c in range(16)}
    return _grey(coef, w, h, np.ones(64, dtype=np.int64), {("dc", 0): sw.table_from_lengths(dc), ("ac", 0): sw.table_from_lengths(ac)}, dri=dri)


def stuffing_rst():
    return _stuffing(130, 104, 80, 1)


def stuffing_norst():
    return _stuffing(128, 128, 64, 0)


def _int16_edge(over):
    """Dequantised values at the int16 edge: DC +32767 and -32768 reached through the predictor (category-15 differences of
    an 8-bit scan), AC +-32767 as +-1 x 32767 and -32768 as -1 x 32768 (16-bit quantiser entries). `over`: one coefficient
    +1 x 32768, one beyond the store."""
    coef = np.zeros((1, 8, 8, 8), dtype=np.int32)
    for b, dc in enumerate([16383, 32767, 32767, 0, -16384, -32768, -32768, -100]):
        coef[0, b, 0, 0] = dc
    _set(coef, 0, 0, 1, 1)
    _set(coef, 0, 2, 1, -1)
    _set(coef, 0, 3, 2, -1)
    _set(coef, 0, 5, 2, -1)
    if over:
        _set(coef, 0, 7, 2, 1)
    q = np.ones(64, dtype=np.int64)
    q[sw.ZIGZAG[1]] = 32767
    q[sw.ZIGZAG[2]] = 32768
    tables = {("dc", 0): sw.table_from_counts({c: 1 for c in DC_ALL}),
              ("ac", 0): sw.table_from_counts({0x00: 8, 0x01: 3, 0x11: 2, 0xF0: 1})}
    return _grey(coef, 64, 8, q, tables, dqt16=True)


def int16_edge():
    return _int16_edge(False)


def int16_over():
    return _int16_edge(True)


PROG_SCRIPT_420 = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([1], 1, 63, 0, 1), ([2], 1, 63, 0, 1), ([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1),
                   ([0], 1, 63, 1, 0), ([1], 1, 63, 1, 0), ([2], 1, 63, 1, 0), ([0, 1, 2], 0, 0, 1, 0)]


def prog_long_420():
    """Ten scans (DC first and refinement, AC bands with Al 1 and 2, AC refinement) on long-code tables, restart interval 2."""
    rng = np.random.default_rng(109)
    comps = [Component(sparse(rng, 4, 6, density=0.35, max_size=8), 2, 2, 0), Component(sparse(rng, 2, 3, density=0.35, max_size=8), 1, 1, 1),
             Component(sparse(rng, 2, 3, density=0.35, max_size=8), 1, 1, 1)]
    scans = []
    for comps_, ss, se, ah, al in PROG_SCRIPT_420:
        if ss == 0:
            t = {("dc", 0): all_lengths_dc(), ("dc", 1): long_table(DC_ALL, rng)} if ah == 0 else {}
            scans.append(Scan(comps_, [0, 1, 1], [0, 0, 0], ss, se, ah, al, t))
        else:
            t = {("ac", 0): long_table(PROG_REFINE if ah else PROG_AC_FIRST, rng, force={0xE0: 16})}
            scans.append(Scan(comps_, [0], [0], ss, se, ah, al, t))
    return Frame(48, 32, comps, {0: rng.integers(1, 4, 64), 1: rng.integers(1, 4, 64)}, scans, restart_interval=2, progressive=True)


PROG_BANDS = [(1, 1, 0, 1), (2, 5, 0, 1), (6, 14, 0, 1), (15, 27, 0, 1), (28, 63, 0, 1), (1, 63, 1, 0)]


def prog_big_6scans():
    """Six AC scans of the luma component, each on its own table of all 256 symbols on 12/13-bit codes (DHT in front of every scan):
    the component-fused AC kernel holds six distinct LUTs of about 6,100 words in shared memory."""
    rng = np.random.default_rng(110)
    comps = [Component(sparse(rng, 4, 4, density=0.35, max_size=8), 1, 1, c) for c in range(3)]
    scans = [Scan([0, 1, 2], [0, 1, 2], [0, 0, 0], 0, 0, 0, 0, {("dc", c): wide_table(DC_ALL, c) for c in range(3)})]
    for i, (ss, se, ah, al) in enumerate(PROG_BANDS):
        scans.append(Scan([0], [0], [0], ss, se, ah, al, {("ac", 0): wide_table(list(range(256)), i)}))
    for c in (1, 2):  # (the chroma components in one scan each: the scan count stays within what the oracle keeps)
        scans.append(Scan([c], [0], [c], 1, 63, 0, 0, {("ac", c): wide_table(list(range(256)), 6 + c)}))
    return Frame(32, 32, comps, {c: rng.integers(1, 4, 64) for c in range(3)}, scans, restart_interval=4, progressive=True)


def prog_eobrun_max():
    """A grey frame of 184 x 184 blocks, nearly all of them zero in the AC band: the first EOB run reaches 32767 (EOB14 plus
    fourteen 1-bits, on a 16-bit code), the refinement scan carries correction bits behind its runs."""
    rng = np.random.default_rng(111)
    n = 184
    coef = np.zeros((n, n, 8, 8), dtype=np.int32)
    coef[..., 0, 0] = rng.integers(-3, 4, size=(n, n))
    _set(coef, 0, 0, 5, 6)
    by, bx = divmod(32768, n)
    _set(coef, by, bx, 1, 3)
    _set(coef, by, bx, 63, -2)
    t_dc = long_table(DC_ALL, rng)
    t_first = long_table(PROG_AC_FIRST, rng, force={0xE0: 16})
    t_ref = long_table(PROG_REFINE, rng, force={0xE0: 16})
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, {("dc", 0): t_dc}), Scan([0], [0], [0], 1, 63, 0, 1, {("ac", 0): t_first}),
             Scan([0], [0], [0], 1, 63, 1, 0, {("ac", 0): t_ref})]
    return Frame(8 * n, 8 * n, [Component(coef)], {0: rng.integers(1, 4, 64)}, scans, progressive=True)


CASES = {f.__name__: f for f in [long_420, long_444_12bit, big_lut_420_rst, big_lut_4c_norst, degenerate_1bit, degenerate_16bit, dense_8bit,
                                 dense_12bit, run_edges, zrl_tail, stuffing_rst, stuffing_norst, int16_edge, int16_over, prog_long_420,
                                 prog_big_6scans, prog_eobrun_max]}
NAMES = list(CASES)
# the frame whose dequantised coefficient +32768 leaves the int16 coefficient store: MALFORMED_STREAM on the GPU, decoded by the
# reference (DESIGN.md section 7)
BEYOND_INT16 = {"int16_over"}


@functools.lru_cache(maxsize=None)
def case(name):
    frame = CASES[name]()
    return frame, sw.encode(frame)


def quantised(frame):
    return [c.coef for c in frame.components]


def dequantised(frame):
    """[per component int32 [bh, bw, 8, 8]]: the coefficients times the component's quantiser (raster order)."""
    return [c.coef * np.asarray(frame.quant[c.tq], dtype=np.int64).reshape(8, 8) for c in frame.components]
