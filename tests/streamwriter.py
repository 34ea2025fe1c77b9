"""A coefficient-first JPEG codestream writer for tests, written from ITU-T T.81 alone.

Input: quantised coefficients per component ([bh, bw, 8, 8] int32, raster order inside the block, over the MCU-padded block
grid), the precision, the quantisation tables, Huffman tables given as BITS / HUFFVAL, a scan script and a restart interval.
Output: SOI ... EOI with byte stuffing. Nothing is chosen for the caller: a coefficient whose symbol is missing from the table
in effect, or an illegal table, raises ValueError.

  Annex C   canonical code assignment (Figures C.1-C.3), with the all-ones code word of every length kept free
  Annex K.2 code lengths from symbol counts, limited to 16 bits (Figure K.3)
  F.1.2     sequential DC / AC coding (DIFF categories, run / size symbols, ZRL, EOB)
  G.1.2     progressive coding: DC first and refinement scans, AC spectral selection with EOBRUN, AC successive approximation
            with correction bits
"""
import heapq
from dataclasses import dataclass, field

import numpy as np

# zig-zag position k -> raster index (T.81 Figure A.6)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63])


class HuffTable:
    """BITS[16] / HUFFVAL with the canonical codes of Annex C: codes[symbol] = (code, length)."""

    def __init__(self, bits, vals):
        bits, vals = [int(b) for b in bits], [int(v) for v in vals]
        if len(bits) != 16 or min(bits) < 0:
            raise ValueError("BITS must hold 16 counts")
        if sum(bits) != len(vals) or not 1 <= len(vals) <= 256:
            raise ValueError("BITS and HUFFVAL disagree")
        if len(set(vals)) != len(vals) or min(vals) < 0 or max(vals) > 255:
            raise ValueError("HUFFVAL must hold distinct byte values")
        self.bits, self.vals, self.codes = bits, vals, {}
        code, i = 0, 0
        for length in range(1, 17):
            for _ in range(bits[length - 1]):
                if code >= (1 << length):
                    raise ValueError("over-full code: the Kraft sum exceeds one")
                if code == (1 << length) - 1:
                    raise ValueError("the all-ones code word of length %d is reserved" % length)
                self.codes[vals[i]] = (code, length)
                code += 1
                i += 1
            code <<= 1

    def dht_payload(self, tc, th):
        return bytes([(tc << 4) | th] + self.bits + self.vals)


def table_from_lengths(lengths):
    """{symbol: code length} -> HuffTable, symbols of one length in ascending order."""
    bits = [0] * 16
    for sym, n in lengths.items():
        if not 1 <= n <= 16:
            raise ValueError("code lengths are 1..16")
        bits[n - 1] += 1
    return HuffTable(bits, sorted(lengths, key=lambda s: (lengths[s], s)))


def table_from_counts(counts):
    """Annex K.2: Huffman code lengths for {symbol: count}, limited to 16 bits, all-ones code kept free."""
    syms = sorted(s for s, c in counts.items() if c > 0)
    if not syms:
        raise ValueError("no symbols")
    reserved = 256  # K.2: one extra symbol of frequency 1 takes the all-ones code
    heap = [(counts[s], s, [s]) for s in syms] + [(1, reserved, [reserved])]
    heapq.heapify(heap)
    size = {s: 0 for s in syms + [reserved]}
    while len(heap) > 1:
        f1, k1, a = heapq.heappop(heap)
        f2, k2, b = heapq.heappop(heap)
        for s in a + b:
            size[s] += 1
        heapq.heappush(heap, (f1 + f2, min(k1, k2), a + b))
    hist = [0] * 64
    for s in size:
        hist[size[s]] += 1
    for i in range(63, 16, -1):  # Figure K.3
        while hist[i] > 0:
            j = i - 2
            while hist[j] == 0:
                j -= 1
            hist[i] -= 2
            hist[i - 1] += 1
            hist[j + 1] += 2
            hist[j] -= 1
    i = 16
    while hist[i] == 0:
        i -= 1
    hist[i] -= 1  # the reserved symbol leaves
    order = sorted(syms, key=lambda s: (-counts[s], s))
    lengths, at = {}, 0
    for n in range(1, 17):
        for _ in range(hist[n]):
            lengths[order[at]] = n
            at += 1
    return table_from_lengths(lengths)


def category(v):
    return abs(int(v)).bit_length()


def value_bits(v, s):
    """F.1.2.1: the s low bits of v, of v - 1 for negative v."""
    return (int(v) if v >= 0 else int(v) + (1 << s) - 1) & ((1 << s) - 1)


class BitWriter:
    """Entropy-coded segment bytes with FF 00 stuffing (B.1.1.5); records the start bit and length of every coded symbol
    (Huffman code + value bits) in the unstuffed bit stream of the current interval."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0
        self.bit = 0          # bits written in the current interval
        self.symbols = []     # (start bit within the interval, code length + value bits)
        self.blocks = []      # start bit within the interval of every block of a sequential scan, in coding order
        self.intervals = []   # unstuffed bytes of every finished interval

    def put(self, value, n):
        if n == 0:
            return
        self.acc = (self.acc << n) | (int(value) & ((1 << n) - 1))
        self.n += n
        self.bit += n
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 0xFF
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)
        self.acc &= (1 << self.n) - 1

    def symbol(self, table, sym, value=0, s=0):
        if sym not in table.codes:
            raise ValueError("symbol 0x%02x is not in the table" % sym)
        code, length = table.codes[sym]
        self.symbols.append((self.bit, length + s))
        self.put(code, length)
        self.put(value_bits(value, s), s)

    def end_interval(self):
        """Pads the interval with 1-bits to a byte boundary (F.1.2.3)."""
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        self.intervals.append(self.bit // 8)
        self.bit = 0


@dataclass
class Component:
    coef: np.ndarray      # [bh, bw, 8, 8] quantised, raster order inside the block, MCU-padded grid
    h: int = 1
    v: int = 1
    tq: int = 0


@dataclass
class Scan:
    comps: list           # frame component indices, in SOS order
    td: list = None       # DC table slot per scan component (default 0)
    ta: list = None       # AC table slot per scan component (default 0)
    ss: int = 0
    se: int = 63
    ah: int = 0
    al: int = 0
    tables: dict = field(default_factory=dict)  # {("dc" | "ac", slot): HuffTable} defined right in front of this scan


@dataclass
class Frame:
    width: int
    height: int
    components: list
    quant: dict                                # {slot: 64 quantiser values in RASTER order}
    scans: list
    tables: dict = field(default_factory=dict)  # {("dc" | "ac", slot): HuffTable} defined in front of the first scan
    precision: int = 8
    dqt16: bool = False
    restart_interval: int = 0
    progressive: bool = False
    end_with_zrl: bool = False                 # sequential: trailing zeros end with ZRLs that step over k = 63 instead of EOB
    stats: dict = field(default_factory=dict)   # filled by encode(): "symbols", "intervals" (per scan)


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def _dht(tables):
    payload = b""
    for (kind, slot), t in sorted(tables.items()):
        payload += t.dht_payload(0 if kind == "dc" else 1, slot)
    return _segment(0xC4, payload) if payload else b""


def _cdiv(a, b):
    return -(-a // b)


def geometry(frame):
    """(hmax, vmax, mcu_cols, mcu_rows, [(bw, bh) of the component's own block grid])"""
    hmax = max(c.h for c in frame.components)
    vmax = max(c.v for c in frame.components)
    mcx = -(-frame.width // (8 * hmax))
    mcy = -(-frame.height // (8 * vmax))
    own = [(_cdiv(_cdiv(frame.width * c.h, hmax), 8), _cdiv(_cdiv(frame.height * c.v, vmax), 8)) for c in frame.components]
    return hmax, vmax, mcx, mcy, own


def _scan_units(frame, scan):
    """Per MCU of the scan: the list of (scan component index, block row, block column) in coding order (A.2)."""
    hmax, vmax, mcx, mcy, own = geometry(frame)
    if len(scan.comps) == 1:
        ci = scan.comps[0]
        bw, bh = own[ci]
        return [[(0, by, bx)] for by in range(bh) for bx in range(bw)]
    units = []
    for my in range(mcy):
        for mx in range(mcx):
            u = []
            for k, ci in enumerate(scan.comps):
                c = frame.components[ci]
                for y in range(c.v):
                    for x in range(c.h):
                        u.append((k, my * c.v + y, mx * c.h + x))
            units.append(u)
    return units


def _zz(blk):
    return blk.reshape(64)[ZIGZAG]


class _ScanCoder:
    def __init__(self, frame, scan, w, dc, ac):
        self.f, self.s, self.w, self.dc, self.ac = frame, scan, w, dc, ac
        self.pred = [0] * 4
        self.eobrun = 0
        self.be = []  # correction bits that follow the pending EOB run

    def restart(self):
        self.flush_eobrun()
        self.pred = [0] * 4

    def dc_diff(self, k, v):
        diff = int(v) - self.pred[k]
        self.pred[k] = int(v)
        s = category(diff)
        if s > 15:
            raise ValueError("DC difference %d has no category" % diff)
        self.w.symbol(self.dc[k], s, diff, s)

    def sequential(self, k, blk):
        zz = _zz(blk)
        self.dc_diff(k, zz[0])
        nz = np.nonzero(zz[1:])[0]
        last = int(nz[-1]) + 1 if len(nz) else 0
        r = 0
        for i in range(1, last + 1):
            v = int(zz[i])
            if v == 0:
                r += 1
                continue
            while r > 15:
                self.w.symbol(self.ac[k], 0xF0)
                r -= 16
            s = category(v)
            if s > 15:
                raise ValueError("AC coefficient %d has no category" % v)
            self.w.symbol(self.ac[k], (r << 4) | s, v, s)
            r = 0
        if last < 63:
            if self.f.end_with_zrl:
                for _ in range(-(-(63 - last) // 16)):
                    self.w.symbol(self.ac[k], 0xF0)
            else:
                self.w.symbol(self.ac[k], 0x00)

    def flush_eobrun(self):
        if self.eobrun:
            n = self.eobrun.bit_length() - 1
            self.w.symbol(self.ac[0], n << 4, self.eobrun - (1 << n), n)
            for b in self.be:
                self.w.put(b, 1)
            self.eobrun, self.be = 0, []

    def ac_first(self, blk):
        zz, al = _zz(blk), self.s.al
        if not np.any(np.abs(zz[self.s.ss:self.s.se + 1]) >> al):  # nothing in the band: the block joins the EOB run
            self.eobrun += 1
            if self.eobrun == 0x7FFF:
                self.flush_eobrun()
            return
        r = 0
        for i in range(self.s.ss, self.s.se + 1):
            v = int(zz[i])
            t = (abs(v) >> al) * (1 if v >= 0 else -1)  # G.1.2.2: point transform of AC coefficients rounds towards zero
            if t == 0:
                r += 1
                continue
            self.flush_eobrun()
            while r > 15:
                self.w.symbol(self.ac[0], 0xF0)
                r -= 16
            s = category(t)
            self.w.symbol(self.ac[0], (r << 4) | s, t, s)
            r = 0
        if r > 0:
            self.eobrun += 1
            if self.eobrun == 0x7FFF:
                self.flush_eobrun()

    def ac_refine(self, blk):
        zz, al = _zz(blk), self.s.al
        if not np.any(np.abs(zz[self.s.ss:self.s.se + 1]) >> al):
            self.eobrun += 1
            if self.eobrun == 0x7FFF:
                self.flush_eobrun()
            return
        absv = [abs(int(zz[i])) >> al for i in range(64)]
        eob = max([i for i in range(self.s.ss, self.s.se + 1) if absv[i] == 1], default=-1)
        r, br = 0, []
        for i in range(self.s.ss, self.s.se + 1):
            t = absv[i]
            if t == 0:
                r += 1
                continue
            while r > 15 and i <= eob:
                self.flush_eobrun()
                self.w.symbol(self.ac[0], 0xF0)
                r -= 16
                for b in br:
                    self.w.put(b, 1)
                br = []
            if t > 1:  # already non-zero: one correction bit
                br.append(t & 1)
                continue
            self.flush_eobrun()
            self.w.symbol(self.ac[0], (r << 4) | 1)
            self.w.put(1 if zz[i] > 0 else 0, 1)
            for b in br:
                self.w.put(b, 1)
            br, r = [], 0
        if r > 0 or br:
            self.eobrun += 1
            self.be += br
            if self.eobrun == 0x7FFF:
                self.flush_eobrun()

    def block(self, k, blk):
        s = self.s
        if not self.f.progressive:
            self.w.blocks.append(self.w.bit)
            self.sequential(k, blk)
        elif s.ss == 0:
            dc = int(blk[0, 0])
            if s.ah == 0:
                self.dc_diff(k, dc >> s.al)
            else:
                self.w.put((dc >> s.al) & 1, 1)
        elif s.ah == 0:
            self.ac_first(blk)
        else:
            self.ac_refine(blk)


def _check_scan(frame, scan):
    if frame.progressive:
        if scan.ss == 0 and scan.se != 0:
            raise ValueError("progressive DC scans code coefficient 0 alone")
        if scan.ss > 0 and len(scan.comps) != 1:
            raise ValueError("progressive AC scans hold one component")
        if scan.ah and scan.al != scan.ah - 1:
            raise ValueError("successive approximation refines one bit at a time")
    elif (scan.ss, scan.se, scan.ah, scan.al) != (0, 63, 0, 0):
        raise ValueError("sequential scans code the whole block")


def encode(frame):
    """-> the codestream (bytes). frame.stats receives, per scan, the coded symbols, the unstuffed interval lengths and the start
    bits of the blocks of a sequential scan."""
    if frame.precision not in (8, 12):
        raise ValueError("precision is 8 or 12")
    hmax, vmax, mcx, mcy, own = geometry(frame)
    for ci, c in enumerate(frame.components):
        if c.coef.shape != (mcy * c.v, mcx * c.h, 8, 8):
            raise ValueError("component %d: coefficients must cover the MCU-padded grid %r" % (ci, (mcy * c.v, mcx * c.h)))
    out = bytearray(b"\xff\xd8")
    dqt = b""
    for slot, q in sorted(frame.quant.items()):
        q = np.asarray(q).reshape(64)[ZIGZAG]
        if q.min() < 1 or q.max() > (65535 if frame.dqt16 else 255):
            raise ValueError("quantiser out of range")
        dqt += bytes([(0x10 if frame.dqt16 else 0) | slot]) + (b"".join(int(v).to_bytes(2, "big") for v in q) if frame.dqt16 else bytes(int(v) for v in q))
    out += _segment(0xDB, dqt)
    baseline = (frame.precision == 8 and not frame.dqt16 and not frame.progressive and
                all(slot < 2 for scan in frame.scans for slot in (scan.td or [0]) + (scan.ta or [0])) and
                all(slot < 2 for (_, slot) in frame.tables))
    sof = 0xC2 if frame.progressive else (0xC0 if baseline else 0xC1)
    payload = [frame.precision] + list(frame.height.to_bytes(2, "big")) + list(frame.width.to_bytes(2, "big")) + [len(frame.components)]
    for ci, c in enumerate(frame.components):
        payload += [ci + 1, (c.h << 4) | c.v, c.tq]
    out += _segment(sof, payload)
    out += _dht(frame.tables)
    if frame.restart_interval:
        out += _segment(0xDD, list(frame.restart_interval.to_bytes(2, "big")))
    current = dict(frame.tables)
    frame.stats = {"symbols": [], "intervals": [], "blocks": []}
    for scan in frame.scans:
        _check_scan(frame, scan)
        out += _dht(scan.tables)
        current.update(scan.tables)
        ns = len(scan.comps)
        td, ta = scan.td or [0] * ns, scan.ta or [0] * ns
        dc = [current.get(("dc", td[k])) for k in range(ns)]
        ac = [current.get(("ac", ta[k])) for k in range(ns)]
        sos = [ns]
        for k, ci in enumerate(scan.comps):
            sos += [ci + 1, (td[k] << 4) | ta[k]]
        sos += [scan.ss, scan.se, (scan.ah << 4) | scan.al]
        out += _segment(0xDA, sos)
        w = BitWriter()
        coder = _ScanCoder(frame, scan, w, dc, ac)
        units = _scan_units(frame, scan)
        if ns == 1:  # blocks of the padded grid outside the component's own grid are not coded: they must be zero
            c = frame.components[scan.comps[0]]
            bw, bh = own[scan.comps[0]]
            if np.any(c.coef[bh:]) or np.any(c.coef[:, bw:]):
                raise ValueError("component %d has coefficients outside the grid a single-component scan codes" % scan.comps[0])
        ri, rst = frame.restart_interval, 0
        for m, unit in enumerate(units):
            if ri and m and m % ri == 0:
                coder.restart()
                w.end_interval()
                w.out += bytes([0xFF, 0xD0 + (rst & 7)])
                rst += 1
            for (k, by, bx) in unit:
                coder.block(k, frame.components[scan.comps[k]].coef[by, bx])
        coder.flush_eobrun()
        w.end_interval()
        out += w.out
        frame.stats["symbols"].append(w.symbols)
        frame.stats["intervals"].append(w.intervals)
        frame.stats["blocks"].append(w.blocks)
    out += b"\xff\xd9"
    return bytes(out)
