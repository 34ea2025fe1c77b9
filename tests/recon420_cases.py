"""Hand-built 4:2:0 frames aimed at the seams of reconstruct420_kernel (libjpeg_b200/csrc/recon_sm100.cu), plus a plain 64-bit
model of the upsampling and colour stage. tests/streamwriter.py writes the frames from chosen quantised coefficients (seeded,
deterministic); every quantiser entry is 1, so the quantised coefficients are the dequantised ones.

A CTA of reconstruct420_kernel covers 256 x 32 luma pixels: chroma block columns 16k .. 16k + 15 and chroma block rows
2r, 2r + 1 (its tile), the line above / below (row 7 of chroma block row 2r - 1, row 0 of row 2r + 2: tile_idct_rows with
only = 7 / 0) and the column left / right (column 7 of chroma block column 16k - 1, column 0 of 16k + 16: phase 1b). In phase
1a, lane L of a warp holds block L & 15 of the component L >> 4 (Cb, Cr) of one chroma block row.

case(name) -> (Frame, codestream bytes); meta(name) -> what the case is there for (see Meta)."""
import dataclasses
import functools

import numpy as np

from tests import entropy_cases as ec
from tests import streamwriter as sw
from tests.streamwriter import Component, Frame, Scan

CTA_W, CTA_H = 256, 32       # luma pixels per CTA
CTA_CBX, CTA_CBY = 16, 2     # chroma blocks per CTA (4:2:0)
ONES = np.ones(64, dtype=np.int64)
WIDE = 32767                 # coefficient row (column) 0 all WIDE: column (row) 0 of the samples near 491,000 (oracle.idct)
WIDE_DC = 32700              # its DC: the DC difference to a neighbour (DC within +-60) stays within category 15
BRIGHT = 25000               # luma DC: samples 52,048, inside +-65535, enough for Cb ~ 122,000 to wrap the 32-bit blue sum
# (DC, coefficient 1) of a block whose extreme sample is exactly the key, in column 0 of every row and nowhere else
# (found with oracle.idct; tests/test_recon420_cases.py checks them)
EDGE = {32767: (15358, 1), 32768: (15357, 2), -32768: (-17404, -3), -32769: (-17407, -1)}


@dataclasses.dataclass
class Meta:
    sense: list = dataclasses.field(default_factory=list)    # [(component, by, bx, 8x8 bool mask)]: the targeted coefficients
    sense_px: list = dataclasses.field(default_factory=list)  # [(y0, y1, x0, x1)]: pixels that must change when they are zeroed
    sense_min: int = 0                                        # ... in at least this many bytes
    extreme: tuple = None                                     # (component, by, bx) of the block that leaves the fast ranges
    peak: int = None                                          # the exact extreme chroma sample of the frame
    narrow: bool = False                                      # some chroma sample leaves int16: the int32 instance redoes it
    twin: str = None                                          # the same frame without the extreme block
    wrap_px: list = dataclasses.field(default_factory=list)   # [(y0, y1, x0, x1)]: 32-bit colour differs from 64-bit in here
    unsat_px: list = dataclasses.field(default_factory=list)  # [(y0, y1, x0, x1)]: mostly unsaturated output bytes


def _table(syms, weight):
    return sw.table_from_counts({s: weight(s) for s in syms})


# ordinary tables: short codes for EOB and small values, every symbol a sequential scan may need
AC_TABLE = _table(ec.SEQ_AC, lambda s: 4000 if s == 0 else (20 if s == 0xF0 else max(1, 2000 >> (2 * (s & 15) + (s >> 4)))))
DC_TABLE = _table(ec.DC_ALL, lambda s: max(1, 1000 >> s))
TABLES = {("dc", 0): DC_TABLE, ("ac", 0): AC_TABLE, ("dc", 1): DC_TABLE, ("ac", 1): AC_TABLE}


def _cdiv(a, b):
    return -(-a // b)


def _luma(rng, bh, bw):
    """Near mid-grey: DC +-16 (pixels 128 +- 2), a few small low-frequency terms."""
    c = np.zeros((bh, bw, 8, 8), dtype=np.int32)
    c[..., 0, 0] = rng.integers(-16, 17, (bh, bw))
    c[..., 0, 1] = rng.integers(-6, 7, (bh, bw))
    c[..., 1, 0] = rng.integers(-6, 7, (bh, bw))
    return c


def _chroma(rng, bh, bw):
    """Sparse, low-frequency, moderate: coefficient rows 0 .. 2 only."""
    c = np.zeros((bh, bw, 8, 8), dtype=np.int32)
    c[..., 0, 0] = rng.integers(-60, 61, (bh, bw))
    for r, k in ((0, 1), (1, 0), (1, 1), (0, 2), (2, 0)):
        c[..., r, k] = np.where(rng.random((bh, bw)) < 0.5, rng.integers(-20, 21, (bh, bw)), 0)
    return c


def dense(rng, cols=True, rows=False):
    """All 64 coefficients non-zero. cols: large pairs in coefficient columns 5 and 7 of every row, with 402 v5 + 141 v7 ~ 0, so
    that column 0 and 7 of the samples (the halo columns of phase 1b) stay moderate while the 402 and 141 terms of its dot
    products are large. rows: the same in coefficient rows 5 and 7 (the `only` dot products of the line above / below)."""
    b = rng.integers(1, 13, (8, 8)) * np.where(rng.random((8, 8)) < 0.5, -1, 1)
    big = lambda n: rng.integers(300, 601, n) * np.where(rng.random(n) < 0.5, -1, 1)
    if cols:
        b[:, 7] = big(8)
        b[:, 5] = -np.rint(141 * b[:, 7] / 402).astype(np.int64) + rng.integers(-3, 4, 8)
    if rows:
        b[7, :] = big(8)
        b[5, :] = -np.rint(141 * b[7, :] / 402).astype(np.int64) + rng.integers(-3, 4, 8)
    b[b == 0] = 1
    return b.astype(np.int32)


def frame(w, h, comps, sub=(2, 2)):
    """Sequential, one interleaved scan, ordinary tables, every quantiser entry 1. comps = [Y, Cb, Cr] quantised [bh, bw, 8, 8]."""
    hv = [sub, (1, 1), (1, 1)]
    return Frame(w, h, [Component(c, hv[i][0], hv[i][1], min(i, 1)) for i, c in enumerate(comps)], {0: ONES, 1: ONES},
                 [Scan([0, 1, 2], [0, 1, 1], [0, 1, 1])], dict(TABLES))


def base(w, h, seed, sub=(2, 2)):
    """[Y, Cb, Cr] over the MCU-padded grids: luma near grey, chroma sparse and low-frequency."""
    rng = np.random.default_rng(seed)
    mcx, mcy = _cdiv(w, 8 * sub[0]), _cdiv(h, 8 * sub[1])
    return rng, [_luma(rng, mcy * sub[1], mcx * sub[0]), _chroma(rng, mcy, mcx), _chroma(rng, mcy, mcx)]


def reach(f, comp, by, bx):
    """(y0, y1, x0, x1), half-open and clipped to the frame: the pixels whose value depends on block (by, bx) of component comp.
    A chroma sample feeds the output pixels of its own position and of the neighbouring sample on either side (both filter
    cores, including HorizontalFilterCore<2>'s read of the new out[2], and the edge replication)."""
    sx, sy = (f.components[0].h, f.components[0].v) if comp else (1, 1)
    y0, y1, x0, x1 = 8 * by * sy, 8 * (by + 1) * sy, 8 * bx * sx, 8 * (bx + 1) * sx
    if sx == 2:
        x0, x1 = x0 - 2, x1 + 2
    if sy == 2:
        y0, y1 = y0 - 2, y1 + 2
    return max(y0, 0), min(y1, f.height), max(x0, 0), min(x1, f.width)


def _mask(rows=range(8), cols=range(8)):
    m = np.zeros((8, 8), dtype=bool)
    m[np.ix_(list(rows), list(cols))] = True
    return m


# ---------------------------------------------------------------------------------------------------------------------------
def _seams(w, h, seed, cols, rows):
    """Dense blocks in both chroma components at the CTA seams: block columns 16k - 1, 16k (cols) and block rows 2r - 1,
    2r + 2 (rows; 2r + 2 is the first row of the next CTA row, so that is block rows 2r - 1 and 2r for r >= 1)."""
    rng, (y, cb, cr) = base(w, h, seed)
    bh, bw = cb.shape[:2]
    seam_c = [c for k in range(1, _cdiv(bw, CTA_CBX)) for c in (CTA_CBX * k - 1, CTA_CBX * k) if c < bw] if cols else []
    seam_r = [r for k in range(1, _cdiv(bh, CTA_CBY)) for r in (CTA_CBY * k - 1, CTA_CBY * k) if r < bh] if rows else []
    for comp in (cb, cr):
        for by in range(bh):
            for bx in range(bw):
                c, r = bx in seam_c, by in seam_r
                if c or r:
                    comp[by, bx] = dense(rng, cols=c, rows=r)
    return [y, cb, cr], seam_c, seam_r


def seam_cols():
    """Phase 1b: dense chroma blocks at block columns 16k - 1 and 16k of a 3 x 3 CTA frame. Column 7 of block 16k - 1 is CTA k's
    left halo column, column 0 of block 16k is CTA k - 1's right halo column; both carry the 402 / 141 terms of the row-pass dot
    products. Sensitivity: coefficient columns 5 .. 7 of the blocks at column 16k - 1 alone feed luma column 256k only through
    CTA k's left halo."""
    comps, sc, _ = _seams(768, 96, 201, True, False)
    f = frame(768, 96, comps)
    left = [c for c in sc if c % CTA_CBX == CTA_CBX - 1]
    m = Meta(sense=[(comp, by, bx, _mask(cols=range(5, 8))) for comp in (1, 2) for by in range(comps[1].shape[0]) for bx in left],
             sense_px=[(0, 96, 16 * (bx + 1), 16 * (bx + 1) + 1) for bx in left], sense_min=100,
             unsat_px=[(0, 96, 16 * c + d, 16 * c + d + 1) for c in left for d in (15, 16)])
    return f, m


def seam_rows():
    """The `only` dot products: dense chroma blocks at block rows 2r - 1 and 2r + 2 (coefficient rows 5 .. 7 included) of a 3 x 3
    CTA frame: row 7 of block row 2r - 1 is the line above of CTA row r, row 0 of block row 2r is the line below of CTA row
    r - 1. Sensitivity: coefficient rows 5 .. 7 of block row 2r - 1 alone feed luma row 32r only through the line above."""
    comps, _, sr = _seams(768, 96, 202, False, True)
    f = frame(768, 96, comps)
    above = [r for r in sr if r % CTA_CBY == CTA_CBY - 1]
    m = Meta(sense=[(comp, by, bx, _mask(rows=range(5, 8))) for comp in (1, 2) for by in above for bx in range(comps[1].shape[1])],
             sense_px=[(16 * (by + 1), 16 * (by + 1) + 1, 0, 768) for by in above], sense_min=300,
             unsat_px=[(16 * r + d, 16 * r + d + 1, 0, 768) for r in above for d in (15, 16)])
    return f, m


def seam_corners():
    """The window corners (line 0 / 17 x column 3 / 132): chroma content only in the four blocks around every inner corner of
    the CTA grid (block rows 2r - 1, 2r x columns 16k - 1, 16k), each the diagonal neighbour of one CTA; everything else flat.
    Sensitivity: block (2r - 1, 16k - 1) alone feeds pixel (32r, 256k) only through CTA (r, k)'s corner (line 0, column 3)."""
    rng, (y, cb, cr) = base(768, 96, 203)
    cb[...], cr[...] = 0, 0
    for comp in (cb, cr):
        for r in (1, 2):
            for k in (1, 2):
                for by in (2 * r - 1, 2 * r):
                    for bx in (16 * k - 1, 16 * k):
                        comp[by, bx] = dense(rng, cols=True, rows=True)
    f = frame(768, 96, [y, cb, cr])
    m = Meta(sense=[(comp, 2 * r - 1, 16 * k - 1, _mask()) for comp in (1, 2) for r in (1, 2) for k in (1, 2)],
             sense_px=[(32 * r, 32 * r + 1, 256 * k, 256 * k + 1) for r in (1, 2) for k in (1, 2)], sense_min=4)
    return f, m


# lane -> (component, block column within the CTA); the right-edge partial warp of skip_rule has 5 blocks per component
SKIP_LANES = {0: (1, 0), 15: (1, 15), 16: (2, 0), 31: (2, 15)}
SKIP_PARTIAL = {0: (1, 0), 4: (1, 4), 16: (2, 0), 20: (2, 4)}


def skip_rule():
    """tile_idct's per-warp rule that skips coefficient rows 6 and 7. 4 full CTA columns plus a partial one (5 chroma blocks per
    component) x 4 CTA rows. In every chroma block row of a CTA (one warp) each block has coefficients in rows 0 .. 5 only,
    except in the warps listed here, where one block has a single coefficient in row 6 or 7, column 0 or 7, in lane 0, 15, 16
    or 31 (first / last Cb, first / last Cr block), and in the partial warp in its first / last Cb and Cr block. The same block
    row is the line above or below of the neighbouring CTA row (the `only` branch)."""
    w, h = 4 * CTA_W + 72, 4 * CTA_H
    rng, (y, cb, cr) = base(w, h, 204)
    for comp in (cb, cr):
        comp[..., :6, :] = rng.integers(-6, 7, comp[..., :6, :].shape)
    slots = [(k, by) for by in range(8) for k in range(4)]
    place = [(k, by, lane, row, col) for (lane, (row, col)), (k, by) in
             zip([(lane, (row, col)) for lane in SKIP_LANES for row in (6, 7) for col in (0, 7)], slots[::2])]
    place += [(4, by, lane, row, col) for by, (lane, row, col) in zip((0, 3, 4, 7), [(0, 7, 0), (4, 6, 7), (16, 6, 0), (20, 7, 7)])]
    m = Meta(sense_min=0)
    comps = [y, cb, cr]
    f = frame(w, h, comps)
    for k, by, lane, row, col in place:
        c, j = (SKIP_PARTIAL if k == 4 else SKIP_LANES)[lane]
        bx = CTA_CBX * k + j
        v = int(rng.integers(120, 200)) * (1 if rng.random() < 0.5 else -1)
        comps[c][by, bx, row, col] = v
        m.sense.append((c, by, bx, _mask(rows=[row], cols=[col])))
        m.sense_px.append(reach(f, c, by, bx))
    m.sense_min = 20 * len(place)
    m.unsat_px = list(m.sense_px)
    return f, m


SWEEP = [(3 * CTA_W - 1, 3 * CTA_H - 1), (2 * CTA_W + 1, 2 * CTA_H + 1), (2 * CTA_W + 8, 2 * CTA_H + 8), (2 * CTA_W + 9, 2 * CTA_H + 9),
         (2 * CTA_W + 16, 2 * CTA_H + 16), (2 * CTA_W + 17, 2 * CTA_H + 17), (1, 3 * CTA_H + 1), (3 * CTA_W + 1, 1)]


def _sweep(w, h):
    def make():
        comps, _, _ = _seams(w, h, 205 + w + h, True, True)
        return frame(w, h, comps), Meta()
    make.__name__ = "sweep_%dx%d" % (w, h)
    make.__doc__ = ("Geometry: %d x %d, seam columns and rows as in seam_cols / seam_rows: partial CTAs, odd chroma sizes, an "
                    "MCU-padded luma grid wider than the visible blocks where ceil(W / 8) is odd." % (w, h))
    return make


def _edge(target, seam):
    def make():
        rng, (y, cb, cr) = base(512, 64, 206)
        bx = CTA_CBX if seam else 5
        cb[1, bx] = 0
        cb[1, bx, 0, 0], cb[1, bx, 0, 1] = EDGE[target]
        f = frame(512, 64, [y, cb, cr])
        twin = {32767: 32768, 32768: 32767, -32768: -32769, -32769: -32768}[target]
        return f, Meta(extreme=(1, 1, bx), peak=target, narrow=target in (32768, -32769), twin=_edge_name(twin, seam))
    make.__name__ = _edge_name(target, seam)
    make.__doc__ = ("The int16 edge of the window: the extreme chroma sample of the frame is exactly %d, in column 0 of Cb block "
                    "(1, %d)%s. Beyond int16 the frame is flagged `narrow` and redone by the int32 instance."
                    % (target, CTA_CBX if seam else 5, ", CTA 1's first column and CTA 0's right halo" if seam else ", inside CTA 0's tile"))
    return make


def _edge_name(target, seam):
    return "narrow_%s%d_%s" % ("p" if target > 0 else "m", abs(target), "seam" if seam else "tile")


def _wide(kind, twin):
    """kind: where the block beyond the 32-bit colour range sits (2 x 3 CTAs, 512 x 96):
    right: Cb block (2, 16) (CTA (1, 1)) with column 0 at 491,633: CTA (1, 0)'s right halo. Every sample of CTA (1, 0)'s own
           blocks stays within +-65535 (luma 52,048 under the seam), so only phase 1b's range check gives it 64-bit colour;
    below: Cb block (4, 5) (CTA (2, 0)) with row 0 at 491,633: the line below of CTA (1, 0) (the `only` = 0 branch);
    above: Cb block (1, 5) (CTA (0, 0)) with row 7 at 491,633: the line above of CTA (1, 0) (the `only` = 7 branch);
    luma:  luma block (5, 7) with column 0 at 491,633 and moderate chroma: the per-lane luma guard of reconstruct_tile.
    The twin has an ordinary block in its place."""
    def make():
        rng, (y, cb, cr) = base(512, 96, 207)
        blk = np.zeros((8, 8), dtype=np.int32)
        if kind in ("right", "luma"):
            blk[0, :] = WIDE
        elif kind == "below":
            blk[:, 0] = WIDE
        else:
            blk[:, 0] = WIDE * (-1) ** np.arange(8)
        blk[0, 0] = WIDE_DC
        at = {"right": (1, 2, 16), "below": (1, 4, 5), "above": (1, 1, 5), "luma": (0, 5, 7)}[kind]
        if kind == "right":      # bright luma at luma column 255 (block column 31), block rows 4, 5
            y[4:6, 31, 0, 0] = BRIGHT
            wrap = [(32, 48, 255, 256)]
        elif kind == "below":    # luma row 63 (block row 7), under chroma columns 40 .. 47
            y[7, 10:12, 0, 0] = BRIGHT
            wrap = [(63, 64, 80, 96)]
        elif kind == "above":    # luma row 32 (block row 4)
            y[4, 10:12, 0, 0] = BRIGHT
            wrap = [(32, 33, 80, 96)]
        else:
            wrap = [(40, 48, 56, 57)]
        comps = [y, cb, cr]
        if not twin:
            comps[at[0]][at[1], at[2]] = blk
        f = frame(512, 96, comps)
        return f, Meta(extreme=at, narrow=kind != "luma" and not twin, twin=_wide_name(kind, not twin), wrap_px=[] if twin else wrap)
    make.__name__ = _wide_name(kind, twin)
    make.__doc__ = _wide.__doc__.replace("kind: where", "%s%s: where" % (kind, " (twin)" if twin else ""))
    return make


def _wide_name(kind, twin):
    return "wide_%s%s" % (kind, "_twin" if twin else "")


def _wide_b12(sub, twin):
    def make():
        w, h = 128, 48
        rng, (y, cb, cr) = base(w, h, 208, sub)
        at = (1, 2, 3)
        if not twin:
            cb[2, 3] = 0
            cb[2, 3, 0, :] = WIDE
            cb[2, 3, 0, 0] = WIDE_DC
        y[:, :, 0, 0] = np.where(np.arange(y.shape[1]) >= 2 * sub[0] + 1, BRIGHT, y[:, :, 0, 0])  # luma x >= 24 / 40
        f = frame(w, h, [y, cb, cr], sub)
        x = 8 * 3 * sub[0]
        return f, Meta(extreme=at, narrow=not twin, twin=_b12_name(sub, not twin), wrap_px=[] if twin else [(16, 24, x - 2, x + 8 * sub[0])])
    make.__name__ = _b12_name(sub, twin)
    make.__doc__ = ("b1 + b2 at %s: Cb block (2, 3) with column 0 at 491,633 over bright luma: idct_planes_kernel<int32_t> must "
                    "flag the frame `wide` and reconstruct_kernel<int32_t> take 64-bit colour (reconstruct_tile's MODE 1)%s."
                    % ({(1, 1): "4:4:4", (2, 1): "4:2:2"}[sub], " -- twin: an ordinary block in its place" if twin else ""))
    return make


def _b12_name(sub, twin):
    return "wide_%s%s" % ({(1, 1): "444", (2, 1): "422"}[sub], "_twin" if twin else "")


CASES = {f.__name__: f for f in [seam_cols, seam_rows, seam_corners, skip_rule] + [_sweep(w, h) for w, h in SWEEP] +
         [_edge(t, s) for s in (False, True) for t in (32767, 32768, -32768, -32769)] +
         [_wide(k, t) for k in ("right", "below", "above", "luma") for t in (False, True)] +
         [_wide_b12(s, t) for s in ((1, 1), (2, 1)) for t in (False, True)]}
NAMES = list(CASES)


@functools.lru_cache(maxsize=None)
def _built(name):
    f, m = CASES[name]()
    for c in f.components:
        if ec.idct_peak(c.coef.reshape(-1, 64), 128) >= 2 ** 31 - 2 ** 20:
            raise ValueError("%s: an IDCT intermediate leaves 32-bit arithmetic" % name)
    return f, sw.encode(f), m


def case(name):
    f, data, _ = _built(name)
    return f, data


def meta(name):
    return _built(name)[2]


def subsampling(f):
    return f.components[0].h, f.components[0].v


def with_zeroed(f, sense):
    """The frame with the coefficients `sense` [(component, by, bx, mask)] set to zero, re-encoded."""
    comps = [dataclasses.replace(c, coef=c.coef.copy()) for c in f.components]
    for c, by, bx, mask in sense:
        comps[c].coef[by, bx][mask] = 0
    return sw.encode(dataclasses.replace(f, components=comps, stats={}))


# ---------------------------------------------------------------------------------------------------------------------------
# A plain model of the reference's upsampling and colour stage for sequential 8-bit frames with chroma factors (1 | 2, 1 | 2),
# in int64; the IDCT comes from the oracle (oracle.idct = dct/idct.cpp:226-339).
def sample_planes(oracle, f):
    """[per component int64 [8 bh, 8 bw]]: the IDCT of every block (dcoffset 128), 4 fractional bits."""
    out = []
    for c in f.components:
        q = np.asarray(f.quant[c.tq], dtype=np.uint16).reshape(64)
        bh, bw = c.coef.shape[:2]
        p = np.zeros((8 * bh, 8 * bw), dtype=np.int64)
        for by in range(bh):
            for bx in range(bw):
                p[8 * by:8 * by + 8, 8 * bx:8 * bx + 8] = oracle.idct(c.coef[by, bx].reshape(64), q)
        out.append(p)
    return out


def upsample(p, w, h, cw, ch, sx, sy):
    """Component samples p (true size cw x ch) -> [h, w] at the frame's resolution.
      edge replication dest[-1] = dest[0], dest[cw] = dest[cw - 1] of every line       upsampling/upsamplerbase.cpp:322-323
      VerticalFilterCore<2>: output line 2y leans on line y - 1, 2y + 1 on y + 1, weights 1:3, the rounding (2 / 1) alternates
        with the column; the first / last line is duplicated                            upsampling/upsampler.cpp:100-106, 136-168
      HorizontalFilterCore<2>: in place, in the reference's store order: output 8j + 1 reads the freshly written output 8j + 2
                                                                                         upsampling/upsampler.cpp:283-307 (301-302)
    """
    line = np.concatenate([p[:ch, :1], p[:ch, :cw], p[:ch, cw - 1:cw]], axis=1)  # column cx at cx + 1, cx = -1 .. cw
    if sy == 2:
        yo = np.arange(h)
        cur = yo // 2
        nb = np.where(yo % 2 == 0, np.maximum(cur - 1, 0), np.minimum(cur + 1, ch - 1))
        cx = np.arange(-1, cw + 1)
        rnd = np.where(((cx + 1) & 1)[None, :] == (yo & 1)[:, None], 2, 1)
        v = (line[nb] + 3 * line[cur] + rnd) >> 2
    else:
        v = line[:h]
    if sx == 1:
        return v[:, 1:w + 1]
    xo = np.arange(w)
    c = xo // 2 + 1
    even = (v[:, c - 1] + 3 * v[:, c] + 2) >> 2
    odd = (v[:, c + 1] + 3 * v[:, c] + 1) >> 2
    out = np.where(xo % 2 == 0, even, odd)
    j = xo[xo % 8 == 1]
    c = j // 2 + 1
    new2 = (v[:, c] + 3 * v[:, c + 1] + 2) >> 2
    out[:, j] = (new2 + 3 * v[:, c] + 1) >> 2
    return out


def _wrap32(v):
    return ((v + 2 ** 31) % 2 ** 32) - 2 ** 31


def model(oracle, f, color_transform=True, int32_colour=False):
    """-> [H, W, 3] uint8: the frame's pixels.
      YCbCr -> RGB in 64 bits, 13 fractional bits, + 65536 >> 17, CLAMP(255)  colortrafo/ycbcrtrafo.cpp:842-850, matrix
                                                                               colortransformerfactory.cpp:136-138
      int32_colour: the same sums wrapped to 32 bits (what 32-bit colour arithmetic gives)
      color_transform = False: COLOR_TO_INT (v + 8) >> 4 and CLAMP(255) per component   tools/numerics.hpp:69"""
    sx, sy = subsampling(f)
    planes = sample_planes(oracle, f)
    w, h = f.width, f.height
    cw, ch = _cdiv(w, sx), _cdiv(h, sy)
    yv = planes[0][:h, :w]
    cb, cr = (upsample(p, w, h, cw, ch, sx, sy) for p in planes[1:])
    if not color_transform:
        rgb = [(v + 8) >> 4 for v in (yv, cb, cr)]
    else:
        cb, cr = cb - 2048, cr - 2048
        sums = [yv * 8192 + cr * 11485 + 65536, yv * 8192 - cb * 2819 - cr * 5850 + 65536, yv * 8192 + cb * 14516 + 65536]
        rgb = [(_wrap32(s) if int32_colour else s) >> 17 for s in sums]
    return np.clip(np.stack(rgb, axis=-1), 0, 255).astype(np.uint8)
