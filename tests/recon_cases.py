"""Hand-built frames aimed at the reconstruction paths other than reconstruct420_kernel (libjpeg_b200/csrc/recon_sm100.cu) and at
the 32-bit limits of the IDCT. tests/streamwriter.py writes the frames from chosen quantised coefficients (seeded, deterministic);
every quantiser entry is 1, so the quantised coefficients are the dequantised ones. Shaped like tests/recon420_cases.py, whose
Meta, dense(), reach() and with_zeroed() it reuses.

  Tiled (idct_planes_kernel + reconstruct_kernel: grey, 4:4:4, 4:2:2, 4:4:0). A CTA covers 32 luma block columns x 4 luma block
    rows (256 x 32 pixels): seams at luma block columns 32k - 1 / 32k and rows 4r - 1 / 4r. Lane L of a warp holds luma block
    column 32k + L; it reads its chroma through the warp-uniform `fast` load (load_row_own) when all 32 blocks are visible, else
    per lane (load_row, `interior` or clamped). 4:2:2 lanes also read the chroma columns xl / xr either side of their own four;
    4:4:0 lanes keep three chroma lines (top / cur / bot) and fetch a new one after every odd output line.
  Generic (idct_planes_kernel<int32_t> + generic_reconstruct_kernel / planes_out_kernel): factors 3 and 4, unequal chroma
    factors, a subsampled first component, two and four components, 12 bit.
  IDCT limits: the row pass of the kernels works on the raw coefficients (unpack_row_raw), which is exact only while the
    reference's row pass on 16 x the coefficients stays inside int32; the column pass wraps in 32 bits like the reference's.

case(name) -> (Frame, codestream bytes); meta(name) -> what the case is there for (Meta)."""
import dataclasses
import functools

import numpy as np

from tests import entropy_cases as ec
from tests import recon420_cases as r4
from tests import streamwriter as sw
from tests.recon420_cases import EDGE, WIDE, WIDE_DC, BRIGHT, dense, reach, with_zeroed  # noqa: F401 (re-exported)
from tests.streamwriter import Component, Frame, Scan

CTA_W, CTA_H = 256, 32  # luma pixels per CTA of reconstruct_kernel
TILED = {"grey": [(1, 1)], "444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "440": [(1, 2), (1, 1), (1, 1)]}
# the largest value the reference's row pass takes for coefficients within +-32767 (row_max_block: every output index alike)
ROW_MAX = {8: 2013729264, 12: 2139558384}
# ... and for any int16 coefficients (a dequantised -32768 where a weight is negative): reached at output 1, still below 2^31
INT16_ROW_MAX = {8: 2013768208, 12: 2139597328}


@dataclasses.dataclass
class Meta(r4.Meta):
    rowmax: list = dataclasses.field(default_factory=list)  # [(component, by, bx, output index)]: row 0 attains the bound
    colwrap: bool = False                                    # some block's column pass leaves int32 (and wraps)


def _cdiv(a, b):
    return -(-a // b)


def grids(w, h, factors):
    """[(bh, bw)] of every component over the MCU-padded grid"""
    hmax, vmax = max(f[0] for f in factors), max(f[1] for f in factors)
    mcx, mcy = _cdiv(w, 8 * hmax), _cdiv(h, 8 * vmax)
    return [(mcy * v, mcx * hh) for hh, v in factors]


def frame(w, h, comps, factors, precision=8):
    """Sequential, every quantiser entry 1, component 0 on table slot 0 and the others on slot 1. One interleaved scan while an
    MCU has at most 10 blocks, else one scan per component (whose blocks outside the component's own grid are zeroed)."""
    n = len(comps)
    slot = [min(c, 1) for c in range(n)]
    if n == 1 or sum(a * b for a, b in factors) <= 10:
        scans = [Scan(list(range(n)), slot, slot)]
    else:
        scans = [Scan([c], [slot[c]], [slot[c]]) for c in range(n)]
    f = Frame(w, h, [Component(comps[c], factors[c][0], factors[c][1], slot[c]) for c in range(n)], {0: r4.ONES, 1: r4.ONES},
              scans, dict(r4.TABLES), precision)
    if len(scans) > 1:
        for (bw, bh), c in zip(sw.geometry(f)[4], f.components):
            c.coef[bh:] = 0
            c.coef[:, bw:] = 0
    return f


def base(w, h, seed, factors):
    """Component 0 near mid-grey, the others sparse and low-frequency, over the MCU-padded grids (padding included)."""
    rng = np.random.default_rng(seed)
    return rng, [(r4._luma if c == 0 else r4._chroma)(rng, bh, bw) for c, (bh, bw) in enumerate(grids(w, h, factors))]


def _mask(rows=range(8), cols=range(8)):
    return r4._mask(rows, cols)


def subsampling(f):
    """(subx, suby) per component: the factor by which it is subsampled"""
    hmax, vmax = max(c.h for c in f.components), max(c.v for c in f.components)
    return [hmax // c.h for c in f.components], [vmax // c.v for c in f.components]


def path(f):
    """The reconstruction path of the frame (abi.cpp recon_path): 'Fused420', 'Tiled' or 'Generic'"""
    fac = [(c.h, c.v) for c in f.components]
    if f.precision != 8:
        return "Generic"
    if len(fac) == 1:
        return "Tiled"
    if len(fac) != 3 or fac[1] != fac[2] or fac[1] != (1, 1) or fac[0] not in ((1, 1), (2, 1), (1, 2), (2, 2)):
        return "Generic"
    return "Fused420" if fac[0] == (2, 2) else "Tiled"


# ---- the reference's integer IDCT in Python ---------------------------------------------------------------------------------
def _pass(x):
    """the 8 outputs of one 8-point pass (dct/idct.cpp:237-334, idct8t) in front of their rounding, exact int64 over [..., 8]"""
    z1 = (x[..., 2] + x[..., 6]) * 277
    t2, t3 = z1 - x[..., 6] * 946, z1 + x[..., 2] * 392
    a10, a13 = ((x[..., 0] + x[..., 4]) << 9) + t3, ((x[..., 0] + x[..., 4]) << 9) - t3
    a11, a12 = ((x[..., 0] - x[..., 4]) << 9) + t2, ((x[..., 0] - x[..., 4]) << 9) - t2
    o0, o1, o2, o3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z5 = (o0 + o2 + o1 + o3) * 602
    z1o, z2 = (o0 + o3) * -461, (o1 + o2) * -1312
    z3, z4 = (o0 + o2) * -1004 + z5, (o1 + o3) * -200 + z5
    e0, e1, e2, e3 = o0 * 153 + z1o + z3, o1 * 1051 + z2 + z4, o2 * 1573 + z2 + z3, o3 * 769 + z1o + z4
    return np.stack([a10 + e3, a11 + e2, a12 + e1, a13 + e0, a13 - e0, a12 - e1, a11 - e2, a10 - e3], axis=-1)


def _wrap32(v):
    return ((v + 2 ** 31) % 2 ** 32) - 2 ** 31


def row_weights():
    """W [8 outputs, 8 inputs]: one pass of idct8t is the linear map x -> W x in front of its rounding"""
    return _pass(np.eye(8, dtype=np.int64)).T


def row_pass_sums(deq, dcoffset):
    """[n, 8 rows, 8 outputs]: the reference's row pass sums (16 x the coefficients, dcoffset << 7 on the DC, + 256) in int64"""
    x = np.asarray(deq, dtype=np.int64).reshape(-1, 8, 8) * 16
    x[:, 0, 0] += dcoffset << 7
    return _pass(x) + 256


def idct(deq, dcoffset, wrap=True):
    """[n, 8, 8] samples of the reference's IDCT (oracle.idct) for the dequantised raster blocks deq [n, 64]; wrap=False: the
    same arithmetic in 64 bits, what the IDCT gives where nothing wraps"""
    w = _wrap32 if wrap else (lambda v: v)
    rows = w(row_pass_sums(deq, dcoffset)) >> 9
    return np.swapaxes(w(_pass(np.swapaxes(rows, 1, 2)) + 2048) >> 12, 1, 2)


def row_max_block(i, precision):
    """The block whose row 0 gives output i of the row pass its largest value: DC 32767, every AC coefficient of the row 32767
    with the sign of its weight. -> (8x8 block, that value)"""
    wts = row_weights()[i]
    blk = np.zeros((8, 8), dtype=np.int32)
    blk[0] = 32767 * np.where(wts < 0, -1, 1)
    blk[0, 0] = 32767
    dcoffset = 1 << (precision - 1)
    bound = 16 * (int(np.abs(wts).sum()) * 32767 + 512 * (dcoffset << 3)) + 256
    return blk, bound


def wrapping_block(rng, dcoffset):
    """All 64 coefficients large (|v| 12,000 .. 32,767, DC within +-16,000): column-pass sums far beyond int32, and samples that
    differ from the 64-bit IDCT's"""
    while True:
        b = rng.integers(12000, 32768, (8, 8)) * np.where(rng.random((8, 8)) < 0.5, -1, 1)
        b[0, 0] = rng.integers(-16000, 16001)
        if not np.array_equal(idct(b.reshape(1, 64), dcoffset), idct(b.reshape(1, 64), dcoffset, wrap=False)):
            return b.astype(np.int32)


# ---- Tiled ------------------------------------------------------------------------------------------------------------------
def _tile_blocks(fmt):
    """(block columns, block rows) of component 1 (grey: 0) under one CTA"""
    sx, sy = TILED[fmt][0] if fmt != "grey" else (1, 1)
    return 32 // sx, 4 // sy


def _seams(fmt, w, h, seed, edge=False):
    """Dense blocks in every chroma component (grey: luma) at the CTA seams (block columns / rows TW k - 1, TW k); edge: also in
    the last block column and row of the visible frame and the padded grid."""
    factors = TILED[fmt]
    rng, comps = base(w, h, seed, factors)
    tw, th = _tile_blocks(fmt)
    targets = comps[1:] if len(comps) > 1 else comps
    bh, bw = targets[0].shape[:2]
    sc = [c for k in range(1, _cdiv(bw, tw)) for c in (tw * k - 1, tw * k) if c < bw]
    sr = [r for k in range(1, _cdiv(bh, th)) for r in (th * k - 1, th * k) if r < bh]
    if edge:
        sx, sy = (factors[0] if len(comps) > 1 else (1, 1))
        vis_c, vis_r = _cdiv(_cdiv(w, sx), 8), _cdiv(_cdiv(h, sy), 8)
        sc = sorted(set(sc) | {vis_c - 1, bw - 1})
        sr = sorted(set(sr) | {vis_r - 1, bh - 1})
    for comp in targets:
        for by in range(bh):
            for bx in range(bw):
                if bx in sc or by in sr:
                    comp[by, bx] = dense(rng, cols=bx in sc, rows=by in sr)
    return comps, sc, sr


def _seam(fmt):
    def make():
        w, h = 3 * CTA_W, 3 * CTA_H
        comps, sc, sr = _seams(fmt, w, h, 301 + len(fmt) + sum(map(ord, fmt)))
        f = frame(w, h, comps, TILED[fmt])
        tw, th = _tile_blocks(fmt)
        cs = [1, 2] if fmt != "grey" else [0]
        m = Meta()
        if fmt == "422":    # coefficient columns 5 .. 7 of chroma block column 16k - 1 reach luma column 256k only as tile k's xl
            left = [c for c in sc if c % tw == tw - 1]
            m.sense = [(c, by, bx, _mask(cols=range(5, 8))) for c in cs for by in range(comps[1].shape[0]) for bx in left]
            m.sense_px, m.sense_min = [(0, h, 16 * (bx + 1), 16 * (bx + 1) + 1) for bx in left], 100
        elif fmt == "440":  # coefficient rows 5 .. 7 of chroma block row 2r - 1 reach luma row 32r only as tile r's line above
            above = [r for r in sr if r % th == th - 1]
            m.sense = [(c, by, bx, _mask(rows=range(5, 8))) for c in cs for by in above for bx in range(comps[1].shape[1])]
            m.sense_px, m.sense_min = [(16 * (by + 1), 16 * (by + 1) + 1, 0, w) for by in above], 300
        else:               # the blocks either side of every seam: the first / last lane and warp of a CTA
            first = [c for c in sc if c % tw == 0]
            m.sense = [(c, by, bx, _mask()) for c in cs for by in (0, 5) for bx in first]
            m.sense_px = [r for bx in first for r in (reach(f, cs[0], 0, bx), reach(f, cs[0], 5, bx))]
            m.sense_min = 100
        return f, m
    make.__name__ = "seam_%s" % fmt
    make.__doc__ = ("%s, 3 x 3 CTAs: dense blocks at every CTA seam (block columns 32k - 1 / 32k, rows 4r - 1 / 4r of the luma "
                    "grid) in the chroma components (grey: luma)." % fmt)
    return make


SWEEP = {
    "grey": [(513, 33), (767, 95), (1, 97), (769, 7)],
    "444": [(514, 66), (513, 33), (767, 95), (1, 97), (769, 1)],
    "422": [(532, 70), (513, 33), (766, 95), (2, 97), (769, 9)],
    "440": [(515, 67), (512, 65), (767, 95), (9, 129), (769, 2)],
}


def _sweep(fmt, w, h):
    def make():
        comps, _, _ = _seams(fmt, w, h, 305 + w + h, edge=True)
        return frame(w, h, comps, TILED[fmt]), Meta()
    make.__name__ = "sweep_%s_%dx%d" % (fmt, w, h)
    make.__doc__ = ("%s, %d x %d: partial CTAs and warps (the per-lane load in place of the `fast` one), odd chroma sizes, "
                    "dense blocks at the seams and at the last visible and the last padded block column / row, where the "
                    "MCU-padded chroma grid is wider than the visible chroma." % (fmt, w, h))
    return make


def _edge_name(fmt, target, seam):
    return "narrow_%s_%s%d_%s" % (fmt, "p" if target > 0 else "m", abs(target), "seam" if seam else "tile")


def _edge(fmt, target, seam):
    def make():
        w, h = 2 * CTA_W, 2 * CTA_H
        rng, comps = base(w, h, 306, TILED[fmt])
        bx = _tile_blocks(fmt)[0] if seam else 5
        comps[1][1, bx] = 0
        comps[1][1, bx, 0, 0], comps[1][1, bx, 0, 1] = EDGE[target]
        twin = {32767: 32768, 32768: 32767, -32768: -32769, -32769: -32768}[target]
        return frame(w, h, comps, TILED[fmt]), Meta(extreme=(1, 1, bx), peak=target, narrow=target in (32768, -32769),
                                                   twin=_edge_name(fmt, twin, seam))
    make.__name__ = _edge_name(fmt, target, seam)
    make.__doc__ = ("%s: the extreme chroma sample of the frame is exactly %d, in column 0 of Cb block (1, %s)%s." %
                    (fmt, target, "first of CTA 1" if seam else "5", " (CTA 1's first column)" if seam else ""))
    return make


# where the block beyond the 32-bit colour range sits, and the pixels whose 32-bit colour wraps
WIDE_AT = {
    ("422", "xr"): ((1, 2, 16), [(16, 24, 255, 256)]),    # chroma column 128: CTA 0's last lane reads it as xr only
    ("422", "xl"): ((1, 2, 15), [(16, 24, 256, 257)]),    # chroma column 127: CTA 1's first lane reads it as xl only
    ("440", "below"): ((1, 2, 5), [(31, 32, 40, 48)]),    # chroma line 16: CTA row 0's last output line leans on it (bot)
    ("440", "above"): ((1, 1, 5), [(32, 33, 40, 48)]),    # chroma line 15: CTA row 1's first output line leans on it (top)
    ("444", "luma"): ((0, 2, 7), [(16, 24, 56, 57)]),
    ("422", "luma"): ((0, 2, 7), [(16, 24, 56, 57)]),
    ("440", "luma"): ((0, 2, 7), [(16, 24, 56, 57)]),
}


def _wide_name(fmt, kind, twin):
    return "wide_%s_%s%s" % (fmt, kind, "_twin" if twin else "")


def _wide(fmt, kind, twin):
    def make():
        w, h = 2 * CTA_W, 2 * CTA_H
        rng, comps = base(w, h, 307, TILED[fmt])
        at, wrap = WIDE_AT[(fmt, kind)]
        blk = np.zeros((8, 8), dtype=np.int32)
        if kind in ("xr", "luma"):    # sample column 0
            blk[0, :] = WIDE
        elif kind == "xl":            # sample column 7
            blk[0, :] = WIDE * (-1) ** np.arange(8)
        elif kind == "below":         # sample row 0
            blk[:, 0] = WIDE
        else:                         # sample row 7
            blk[:, 0] = WIDE * (-1) ** np.arange(8)
        blk[0, 0] = WIDE_DC
        y0, y1, x0, x1 = wrap[0]
        comps[0][y0 // 8:_cdiv(y1, 8), x0 // 8:_cdiv(x1, 8), 0, 0] = BRIGHT
        if not twin:
            comps[at[0]][at[1], at[2]] = blk
        f = frame(w, h, comps, TILED[fmt])
        return f, Meta(extreme=at, narrow=kind != "luma" and not twin, twin=_wide_name(fmt, kind, not twin),
                       wrap_px=[] if twin else wrap)
    make.__name__ = _wide_name(fmt, kind, twin)
    make.__doc__ = ("%s: a block with one sample line near 491,000 (%s) over bright luma: 64-bit colour%s."
                    % (fmt, kind, " -- twin: an ordinary block in its place" if twin else ""))
    return make


def grey_beyond_int16():
    """Grey (the NC == 1 branch of reconstruct_tile): luma samples near +-491,000 in blocks at a seam, saturating both ways."""
    w, h = 2 * CTA_W, CTA_H
    rng, (y,) = base(w, h, 308, TILED["grey"])
    for bx, s in ((31, 1), (32, 1), (40, -1)):
        y[1, bx] = 0
        y[1, bx, 0, :] = s * WIDE
        y[1, bx, 0, 0] = s * WIDE_DC
    return frame(w, h, [y], TILED["grey"]), Meta(extreme=(0, 1, 31))


# ---- Generic ----------------------------------------------------------------------------------------------------------------
GENERIC = {
    "31": [(3, 1), (1, 1), (1, 1)], "13": [(1, 3), (1, 1), (1, 1)], "411": [(4, 1), (1, 1), (1, 1)],
    "14": [(1, 4), (1, 1), (1, 1)], "410": [(4, 2), (1, 1), (1, 1)], "33": [(3, 3), (1, 1), (1, 1)],
    "44": [(4, 4), (1, 1), (1, 1)], "32": [(3, 2), (1, 1), (1, 1)],
    "first_sub": [(1, 1), (2, 2), (2, 2)], "first_sub_mixed": [(1, 2), (2, 2), (2, 1)], "unequal": [(2, 2), (1, 1), (2, 1)],
    "two_11": [(1, 1), (1, 1)], "two_21": [(2, 2), (1, 1)],
    "four_11": [(1, 1)] * 4, "four_own": [(2, 2), (1, 1), (1, 1), (2, 1)],
}
GENERIC_SIZES = {"31": [(511, 13), (515, 29)], "13": [(509, 31)], "411": [(513, 17)], "14": [(35, 70)], "410": [(514, 35)],
                 "33": [(517, 50)], "44": [(520, 65)], "32": [(100, 37)], "first_sub": [(513, 33)], "first_sub_mixed": [(97, 61)],
                 "unequal": [(130, 41)], "two_11": [(513, 20)], "two_21": [(99, 35)], "four_11": [(515, 19)],
                 "four_own": [(133, 47)]}


def _generic(layout, w, h):
    def make():
        factors = GENERIC[layout]
        rng, comps = base(w, h, 309 + w + 3 * h, factors)
        for c in comps[1:]:  # every component its own content: a dense block in each, at a different place
            bh, bw = c.shape[:2]
            c[rng.integers(0, bh), rng.integers(0, bw)] = dense(rng, True, True)
        return frame(w, h, comps, factors), Meta()
    make.__name__ = "generic_%s_%dx%d" % (layout, w, h)
    make.__doc__ = "Generic path, factors %s, %d x %d" % (GENERIC[layout], w, h)
    return make


def _deep_wide(sub, twin):
    def make():
        w, h = 96, 40
        factors = [sub, (1, 1), (1, 1)]
        rng, comps = base(w, h, 310, factors)
        if not twin:
            comps[1][1, 2] = 0
            comps[1][1, 2, 0, :] = WIDE
            comps[1][1, 2, 0, 0] = WIDE_DC
        f = frame(w, h, comps, factors, precision=12)
        return f, Meta(extreme=(1, 1, 2), narrow=not twin, twin=_deep_name(sub, not twin))
    make.__name__ = _deep_name(sub, twin)
    make.__doc__ = "12 bit, Y %s: a Cb block with sample column 0 near 491,000 (beyond +-65535) over bright luma" % (sub,)
    return make


def _deep_name(sub, twin):
    return "deep12_wide_%d%d%s" % (sub[0], sub[1], "_twin" if twin else "")


# ---- IDCT limits ------------------------------------------------------------------------------------------------------------
def _rowmax(precision):
    def make():
        w, h = 128, 16
        factors = TILED["444"]
        rng, comps = base(w, h, 311 + precision, factors)
        m = Meta(narrow=True)
        for c in comps[:2]:  # DC differences to the blocks with DC 32767 stay within category 15
            c[..., 0, 0] = 0
        for i in range(8):
            blk, _ = row_max_block(i, precision)
            comps[0][0, 2 * i] = blk
            comps[1][1, 2 * i + 1] = blk
            m.rowmax += [(0, 0, 2 * i, i), (1, 1, 2 * i + 1, i)]
        return frame(w, h, comps, factors, precision), m
    make.__name__ = "rowmax_%d" % precision
    make.__doc__ = ("%d bit 4:4:4: for every output index i of the row pass, a luma and a Cb block whose row 0 gives it the "
                    "largest value int16 coefficients allow (DC 32767, the AC signs of its weights)" % precision)
    return make


COLWRAP = {"420": ([(2, 2), (1, 1), (1, 1)], 8), "444": ([(1, 1)] * 3, 8), "411": ([(4, 1), (1, 1), (1, 1)], 8),
           "grey": ([(1, 1)], 8), "422_12": ([(2, 1), (1, 1), (1, 1)], 12)}


def _colwrap(kind):
    def make():
        factors, precision = COLWRAP[kind]
        w, h = 2 * CTA_W + 24, 40
        rng, comps = base(w, h, 312 + len(kind), factors)
        dco = 1 << (precision - 1)
        for c in comps:
            bh, bw = c.shape[:2]
            for by, bx in {(0, 0), (1, bw // 2 - 1), (1, bw // 2), (bh - 1, bw - 1), (2 % bh, 16 % bw), (2 % bh, 15 % bw)}:
                c[by, bx] = wrapping_block(rng, dco)
        return frame(w, h, comps, factors, precision), Meta(colwrap=True, narrow=len(comps) > 1)
    make.__name__ = "colwrap_%s" % kind
    make.__doc__ = ("%s: dense blocks whose column-pass sums leave int32 in every component, at the corners, the CTA seams "
                    "and the middle: the samples are the reference's 32-bit wrap" % kind)
    return make


CASES = {f.__name__: f for f in
         [_seam(k) for k in TILED] + [_sweep(k, w, h) for k in TILED for w, h in SWEEP[k]] +
         [_edge(k, t, s) for k in ("444", "422", "440") for s in (False, True) for t in (32767, 32768, -32768, -32769)] +
         [_wide(k, kind, t) for (k, kind) in WIDE_AT for t in (False, True)] + [grey_beyond_int16] +
         [_generic(lay, w, h) for lay in GENERIC for w, h in GENERIC_SIZES[lay]] +
         [_deep_wide(s, t) for s in ((1, 1), (2, 2)) for t in (False, True)] +
         [_rowmax(8), _rowmax(12)] + [_colwrap(k) for k in COLWRAP]}
NAMES = list(CASES)


@functools.lru_cache(maxsize=None)
def _built(name):
    f, m = CASES[name]()
    if not m.colwrap:
        for c in f.components:
            if ec.idct_peak(c.coef.reshape(-1, 64), 1 << (f.precision - 1)) >= 2 ** 31 - 2 ** 20:
                raise ValueError("%s: an IDCT intermediate leaves 32-bit arithmetic" % name)
    return f, sw.encode(f), m


def case(name):
    f, data, _ = _built(name)
    return f, data


def meta(name):
    return _built(name)[2]
