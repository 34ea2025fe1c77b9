"""Hand-built progressive (SOF2) frames for both GPU decode paths: the component-fused kernels (progfused_sm100.cu) and the
scan-by-scan kernels (progressive_sm100.cu). Every case is seeded and names the path the batch planner must give it: "fused"
takes the scripts whose scans are interleaved DC scans of all components or single-component AC scans, at most kPfMaxScans (6)
per group, restart intervals equal within a group; "scan" takes the rest. tests/progressive_model.py says what each frame must
decode to; tests/golden/progressive_cases/ holds what the reference decoder made of each stream.

  scripts     libjpeg's jpeg_simple_progression, DC-only frames, a component without AC scans, non-interleaved DC scans, seven
              AC scans of one component, successive approximation from Al = 13 down to 0 on 8- and 12-bit frames, a DRI
              changed between scans and the same DRI sent again
  geometry    grey, 4:4:4, 4:2:2, 4:2:0, 3x and 4x factors, sizes whose MCU-padded grid exceeds the component grids
  symbols     EOB runs that end at a restart boundary, ZRL followed by correction bits, refinement symbols of sizes 2..15
  quantisers  a DQT redefined between scans (one slot shared by components that first appear in different scans), 16-bit DQT
  int16 edge  DC first pass, DC refinement, AC first pass, AC refinement (correction and new coefficient) and the fused path's
              level x (q << Al) product: coefficients exactly at -32768 / 32767 and one step beyond
  refused     q << Al >= 2^24
"""
import functools

import numpy as np

from tests import entropy_cases as ec
from tests import streamwriter as sw
from tests.streamwriter import Component, Frame, Scan

ZZ = sw.ZIGZAG

PROG_AC_ALL = ec.PROG_AC_FIRST + [(r << 4) | 15 for r in range(16)]  # with size 15: +-32767 at Al 0
PROG_REFINE_ODD = ec.PROG_REFINE + list(range(2, 16))  # run 0, sizes 2..15: sizes refinement scans do not define


def _counts_table(syms):
    return sw.table_from_counts({s: 1 + (s % 7) for s in syms})


def _tables(dc_slots=(0,), ac_slots=(0,)):
    t = {("dc", s): _counts_table(ec.DC_ALL) for s in dc_slots}
    t.update({("ac", s): _counts_table(PROG_AC_ALL) for s in ac_slots})
    return t


def _refine_tables(ac_slots=(0,), odd=False):
    return {("ac", s): _counts_table(PROG_REFINE_ODD if odd else ec.PROG_REFINE) for s in ac_slots}


def _coef(rng, bh, bw, density=0.3, max_size=7, dc=300, own=None):
    c = ec.sparse(rng, bh, bw, density=density, max_size=max_size, dc=dc)
    if own is not None:  # blocks outside the component's own grid are never coded by its AC scans: zero there
        obw, obh = own
        c[obh:] = 0
        c[:, obw:] = 0
    return c.astype(np.int64)


def _components(rng, w, h, factors, tq=None, **kw):
    hmax = max(f[0] for f in factors)
    vmax = max(f[1] for f in factors)
    mcx, mcy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    comps = []
    for i, (fh, fv) in enumerate(factors):
        own = (-(-(-(-w * fh) // hmax) // 8), -(-(-(-h * fv) // vmax) // 8))  # the component's own block grid
        comps.append(Component(_coef(rng, mcy * fv, mcx * fh, own=own, **kw), fh, fv, (tq or [0, 1, 1, 1])[i]))
    return comps


def _quant(rng, slots, lo=1, hi=6):
    return {s: rng.integers(lo, hi, 64) for s in slots}


def _simple_script(nc, dc_td):
    """libjpeg's jpeg_simple_progression (jcparam.c) for 1 or 3 components: DC Al 1, luma 1-5 Al 2, chroma 1-63 Al 1, luma 6-63
    Al 2, luma 1-63 refinement to Al 1, DC refinement, chroma refinements, luma refinement to Al 0"""
    all_ = list(range(nc))
    dc_t = _tables(dc_slots=sorted(set(dc_td)), ac_slots=())
    if nc == 1:
        return [Scan([0], [0], [0], 0, 0, 0, 1, dc_t), Scan([0], [0], [0], 1, 5, 0, 2, _tables((), (0,))), Scan([0], [0], [0], 6, 63, 0, 2),
                Scan([0], [0], [0], 1, 63, 2, 1, _refine_tables()), Scan([0], [0], [0], 0, 0, 1, 0), Scan([0], [0], [0], 1, 63, 1, 0)]
    return [Scan(all_, dc_td, [0] * nc, 0, 0, 0, 1, dc_t),
            Scan([0], [0], [0], 1, 5, 0, 2, _tables((), (0, 1))),
            Scan([2], [0], [1], 1, 63, 0, 1), Scan([1], [0], [1], 1, 63, 0, 1),
            Scan([0], [0], [0], 6, 63, 0, 2),
            Scan([0], [0], [0], 1, 63, 2, 1, _refine_tables((0, 1))),
            Scan(all_, dc_td, [0] * nc, 0, 0, 1, 0),
            Scan([2], [0], [1], 1, 63, 1, 0), Scan([1], [0], [1], 1, 63, 1, 0), Scan([0], [0], [0], 1, 63, 1, 0)]


# ---- scripts and geometry ------------------------------------------------------------------------------------------------
def simple_420_37x21(seed):
    rng = np.random.default_rng(seed)
    comps = _components(rng, 37, 21, [(2, 2), (1, 1), (1, 1)])
    return Frame(37, 21, comps, _quant(rng, (0, 1)), _simple_script(3, [0, 1, 1]), progressive=True)


def simple_444_rst_45x30(seed):
    rng = np.random.default_rng(seed)
    comps = _components(rng, 45, 30, [(1, 1)] * 3, density=0.15)
    return Frame(45, 30, comps, _quant(rng, (0, 1)), _simple_script(3, [0, 1, 1]), restart_interval=3, progressive=True)


def simple_422_50x17(seed):
    rng = np.random.default_rng(seed)
    comps = _components(rng, 50, 17, [(2, 1), (1, 1), (1, 1)])
    return Frame(50, 17, comps, _quant(rng, (0, 1)), _simple_script(3, [0, 1, 1]), progressive=True)


def simple_grey_29x19(seed):
    rng = np.random.default_rng(seed)
    comps = _components(rng, 29, 19, [(1, 1)], dc=900)
    return Frame(29, 19, comps, _quant(rng, (0,)), _simple_script(1, [0]), progressive=True)


def factors_3x_4x_61x47(seed):
    """luma sampled 3 x 1 against 1 x 1 chroma"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 61, 47, [(3, 1), (1, 1), (1, 1)])
    return Frame(61, 47, comps, _quant(rng, (0, 1)), _simple_script(3, [0, 1, 1]), progressive=True)


def factors_4x4_70x40(seed):
    rng = np.random.default_rng(seed)
    comps = _components(rng, 70, 40, [(4, 4), (1, 1), (1, 1)], density=0.1)
    return Frame(70, 40, comps, _quant(rng, (0, 1)), _simple_script(3, [0, 1, 1]), restart_interval=2, progressive=True)


def dc_only_grey_13x9(seed):
    """no AC scans at all: DC first pass at Al 2, two refinements, negative DCs; the DC kernel completes every block"""
    rng = np.random.default_rng(seed)
    coef = np.zeros((2, 2, 8, 8), dtype=np.int64)
    coef[..., 0, 0] = rng.integers(-700, 700, size=(2, 2))
    coef[0, 0, 0, 0] = -1
    scans = [Scan([0], [0], [0], 0, 0, 0, 2, _tables((0,), ())), Scan([0], [0], [0], 0, 0, 2, 1), Scan([0], [0], [0], 0, 0, 1, 0)]
    return Frame(13, 9, [Component(coef)], _quant(rng, (0,)), scans, progressive=True)


def chroma_without_ac_422(seed):
    """4:2:2 whose chroma components have no AC scans: their blocks are the DC alone"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 40, 24, [(2, 1), (1, 1), (1, 1)])
    for c in comps[1:]:
        c.coef[..., 1:] = 0
        c.coef[..., 1:, 0] = 0
    scans = [Scan([0, 1, 2], [0, 1, 1], [0, 0, 0], 0, 0, 0, 0, _tables((0, 1), ())), Scan([0], [0], [0], 1, 63, 0, 0, _tables((), (0,)))]
    return Frame(40, 24, comps, _quant(rng, (0, 1)), scans, progressive=True)


def noninterleaved_dc_444(seed):
    """every DC scan holds one component: the scan-by-scan path"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 24, 16, [(1, 1)] * 3)
    t = _tables((0,), (0,))
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, t), Scan([1], [0], [0], 0, 0, 0, 0), Scan([2], [0], [0], 0, 0, 0, 0)]
    scans += [Scan([c], [0], [0], 1, 63, 0, 0) for c in range(3)]
    return Frame(24, 16, comps, _quant(rng, (0, 1)), scans, progressive=True)


def seven_ac_scans_grey(seed):
    """seven AC scans of one component, one more than the fused AC kernel carries"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 32, 24, [(1, 1)], density=0.5, max_size=9)
    bands = [(1, 2), (3, 5), (6, 9), (10, 20), (21, 35), (36, 50), (51, 63)]
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), (0,)))] + [Scan([0], [0], [0], a, b, 0, 0) for a, b in bands]
    return Frame(32, 24, comps, _quant(rng, (0,)), scans, progressive=True)


def _deep(seed, precision, dc_scale, ac_max):
    """DC from Al 13 down to 0 one bit per scan, the AC band once at Al 0, negative DCs: fifteen scans"""
    rng = np.random.default_rng(seed)
    coef = np.zeros((2, 3, 8, 8), dtype=np.int64)
    coef[..., 0, 0] = rng.integers(-dc_scale, dc_scale, size=(2, 3))
    coef[0, 0, 0, 0], coef[0, 1, 0, 0] = -dc_scale, dc_scale - 1
    for by in range(2):
        for bx in range(3):
            for k in rng.choice(np.arange(1, 64), 6, replace=False):
                coef[by, bx].reshape(64)[ZZ[k]] = int(rng.integers(-ac_max, ac_max + 1))
    scans = [Scan([0], [0], [0], 0, 0, 0, 13, _tables((0,), ()))]
    scans += [Scan([0], [0], [0], 0, 0, a + 1, a) for a in range(12, -1, -1)]
    scans += [Scan([0], [0], [0], 1, 63, 0, 0, _tables((), (0,)))]
    return Frame(24, 16, [Component(coef)], {0: np.ones(64, dtype=np.int64)}, scans, precision=precision, progressive=True)


def deep_sa_8bit(seed):
    return _deep(seed, 8, 2040, 600)


def deep_sa_12bit(seed):
    return _deep(seed, 12, 16380, 9000)


def deep_ac_sa_grey(seed):
    """the AC band from Al 5 down to 0 (one first pass, five refinements), DC in one pass: six AC scans, the fused limit"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 24, 24, [(1, 1)], density=0.4, max_size=9)
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), ())), Scan([0], [0], [0], 1, 63, 0, 5, _tables((), (0,)))]
    scans += [Scan([0], [0], [0], 1, 63, a + 1, a, _refine_tables() if a == 4 else {}) for a in range(4, -1, -1)]
    return Frame(24, 24, comps, _quant(rng, (0,)), scans, progressive=True)


def dri_changed_between_scans(seed):
    """restart interval 2 for the DC scan, 3 and then none for the AC scans"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 40, 32, [(1, 1)], density=0.2)
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), ()), restart_interval=2),
             Scan([0], [0], [0], 1, 9, 0, 0, _tables((), (0,)), restart_interval=3), Scan([0], [0], [0], 10, 63, 0, 0, restart_interval=0)]
    return Frame(40, 32, comps, _quant(rng, (0,)), scans, progressive=True)


def dri_resent_same(seed):
    """the same DRI in front of every scan"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 40, 32, [(2, 2), (1, 1), (1, 1)], density=0.2)
    scans = _simple_script(3, [0, 1, 1])
    for s in scans:
        s.restart_interval = 2
    return Frame(40, 32, comps, _quant(rng, (0, 1)), scans, restart_interval=2, progressive=True)


# ---- symbols ---------------------------------------------------------------------------------------------------------------
def eobrun_at_restart(seed):
    """restart interval 4 with the AC band of blocks 0..3, 4..7 and 12..15 all zero: EOB runs of exactly one interval, ended by
    the restart marker, and a refinement scan whose runs end there too"""
    rng = np.random.default_rng(seed)
    coef = _coef(rng, 2, 8, density=0.3).reshape(16, 8, 8)
    coef[0:8, :, :][:, 1:, :] = 0
    coef[0:8, 0, 1:] = 0
    coef[12:16, 1:, :] = 0
    coef[12:16, 0, 1:] = 0
    coef = coef.reshape(2, 8, 8, 8)
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), ())), Scan([0], [0], [0], 1, 63, 0, 1, _tables((), (0,))),
             Scan([0], [0], [0], 1, 63, 1, 0, _refine_tables())]
    return Frame(64, 16, [Component(coef)], _quant(rng, (0,)), scans, restart_interval=4, progressive=True)


def zrl_then_correction(seed):
    """refinement runs longer than 16 zeros that pass coefficients already significant: ZRL symbols followed by the correction
    bits of the positions they passed"""
    rng = np.random.default_rng(seed)
    coef = np.zeros((2, 2, 8, 8), dtype=np.int64)
    for b, blk in enumerate(coef.reshape(4, 8, 8)):
        blk[0, 0] = int(rng.integers(-50, 50))
        f = blk.reshape(64)
        f[ZZ[3 + b]] = int(rng.choice([-3, -2, 2, 3]))       # significant after the first pass
        f[ZZ[12 + b]] = int(rng.choice([-3, 3]))
        f[ZZ[40 + 3 * b]] = int(rng.choice([-1, 1]))         # newly significant at the refinement, 20+ zeros behind
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), ())), Scan([0], [0], [0], 1, 63, 0, 1, _tables((), (0,))),
             Scan([0], [0], [0], 1, 63, 1, 0, _refine_tables())]
    return Frame(16, 16, [Component(coef)], _quant(rng, (0,)), scans, progressive=True)


def refine_odd_sizes(seed):
    """every refinement size 2..15 once, on blocks 0..13 of the scan"""
    rng = np.random.default_rng(seed)
    coef = _coef(rng, 2, 8, density=0.3)
    coef.reshape(16, 64)[:, ZZ[1]] = 0  # position 1 stays zero: the odd symbol passes it
    scans = [Scan([0], [0], [0], 0, 0, 0, 0, _tables((0,), ())), Scan([0], [0], [0], 1, 63, 0, 1, _tables((), (0,))),
             Scan([0], [0], [0], 1, 63, 1, 0, _refine_tables(odd=True), odd_sizes={i: 2 + i for i in range(14)})]
    return Frame(64, 16, [Component(coef)], _quant(rng, (0,)), scans, progressive=True)


# ---- quantisers --------------------------------------------------------------------------------------------------------------
def dqt_redefined_fused(seed):
    """both slots redefined behind the DC scan and again in the middle of the AC scans: the AC scans must keep the tables of
    the DC scan, where each component first appears"""
    rng = np.random.default_rng(seed)
    f = simple_420_37x21(seed)
    f.scans[1].quant = _quant(rng, (0, 1), 7, 40)
    f.scans[4].quant = _quant(rng, (0,), 7, 40)
    f.scans[7].quant = _quant(rng, (1,), 7, 40)
    return f


def dqt_redefined_scan(seed):
    """non-interleaved DC scans with slot 1 redefined between the scans of Cb and Cr: the two components of the slot latch
    different tables"""
    rng = np.random.default_rng(seed)
    f = noninterleaved_dc_444(seed)
    for c in f.components[1:]:
        c.tq = 1
    f.scans[2].quant = _quant(rng, (1,), 7, 40)
    f.scans[3].quant = _quant(rng, (0, 1), 41, 90)
    return f


def dqt16_444(seed):
    """16-bit DQT entries up to 1000 on small levels"""
    rng = np.random.default_rng(seed)
    comps = _components(rng, 24, 16, [(1, 1)] * 3, max_size=3, dc=20)
    q = {s: rng.integers(256, 1000, 64) for s in (0, 1)}
    return Frame(24, 16, comps, q, _simple_script(3, [0, 1, 1]), dqt16=True, progressive=True)


# ---- the int16 edge: a grey frame of five blocks, coefficients placed by (block, zig-zag k) -----------------------------------
def _edge_frame(seed, values, q, script, dqt16=False):
    """values: {(block, k): coefficient}; q: {k: quantiser} over a base of ones; script: [(ss, se, ah, al)] after a DC pass"""
    rng = np.random.default_rng(seed)
    coef = np.zeros((1, 5, 8, 8), dtype=np.int64)
    for b in range(5):
        coef[0, b, 0, 0] = int(rng.integers(-3, 4))
    for (b, k), v in values.items():
        coef[0, b].reshape(64)[ZZ[k]] = v
    qq = np.ones(64, dtype=np.int64)
    for k, v in q.items():
        qq[ZZ[k]] = v
    scans = []
    for i, (ss, se, ah, al) in enumerate(script):
        t = {}
        if ss == 0 and ah == 0:
            t = _tables((0,), ())
        elif ss > 0 and i == next(j for j, s in enumerate(script) if s[0] > 0):
            t = {**_tables((), (0,)), **_refine_tables((1,))}
        scans.append(Scan([0], [0], [1 if ah and ss else 0], ss, se, ah, al, t))
    return Frame(40, 8, [Component(coef)], {0: qq}, scans, dqt16=dqt16, progressive=True)


DC_PASS = [(0, 0, 0, 0)]


def i16_dc_first(seed, over):
    """DC levels 32767 and -32768 reached through the predictor (q = 1); beyond: 32768"""
    f = _edge_frame(seed, {}, {}, DC_PASS + [(1, 63, 0, 0)])
    f.components[0].coef[0, :, 0, 0] = [16384, 32768, 16384, 0, -16384] if over else [16384, 32767, 0, -16384, -32768]
    return f


def i16_dc_refine(seed, over):
    """DC first pass at Al 1, refinement to Al 0: 4681 x 7 = 32767 (odd level, the refinement bit sets it); beyond: 10923 x 3"""
    f = _edge_frame(seed, {}, {}, [(0, 0, 0, 1), (0, 0, 1, 0), (1, 63, 0, 0)])
    f.components[0].coef[0, :, 0, 0] = [10923 if over else 4681, -4681, 0, 1, -1]
    f.quant[0][0] = 3 if over else 7
    return f


def i16_ac_first(seed, over):
    """AC first pass at Al 0 (k = 1: +-32767) and at Al 6 (k = 2: -512 << 6 = -32768); beyond: 512 << 6 = 32768"""
    return _edge_frame(seed, {(0, 1): 32767, (1, 1): -32767, (2, 2): (512 if over else 511) << 6, (3, 2): -512 << 6},
                       {}, DC_PASS + [(1, 1, 0, 0), (2, 63, 0, 6)])


def i16_ac_refine(seed, over):
    """AC first pass at Al 1, refinement to Al 0: the correction bit lifts 4680 x 7 to 4681 x 7 = 32767 (and -32767); beyond:
    10922 x 3 = 32766 lifted to 10923 x 3 = 32769"""
    k, q = 5, (3 if over else 7)
    v = 10923 if over else 4681
    return _edge_frame(seed, {(0, k): v, (1, k): -v, (2, k + 1): 6}, {k: q}, DC_PASS + [(1, 63, 0, 1), (1, 63, 1, 0)])


def i16_ac_refine_new(seed, over):
    """a coefficient that becomes significant in the refinement, -1 x 32768 = -32768 (16-bit DQT); beyond: +1 x 32768"""
    return _edge_frame(seed, {(0, 7): -1, (3, 7): 1 if over else -1, (1, 9): 4}, {7: 32768}, DC_PASS + [(1, 63, 0, 1), (1, 63, 1, 0)],
                       dqt16=True)


def i16_product(seed, over):
    """AC first pass at Al 13 with q = 4: -1 x (4 << 13) = -32768; beyond: 2^14 x (32 << 13) = 2^32, which an int32 product
    wraps to 0"""
    if over:
        return _edge_frame(seed, {(0, 3): (1 << 14) << 13}, {3: 32}, DC_PASS + [(1, 63, 0, 13)])
    return _edge_frame(seed, {(0, 3): -(1 << 13), (2, 4): 1 << 13}, {3: 4}, DC_PASS + [(1, 63, 0, 13)])


def refused_q_shift(seed):
    """q << Al = 2048 << 13 = 2^24: beyond what the GPU tables hold, NOT_IMPLEMENTED"""
    return _edge_frame(seed, {(0, 3): 1 << 13}, {3: 2048}, DC_PASS + [(1, 63, 0, 13)], dqt16=True)


def _pair(fn):
    return [("%s_edge" % fn.__name__, functools.partial(fn, over=False)), ("%s_over" % fn.__name__, functools.partial(fn, over=True))]


# name -> (builder, seed, path)
CASES = {}
for _i, (_name, _fn, _path) in enumerate(
        [(f.__name__, f, p) for f, p in [(simple_420_37x21, "fused"), (simple_444_rst_45x30, "fused"), (simple_422_50x17, "fused"),
                                         (simple_grey_29x19, "fused"), (factors_3x_4x_61x47, "fused"), (factors_4x4_70x40, "fused"),
                                         (dc_only_grey_13x9, "fused"), (chroma_without_ac_422, "fused"), (noninterleaved_dc_444, "scan"),
                                         (seven_ac_scans_grey, "scan"), (deep_sa_8bit, "scan"), (deep_sa_12bit, "scan"),
                                         (deep_ac_sa_grey, "fused"), (dri_changed_between_scans, "scan"), (dri_resent_same, "fused"),
                                         (eobrun_at_restart, "fused"), (zrl_then_correction, "fused"), (refine_odd_sizes, "fused"),
                                         (dqt_redefined_fused, "fused"), (dqt_redefined_scan, "scan"), (dqt16_444, "fused"),
                                         (refused_q_shift, None)]] +
        [(n, f, "fused") for fn in (i16_dc_first, i16_dc_refine, i16_ac_first, i16_ac_refine, i16_ac_refine_new, i16_product)
         for n, f in _pair(fn)]):
    CASES[_name] = (_fn, 7001 + _i, _path)
NAMES = list(CASES)
REFUSED = {"refused_q_shift": -1034}


@functools.lru_cache(maxsize=None)
def case(name):
    fn, seed, _ = CASES[name]
    frame = fn(seed)
    return frame, sw.encode(frame)


def path(name):
    return CASES[name][2]
