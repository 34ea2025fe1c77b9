"""What a progressive (SOF2) scan script leaves in the coefficient store, written from ITU-T T.81 alone, for tests.

Input: a tests/streamwriter.py Frame (the coefficients the writer codes, its scan script, the DQTs in front of the frame and of
its scans). Output, per component, over the MCU-padded block grid ([bh, bw, 8, 8] int64, raster order inside the block):
  levels        the quantised levels the script codes: the DC of a block shifted right by the lowest Al of the DC scans that
                hold the component (arithmetic shift, G.1.2.1), each AC coefficient's magnitude by the lowest Al of the AC
                scans whose band holds it (rounded toward zero, G.1.2.2), both shifted back; zero where no scan reaches
  quantisers    the table each component dequantises with under a named rule:
                  "frame_first"      the tables in effect at the frame's first scan
                  "component_first"  the tables in effect at the first scan that holds the component
                  "last"             the last definition of each slot in the stream
  dequantised   levels x quantiser, exact (int64)
  fits_int16    whether every dequantised coefficient fits the int16 coefficient store
"""
import numpy as np

from tests.streamwriter import ZIGZAG

RULES = ("frame_first", "component_first", "last")


def levels(frame):
    out = []
    for ci, comp in enumerate(frame.components):
        coef = np.asarray(comp.coef, dtype=np.int64)
        dc_al = [s.al for s in frame.scans if s.ss == 0 and ci in s.comps]
        ac_al = np.full(64, -1)  # per raster position: the lowest Al that reaches it
        for s in frame.scans:
            if s.ss > 0 and ci in s.comps:
                for k in range(s.ss, s.se + 1):
                    r = ZIGZAG[k]
                    ac_al[r] = s.al if ac_al[r] < 0 else min(ac_al[r], s.al)
        lv = np.zeros_like(coef)
        if dc_al:
            a = min(dc_al)
            lv[..., 0, 0] = (coef[..., 0, 0] >> a) << a
        flat = coef.reshape(coef.shape[:2] + (64,))
        lflat = lv.reshape(flat.shape)
        for r in range(1, 64):
            if ac_al[r] >= 0:
                a = int(ac_al[r])
                lflat[..., r] = np.sign(flat[..., r]) * ((np.abs(flat[..., r]) >> a) << a)
        out.append(lflat.reshape(coef.shape))
    return out


def _tables_at_scans(frame):
    """[per scan: {slot: 64 raster values} in effect at that scan], and the last definitions"""
    cur = {k: np.asarray(v, dtype=np.int64).reshape(64) for k, v in frame.quant.items()}
    at = []
    for s in frame.scans:
        cur.update({k: np.asarray(v, dtype=np.int64).reshape(64) for k, v in s.quant.items()})
        at.append(dict(cur))
    return at, cur


def quantisers(frame, rule):
    """[per component: 64 raster quantiser values] under `rule`"""
    at, last = _tables_at_scans(frame)
    out = []
    for ci, comp in enumerate(frame.components):
        if rule == "frame_first":
            tabs = at[0]
        elif rule == "component_first":
            tabs = next((at[i] for i, s in enumerate(frame.scans) if ci in s.comps), last)
        elif rule == "last":
            tabs = last
        else:
            raise ValueError(rule)
        out.append(tabs[comp.tq])
    return out


def dequantised(frame, rule="component_first"):
    return [lv * q.reshape(8, 8) for lv, q in zip(levels(frame), quantisers(frame, rule))]


def fits_int16(frame, rule="component_first"):
    return all(d.min() >= -32768 and d.max() <= 32767 for d in dequantised(frame, rule))
