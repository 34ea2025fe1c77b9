"""Executable specification of BatchDecoder(draft=...) / b200jpg_batch_create_draft (DESIGN §17). TEST-ONLY.

libjpeg-turbo's reconstruction at scale 1/k, as Pillow's Image.draft(mode, (w, h)) asks for it, from dequantised coefficients on:
Pillow's choice of k, the IDCT size of every component (jdmaster.c), the reduced IDCTs of jidctred.c in their C form with 64-bit
intermediates, upsampling by the ratios after them (fancy for k = 2 and 4, replicated for k = 8) and tests/turbo_model.py's
colour conversion. tests/test_draft_cpu.py checks it byte for byte against Pillow; tests/test_draft.py checks the GPU against it."""
import numpy as np

from tests import turbo_model as tm


def draft_scale(width, height, req_w, req_h):
    """Pillow's JpegImageFile.draft: the largest k of 8, 4, 2, 1 with k <= min(W // w, H // h), 1 when none fits"""
    s = min(width // req_w, height // req_h)
    return next((k for k in (8, 4, 2) if k <= s), 1)


def idct_size(hs, vs, c, k):
    """s_c: 8 / k, doubled while below 8 and (hmax m) % (2 h_c s) == 0 and (vmax m) % (2 v_c s) == 0 (jdmaster.c)"""
    m = 8 // k
    hmax, vmax = max(hs), max(vs)
    s = m
    while s < 8 and (hmax * m) % (hs[c] * s * 2) == 0 and (vmax * m) % (vs[c] * s * 2) == 0:
        s *= 2
    return s


def red4_line(d, shift, record=None):
    """one line of jpeg_idct_4x4 over d[0..8) (d[4] unused) -> 4 outputs (x + 2^(shift-1)) >> shift. record: receives every sum"""
    def r(v):
        if record is not None:
            record.append(v)
        return v
    t0 = r(d[0] * 16384)
    t2 = r(r(d[2] * 15137) + r(d[6] * -6270))
    t10, t12 = r(t0 + t2), r(t0 - t2)
    o0 = r(r(r(r(d[7] * -1730) + r(d[5] * 11893)) + r(d[3] * -17799)) + r(d[1] * 8697))
    o2 = r(r(r(r(d[7] * -4176) + r(d[5] * -4926)) + r(d[3] * 7373)) + r(d[1] * 20995))
    rnd = 1 << (shift - 1)
    return [(r(v) + rnd) >> shift for v in (t10 + o2, t12 + o0, t12 - o0, t10 - o2)]


def red2_line(d, shift, record=None):
    """one line of jpeg_idct_2x2 over d[0..8) (d[2], d[4], d[6] unused) -> 2 outputs"""
    def r(v):
        if record is not None:
            record.append(v)
        return v
    t10 = r(d[0] * 32768)
    t0 = r(r(r(r(d[7] * -5906) + r(d[5] * 6967)) + r(d[3] * -10426)) + r(d[1] * 29692))
    rnd = 1 << (shift - 1)
    return [(r(v) + rnd) >> shift for v in (t10 + t0, t10 - t0)]


def idct_blocks(F, s):
    """F [..., 8, 8] dequantised (raster: row = vertical frequency) -> [..., s, s] uint8 samples of the s-point IDCT"""
    F = np.asarray(F, dtype=np.int64)
    if s == 8:
        return tm.idct_blocks(F)
    if s == 1:
        return tm.range_limit((F[..., 0, 0] + 4) >> 3)[..., None, None]
    line, p1, p2 = (red4_line, 12, 19) if s == 4 else (red2_line, 13, 20)
    ws = np.stack(line([F[..., u, :] for u in range(8)], p1), axis=-2)  # [..., s, 8]: pass 1 down every column
    return tm.range_limit(np.stack(line([ws[..., :, u] for u in range(8)], p2), axis=-1))  # [..., s, s]


def idct_plane(coef, s):
    """coef [bh, bw, 8, 8] -> uint8 plane [s bh, s bw]"""
    bh, bw = coef.shape[:2]
    return idct_blocks(coef, s).transpose(0, 2, 1, 3).reshape(s * bh, s * bw)


def reconstruct(coef, width, height, hs, vs, k, colorspace, mode=None, color_transform=True):
    """tests/turbo_model.reconstruct at scale 1/k: coef per component [bh, bw, 8, 8] dequantised, width x height the codestream's
    size -> [ceil(H / k), ceil(W / k), C] uint8"""
    if k == 1:
        return tm.reconstruct(coef, width, height, hs, vs, colorspace, mode, color_transform)
    nc = len(coef)
    hs, vs = list(hs[:nc]), list(vs[:nc])
    hmax, vmax, m = max(hs), max(vs), 8 // k
    W, H = -(-width // k), -(-height // k)
    comps = range(1 if (mode == "L" and colorspace == "YCbCr") else nc)

    def plane(c):
        s = idct_size(hs, vs, c, k)
        fx, fy = hmax * m // (hs[c] * s), vmax * m // (vs[c] * s)
        assert fx * hs[c] * s == hmax * m and fy * vs[c] * s == vmax * m, "fractional sampling ratios are not upsampled"
        w, h = -(-W // fx), -(-H // fy)
        a = idct_plane(coef[c], s)
        if k == 8:  # fancy upsampling is off at 1/8: every ratio replicates
            up = np.repeat(np.repeat(a[:h, :w].astype(np.int64), fy, axis=0), fx, axis=1)
        else:
            up = tm.upsample(a, fx, fy, w, h)
        return up[:H, :W].astype(np.uint8)
    p = [plane(c) for c in comps]
    if len(p) == 3 and colorspace == "YCbCr" and color_transform:
        out = tm.ycc_to_rgb(*p)
    else:
        out = np.stack(p, axis=-1)
    if mode == "RGB" and out.shape[-1] == 1:
        out = np.repeat(out, 3, axis=-1)
    if mode == "L" and out.shape[-1] == 3:
        out = tm.luma(out)[..., None]
    return out


def decode(oracle, data, colorspace, k, mode=None, color_transform=True):
    """the model on one intact codestream at scale 1/k, its coefficients from the oracle -> [H', W', C] uint8"""
    rc, info, planes = oracle.coefficients(data)
    assert rc == 0, rc
    return reconstruct(tm.dequantised(info, planes), info.width, info.height, list(info.hs), list(info.vs), k, colorspace, mode,
                       color_transform)
