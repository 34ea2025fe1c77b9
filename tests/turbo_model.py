"""Executable specification of B200JPG_FLAG_LIBJPEG_TURBO (DESIGN §16). TEST-ONLY.

libjpeg-turbo's reconstruction as Pillow runs it, from dequantised coefficients on: the JDCT_ISLOW IDCT in its C form with 64-bit
intermediates (LP64), the post-IDCT range-limit table, the "fancy" upsamplers (h2v1, h1v2, h2v2; every other integer ratio
replicates) and the fixed-point YCbCr -> RGB conversion. All in int64. tests/test_turbo_cpu.py checks it byte for byte against
Pillow; tests/test_turbo.py checks the GPU against it."""
import numpy as np

# the 13-bit constants of the islow butterfly, round(2^13 * x)
C0_298, C0_390, C0_541, C0_765, C0_899, C1_175 = 2446, 3196, 4433, 6270, 7373, 9633
C1_501, C1_847, C1_961, C2_053, C2_562, C3_072 = 12299, 15137, 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2
PASS1_SHIFT = CONST_BITS - PASS1_BITS          # 11
PASS2_SHIFT = CONST_BITS + PASS1_BITS + 3      # 18


def idct1d(d, shift, record=None):
    """one 8-point pass over d[0..8) (int64 arrays or Python ints, any matching shapes) -> 8 outputs (x + 2^(shift-1)) >> shift.
    record: a list that receives every intermediate of the butterfly (tests/test_turbo_cpu.py derives the int32 bounds from it)."""
    def r(v):
        if record is not None:
            record.append(v)
        return v
    # even part
    z1 = r(r(d[2] + d[6]) * C0_541)
    tmp2 = r(z1 + r(d[6] * -C1_847))
    tmp3 = r(z1 + r(d[2] * C0_765))
    tmp0 = r(r(d[0] + d[4]) * (1 << CONST_BITS))
    tmp1 = r(r(d[0] - d[4]) * (1 << CONST_BITS))
    t10, t13 = r(tmp0 + tmp3), r(tmp0 - tmp3)
    t11, t12 = r(tmp1 + tmp2), r(tmp1 - tmp2)
    # odd part
    o0, o1, o2, o3 = d[7], d[5], d[3], d[1]
    z1, z2, z3, z4 = r(o0 + o3), r(o1 + o2), r(o0 + o2), r(o1 + o3)
    z5 = r(r(z3 + z4) * C1_175)
    o0, o1, o2, o3 = r(o0 * C0_298), r(o1 * C2_053), r(o2 * C3_072), r(o3 * C1_501)
    z1, z2, z3, z4 = r(z1 * -C0_899), r(z2 * -C2_562), r(z3 * -C1_961), r(z4 * -C0_390)
    z3, z4 = r(z3 + z5), r(z4 + z5)
    o0 = r(o0 + r(z1 + z3))
    o1 = r(o1 + r(z2 + z4))
    o2 = r(o2 + r(z2 + z3))
    o3 = r(o3 + r(z1 + z4))
    rnd = 1 << (shift - 1)
    outs = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return [(r(v) + rnd) >> shift for v in outs]


def range_limit(v):
    """the post-IDCT table at index v & 1023: 0..127 -> v + 128, 128..511 -> 255, 512..895 -> 0, 896..1023 -> v - 896"""
    i = np.asarray(v, dtype=np.int64) & 1023
    return np.where(i < 128, i + 128, np.where(i < 512, 255, np.where(i < 896, 0, i - 896))).astype(np.uint8)


def idct_pass1(F):
    """F [..., 8, 8] dequantised (raster: row = vertical frequency) -> the pass-1 workspace [..., 8, 8] (columns, descale 11)"""
    F = np.asarray(F, dtype=np.int64)
    cols = idct1d([F[..., u, :] for u in range(8)], PASS1_SHIFT)
    return np.stack(cols, axis=-2)


def idct_blocks(F):
    """F [..., 8, 8] dequantised -> [..., 8, 8] uint8 samples"""
    ws = idct_pass1(F)
    rows = idct1d([ws[..., :, u] for u in range(8)], PASS2_SHIFT)
    return range_limit(np.stack(rows, axis=-1))


def idct_plane(coef):
    """coef [bh, bw, 8, 8] dequantised -> uint8 plane [8 bh, 8 bw]"""
    bh, bw = coef.shape[:2]
    return idct_blocks(coef).transpose(0, 2, 1, 3).reshape(8 * bh, 8 * bw)


def upsample(a, fx, fy, w, h):
    """the plane a (at least h x w, real size h x w) upsampled by the integer factors fx x fy -> [fy h, fx w] int64: h2v1 and h2v2
    fancy for w > 2, h1v2 fancy, every other ratio replicated. The row above the first and below row h - 1 is that row itself."""
    a = np.asarray(a, dtype=np.int64)[:h, :w]
    if (fx, fy) in ((2, 1), (2, 2)) and w <= 2 or (fx, fy) not in ((1, 1), (2, 1), (1, 2), (2, 2)):
        return np.repeat(np.repeat(a, fy, axis=0), fx, axis=1)
    if fx == 1 and fy == 1:
        return a
    above = np.concatenate([a[:1], a[:-1]], axis=0)
    below = np.concatenate([a[1:], a[-1:]], axis=0)
    if fx == 1:  # h1v2
        out = np.empty((2 * h, w), dtype=np.int64)
        out[0::2] = (3 * a + above + 1) >> 2
        out[1::2] = (3 * a + below + 2) >> 2
        return out

    def h2(cs, sh, r0, r1, edge0, edge1):
        left = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        out = np.empty((cs.shape[0], 2 * w), dtype=np.int64)
        out[:, 0::2] = (3 * cs + left + r0) >> sh
        out[:, 1::2] = (3 * cs + right + r1) >> sh
        out[:, 0] = edge0(cs[:, 0])
        out[:, -1] = edge1(cs[:, -1])
        return out
    if fy == 1:  # h2v1
        return h2(a, 2, 1, 2, lambda c: c, lambda c: c)
    out = np.empty((2 * h, 2 * w), dtype=np.int64)  # h2v2
    for k, far in ((0, above), (1, below)):
        out[k::2] = h2(3 * a + far, 4, 8, 7, lambda c: (4 * c + 8) >> 4, lambda c: (4 * c + 7) >> 4)
    return out


def ycc_to_rgb(y, cb, cr):
    """libjpeg-turbo's ycc_rgb_convert on 8-bit samples (arithmetic shifts, clamped) -> [..., 3] uint8"""
    y, b, r = (np.asarray(v, dtype=np.int64) for v in (y, cb, cr))
    b, r = b - 128, r - 128
    rgb = [y + ((91881 * r + 32768) >> 16), y + ((-22554 * b - 46802 * r + 32768) >> 16), y + ((116130 * b + 32768) >> 16)]
    return np.clip(np.stack(rgb, axis=-1), 0, 255).astype(np.uint8)


def luma(rgb):
    """Pillow's convert("L") of uint8 RGB (the existing L formula)"""
    v = np.asarray(rgb, dtype=np.int64)
    return ((19595 * v[..., 0] + 38470 * v[..., 1] + 7471 * v[..., 2] + 32768) >> 16).astype(np.uint8)


def dequantised(info, planes):
    """the oracle's quantised coefficients (tests/oracle_binding.Oracle.coefficients) times the component's quantiser, int64"""
    out = []
    for c, p in enumerate(planes):
        q = np.array(info.quant[info.tq[c]][:], dtype=np.int64).reshape(8, 8)
        out.append(np.asarray(p, dtype=np.int64) * q)
    return out


def reconstruct(coef, width, height, hs, vs, colorspace, mode=None, color_transform=True):
    """coef: per component [bh, bw, 8, 8] dequantised; hs / vs the sampling factors; colorspace "L", "YCbCr" or "RGB" (as
    b200jpg_colorspace reads the frame) -> [height, width, C] uint8, C as the batch writes it: the frame's components, 3 with
    mode "RGB", 1 with mode "L". color_transform=False delivers the upsampled components as they are."""
    nc = len(coef)
    hmax, vmax = max(hs[:nc]), max(vs[:nc])
    comps = range(1 if (mode == "L" and colorspace == "YCbCr") else nc)

    def plane(c):
        fx, fy = hmax // hs[c], vmax // vs[c]
        assert fx * hs[c] == hmax and fy * vs[c] == vmax, "fractional sampling ratios are not upsampled"
        w, h = -(-width * hs[c] // hmax), -(-height * vs[c] // vmax)
        return upsample(idct_plane(coef[c]), fx, fy, w, h)[:height, :width].astype(np.uint8)
    p = [plane(c) for c in comps]
    if len(p) == 3 and colorspace == "YCbCr" and color_transform:
        out = ycc_to_rgb(*p)
    else:
        out = np.stack(p, axis=-1)
    if mode == "RGB" and out.shape[-1] == 1:
        out = np.repeat(out, 3, axis=-1)
    if mode == "L" and out.shape[-1] == 3:
        out = luma(out)[..., None]
    return out


def decode(oracle, data, colorspace, mode=None, color_transform=True):
    """the model on one intact codestream, its coefficients from the oracle -> [H, W, C] uint8"""
    rc, info, planes = oracle.coefficients(data)
    assert rc == 0, rc
    return reconstruct(dequantised(info, planes), info.width, info.height, list(info.hs), list(info.vs), colorspace, mode, color_transform)
