"""Executable specification of downscaled decoding (B200JPG_FLAG_DOWNSCALE_k, DESIGN §10). TEST-ONLY.

scaled_planes: the fixed-point scaled IDCT, dequantised coefficients -> int32 sample planes of (8/k) x (8/k) samples per block,
4 fractional bits, level shifted. reconstruct_samples: the reference's rules from sample planes on (upsampler cores for factors
1..4 with their in-place store order and edge replication, colour transformation, clamp, 8- / 16-bit samples), written after
upsampling/upsampler.cpp:83-386 and colortrafo/ycbcrtrafo.cpp:842-850; tests/test_downscale_cpu.py checks it byte for byte
against the oracle's full-size decode."""
import numpy as np

# round(2^20 * A_k(m, u)), A_k(m, u) = 1/k sum_{j<k} C(u)/2 cos((2 (k m + j) + 1) u pi / 16)
BASIS = {
    2: np.array([[370728, 475072, 342508, 166823, 0, -111468, -141871, -94498],
                 [370728, 196781, -342508, -402746, 0, 269107, 141871, -39142],
                 [370728, -196781, -342508, 402746, 0, -269107, 141871, 39142],
                 [370728, -475072, 342508, -166823, 0, 111468, -141871, 94498]], dtype=np.int64),
    4: np.array([[370728, 335926, 0, -117962, 0, 78819, 0, -66820],
                 [370728, -335926, 0, 117962, 0, -78819, 0, 66820]], dtype=np.int64),
}


def basis(k):
    """A_k as float64: row m = output sample, column u = frequency"""
    n = 8 // k
    a = np.zeros((n, 8))
    for m in range(n):
        for u in range(8):
            cu = (1 / np.sqrt(2) if u == 0 else 1.0) / 2
            a[m, u] = np.mean([cu * np.cos((2 * (k * m + j) + 1) * u * np.pi / 16) for j in range(k)])
    return a


def idct8_matrix():
    """the exact 8-point IDCT: x = M @ F"""
    return basis(1)


def scaled_blocks(F, k, precision):
    """F [..., 8, 8] dequantised coefficients (raster, row = vertical frequency) -> [..., 8/k, 8/k] int samples"""
    F = np.asarray(F, dtype=np.int64)
    level = 8 << precision
    if k == 8:
        return (2 * F[..., 0:1, 0:1] + level).astype(np.int64)
    a = BASIS[k]
    p = (np.einsum("...ru,mu->...rm", F, a) + (1 << 7)) >> 8      # row pass, |p| < 2^28
    assert np.abs(p).max(initial=0) < 2 ** 28
    return ((np.einsum("nr,...rm->...nm", a, p) + (1 << 27)) >> 28) + level  # column pass


def exact_box_average(F, k, precision):
    """float64 k x k box average of the exact IDCT, in the same domain (x 16, level shifted)"""
    F = np.asarray(F, dtype=np.float64)
    a = basis(k)
    return 16 * np.einsum("nr,...ru,mu->...nm", a, F, a) + (8 << precision)


def scaled_planes(coef, k, precision):
    """coef [bh, bw, 8, 8] dequantised -> plane [(8/k) bh, (8/k) bw] int64"""
    bh, bw = coef.shape[:2]
    n = 8 // k
    s = scaled_blocks(coef, k, precision)
    return s.transpose(0, 2, 1, 3).reshape(bh * n, bw * n)


def full_planes(oracle, coef, precision):
    """coef [bh, bw, 8, 8] dequantised -> the reference's full-size IDCT planes through jpgo_idct_block"""
    bh, bw = coef.shape[:2]
    out = np.zeros((bh * 8, bw * 8), dtype=np.int64)
    ones = np.ones(64, dtype=np.uint16)
    for y in range(bh):
        for x in range(bw):
            out[8 * y:8 * y + 8, 8 * x:8 * x + 8] = oracle.idct(coef[y, x].reshape(64).astype(np.int32), ones, 1 << (precision - 1))
    return out


def _mix(a, wa, b, wb, rnd, sh):
    return (wa * a + wb * b + rnd) >> sh


def upsample(plane, w, h, sx, sy, W, H):
    """Upsampler<sx, sy>::UpsampleRegion over a W x H frame: plane = IDCT output whose true extent is w x h"""
    if sx == 1 and sy == 1:
        return plane[:H, :W].astype(np.int64)
    p = plane.astype(np.int64)
    bw, bh = (W + 7) // 8, (H + 7) // 8
    out = np.zeros((bh * 8, bw * 8), dtype=np.int64)
    X = 8 * np.arange(bw)
    x0 = X // sx - (1 if sx > 1 else 0)
    xmod = X % sx
    for by in range(bh):
        Y = 8 * by
        y = Y // sy
        top, cur, bot = (y - 1 if y > 0 else y), y, (y + 1 if y + 1 < h else y)
        ymod = Y % sy

        def at(j, yy):
            return p[yy, np.clip(x0 + j, 0, w - 1)]

        for row in range(8):
            o = [None] * 8
            advance = False
            if sy == 1:
                for j in range(8):
                    o[j] = at(j, cur)
                if cur + 1 < h:
                    cur += 1
            elif sy == 2:
                nb = top if ymod == 0 else bot
                for j in range(8):
                    o[j] = _mix(at(j, nb), 1, at(j, cur), 3, 2 if (j & 1) == ymod else 1, 2)
                advance = ymod == 1
            elif sy == 3:
                if ymod == 1:
                    for j in range(8):
                        o[j] = at(j, cur)
                else:
                    nb = top if ymod == 0 else bot
                    for j in range(8):
                        o[j] = _mix(at(j, nb), 1, at(j, cur), 3, 2 if ((j & 1) == 0) == (ymod == 0) else 1, 2)
                advance = ymod == 2
            else:
                nb = top if ymod < 2 else bot
                far = ymod in (0, 3)
                for j in range(8):
                    if ymod in (0, 2, 3):
                        rnd = 3 if j & 1 else 4
                    else:
                        rnd = 4 if j & 1 else 3
                    o[j] = _mix(at(j, nb), 3 if far else 1, at(j, cur), 5 if far else 7, rnd, 3)
                advance = ymod == 3
            if sy > 1:
                if advance:
                    ymod, top, cur = 0, cur, bot
                    if bot + 1 < h:
                        bot += 1
                else:
                    ymod += 1
            # horizontal cores, in place in the reference's store order: src[i] = o[i + 1]
            s = lambda i: o[i + 1]
            if sx == 2:
                o[7] = _mix(s(4), 1, s(3), 3, 1, 2)
                o[6] = _mix(s(2), 1, s(3), 3, 2, 2)
                o[5] = _mix(s(3), 1, s(2), 3, 1, 2)
                o[4] = _mix(s(1), 1, s(2), 3, 2, 2)
                o[3] = _mix(s(2), 1, s(1), 3, 1, 2)
                o[2] = _mix(s(0), 1, s(1), 3, 2, 2)
                t = s(0)
                o[1] = _mix(s(1), 1, t, 3, 1, 2)
                o[0] = _mix(s(-1), 1, t, 3, 2, 2)
            elif sx == 3:
                variants = []
                for xm in range(3):
                    q = list(o)
                    r = lambda i: q[i + 1]
                    if xm == 0:
                        q[7] = r(2); q[6] = _mix(r(1), 1, r(2), 3, 2, 2); q[5] = _mix(r(2), 1, r(1), 3, 1, 2); q[4] = r(1)
                        q[3] = _mix(r(0), 1, r(1), 3, 2, 2); q[2] = _mix(r(1), 1, r(0), 3, 1, 2); q[0] = _mix(r(-1), 1, r(0), 3, 2, 2)
                        q[1] = r(0)
                    elif xm == 1:
                        q[7] = _mix(r(3), 1, r(2), 3, 1, 2); q[6] = r(2); q[5] = _mix(r(1), 1, r(2), 3, 2, 2)
                        q[4] = _mix(r(2), 1, r(1), 3, 1, 2); q[3] = r(1); t = r(0); q[2] = _mix(t, 1, r(1), 3, 2, 2)
                        q[1] = _mix(r(1), 1, t, 3, 1, 2); q[0] = t
                    else:
                        q[7] = _mix(r(2), 1, r(3), 3, 2, 2); q[6] = _mix(r(3), 1, r(2), 3, 1, 2); q[5] = r(2)
                        q[4] = _mix(r(1), 1, r(2), 3, 2, 2); q[3] = _mix(r(2), 1, r(1), 3, 1, 2); q[2] = r(1); t = r(0)
                        q[1] = _mix(t, 1, r(1), 3, 2, 2); q[0] = _mix(r(1), 1, t, 3, 1, 2)
                    variants.append(q)
                o = [np.select([xmod == 0, xmod == 1], [variants[0][j], variants[1][j]], variants[2][j]) for j in range(8)]
            elif sx == 4:
                o[7] = _mix(s(2), 3, s(1), 5, 1, 3)
                o[6] = _mix(s(2), 1, s(1), 7, 2, 3)
                o[5] = _mix(s(0), 1, s(1), 7, 1, 3)
                o[4] = _mix(s(0), 3, s(1), 5, 2, 3)
                t = s(0)
                o[3] = _mix(s(1), 3, t, 5, 1, 3)
                o[2] = _mix(s(1), 1, t, 7, 2, 3)
                o[1] = _mix(s(-1), 1, t, 7, 1, 3)
                o[0] = _mix(s(-1), 3, t, 5, 2, 3)
            for j in range(8):
                out[Y + row, X + j] = o[j]
    return out[:H, :W]


def reconstruct_samples(planes, subx, suby, W, H, precision, ycbcr, out16=False):
    """the frame W x H from its IDCT output planes (component c's true extent ceil(W / subx) x ceil(H / suby)):
    -> [H, W, ncomp] uint8 (8-bit frames) or uint16 (out16, or 12-bit frames)"""
    nc = len(planes)
    up = [upsample(planes[c], -(-W // subx[c]), -(-H // suby[c]), subx[c], suby[c], W, H) for c in range(nc)]
    maxval = (1 << precision) - 1
    if nc == 3 and ycbcr:
        coff = 16 << (precision - 1)
        yv, cb, cr = up[0], up[1] - coff, up[2] - coff
        v = [(yv * 8192 + cr * 11485 + 65536) >> 17, (yv * 8192 - cb * 2819 - cr * 5850 + 65536) >> 17,
             (yv * 8192 + cb * 14516 + 65536) >> 17]
    else:
        v = [(u + 8) >> 4 for u in up]
    out = np.stack([np.clip(x, 0, maxval) for x in v], axis=-1)
    return out.astype(np.uint16 if (out16 or precision > 8) else np.uint8)


def planes_out(planes, subx, suby, W, H, precision):
    """B200JPG_FLAG_NO_UPSAMPLE: component c as ceil(W / subx) x ceil(H / suby) samples, COLOR_TO_INT + clamp"""
    maxval = (1 << precision) - 1
    res = []
    for c, p in enumerate(planes):
        w, h = -(-W // subx[c]), -(-H // suby[c])
        res.append(np.clip((p[:h, :w].astype(np.int64) + 8) >> 4, 0, maxval).astype(np.uint16 if precision > 8 else np.uint8))
    return res


def scaled_extent(W, H, k):
    return -(-W // k), -(-H // k)


def expected(coefs, subx, suby, W, H, precision, ycbcr, k, upsample_=True):
    """coefs[c] [bh, bw, 8, 8] dequantised -> the frame decoded at 1/k: [H', W', C] array, or the planes without upsampling"""
    planes = [scaled_planes(cf, k, precision) for cf in coefs]
    Wk, Hk = scaled_extent(W, H, k)
    if not upsample_:
        return planes_out(planes, subx, suby, Wk, Hk, precision)
    return reconstruct_samples(planes, subx, suby, Wk, Hk, precision, ycbcr)
