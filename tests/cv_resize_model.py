"""numpy model of OpenCV's cv2.resize(C, (W_t, H_t), interpolation=INTER_LINEAR | INTER_AREA) of a uint8 [h, w, C] image, every
channel on its own (DESIGN §20). inv = W_t / w and scale = 1 / inv in double, as OpenCV computes them; rint is round-half-even,
what OpenCV's saturate_cast / cvRound do. Float arithmetic is float32, one rounding per operation, in OpenCV's order.

  rule 1, INTER_LINEAR: two taps per output with 11-bit int16 weights; the horizontal pass keeps int32 sums, the vertical pass is
          (((b0 (T0 >> 4)) >> 16) + ((b1 (T1 >> 4)) >> 16) + 2) >> 2, clamped. Horizontally the fraction is clamped with the index at
          the edges, vertically only the two row indices are.
  rule 2, INTER_AREA with integer factors on both axes (OpenCV's |scale - round(scale)| < DBL_EPSILON): block sums, (s + 2) >> 2
          for 2 x 2 blocks, rint((float)s * (1.0f / (fx fy))) for the others.
  rule 3, INTER_AREA, both axes at a scale >= 1, not both integer: computeResizeAreaTab's float tables, horizontal then vertical,
          float sums in table order.
  rule 4, INTER_AREA when either axis upscales: rule 1's machinery on both axes with the "area mode" fractions.
A W_t x H_t equal to w x h is a copy."""
import numpy as np

LINEAR, AREA = 0x101, 0x103  # B200JPG_RESAMPLE_CV_LINEAR / _CV_AREA: 0x100 | cv2.INTER_LINEAR / cv2.INTER_AREA
NAMES = {"cv2-linear": LINEAR, "cv2-area": AREA}
TABLE_VERTICAL, TABLE_LINEAR = 0x1000, 0x2000  # b200jpg_resample_coefficients: the vertical axis; rule 4 on a non-upscaling axis
DBL_EPSILON = np.finfo(np.float64).eps
F32 = np.float32


def _scale(in_size, out_size):
    inv = out_size / in_size
    return inv, 1.0 / inv


def linear_table(in_size, out_size, area=False, vertical=False):
    """rules 1 / 4 for one axis -> (i0, i1, a0, a1): the two source indices (clamped) and int16 weights of every output"""
    inv, scale = _scale(in_size, out_size)
    d = np.arange(out_size, dtype=np.float64)
    if not area:
        fx = ((d + 0.5) * scale - 0.5).astype(F32)
        sx = np.floor(fx).astype(np.int64)
        fx = (fx - sx.astype(F32)).astype(F32)
    else:
        sx = np.floor(d * scale).astype(np.int64)
        fx = ((d + 1) - (sx + 1) * inv).astype(F32)
        fx = np.where(fx <= 0, F32(0), (fx - np.floor(fx)).astype(F32)).astype(F32)
    if not vertical:
        low, high = sx < 0, sx >= in_size - 1
        fx = np.where(low | high, F32(0), fx).astype(F32)
        sx = np.where(low, 0, np.where(high, in_size - 1, sx))
    a0 = np.rint((F32(1) - fx).astype(F32) * F32(2048)).astype(np.int64)
    a1 = np.rint(fx * F32(2048)).astype(np.int64)
    i0 = np.clip(sx, 0, in_size - 1)
    i1 = np.clip(sx + 1, 0, in_size - 1)
    return i0, i1, a0, a1


def area_table(in_size, out_size):
    """rule 3 for one axis, OpenCV's computeResizeAreaTab -> (first [out], taps [out], weights [out, ksize] float32)"""
    _, scale = _scale(in_size, out_size)
    firsts, counts, rows = [], [], []
    for dx in range(out_size):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, in_size - fsx1)
        sx1, sx2 = int(np.ceil(fsx1)), int(np.floor(fsx2))
        sx2 = min(sx2, in_size - 1)
        sx1 = min(sx1, sx2)
        first, w = None, []
        if sx1 - fsx1 > 1e-3:
            first = sx1 - 1
            w.append(np.float32((sx1 - fsx1) / cell))
        for _sx in range(sx1, sx2):
            w.append(np.float32(1.0 / cell))
        if first is None:
            first = sx1
        if fsx2 - sx2 > 1e-3:
            w.append(np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell))
        firsts.append(first), counts.append(len(w)), rows.append(w)
    k = max(counts)
    weights = np.zeros((out_size, k), dtype=F32)
    for j, w in enumerate(rows):
        weights[j, :len(w)] = w
    return np.array(firsts, dtype=np.int64), np.array(counts, dtype=np.int64), weights


def integer_factor(in_size, out_size):
    """OpenCV's is_area_fast test for one axis: the integer factor, or None"""
    _, scale = _scale(in_size, out_size)
    k = int(np.rint(scale))
    return k if abs(scale - k) < DBL_EPSILON else None


def rule(w, h, width, height, interpolation):
    """which rule cv2.resize applies: "copy", 1, 2, 3 or 4"""
    if (w, h) == (width, height):
        return "copy"
    if interpolation == LINEAR:
        return 1
    _, sx = _scale(w, width)
    _, sy = _scale(h, height)
    if sx >= 1 and sy >= 1:
        return 2 if integer_factor(w, width) and integer_factor(h, height) else 3
    return 4


def _linear(img, width, height, area):
    h, w, _ = img.shape
    i0, i1, a0, a1 = linear_table(w, width, area)
    s = img.astype(np.int64)
    t = s[:, i0, :] * a0[None, :, None] + s[:, i1, :] * a1[None, :, None]
    r0, r1, b0, b1 = linear_table(h, height, area, vertical=True)
    v = (((b0[:, None, None] * (t[r0] >> 4)) >> 16) + ((b1[:, None, None] * (t[r1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def _weighted(src, first, count, weights, axis):
    """float32 sums along `axis` in table order (a zero weight behind the taps adds nothing)"""
    n = src.shape[axis]
    acc = None
    for t in range(weights.shape[1]):
        idx = np.minimum(first + t, n - 1)
        tap = np.take(src, idx, axis=axis)
        wt = np.where(t < count, weights[:, t], F32(0)).astype(F32)
        wt = wt[:, None, None] if axis == 0 else wt[None, :, None]
        prod = (tap * wt).astype(F32)
        acc = prod if acc is None else (acc + prod).astype(F32)
    return acc


def _area(img, width, height):
    h, w, _ = img.shape
    fx, fy = integer_factor(w, width), integer_factor(h, height)
    if fx and fy:
        s = img.astype(np.int64).reshape(height, fy, width, fx, -1).sum(axis=(1, 3))
        if (fx, fy) == (2, 2):
            return ((s + 2) >> 2).astype(np.uint8)
        return np.clip(np.rint(s.astype(F32) * F32(F32(1.0) / F32(fx * fy))), 0, 255).astype(np.uint8)
    xf, xc, xw = area_table(w, width)
    yf, yc, yw = area_table(h, height)
    buf = _weighted(img.astype(F32), xf, xc, xw, axis=1)
    out = _weighted(buf, yf, yc, yw, axis=0)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def resize(img, width, height, interpolation):
    """cv2.resize(img, (width, height), interpolation=...) of a uint8 [h, w] or [h, w, C] image; LINEAR / AREA or their names"""
    interpolation = NAMES.get(interpolation, interpolation)
    a = img[..., None] if img.ndim == 2 else img
    r = rule(a.shape[1], a.shape[0], width, height, interpolation)
    if r == "copy":
        out = a.copy()
    elif r in (1, 4):
        out = _linear(a, width, height, r == 4)
    else:
        out = _area(a, width, height)
    return out[..., 0] if img.ndim == 2 else out


def resize_window(img, width, height, interpolation, window=None):
    """resize() then the window (x, y, width, height) of the result, [h, w, C]"""
    out = resize(img, width, height, interpolation)
    if window is not None:
        x, y, ww, wh = window
        out = out[y:y + wh, x:x + ww]
    return out


def coefficients(in_size, out_size, resample):
    """the tables of b200jpg_resample_coefficients for a cv id (| TABLE_VERTICAL, | TABLE_LINEAR) -> (bounds [2 out] int32,
    coeffs [out * ksize] int32, ksize). Rules 1 / 4: bounds = the two source indices, coeffs = the two int16 weights; rule 3:
    bounds = (first, taps), coeffs = the float32 weights' bits."""
    base = resample & 0xFFF
    vertical = bool(resample & TABLE_VERTICAL)
    if base == AREA and in_size >= out_size and not resample & TABLE_LINEAR:
        first, count, weights = area_table(in_size, out_size)
        bounds = np.stack([first, count], axis=1).reshape(-1).astype(np.int32)
        return bounds, weights.view(np.int32).reshape(-1).copy(), weights.shape[1]
    i0, i1, a0, a1 = linear_table(in_size, out_size, base == AREA, vertical)
    return (np.stack([i0, i1], axis=1).reshape(-1).astype(np.int32), np.stack([a0, a1], axis=1).reshape(-1).astype(np.int32), 2)
