"""Host-side mirror of the batch decode interface (include/b200jpg.h) for Python callers.

PyTorch is plumbing here: it owns the output tensor and the CUDA stream; every byte of decode work happens
in the hand-written kernels of libb200jpg.so.
"""
import ctypes
import math
import threading
from dataclasses import dataclass

import numpy as np

from . import native
from .native import lib


@dataclass
class FrameInfo:
    width: int
    height: int
    ncomp: int
    precision: int
    ycbcr: bool
    hs: tuple
    vs: tuple
    subx: tuple
    suby: tuple
    mcu_cols: int
    mcu_rows: int
    blocks_w: tuple
    blocks_h: tuple
    nscans: int
    restart_interval: int
    n_intervals: int
    ecs_bytes: int
    stored_blocks: int

    @staticmethod
    def from_struct(s):
        n = s.ncomp
        return FrameInfo(s.width, s.height, n, s.precision, bool(s.ycbcr), tuple(s.hs[:n]), tuple(s.vs[:n]),
                         tuple(s.subx[:n]), tuple(s.suby[:n]), s.mcu_cols, s.mcu_rows, tuple(s.blocks_w[:n]),
                         tuple(s.blocks_h[:n]), s.nscans, s.restart_interval, s.n_intervals, s.ecs_bytes,
                         s.stored_blocks)


def _as_buffer(data):
    """bytes / bytearray / numpy uint8 array -> (address, length, keepalive)."""
    if isinstance(data, np.ndarray):
        arr = np.ascontiguousarray(data, dtype=np.uint8)
        return arr.ctypes.data, arr.size, arr
    if hasattr(data, "data_ptr"):  # torch CPU tensor (possibly pinned)
        return data.data_ptr(), data.numel(), data
    buf = (ctypes.c_uint8 * len(data)).from_buffer_copy(data) if not isinstance(data, bytearray) else (
        ctypes.c_uint8 * len(data)).from_buffer(data)
    return ctypes.addressof(buf), len(data), buf


def parse(data):
    """Marker-level parse of one codestream on the host (no GPU). Raises NativeError on malformed input."""
    addr, n, keep = _as_buffer(data)
    s = native.FrameInfoStruct()
    rc = lib.b200jpg_parse(addr, n, ctypes.byref(s))
    native.check(rc)
    del keep
    return FrameInfo.from_struct(s)


def exif_orientation(data):
    """The Exif orientation 1..8 of one codestream (1 without a valid one), the value BatchDecoder(exif_orientation=True)
    applies; host only, no GPU. Raises NativeError where parse() does."""
    addr, n, keep = _as_buffer(data)
    rc = lib.b200jpg_exif_orientation(addr, n)
    del keep
    if rc < 0:
        native.check(rc)
    return rc


def colorspace(data):
    """The colour space BatchDecoder(mode=...) reads one codestream's samples in (b200jpg_colorspace, DESIGN §15): "L", "YCbCr",
    "RGB", "CMYK", "YCCK", or None for a frame a mode refuses (two components, four without an Adobe segment in front of the first
    scan, or four of 12 bits). Host only, no GPU. Raises NativeError where parse() does."""
    addr, n, keep = _as_buffer(data)
    rc = lib.b200jpg_colorspace(addr, n)
    del keep
    if rc < 0:
        native.check(rc)
    return native.COLORSPACES[rc]


def output_size(data, downscale=1, exif_orientation=False):
    """(h, w) of the whole output image of one codestream as BatchDecoder(frames, downscale=..., exif_orientation=...) writes it
    without a crop: the frame size divided by `downscale` (rounded up), height and width swapped for the Exif orientations 5..8
    when exif_orientation is set. The coordinates the `crop` rectangles of BatchDecoder are given in; host only, no GPU. Raises
    NativeError where parse() does."""
    if isinstance(downscale, bool) or not isinstance(downscale, int) or downscale not in native.DOWNSCALE_FLAGS:
        raise ValueError("downscale must be 1, 2, 4 or 8, got %r" % (downscale,))
    flags = native.DOWNSCALE_FLAGS[downscale] | (native.FLAG_EXIF_ORIENTATION if exif_orientation else 0)
    addr, n, keep = _as_buffer(data)
    w, h = ctypes.c_uint32(), ctypes.c_uint32()
    rc = lib.b200jpg_output_size(addr, n, flags, ctypes.byref(w), ctypes.byref(h))
    del keep
    native.check(rc)
    return h.value, w.value


def draft_scale(data, size):
    """Pillow's draft scale k (8, 4, 2 or 1) of one codestream for the requested size = (h, w) -- Image.draft(mode, (w, h)) takes
    (w, h) --, from the codestream's own size before any Exif orientation: the largest k <= min(W // w, H // h), 1 when none fits.
    BatchDecoder(frames, draft=size) decodes the frame at ceil(W / k) x ceil(H / k); output_size(data, downscale=k,
    exif_orientation=...) is then the image crop rectangles are given in. Host only, no GPU. Raises ValueError for a size that is
    not two positive integers, NativeError where parse() does."""
    import numbers
    hw = tuple(size) if isinstance(size, (tuple, list)) else None
    if hw is None or len(hw) != 2 or any(isinstance(v, bool) or not isinstance(v, numbers.Integral) for v in hw) or \
            any(v < 1 or v > 0xFFFFFFFF for v in hw):
        raise ValueError("draft size must be two integers (h, w) of 1 .. 2**32 - 1, got %r" % (size,))
    addr, n, keep = _as_buffer(data)
    rc = lib.b200jpg_draft_scale(addr, n, int(hw[1]), int(hw[0]))
    del keep
    if rc < 0:
        native.check(rc)
    return rc


def _hw(size, what):
    """(h, w) of two positive integers; raises ValueError"""
    import numbers
    hw = tuple(size) if isinstance(size, (tuple, list)) else None
    if hw is None or len(hw) != 2 or any(isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 1 for v in hw):
        raise ValueError("%s must be two positive integers (h, w), got %r" % (what, size))
    return int(hw[0]), int(hw[1])


def thumbnail_args(data, size, reducing_gap=2.0, exif_orientation=False):
    """The BatchDecoder entries of one codestream for Pillow's thumbnail, as a dict of "draft", "resize" and "box" (each None or
    the entry) -- host only, no GPU. size = (h, w); Image.thumbnail takes (w, h). With exif_orientation=False the chain is
        im = Image.open(f); im.thumbnail((w, h), reducing_gap=reducing_gap)
    and with exif_orientation=True (the batch's flag too) ImageOps.exif_transpose(Image.open(f)).thumbnail((w, h), ...), which
    draws no draft: exif_transpose has loaded the image. The batch takes resample="bicubic" and the same reducing_gap (None for
    None). An image already within the size is left untouched (every entry None), and a frame whose draft already has the
    thumbnail's size is drafted but not resized. The image the batch resizes is the frame's own, so this holds for grey and
    YCbCr frames under mode None or "RGB" (DESIGN §19). Raises ValueError, NativeError where parse() does."""
    h, w = _hw(size, "size")
    if reducing_gap is not None:
        reducing_gap_value(reducing_gap)
    H, W = output_size(data, exif_orientation=exif_orientation)
    out = {"draft": None, "resize": None, "box": None}
    if w >= W and h >= H:  # preserve_aspect_ratio: None
        return out
    aspect = W / H

    def round_aspect(number, key):
        return max(min(math.floor(number), math.ceil(number), key=key), 1)

    x, y = w, h
    if x / y >= aspect:
        x = round_aspect(y * aspect, key=lambda n: abs(aspect - n / y))
    else:
        y = round_aspect(x / aspect, key=lambda n: 0 if n == 0 else abs(aspect - x / n))
    cur_h, cur_w = H, W
    if reducing_gap is not None and not exif_orientation:
        dh, dw = int(h * reducing_gap), int(w * reducing_gap)
        k = draft_scale(data, (dh, dw))
        out["draft"] = (dh, dw)
        cur_h, cur_w = (H + k - 1) // k, (W + k - 1) // k
        out["box"] = (0.0, 0.0, W / k, H / k)
    if (cur_w, cur_h) != (x, y):
        out["resize"] = (y, x)
    else:
        out["box"] = None
    return out


def fit_args(data, size, bleed=0.0, centering=(0.5, 0.5), exif_orientation=False):
    """The BatchDecoder entries of one codestream for ImageOps.fit(im, (w, h), bleed=bleed, centering=centering) of the image the
    batch writes without a size (Image.open(f), or its exif_transpose with exif_orientation=True), as a dict of "resize" and "box":
    Pillow's own box arithmetic, including its fallbacks (a centering outside [0, 1] is 0.5, a bleed outside [0, 0.5) is 0). The
    batch takes resample="bicubic" (fit's default method) and no reducing_gap. size = (h, w). Host only; raises ValueError,
    NativeError where parse() does."""
    h, w = _hw(size, "size")
    H, W = output_size(data, exif_orientation=exif_orientation)
    cx, cy = centering
    if not 0.0 <= cx <= 1.0:
        cx = 0.5
    if not 0.0 <= cy <= 1.0:
        cy = 0.5
    if not 0.0 <= bleed < 0.5:
        bleed = 0.0
    bx, by = bleed * W, bleed * H
    lw, lh = W - bx * 2, H - by * 2
    live_ratio, out_ratio = lw / lh, w / h
    if live_ratio == out_ratio:
        cw, ch = lw, lh
    elif live_ratio >= out_ratio:
        cw, ch = out_ratio * lh, lh
    else:
        cw, ch = lw, lw / out_ratio
    left, top = bx + (lw - cw) * cx, by + (lh - ch) * cy
    return {"resize": (h, w), "box": (left, top, left + cw, top + ch)}


def resize_center_crop_args(data, resize, crop, exif_orientation=False):
    """The BatchDecoder entries of one codestream for torchvision's Resize(resize) then CenterCrop(crop) on the PIL image the batch
    writes without a size, as a dict of "resize" and "window". resize is an int (the shorter side: the longer becomes
    int(resize * long / short)) or (h, w); crop an int or (h, w). The window is at (int(round((W_r - w) / 2)), int(round((H_r - h)
    / 2))) of the resized W_r x H_r image, Python's round. The batch takes resample="bilinear" (Resize's default) and no
    reducing_gap. A crop larger than the resized image raises ValueError: torchvision pads there. Host only; NativeError where
    parse() does."""
    import numbers
    H, W = output_size(data, exif_orientation=exif_orientation)
    if isinstance(resize, numbers.Integral) and not isinstance(resize, bool):
        if resize < 1:
            raise ValueError("resize must be positive, got %r" % (resize,))
        short, long = (W, H) if W <= H else (H, W)
        new_short, new_long = int(resize), int(resize * long / short)
        rw, rh = (new_short, new_long) if W <= H else (new_long, new_short)
    else:
        rh, rw = _hw(resize, "resize")
    if isinstance(crop, numbers.Integral) and not isinstance(crop, bool):
        crop = (crop, crop)
    ch, cw = _hw(crop, "crop")
    if ch > rh or cw > rw:
        raise ValueError("crop %d x %d is larger than the resized %d x %d image (torchvision pads there)" % (ch, cw, rh, rw))
    top, left = int(round((rh - ch) / 2.0)), int(round((rw - cw) / 2.0))
    return {"resize": (rh, rw), "window": (left, top, cw, ch)}


def crop_table(crop, n, name="crop"):
    """The b200jpg_rect table of BatchDecoder(crop=...) (or of `name`=..., window): n entries, each None (the whole frame) or (x, y,
    width, height) as non-negative integers. Raises ValueError; the rectangles themselves are checked against the frames by the
    batch."""
    import numbers
    if len(crop) != n:
        raise ValueError("%s: %d rectangles for %d frames" % (name, len(crop), n))
    table = (native.RectStruct * n)()
    for i, r in enumerate(crop):
        if r is None:
            continue
        vals = tuple(r)
        if len(vals) != 4 or any(isinstance(v, bool) or not isinstance(v, numbers.Integral) for v in vals):
            raise ValueError("%s[%d]: expected None or four integers (x, y, width, height), got %r" % (name, i, r))
        if any(v < 0 or v > 0xFFFFFFFF for v in vals):
            raise ValueError("%s[%d]: x, y, width and height must be 0 .. 2**32 - 1, got %r" % (name, i, vals))
        table[i].x, table[i].y, table[i].width, table[i].height = (int(v) for v in vals)
    return table


def flip_table(hflip, vflip, n):
    """The flips of b200jpg_batch_create_flip for BatchDecoder(hflip=..., vflip=...): each of hflip and vflip is None, one bool
    for every frame, or a sequence of n bools. None when no frame is flipped (the batch of b200jpg_batch_create_resample). Raises
    ValueError for a wrong length or a value that is not a bool."""
    def is_bool(v):
        return isinstance(v, (bool, np.bool_))

    table = (ctypes.c_uint8 * n)()
    for name, arg, bit in (("hflip", hflip, native.FLIP_H), ("vflip", vflip, native.FLIP_V)):
        if arg is None:
            continue
        if is_bool(arg):
            arg = [arg] * n
        elif isinstance(arg, (str, bytes)) or not hasattr(arg, "__len__"):
            raise ValueError("%s must be None, a bool or one bool per frame, got %r" % (name, arg))
        if len(arg) != n:
            raise ValueError("%s: %d entries for %d frames" % (name, len(arg), n))
        for i, v in enumerate(arg):
            if not is_bool(v):
                raise ValueError("%s[%d]: expected a bool, got %r" % (name, i, v))
            if v:
                table[i] |= bit
    return table if any(table) else None


def resize_table(resize, n, name="resize"):
    """The b200jpg_size table of BatchDecoder(resize=...) (or of `name`=..., draft): one (h, w) for every frame, or n entries each
    None or (h, w), as non-negative integers; (0, 0) leaves a frame unresized (undrafted). Raises ValueError."""
    import numbers

    def is_int(v):
        return not isinstance(v, bool) and isinstance(v, numbers.Integral)

    vals = tuple(resize)
    if len(vals) == 2 and all(is_int(v) for v in vals):
        vals = (vals,) * n
    elif len(vals) != n:
        raise ValueError("%s: %d sizes for %d frames" % (name, len(vals), n))
    table = (native.SizeStruct * n)()
    for i, r in enumerate(vals):
        if r is None:
            continue
        hw = tuple(r) if isinstance(r, (tuple, list)) else None
        if hw is None or len(hw) != 2 or not all(is_int(v) for v in hw):
            raise ValueError("%s[%d]: expected None or two integers (h, w), got %r" % (name, i, r))
        if any(v < 0 or v > 0xFFFFFFFF for v in hw):
            raise ValueError("%s[%d]: h and w must be 0 .. 2**32 - 1, got %r" % (name, i, hw))
        if (hw[0] == 0) != (hw[1] == 0):
            raise ValueError("%s[%d]: exactly one of h and w is zero: %r" % (name, i, hw))
        table[i].height, table[i].width = int(hw[0]), int(hw[1])
    return table


def box_table(box, n):
    """The b200jpg_box table of BatchDecoder(box=...): n entries, each None (the default box) or (x0, y0, x1, y1) as finite real
    numbers, Pillow's Image.resize(box=...) order. Raises ValueError; the boxes themselves are checked against the frames by the
    batch."""
    import math
    import numbers
    if len(box) != n:
        raise ValueError("box: %d boxes for %d frames" % (len(box), n))
    table = (native.BoxStruct * n)()
    for i, b in enumerate(box):
        if b is None:
            continue
        vals = tuple(b) if isinstance(b, (tuple, list)) else None
        if vals is None or len(vals) != 4 or any(isinstance(v, bool) or not isinstance(v, numbers.Real) for v in vals):
            raise ValueError("box[%d]: expected None or four numbers (x0, y0, x1, y1), got %r" % (i, b))
        if not all(math.isfinite(v) for v in vals):
            raise ValueError("box[%d]: every coordinate must be finite, got %r" % (i, vals))
        if vals[0] < 0 or vals[1] < 0 or vals[2] < vals[0] or vals[3] < vals[1]:
            raise ValueError("box[%d]: expected 0 <= x0 <= x1 and 0 <= y0 <= y1, got %r" % (i, vals))
        table[i].x0, table[i].y0, table[i].x1, table[i].y1 = (float(v) for v in vals)
    return table


def reducing_gap_value(gap):
    """The reducing_gap of b200jpg_batch_create_resample: 0.0 for None, else a real number of at least 1.0. Raises ValueError."""
    import numbers
    if gap is None:
        return 0.0
    if isinstance(gap, bool) or not isinstance(gap, numbers.Real) or not gap >= 1.0:
        raise ValueError("reducing_gap must be None or a number >= 1.0, got %r" % (gap,))
    return float(gap)


def resample_filter(name):
    """B200JPG_RESAMPLE_* of a filter name: Pillow's "box", "bilinear", "hamming", "bicubic" or "lanczos", or OpenCV's
    "cv2-linear" or "cv2-area" (INTER_LINEAR / INTER_AREA, DESIGN §20). Raises ValueError."""
    if not isinstance(name, str) or name not in native.RESAMPLE:
        raise ValueError("resample must be one of %s, got %r" % (", ".join(sorted(native.RESAMPLE)), name))
    return native.RESAMPLE[name]


def component_shapes(info, upsample=True):
    """[(h, w)] of every component of a frame as the decoder writes it: the frame size, or without upsampling each
    component's own ceil(H / suby) x ceil(W / subx)."""
    if upsample:
        return [(info.height, info.width)] * info.ncomp
    return [((info.height + info.suby[c] - 1) // info.suby[c], (info.width + info.subx[c] - 1) // info.subx[c])
            for c in range(info.ncomp)]


def _sample_types():
    """torch float dtype -> B200JPG_SAMPLE_* of the float destinations"""
    import torch
    return {torch.float32: native.SAMPLE_F32, torch.float16: native.SAMPLE_F16, torch.bfloat16: native.SAMPLE_BF16}


def _check_dtype(dtype, deep, first, where):
    """integer destinations: uint8 for 8-bit, int16 for 12-bit frames; float destinations: any frame, one dtype per call
    (`first` = the dtype of the call's first tensor)"""
    import torch
    floats = _sample_types()
    if (dtype in floats or first in floats) and dtype != first:
        raise TypeError("%sdtype %s, but the call's first destination is %s: one float dtype per call" % (where, dtype, first))
    want = torch.int16 if deep else torch.uint8
    if dtype not in floats and dtype != want:
        raise TypeError("%sdtype %s, expected %s" % (where, dtype, want))


def destination_dtype(dst):
    """The dtype of the first tensor of a decode_into destination (None when it holds no tensor)."""
    if hasattr(dst, "dtype"):
        return dst.dtype
    for entry in dst:
        for t in entry or ():
            return getattr(t, "dtype", None)
    return None


def table_args(dtype, table, ncomp=1):
    """The b200jpg_convert_table of a decode_into call into `dtype` tensors with `table`, a [C, 256] float32 tensor or array
    (ncomp <= C <= 4, ncomp: the most output components a live frame of the batch has): row c maps the samples of output
    component c. Raises TypeError for an integer destination or a table that is not float32, ValueError for a table of another
    shape or with fewer rows than the batch's components."""
    floats = _sample_types()
    if dtype not in floats:
        raise TypeError("a sample table needs a float32, float16 or bfloat16 destination, not %s" % dtype)
    if hasattr(table, "detach"):
        table = table.detach().cpu().numpy()
    a = np.asarray(table)
    if a.dtype != np.float32:
        raise TypeError("the sample table must be float32, got %s" % a.dtype)
    if a.ndim != 2 or a.shape[1] != 256 or not 1 <= a.shape[0] <= 4:
        raise ValueError("the sample table must be [C, 256] with C <= 4, got %s" % (a.shape,))
    if a.shape[0] < ncomp:
        raise ValueError("the sample table has %d rows, but frames of the batch are written with %d components: one row per "
                         "component" % (a.shape[0], ncomp))
    t = native.ConvertTableStruct()
    t.type = floats[dtype]
    ctypes.memmove(ctypes.addressof(t.table), np.ascontiguousarray(a).ctypes.data, a.nbytes)
    return t


def sample_table(fn, ncomp=3):
    """The [ncomp, 256] float32 sample table of decode_into(..., table=...) that a per-sample transform gives: fn runs once on the
    [ncomp, 1, 256] uint8 CPU tensor of every sample value (each component's row is arange(256)) and returns a tensor of the same
    shape, whose values become the table. For torchvision's ToTensor() + Normalize(mean, std):
        sample_table(lambda t: TF.normalize(t.float().div(255), mean, std))
    fn must act sample by sample (component c of sample v -> one value): a transform that mixes samples, like a blur or a
    resize, has no table."""
    import torch
    if isinstance(ncomp, bool) or not isinstance(ncomp, int) or not 1 <= ncomp <= 4:
        raise ValueError("ncomp must be 1 .. 4, got %r" % (ncomp,))
    x = torch.arange(256, dtype=torch.uint8).view(1, 1, 256).expand(ncomp, 1, 256).contiguous()
    y = torch.as_tensor(fn(x)).detach().cpu()  # (fn may return a CUDA tensor, or one that requires grad)
    if tuple(y.shape) != (ncomp, 1, 256):
        raise ValueError("fn must return a [%d, 1, 256] tensor, got %s" % (ncomp, tuple(y.shape)))
    return y.reshape(ncomp, 256).to(torch.float32).numpy()


def convert_args(dtype, scale=None, bias=None, ncomp=4):
    """The b200jpg_convert of a decode_into call into `dtype` tensors: None for uint8 / int16 destinations (scale and bias
    must then be left out), else the element type and the map y = v * scale[c] + bias[c]. scale and bias are a scalar, which
    applies to every component, or one value per component (ncomp of them); the defaults are 1 and 0. Both are rounded to
    float32 and must be finite there. Raises ValueError / TypeError."""
    import numbers
    floats = _sample_types()
    if dtype not in floats:
        if scale is not None or bias is not None:
            raise TypeError("scale and bias need a float32, float16 or bfloat16 destination, not %s" % dtype)
        return None
    c = native.ConvertStruct()
    c.type = floats[dtype]
    for name, v, default in (("scale", scale, 1.0), ("bias", bias, 0.0)):
        if v is None:
            vals = [default] * 4
        elif isinstance(v, numbers.Real) or getattr(v, "ndim", None) == 0:
            vals = [float(v)] * 4
        else:
            vals = [float(x) for x in v]
            if len(vals) != ncomp:
                raise ValueError("%s: %d values for %d components" % (name, len(vals), ncomp))
            vals += [default] * (4 - ncomp)
        with np.errstate(over="ignore"):
            f32 = np.asarray(vals, dtype=np.float32)
        if not np.isfinite(f32).all():
            raise ValueError("%s must be finite in float32, got %s" % (name, vals[:ncomp]))
        getattr(c, name)[:] = [float(x) for x in f32]
    return c


def plane_table(geometry, dst, device_type="cuda"):
    """The b200jpg_plane table of BatchDecoder.decode_into (4 entries per frame).

    geometry[i] = (component shapes [(h, w)], deep) of frame i, or None for a frame that failed to parse. dst[i] is a
    sequence of one 2-D tensor per component (a [C, H, W] tensor is one), uint8 for 8-bit and int16 for 12-bit (`deep`)
    frames, or float32 / float16 / bfloat16 for any frame (one of them for the whole call), or None where geometry[i] is
    None. Component c's sample (x, y) goes to t[y, x]: bytes_per_pixel = stride(1) * itemsize, bytes_per_row = stride(0) *
    itemsize. Raises ValueError / TypeError on a wrong count, shape, dtype or device; nothing has been launched then."""
    import torch
    n = len(geometry)
    if len(dst) != n:
        raise ValueError("decode_into: %d destinations for %d frames" % (len(dst), n))
    if isinstance(dst, torch.Tensor) and dst.dim() == 4:
        return _batch_tensor_table(geometry, dst, device_type)
    table = (native.PlaneStruct * (4 * n))()
    first = None
    for i, (geo, entry) in enumerate(zip(geometry, dst)):
        if geo is None:
            if entry is not None:
                raise ValueError("frame %d failed to parse: its destination must be None" % i)
            continue
        if entry is None:
            raise ValueError("frame %d needs a destination" % i)
        shapes, deep = geo
        if len(entry) != len(shapes):
            raise ValueError("frame %d has %d components, its destination %d" % (i, len(shapes), len(entry)))
        for c, t in enumerate(entry):
            if not isinstance(t, torch.Tensor):
                raise TypeError("frame %d component %d: expected a tensor, got %s" % (i, c, type(t).__name__))
            if t.device.type != device_type:
                raise ValueError("frame %d component %d: a %s tensor, expected %s" % (i, c, t.device.type, device_type))
            first = t.dtype if first is None else first
            _check_dtype(t.dtype, deep, first, "frame %d component %d: " % (i, c))
            if tuple(t.shape) != tuple(shapes[c]):
                raise ValueError("frame %d component %d: shape %s, expected %s" % (i, c, tuple(t.shape), tuple(shapes[c])))
            e = table[4 * i + c]
            e.data = t.data_ptr()
            e.bytes_per_pixel = t.stride(1) * t.element_size()
            e.bytes_per_row = t.stride(0) * t.element_size()
    return table


def _batch_tensor_table(geometry, t, device_type):
    """plane_table for one [N, C, H, W] tensor, without a view per component (a batch of thousands of frames would spend
    longer building views than the GPU spends decoding it)"""
    import torch
    live = [i for i, g in enumerate(geometry) if g is not None]
    if not live:
        return (native.PlaneStruct * (4 * len(geometry)))()
    shapes, deep = geometry[live[0]]
    same_depth = t.dtype not in _sample_types()  # a float tensor takes 8- and 12-bit frames alike
    if any(geometry[i][0] != shapes or (same_depth and geometry[i][1] != deep) for i in live) or len(set(shapes)) != 1:
        raise ValueError("a [N, C, H, W] destination needs frames of one geometry")
    want = (len(geometry), len(shapes)) + tuple(shapes[0])
    if t.device.type != device_type:
        raise ValueError("a %s tensor, expected %s" % (t.device.type, device_type))
    _check_dtype(t.dtype, deep, t.dtype, "")
    if tuple(t.shape) != want:
        raise ValueError("shape %s, expected %s" % (tuple(t.shape), want))
    arr = np.zeros(4 * len(geometry), dtype=np.dtype([("data", "<u8"), ("bpp", "<i4"), ("pad", "<i4"), ("bpr", "<i8")]))
    assert arr.itemsize == ctypes.sizeof(native.PlaneStruct)
    isz, st, idx = t.element_size(), t.stride(), np.asarray(live, dtype=np.int64)
    for c in range(len(shapes)):
        arr["data"][4 * idx + c] = t.data_ptr() + (idx * st[0] + c * st[1]) * isz
        arr["bpp"][4 * idx + c] = st[3] * isz
        arr["bpr"][4 * idx + c] = st[2] * isz
    return (native.PlaneStruct * (4 * len(geometry))).from_buffer_copy(arr.tobytes())


class Context:
    def __init__(self, device=-1):
        self.handle = ctypes.c_void_p()
        self._batches = 0  # live BatchDecoders on this context (batches may be created on several threads: under the lock)
        self._closing = False
        self._lock = threading.Lock()
        rc = lib.b200jpg_create(device, ctypes.byref(self.handle))
        native.check(rc)

    def trim(self):
        """Returns the pooled (idle) device / pinned buffers to the driver."""
        if self.handle:
            lib.b200jpg_trim(self.handle)

    def close(self):
        """Destroys the context; with batches still open, when the last of them closes: a batch returns its buffers to the
        context's pool. (The garbage collector may finalise a context before the batches of the same reference cycle.)"""
        lock = getattr(self, "_lock", None)
        if lock is None:  # b200jpg_create failed
            return
        with lock:
            if self._batches:
                self._closing = True
                return
            if self.handle:
                lib.b200jpg_destroy(self.handle)
                self.handle = ctypes.c_void_p()

    def _batch_opened(self):
        with self._lock:
            self._batches += 1

    def _batch_closed(self):
        with self._lock:
            self._batches -= 1
            if not (self._closing and self._batches == 0):
                return
            self._closing = False
        self.close()

    def __del__(self):
        self.close()


class BatchDecoder:
    """One batch of codestreams: parse + pack on construction, then upload() / decode() on a CUDA stream."""

    def __init__(self, frames, device=-1, tolerate_bad=False, ctx=None, color_transform=True, upsample=True, downscale=1,
                 exif_orientation=False, crop=None, resize=None, resample="bilinear", mode=None, reconstruction="reference", draft=None,
                 box=None, reducing_gap=None, window=None, hflip=None, vflip=None):
        """downscale = 2, 4 or 8 decodes every frame at ceil(W / k) x ceil(H / k) (B200JPG_FLAG_DOWNSCALE_k): each 8x8 block is
        inverse transformed straight to (8/k) x (8/k) samples, the k x k box average of its IDCT, and the rest of the
        reconstruction runs on the smaller frame. geometry(), frame_view() and plane_views() give the reduced sizes. Not to be
        confused with the `scale` of decode_into, which maps sample values.

        exif_orientation=True (B200JPG_FLAG_EXIF_ORIENTATION) writes every frame as its Exif-oriented image, what PIL's
        ImageOps.exif_transpose gives: mirrored and rotated in the reconstruction's store, width and height swapped for the
        orientations 5..8. output_shape(), geometry(), frame_view(), plane_views() and the destinations of decode_into() are
        then in oriented shapes. orientation(i) gives a frame's Exif value either way.

        crop (b200jpg_batch_create_crop) is one entry per frame: None for the whole frame, or (x, y, width, height) -- the order
        of b200jpg_rect -- a rectangle of the frame's output image after downscaling and Exif orientation (output_size() gives that
        image's (h, w)). The frame is then written as exactly out[y:y + height, x:x + width] of its uncropped output, bit for bit,
        and output_shape(), geometry(), frame_view() and the destinations of decode_into() are the rectangle's. Only the tiles
        under the rectangle are reconstructed; every scan is still decoded, and status(i) is the frame's status without the
        crop. A rectangle that is empty or leaves the frame raises NativeError (B200JPG_ERR_INVALID_PARAMETER), as does a
        crop with upsample=False (B200JPG_ERR_NOT_IMPLEMENTED); a wrong length or an entry that is not four non-negative
        integers raises ValueError.

        resize (b200jpg_batch_create_resize) is one (h, w) for every frame, or one entry per frame: None, or (h, w). The frame's
        output -- after downscaling, Exif orientation and the crop -- is then resized to h x w with `resample`, one of "box",
        "bilinear", "hamming", "bicubic" and "lanczos": bit for bit what PIL's Image.resize((w, h), filter) gives for that uint8
        image (DESIGN §13), and a float destination of decode_into() receives the resized samples through its map; OpenCV's
        "cv2-linear" and "cv2-area" are described below.
        output_shape(), geometry(), frame_view() and the destinations of decode_into() are then h x w, so one [N, C, h, w] tensor
        takes frames of any size. status(i) is the frame's status without the size; a 12-bit frame with a size is
        B200JPG_ERR_NOT_IMPLEMENTED, and a size with upsample=False raises NativeError (B200JPG_ERR_NOT_IMPLEMENTED). A wrong length,
        an entry that is not two non-negative integers, exactly one zero in a size or an unknown filter name raises ValueError.

        mode (B200JPG_FLAG_OUTPUT_RGB / _L, DESIGN §14), named after PIL's Image.convert(mode): None writes every frame with its own
        components; "RGB" writes every frame with three -- a grey frame's sample in all three, as convert("RGB") does -- and "L"
        with one: a YCbCr frame's luma (the component 0 that color_transform=False gives, reconstructed without its chroma), an
        RGB-coded or JPEG XT frame's (19595 R + 38470 G + 7471 B + 32768) >> 16, as convert("L") does. The mode comes before the
        orientation, the crop, the resize and the float map (scale[c] / bias[c] of the output component c), so a batch of grey and
        colour frames fills one [N, 3, H, W] tensor. output_components(i) gives the count; geometry(), frame_view() and the
        destinations of decode_into() follow it. A CMYK or YCCK frame (an 8-bit four-component frame with an Adobe segment,
        colorspace(data); DESIGN §15) is written as Pillow's convert("RGB") / convert("L") of the image it reads as Adobe-inverted
        CMYK. A frame colorspace() gives None for -- two components, four without an Adobe segment or of 12 bits -- is then
        B200JPG_ERR_NOT_IMPLEMENTED (skipped with tolerate_bad); a mode with color_transform=False raises NativeError (B200JPG_ERR_INVALID_PARAMETER), with upsample=False
        NativeError (B200JPG_ERR_NOT_IMPLEMENTED); any other value than None, "RGB" and "L" raises ValueError.

        reconstruction (B200JPG_FLAG_LIBJPEG_TURBO, DESIGN §16): "reference" (the default) reconstructs as the reference decoder
        does; "libjpeg-turbo" as libjpeg-turbo does, so as Pillow's Image.open(f) -- its islow IDCT, fancy upsampling and YCbCr ->
        RGB conversion -- with "L" of a YCbCr frame as Pillow's draft("L") and a JPEG XT frame as its base codestream alone.
        Orientation, crop, resize and the float map follow unchanged, so Image.open(f).convert("RGB").crop(box).resize(size)
        is what the GPU writes, byte for byte, for intact codestreams. Under mode "RGB" or "L" that holds for CMYK and YCCK frames
        too (DESIGN §18): libjpeg-turbo's IDCT and upsampling of all four components, then §15's conversion, as Pillow's
        convert(mode) of the "CMYK" image it opens. A 12-bit or two-component frame, a four-component frame without a mode and
        one colorspace() gives None for are then B200JPG_ERR_NOT_IMPLEMENTED (skipped with tolerate_bad); "libjpeg-turbo" with
        downscale > 1 or upsample=False raises
        NativeError (B200JPG_ERR_NOT_IMPLEMENTED); any other value raises ValueError before a device is touched.

        draft (b200jpg_batch_create_draft, DESIGN §17) is one (h, w) for every frame, or one entry per frame: None, or (h, w) -- the
        order of `resize`; Pillow's Image.draft(mode, (w, h)) takes (w, h). A frame with a request is decoded as Pillow's draft gives
        it: at scale 1/k, k = draft_scale(data, (h, w)) of 8, 4, 2 and 1 from the codestream's own size, ceil(W / k) x ceil(H / k),
        with libjpeg-turbo's reduced IDCTs and its upsampling at that scale. Everything else follows on that image, so for intact
        codestreams the batch writes, byte for byte, what
            im = Image.open(f); im.draft(mode, (w, h))
            ImageOps.exif_transpose(im).convert(mode).crop(box).resize(size, filter)
        gives, CMYK and YCCK frames under a mode included (their four components at their reduced IDCT sizes, DESIGN §18); crop
        rectangles are given in output_size(data, downscale=k, exif_orientation=...). A frame whose k is 1 is decoded
        exactly as without a draft; status(i) is unchanged. A draft needs reconstruction="libjpeg-turbo" (else NativeError,
        B200JPG_ERR_NOT_IMPLEMENTED); a wrong length, an entry that is not two non-negative integers or exactly one zero in an
        entry raises ValueError.

        box, reducing_gap and window (b200jpg_batch_create_resample, DESIGN §19) are the rest of Pillow's Image.resize, for frames
        with a `resize` entry. box is one entry per frame: None, or Pillow's (x0, y0, x1, y1) in floats, in the coordinates of the
        image the resize takes (after draft, downscaling, Exif orientation and the crop). reducing_gap is None or a number >= 1.0
        for the whole batch, Pillow's reducing_gap: Image.reduce() runs first when the box is at least twice `gap` times the
        target. window is one entry per frame: None, or (x, y, width, height) -- the order of `crop` -- a rectangle of the resized
        h x w image. The frame is then written as, byte for byte,
            Image.fromarray(C).resize((w, h), filter, box=box, reducing_gap=gap).crop((x, y, x + width, y + height))
        of its image C without the size, and output_shape() and the destinations of decode_into() are the window's (height, width),
        so a Resize(256) + CenterCrop(224) batch fills one [N, 3, 224, 224] tensor. Only the part of C the resize reads is
        reconstructed. thumbnail_args(), fit_args() and resize_center_crop_args() give the entries of Pillow's thumbnail(),
        ImageOps.fit() and torchvision's Resize + CenterCrop. A box or window on a frame without a size, a box outside C, a window
        outside h x w, or a reduce box that is empty raises NativeError (B200JPG_ERR_INVALID_PARAMETER); a wrong length, an entry
        of the wrong form, a box that is not finite or has x1 < x0 or y1 < y0 and a reducing_gap below 1.0 raise ValueError.

        resample="cv2-linear" or "cv2-area" (B200JPG_RESAMPLE_CV_LINEAR / _CV_AREA, DESIGN §20) resizes as OpenCV does instead of
        Pillow: the frame is written, byte for byte, as
            cv2.resize(C, (w, h), interpolation=cv2.INTER_LINEAR or cv2.INTER_AREA)[y:y + height, x:x + width]
        of OpenCV 4.13, with C the frame's image without the size and (x, y, width, height) the window (the whole h x w image
        without one). With reconstruction="libjpeg-turbo", C of a YCbCr or grey frame is cv2.imdecode(data, IMREAD_COLOR)
        in RGB order (IMREAD_GRAYSCALE under mode "L"), so an OpenCV loader's pixels come out unchanged; a BGR tensor is a
        decode_into() with the planes in the other order. cv2.resize has no box and no reducing_gap: either with a cv2 filter
        raises NativeError (B200JPG_ERR_INVALID_PARAMETER).

        hflip and vflip (b200jpg_batch_create_flip, DESIGN §21) are None, one bool for every frame, or one bool per frame:
        torchvision's RandomHorizontalFlip / RandomVerticalFlip with the coin already tossed. The flip is the last geometric step,
        after the resize and the window: a frame whose output without it is O ([h, w, C]) is written as O[:, ::-1] with hflip,
        O[::-1, :] with vflip and O[::-1, ::-1] with both, so hflip(img.crop(box).resize(size)) fills the batch tensor with no pass
        of its own. crop, box and window keep the coordinates of the unflipped image; output_shape(), status() and orientation()
        do not change. A frame without a size is reconstructed mirrored (the flip composed with its Exif orientation); a resized
        frame's resample pass stores mirrored, with the launches of the unflipped batch. A wrong length or a value that is not a
        bool raises ValueError."""
        if not isinstance(mode, (str, type(None))) or mode not in native.MODE_FLAGS:
            raise ValueError('mode must be None, "RGB" or "L", got %r' % (mode,))
        if not isinstance(reconstruction, str) or reconstruction not in native.RECONSTRUCTION_FLAGS:
            raise ValueError('reconstruction must be "reference" or "libjpeg-turbo", got %r' % (reconstruction,))
        if isinstance(downscale, bool) or not isinstance(downscale, int) or downscale not in native.DOWNSCALE_FLAGS:
            raise ValueError("downscale must be 1, 2, 4 or 8, got %r" % (downscale,))
        rects = None if crop is None else crop_table(crop, len(frames))
        sizes = None if resize is None else resize_table(resize, len(frames))
        drafts = None if draft is None else resize_table(draft, len(frames), "draft")
        boxes = None if box is None else box_table(box, len(frames))
        windows = None if window is None else crop_table(window, len(frames), "window")
        gap = reducing_gap_value(reducing_gap)
        filt = resample_filter(resample)
        flips = flip_table(hflip, vflip, len(frames))
        self.ctx = ctx or Context(device)
        self._keep = []
        n = len(frames)
        ptrs = (ctypes.c_void_p * n)()
        lens = (ctypes.c_size_t * n)()
        for i, f in enumerate(frames):
            addr, ln, keep = _as_buffer(f)
            ptrs[i] = addr
            lens[i] = ln
            self._keep.append(keep)
        self.handle = ctypes.c_void_p()
        flags = 0 if color_transform else 1  # B200JPG_FLAG_NO_COLOR_TRANSFORM (JPGTAG_MATRIX_LTRAFO = none)
        if not upsample:
            flags = 3  # B200JPG_FLAG_NO_UPSAMPLE (JPGTAG_DECODER_UPSAMPLE = false): planes, no colour transformation
        self.upsample = bool(upsample)
        self.downscale = downscale
        flags |= native.DOWNSCALE_FLAGS[downscale]
        self.exif_orientation = bool(exif_orientation)
        if exif_orientation:
            flags |= native.FLAG_EXIF_ORIENTATION
        self.mode = mode
        flags |= native.MODE_FLAGS[mode]
        self.reconstruction = reconstruction
        flags |= native.RECONSTRUCTION_FLAGS[reconstruction]
        rc = lib.b200jpg_batch_create_flip(self.ctx.handle, ptrs, lens, n, int(tolerate_bad), flags, drafts, rects, sizes, boxes, windows,
                                           filt, gap, flips, ctypes.byref(self.handle))
        native.check(rc, self.ctx.handle)
        self.ctx._batch_opened()
        self._keep = []  # the batch holds its own pinned copy
        self.n = n
        self.out_bytes = lib.b200jpg_batch_out_bytes(self.handle, -1)

    # ---- geometry ----------------------------------------------------------------------------------
    def info(self, i):
        s = native.FrameInfoStruct()
        lib.b200jpg_batch_frame_info(self.handle, i, ctypes.byref(s))
        return FrameInfo.from_struct(s)

    def output_shape(self, i, c):
        """(h, w) of component c of frame i as decode() / decode_into() write it: the frame size divided by `downscale`
        (rounded up), or without upsampling the component's own size; the rectangle's size for a cropped frame, the target size
        for a resized one. Raises NativeError for a frame that failed."""
        w, h = ctypes.c_uint32(), ctypes.c_uint32()
        native.check(lib.b200jpg_batch_output_extent(self.handle, i, c, ctypes.byref(w), ctypes.byref(h)), self.ctx.handle)
        return h.value, w.value

    def output_components(self, i):
        """The number of components frame i is written with: its own without a mode, 3 with mode="RGB", 1 with mode="L". Raises
        NativeError for a frame that failed."""
        rc = lib.b200jpg_batch_output_components(self.handle, i)
        if rc < 0:
            native.check(rc, self.ctx.handle)
        return rc

    def _components(self, i, fi):
        """output_components, or for a frame that failed the component count of its partial frame info"""
        rc = lib.b200jpg_batch_output_components(self.handle, i)
        return rc if rc > 0 else fi.ncomp

    def orientation(self, i):
        """Frame i's Exif orientation 1..8, whether or not the batch applies it; the (negative) status of a frame that failed."""
        return lib.b200jpg_batch_frame_orientation(self.handle, i)

    def _shape(self, i, c, fi):
        """output_shape, or for a frame that failed the shape its partial frame info gives (such a frame has no samples)"""
        w, h = ctypes.c_uint32(), ctypes.c_uint32()
        if lib.b200jpg_batch_output_extent(self.handle, i, c, ctypes.byref(w), ctypes.byref(h)) != 0:
            shapes = component_shapes(fi, self.upsample)
            return shapes[c] if c < len(shapes) else (fi.height, fi.width)
        return h.value, w.value

    def out_offset(self, i):
        return lib.b200jpg_batch_out_offset(self.handle, i)

    def frame_bytes(self, i):
        return lib.b200jpg_batch_out_bytes(self.handle, i)

    @property
    def ecs_bytes(self):
        return lib.b200jpg_batch_ecs_bytes(self.handle)

    @property
    def stored_blocks(self):
        return lib.b200jpg_batch_stored_blocks(self.handle)

    @property
    def h2d_bytes(self):
        return lib.b200jpg_batch_h2d_bytes(self.handle)

    # ---- tables (multi-GPU broadcast) --------------------------------------------------------------
    def export_tables(self):
        size = lib.b200jpg_batch_export_tables(self.handle, None, 0)
        if size == 0:
            raise native.NativeError(-1024, "batch does not have exactly one table set")
        buf = np.zeros(size, dtype=np.uint8)
        lib.b200jpg_batch_export_tables(self.handle, buf.ctypes.data, size)
        return buf

    def import_tables(self, blob):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        native.check(lib.b200jpg_batch_import_tables(self.handle, blob.ctypes.data, blob.size), self.ctx.handle)

    # ---- device work ---------------------------------------------------------------------------------
    @staticmethod
    def _stream_ptr(stream):
        if stream is None:
            import torch
            return torch.cuda.current_stream().cuda_stream
        if hasattr(stream, "cuda_stream"):
            return stream.cuda_stream
        return int(stream)

    def upload(self, stream=None):
        native.check(lib.b200jpg_batch_upload(self.handle, self._stream_ptr(stream)), self.ctx.handle)

    def reindex(self, stream=None):
        """Re-runs the device-side restart index alone (upload() already built it); for timing."""
        native.check(lib.b200jpg_batch_reindex(self.handle, self._stream_ptr(stream)), self.ctx.handle)

    def new_output(self, device=None):
        import torch
        return torch.empty(self.out_bytes, dtype=torch.uint8, device=device or "cuda")

    def decode(self, out, stream=None):
        """Launches both stages on `stream`; `out` is a CUDA uint8 tensor of at least out_bytes elements."""
        assert out.is_cuda and out.numel() >= self.out_bytes
        native.check(lib.b200jpg_batch_decode(self.handle, out.data_ptr(), self._stream_ptr(stream)), self.ctx.handle)
        return out

    def geometry(self):
        """Per frame (component shapes [(h, w)], deep), or None for a frame that failed to parse: what decode_into expects."""
        if getattr(self, "_geometry", None) is None:
            geo = []
            for i in range(self.n):
                s = native.FrameInfoStruct()
                rc = lib.b200jpg_batch_frame_info(self.handle, i, ctypes.byref(s))
                fi = FrameInfo.from_struct(s)
                geo.append(None if rc != 0 else ([self.output_shape(i, c) for c in range(self._components(i, fi))], fi.precision > 8))
            self._geometry = geo
        return self._geometry

    def decode_into(self, dst, stream=None, scale=None, bias=None, table=None):
        """decode() into caller-described tensors: dst[i] holds one 2-D CUDA tensor per component of frame i ([H, W], or
        each component's own size with upsample=False), so a [N, C, H, W] batch tensor can be passed as it is, an NHWC
        tensor t as t.permute(0, 3, 1, 2), BGR as [t[i, ..., 2], t[i, ..., 1], t[i, ..., 0]]. uint8 for 8-bit frames,
        int16 for 12-bit frames; None for frames that failed to parse. Only the samples are written. Returns dst.

        float32, float16 or bfloat16 destinations (one dtype per call, any frame) receive every integer sample v (0..255,
        or 0..4095 for 12-bit frames) converted in the reconstruction kernels' store, with no extra pass:
            y = float32(float32(v * scale[c]) + bias[c]), then rounded to nearest even into float16 / bfloat16
        which is what t.float() * scale + bias followed by .half() / .bfloat16() gives. c is the output component (R, G, B
        after the colour transformation). scale and bias are a scalar or one value per component (defaults 1 and 0),
        rounded to float32. scale = 1 / (255 * std), bias = -mean / std is close to ImageNet-style normalisation but not equal
        to it: torchvision's ToTensor() + Normalize(mean, std) computes v / 255, then - mean, then / std, three roundings, and differs
        from the map in the last bit for many (v, c).

        table (b200jpg_batch_decode_into_table, DESIGN §22), a [C, 256] float32 tensor or array with C <= 4, replaces the map: every
        8-bit sample v of output component c is written as table[c][v], stored as float32 or rounded to nearest even into float16 /
        bfloat16 as above. sample_table(fn) builds it from any per-sample transform, so ToTensor() + Normalize() is matched bit
        for bit. A table with fewer rows than the batch's output components, or with scale or bias, raises ValueError, with an integer destination TypeError; a batch with a live 12-bit
        frame raises NativeError (B200JPG_ERR_NOT_IMPLEMENTED)."""
        if table is not None and (scale is not None or bias is not None):
            raise ValueError("a sample table replaces scale and bias: pass one or the other")
        geo = self.geometry()
        planes = plane_table(geo, dst)
        ncomp = max([len(g[0]) for g in geo if g is not None] or [1])
        if table is not None:
            conv = table_args(destination_dtype(dst), table, ncomp)
            native.check(lib.b200jpg_batch_decode_into_table(self.handle, planes, ctypes.byref(conv), self._stream_ptr(stream)), self.ctx.handle)
            return dst
        conv = convert_args(destination_dtype(dst), scale, bias, ncomp)
        if conv is None:
            native.check(lib.b200jpg_batch_decode_into(self.handle, planes, self._stream_ptr(stream)), self.ctx.handle)
        else:
            native.check(lib.b200jpg_batch_decode_into_ex(self.handle, planes, ctypes.byref(conv), self._stream_ptr(stream)), self.ctx.handle)
        return dst

    def decode_entropy(self, stream=None):
        native.check(lib.b200jpg_batch_decode_entropy(self.handle, self._stream_ptr(stream)), self.ctx.handle)

    def reconstruct(self, out, stream=None):
        native.check(lib.b200jpg_batch_reconstruct(self.handle, out.data_ptr(), self._stream_ptr(stream)), self.ctx.handle)
        return out

    def status(self, i):
        return lib.b200jpg_batch_frame_status(self.handle, i)

    def coefficients(self, i, c):
        fi = self.info(i)
        n = fi.blocks_w[c] * fi.blocks_h[c] * 64
        buf = np.empty(n, dtype=np.int16)
        native.check(lib.b200jpg_batch_read_coefficients(self.handle, i, c, buf.ctypes.data, n), self.ctx.handle)
        return buf.reshape(fi.blocks_h[c], fi.blocks_w[c], 8, 8)

    @property
    def launches(self):
        return lib.b200jpg_batch_last_launch_count(self.handle)

    def enable_timing(self, on=True):
        lib.b200jpg_batch_enable_timing(self.handle, int(on))

    def last_timing(self):
        a, b = ctypes.c_float(), ctypes.c_float()
        native.check(lib.b200jpg_batch_last_timing(self.handle, ctypes.byref(a), ctypes.byref(b)), self.ctx.handle)
        return a.value, b.value

    def last_unstuff_ms(self):
        return lib.b200jpg_batch_last_unstuff_ms(self.handle)

    def frame_view(self, out, i):
        """Frame i of a decoded output tensor as [H, W, C] (H x W reduced by `downscale`, swapped by an applied Exif orientation
        5..8, the rectangle's size for a cropped frame, the target size for a resized one)."""
        fi = self.info(i)
        off = self.out_offset(i)
        h, w = self._shape(i, 0, fi)
        nc = self._components(i, fi)
        n = w * h * nc
        if fi.precision > 8:  # 12-bit frames: native-endian 16-bit samples
            import torch
            return out[off:off + 2 * n].view(torch.int16).view(h, w, nc)
        return out[off:off + n].view(h, w, nc)

    def plane_views(self, out, i):
        """upsample=False: the components of frame i as planes [ceil(H/suby), ceil(W/subx)] at their own resolution (H x W
        reduced by `downscale`)."""
        import torch
        assert not self.upsample
        fi = self.info(i)
        off, deep, planes = self.out_offset(i), fi.precision > 8, []
        for c in range(fi.ncomp):
            h, w = self._shape(i, c, fi)
            n = h * w * (2 if deep else 1)
            p = out[off:off + n]
            planes.append(p.view(torch.int16).view(h, w) if deep else p.view(h, w))
            off += n
        return planes

    def close(self):
        if getattr(self, "handle", None):
            lib.b200jpg_batch_destroy(self.handle)
            self.handle = ctypes.c_void_p()
            self.ctx._batch_closed()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
