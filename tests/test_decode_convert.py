"""GPU: float32 / float16 / bfloat16 destinations of BatchDecoder.decode_into / b200jpg_batch_decode_into_ex. Every written
element must be, bit for bit, the numpy conversion of the integer sample decode() writes for the same batch; every other byte
keeps its sentinel, and the call issues as many launches as decode()."""
import ctypes
import glob
import os

import numpy as np
import pytest

from tests import recon420_cases as rc
from tests.test_decode_convert_cpu import convert
from tests.test_decode_into import GOLDEN, SETS, _read, _recon_case_batches, _reference, _set

pytestmark = pytest.mark.gpu

SENT = 0xA5
# a different map per component, negative scales and offsets included (ImageNet-like in the first three)
SCALE = [1 / (255 * 0.229), 1 / (255 * 0.224), -1 / (255 * 0.225), 0.37]
BIAS = [-0.485 / 0.229, -0.456 / 0.224, 0.406 / 0.225, -11.0]


def _dtypes():
    import torch
    return {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _batch(built, ctx, frames, **kw):
    dec = built.BatchDecoder(frames, ctx=ctx, tolerate_bad=True, **kw)
    dec.upload()
    return dec


def _ncomp(geometry):
    return max([len(g[0]) for g in geometry if g is not None] or [1])


def _alloc(shape, dtype):
    """a sentinel-filled byte buffer and its `dtype` view of `shape`"""
    import torch
    esz = torch.empty(0, dtype=dtype).element_size()
    buf = torch.full((int(np.prod(shape)) * esz,), SENT, dtype=torch.uint8, device="cuda")
    return buf, buf.view(dtype).view(*shape)


def _uniform(geometry):
    live = [g for g in geometry if g is not None]
    return len(live) == len(geometry) and all(g[0] == live[0][0] for g in live) and len(set(live[0][0])) == 1


def _dims(g):
    return len(g[0]), max(h for h, _ in g[0]), max(w for _, w in g[0])


# ---- layouts: (geometry, dtype) -> (byte buffers, dst) with dst a tensor, a list of tensor lists, or a raw plane table ----------
def layout_nchw(geometry, dtype):
    if _uniform(geometry):
        c, h, w = _dims(geometry[0])
        buf, t = _alloc((len(geometry), c, h, w), dtype)
        return [buf], t
    bufs, dst = [], []
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        comps = []
        for (h, w) in g[0]:
            buf, t = _alloc((h, w), dtype)
            bufs.append(buf)
            comps.append(t)
        dst.append(comps)
    return bufs, dst


def layout_padded(geometry, dtype):
    live = [_dims(g) for g in geometry if g is not None]
    c, h, w = (max(d[k] for d in live) for k in range(3))
    buf, big = _alloc((len(geometry), c, h + 3, w + 5), dtype)
    return [buf], [None if g is None else [big[i, k, :hh, :ww] for k, (hh, ww) in enumerate(g[0])] for i, g in enumerate(geometry)]


def layout_channels_last(geometry, dtype):
    """an NHWC tensor as t.permute(0, 3, 1, 2) when the frames allow one, else one HWC tensor per frame"""
    if _uniform(geometry):
        c, h, w = _dims(geometry[0])
        buf, t = _alloc((len(geometry), h, w, c), dtype)
        return [buf], t.permute(0, 3, 1, 2)
    return _interleaved(geometry, dtype, False)


def _interleaved(geometry, dtype, reverse):
    bufs, dst = [], []
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        c, h, w = _dims(g)
        buf, t = _alloc((h, w, c), dtype)
        bufs.append(buf)
        dst.append([t[:hh, :ww, (c - 1 - k) if reverse else k] for k, (hh, ww) in enumerate(g[0])])
    return bufs, dst


def layout_bgr(geometry, dtype):
    return _interleaved(geometry, dtype, True)


def layout_bottom_up(geometry, dtype):
    from libjpeg_b200 import native
    import torch
    esz = torch.empty(0, dtype=dtype).element_size()
    bufs, table = [], (native.PlaneStruct * (4 * len(geometry)))()
    for i, g in enumerate(geometry):
        if g is None:
            continue
        c, h, w = _dims(g)
        buf, _ = _alloc((h, w, c), dtype)
        bufs.append(buf)
        for k, (hh, ww) in enumerate(g[0]):
            e = table[4 * i + k]
            e.data = buf.data_ptr() + ((hh - 1) * w * c + k) * esz
            e.bytes_per_pixel = c * esz
            e.bytes_per_row = -w * c * esz
    return bufs, table


def layout_unaligned(geometry, dtype):
    """planar, but every plane starts one element past a 16-byte boundary: the per-element path of the planar kind"""
    import torch
    bufs, dst = [], []
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        n = 1 + sum(h * w for h, w in g[0])
        buf, flat = _alloc((n,), dtype)
        bufs.append(buf)
        comps, off = [], 1
        for (h, w) in g[0]:
            comps.append(torch.as_strided(flat, (h, w), (w, 1), off))
            off += h * w
        dst.append(comps)
    return bufs, dst


LAYOUTS = {"nchw": layout_nchw, "padded": layout_padded, "channels_last": layout_channels_last, "bgr": layout_bgr,
           "bottom_up": layout_bottom_up}


def _map(geometry, dtype, scale, bias):
    from libjpeg_b200.decoder import convert_args
    n = _ncomp(geometry)
    pick = (lambda v: v if np.ndim(v) == 0 else list(v)[:n])
    return pick(scale), pick(bias), convert_args(dtype, pick(scale), pick(bias), n)


def _launch(dec, dst, dtype, scale, bias):
    from libjpeg_b200 import native
    s, b, conv = _map(dec.geometry(), dtype, scale, bias)
    if hasattr(dst, "data_ptr") or isinstance(dst, list):
        assert dec.decode_into(dst, scale=s, bias=b) is dst
        from libjpeg_b200.decoder import plane_table
        return plane_table(dec.geometry(), dst), conv
    native.check(native.lib.b200jpg_batch_decode_into_ex(dec.handle, dst, ctypes.byref(conv), dec._stream_ptr(None)), dec.ctx.handle)
    return dst, conv


def _expected(buf, table, refs, conv, dtype):
    want = np.full(buf.numel(), SENT, dtype=np.uint8)
    base = buf.data_ptr()
    for i, comps in enumerate(refs):
        for c, ref in enumerate(comps or []):
            e = table[4 * i + c]
            off = (e.data or 0) - base
            if not 0 <= off < buf.numel():
                continue
            h, w = ref.shape
            el = convert(ref.astype(np.int64), conv.scale[c], conv.bias[c], dtype)
            el = np.ascontiguousarray(el).view(np.uint8).reshape(h, w, -1)
            ys, xs = np.mgrid[0:h, 0:w]
            at = off + xs.astype(np.int64) * e.bytes_per_pixel + ys.astype(np.int64) * e.bytes_per_row
            for k in range(el.shape[2]):
                want[at + k] = el[..., k]
    return want


def _check(bufs, table, refs, conv, dtype, what):
    import torch
    torch.cuda.synchronize()
    for k, buf in enumerate(bufs):
        got, want = buf.cpu().numpy(), _expected(buf, table, refs, conv, dtype)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, "%s: buffer %d, %d bytes differ, first at %d (got %d, want %d)" % (
            what, k, len(bad), bad[0], got[bad[0]], want[bad[0]])


def _roundtrip(dec, refs, launches, layout, dtype, what, scale=SCALE, bias=BIAS):
    bufs, dst = layout(dec.geometry(), dtype)
    table, conv = _launch(dec, dst, dtype, scale, bias)
    _check(bufs, table, refs, conv, dtype, what)
    assert dec.launches == launches, what


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("vectors", sorted(SETS))
def test_golden_vectors_into_every_layout(built, ctx, vectors, dt):
    dtype = _dtypes()[dt]
    dec = _batch(built, ctx, SETS[vectors]())
    refs, launches = _reference(dec)
    if vectors == "damaged":
        assert refs[-1] is None and all(r is not None for r in refs[:-1])
    for name, layout in sorted(LAYOUTS.items()):
        _roundtrip(dec, refs, launches, layout, dtype, "%s/%s/%s" % (vectors, dt, name))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("kw", [{"upsample": False}, {"color_transform": False}])
def test_planes_and_untransformed_components(built, ctx, kw, dt):
    dtype = _dtypes()[dt]
    for frames in (_set("") + _set("subsampling"), _set("deep12")):
        dec = _batch(built, ctx, frames, **kw)
        refs, launches = _reference(dec)
        for name in ("nchw", "channels_last", "bottom_up"):
            _roundtrip(dec, refs, launches, LAYOUTS[name], dtype, "%s/%s/%s" % (kw, dt, name))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_recon420_cases_through_the_float_stores(built, ctx, dt):
    """tile seams, the int32 instance and the 64-bit colour mode of reconstruct420_kernel through both float kinds"""
    names = rc.NAMES
    assert any(rc.meta(n).narrow for n in names)
    dec = _batch(built, ctx, [rc.case(n)[1] for n in names])
    refs, launches = _reference(dec)
    for name in ("nchw", "channels_last", "bottom_up"):
        _roundtrip(dec, refs, launches, LAYOUTS[name], _dtypes()[dt], "recon420/%s/%s" % (dt, name))
    _roundtrip(dec, refs, launches, layout_unaligned, _dtypes()[dt], "recon420/%s/unaligned" % dt)


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_recon_cases_through_the_float_stores(built, ctx, dt):
    """the Tiled, Generic and wrapping-IDCT cases of tests/recon_cases.py (8- and 12-bit batches) through both float kinds"""
    for k, frames in enumerate(_recon_case_batches()):
        dec = _batch(built, ctx, frames)
        refs, launches = _reference(dec)
        for name in ("nchw", "channels_last", "bottom_up"):
            _roundtrip(dec, refs, launches, LAYOUTS[name], _dtypes()[dt], "recon/%d/%s/%s" % (k, dt, name))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_unaligned_rows_take_the_per_element_path(built, ctx, dt):
    dec = _batch(built, ctx, _set("") + _set("subsampling"))
    refs, launches = _reference(dec)
    _roundtrip(dec, refs, launches, layout_unaligned, _dtypes()[dt], "unaligned/%s" % dt)


def test_map_edges(built, ctx):
    """identity, a negative scale, fp16 overflow to inf, fp16 subnormal results, 12-bit samples rounded in bf16"""
    import torch
    d = _dtypes()
    dec = _batch(built, ctx, _set(""))
    refs, launches = _reference(dec)
    for dt in ("f32", "f16", "bf16"):
        bufs, dst = layout_nchw(dec.geometry(), d[dt])
        dec.decode_into(dst)  # identity: the integers themselves
        torch.cuda.synchronize()
        for i, comps in enumerate(refs):
            t = dst[i] if isinstance(dst, list) else dst[i].unbind(0)
            for c, ref in enumerate(comps):
                assert np.array_equal(t[c].float().cpu().numpy(), ref.astype(np.float32)), ("identity", dt, i, c)
    _roundtrip(dec, refs, launches, layout_nchw, d["f32"], "negative", scale=-2.5, bias=7.0)
    _roundtrip(dec, refs, launches, layout_nchw, d["f16"], "overflow", scale=300.0, bias=0.0)
    _roundtrip(dec, refs, launches, layout_nchw, d["f16"], "subnormal", scale=2.0 ** -22, bias=0.0)
    bufs, dst = layout_nchw(dec.geometry(), d["f16"])
    dec.decode_into(dst, scale=300.0)
    torch.cuda.synchronize()
    flat = torch.cat([t.reshape(-1) for e in (dst if isinstance(dst, list) else [dst]) for t in e])
    assert bool(torch.isinf(flat).any())  # the values above 218 really left the fp16 range
    dec12 = _batch(built, ctx, _set("deep12"))
    refs12, launches12 = _reference(dec12)
    assert max(int(c.max()) for comps in refs12 for c in comps) > 256  # 12-bit values bf16 cannot hold exactly
    _roundtrip(dec12, refs12, launches12, layout_nchw, d["bf16"], "deep12 bf16", scale=1.0, bias=0.0)
    _roundtrip(dec12, refs12, launches12, layout_bgr, d["f16"], "deep12 f16", scale=1 / 4095, bias=-0.5)


def test_mixed_batch_and_back_to_back_calls(built, ctx):
    """4:2:0, 4:4:4, grey and 12-bit frames in one call; then two calls with different maps and types without a
    synchronisation between them"""
    import torch
    d = _dtypes()
    names = ["c420_96x80_z6_q75", "c444_64x64_z16_q90", "g_40x24_z2_q75", "c420_127x255_z7_q30"]
    frames = [_read(os.path.join(GOLDEN, n + ".jpg")) for n in names]
    frames.append(_read(sorted(glob.glob(os.path.join(GOLDEN, "deep12", "*.jpg")))[0]))
    dec = _batch(built, ctx, frames)
    refs, launches = _reference(dec)
    _roundtrip(dec, refs, launches, layout_padded, d["f16"], "mixed/padded")
    a_bufs, a = layout_nchw(dec.geometry(), d["bf16"])
    b_bufs, b = layout_bgr(dec.geometry(), d["f32"])
    torch.cuda.synchronize()
    ta, ca = _launch(dec, a, d["bf16"], SCALE, BIAS)
    tb, cb = _launch(dec, b, d["f32"], 0.5, -3.0)
    _check(a_bufs, ta, refs, ca, d["bf16"], "first call")
    _check(b_bufs, tb, refs, cb, d["f32"], "second call")


@pytest.mark.parametrize("rule", ["unknown_type", "nan_scale", "inf_scale", "nan_bias", "inf_bias", "misaligned_data",
                                  "misaligned_stride", "misaligned_pixel_stride", "pixel_stride_below_element"])
@pytest.mark.parametrize("dt", ["f32", "f16"])
def test_invalid_requests_are_refused_before_any_launch(built, ctx, rule, dt):
    import torch
    from libjpeg_b200 import native
    from libjpeg_b200.decoder import plane_table
    dtype = _dtypes()[dt]
    esz = 4 if dt == "f32" else 2
    dec = _batch(built, ctx, [_read(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"))])
    dec.decode(dec.new_output())
    torch.cuda.synchronize()
    bufs, dst = layout_nchw(dec.geometry(), dtype)
    table = plane_table(dec.geometry(), dst)
    _, _, conv = _map(dec.geometry(), dtype, SCALE, BIAS)
    e = table[1]
    if rule == "unknown_type":
        conv.type = 7
    elif rule.endswith("_scale") or rule.endswith("_bias"):
        getattr(conv, rule.split("_")[1])[2] = float("nan") if rule.startswith("nan") else -float("inf")
    elif rule == "misaligned_data":
        e.data += esz // 2
    elif rule == "misaligned_stride":
        e.bytes_per_row += esz // 2
    elif rule == "misaligned_pixel_stride":
        e.bytes_per_pixel += esz // 2
    else:
        e.bytes_per_pixel = esz // 2
    launches = dec.launches
    rc_ = native.lib.b200jpg_batch_decode_into_ex(dec.handle, table, ctypes.byref(conv), dec._stream_ptr(None))
    assert rc_ == -1024, rule
    torch.cuda.synchronize()
    for buf in bufs:
        assert bool((buf == SENT).all()), rule
    assert dec.launches == launches
    code, msg = native.last_error(ctx.handle)
    assert code == -1024 and msg, rule


def test_non_finite_map_of_an_absent_component_is_accepted(built, ctx):
    """only the components some live frame has are checked: scale[3] of a three-component batch is never read"""
    import torch
    from libjpeg_b200 import native
    from libjpeg_b200.decoder import plane_table
    dec = _batch(built, ctx, [_read(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg"))])
    refs, launches = _reference(dec)
    bufs, dst = layout_nchw(dec.geometry(), _dtypes()["f16"])
    _, _, conv = _map(dec.geometry(), _dtypes()["f16"], SCALE, BIAS)
    conv.scale[3], conv.bias[3] = float("nan"), float("inf")
    table = plane_table(dec.geometry(), dst)
    native.check(native.lib.b200jpg_batch_decode_into_ex(dec.handle, table, ctypes.byref(conv), dec._stream_ptr(None)), dec.ctx.handle)
    _check(bufs, table, refs, conv, _dtypes()["f16"], "absent component")
    assert dec.launches == launches
    torch.cuda.synchronize()
