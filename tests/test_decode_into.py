"""GPU: BatchDecoder.decode_into / b200jpg_batch_decode_into. Every destination layout must receive exactly the samples decode()
writes into the packed slots of the same batch, rearranged, and nothing else: every byte the descriptors do not name keeps
its sentinel."""
import glob
import os

import numpy as np
import pytest

from tests import recon420_cases as rc
from tests import recon_cases

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SENT = 0xA5


def _read(path):
    return open(path, "rb").read()


def _set(sub, skip_suffix=None):
    d = os.path.join(GOLDEN, sub) if sub else GOLDEN
    return [_read(p) for p in sorted(glob.glob(os.path.join(d, "*.jpg"))) if not (skip_suffix and p.endswith(skip_suffix + ".jpg"))]


# every golden vector, set by set: sequential, 4:2:2 / 4:4:0 / 4:4:4 / grey, progressive, 3x / 4x factors, 12-bit, damaged
# (plus one stream that does not parse), DNL, JPEG XT
SETS = {
    "baseline": lambda: _set(""),
    "progressive": lambda: _set("progressive"),
    "subsampling": lambda: _set("subsampling"),
    "deep12": lambda: _set("deep12"),
    "damaged": lambda: _set("damaged") + [b"\xff\xd8\xff\xd9"],
    "dnl": lambda: _set("dnl"),
    "xt": lambda: _set("xt", "__nimpl"),
}


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _batch(built, ctx, frames, **kw):
    dec = built.BatchDecoder(frames, ctx=ctx, tolerate_bad=True, **kw)
    dec.upload()
    return dec


def _reference(dec):
    """decode() of the batch, per frame a list of per-component arrays (uint8, or uint16 for 12-bit frames); None = no frame."""
    import torch
    out = dec.new_output()
    out.fill_(0x5A)
    dec.decode(out)
    torch.cuda.synchronize()
    refs = []
    for i, geo in enumerate(dec.geometry()):
        if geo is None:
            refs.append(None)
            continue
        if dec.upsample:
            v = dec.frame_view(out, i).cpu().numpy()
            comps = [np.ascontiguousarray(v[..., c]) for c in range(v.shape[2])]
        else:
            comps = [p.cpu().numpy() for p in dec.plane_views(out, i)]
        refs.append([c.view(np.uint16) if c.dtype == np.int16 else c for c in comps])
    return refs, dec.launches


def _alloc(shape, deep):
    """a sentinel-filled byte buffer and its typed view of `shape`"""
    import torch
    n = int(np.prod(shape)) * (2 if deep else 1)
    buf = torch.full((n,), SENT, dtype=torch.uint8, device="cuda")
    return buf, (buf.view(torch.int16) if deep else buf).view(*shape)


def _dims(geo):
    shapes, deep = geo
    return len(shapes), max(h for h, _ in shapes), max(w for _, w in shapes), deep


# ---- layouts: geometry -> (byte buffers, dst) with dst a list of tensor lists, or a raw b200jpg_plane table -------------------
def layout_nchw(geometry):
    bufs, dst = [], []
    live = [g for g in geometry if g is not None]
    if len(live) == len(geometry) and all(g == live[0] for g in live) and len(set(live[0][0])) == 1:
        c, h, w, deep = _dims(live[0])
        buf, t = _alloc((len(geometry), c, h, w), deep)
        return [buf], t  # the [N, C, H, W] tensor as it is
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        comps = []
        for (h, w) in g[0]:
            buf, t = _alloc((h, w), g[1])
            bufs.append(buf)
            comps.append(t)
        dst.append(comps)
    return bufs, dst


def layout_padded(geometry):
    live = [_dims(g) for g in geometry if g is not None]
    c, h, w = max(d[0] for d in live), max(d[1] for d in live), max(d[2] for d in live)
    deep = {d[3] for d in live}
    assert len(deep) == 1
    buf, big = _alloc((len(geometry), c, h + 3, w + 5), deep.pop())
    return [buf], [None if g is None else [big[i, k, :hh, :ww] for k, (hh, ww) in enumerate(g[0])] for i, g in enumerate(geometry)]


def _interleaved(geometry, extra, reverse):
    bufs, dst = [], []
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        c, h, w, deep = _dims(g)
        buf, t = _alloc((h, w, c + extra), deep)
        bufs.append(buf)
        dst.append([t[:hh, :ww, (c - 1 - k) if reverse else k] for k, (hh, ww) in enumerate(g[0])])
    return bufs, dst


def layout_bgr(geometry):
    return _interleaved(geometry, 0, True)


def layout_rgbx(geometry):
    return _interleaved(geometry, 1, False)


def layout_bottom_up(geometry):
    from libjpeg_b200 import native
    bufs = []
    table = (native.PlaneStruct * (4 * len(geometry)))()
    for i, g in enumerate(geometry):
        if g is None:
            continue
        c, h, w, deep = _dims(g)
        size = 2 if deep else 1
        buf, _ = _alloc((h, w, c), deep)
        bufs.append(buf)
        for k, (hh, ww) in enumerate(g[0]):
            e = table[4 * i + k]
            e.data = buf.data_ptr() + ((hh - 1) * w * c + k) * size
            e.bytes_per_pixel = c * size
            e.bytes_per_row = -w * c * size
    return bufs, table


def layout_odd(geometry):
    """one allocation per frame, every plane at an odd element offset with an odd element pitch: no row is 8-byte aligned"""
    import torch
    bufs, dst = [], []
    for g in geometry:
        if g is None:
            dst.append(None)
            continue
        shapes, deep = g
        pitches = [w + 1 if (w + 1) % 2 else w + 2 for _, w in shapes]
        n = 1 + sum(h * p for (h, _), p in zip(shapes, pitches)) + 1
        buf, flat = _alloc((n,), deep)
        bufs.append(buf)
        comps, off = [], 1
        for (h, w), p in zip(shapes, pitches):
            comps.append(torch.as_strided(flat, (h, w), (p, 1), off))
            off += h * p
        dst.append(comps)
    return bufs, dst


LAYOUTS = {"nchw": layout_nchw, "padded": layout_padded, "bgr": layout_bgr, "rgbx": layout_rgbx, "bottom_up": layout_bottom_up,
           "odd": layout_odd}


def _table_of(dec, dst):
    from libjpeg_b200.decoder import plane_table
    return dst if not isinstance(dst, (list, tuple)) and not hasattr(dst, "data_ptr") else plane_table(dec.geometry(), dst)


def _launch(dec, dst, stream=None):
    from libjpeg_b200 import native
    if hasattr(dst, "data_ptr") or isinstance(dst, list):
        assert dec.decode_into(dst, stream) is dst
    else:
        native.check(native.lib.b200jpg_batch_decode_into(dec.handle, dst, dec._stream_ptr(stream)), dec.ctx.handle)


def _expected(buf, table, refs):
    """the sentinel buffer with every described sample of every frame at its place"""
    want = np.full(buf.numel(), SENT, dtype=np.uint8)
    base = buf.data_ptr()
    for i, comps in enumerate(refs):
        for c, ref in enumerate(comps or []):
            e = table[4 * i + c]
            off = (e.data or 0) - base
            if not 0 <= off < buf.numel():
                continue
            h, w = ref.shape
            ys, xs = np.mgrid[0:h, 0:w]
            at = off + xs.astype(np.int64) * e.bytes_per_pixel + ys.astype(np.int64) * e.bytes_per_row
            if ref.dtype == np.uint16:
                want[at] = (ref & 0xFF).astype(np.uint8)
                want[at + 1] = (ref >> 8).astype(np.uint8)
            else:
                want[at] = ref
    return want


def _check(bufs, table, refs, what):
    import torch
    torch.cuda.synchronize()
    for k, buf in enumerate(bufs):
        got, want = buf.cpu().numpy(), _expected(buf, table, refs)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, "%s: buffer %d, %d bytes differ, first at %d (got %d, want %d)" % (
            what, k, len(bad), bad[0], got[bad[0]], want[bad[0]])


def _roundtrip(dec, refs, layout, what):
    bufs, dst = LAYOUTS[layout](dec.geometry())
    _launch(dec, dst)
    _check(bufs, _table_of(dec, dst), refs, what)


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("vectors", sorted(SETS))
def test_golden_vectors_into_every_layout(built, ctx, vectors, layout):
    frames = SETS[vectors]()
    dec = _batch(built, ctx, frames)
    refs, launches = _reference(dec)
    if vectors == "damaged":
        assert refs[-1] is None and all(r is not None for r in refs[:-1])
    if layout == "padded" and len({g[1] for g in dec.geometry() if g is not None}) > 1:
        pytest.skip("one padded tensor holds one sample type")
    _roundtrip(dec, refs, layout, "%s/%s" % (vectors, layout))
    assert dec.launches == launches


def test_every_golden_vector_alone_planar_and_strided(built, ctx):
    """one frame per batch: every group of the launch is uniform, so each store kind runs on its own"""
    for vectors in sorted(SETS):
        for data in SETS[vectors]():
            dec = _batch(built, ctx, [data])
            if dec.geometry()[0] is None:
                continue
            refs, _ = _reference(dec)
            for layout in ("nchw", "odd", "bottom_up"):
                _roundtrip(dec, refs, layout, "%s alone/%s" % (vectors, layout))


@pytest.mark.parametrize("layout", ["nchw", "odd", "rgbx", "bottom_up"])
def test_recon420_cases_through_the_new_stores(built, ctx, layout):
    """the seam / skip / narrow / wide frames: the int32 instance of reconstruct420_kernel and 64-bit colour store through
    the planar and the strided kind too"""
    names = rc.NAMES
    assert any(rc.meta(n).narrow for n in names)
    dec = _batch(built, ctx, [rc.case(n)[1] for n in names])
    refs, launches = _reference(dec)
    _roundtrip(dec, refs, layout, "recon420/%s" % layout)
    assert dec.launches == launches


def _recon_case_batches():
    """the cases of tests/recon_cases.py in two batches: 8-bit frames (Tiled, Fused420, Generic) and 12-bit frames"""
    names = recon_cases.NAMES
    return [[recon_cases.case(n)[1] for n in names if recon_cases.case(n)[0].precision == p] for p in (8, 12)]


@pytest.mark.parametrize("layout", ["nchw", "odd", "bottom_up"])
def test_recon_cases_through_the_new_stores(built, ctx, layout):
    """tile seams, the `narrow` exact pass, 64-bit colour, the generic layouts and wrapping IDCTs of tests/recon_cases.py
    through the planar and the strided kinds"""
    for k, frames in enumerate(_recon_case_batches()):
        dec = _batch(built, ctx, frames)
        refs, launches = _reference(dec)
        _roundtrip(dec, refs, layout, "recon/%d/%s" % (k, layout))
        assert dec.launches == launches


@pytest.mark.parametrize("kw", [{"upsample": False}, {"color_transform": False}])
@pytest.mark.parametrize("layout", ["nchw", "padded", "bgr", "odd"])
def test_planes_and_untransformed_components(built, ctx, kw, layout):
    frames = _set("") + _set("subsampling")
    dec = _batch(built, ctx, frames, **kw)
    refs, launches = _reference(dec)
    _roundtrip(dec, refs, layout, "%s/%s" % (kw, layout))
    assert dec.launches == launches
    if not kw.get("upsample", True):
        dec12 = _batch(built, ctx, _set("deep12"), **kw)
        refs12, _ = _reference(dec12)
        _roundtrip(dec12, refs12, layout, "deep12 %s/%s" % (kw, layout))


def test_mixed_batch_with_a_layout_per_frame(built, ctx):
    """4:2:0, 4:4:4, grey and 12-bit frames, each 4:2:0 frame in another layout: the 4:2:0 group falls back to the strided kind"""
    import torch
    names = ["c420_96x80_z6_q75", "c444_64x64_z16_q90", "c420_130x70_z9_q98", "g_40x24_z2_q75", "c420_127x255_z7_q30"]
    frames = [_read(os.path.join(GOLDEN, n + ".jpg")) for n in names]
    frames.append(_read(sorted(glob.glob(os.path.join(GOLDEN, "deep12", "*.jpg")))[0]))
    dec = _batch(built, ctx, frames)
    refs, launches = _reference(dec)
    geo = dec.geometry()
    pieces = [layout_nchw([geo[0]]), layout_bgr([geo[1]]), layout_rgbx([geo[2]]), layout_odd([geo[3]]), layout_padded([geo[4]]),
              layout_odd([geo[5]])]
    bufs, dst = [], []
    for b, d in pieces:
        bufs += b
        dst.append(d[0] if isinstance(d, list) else d[0].unbind(0))
    assert dec.decode_into(dst) is dst
    _check(bufs, _table_of(dec, dst), refs, "mixed")
    assert dec.launches == launches
    torch.cuda.synchronize()


def test_back_to_back_calls_write_where_their_own_descriptors_say(built, ctx):
    """two calls on one batch, different destinations, no synchronisation between them: the second call's descriptor table
    must not overwrite the first one's before the first call's kernels have read it"""
    import torch
    frames = _set("")
    dec = _batch(built, ctx, frames)
    refs, _ = _reference(dec)
    stream = torch.cuda.Stream()
    a_bufs, a = layout_nchw(dec.geometry())
    b_bufs, b = layout_bgr(dec.geometry())
    torch.cuda.synchronize()
    dec.decode_into(a, stream)
    dec.decode_into(b, stream)
    stream.synchronize()
    _check(a_bufs, _table_of(dec, a), refs, "first call")
    _check(b_bufs, _table_of(dec, b), refs, "second call")


def test_launch_count_equals_decode(built, ctx):
    dec = _batch(built, ctx, _set("") + _set("progressive") + _set("deep12"))
    _, launches = _reference(dec)
    for layout in ("nchw", "bgr"):
        _, dst = LAYOUTS[layout](dec.geometry())
        _launch(dec, dst)
        assert dec.launches == launches


def _raw(dec, table):
    from libjpeg_b200 import native
    return native.lib.b200jpg_batch_decode_into(dec.handle, table, dec._stream_ptr(None))


@pytest.mark.parametrize("rule", ["host_pointer", "null_live_frame", "pixel_stride", "row_stride", "row_stride_negative",
                                  "misaligned_16bit_data", "misaligned_16bit_stride"])
def test_invalid_descriptors_are_refused_before_any_launch(built, ctx, rule):
    import torch
    frames = [_read(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg")), _read(sorted(glob.glob(os.path.join(GOLDEN, "deep12", "*.jpg")))[0])]
    dec = _batch(built, ctx, frames)
    dec.decode(dec.new_output())
    torch.cuda.synchronize()
    bufs, dst = layout_nchw(dec.geometry())
    from libjpeg_b200.decoder import plane_table
    table = plane_table(dec.geometry(), dst)
    host = torch.zeros(16, dtype=torch.uint8)
    frame, comp = (1, 0) if "16bit" in rule else (0, 1)
    e = table[4 * frame + comp]
    if rule == "host_pointer":
        e.data = host.data_ptr()
    elif rule == "null_live_frame":
        e.data = None
    elif rule == "pixel_stride":
        e.bytes_per_pixel = 0
    elif rule == "row_stride":
        e.bytes_per_row = 95  # width 96
    elif rule == "row_stride_negative":
        e.bytes_per_row = -95
    elif rule == "misaligned_16bit_data":
        e.data += 1
    else:
        e.bytes_per_row += 1
    launches = dec.launches
    assert _raw(dec, table) == -1024
    torch.cuda.synchronize()
    for buf in bufs:
        assert bool((buf == SENT).all()), rule
    assert dec.launches == launches  # nothing was launched: the count still belongs to the last decode
    from libjpeg_b200 import native
    code, msg = native.last_error(ctx.handle)
    assert code == -1024 and msg, rule
