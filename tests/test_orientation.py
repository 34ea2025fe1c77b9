"""GPU: BatchDecoder(exif_orientation=True) / B200JPG_FLAG_EXIF_ORIENTATION. The oracle is the same batch decoded without the flag
(itself pinned to the reference by the other suites), oriented by the numpy table of tests/orientation_model.py, bit for bit; every
frame's status is that of the unflagged batch."""
import ctypes
import glob
import os

import numpy as np
import pytest

from tests import orientation_model as om
from tests import recon420_cases as rc
from tests import recon_cases
from tests import spec_cases as sc
from tests.test_decode_into import GOLDEN, SETS, _read

pytestmark = pytest.mark.gpu

SENT = 0xA5
ORIENT_SETS = dict(SETS)
ORIENT_SETS["reference"] = lambda: [_read(p) for p in sorted(glob.glob(os.path.join(GOLDEN, "reference", "sub_*.jpg")))]
ORIENT_SETS["restartless"] = lambda: [sc.case(n)[1] for n in sc.NAMES]
ORIENT_SETS["recon420"] = lambda: [rc.case(n)[1] for n in rc.NAMES]
ORIENT_SETS["recon"] = lambda: [recon_cases.case(n)[1] for n in recon_cases.NAMES]


def _synth(w, h, seed, sub=(2, 2), q=80, restart=0):
    from libjpeg_b200 import synth
    return synth.encode(synth.source_image(w, h, seed), q, sub, restart).tobytes()


ORIENT_SETS["synth"] = lambda: [_synth(1920, 1080, 1), _synth(1000, 333, 2), _synth(333, 1000, 3, (1, 1)), _synth(1000, 333, 4, (2, 1)),
                                _synth(257, 33, 5), _synth(33, 257, 6, (1, 1))]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _batch(built, ctx, frames, **kw):
    dec = built.BatchDecoder(frames, ctx=ctx, tolerate_bad=True, **kw)
    dec.upload()
    return dec


def _decode(dec):
    import torch
    out = dec.new_output()
    out.fill_(0x5A)
    dec.decode(out)
    torch.cuda.synchronize()
    return out


def _images(dec, out):
    """per frame the decoded image as [H, W, C] (upsample) or a list of planes, uint16 for 12-bit frames; None for no frame"""
    res = []
    for i, geo in enumerate(dec.geometry()):
        if geo is None:
            res.append(None)
            continue
        deep = geo[1]
        if dec.upsample:
            a = dec.frame_view(out, i).cpu().numpy()
            res.append(a.view(np.uint16) if deep else a)
        else:
            res.append([p.cpu().numpy().view(np.uint16) if deep else p.cpu().numpy() for p in dec.plane_views(out, i)])
    return res


def _tagged(frames):
    """every frame with each of the eight orientations: (frames, orientations)"""
    tagged, orients = [], []
    for f in frames:
        for o in om.ORIENTATIONS:
            tagged.append(om.tag(f, o))
            orients.append(o)
    return tagged, orients


def _expected(ref, o):
    if ref is None:
        return None
    if isinstance(ref, list):
        return [np.ascontiguousarray(om.orient(p, o)) for p in ref]
    return np.ascontiguousarray(om.orient(ref, o))


def _check_packed(built, ctx, frames, **kw):
    tagged, orients = _tagged(frames)
    plain = _batch(built, ctx, tagged, **kw)
    ref = _images(plain, _decode(plain))
    dec = _batch(built, ctx, tagged, exif_orientation=True, **kw)
    got = _images(dec, _decode(dec))
    live = 0
    for i, o in enumerate(orients):
        assert dec.status(i) == plain.status(i), "frame %d" % i
        want = _expected(ref[i], o)
        if want is None:
            assert got[i] is None
            continue
        assert dec.orientation(i) == o
        if isinstance(want, list):
            for c, (g, w) in enumerate(zip(got[i], want)):
                assert np.array_equal(g, w), "frame %d (orientation %d) component %d" % (i, o, c)
        else:
            assert np.array_equal(got[i], want), "frame %d (orientation %d)" % (i, o)
        live += 1
    assert live > 0


@pytest.mark.parametrize("name", list(ORIENT_SETS))
def test_packed(built, ctx, name):
    _check_packed(built, ctx, ORIENT_SETS[name]())


@pytest.mark.parametrize("k", [2, 4, 8])
def test_downscale(built, ctx, k):
    frames = SETS["baseline"]() + SETS["deep12"]() + SETS["subsampling"]() + [_synth(1000, 333, 7), _synth(333, 1000, 8, (1, 1))]
    _check_packed(built, ctx, frames, downscale=k)


@pytest.mark.parametrize("mode", ["no_color", "no_upsample", "no_upsample_k2"])
def test_flags(built, ctx, mode):
    frames = SETS["baseline"]() + SETS["subsampling"]() + SETS["deep12"]() + SETS["progressive"]()
    if mode == "no_color":
        _check_packed(built, ctx, frames, color_transform=False)
    elif mode == "no_upsample":
        _check_packed(built, ctx, frames, upsample=False)
    else:
        _check_packed(built, ctx, frames, upsample=False, downscale=2)


def _oriented_refs(built, ctx, frames, orients, **kw):
    """the upright decode of every frame, oriented: [N, C, H, W] (torch, on the device)"""
    import torch
    plain = _batch(built, ctx, [om.tag(f, o) for f, o in zip(frames, orients)], **kw)
    ref = _images(plain, _decode(plain))
    return torch.stack([torch.from_numpy(_expected(r, o).copy()) for r, o in zip(ref, orients)]).permute(0, 3, 1, 2).contiguous().cuda()


def _view_as_int(t):
    import torch
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


@pytest.mark.parametrize("group", ["upright", "transposed"])
@pytest.mark.parametrize("size", [(97, 61), (1000, 333), (256, 64)])
def test_destinations(built, ctx, group, size):
    """decode_into: uint8 into [N, C, H, W] (contiguous, and with padded rows at an odd offset), an NHWC view, and float32 /
    float16 / bfloat16 into [N, C, H, W] and NHWC with a per-component map; only the samples are written, every float is the
    PyTorch conversion of the uint8 result. One batch per group of orientations whose oriented shapes agree."""
    import torch
    w, h = size
    orients = [1, 2, 3, 4] if group == "upright" else [5, 6, 7, 8]
    src = [_synth(w, h, 20, (2, 2)), _synth(w, h, 21, (1, 1))]
    frames = src + src  # a 4:2:0 (Fused420) and a 4:4:4 (Tiled) source, each under two orientations
    want_u8 = _oriented_refs(built, ctx, frames, orients)
    dec = _batch(built, ctx, [om.tag(f, o) for f, o in zip(frames, orients)], exif_orientation=True)
    n, _, oh, ow = want_u8.shape
    assert [dec.output_shape(i, 0) for i in range(n)] == [(oh, ow)] * n
    scale, bias = [1 / 58.4, 1 / 57.1, 1 / 57.4], [-2.1, -2.0, -1.8]
    cases = [(torch.uint8, "nchw"), (torch.uint8, "padded"), (torch.uint8, "nhwc")]
    cases += [(dt, lay) for dt in (torch.float32, torch.float16, torch.bfloat16) for lay in ("nchw", "nhwc")]
    for dtype, layout in cases:
        esz = torch.empty(0, dtype=dtype).element_size()
        if layout == "nchw":
            buf = torch.full((n * 3 * oh * ow * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, 3, oh, ow)
            dst, region = full_t, (slice(None),) * 4
        elif layout == "padded":  # rows padded by 3, the plane starting at an odd element offset
            buf = torch.full((n * 3 * (oh + 2) * (ow + 3) * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, 3, oh + 2, ow + 3)
            region = (slice(None), slice(None), slice(1, oh + 1), slice(1, ow + 1))
            dst = full_t[region]
        else:
            buf = torch.full((n * (oh + 1) * (ow + 2) * 4 * esz,), SENT, dtype=torch.uint8, device="cuda")
            full_t = buf.view(dtype).view(n, oh + 1, ow + 2, 4)
            region = (slice(None), slice(0, oh), slice(1, ow + 1), slice(0, 3))
            dst = full_t[region].permute(0, 3, 1, 2)
        if dtype == torch.uint8:
            dec.decode_into(dst)
            want = want_u8
        else:
            dec.decode_into(dst, scale=scale, bias=bias)
            want = (want_u8.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) +
                    torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
        torch.cuda.synchronize()
        assert torch.equal(_view_as_int(dst), _view_as_int(want)), (dtype, layout)
        mask = torch.ones(full_t.shape, dtype=torch.bool, device="cuda")
        mask[region] = False
        sent = int(np.frombuffer(bytes([SENT] * esz), dtype={1: np.uint8, 2: np.int16, 4: np.int32}[esz])[0])
        assert bool((_view_as_int(full_t)[mask] == sent).all()), (dtype, layout)


def test_deep12_into_int16(built, ctx):
    """12-bit frames into int16 [C, H, W] destinations per frame (the generic kernels' strided store)"""
    import torch
    frames, orients = _tagged(SETS["deep12"]())
    plain = _batch(built, ctx, frames)
    ref = _images(plain, _decode(plain))
    dec = _batch(built, ctx, frames, exif_orientation=True)
    dst = []
    for i, geo in enumerate(dec.geometry()):
        shapes, deep = geo
        assert deep
        dst.append(torch.full((len(shapes),) + tuple(shapes[0]), -1, dtype=torch.int16, device="cuda"))
    dec.decode_into([list(t) for t in dst])
    torch.cuda.synchronize()
    for i, o in enumerate(orients):
        want = _expected(ref[i], o)
        assert np.array_equal(dst[i].cpu().numpy().view(np.uint16), np.moveaxis(want, 2, 0)), "frame %d" % i


def test_mixed_batch(built, ctx):
    """all eight orientations, a frame without Exif and one that fails to parse in one tolerant batch: packed decode and per-frame
    [C, H, W] destinations, every byte outside the samples keeps its sentinel"""
    import torch
    srcs = [_read(os.path.join(GOLDEN, n)) for n in ("c420_127x255_z7_q30.jpg", "c444_64x64_z16_q90.jpg", "c422_100x60_z5_q80.jpg",
                                                     "g_40x24_z2_q75.jpg")]
    srcs.append(_read(os.path.join(GOLDEN, "deep12", "d12_420_96x80_z3_q80.jpg")))
    frames, orients = [], []
    for o in om.ORIENTATIONS:
        frames.append(om.tag(srcs[o % len(srcs)], o))
        orients.append(o)
    frames.append(srcs[0])
    orients.append(1)
    frames.append(om.tag(b"\xff\xd8\xff\xd9", 6))
    orients.append(None)
    plain = _batch(built, ctx, frames)
    ref = _images(plain, _decode(plain))
    dec = _batch(built, ctx, frames, exif_orientation=True)
    out = _decode(dec)
    got = _images(dec, out)
    for i, o in enumerate(orients):
        assert dec.status(i) == plain.status(i)
        if o is None:
            assert got[i] is None and dec.orientation(i) == dec.status(i) < 0
            continue
        assert dec.orientation(i) == o
        assert np.array_equal(got[i], _expected(ref[i], o)), "frame %d" % i
    # the packed output outside the frames' slots is untouched
    o_np = out.cpu().numpy()
    mask = np.ones(o_np.size, dtype=bool)
    for i in range(len(frames)):
        if dec.geometry()[i] is not None:
            mask[dec.out_offset(i):dec.out_offset(i) + dec.frame_bytes(i)] = False
    assert (o_np[mask] == 0x5A).all()
    bufs, dst = [], []
    for i, geo in enumerate(dec.geometry()):
        if geo is None:
            dst.append(None)
            continue
        shapes, deep = geo
        h, w = shapes[0]
        b = torch.full(((h + 1) * (w + 2) * len(shapes) * (2 if deep else 1),), SENT, dtype=torch.uint8, device="cuda")
        full_t = (b.view(torch.int16) if deep else b).view(len(shapes), h + 1, w + 2)
        bufs.append((i, full_t))
        dst.append(list(full_t[:, 1:, 1:w + 1]))
    dec.decode_into(dst)
    torch.cuda.synchronize()
    for i, full_t in bufs:
        want = np.moveaxis(_expected(ref[i], orients[i]), 2, 0)
        a = full_t.cpu().numpy()
        a = a.view(np.uint16) if a.dtype == np.int16 else a
        assert np.array_equal(a[:, 1:, 1:-1], want), "frame %d" % i
        m = np.ones(a.shape, dtype=bool)
        m[:, 1:, 1:-1] = False
        sent = 0xA5A5 if a.dtype == np.uint16 else SENT
        assert (a[m] == sent).all(), "frame %d" % i


def test_upright_frames_are_the_plain_batch(built, ctx):
    """with the flag and every frame at orientation 1 (tagged or not), the batch launches and writes what it does without it"""
    import torch
    frames = SETS["baseline"]() + SETS["deep12"]() + SETS["subsampling"]() + SETS["progressive"]()
    frames = [om.tag(f, 1) if j % 2 else f for j, f in enumerate(frames)]
    a = _batch(built, ctx, frames)
    b = _batch(built, ctx, frames, exif_orientation=True)
    oa, ob = _decode(a), _decode(b)
    assert a.out_bytes == b.out_bytes and a.launches == b.launches
    assert torch.equal(oa, ob)


def test_without_the_flag_exif_is_not_applied(built, ctx):
    import torch
    frames = SETS["baseline"]() + SETS["subsampling"]()
    tagged = [om.tag(f, 1 + j % 8) for j, f in enumerate(frames)]
    a = _batch(built, ctx, frames)
    b = _batch(built, ctx, tagged)
    oa, ob = _decode(a), _decode(b)
    assert a.out_bytes == b.out_bytes and a.launches == b.launches
    assert torch.equal(oa, ob)
    assert [b.orientation(i) for i in range(len(tagged))] == [1 + j % 8 for j in range(len(tagged))]


def test_decode_to_host_ex(built, ctx):
    """the one-call C entry point takes the flag: the same bytes as BatchDecoder(exif_orientation=True)"""
    from libjpeg_b200 import native
    frames = [om.tag(_read(os.path.join(GOLDEN, n)), o) for n, o in (("c420_96x80_z6_q75.jpg", 6), ("c444_64x64_z16_q90.jpg", 3),
                                                                      ("c420_33x17_q50.jpg", 7))]
    dec = _batch(built, ctx, frames, exif_orientation=True)
    want = _decode(dec)[:dec.out_bytes].cpu().numpy()
    n = len(frames)
    bufs = [(ctypes.c_uint8 * len(f)).from_buffer_copy(f) for f in frames]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    got = np.zeros(dec.out_bytes, dtype=np.uint8)
    native.check(native.lib.b200jpg_decode_to_host_ex(ctx.handle, ptrs, lens, n, got.ctypes.data, got.size, native.FLAG_EXIF_ORIENTATION),
                 ctx.handle)
    for i in range(n):
        a, b = dec.out_offset(i), dec.out_offset(i) + dec.frame_bytes(i)
        assert np.array_equal(got[a:b], want[a:b]), "frame %d" % i
