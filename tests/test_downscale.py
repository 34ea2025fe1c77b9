"""GPU: BatchDecoder(downscale=k) / B200JPG_FLAG_DOWNSCALE_k, bit for bit against the specification of tests/downscale_model.py
(scaled IDCT of the batch's own coefficients, then the reference's reconstruction rules on the W' x H' frame)."""
import glob
import os

import numpy as np
import pytest

from tests import downscale_model as dm
from tests import recon420_cases as rc
from tests import recon_cases
from tests import spec_cases as sc
from tests.test_decode_into import GOLDEN, SETS, _read, _set

pytestmark = pytest.mark.gpu

SENT = 0xA5
NOT_IMPLEMENTED = -1034
DOWN_SETS = {name: fn for name, fn in SETS.items() if name != "xt"}
DOWN_SETS["noeoi"] = lambda: _set("noeoi")
DOWN_SETS["reference"] = lambda: [_read(p) for p in sorted(glob.glob(os.path.join(GOLDEN, "reference", "sub_*.jpg")))]
DOWN_SETS["restartless"] = lambda: [sc.case(n)[1] for n in sc.NAMES]
DOWN_SETS["recon"] = lambda: [recon_cases.case(n)[1] for n in recon_cases.NAMES]


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


def _expected(dec, i, k, color=True, upsample=True):
    fi = dec.info(i)
    coefs = [dec.coefficients(i, c).astype(np.int64) for c in range(fi.ncomp)]
    return dm.expected(coefs, fi.subx, fi.suby, fi.width, fi.height, fi.precision, fi.ycbcr and color, k, upsample)


def _as_samples(t, deep):
    a = t.cpu().numpy()
    return a.view(np.uint16) if deep else a


def _check_batch(built, ctx, frames, k, color=True, upsample=True):
    full = _batch(built, ctx, frames, color_transform=color, upsample=upsample)
    _decode(full)
    dec = _batch(built, ctx, frames, color_transform=color, upsample=upsample, downscale=k)
    out = _decode(dec)
    live = 0
    for i in range(len(frames)):
        assert dec.status(i) == full.status(i), "frame %d" % i
        if dec.geometry()[i] is None:
            continue
        fi = dec.info(i)
        want = _expected(dec, i, k, color, upsample)
        if upsample:
            got = _as_samples(dec.frame_view(out, i), fi.precision > 8)
            assert got.shape == (-(-fi.height // k), -(-fi.width // k), fi.ncomp)
            assert np.array_equal(got, want), "frame %d (%dx%d, k = %d)" % (i, fi.width, fi.height, k)
        else:
            for c, p in enumerate(dec.plane_views(out, i)):
                assert np.array_equal(_as_samples(p, fi.precision > 8), want[c]), "frame %d component %d" % (i, c)
        live += 1
    assert live > 0


@pytest.mark.parametrize("k", [2, 4, 8])
@pytest.mark.parametrize("name", list(DOWN_SETS))
def test_golden_sets(built, ctx, name, k):
    _check_batch(built, ctx, DOWN_SETS[name](), k)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_recon420_cases(built, ctx, k):
    _check_batch(built, ctx, [rc.case(n)[1] for n in rc.NAMES], k)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_size_sweep(built, ctx, k):
    """widths and heights around the reduced frame's 8-sample blocks and the generic kernel's 64-block rows, 1x1 .. 17x9"""
    from libjpeg_b200 import synth
    sizes = [(1, 1), (8, 8), (17, 9), (9, 17), (2 * k - 1, 2 * k + 1), (8 * k - 1, 8 * k + 1), (8 * k, 8 * k), (8 * k + 1, 3),
             (64 * 8 * k + 8, 2 * k + 3), (16 * k + 5, 16 * k - 3)]
    frames = []
    for j, (w, h) in enumerate(sizes):
        for sub in ((2, 2), (1, 1)):
            frames.append(synth.encode(synth.source_image(w, h, j + 1), 80, sub, 0).tobytes())
    _check_batch(built, ctx, frames, k)


@pytest.mark.parametrize("k", [2, 4, 8])
@pytest.mark.parametrize("mode", ["no_color", "no_upsample"])
def test_flags(built, ctx, k, mode):
    frames = DOWN_SETS["baseline"]() + DOWN_SETS["subsampling"]() + DOWN_SETS["deep12"]()
    if mode == "no_color":
        _check_batch(built, ctx, frames, k, color=False)
    else:
        _check_batch(built, ctx, frames, k, upsample=False)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_store_kinds(built, ctx, k):
    """decode_into: uint8 into a planar [N, C, H', W'] view and an NHWC view, float32 / float16 / bfloat16 in both; only the
    samples are written, and every float is the PyTorch conversion of the uint8 result"""
    import torch
    from libjpeg_b200 import synth
    frames = [synth.encode(synth.source_image(97, 61, s), 75, (2, 2), 0).tobytes() for s in (1, 2, 3)]
    dec = _batch(built, ctx, frames, downscale=k)
    out = _decode(dec)
    ref = torch.stack([dec.frame_view(out, i) for i in range(len(frames))]).permute(0, 3, 1, 2).contiguous()  # [N, 3, H', W']
    n, _, h, w = ref.shape
    assert (h, w) == (-(-61 // k), -(-97 // k))
    scale, bias = [1 / 58.4, 1 / 57.1, 1 / 57.4], [-2.1, -2.0, -1.8]
    for dtype in (torch.uint8, torch.float32, torch.float16, torch.bfloat16):
        for layout in ("nchw", "nhwc"):
            esz = torch.empty(0, dtype=dtype).element_size()
            if layout == "nchw":
                buf = torch.full(((n * 3 * (h + 2) * (w + 3)) * esz,), SENT, dtype=torch.uint8, device="cuda")
                full_t = buf.view(dtype).view(n, 3, h + 2, w + 3)
                dst = full_t[:, :, 1:h + 1, 2:w + 2]
            else:
                buf = torch.full(((n * (h + 1) * (w + 2) * 4) * esz,), SENT, dtype=torch.uint8, device="cuda")
                full_t = buf.view(dtype).view(n, h + 1, w + 2, 4)
                dst = full_t[:, :h, 1:w + 1, :3].permute(0, 3, 1, 2)
            if dtype == torch.uint8:
                dec.decode_into(dst)
                want = ref
            else:
                dec.decode_into(dst, scale=scale, bias=bias)
                want = (ref.float() * torch.tensor(scale, device="cuda").view(1, 3, 1, 1) + torch.tensor(bias, device="cuda").view(1, 3, 1, 1)).to(dtype)
            torch.cuda.synchronize()
            assert torch.equal(dst.contiguous().view(torch.uint8 if esz == 1 else torch.int16 if esz == 2 else torch.int32),
                               want.contiguous().view(torch.uint8 if esz == 1 else torch.int16 if esz == 2 else torch.int32)), (dtype, layout)
            mask = torch.ones_like(full_t, dtype=torch.bool)
            if layout == "nchw":
                mask[:, :, 1:h + 1, 2:w + 2] = False
            else:
                mask[:, :h, 1:w + 1, :3] = False
            outside = full_t.view(torch.uint8) if esz == 1 else full_t.view(torch.int16 if esz == 2 else torch.int32)
            sent = int(np.frombuffer(bytes([SENT] * esz), dtype={1: np.uint8, 2: np.int16, 4: np.int32}[esz])[0])
            assert bool((outside[mask] == sent).all()), (dtype, layout)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_mixed_tolerant_batch(built, ctx, k):
    xt = sorted(glob.glob(os.path.join(GOLDEN, "xt", "xt_420_96x80*.jpg")))[0]
    frames = [_read(os.path.join(GOLDEN, "c420_96x80_z6_q75.jpg")), b"\xff\xd8\xff\xd9", _read(os.path.join(GOLDEN, "c444_64x64_z16_q90.jpg")),
              _read(xt), _read(os.path.join(GOLDEN, "deep12", "d12_420_96x80_z3_q80.jpg")), _read(os.path.join(GOLDEN, "c420_127x255_z7_q30.jpg"))]
    full = _batch(built, ctx, frames)
    _decode(full)
    dec = _batch(built, ctx, frames, downscale=k)
    out = _decode(dec)
    for i in range(len(frames)):
        want = NOT_IMPLEMENTED if i == 3 else full.status(i)
        assert dec.status(i) == want, "frame %d" % i
    assert dec.geometry()[1] is None and dec.geometry()[3] is None
    for i in (0, 2, 4, 5):
        fi = dec.info(i)
        assert np.array_equal(_as_samples(dec.frame_view(out, i), fi.precision > 8), _expected(dec, i, k)), "frame %d" % i


def test_downscale_1_is_the_plain_batch(built, ctx):
    frames = DOWN_SETS["baseline"]() + DOWN_SETS["deep12"]() + DOWN_SETS["subsampling"]()
    a = _batch(built, ctx, frames)
    b = _batch(built, ctx, frames, downscale=1)
    oa, ob = _decode(a), _decode(b)
    assert a.out_bytes == b.out_bytes
    assert a.launches == b.launches
    import torch
    assert torch.equal(oa, ob)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_fused_tile_sweep(built, ctx, k):
    """4:2:0 frames whose reduced size lies on either side of reconstruct420_scaled_kernel's tile (256 x 32 reduced samples) and
    of its chroma window's block rows and columns"""
    from libjpeg_b200 import synth
    sizes = [(k * 256, k * 32), (k * 256 - 1, k * 32 - 1), (k * 257, k * 33), (k * 255 + 1, k * 31 + 1), (k * 512 + 3, k * 8 + 5),
             (5, k * 64 + 9), (k * 129, 7)]
    frames = [synth.encode(synth.source_image(w, h, j + 11), 85, (2, 2), 0).tobytes() for j, (w, h) in enumerate(sizes)]
    _check_batch(built, ctx, frames, k)


@pytest.mark.parametrize("device", [False, True])
def test_decode_to_host_and_device_ex(built, ctx, device):
    """the one-call C entry points take the flag: the same bytes as BatchDecoder(downscale=4)"""
    import ctypes
    import torch
    from libjpeg_b200 import native
    frames = [_read(os.path.join(GOLDEN, n)) for n in ("c420_96x80_z6_q75.jpg", "c444_64x64_z16_q90.jpg", "c420_33x17_q50.jpg")]
    frames.append(_read(os.path.join(GOLDEN, "deep12", "d12_422_127x99_z5_q75.jpg")))
    dec = _batch(built, ctx, frames, downscale=4)
    want = _decode(dec)[:dec.out_bytes].cpu().numpy()
    n = len(frames)
    bufs = [(ctypes.c_uint8 * len(f)).from_buffer_copy(f) for f in frames]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(f) for f in frames])
    flags = native.DOWNSCALE_FLAGS[4]
    if not device:
        got = np.zeros(dec.out_bytes, dtype=np.uint8)
        native.check(native.lib.b200jpg_decode_to_host_ex(ctx.handle, ptrs, lens, n, got.ctypes.data, got.size, flags), ctx.handle)
    else:
        p, size = ctypes.c_void_p(), ctypes.c_uint64()
        native.check(native.lib.b200jpg_decode_to_device_ex(ctx.handle, ptrs, lens, n, flags, ctypes.byref(p), ctypes.byref(size)), ctx.handle)
        assert size.value == dec.out_bytes
        t = torch.empty(size.value, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        native.lib.b200jpg_device_copy_rect(ctx.handle, t.data_ptr(), size.value, p.value, size.value, size.value, 1)
        torch.cuda.synchronize()
        native.lib.b200jpg_device_free(ctx.handle, p.value)
        got = t.cpu().numpy()
    for i in range(n):
        a, b = dec.out_offset(i), dec.out_offset(i) + dec.frame_bytes(i)
        assert np.array_equal(got[a:b], want[a:b]), "frame %d" % i
