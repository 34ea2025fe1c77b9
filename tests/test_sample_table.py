"""GPU: decode_into(..., table=...) / b200jpg_batch_decode_into_table (DESIGN §22). The oracle is the uint8 decode_into of the
same batch into the same layout, gathered through the table by torch and cast to the element type, bit for bit, over every
reconstruction path and destination kind. The end-to-end test holds the batch to torchvision's training transform on Pillow's
pixels."""
import io
import os

import numpy as np
import pytest

from tests import orientation_model as om
from tests.test_decode_into import GOLDEN, SETS, _read
from tests.test_flip import _flip_args
from tests.test_orientation import _batch, _synth

pytestmark = pytest.mark.gpu

TURBO = "libjpeg-turbo"
CMYK_DIR = os.path.join(GOLDEN, "cmyk")
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


@pytest.fixture(scope="module")
def ctx(built):
    from libjpeg_b200.decoder import Context
    return Context()


def _table(seed):
    """distinct rows per component, with values float16 rounds to inf, to subnormals and to -0"""
    t = np.random.default_rng(seed).standard_normal((4, 256)).astype(np.float32) * 3
    t[:, 7], t[:, 250], t[1, 3], t[2, 200] = 70000.0, -1e-6, -0.0, 3e-41
    return t


def _alloc(dec, dtype, layout, fill):
    """per frame its components as separate [h, w] tensors (planar) or views of one [h, w, C] tensor (nhwc); None for no frame"""
    import torch
    out = []
    for geo in dec.geometry():
        if geo is None:
            out.append(None)
            continue
        shapes = geo[0]
        if layout == "planar" or len(set(shapes)) > 1:
            out.append([torch.full(s, fill, dtype=dtype, device="cuda") for s in shapes])
        else:
            t = torch.full(shapes[0] + (len(shapes),), fill, dtype=dtype, device="cuda")
            out.append([t[..., c] for c in range(len(shapes))])
    return out


def _check(built, ctx, frames, dtypes=None, layouts=("planar", "nhwc"), seed=0, **kw):
    import torch
    dec = _batch(built, ctx, frames, **kw)
    tab = _table(seed)
    ttab = torch.from_numpy(tab)
    live = 0
    for layout in layouts:
        ref = _alloc(dec, torch.uint8, layout, 0)
        dec.decode_into(ref)
        for dtype in dtypes or (torch.float32, torch.float16, torch.bfloat16):
            got = _alloc(dec, dtype, layout, 12345.0)
            ncomp = max(len(g) for g in got if g is not None)
            dec.decode_into(got, table=tab[:ncomp])
            torch.cuda.synchronize()
            for i, (r, g) in enumerate(zip(ref, got)):
                if r is None:
                    continue
                for c, (rc, gc) in enumerate(zip(r, g)):
                    want = ttab[c][rc.long().cpu()].to(dtype)
                    iv = torch.int32 if dtype == torch.float32 else torch.int16
                    assert torch.equal(gc.cpu().contiguous().view(iv), want.view(iv)), (i, c, layout, dtype)
                live += 1
    assert live > 0
    return dec


SYNTH = lambda: [_synth(333, 201, 1, (2, 2)), _synth(200, 120, 2, (1, 1)), _synth(97, 61, 3, (2, 1)), _synth(64, 40, 4, (1, 2))]


@pytest.mark.parametrize("reconstruction", ["reference", TURBO])
def test_paths(built, ctx, reconstruction):
    """Fused420, Tiled, Generic (3x / 4x factors, progressive) and the turbo kernels, grey frames included"""
    frames = SYNTH() + SETS["baseline"]() + SETS["subsampling"]() + SETS["progressive"]()
    _check(built, ctx, frames, reconstruction=reconstruction)


@pytest.mark.parametrize("k", [2, 4, 8])
def test_scaled_and_drafted(built, ctx, k):
    """Scaled / Scaled420 (downscale) and the drafted turbo kernels"""
    frames = SYNTH() + SETS["baseline"]()[:4]
    _check(built, ctx, frames, downscale=k)
    _check(built, ctx, frames, draft=[(8, 8)] * len(frames), reconstruction=TURBO, seed=k)


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("reconstruction", ["reference", TURBO])
def test_modes(built, ctx, mode, reconstruction):
    """Replicate (a grey frame's sample through all three tables), Luma and the CMYK / YCCK conversions"""
    cmyk = [_read(os.path.join(CMYK_DIR, f)) for f in sorted(os.listdir(CMYK_DIR)) if f.endswith(".jpg")][:6]
    _check(built, ctx, SYNTH() + SETS["baseline"]() + cmyk, mode=mode, reconstruction=reconstruction)


def test_kinds(built, ctx):
    """Runs (oriented frames), Clip (cropped frames), Strided and Planar, and upsample=False planes"""
    frames = [om.tag(f, o) for f, o in zip(SYNTH() * 2, [2, 3, 6, 8, 5, 4, 7, 1])]
    _check(built, ctx, frames, exif_orientation=True)
    _check(built, ctx, frames, exif_orientation=True, crop=[(3, 5, 30, 20)] * len(frames), seed=1)
    _check(built, ctx, SYNTH() + SETS["baseline"]()[:3], upsample=False, seed=2)


@pytest.mark.parametrize("resample", ["bilinear", "lanczos", "cv2-linear", "cv2-area"])
def test_resized(built, ctx, resample):
    """resized frames: the resample pass looks the resampled samples up, flipped or not"""
    frames = SYNTH() + SETS["baseline"]()[:4]
    n = len(frames)
    _check(built, ctx, frames, resize=[(31 + i, 45 - i) for i in range(n)], resample=resample, mode="RGB",
           **_flip_args([i % 4 for i in range(n)]))


def test_refused(built, ctx):
    """a live 12-bit frame is NOT_IMPLEMENTED, an unknown type or a NULL table INVALID_PARAMETER, nothing launched"""
    import ctypes

    import torch
    from libjpeg_b200 import NativeError, native
    dec = _batch(built, ctx, SETS["deep12"]()[:2] + SYNTH()[:1])
    dst = _alloc(dec, torch.float32, "planar", 0)
    with pytest.raises(NativeError) as e:
        dec.decode_into(dst, table=np.zeros((3, 256), np.float32))
    assert e.value.code == -1034
    dec = _batch(built, ctx, SYNTH())
    dst = _alloc(dec, torch.float32, "planar", 0)
    from libjpeg_b200.decoder import plane_table
    planes = plane_table(dec.geometry(), dst)
    t = native.ConvertTableStruct()
    for ty in (0, 4, -1):
        t.type = ty
        assert native.lib.b200jpg_batch_decode_into_table(dec.handle, planes, ctypes.byref(t), None) == -1024
    assert native.lib.b200jpg_batch_decode_into_table(dec.handle, planes, None, None) == -1024
    with pytest.raises(TypeError):
        dec.decode_into(_alloc(dec, torch.uint8, "planar", 0), table=np.zeros((3, 256), np.float32))
    with pytest.raises(ValueError):  # one row for a batch of three-component frames
        dec.decode_into(dst, table=np.zeros((1, 256), np.float32))


def test_launches_and_affine_unchanged(built, ctx):
    """a table call issues the launches of the affine call, and the affine call after it is unchanged"""
    import torch
    frames = SYNTH() + SETS["baseline"]()[:3]
    dec = _batch(built, ctx, frames, mode="RGB")
    a = _alloc(dec, torch.float16, "planar", 0)
    dec.decode_into(a, scale=1 / 255.0)
    n_affine = dec.launches
    dec.decode_into(_alloc(dec, torch.float16, "planar", 0), table=_table(3)[:3])
    assert dec.launches == n_affine
    b = _alloc(dec, torch.float16, "planar", 0)
    dec.decode_into(b, scale=1 / 255.0)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        for p, q in zip(x, y):
            assert torch.equal(p, q)


def test_torchvision_training_crop(built, ctx):
    """Normalize(ToTensor(flip(Image.open(f).convert("RGB").crop(box).resize((224, 224), BILINEAR)))) of the golden 8-bit vectors,
    bit for bit, as one fp32 [N, 3, 224, 224] tensor of one decode_into call"""
    import torch
    import torchvision.transforms.functional as TF
    from PIL import Image
    from libjpeg_b200 import sample_table
    frames = []
    for f in SETS["baseline"]():
        with Image.open(io.BytesIO(f)) as im:
            if im.mode in ("L", "RGB"):
                frames.append(f)
    rng = np.random.default_rng(3)
    rects, flips = [], []
    for f in frames:
        with Image.open(io.BytesIO(f)) as im:
            w, h = im.size
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        rects.append((x, y, int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))))
        flips.append(int(rng.integers(0, 4)))
    dec = _batch(built, ctx, frames, crop=rects, resize=(224, 224), resample="bilinear", reconstruction=TURBO, mode="RGB",
                 **_flip_args(flips))
    dst = torch.zeros((len(frames), 3, 224, 224), dtype=torch.float32, device="cuda")
    dec.decode_into(dst, table=sample_table(lambda t: TF.normalize(t.float().div(255), MEAN, STD)))
    torch.cuda.synchronize()
    got = dst.cpu()
    for j, (f, (x, y, w, h), fl) in enumerate(zip(frames, rects, flips)):
        with Image.open(io.BytesIO(f)) as im:
            img = im.convert("RGB").crop((x, y, x + w, y + h)).resize((224, 224), Image.Resampling.BILINEAR)
        if fl & 1:
            img = TF.hflip(img)
        if fl & 2:
            img = TF.vflip(img)
        want = TF.normalize(TF.to_tensor(img), MEAN, STD)
        assert torch.equal(got[j].view(torch.int32), want.view(torch.int32)), "frame %d (flip %d)" % (j, fl)
