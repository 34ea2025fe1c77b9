"""CPU: libjpeg_b200.sample_table and the argument checks of decode_into(..., table=...) (DESIGN §22). The table of torchvision's
ToTensor() + Normalize() (and of v2's ToDtype(scale=True) + Normalize()) holds torchvision's own results on the 256 sample values,
bit for bit, in float32 and after rounding to float16 / bfloat16; the affine map of decode_into_ex does not."""
import types

import numpy as np
import pytest

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _values():
    import torch
    return torch.arange(256, dtype=torch.uint8).view(1, 1, 256).expand(3, 1, 256).contiguous()


def _v1(t):
    import torchvision.transforms.functional as TF
    return TF.normalize(TF.to_tensor(t.permute(1, 2, 0).numpy()), MEAN, STD)


def _v2(t):
    import torch
    from torchvision.transforms import v2
    return v2.Normalize(MEAN, STD)(v2.ToDtype(torch.float32, scale=True)(t))


@pytest.mark.parametrize("name,fn", [("ToTensor+Normalize", _v1), ("v2 ToDtype+Normalize", _v2)])
def test_torchvision_tables(name, fn):
    """the table's entries are torchvision's output for every sample value, in every element type"""
    import torch
    pytest.importorskip("torchvision")
    from libjpeg_b200 import sample_table
    tab = torch.from_numpy(sample_table(fn))
    want = fn(_values()).reshape(3, 256)
    assert tab.dtype == torch.float32 and tuple(tab.shape) == (3, 256)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        assert torch.equal(tab.to(dt).view(torch.int16 if dt != torch.float32 else torch.int32),
                           want.to(dt).view(torch.int16 if dt != torch.float32 else torch.int32)), (name, dt)


@pytest.mark.parametrize("fn,count", [(_v1, 562), (_v2, 643)])
def test_affine_map_is_not_torchvision(fn, count):
    """fp32(fp32(v s) + b) with s = 1 / (255 std), b = -mean / std differs from ToTensor + Normalize in 562 of the 768 (v, c) in
    float32, and from v2's ToDtype + Normalize in 643: the reason for the table (float16 / bfloat16 happen to agree here)"""
    import torch
    pytest.importorskip("torchvision")
    v = torch.arange(256, dtype=torch.float32)
    s = torch.tensor([1 / (255 * x) for x in STD], dtype=torch.float32)
    b = torch.tensor([-m / x for m, x in zip(MEAN, STD)], dtype=torch.float32)
    affine = (v.view(1, 256) * s.view(3, 1)) + b.view(3, 1)  # two roundings, as the kernels compute
    want = fn(_values()).reshape(3, 256)
    assert int((affine != want).sum()) == count
    assert torch.equal(affine.half(), want.half()) and torch.equal(affine.bfloat16(), want.bfloat16())


def test_sample_table_arguments():
    from libjpeg_b200 import sample_table
    assert sample_table(lambda t: t.float(), ncomp=1).shape == (1, 256)
    assert np.array_equal(sample_table(lambda t: t.float() * 2, ncomp=4)[3], np.arange(256, dtype=np.float32) * 2)
    for bad in (0, 5, True, 2.0):
        with pytest.raises(ValueError):
            sample_table(lambda t: t.float(), ncomp=bad)
    with pytest.raises(ValueError):
        sample_table(lambda t: t.float().flatten())
    # a result that requires grad is taken as its values
    w = __import__("torch").ones(1, requires_grad=True)
    assert np.array_equal(sample_table(lambda t: t.float() * w, ncomp=2)[1], np.arange(256, dtype=np.float32))


def test_table_args():
    """integer destinations and non-float32 tables are TypeError, other shapes ValueError; the struct holds the rows"""
    import torch
    from libjpeg_b200 import native
    from libjpeg_b200.decoder import table_args
    tab = np.random.default_rng(0).standard_normal((3, 256)).astype(np.float32)
    for dt in (torch.uint8, torch.int16):
        with pytest.raises(TypeError):
            table_args(dt, tab)
    with pytest.raises(TypeError):
        table_args(torch.float32, tab.astype(np.float64))
    for shape in ((5, 256), (3, 255), (256,), (0, 256)):
        with pytest.raises(ValueError):
            table_args(torch.float16, np.zeros(shape, np.float32))
    for rows, ncomp in ((1, 3), (3, 4), (2, 3)):
        with pytest.raises(ValueError):  # a row per output component: a missing one would write zeros
            table_args(torch.float32, tab[:rows], ncomp)
    t = table_args(torch.bfloat16, torch.from_numpy(tab), 3)
    assert t.type == native.SAMPLE_BF16
    got = np.ctypeslib.as_array(t.table)
    assert np.array_equal(got[:3], tab) and not got[3].any()


def test_table_with_scale_or_bias():
    """a table with scale or bias is refused before anything else"""
    from libjpeg_b200 import BatchDecoder
    tab = np.zeros((3, 256), np.float32)
    for kw in ({"scale": 1.0}, {"bias": 0.5}):
        with pytest.raises(ValueError):
            BatchDecoder.decode_into(types.SimpleNamespace(), None, table=tab, **kw)
