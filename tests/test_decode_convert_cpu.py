"""CPU: float destinations of BatchDecoder.decode_into -- the plane table of float tensors, the b200jpg_convert Python builds,
and the numpy rounding functions the GPU tests use as their expectation, pinned against torch on CPU."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

FLOATS = [torch.float32, torch.float16, torch.bfloat16]
G420 = ([(6, 10)] * 3, False)  # a 10 x 6 frame, three components, upsampled
G12 = ([(6, 10)] * 3, True)    # the same, 12-bit


# ---- the expectation: what decode_into writes for an integer sample array `v` --------------------------------------------
def to_f16_bits(y):
    """float32 array -> float16 bit patterns, round to nearest even, overflow to inf, subnormals kept"""
    with np.errstate(over="ignore"):
        return np.asarray(y, dtype=np.float32).astype(np.float16).view(np.uint16)


def to_bf16_bits(y):
    """float32 array -> bfloat16 bit patterns, round to nearest even (the inputs are never NaN)"""
    u = np.asarray(y, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def convert(v, scale, bias, dtype):
    """the element bytes of fp32_round(fp32_round(v * scale) + bias) in `dtype` (a torch float dtype)"""
    with np.errstate(over="ignore"):
        y = np.asarray(v).astype(np.float32) * np.float32(scale)
        y = y + np.float32(bias)
    if dtype == torch.float32:
        return y.view(np.uint32)
    return to_f16_bits(y) if dtype == torch.float16 else to_bf16_bits(y)


def _bit_classes():
    """float32 values from every class the roundings treat differently"""
    rng = np.random.default_rng(7)
    parts = [
        rng.integers(0, 1 << 32, 200000, dtype=np.uint64).astype(np.uint32).view(np.float32),  # every exponent
        np.float32([0.0, -0.0, 1.0, -1.0, 65504.0, 65519.99, 65520.0, 65536.0, 1e30, -1e30, 3.4e38, -3.4e38]),
        np.float32([2.0 ** -14, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -26, 2.0 ** -15 * 1.0009765625]),  # fp16 subnormals
        np.float32([2.0 ** -126, 2.0 ** -149, 1e-40, -1e-40]),  # fp32 subnormals: bf16 keeps them
    ]
    # ties: exactly half-way between two neighbours of the narrow type, odd and even below
    base = rng.integers(0x3000_0000, 0x4700_0000, 20000, dtype=np.uint64).astype(np.uint32)
    parts.append(((base & ~np.uint32(0x1FFF)) | np.uint32(0x1000)).view(np.float32))  # fp16 ties (13 dropped bits)
    parts.append(((base & ~np.uint32(0xFFFF)) | np.uint32(0x8000)).view(np.float32))  # bf16 ties
    parts.append(((base & ~np.uint32(0xFFFF)) | np.uint32(0x18000)).view(np.float32))
    parts.append(np.float32([np.finfo(np.float32).max, -np.finfo(np.float32).max, np.inf, -np.inf]))
    y = np.concatenate(parts)
    return y[np.isfinite(y) | np.isinf(y)]  # no NaN: the map of finite parameters never makes one


def test_f16_rounding_matches_torch():
    y = _bit_classes()
    want = torch.from_numpy(y.copy()).half().view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(to_f16_bits(y), want)


def test_bf16_rounding_matches_torch():
    y = _bit_classes()
    want = torch.from_numpy(y.copy()).bfloat16().view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(to_bf16_bits(y), want)


@pytest.mark.parametrize("dtype", FLOATS)
def test_conversion_is_torch_float_multiply_add(dtype):
    """convert() is t.float() * scale + bias followed by the cast, for 8- and 12-bit sample values and awkward maps"""
    v = np.arange(4096, dtype=np.int32)
    for scale, bias in [(1.0, 0.0), (1 / (255 * 0.229), -0.485 / 0.229), (-3.7, 12.5), (300.0, 0.0), (1e-9, 0.0), (2.0 ** -30, 1e-7)]:
        t = torch.from_numpy(v).float() * torch.tensor(scale, dtype=torch.float32) + torch.tensor(bias, dtype=torch.float32)
        want = t.to(dtype).view(torch.int32 if dtype == torch.float32 else torch.int16).numpy()
        got = convert(v, scale, bias, dtype)
        assert np.array_equal(got, want.view(got.dtype)), (dtype, scale, bias)


# ---- the plane table of float tensors ----------------------------------------------------------------------------------------
def _table(geometry, dst):
    from libjpeg_b200.decoder import plane_table
    return plane_table(geometry, dst, device_type="cpu")


def _entry(table, i, c):
    e = table[4 * i + c]
    return e.data, e.bytes_per_pixel, e.bytes_per_row


@pytest.mark.parametrize("dtype", FLOATS)
def test_nchw_float_strides_in_bytes(built, dtype):
    t = torch.zeros(2, 3, 6, 10, dtype=dtype)
    isz = t.element_size()
    table = _table([G420, G12], t)
    for i in range(2):
        for c in range(3):
            assert _entry(table, i, c) == (t.data_ptr() + (3 * i + c) * 60 * isz, isz, 10 * isz)


@pytest.mark.parametrize("dtype", FLOATS)
def test_float_batch_tensor_equals_its_frames(built, dtype):
    t = torch.zeros(5, 10, 6, 8, dtype=dtype).permute(0, 3, 2, 1)[:, :3]
    geo = [G420] * 5
    geo[3] = None
    whole, parts = _table(geo, t), _table(geo, [None if g is None else t[i] for i, g in enumerate(geo)])
    assert [_entry(whole, k // 4, k % 4) for k in range(20)] == [_entry(parts, k // 4, k % 4) for k in range(20)]


@pytest.mark.parametrize("dtype", FLOATS)
def test_channels_last_float(built, dtype):
    t = torch.zeros(2, 6, 10, 3, dtype=dtype)
    isz = t.element_size()
    table = _table([G420, G420], t.permute(0, 3, 1, 2))
    for i in range(2):
        for c in range(3):
            assert _entry(table, i, c) == (t.data_ptr() + (i * 180 + c) * isz, 3 * isz, 30 * isz)
    bgr = _table([G420], [[t[0, ..., 2], t[0, ..., 1], t[0, ..., 0]]])
    assert [_entry(bgr, 0, c) for c in range(3)] == [(t.data_ptr() + (2 - c) * isz, 3 * isz, 30 * isz) for c in range(3)]


def test_one_dtype_per_call(built):
    a, b = torch.zeros(3, 6, 10, dtype=torch.float16), torch.zeros(3, 6, 10, dtype=torch.bfloat16)
    u8 = torch.zeros(3, 6, 10, dtype=torch.uint8)
    for dst in ([a, b], [a, u8], [u8, a], [[a[0], b[1], a[2]], a]):
        with pytest.raises(TypeError):
            _table([G420, G420], dst)
    _table([G420, G12], [a, a.clone()])  # a float dtype serves 8- and 12-bit frames alike


def test_integer_rules_are_unchanged(built):
    """int16 for an 8-bit frame and uint8 for a 12-bit frame still raise; uint8 and int16 still mix in one call"""
    with pytest.raises(TypeError):
        _table([G420], [torch.zeros(3, 6, 10, dtype=torch.int16)])
    with pytest.raises(TypeError):
        _table([G12], [torch.zeros(3, 6, 10, dtype=torch.uint8)])
    with pytest.raises(TypeError):
        _table([G420], torch.zeros(1, 3, 6, 10, dtype=torch.int32))
    _table([G420, G12], [torch.zeros(3, 6, 10, dtype=torch.uint8), torch.zeros(3, 6, 10, dtype=torch.int16)])


# ---- the b200jpg_convert -------------------------------------------------------------------------------------------------------
def _conv(*a, **k):
    from libjpeg_b200.decoder import convert_args
    return convert_args(*a, **k)


def test_convert_types_and_defaults(built):
    from libjpeg_b200 import native
    assert [_conv(d, ncomp=3).type for d in FLOATS] == [native.SAMPLE_F32, native.SAMPLE_F16, native.SAMPLE_BF16]
    c = _conv(torch.float16, ncomp=3)
    assert list(c.scale) == [1.0] * 4 and list(c.bias) == [0.0] * 4
    assert _conv(torch.uint8) is None and _conv(torch.int16) is None
    with pytest.raises(TypeError):
        _conv(torch.uint8, scale=2.0)


def test_convert_scalar_broadcast_and_lists(built):
    c = _conv(torch.float32, scale=0.5, bias=np.float64(-2.0), ncomp=3)
    assert list(c.scale) == [0.5] * 4 and list(c.bias) == [-2.0] * 4
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    c = _conv(torch.bfloat16, scale=[1 / (255 * s) for s in std], bias=torch.tensor([-m / s for m, s in zip(mean, std)]), ncomp=3)
    assert list(c.scale)[:3] == [float(np.float32(1 / (255 * s))) for s in std] and c.scale[3] == 1.0
    assert list(c.bias)[:3] == [float(np.float32(-m / s)) for m, s in zip(mean, std)] and c.bias[3] == 0.0
    c = _conv(torch.float16, scale=torch.tensor(3.0), ncomp=1)
    assert list(c.scale) == [3.0] * 4


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf"), 1e39])
def test_convert_refuses_non_finite(built, bad):
    with pytest.raises(ValueError):
        _conv(torch.float16, scale=bad, ncomp=3)
    with pytest.raises(ValueError):
        _conv(torch.float32, bias=[0.0, bad, 0.0], ncomp=3)


def test_convert_refuses_wrong_lengths(built):
    for v in ([1.0, 2.0], [1.0] * 4, []):
        with pytest.raises(ValueError):
            _conv(torch.float32, scale=v, ncomp=3)
        with pytest.raises(ValueError):
            _conv(torch.float32, bias=v, ncomp=3)
    assert math.isclose(_conv(torch.float32, scale=[2.0], ncomp=1).scale[0], 2.0)
