"""CPU: the tensor -> b200jpg_plane table of BatchDecoder.decode_into (libjpeg_b200.decoder.plane_table), on CPU tensors."""
import pytest

torch = pytest.importorskip("torch")


def _table(built, geometry, dst, device_type="cpu"):
    from libjpeg_b200.decoder import plane_table
    return plane_table(geometry, dst, device_type=device_type)


def _entry(table, i, c):
    e = table[4 * i + c]
    return e.data, e.bytes_per_pixel, e.bytes_per_row


G420 = ([(6, 10)] * 3, False)  # a 10 x 6 frame, three components, upsampled


def test_nchw_batch_tensor(built):
    t = torch.zeros(2, 3, 6, 10, dtype=torch.uint8)
    table = _table(built, [G420, G420], t)
    assert len(table) == 8
    for i in range(2):
        for c in range(3):
            assert _entry(table, i, c) == (t.data_ptr() + (3 * i + c) * 60, 1, 10)
        assert not table[4 * i + 3].data


def test_batch_tensor_equals_its_frames(built):
    """a 4-D tensor is described without a view per component: the same table as its frames one by one"""
    t = torch.zeros(5, 10, 6, 8, dtype=torch.int16).permute(0, 3, 2, 1)[:, :3]  # [5, 3, 6, 10] out of an odd layout
    geo = [([(6, 10)] * 3, True)] * 5
    geo[2] = None
    whole, parts = _table(built, geo, t), _table(built, geo, [None if g is None else t[i] for i, g in enumerate(geo)])
    assert [_entry(whole, k // 4, k % 4) for k in range(20)] == [_entry(parts, k // 4, k % 4) for k in range(20)]
    assert not whole[8].data
    with pytest.raises(ValueError):
        _table(built, [G420, ([(4, 7)] * 3, False)], torch.zeros(2, 3, 6, 10, dtype=torch.uint8))  # two geometries
    with pytest.raises(ValueError):
        _table(built, [G420], torch.zeros(1, 3, 6, 11, dtype=torch.uint8))


def test_nhwc_permuted(built):
    t = torch.zeros(2, 6, 10, 3, dtype=torch.uint8)
    table = _table(built, [G420, G420], t.permute(0, 3, 1, 2))
    for i in range(2):
        for c in range(3):
            assert _entry(table, i, c) == (t.data_ptr() + i * 180 + c, 3, 30)


def test_padded_slices(built):
    big = torch.zeros(2, 3, 6 + 3, 10 + 5, dtype=torch.uint8)
    table = _table(built, [G420, ([(4, 7)] * 3, False)], [big[0, :, :6, :10], big[1, :, :4, :7]])
    for c in range(3):
        assert _entry(table, 0, c) == (big.data_ptr() + c * 9 * 15, 1, 15)
        assert _entry(table, 1, c) == (big.data_ptr() + (3 + c) * 9 * 15, 1, 15)


def test_bgr_list(built):
    t = torch.zeros(6, 10, 3, dtype=torch.uint8)
    table = _table(built, [G420], [[t[..., 2], t[..., 1], t[..., 0]]])
    for c in range(3):
        assert _entry(table, 0, c) == (t.data_ptr() + 2 - c, 3, 30)


def test_12bit_int16_views_and_own_sizes(built):
    geo = ([(6, 10), (3, 5), (3, 5)], True)  # 12-bit 4:2:0 without upsampling
    y = torch.zeros(6, 10, dtype=torch.int16)
    cbcr = torch.zeros(2, 3, 8, dtype=torch.int16)[:, :, 1:6]
    table = _table(built, [geo], [[y, cbcr[0], cbcr[1]]])
    assert _entry(table, 0, 0) == (y.data_ptr(), 2, 20)
    assert _entry(table, 0, 1) == (cbcr.data_ptr(), 2, 16)
    assert _entry(table, 0, 2) == (cbcr.data_ptr() + 48, 2, 16)


def test_failed_frame_takes_none(built):
    t = torch.zeros(3, 6, 10, dtype=torch.uint8)
    table = _table(built, [None, G420], [None, t])
    assert all(not table[k].data for k in range(4))
    assert _entry(table, 1, 0) == (t.data_ptr(), 1, 10)
    with pytest.raises(ValueError):
        _table(built, [None, G420], [t, t])  # a failed frame has no destination
    with pytest.raises(ValueError):
        _table(built, [G420, G420], [None, t])  # a live frame needs one


@pytest.mark.parametrize("bad", ["shape", "dtype", "components", "frames", "not_a_tensor"])
def test_wrong_destinations_raise(built, bad):
    t = torch.zeros(3, 6, 10, dtype=torch.uint8)
    dst = {"shape": [torch.zeros(3, 6, 11, dtype=torch.uint8)],
           "dtype": [t.to(torch.int16)],
           "components": [t[:2]],
           "frames": [t, t],
           "not_a_tensor": [[t[0].numpy(), t[1], t[2]]]}[bad]
    with pytest.raises((ValueError, TypeError)):
        _table(built, [G420], dst)


def test_12bit_frame_refuses_uint8(built):
    with pytest.raises(TypeError):
        _table(built, [([(6, 10)], True)], [[torch.zeros(6, 10, dtype=torch.uint8)]])


def test_cpu_tensor_is_refused_for_the_device(built):
    t = torch.zeros(3, 6, 10, dtype=torch.uint8)
    with pytest.raises(ValueError):
        _table(built, [G420], [t], device_type="cuda")
