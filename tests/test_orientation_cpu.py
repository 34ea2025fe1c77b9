"""CPU: the Exif orientation the parser reads (b200jpg_exif_orientation), on APP1 segments spliced into golden vectors. A segment
never changes the parse status or the frame info. Also the numpy definition of the eight orientations and the descriptor rewrite
that applies them, on small arrays. No device needed."""
import ctypes
import glob
import os
import struct

import numpy as np
import pytest

from tests import orientation_model as om

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BASE = ["c420_96x80_z6_q75.jpg", "c444_17x9_q95.jpg", "g_40x24_z2_q75.jpg", os.path.join("deep12", "d12_422_127x99_z5_q75.jpg")]


def _read(name):
    return open(os.path.join(GOLDEN, name), "rb").read()


def _parse(built, data):
    from libjpeg_b200 import native
    s = native.FrameInfoStruct()
    rc = native.lib.b200jpg_parse(data, len(data), ctypes.byref(s))
    return rc, bytes(s)


def _check(built, data, segments, want):
    from libjpeg_b200 import decoder
    tagged = om.splice(data, *segments)
    assert decoder.exif_orientation(tagged) == want
    assert _parse(built, tagged) == _parse(built, data)


@pytest.mark.parametrize("name", BASE)
@pytest.mark.parametrize("order", ["II", "MM"])
@pytest.mark.parametrize("o", list(om.ORIENTATIONS))
def test_values(built, name, order, o):
    _check(built, _read(name), [om.exif_segment(o, order)], o)


@pytest.mark.parametrize("order", ["II", "MM"])
@pytest.mark.parametrize("value", [0, 9, 0xFFFF])
def test_values_out_of_range(built, order, value):
    _check(built, _read(BASE[0]), [om.exif_segment(value, order)], 1)


@pytest.mark.parametrize("order", ["II", "MM"])
def test_type_and_count(built, order):
    data = _read(BASE[0])
    _check(built, data, [om.exif_segment(6, order, typ=4)], 1)    # LONG
    _check(built, data, [om.exif_segment(6, order, count=2)], 1)  # two SHORTs


@pytest.mark.parametrize("order", ["II", "MM"])
def test_offsets_outside_the_segment(built, order):
    data = _read(BASE[0])
    seg = om.exif_segment(6, order, ifd_offset=8)
    _check(built, data, [seg], 6)
    # IFD0 beyond the segment, or its count field half inside
    _check(built, data, [om.app1(b"Exif\0\0" + om.tiff(6, order, ifd_offset=4000)[:8])], 1)
    t = om.tiff(6, order)
    _check(built, data, [om.app1(b"Exif\0\0" + t[:9])], 1)
    # the entry count runs past the end: the orientation entry is the one cut off
    e = "<" if order == "II" else ">"
    make = (0x010F, 2, 4, b"abc\0")
    orient = (0x0112, 3, 1, struct.pack(e + "HH", 6, 0))
    t = om.tiff(order=order, entries=[make, orient])
    _check(built, data, [om.app1(b"Exif\0\0" + t[:8 + 2 + 12 + 11])], 1)
    _check(built, data, [om.app1(b"Exif\0\0" + t[:8 + 2 + 12 + 12])], 6)  # the entry whole, the next-IFD offset cut: still read
    # an IFD0 count far past the segment: the entries that are inside are still read
    big = bytearray(om.tiff(6, order))
    big[8:10] = struct.pack(e + "H", 500)
    _check(built, data, [om.app1(b"Exif\0\0" + bytes(big))], 6)


@pytest.mark.parametrize("cut", [0, 1, 3, 4, 7])
def test_cut_inside_the_tiff_header(built, cut):
    _check(built, _read(BASE[0]), [om.app1(b"Exif\0\0" + om.tiff(6)[:cut])], 1)


@pytest.mark.parametrize("order", ["II", "MM"])
def test_bad_tiff_header(built, order):
    t = bytearray(om.tiff(6, order))
    t[2] ^= 0xFF
    _check(built, _read(BASE[0]), [om.app1(b"Exif\0\0" + bytes(t))], 1)


@pytest.mark.parametrize("order", ["II", "MM"])
def test_tag_only_in_ifd1(built, order):
    make = (0x010F, 2, 4, b"abc\0")
    e = "<" if order == "II" else ">"
    t = om.tiff(order=order, entries=[make], ifd1=[(0x0112, 3, 1, struct.pack(e + "HH", 6, 0))])
    _check(built, _read(BASE[0]), [om.app1(b"Exif\0\0" + t)], 1)


def test_first_exif_segment_decides(built):
    data = _read(BASE[0])
    _check(built, data, [om.exif_segment(3), om.exif_segment(6)], 3)
    _check(built, data, [om.exif_segment(8, "MM"), om.exif_segment(2, "II")], 8)
    _check(built, data, [om.app1(b"Exif\0\0" + b"XX*\0" + bytes(8)), om.exif_segment(6)], 1)  # a malformed first one: 1


def test_not_exif(built):
    data = _read(BASE[0])
    bad_id = om.app1(b"Exif\0X" + om.tiff(6))
    xmp = om.app1(b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta xmlns:x='adobe:ns:meta/'><tiff:Orientation>6</tiff:Orientation></x:xmpmeta>")
    _check(built, data, [bad_id], 1)
    _check(built, data, [xmp], 1)
    _check(built, data, [bad_id, om.exif_segment(8)], 8)  # neither is an Exif segment: the next one decides
    _check(built, data, [xmp, om.exif_segment(5)], 5)
    _check(built, data, [om.app1(b"")], 1)


def test_exif_after_the_first_scan_is_ignored(built):
    from libjpeg_b200 import decoder
    path = sorted(glob.glob(os.path.join(GOLDEN, "progressive", "*.jpg")))[0]
    data = open(path, "rb").read()
    first = data.find(b"\xff\xda")
    second = data.find(b"\xff\xda", first + 2)
    assert first > 0 and second > first
    tagged = data[:second] + om.exif_segment(6) + data[second:]
    assert decoder.exif_orientation(tagged) == 1
    assert _parse(built, tagged) == _parse(built, data)
    assert decoder.exif_orientation(om.splice(tagged, om.exif_segment(3))) == 3


def test_reference_vectors_with_an_empty_ifd0(built):
    from libjpeg_b200 import decoder
    names = ["g_40x24_z2_q75.jpg"] + [os.path.join("xt", os.path.basename(p)) for p in sorted(glob.glob(os.path.join(GOLDEN, "xt", "*.jpg")))
                                      if "__nimpl" not in p]
    for name in names:
        data = _read(name)
        assert b"Exif\0\0" in data, name
        assert decoder.exif_orientation(data) == 1, name


def test_parse_errors_pass_through(built):
    from libjpeg_b200 import decoder, native
    with pytest.raises(native.NativeError) as e:
        decoder.exif_orientation(om.exif_segment(6))
    rc, _ = _parse(built, om.exif_segment(6))
    assert e.value.code == rc < 0
    assert native.lib.b200jpg_exif_orientation(b"\xff\xd8" + om.exif_segment(6), 2 + len(om.exif_segment(6))) < 0


def test_numpy_table_against_the_definition():
    a, b, c, d, e, f = range(1, 7)
    D = np.array([[a, b, c], [d, e, f]])
    want = {
        1: [[a, b, c], [d, e, f]],
        2: [[c, b, a], [f, e, d]],
        3: [[f, e, d], [c, b, a]],
        4: [[d, e, f], [a, b, c]],
        5: [[a, d], [b, e], [c, f]],
        6: [[d, a], [e, b], [f, c]],
        7: [[f, c], [e, b], [d, a]],
        8: [[c, f], [b, e], [a, d]],
    }
    for o in om.ORIENTATIONS:
        assert om.orient(D, o).tolist() == want[o], o


@pytest.mark.parametrize("o", list(om.ORIENTATIONS))
@pytest.mark.parametrize("layout", ["planar", "interleaved", "padded"])
def test_descriptor_rewrite(o, layout):
    """the rewritten descriptor, walked in decoded coordinates, writes exactly the oriented image into the destination that
    the original descriptor describes in output coordinates"""
    h, w, nc = 5, 7, 3
    D = np.arange(h * w * nc, dtype=np.int64).reshape(h, w, nc) + 1
    want = om.orient(D, o)
    oh, ow = want.shape[:2]
    if layout == "planar":
        p, r, cstep, size = 1, ow, oh * ow, nc * oh * ow
    elif layout == "interleaved":
        p, r, cstep, size = nc, ow * nc, 1, oh * ow * nc
    else:
        p, r, cstep, size = nc + 1, (ow + 3) * (nc + 1), 1, (oh + 1) * (ow + 3) * (nc + 1)
    buf = np.zeros(size + 16, dtype=np.int64)
    for c in range(nc):
        data, pp, rr = om.orient_plane(2 + c * cstep, p, r, o, w, h)
        for y in range(h):
            for x in range(w):
                buf[data + x * pp + y * rr] = D[y, x, c]
    for c in range(nc):
        for i in range(oh):
            for j in range(ow):
                assert buf[2 + c * cstep + j * p + i * r] == want[i, j, c]
    assert np.count_nonzero(buf) == h * w * nc
