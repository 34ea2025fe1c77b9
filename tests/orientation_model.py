"""Exif orientation: APP1 segments for the tests, the numpy definition of the eight orientations, and a restatement of the
descriptor rewrite the batch path applies (abi.cpp: orient_plane, DESIGN §11)."""
import struct

import numpy as np

ORIENTATIONS = range(1, 9)


def orient(d, o):
    """D ([H, W, ...] as written without the flag) -> O as written with orientation o (PIL's ImageOps.exif_transpose)"""
    return {
        1: lambda a: a,
        2: lambda a: a[:, ::-1],
        3: lambda a: a[::-1, ::-1],
        4: lambda a: a[::-1, :],
        5: lambda a: a.swapaxes(0, 1),
        6: lambda a: np.rot90(a, -1),
        7: lambda a: a[::-1, ::-1].swapaxes(0, 1),
        8: lambda a: np.rot90(a, 1),
    }[o](d)


def orient_plane(data, p, r, o, w, h):
    """(data, bytes_per_pixel, bytes_per_row) in output coordinates -> the same destination in the decoded coordinates of a
    component of decoded extent w x h"""
    W, H = w - 1, h - 1
    return {
        1: (data, p, r),
        2: (data + W * p, -p, r),
        3: (data + W * p + H * r, -p, -r),
        4: (data + H * r, p, -r),
        5: (data, r, p),
        6: (data + H * p, r, -p),
        7: (data + H * p + W * r, -r, -p),
        8: (data + W * r, -r, p),
    }[o]


def tiff(value=None, order="II", typ=3, count=1, ifd_offset=8, entries=None, ifd1=None):
    """A TIFF structure: header, IFD0 with `entries` ([(tag, type, count, 4-byte value field)]; default: one orientation entry of
    `value`), the offset of IFD1, and IFD1 with the entries `ifd1` if given"""
    e = "<" if order == "II" else ">"
    if entries is None:
        entries = [(0x0112, typ, count, struct.pack(e + "HH", value, 0) if typ == 3 else struct.pack(e + "I", value))]
    hdr = (b"II*\0" if order == "II" else b"MM\0*") + struct.pack(e + "I", ifd_offset)
    body = b"\0" * (ifd_offset - 8)

    def ifd(ents, next_off):
        return struct.pack(e + "H", len(ents)) + b"".join(struct.pack(e + "HHI", t, ty, c) + v for t, ty, c, v in ents) + \
            struct.pack(e + "I", next_off)

    ifd0_len = 2 + 12 * len(entries) + 4
    next_off = ifd_offset + ifd0_len if ifd1 else 0
    out = hdr + body + ifd(entries, next_off)
    if ifd1:
        out += ifd(ifd1, 0)
    return out


def app1(payload):
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def exif_segment(value, order="II", **kw):
    return app1(b"Exif\0\0" + tiff(value, order, **kw))


def splice(data, *segments):
    """the segments behind SOI"""
    return data[:2] + b"".join(segments) + data[2:]


def tag(data, o):
    """data with an Exif segment of orientation o behind SOI"""
    return splice(data, exif_segment(o))
