"""The CMYK and YCCK conversions of the output modes (DESIGN §15) in numpy, and the codestreams the tests feed them: Adobe APP14
segments spliced into four-component streams. No Pillow here: tests/test_cmyk_cpu.py pins these functions on Pillow, and the GPU
tests use them as their oracle on top of the library's own decode without the mode."""
import numpy as np

CMYK, YCCK = "CMYK", "YCCK"


def muldiv255(a, b):
    t = a * b + 128
    return ((t >> 8) + t) >> 8


def ycc_to_rgb(y, cb, cr):
    """libjpeg's ycck_cmyk_convert before its inversion: R, G, B of Y, Cb - 128, Cr - 128 with its tables (arithmetic shifts),
    clamped to 0..255"""
    cb, cr = cb - 128, cr - 128
    r = y + ((91881 * cr + 32768) >> 16)
    g = y + ((-22554 * cb - 46802 * cr + 32768) >> 16)
    b = y + ((116130 * cb + 32768) >> 16)
    return [np.clip(v, 0, 255) for v in (r, g, b)]


def luma(rgb):
    rgb = np.asarray(rgb).astype(np.int64)
    return (19595 * rgb[..., 0] + 38470 * rgb[..., 1] + 7471 * rgb[..., 2] + 32768) >> 16


def to_rgb(s, space):
    """[..., 4] samples as the batch writes them without a mode -> [..., 3] uint8, Pillow's convert("RGB")"""
    s = np.asarray(s).astype(np.int64)
    if space == YCCK:
        a = ycc_to_rgb(s[..., 0], s[..., 1], s[..., 2])
    else:
        a = [255 - s[..., c] for c in range(3)]
    k = s[..., 3]
    return np.stack([k - muldiv255(a[c], k) for c in range(3)], axis=-1).astype(np.uint8)


def convert(s, space, mode):
    """the image BatchDecoder(mode=mode) writes for a CMYK / YCCK frame whose mode-less decode is s ([h, w, 4])"""
    rgb = to_rgb(s, space)
    return rgb if mode == "RGB" else luma(rgb)[..., None].astype(np.uint8)


def adobe(transform, payload=12, tag=b"Adobe"):
    """an APP14 segment whose payload is `payload` bytes: the tag, version 100, flags 0, and the transform byte at payload[11]
    (the payload is cut there when shorter)"""
    body = (tag + bytes([0, 100, 0, 0, 0, 0, transform]))[:payload].ljust(payload, b"\0")
    return b"\xff\xee" + (len(body) + 2).to_bytes(2, "big") + body


def after_soi(data, seg):
    return data[:2] + seg + data[2:]


def before_sos(data, seg, k=0):
    """seg in front of the k-th SOS marker (k = 0: between the frame header and the first scan)"""
    at = -1
    for _ in range(k + 1):
        at = data.find(b"\xff\xda", at + 1)
        assert at > 0
    return data[:at] + seg + data[at:]


def four_component(w, h, seed, sub=(1, 1), restart=0):
    """an unmarked 8-bit four-component stream, one scan per component: oracle_binding.with_fourth_component of a synthetic
    frame (the fourth component repeats the third)"""
    from libjpeg_b200 import synth
    from tests import oracle_binding
    return oracle_binding.with_fourth_component(synth.encode(synth.source_image(w, h, seed), 80, sub, restart, synth.NON_INTERLEAVED))


def deep12_four(w=64, h=32):
    """an unmarked 12-bit four-component stream (hand-built, tests/recon_cases.py)"""
    from tests import recon_cases as rc
    from tests import streamwriter as sw
    factors = [(1, 1)] * 4
    _, comps = rc.base(w, h, 7, factors)
    return sw.encode(rc.frame(w, h, comps, factors, precision=12))
