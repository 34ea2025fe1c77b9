"""Writes the CMYK / YCCK fixtures of tests/test_cmyk.py (DESIGN §15): small four-component JPEGs written by Pillow, their YCCK
twins, and expected.npz with Pillow's own convert("RGB") and convert("L") of each, so the GPU tests need no Pillow.

    python tests/golden/cmyk/make_cmyk.py

Pillow writes a CMYK image as Adobe-inverted samples with an APP14 "Adobe" segment of transform 0 right behind SOI. A YCCK twin is
the same file with that transform byte set to 2: libjpeg then reads its first three components as YCC (the same coefficients, a
different colour space). Pillow decodes either through libjpeg to CMYK and converts that.
"""
import io
import os

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))

# (width, height, quality, subsampling, restart_marker_rows): 4:4:4, the first component 2 x 2 (Pillow's subsampling=2 on CMYK),
# and restart markers
FILES = [(64, 48, 90, 0, 0), (97, 61, 75, 2, 0), (123, 45, 80, 0, 1), (40, 72, 85, 2, 2)]


def source(w, h, seed):
    """smooth ramps per channel plus noise: every channel covers most of 0..255, so the conversion is exercised everywhere"""
    rng = np.random.default_rng(seed)
    x = np.arange(w, dtype=np.float32)[None, :] / max(w - 1, 1)
    y = np.arange(h, dtype=np.float32)[:, None] / max(h - 1, 1)
    img = np.stack([255 * x + 0 * y, 255 * y + 0 * x, 255 * (1 - x) * (1 - y), 127 + 128 * np.sin(6 * x + 4 * y)], axis=-1)
    img = img + rng.normal(0, 10, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def write_cmyk(pixels, quality, subsampling, restart_rows):
    kw = dict(quality=quality, subsampling=subsampling)
    if restart_rows:
        kw["restart_marker_rows"] = restart_rows
    buf = io.BytesIO()
    Image.fromarray(pixels, "CMYK").save(buf, "JPEG", **kw)
    return buf.getvalue()


def adobe_transform_at(data):
    """the offset of the transform byte of the first APP14 "Adobe" segment"""
    i = data.find(b"\xff\xee")
    assert i >= 0 and data[i + 4:i + 9] == b"Adobe"
    return i + 4 + 11


def with_transform(data, transform):
    at = adobe_transform_at(data)
    return data[:at] + bytes([transform]) + data[at + 1:]


def main():
    expected = {}
    for k, (w, h, q, sub, rst) in enumerate(FILES):
        base = "%dx%d_s%d_q%d%s" % (w, h, sub, q, "_r%d" % rst if rst else "")
        cmyk = write_cmyk(source(w, h, k + 1), q, sub, rst)
        assert cmyk[adobe_transform_at(cmyk)] == 0
        for name, data in (("cmyk_" + base, cmyk), ("ycck_" + base, with_transform(cmyk, 2))):
            with open(os.path.join(HERE, name + ".jpg"), "wb") as f:
                f.write(data)
            im = Image.open(io.BytesIO(data))
            assert im.mode == "CMYK"
            expected[name + "_RGB"] = np.asarray(im.convert("RGB"))
            expected[name + "_L"] = np.asarray(im.convert("L"))
    np.savez_compressed(os.path.join(HERE, "expected.npz"), **expected)
    print("wrote %d files" % (2 * len(FILES)))


if __name__ == "__main__":
    main()
