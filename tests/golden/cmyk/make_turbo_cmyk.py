"""Writes turbo_digests.json: for every CMYK / YCCK fixture of this directory, at k = 1, 2, 4 and 8 and under the modes "RGB" and
"L", the request (w, h) = (max(1, W // k), max(1, H // k)), the scale Pillow's draft picks for it (decoderconfig[0], 1 undrafted)
and the SHA-256 and shape of np.asarray(im.convert(mode)) after im.draft(mode, (w, h)) (no draft at k = 1). tests/test_turbo_cmyk.py
compares the GPU's output under reconstruction="libjpeg-turbo" with these digests on machines without Pillow;
tests/test_turbo_cmyk_cpu.py checks them against Pillow wherever it is installed (DESIGN §18).

    python tests/golden/cmyk/make_turbo_cmyk.py
"""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SCALES = (1, 2, 4, 8)
MODES = ("RGB", "L")


def fixtures():
    return sorted(f[:-4] for f in os.listdir(HERE) if f.endswith(".jpg"))


def request(size, k):
    return max(1, size[0] // k), max(1, size[1] // k)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def pillow(data, mode, k):
    """(Pillow's scale, its pixels under `mode`) of a codestream asked for 1/k (k = 1: Image.open(f).convert(mode))"""
    import io
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        if k > 1:
            im.draft(mode, request(im.size, k))
        scale = im.decoderconfig[0] if im.decoderconfig else 1
        return scale, np.ascontiguousarray(np.asarray(im.convert(mode)))


def table():
    out = {}
    for name in fixtures():
        with open(os.path.join(HERE, name + ".jpg"), "rb") as f:
            data = f.read()
        for k in SCALES:
            for mode in MODES:
                scale, px = pillow(data, mode, k)
                out["%s|%s|%d" % (name, mode, k)] = {"scale": scale, "shape": list(px.shape), "sha256": digest(px)}
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "turbo_digests.json"), "w") as f:
        json.dump(table(), f, indent=1, sort_keys=True)
        f.write("\n")
