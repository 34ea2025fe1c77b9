"""Writes pil_digests.json: for every stored vector Pillow decodes, the SHA-256 of np.asarray(Image.open(f)) (uint8, [H, W] or
[H, W, 3] in C order) and its shape, keyed by the path under tests/golden. tests/test_turbo.py compares the GPU's
reconstruction="libjpeg-turbo" output with these digests on machines without Pillow; tests/test_turbo_cpu.py checks them against
Pillow wherever it is installed. Run from the repository root: python tests/golden/turbo/make_turbo.py"""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.dirname(HERE)
# the sets whose intact, 8-bit, one- or three-component codestreams the digests cover (Pillow refuses more than 10 blocks per MCU)
DIRS = ["", "progressive", "subsampling", "reference", "xt"]


def vectors():
    for d in DIRS:
        for name in sorted(os.listdir(os.path.join(GOLDEN, d))):
            if name.endswith(".jpg") and "__nimpl" not in name:
                yield os.path.join(d, name) if d else name


def pillow_pixels(rel):
    from PIL import Image
    try:
        with Image.open(os.path.join(GOLDEN, rel)) as im:
            return np.ascontiguousarray(np.asarray(im))
    except OSError:
        return None


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def table():
    out = {}
    for rel in vectors():
        a = pillow_pixels(rel)
        if a is not None:
            out[rel] = {"shape": list(a.shape), "sha256": digest(a)}
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "pil_digests.json"), "w") as f:
        json.dump(table(), f, indent=1, sort_keys=True)
        f.write("\n")
