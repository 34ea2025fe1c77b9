"""Writes the fixtures of tests/test_resize_box.py: Pillow-written JPEGs (seeded smooth images) and the SHA-256 digests of what
Pillow 12.2 and torchvision 0.26 make of them -- thumbnail(), ImageOps.fit() and Resize(256) + CenterCrop(224) -- as uint8
[h, w, C] arrays. Run from the repository root: python tests/golden/resize_box/make_resize_box.py"""
import hashlib
import io
import json
import os

import numpy as np
from PIL import Image, ImageOps

HERE = os.path.dirname(os.path.abspath(__file__))
# (name, width, height, mode, subsampling)
IMAGES = [("a_800x600_420", 800, 600, "RGB", 2), ("b_517x389_420", 517, 389, "RGB", 2), ("c_640x480_444", 640, 480, "RGB", 0),
          ("d_333x1000_grey", 333, 1000, "L", 0), ("e_901x507_422", 901, 507, "RGB", 1), ("f_300x200_420", 300, 200, "RGB", 2)]
THUMBS = [(128, 128), (64, 64), (100, 37), (2000, 2000)]  # (w, h), Pillow's order
FITS = [((224, 224), 0.0, (0.5, 0.5)), ((160, 90), 0.1, (0.2, 0.9))]


def smooth(w, h, seed, ch):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    planes = []
    for _ in range(ch):
        a, b, c, d = rng.uniform(0.005, 0.05, 4)
        planes.append(127.5 + 60 * np.sin(a * x + b * y) + 60 * np.cos(c * x - d * y) + rng.normal(0, 4, (h, w)))
    return np.clip(np.stack(planes, -1), 0, 255).astype(np.uint8)


def jpeg(name, w, h, mode, sub, seed):
    img = smooth(w, h, seed, 3 if mode == "RGB" else 1)
    im = Image.fromarray(img if mode == "RGB" else img[..., 0], mode)
    buf = io.BytesIO()
    im.save(buf, "JPEG", quality=75, subsampling=sub)
    return buf.getvalue()


def digest(im):
    a = np.asarray(im)
    a = a[..., None] if a.ndim == 2 else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":%dx%dx%d" % a.shape


def chains(data):
    """{chain name: digest} of one JPEG"""
    import torchvision.transforms as T
    out = {}
    for w, h in THUMBS:
        im = Image.open(io.BytesIO(data))
        im.thumbnail((w, h))
        out["thumbnail_%dx%d" % (w, h)] = digest(im)
    for (w, h), bleed, cen in FITS:
        out["fit_%dx%d_%g_%g_%g" % (w, h, bleed, cen[0], cen[1])] = digest(ImageOps.fit(Image.open(io.BytesIO(data)), (w, h), bleed=bleed,
                                                                                       centering=cen))
    t = T.Compose([T.Resize(256), T.CenterCrop(224)])
    out["resize256_crop224"] = digest(t(Image.open(io.BytesIO(data)).convert("RGB")))
    return out


def main():
    digests = {}
    for k, (name, w, h, mode, sub) in enumerate(IMAGES):
        data = jpeg(name, w, h, mode, sub, 100 + k)
        with open(os.path.join(HERE, name + ".jpg"), "wb") as f:
            f.write(data)
        digests[name] = chains(data)
    with open(os.path.join(HERE, "digests.json"), "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
