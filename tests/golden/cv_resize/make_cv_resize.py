"""Writes tests/golden/cv_resize/digests.json: the SHA-256 digests of what OpenCV 4.13 makes of the stored fixtures
(tests/golden/*.jpg and tests/golden/resize_box/*.jpg) under cv2.resize -- cv2.imdecode(data, IMREAD_COLOR) (BGR) and
cv2.imdecode(data, IMREAD_GRAYSCALE), each resized to every size of sizes() with INTER_LINEAR and INTER_AREA -- as uint8
[h, w, C] arrays. Run from the repository root: python tests/golden/cv_resize/make_cv_resize.py"""
import glob
import hashlib
import json
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.dirname(HERE)


def fixtures():
    """(name, path) of the stored fixtures, name relative to tests/golden"""
    paths = sorted(glob.glob(os.path.join(GOLDEN, "*.jpg"))) + sorted(glob.glob(os.path.join(GOLDEN, "resize_box", "*.jpg")))
    return [(os.path.relpath(p, GOLDEN), p) for p in paths]


def sizes(w, h):
    """(W_t, H_t) targets of a w x h image: ultralytics' long side 640 (ceil(w r)), 224 x 224, an integer shrink, a fractional
    shrink and a growth on one axis with a shrink on the other"""
    r = 640 / max(w, h)
    return [(min(math.ceil(w * r), 640), min(math.ceil(h * r), 640)), (224, 224), (max(1, w // 2), max(1, h // 2)),
            (max(1, w * 2 // 3), max(1, h * 3 // 5)), (w + 7, max(1, h // 3))]


def digest(a):
    a = a[..., None] if a.ndim == 2 else a
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":%dx%dx%d" % a.shape


def main():
    import cv2
    out = {"opencv": cv2.__version__, "frames": {}}
    for name, path in fixtures():
        data = np.fromfile(path, dtype=np.uint8)
        entry = {}
        for mode, flag in (("color", cv2.IMREAD_COLOR), ("gray", cv2.IMREAD_GRAYSCALE)):
            img = cv2.imdecode(data, flag)
            h, w = img.shape[:2]
            for interp, iname in ((cv2.INTER_LINEAR, "linear"), (cv2.INTER_AREA, "area")):
                for tw, th in sizes(w, h):
                    entry["%s_%s_%dx%d" % (mode, iname, tw, th)] = digest(cv2.resize(img, (tw, th), interpolation=interp))
        out["frames"][name] = entry
    with open(os.path.join(HERE, "digests.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
