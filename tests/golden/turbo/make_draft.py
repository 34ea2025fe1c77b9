"""Writes draft_digests.json: for every stored vector of make_turbo.py's sets that Pillow decodes, at k = 2, 4 and 8 and under the
modes "RGB" and "L", the request (w, h) = (max(1, W // k), max(1, H // k)), the scale Pillow's draft picks for it
(decoderconfig[0]) and the SHA-256 and shape of np.asarray(im.convert(mode)) after im.draft(mode, (w, h)). tests/test_draft.py
compares the GPU's drafted output with these digests on machines without Pillow; tests/test_draft_cpu.py checks them against
Pillow wherever it is installed. Run from the repository root: python tests/golden/turbo/make_draft.py"""
import importlib.util
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.dirname(HERE)
SCALES = (2, 4, 8)
MODES = ("RGB", "L")


def _make_turbo():
    spec = importlib.util.spec_from_file_location("make_turbo", os.path.join(HERE, "make_turbo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def request(size, k):
    """the (w, h) Pillow's draft is asked for to decode a W x H frame at 1/k (a smaller k where the frame is too small for it)"""
    return max(1, size[0] // k), max(1, size[1] // k)


def pillow_draft(rel, mode, k):
    """(Pillow's scale, its drafted pixels under `mode`), or None for a vector Pillow does not read"""
    from PIL import Image
    try:
        with Image.open(os.path.join(GOLDEN, rel)) as im:
            im.draft(mode, request(im.size, k))
            scale = im.decoderconfig[0] if im.decoderconfig else 1
            return scale, np.ascontiguousarray(np.asarray(im.convert(mode)))
    except OSError:
        return None


def table():
    mk = _make_turbo()
    out = {}
    for rel in mk.vectors():
        for k in SCALES:
            for mode in MODES:
                r = pillow_draft(rel, mode, k)
                if r is not None:
                    out["%s|%s|%d" % (rel, mode, k)] = {"scale": r[0], "shape": list(r[1].shape), "sha256": mk.digest(r[1])}
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "draft_digests.json"), "w") as f:
        json.dump(table(), f, indent=1, sort_keys=True)
        f.write("\n")
