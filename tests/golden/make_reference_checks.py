"""Regenerates tests/golden/reference/: what the UNMODIFIED reference (oracle/_ref/refharness, oracle/_ref/jpeg) makes of the
streams that tests/test_oracle.py builds with the repo's generator and its damage helpers, so that the oracle is pinned on the
reference without the reference being present:
  * reference_digests.json: per case the SHA-256 of the input stream and, where the reference decoded it, the shape and the
    SHA-256 of its samples (null where it refused the stream);
  * sub_<factors>.jpg: streams that the reference's ENCODER wrote for other chroma subsampling factors (`jpeg -s`);
  * tagitem_check.txt: the transcript of tests/client/tagitem_check.cpp compiled against the reference (oracle/_ref/tagitem_ref;
    tests/test_shim_cpu.py).

Run in the build container only (needs `make -C oracle ref`):  python tests/golden/make_reference_checks.py
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "reference")

from tests import oracle_binding  # noqa: E402
from tests import test_oracle as t  # noqa: E402


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def entry(data, px):
    d = {"input_sha256": sha(data), "shape": None, "sha256": None}
    if px is not None:
        d["shape"] = list(px.shape)
        d["sha256"] = sha(np.ascontiguousarray(px).tobytes())
    return d


def ref_decode(tmp, data):
    jpg = os.path.join(tmp, "s.jpg")
    open(jpg, "wb").write(data)
    return oracle_binding.reference_decode(jpg, os.path.join(tmp, "s.raw"))


def main():
    assert oracle_binding.have_reference(), "needs the reference build (make -C oracle ref)"
    os.makedirs(OUT, exist_ok=True)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for key, data in t.reference_cases():
            out[key] = entry(data, ref_decode(tmp, data))
        for sub in t.OTHER_SUBSAMPLING:
            w, h = 75, 61
            from libjpeg_b200 import synth
            ppm = os.path.join(tmp, "in.ppm")
            open(ppm, "wb").write(b"P6\n%d %d\n255\n" % (w, h) + synth.source_image(w, h, 17).tobytes())
            jpg = os.path.join(OUT, t.other_subsampling_name(sub) + ".jpg")
            subprocess.run([oracle_binding.REF_CLI, "-q", "80", "-bl", "-s", sub, "-z", "3", ppm, jpg], check=True, capture_output=True)
            data = open(jpg, "rb").read()
            out["other_subsampling[%s]" % sub] = entry(data, ref_decode(tmp, data))
        for name in t.NO_COLOR_TRANSFORM:
            src = os.path.join(t.GOLDEN, name + ".jpg")
            ppm = os.path.join(tmp, "o.ppm")
            subprocess.run([oracle_binding.REF_CLI, "-c", src, ppm], check=True, capture_output=True)
            magic, dims, maxv, rest = open(ppm, "rb").read().split(b"\n", 3)
            w, h = map(int, dims.split())
            out["no_color_transform[%s]" % name] = entry(open(src, "rb").read(), np.frombuffer(rest, dtype=np.uint8).reshape(h, w, 3))
    exe = os.path.join(ROOT, "oracle", "_ref", "tagitem_ref")
    open(os.path.join(OUT, "tagitem_check.txt"), "w").write(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    json.dump(out, open(os.path.join(OUT, "reference_digests.json"), "w"), indent=1, sort_keys=True)
    print(len(out), "cases")


if __name__ == "__main__":
    main()
