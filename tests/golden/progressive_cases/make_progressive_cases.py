"""Regenerates tests/golden/progressive_cases/reference.json: what the UNMODIFIED reference decoder (oracle/_ref/refharness) makes of
every stream of tests/progressive_cases.py -- per case the SHA-256 of the stream, the reference's return code (0, or the error
code it reports) and, where it decoded the stream, the shape and the SHA-256 of its samples (null where it refused it).

Run where the reference is built (make -C oracle ref):  python tests/golden/progressive_cases/make_progressive_cases.py
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)

from tests import oracle_binding  # noqa: E402
from tests import progressive_cases as pc  # noqa: E402


def main():
    assert oracle_binding.have_reference(), "needs the reference build (make -C oracle ref)"
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in pc.NAMES:
            data = pc.case(name)[1]
            jpg, raw = os.path.join(tmp, "s.jpg"), os.path.join(tmp, "s.raw")
            open(jpg, "wb").write(data)
            r = subprocess.run([oracle_binding.REF_HARNESS, "decode", jpg, raw], capture_output=True, text=True)
            d = {"input_sha256": hashlib.sha256(data).hexdigest(), "rc": 0, "shape": None, "sha256": None}
            if r.returncode != 0:
                m = re.search(r"reference error (-?\d+)", r.stderr)
                d["rc"] = int(m.group(1)) if m else -1
            else:
                f = r.stdout.split()
                w, h, depth = map(int, f[:3])
                px = np.fromfile(raw, dtype=np.uint16 if len(f) > 3 else np.uint8).reshape(h, w, depth)
                d["shape"] = [h, w, depth]
                d["sha256"] = hashlib.sha256(np.ascontiguousarray(px).tobytes()).hexdigest()
            out[name] = d
    json.dump(out, open(os.path.join(HERE, "reference.json"), "w"), indent=1, sort_keys=True)
    print(len(out), "cases")


if __name__ == "__main__":
    main()
