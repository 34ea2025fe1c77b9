"""Device time per step of CMYK frames under reconstruction="libjpeg-turbo" and mode="RGB" (DESIGN §18), against the reference
path (§15), one GPU:

    python tools/turbo_cmyk_bench.py [--frames 256] [--steps 5] [--warmup 1] [--rounds 3] [--distinct 8] [--replace 3]

Timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds; the best round is reported next to
all of them. The frames are tools/cmyk_bench.py's: 1920x1080 CMYK (an Adobe segment of transform 0 on an 8-bit four-component
stream, one scan per component). Cases:
  ref_rgb         BatchDecoder(mode="RGB"), decode_into a uint8 [N, 3, H, W] tensor (the reference path's CMYK conversion)
  turbo_rgb       the same with reconstruction="libjpeg-turbo"
  turbo_draft_k   the same drafted to 1/k (k = 2, 4, 8), into [N, 3, ceil(H / k), ceil(W / k)]
  ref_mixed / turbo_mixed   tools/cmyk_bench.py's mixed_resized: 256 frames of bench.py's cfg2 (1080p 4:2:0) with `--replace` of
                  them CMYK, RandomResizedCrop-like rectangles, mode="RGB", resized to fp16 [N, 3, 224, 224] with the ImageNet map, on
                  each path
The entropy / reconstruction split of every case comes from the batch's event timing in a step of its own. Prints one JSON line
with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tests import crop_model as cm  # noqa: E402
from tools import bench_inputs  # noqa: E402
from tools.cmyk_bench import T, cmyk_frames  # noqa: E402
from tools.mode_bench import _timed  # noqa: E402
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

TURBO = "libjpeg-turbo"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--replace", type=int, default=3, help="CMYK frames in the mixed batch")
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    from libjpeg_b200 import decoder
    assert torch.cuda.is_available(), "turbo_cmyk_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    N = args.frames
    stream = torch.cuda.Stream()

    cmyk_base = cmyk_frames(args.distinct)
    cmyk = [cmyk_base[i % len(cmyk_base)] for i in range(N)]
    ycc_base = bench_inputs.make_frames("cfg2", 32, max(1, min(16, os.cpu_count() or 1)))
    ycc = [bytes(ycc_base[i % len(ycc_base)]) for i in range(N)]
    step = max(1, N // max(1, args.replace))
    mixed = [cmyk_base[i % len(cmyk_base)] if i % step == 0 and i // step < args.replace else f for i, f in enumerate(ycc)]
    r = np.random.default_rng(1)
    rects = [cm.rectangles(*decoder.output_size(f)[::-1], r, n_random=1)[-1] for f in mixed]

    decs = {"ref_rgb": libjpeg_b200.BatchDecoder(cmyk, mode="RGB"),
            "turbo_rgb": libjpeg_b200.BatchDecoder(cmyk, mode="RGB", reconstruction=TURBO)}
    H, W = decs["ref_rgb"].output_shape(0, 0)
    for k in (2, 4, 8):
        decs["turbo_draft_%d" % k] = libjpeg_b200.BatchDecoder(cmyk, mode="RGB", reconstruction=TURBO, draft=(H // k, W // k))
    decs["ref_mixed"] = libjpeg_b200.BatchDecoder(mixed, mode="RGB", crop=rects, resize=(T, T))
    decs["turbo_mixed"] = libjpeg_b200.BatchDecoder(mixed, mode="RGB", crop=rects, resize=(T, T), reconstruction=TURBO)
    for d in decs.values():
        d.upload(stream)
    torch.cuda.synchronize()
    dst = {}
    for v, d in decs.items():
        if v.endswith("mixed"):
            dst[v] = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
        else:
            h, w = d.output_shape(0, 0)
            dst[v] = torch.empty(N, 3, h, w, dtype=torch.uint8, device="cuda")

    def stepper(v):
        if v.endswith("mixed"):
            return lambda: decs[v].decode_into(dst[v], stream, scale=SCALE, bias=BIAS)
        return lambda: decs[v].decode_into(dst[v], stream)
    steps = {v: stepper(v) for v in decs}
    times = {v: [] for v in steps}
    for rnd in range(args.rounds):
        for v in (list(steps) if rnd % 2 == 0 else list(steps)[::-1]):
            times[v].append(_timed(steps[v], args, stream))
    split = {}
    for v, d in decs.items():
        d.enable_timing(True)
        steps[v]()
        torch.cuda.synchronize()
        split[v] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    failed = {v: sum(d.status(i) != 0 for i in range(N)) for v, d in decs.items()}
    shapes = {v: list(dst[v].shape) for v in dst}
    for d in decs.values():
        d.close()
    torch.cuda.empty_cache()
    line = {"metric": "device ms per step (CUDA events): 1080p CMYK frames under mode=RGB, reference path vs libjpeg-turbo path (full "
                      "size and drafted); a 1080p YCbCr batch with CMYK frames in it resized to fp16 [N, 3, 224, 224] on each path",
            "gpu": bench.gpu_facts(0), "frames": N, "size": "%dx%d" % (W, H), "cmyk_in_mixed": args.replace,
            "steps": args.steps, "rounds": args.rounds, "shapes": shapes,
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in times},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in times},
            "entropy_recon_ms": split, "failed_frames": failed}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
