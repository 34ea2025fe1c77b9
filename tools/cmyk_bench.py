"""Device time per step of CMYK frames under an output mode (BatchDecoder(mode="RGB"), DESIGN §15), one GPU:

    python tools/cmyk_bench.py [--frames 256] [--steps 5] [--warmup 1] [--rounds 3] [--distinct 8] [--replace 3]

Timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds; the best round is reported next to
all of them. Cases:
  cmyk_rgb        256 synthetic 1920x1080 CMYK frames (an Adobe segment of transform 0 on an 8-bit four-component stream, one
                  scan per component), BatchDecoder(mode="RGB"), decode_into a uint8 [N, 3, H, W] tensor
  cmyk_plain      the same frames without a mode, decode_into a uint8 [N, 4, H, W] tensor: the same entropy decode and IDCT,
                  four components stored instead of three converted ones
  ycbcr_resized   256 frames of bench.py's cfg2 (1080p 4:2:0) with RandomResizedCrop-like rectangles, mode="RGB", resized to
                  fp16 [N, 3, 224, 224] with the ImageNet map
  mixed_resized   the same batch with `--replace` of its frames replaced by CMYK ones (their own rectangles)
The entropy / reconstruction split of every case comes from the batch's event timing in a step of its own. Prints one
JSON line with the card's name and power limit, read in the same run.
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
from tests import cmyk_model as km  # noqa: E402
from tests import crop_model as cm  # noqa: E402
from tools import bench_inputs  # noqa: E402
from tools.mode_bench import _timed  # noqa: E402
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

T = 224


def cmyk_frames(distinct, w=1920, h=1080):
    return [km.after_soi(km.four_component(w, h, 100 + s, (1, 1), (w + 7) // 8), km.adobe(0)) for s in range(distinct)]


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
    assert torch.cuda.is_available(), "cmyk_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    N = args.frames
    stream = torch.cuda.Stream()

    cmyk_base = cmyk_frames(args.distinct)
    cmyk = [cmyk_base[i % len(cmyk_base)] for i in range(N)]
    ycc_base = bench_inputs.make_frames("cfg2", 32, max(1, min(16, os.cpu_count() or 1)))
    ycc = [bytes(ycc_base[i % len(ycc_base)]) for i in range(N)]
    step = max(1, N // max(1, args.replace))
    mixed = [cmyk_base[i % len(cmyk_base)] if i % step == 0 and i // step < args.replace else f for i, f in enumerate(ycc)]
    rects = {}
    for name, frames in (("ycbcr_resized", ycc), ("mixed_resized", mixed)):
        r = np.random.default_rng(1)
        rects[name] = [cm.rectangles(*decoder.output_size(f)[::-1], r, n_random=1)[-1] for f in frames]

    rgb = libjpeg_b200.BatchDecoder(cmyk, mode="RGB")
    plain = libjpeg_b200.BatchDecoder(cmyk)
    resized = {name: libjpeg_b200.BatchDecoder(frames, mode="RGB", crop=rects[name], resize=(T, T))
               for name, frames in (("ycbcr_resized", ycc), ("mixed_resized", mixed))}
    decs = [rgb, plain] + list(resized.values())
    for d in decs:
        d.upload(stream)
    torch.cuda.synchronize()
    H, W = rgb.output_shape(0, 0)
    t3 = torch.empty(N, 3, H, W, dtype=torch.uint8, device="cuda")
    t4 = torch.empty(N, 4, H, W, dtype=torch.uint8, device="cuda")
    out = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
    steps = {
        "cmyk_rgb": lambda: rgb.decode_into(t3, stream),
        "cmyk_plain": lambda: plain.decode_into(t4, stream),
        "ycbcr_resized": lambda: resized["ycbcr_resized"].decode_into(out, stream, scale=SCALE, bias=BIAS),
        "mixed_resized": lambda: resized["mixed_resized"].decode_into(out, stream, scale=SCALE, bias=BIAS),
    }
    times = {v: [] for v in steps}
    for rnd in range(args.rounds):
        for v in (list(steps) if rnd % 2 == 0 else list(steps)[::-1]):
            times[v].append(_timed(steps[v], args, stream))
    split = {}
    for v, d in [("cmyk_rgb", rgb), ("cmyk_plain", plain)] + list(resized.items()):
        d.enable_timing(True)
        steps[v]()
        torch.cuda.synchronize()
        split[v] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    statuses = {v: sum(d.status(i) != 0 for i in range(N)) for v, d in (("cmyk_rgb", rgb), ("mixed_resized", resized["mixed_resized"]))}
    for d in decs:
        d.close()
    torch.cuda.empty_cache()
    line = {"metric": "device ms per step (CUDA events): 1080p CMYK frames under mode=RGB vs without a mode; a 1080p YCbCr batch "
                      "resized to fp16 [N, 3, 224, 224] under mode=RGB with and without CMYK frames in it",
            "gpu": bench.gpu_facts(0), "frames": N, "size": "%dx%d" % (W, H), "cmyk_in_mixed": args.replace,
            "steps": args.steps, "rounds": args.rounds,
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in times},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in times},
            "entropy_recon_ms": split, "failed_frames": statuses}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
