"""Device time per step of the flips (DESIGN §21) and the sample tables (DESIGN §22), one GPU:

    python tools/flip_table_bench.py [--workloads cfg2,cfg3] [--crop-frames 256] [--frames 32] [--steps 5] [--warmup 1] [--rounds 3]

Per workload, timed with CUDA events around `--steps` back-to-back steps in `--rounds` alternating rounds (best and all rounds):
  rrc       RandomResizedCrop(224) of `--crop-frames` frames (seeded rectangles of scale 0.08 .. 1 and ratio 3/4 .. 4/3, the
            libjpeg-turbo reconstruction, mode "RGB", bilinear) into an fp16 [N, 3, 224, 224] tensor with the ImageNet map: without
            flips, and with hflip on every other frame
  full      the whole frames of `--frames` frames (reference reconstruction: reconstruct420_kernel) into an fp16 and an fp32
            [N, 3, H, W] tensor: the affine ImageNet map against the sample table of ToTensor() + Normalize()
Prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402
from tools.cv_resize_bench import _time  # noqa: E402
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def _rrc_rects(w, h, n, rng):
    """torchvision's RandomResizedCrop.get_params (scale 0.08 .. 1, ratio 3/4 .. 4/3, ten tries, then the centre crop)"""
    out = []
    for _ in range(n):
        for _ in range(10):
            area = w * h * rng.uniform(0.08, 1.0)
            ar = math.exp(rng.uniform(math.log(3 / 4), math.log(4 / 3)))
            cw, ch = int(round(math.sqrt(area * ar))), int(round(math.sqrt(area / ar)))
            if 0 < cw <= w and 0 < ch <= h:
                out.append((int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch))
                break
        else:
            out.append((0, 0, w, h))
    return out


def _timed(steps, stream, args):
    names = list(steps)
    times = {v: [] for v in names}
    for rnd in range(args.rounds):
        for v in (names if rnd % 2 == 0 else names[::-1]):
            times[v].append(_time(steps[v], stream, args))
    return {"ms_per_step": {v: [round(t, 3) for t in times[v]] for v in names},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in names}}


def run_workload(libjpeg_b200, workload, args):
    import numpy as np
    import torch
    import torchvision.transforms.functional as TF
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    stream = torch.cuda.Stream()
    res = {}
    # RandomResizedCrop + RandomHorizontalFlip
    frames = [bytes(base[i % len(base)]) for i in range(args.crop_frames)]
    n = len(frames)
    kw = dict(mode="RGB", reconstruction="libjpeg-turbo", resize=(224, 224), resample="bilinear")
    probe = libjpeg_b200.BatchDecoder(frames[:1], mode="RGB")
    h, w = probe.geometry()[0][0][0]
    probe.close()
    rects = _rrc_rects(w, h, n, np.random.default_rng(1))
    dst = torch.empty(n, 3, 224, 224, dtype=torch.float16, device="cuda")
    plain = libjpeg_b200.BatchDecoder(frames, crop=rects, **kw)
    flipped = libjpeg_b200.BatchDecoder(frames, crop=rects, hflip=[i % 2 == 0 for i in range(n)], **kw)
    for d in (plain, flipped):
        d.upload(stream)
    torch.cuda.synchronize()
    res["rrc"] = {"frames": n, "frame_size": [w, h], **_timed({
        "no_flip": lambda: plain.decode_into(dst, stream, scale=SCALE, bias=BIAS),
        "hflip_half": lambda: flipped.decode_into(dst, stream, scale=SCALE, bias=BIAS)}, stream, args)}
    res["rrc"]["launches"] = {"no_flip": plain.launches, "hflip_half": flipped.launches}
    plain.close(), flipped.close()
    # whole frames: affine map against the table
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    n = len(frames)
    dec = libjpeg_b200.BatchDecoder(frames)
    dec.upload(stream)
    table = libjpeg_b200.sample_table(lambda t: TF.normalize(t.float().div(255), MEAN, STD))
    steps = {}
    for dt in (torch.float16, torch.float32):
        d = torch.empty(n, 3, h, w, dtype=dt, device="cuda")
        name = str(dt).split(".")[-1]
        steps[name + "_affine"] = (lambda d=d: dec.decode_into(d, stream, scale=SCALE, bias=BIAS))
        steps[name + "_table"] = (lambda d=d: dec.decode_into(d, stream, table=table))
    torch.cuda.synchronize()
    res["full"] = {"frames": n, "frame_size": [w, h], **_timed(steps, stream, args)}
    dec.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--crop-frames", type=int, default=256)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "flip_table_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): RandomResizedCrop 224 fp16 with and without hflip on half the frames; "
                      "whole frames into fp16 / fp32, affine map against sample table",
            "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for wl in args.workloads.split(","):
        line[wl] = run_workload(libjpeg_b200, wl, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
