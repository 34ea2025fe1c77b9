"""Device time per step of cropped decoding (BatchDecoder(crop=...)) against what a user does without it, one GPU:

    python tools/crop_bench.py [--workloads cfg3,cfg2] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3]

Output: fp16 [N, 3, h, w] with the ImageNet map. Rectangles, seeded per frame: a centered 224 x 224 (c224), a 512 x 512 at a
random origin (r512), half the area at a random origin (half), the full frame (full), and a 224 x 224 at downscale 2 (c224_k2).
Per rectangle, timed with CUDA events around `--steps` back-to-back steps in `--rounds` alternating rounds:
  crop_<r>    decode_into of the cropped batch
  slice_<r>   decode_into of the uncropped batch into a full-size tensor, then a per-frame slice copy into a preallocated one
The two must write the same bytes ("agree"). The stage split (entropy / reconstruction ms) of every crop_<r> comes from the batch's
event timing in a separate step. Prints one JSON line with the card's name and power limit, read in the same run.
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
from tools import bench_inputs  # noqa: E402
from tools.orientation_bench import BIAS, SCALE, _digest  # noqa: E402

RECTS = ("c224", "r512", "half", "full", "c224_k2")


def rectangles(name, H, W, n, seed):
    """(x, y, width, height) per frame of an H x W output"""
    rng = np.random.default_rng(seed)
    if name in ("c224", "c224_k2"):
        return [((W - 224) // 2, (H - 224) // 2, 224, 224)] * n
    if name == "full":
        return [(0, 0, W, H)] * n
    w, h = (512, 512) if name == "r512" else (int(W / 2 ** 0.5), int(H / 2 ** 0.5))
    return [(int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h) for _ in range(n)]


def run_workload(libjpeg_b200, workload, args):
    import torch
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    plain = {k: libjpeg_b200.BatchDecoder(frames, downscale=k) for k in (1, 2)}
    rects, crops = {}, {}
    for r in RECTS:
        k = 2 if r.endswith("_k2") else 1
        H, W = plain[k].output_shape(0, 0)
        rects[r] = rectangles(r, H, W, N, seed=7)
        crops[r] = libjpeg_b200.BatchDecoder(frames, downscale=k, crop=rects[r])
    for d in list(plain.values()) + list(crops.values()):
        d.upload(stream)
    torch.cuda.synchronize()

    def setup(v):
        kind, r = v.split("_", 1)
        h, w = rects[r][0][3], rects[r][0][2]
        dst = torch.empty(N, 3, h, w, dtype=torch.float16, device="cuda")
        if kind == "crop":
            return (lambda: crops[r].decode_into(dst, stream, scale=SCALE, bias=BIAS)), dst
        dec = plain[2 if r.endswith("_k2") else 1]
        H, W = dec.output_shape(0, 0)
        full = torch.empty(N, 3, H, W, dtype=torch.float16, device="cuda")

        def step():
            dec.decode_into(full, stream, scale=SCALE, bias=BIAS)
            with torch.cuda.stream(stream):
                for i, (x, y, rw, rh) in enumerate(rects[r]):
                    dst[i].copy_(full[i, :, y:y + rh, x:x + rw])
        return step, dst

    variants = ["crop_" + r for r in RECTS] + ["slice_" + r for r in RECTS]
    times = {v: [] for v in variants}
    digests = {}
    for rnd in range(args.rounds):
        for v in (variants if rnd % 2 == 0 else variants[::-1]):
            step, keep = setup(v)
            for _ in range(args.warmup):
                step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                step()
            e1.record(stream)
            e1.synchronize()
            times[v].append(e0.elapsed_time(e1) / args.steps)
            if rnd == args.rounds - 1:
                torch.cuda.synchronize()
                digests[v] = _digest(keep[a] for a in range(N))
            del step, keep
            torch.cuda.empty_cache()
    split = {}
    for r in RECTS:  # the stage split, in a step of its own (the events sit on the stream)
        step, keep = setup("crop_" + r)
        crops[r].enable_timing(True)
        step()
        torch.cuda.synchronize()
        split[r] = [round(t, 3) for t in crops[r].last_timing()]
        crops[r].enable_timing(False)
        del step, keep
    agree = {r: digests["crop_" + r] == digests["slice_" + r] for r in RECTS}
    H, W = plain[1].output_shape(0, 0)
    for d in list(plain.values()) + list(crops.values()):
        d.close()
    torch.cuda.empty_cache()
    best = {v: round(min(times[v]), 3) for v in variants}
    return {"frames": N, "size": "%dx%d" % (W, H), "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in variants},
            "ms_per_step_best": best, "crop_entropy_recon_ms": split, "agree": agree}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "crop_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events), fp16 [N, 3, h, w]: cropped decode vs full decode then slice", "gpu": bench.gpu_facts(0),
            "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
