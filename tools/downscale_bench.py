"""Device time per step of downscaled decoding (BatchDecoder(downscale=k)) against what a user does without it, one GPU:

    python tools/downscale_bench.py [--workloads cfg3,cfg2,cfg1] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3]

Per workload and k in 1, 2, 4, 8, timed with CUDA events around `--steps` back-to-back steps in `--rounds` alternating rounds:
  packed_k   decode() of a downscale=k batch into its packed slots
  f16_k      decode_into an fp16 [N, 3, H', W'] tensor with an ImageNet-style map
  pool_k     (k > 1) the full-size batch decode_into an fp16 [N, 3, H, W] tensor, then torch.nn.functional.avg_pool2d(k)
             into a preallocated [N, 3, H / k, W / k] tensor, `POOL_CHUNK` frames at a time (ceil_mode, so that odd sizes agree)
Prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SCALE, BIAS = [1 / (255 * s) for s in STD], [-m / s for m, s in zip(MEAN, STD)]
POOL_CHUNK = 16
KS = (1, 2, 4, 8)


def run_workload(libjpeg_b200, workload, args):
    import torch
    import torch.nn.functional as F
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [base[i % len(base)] for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    decs = {k: libjpeg_b200.BatchDecoder(frames, downscale=k) for k in KS}
    for d in decs.values():
        d.upload(stream)
    torch.cuda.synchronize()
    shapes = {k: decs[k].output_shape(0, 0) for k in KS}

    def setup(v):
        kind, k = v.split("_")
        k = int(k)
        d = decs[k]
        if kind == "packed":
            out = d.new_output()
            return (lambda: d.decode(out, stream)), [out]
        h, w = shapes[k]
        if kind == "f16":
            t = torch.empty(N, 3, h, w, dtype=torch.float16, device="cuda")
            return (lambda: d.decode_into(t, stream, scale=SCALE, bias=BIAS)), [t]
        H, W = shapes[1]
        full = torch.empty(N, 3, H, W, dtype=torch.float16, device="cuda")
        small = torch.empty(N, 3, h, w, dtype=torch.float16, device="cuda")

        def step():
            decs[1].decode_into(full, stream, scale=SCALE, bias=BIAS)
            with torch.cuda.stream(stream):
                for a in range(0, N, POOL_CHUNK):
                    small[a:a + POOL_CHUNK].copy_(F.avg_pool2d(full[a:a + POOL_CHUNK], k, ceil_mode=True))
        return step, [full, small]

    variants = ["packed_%d" % k for k in KS] + ["f16_%d" % k for k in KS] + ["pool_%d" % k for k in KS if k > 1]
    times = {v: [] for v in variants}
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
            del step, keep
            torch.cuda.empty_cache()
    for d in decs.values():
        d.close()
    best = {v: round(min(times[v]), 3) for v in variants}
    return {"frames": N, "size": "%dx%d" % (shapes[1][1], shapes[1][0]), "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in variants},
            "ms_per_step_best": best, "frames_per_s_best": {v: round(N / best[v] * 1000.0, 1) for v in variants}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2,cfg1")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "downscale_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events), downscaled decoding vs full size + avg_pool2d", "gpu": bench.gpu_facts(0),
            "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
