"""Device time per step of BatchDecoder(reconstruction="libjpeg-turbo") (DESIGN §16) against the reference reconstruction, one GPU:

    python tools/turbo_bench.py [--workloads cfg3,cfg2] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3] [--out DIR]

Timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds; the best round is reported next to
all of them. Cases, each for reconstruction="reference" and "libjpeg-turbo" on the same frames:
  packed   decode() into the packed output
  fp16     decode_into an fp16 [N, 3, H, W] tensor with the ImageNet map
  rrc224   RandomResizedCrop rectangles (seeded), resized to fp16 [N, 3, 224, 224] with the ImageNet map
and, for the reference reconstruction only, packed / fp16 with every frame cropped to its whole output (`packed_whole`,
`fp16_whole`): the cost of the described, clipped store that every turbo frame takes (admit_crops), on upright packed and
planar destinations.
The entropy / reconstruction split comes from the batch's event timing in a step of its own. With --out, one packed turbo step
per workload runs again under torch.profiler (CUDA activities) for the times of turbo_idct_kernel, turbo_reconstruct_kernel and
turbo_generic_kernel (whichever run), and turbo_idct_kernel's chroma plane bytes over its time. Prints one JSON line with the card's name and power limit, read in the same run.
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
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

T = 224
RECONS = ("reference", "libjpeg-turbo")


def _timed(step, args, stream):
    import torch
    for _ in range(args.warmup):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(args.steps):
        step()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / args.steps


def rrc_rects(frames, seed):
    """torchvision's RandomResizedCrop rectangle rule (scale 0.08..1, ratio 3/4..4/3, 10 tries, centre fallback), seeded"""
    from libjpeg_b200 import decoder
    rng = np.random.default_rng(seed)
    out = []
    for f in frames:
        h, w = decoder.output_size(f)
        for _ in range(10):
            area = h * w * rng.uniform(0.08, 1.0)
            ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
            cw, ch = int(round(np.sqrt(area * ar))), int(round(np.sqrt(area / ar)))
            if 0 < cw <= w and 0 < ch <= h:
                out.append((int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch))
                break
        else:
            s = min(h, w)
            out.append(((w - s) // 2, (h - s) // 2, s, s))
    return out


def plane_bytes(dec_frames):
    """the bytes turbo_idct_kernel writes for these uncropped three-component frames of the tiled path: 64 per chroma block"""
    from libjpeg_b200 import decoder
    total = 0
    for f in dec_frames:
        info = decoder.parse(f)
        total += sum(64 * info.blocks_w[c] * info.blocks_h[c] for c in range(1, info.ncomp))
    return total


def run_workload(libjpeg_b200, workload, args):
    import torch
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    rects = rrc_rects(frames, 11)
    decs = {}
    for r in RECONS:
        decs["packed", r] = libjpeg_b200.BatchDecoder(frames, reconstruction=r)
        decs["fp16", r] = libjpeg_b200.BatchDecoder(frames, reconstruction=r)
        decs["rrc224", r] = libjpeg_b200.BatchDecoder(frames, reconstruction=r, crop=rects, resize=(T, T))
    whole = [(0, 0, w, h) for h, w in (libjpeg_b200.decoder.output_size(f) for f in frames)]
    decs["packed_whole", "reference"] = libjpeg_b200.BatchDecoder(frames, crop=whole)
    decs["fp16_whole", "reference"] = libjpeg_b200.BatchDecoder(frames, crop=whole)
    for d in decs.values():
        d.upload(stream)
    torch.cuda.synchronize()
    H, W = decs["fp16", "reference"].output_shape(0, 0)
    packed = {r: decs["packed", r].new_output() for r in RECONS}
    packed_whole = decs["packed_whole", "reference"].new_output()
    full = torch.empty(N, 3, H, W, dtype=torch.float16, device="cuda")
    small = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
    steps = {}
    for r in RECONS:
        steps["packed", r] = (lambda r=r: decs["packed", r].decode(packed[r], stream))
        steps["fp16", r] = (lambda r=r: decs["fp16", r].decode_into(full, stream, scale=SCALE, bias=BIAS))
        steps["rrc224", r] = (lambda r=r: decs["rrc224", r].decode_into(small, stream, scale=SCALE, bias=BIAS))
    steps["packed_whole", "reference"] = lambda: decs["packed_whole", "reference"].decode(packed_whole, stream)
    steps["fp16_whole", "reference"] = lambda: decs["fp16_whole", "reference"].decode_into(full, stream, scale=SCALE, bias=BIAS)
    times = {k: [] for k in steps}
    for rnd in range(args.rounds):
        for k in (list(steps) if rnd % 2 == 0 else list(steps)[::-1]):
            times[k].append(_timed(steps[k], args, stream))
    split = {}
    for k in (("packed", "reference"), ("packed", "libjpeg-turbo")):
        d = decs[k]
        d.enable_timing(True)
        steps[k]()
        torch.cuda.synchronize()
        split[k[1]] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    res = {"frames": N, "size": "%dx%d" % (W, H),
           "ms_per_step": {"%s/%s" % k: [round(t, 3) for t in times[k]] for k in times},
           "ms_per_step_best": {"%s/%s" % k: round(min(times[k]), 3) for k in times},
           "entropy_recon_ms_packed": split}
    if args.out:
        from torch.profiler import ProfilerActivity, profile
        step = steps["packed", "libjpeg-turbo"]
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
        kt = {}
        for ev in prof.key_averages():
            for name in ("turbo_idct_kernel", "turbo_reconstruct_kernel", "turbo_generic_kernel"):
                if name in ev.key:
                    kt[name] = round(ev.device_time_total / 1000.0 / args.steps, 3)
        os.makedirs(args.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.out, "turbo_%s.pt.trace.json" % workload))
        res["turbo_kernel_ms"] = kt
        if kt.get("turbo_idct_kernel"):
            res["idct_plane_GBps"] = round(plane_bytes(frames) / (kt["turbo_idct_kernel"] * 1e-3) / 1e9, 1)
    for d in decs.values():
        d.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (kernel times are measured only with it)")
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "turbo_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): reconstruction=reference vs libjpeg-turbo, packed / fp16 [N, 3, H, W] / "
                      "RandomResizedCrop -> fp16 [N, 3, 224, 224], ImageNet map", "gpu": bench.gpu_facts(0), "steps": args.steps,
            "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
