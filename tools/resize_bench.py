"""Device time per step of a training loader's RandomResizedCrop done by the batch (BatchDecoder(crop=..., resize=...)) against what
a loader does without it, one GPU:

    python tools/resize_bench.py [--workloads cfg3,cfg2] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3] [--profile-dir DIR]

Rectangles: torchvision's RandomResizedCrop sampling (scale 0.08 - 1, ratio 3/4 - 4/3), seeded per frame; every frame resized to
224 x 224; fp16 [N, 3, 224, 224] output with the ImageNet map. Per filter (bilinear, bicubic), timed with CUDA events around
`--steps` back-to-back steps in `--rounds` alternating rounds:
  fused_<f>    decode_into of BatchDecoder(crop=rects, resize=(224, 224), resample=f)
  interp_<f>   decode_into of BatchDecoder(crop=rects) into per-frame fp32 [3, h, w] tensors, then per frame
               F.interpolate(antialias=True), the map and .half() into the batch tensor
The two are not bit-equal (F.interpolate works on floats): the maximum absolute difference is reported. Also: the stage split
(entropy / reconstruction ms, the resample launches included in the second) of every fused_<f> from the batch's event timing in a
step of its own; the two resample kernels' device time per step from a torch.profiler run of its own; the bytes and
multiply-adds of the resample pass computed from the shapes, over that time. Prints one JSON line with the card's name and power
limit, read in the same run.
"""
import argparse
import ctypes
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

FILTERS = ("bilinear", "bicubic")
T = 224


def random_resized_crops(H, W, n, seed, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3)):
    """(x, y, width, height) per frame of an H x W output, drawn like torchvision's RandomResizedCrop.get_params"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        for _ in range(10):
            area = H * W * rng.uniform(*scale)
            ar = math.exp(rng.uniform(math.log(ratio[0]), math.log(ratio[1])))
            w, h = int(round(math.sqrt(area * ar))), int(round(math.sqrt(area / ar)))
            if 0 < w <= W and 0 < h <= H:
                out.append((int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h))
                break
        else:
            w, h = W, H
            out.append(((W - w) // 2, (H - h) // 2, w, h))
    return out


def _tables(lib, in_size, out_size, f):
    ks = ctypes.c_uint32()
    lib.b200jpg_resample_coefficients(in_size, out_size, f, None, None, 0, ctypes.byref(ks))
    b = np.zeros(2 * out_size, dtype=np.int32)
    t = np.zeros(out_size * ks.value, dtype=np.int32)
    assert lib.b200jpg_resample_coefficients(in_size, out_size, f, b.ctypes.data, t.ctypes.data, t.size, ctypes.byref(ks)) == 0
    return b.reshape(out_size, 2)


def resample_work(lib, rects, f, ncomp=3, out_bytes=2):
    """bytes the two resample kernels must move (C read, intermediate written and read, destination written) and the
    multiply-adds they do, from the shapes and the tables (DESIGN §13)"""
    nbytes = macs = 0
    for _, _, w, h in rects:
        vb = _tables(lib, h, T, f) if h != T else None
        y0, y1 = (int(vb[0, 0]), int(vb[-1, 0] + vb[-1, 1])) if vb is not None else (0, h)
        if w != T:
            hb = _tables(lib, w, T, f)
            nbytes += (y1 - y0) * w * ncomp + 2 * (y1 - y0) * T * ncomp
            macs += (y1 - y0) * ncomp * int(hb[:, 1].sum())
        else:
            nbytes += h * w * ncomp
        if vb is not None:
            macs += T * ncomp * int(vb[:, 1].sum())
        nbytes += T * T * ncomp * out_bytes
    return nbytes, macs


def run_workload(libjpeg_b200, workload, args):
    import torch
    import torch.nn.functional as F
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    probe = libjpeg_b200.BatchDecoder(frames[:1])
    H, W = probe.output_shape(0, 0)
    probe.close()
    rects = random_resized_crops(H, W, N, seed=11)
    fused = {f: libjpeg_b200.BatchDecoder(frames, crop=rects, resize=(T, T), resample=f) for f in FILTERS}
    crop = libjpeg_b200.BatchDecoder(frames, crop=rects)
    for d in list(fused.values()) + [crop]:
        d.upload(stream)
    torch.cuda.synchronize()
    scale_t = torch.tensor(SCALE, device="cuda").view(3, 1, 1)
    bias_t = torch.tensor(BIAS, device="cuda").view(3, 1, 1)

    def setup(v):
        kind, f = v.split("_", 1)
        dst = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
        if kind == "fused":
            return (lambda: fused[f].decode_into(dst, stream, scale=SCALE, bias=BIAS)), dst
        per = [torch.empty(3, h, w, dtype=torch.float32, device="cuda") for _, _, w, h in rects]
        planes = [[t[0], t[1], t[2]] for t in per]

        def step():
            crop.decode_into(planes, stream)
            with torch.cuda.stream(stream):
                for i, t in enumerate(per):
                    y = F.interpolate(t[None], size=(T, T), mode=f, antialias=True, align_corners=False)[0]
                    dst[i].copy_((y * scale_t + bias_t).half())
        return step, dst

    variants = ["fused_" + f for f in FILTERS] + ["interp_" + f for f in FILTERS]
    times = {v: [] for v in variants}
    outs = {}
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
                outs[v] = keep.float().cpu()
            del step, keep
            torch.cuda.empty_cache()
    split, kernel_ms, work = {}, {}, {}
    lib = libjpeg_b200.native.lib
    for f in FILTERS:  # the stage split, in a step of its own (the events sit on the stream)
        step, keep = setup("fused_" + f)
        fused[f].enable_timing(True)
        step()
        torch.cuda.synchronize()
        split[f] = [round(t, 3) for t in fused[f].last_timing()]
        fused[f].enable_timing(False)
        # the resample kernels' own device time, from a profiler run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
        if args.profile_dir:
            os.makedirs(args.profile_dir, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.profile_dir, "resize_%s_%s.pt.trace.json" % (workload, f)))
        per = {"resample_h_kernel": 0.0, "resample_v_kernel": 0.0}
        for e in prof.key_averages():
            for k in per:
                if k in e.key:
                    per[k] += e.device_time_total / 1000.0 / args.steps
        kernel_ms[f] = {k: round(t, 4) for k, t in per.items()}
        nbytes, macs = resample_work(lib, rects, libjpeg_b200.native.RESAMPLE[f])
        ms = sum(per.values())
        work[f] = {"bytes": nbytes, "macs": macs, "GB_per_s": round(nbytes / ms / 1e6, 1) if ms else None,
                   "GMAC_per_s": round(macs / ms / 1e6, 1) if ms else None}
        del step, keep
    maxdiff = {f: float((outs["fused_" + f] - outs["interp_" + f]).abs().max()) for f in FILTERS}
    for d in list(fused.values()) + [crop]:
        d.close()
    torch.cuda.empty_cache()
    areas = [w * h for _, _, w, h in rects]
    best = {v: round(min(times[v]), 3) for v in variants}
    return {"frames": N, "size": "%dx%d" % (W, H), "crop_pixels_mean": int(np.mean(areas)),
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in variants}, "ms_per_step_best": best,
            "fused_entropy_recon_ms": split, "resample_kernel_ms_per_step": kernel_ms, "resample_work": work,
            "max_abs_diff_fused_vs_interp": maxdiff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--profile-dir", default="", help="where the profiler runs' traces go (default: not written)")
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "resize_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events), RandomResizedCrop to fp16 [N, 3, 224, 224]: fused resize vs crop then "
                      "F.interpolate", "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
