"""Device time per step of OpenCV's resize in the batch (DESIGN §20) against Pillow's bilinear at the same sizes, 4:2:0 frames on
the libjpeg-turbo path, one GPU:

    python tools/cv_resize_bench.py [--workloads cfg2,cfg3] [--frames 128] [--steps 5] [--warmup 1] [--rounds 3]

Per workload and filter (cv2-linear, cv2-area, Pillow's bilinear), timed with CUDA events around `--steps` back-to-back steps in
`--rounds` alternating rounds (best and all rounds):
  letterbox  ultralytics' sizes (long side 640, ceil(w r)) into an fp16 [N, 3, 640, 640] tensor pre-filled with 114 / 255, each
             frame described at its centred offset in BGR order, map x / 255
  sq224      224 x 224 into an fp16 [N, 3, 224, 224] tensor with the ImageNet map
Then, in a separate run under torch.profiler, the summed device time per step of the resize stage's kernels (reduce_kernel,
resample_*, cv_*) for each case. Prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import math
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

FILTERS = ["cv2-linear", "cv2-area", "bilinear"]
RESIZE_KERNELS = ("reduce_kernel", "resample_h_kernel", "resample_v", "cv_resample", "cv_area_block")


def _time(step, stream, args):
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


def _resize_kernel_ms(step, stream, steps):
    """device ms per step of the resize stage's kernels under torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    total = {}
    for e in prof.key_averages():
        if any(k in e.key for k in RESIZE_KERNELS):
            m = re.search(r"(\w+_kernel(<[^>]*>)?)", e.key)
            name = m.group(1) if m else e.key
            dev = getattr(e, "device_time_total", None)
            if dev is None:
                dev = e.cuda_time_total
            total[name] = total.get(name, 0.0) + dev / 1000.0 / steps
    return {k: round(v, 3) for k, v in sorted(total.items())}


def run_workload(libjpeg_b200, workload, args):
    import torch
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    kw = dict(mode="RGB", reconstruction="libjpeg-turbo")
    probe = libjpeg_b200.BatchDecoder(frames[:1], **kw)
    h, w = probe.geometry()[0][0][0]
    probe.close()
    r = 640 / max(w, h)
    lb = (min(math.ceil(h * r), 640), min(math.ceil(w * r), 640))
    y0, x0 = (640 - lb[0]) // 2, (640 - lb[1]) // 2
    fill = 114 / 255
    dst_lb = torch.full((N, 3, 640, 640), fill, dtype=torch.float16, device="cuda")
    dst_sq = torch.empty(N, 3, 224, 224, dtype=torch.float16, device="cuda")
    planes_lb = [[dst_lb[i, 2 - c, y0:y0 + lb[0], x0:x0 + lb[1]] for c in range(3)] for i in range(N)]
    steps, decs = {}, []
    for f in FILTERS:
        d_lb = libjpeg_b200.BatchDecoder(frames, resize=lb, resample=f, **kw)
        d_sq = libjpeg_b200.BatchDecoder(frames, resize=(224, 224), resample=f, **kw)
        for d in (d_lb, d_sq):
            d.upload(stream)
            decs.append(d)
        steps["letterbox_" + f] = (lambda d=d_lb: d.decode_into(planes_lb, stream, scale=1 / 255))
        steps["sq224_" + f] = (lambda d=d_sq: d.decode_into(dst_sq, stream, scale=SCALE, bias=BIAS))
    torch.cuda.synchronize()
    names = list(steps)
    times = {v: [] for v in names}
    for rnd in range(args.rounds):
        for v in (names if rnd % 2 == 0 else names[::-1]):
            times[v].append(_time(steps[v], stream, args))
    try:
        kernels = {v: _resize_kernel_ms(steps[v], stream, args.steps) for v in names}
    except Exception as e:  # the profiler is optional: say so instead of a number
        kernels = "not measured (%s)" % type(e).__name__
    for d in decs:
        d.close()
    torch.cuda.empty_cache()
    return {"frames": N, "frame_size": [w, h], "letterbox_size_wh": [lb[1], lb[0]],
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in names},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in names},
            "resize_kernels_ms_per_step (torch.profiler, separate run)": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "cv_resize_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): cv2.resize (INTER_LINEAR, INTER_AREA) and Pillow's bilinear, letterbox 640 "
                      "and 224 x 224, fp16", "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for wl in args.workloads.split(","):
        line[wl] = run_workload(libjpeg_b200, wl, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
