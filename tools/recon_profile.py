"""Per-kernel device time of the decode path under torch.profiler (CUDA activities), on one GPU:

    python tools/recon_profile.py [--workload cfg3] [--frames 750] [--steps 5] [--out DIR]

Decodes the workload's batch (bench.py's frames: `--distinct` distinct codestreams tiled over the batch) a few times to warm
up, then profiles `--steps` decodes and prints, per kernel, the device time per step and the launches per step. With --out
the table is also written to DIR/recon_profile.json. B200JPG_LIB selects a variant build of the library. Tracing slows the
host, so end-to-end rates come from bench.py, not from here.
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3", choices=sorted(bench_inputs.WORKLOADS))
    ap.add_argument("--frames", type=int, default=750)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import libjpeg_b200
    assert torch.cuda.is_available(), "recon_profile.py needs a CUDA device"
    torch.cuda.set_device(0)
    base = bench_inputs.make_frames(args.workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [base[i % len(base)] for i in range(args.frames)]
    dec = libjpeg_b200.BatchDecoder(frames)
    out = dec.new_output()
    dec.upload()
    for _ in range(args.warmup):
        dec.decode(out)
    torch.cuda.synchronize()
    assert all(dec.status(i) == 0 for i in range(args.frames)), "decode reported errors"

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            dec.decode(out)
        torch.cuda.synchronize()

    per = collections.defaultdict(lambda: [0.0, 0])  # kernel -> [device us, launches]
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.replace("(anonymous namespace)::", "").replace("b200jpg::", "").split("(")[0]
        if name.startswith("void "):
            name = name[5:]
        per[name][0] += ev.time_range.elapsed_us()
        per[name][1] += 1
    rows = sorted(((k, v[0] / 1e3 / args.steps, v[1] / args.steps) for k, v in per.items()), key=lambda r: -r[1])
    gpu = bench.gpu_facts(0)
    print("%s, %s W; %s, %d frames, %d profiled steps; library %s" % (gpu["name"], gpu["power_limit_w"], args.workload, args.frames,
                                                                     args.steps, libjpeg_b200.library_path()))
    print("%10s %9s  %s" % ("ms/step", "launches", "kernel"))
    for name, ms, n in rows:
        print("%10.3f %9.1f  %s" % (ms, n, name))
    print("%10.3f %9s  total" % (sum(r[1] for r in rows), ""))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "recon_profile.json"), "w") as f:
            json.dump({"gpu": gpu, "workload": args.workload, "frames": args.frames, "steps": args.steps,
                       "library": libjpeg_b200.library_path(),
                       "kernels": [{"name": k, "ms_per_step": ms, "launches_per_step": n} for k, ms, n in rows]}, f, indent=1)


if __name__ == "__main__":
    main()
