"""Times spec_sync_kernel and the whole decode of restart-less frames, for one or more builds of libb200jpg.so.

    python tools/spec_sync_bench.py --tree new=. --tree parent=/path/to/a/checkout/of/the/parent

Workloads: 1080p and 4K frames with every component on Huffman table 0 (synth SHARED_TABLES), one frame and a batch, and the
benchmark's cfg2n / cfg3n frames, all written once by this tree. Each build (a built source tree) runs in its own process,
the builds alternate, three rounds; the best round per build is reported. Decode time: CUDA events around decode(); spec_sync_kernel time: the CUDA time of its
launches in a torch.profiler trace of one decode. Prints one JSON line per build and workload, with the card and its power
limit."""
import argparse
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = {  # name: (kind, width, height, frames)
    "shared1080x1": ("shared", 1920, 1080, 1), "shared4kx1": ("shared", 3840, 2160, 1),
    "shared1080x64": ("shared", 1920, 1080, 64), "shared4kx16": ("shared", 3840, 2160, 16),
    "cfg2n": ("bench", 0, 0, 256), "cfg3n": ("bench", 0, 0, 64),
}


def frames_for(name):
    from libjpeg_b200 import synth
    from tools import bench_inputs
    kind, w, h, n = WORKLOADS[name]
    if kind == "shared":
        distinct = [synth.encode(synth.source_image(w, h, s), 75, (2, 2), 0, synth.SHARED_TABLES).tobytes() for s in range(1, 5)]
    else:
        distinct = bench_inputs.make_frames(name, 4, workers=4)
    return [distinct[i % len(distinct)] for i in range(n)]


def child(tree, frames_dir, names, steps):
    import pickle

    import torch
    from torch.profiler import ProfilerActivity, profile
    sys.path.insert(0, tree)
    import libjpeg_b200 as lj
    out = {}
    for name in names:
        with open(os.path.join(frames_dir, name + ".pkl"), "rb") as f:
            dec = lj.BatchDecoder(pickle.load(f))
        buf = dec.new_output()
        dec.upload()
        for _ in range(3):
            dec.decode(buf)
        torch.cuda.synchronize()
        times = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dec.decode(buf)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            dec.decode(buf)
            torch.cuda.synchronize()
        sync_us = sum(e.device_time_total for e in prof.key_averages() if "spec_sync_kernel" in e.key)
        out[name] = {"decode_ms": min(times), "spec_sync_ms": sync_us / 1000.0}
    print(json.dumps(out))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", default=[], help="label=built source tree (repeatable)")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--child", nargs=2, metavar=("TREE", "FRAMES_DIR"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    names = args.workloads.split(",")
    if args.child:
        child(args.child[0], args.child[1], names, args.steps)
        return
    import pickle
    import tempfile
    sys.path.insert(0, ROOT)
    trees = [tuple(s.split("=", 1)) for s in args.tree] or [("tree", ROOT)]
    frames_dir = tempfile.mkdtemp(prefix="spec_sync_bench_")
    for name in names:
        with open(os.path.join(frames_dir, name + ".pkl"), "wb") as f:
            pickle.dump(frames_for(name), f)
    best = {}
    for _ in range(args.rounds):
        for label, tree in trees:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", os.path.abspath(tree), frames_dir, "--workloads", args.workloads,
                                "--steps", str(args.steps)], capture_output=True, text=True, cwd=os.path.abspath(tree))
            if r.returncode:
                sys.stderr.write(r.stderr)
                raise SystemExit("%s failed" % label)
            for name, v in json.loads(r.stdout.strip().splitlines()[-1]).items():
                b = best.setdefault((label, name), dict(v))
                for k in v:  # (a profile that caught no launch of the kernel reports 0: not a measurement)
                    b[k] = min(x for x in (b[k], v[k], float("inf")) if x > 0) if b[k] > 0 or v[k] > 0 else 0.0
    shutil.rmtree(frames_dir)
    gpu = card()
    for (label, name), v in sorted(best.items(), key=lambda kv: (kv[0][1], kv[0][0])):
        print(json.dumps({"build": label, "workload": name, "frames": WORKLOADS[name][3], "gpu": gpu, **{k: round(x, 3) for k, x in v.items()}}))


if __name__ == "__main__":
    main()
