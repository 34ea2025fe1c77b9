"""Device time per step of decode() against BatchDecoder.decode_into on the benchmark's batches, one GPU:

    python tools/layout_bench.py [--workloads cfg3,cfg2] [--steps 10] [--warmup 2] [--rounds 3]

Four variants per workload, timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds:
  decode         decode() into the packed interleaved slots
  into_nchw      decode_into a [N, 3, H, W] tensor (the planar store kind)
  into_rgbx      decode_into an [N, H, W, 4] tensor, X untouched (the strided store kind)
  decode_permute decode() then out.view(N, H, W, 3).permute(0, 3, 1, 2).contiguous() (as a copy_ into a preallocated tensor):
                 what a model that takes NCHW needed so far
Every variant's pixels are reduced to the same per-chunk digest in NCHW order, and the digests must agree. Prints one JSON line
with the card's name and power limit, read in the same run. Each variant allocates its own destination and frees it again:
a cfg3 batch (750 4K frames) needs 18.7 GB per copy of its pixels.
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

VARIANTS = ["decode", "into_nchw", "into_rgbx", "decode_permute"]
# frames per batch: bench.py's for cfg3; half of it for cfg2, whose 4096-frame batch leaves no room on an 80 GB card for the two
# copies of its pixels (25.5 GB each) that decode_permute holds next to the batch's own buffers
FRAMES = {"cfg3": 750, "cfg2": 2048}


def digest(nchw_chunk, chunk_frames, n):
    """per chunk of frames: a weighted int64 sum of the chunk's bytes in NCHW order (wrapping, so exact and order-free)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(1)
    weights, sums = None, []
    for a in range(0, n, chunk_frames):
        words = nchw_chunk(a, min(n, a + chunk_frames)).contiguous().view(-1).view(torch.int32)
        if weights is None or weights.numel() < words.numel():
            weights = torch.randint(1, 1 << 20, (words.numel(),), device="cuda", dtype=torch.int64, generator=g)
        sums.append(int((words.to(torch.int64) * weights[:words.numel()]).sum()))
    return sums


def run_workload(libjpeg_b200, workload, args):
    import torch
    nf = FRAMES.get(workload, bench.DEFAULT_FRAMES[workload])
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [base[i % len(base)] for i in range(nf)]
    dec = libjpeg_b200.BatchDecoder(frames)
    fi = dec.info(0)
    N, H, W = nf, fi.height, fi.width
    fb = H * W * 3
    assert all(dec.out_offset(i) == i * fb for i in range(N)), "the packed slots of this batch are not back to back"
    stream = torch.cuda.Stream()
    dec.upload(stream)
    torch.cuda.synchronize()

    def setup(v):
        """-> (one step, NCHW view of frames [a, b) of the last step's result, the tensors to free)"""
        if v == "decode":
            out = dec.new_output()
            return (lambda: dec.decode(out, stream)), (lambda a, b: out[:N * fb].view(N, H, W, 3)[a:b].permute(0, 3, 1, 2)), [out]
        if v == "into_nchw":
            t = torch.empty(N, 3, H, W, dtype=torch.uint8, device="cuda")
            return (lambda: dec.decode_into(t, stream)), (lambda a, b: t[a:b]), [t]
        if v == "into_rgbx":
            t = torch.empty(N, H, W, 4, dtype=torch.uint8, device="cuda")
            dst = t.permute(0, 3, 1, 2)[:, :3]
            return (lambda: dec.decode_into(dst, stream)), (lambda a, b: t[a:b, :, :, :3].permute(0, 3, 1, 2)), [t]
        out = dec.new_output()
        t = torch.empty(N, 3, H, W, dtype=torch.uint8, device="cuda")

        def step():  # permute(0, 3, 1, 2).contiguous() into a tensor of its own, without a new allocation per step
            dec.decode(out, stream)
            with torch.cuda.stream(stream):
                t.copy_(out[:N * fb].view(N, H, W, 3).permute(0, 3, 1, 2))
        return step, (lambda a, b: t[a:b]), [out, t]

    times = {v: [] for v in VARIANTS}
    digests = {}
    for rnd in range(args.rounds):
        for v in (VARIANTS if rnd % 2 == 0 else VARIANTS[::-1]):
            step, view, keep = setup(v)
            for _ in range(args.warmup):
                step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                step()
            e1.record(stream)
            e1.synchronize()
            times[v].append(e0.elapsed_time(e1) / args.steps)
            if v not in digests:
                digests[v] = digest(view, 16, N)
            del step, view, keep
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    dec.close()
    same = all(digests[v] == digests["decode"] for v in VARIANTS)
    return {"frames": N, "size": "%dx%d" % (W, H), "same_pixels": same,
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in VARIANTS},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in VARIANTS}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=64)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "layout_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events), decode() vs decode_into", "gpu": bench.gpu_facts(0),
            "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))
    if not all(line[w]["same_pixels"] for w in args.workloads.split(",")):
        sys.exit("the variants decoded different pixels")


if __name__ == "__main__":
    main()
