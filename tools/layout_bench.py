"""Device time per step of decode() against BatchDecoder.decode_into on the benchmark's batches, one GPU:

    python tools/layout_bench.py [--workloads cfg3,cfg2] [--steps 10] [--warmup 2] [--rounds 3]

Variants per workload, timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds:
  decode         decode() into the packed interleaved slots
  into_nchw      decode_into a [N, 3, H, W] tensor (the planar store kind)
  into_rgbx      decode_into an [N, H, W, 4] tensor, X untouched (the strided store kind)
  decode_permute decode() then out.view(N, H, W, 3).permute(0, 3, 1, 2).contiguous() (as a copy_ into a preallocated tensor):
                 what a model that takes NCHW needed before decode_into
  into_nchw_f16 / into_nchw_bf16 / into_nchw_f32
                 decode_into a float [N, 3, H, W] tensor with an ImageNet-style per-channel map (the planar float kind);
                 f32 at half the frames: a cfg3 batch in fp32 is 74.6 GB of output
  into_nhwc_f16  decode_into an fp16 [N, H, W, 3] tensor as t.permute(0, 3, 1, 2) (the strided float kind)
  into_nchw_then_torch_f16
                 decode_into a uint8 [N, 3, H, W] tensor, then (t.float() * scale + bias).half() into a preallocated fp16
                 tensor, `CONVERT_CHUNK` frames at a time so the fp32 temporaries stay small: what the float kinds replace
Every variant's output is reduced to the same per-chunk digest in NCHW order. The uint8 variants must agree with decode(); the
float variants with the uint8 result converted by PyTorch. Prints one JSON line with the card's name and power limit, read in
the same run, and the frame count of every variant. Each variant allocates its own destination and frees it again: a cfg3 batch
(750 4K frames) needs 18.7 GB per copy of its pixels in uint8.
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

VARIANTS = ["decode", "into_nchw", "into_rgbx", "decode_permute", "into_nchw_f16", "into_nchw_bf16", "into_nchw_f32", "into_nhwc_f16",
            "into_nchw_then_torch_f16"]
FLOAT = {"into_nchw_f16": "float16", "into_nchw_bf16": "bfloat16", "into_nchw_f32": "float32", "into_nhwc_f16": "float16",
         "into_nchw_then_torch_f16": "float16"}
HALF_FRAMES = {"into_nchw_f32"}
CONVERT_CHUNK = 8
# frames per digest chunk: its int64 temporaries have to fit next to the PyTorch baseline's uint8 and fp16 copies of a cfg3 batch
DIGEST_CHUNK = 4
# (x / 255 - mean) / std per channel
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SCALE, BIAS = [1 / (255 * s) for s in STD], [-m / s for m, s in zip(MEAN, STD)]
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
    scale = torch.tensor(SCALE, dtype=torch.float32, device="cuda").view(1, 3, 1, 1)
    bias = torch.tensor(BIAS, dtype=torch.float32, device="cuda").view(1, 3, 1, 1)

    def torch_convert(u8, dtype):
        return (u8.float() * scale + bias).to(dtype)  # two roundings: separate multiply and add kernels

    def frames_of(v):
        return N // 2 if v in HALF_FRAMES else N

    def setup(v):
        """-> (one step, NCHW view of frames [a, b) of the last step's result, the tensors to free)"""
        if v in FLOAT and v != "into_nchw_then_torch_f16":
            dtype, d, n = getattr(torch, FLOAT[v]), dec, frames_of(v)
            if v in HALF_FRAMES:  # a batch of its own, the first N / 2 frames of `dec`; freed with the variant's tensors
                d = libjpeg_b200.BatchDecoder(frames[:n])
                d.upload(stream)
            if v.startswith("into_nhwc"):
                t = torch.empty(n, H, W, 3, dtype=dtype, device="cuda")
                dst = t.permute(0, 3, 1, 2)
                return (lambda: d.decode_into(dst, stream, scale=SCALE, bias=BIAS)), (lambda a, b: dst[a:b]), [t]
            t = torch.empty(n, 3, H, W, dtype=dtype, device="cuda")
            return (lambda: d.decode_into(t, stream, scale=SCALE, bias=BIAS)), (lambda a, b: t[a:b]), [t] + ([d] if d is not dec else [])
        if v == "into_nchw_then_torch_f16":
            u8 = torch.empty(N, 3, H, W, dtype=torch.uint8, device="cuda")
            t = torch.empty(N, 3, H, W, dtype=torch.float16, device="cuda")

            def step():
                dec.decode_into(u8, stream)
                with torch.cuda.stream(stream):
                    for a in range(0, N, CONVERT_CHUNK):
                        t[a:a + CONVERT_CHUNK].copy_(torch_convert(u8[a:a + CONVERT_CHUNK], torch.float16))
            return step, (lambda a, b: t[a:b]), [u8, t]
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

    def close_batches(keep):  # a function of its own: no loop variable outlives it and pins a tensor
        for k in keep:
            if isinstance(k, libjpeg_b200.BatchDecoder):
                k.close()
                k.ctx.close()

    times = {v: [] for v in VARIANTS}
    digests, converted = {}, {}
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
            torch.cuda.empty_cache()  # the conversion temporaries of the PyTorch baseline: room for the digest's
            if v not in digests:
                digests[v] = digest(view, DIGEST_CHUNK, frames_of(v))
            if v == "into_nchw" and "float16" not in converted:  # what every float variant must equal, from the uint8 result
                for name in set(FLOAT.values()):
                    n = N // 2 if name == "float32" else N
                    converted[name] = digest(lambda a, b: torch_convert(view(a, b), getattr(torch, name)), DIGEST_CHUNK, n)
            torch.cuda.synchronize()
            close_batches(keep)
            del step, view, keep
            torch.cuda.empty_cache()
    dec.close()
    want = {v: converted[FLOAT[v]] if v in FLOAT else digests["decode"] for v in VARIANTS}
    same = {v: digests[v] == want[v] for v in VARIANTS}
    return {"frames": {v: frames_of(v) for v in VARIANTS}, "size": "%dx%d" % (W, H), "same_output": same,
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
    line = {"metric": "device ms per step (CUDA events), decode() vs decode_into (uint8 and float)", "gpu": bench.gpu_facts(0),
            "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))
    if not all(all(line[w]["same_output"].values()) for w in args.workloads.split(",")):
        sys.exit("the variants disagree with decode() or with its PyTorch conversion")


if __name__ == "__main__":
    main()
