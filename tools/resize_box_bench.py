"""Device time per step of the chains DESIGN §19 adds, on 4:2:0 frames, one GPU:

    python tools/resize_box_bench.py [--workloads cfg2,cfg3] [--frames 128] [--steps 5] [--warmup 1] [--rounds 3]

Per workload, timed with CUDA events around `--steps` back-to-back steps in `--rounds` alternating rounds (best and all rounds):
  eval_fused      Resize(256) + CenterCrop(224) as one batch with windows (resize_center_crop_args), decode_into an fp16
                  [N, 3, 224, 224] tensor with the ImageNet map, on the libjpeg-turbo path
  eval_sliced     the same resize without windows into packed uint8 output, then each frame's 224 x 224 centre sliced, mapped
                  and converted to fp16 into the same tensor by PyTorch
  thumb<S>_chain  thumbnail((S, S)) as Pillow does it: draft, fractional box and reduce() (thumbnail_args, reducing_gap=2.0)
  thumb<S>_plain  the drafted resize alone: the same draft and size, no box and no gap
Also the stage split (entropy, reconstruction + resample ms, the batch's event timing in a step of its own) of eval_fused, whose
reconstruction covers only the columns and rows the windows read, against eval_sliced, which reconstructs all of C. eval_fused
and eval_sliced are checked bit-equal. Prints one JSON line with the card's name and
power limit, read in the same run.
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
from tools.orientation_bench import BIAS, SCALE  # noqa: E402

T = 224


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


def run_workload(libjpeg_b200, workload, args):
    import torch
    from libjpeg_b200.decoder import resize_center_crop_args, thumbnail_args
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    kw = dict(mode="RGB", reconstruction="libjpeg-turbo")
    ev = [resize_center_crop_args(f, 256, T) for f in frames]
    rs = [a["resize"] for a in ev]
    decs = {"eval_fused": libjpeg_b200.BatchDecoder(frames, resize=rs, window=[a["window"] for a in ev], **kw),
            "eval_sliced": libjpeg_b200.BatchDecoder(frames, resize=rs, **kw)}
    for s in (128, 64):
        th = [thumbnail_args(f, (s, s)) for f in frames]
        draft, size = [a["draft"] for a in th], [a["resize"] for a in th]
        decs["thumb%d_chain" % s] = libjpeg_b200.BatchDecoder(frames, draft=draft, resize=size, box=[a["box"] for a in th],
                                                              reducing_gap=2.0, resample="bicubic", **kw)
        decs["thumb%d_plain" % s] = libjpeg_b200.BatchDecoder(frames, draft=draft, resize=size, resample="bicubic", **kw)
    for d in decs.values():
        d.upload(stream)
    torch.cuda.synchronize()
    scale_t = torch.tensor(SCALE, device="cuda").view(3, 1, 1)
    bias_t = torch.tensor(BIAS, device="cuda").view(3, 1, 1)
    dst = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
    packed = decs["eval_sliced"].new_output()
    outs = {s: decs["thumb%d_chain" % s].new_output() for s in (128, 64)}
    outs.update({"p%d" % s: decs["thumb%d_plain" % s].new_output() for s in (128, 64)})

    def sliced():
        d = decs["eval_sliced"]
        d.decode(packed, stream)
        with torch.cuda.stream(stream):
            for i, a in enumerate(ev):
                x, y, w, h = a["window"]
                v = d.frame_view(packed, i)[y:y + h, x:x + w].permute(2, 0, 1)
                dst[i].copy_((v.float() * scale_t + bias_t).half())

    steps = {"eval_fused": lambda: decs["eval_fused"].decode_into(dst, stream, scale=SCALE, bias=BIAS), "eval_sliced": sliced}
    for s in (128, 64):
        steps["thumb%d_chain" % s] = (lambda s=s: decs["thumb%d_chain" % s].decode(outs[s], stream))
        steps["thumb%d_plain" % s] = (lambda s=s: decs["thumb%d_plain" % s].decode(outs["p%d" % s], stream))
    names = list(steps)
    times = {v: [] for v in names}
    for rnd in range(args.rounds):
        for v in (names if rnd % 2 == 0 else names[::-1]):
            times[v].append(_time(steps[v], stream, args))
    steps["eval_fused"]()
    torch.cuda.synchronize()
    fused = dst.clone()
    sliced()
    torch.cuda.synchronize()
    equal = bool(torch.equal(fused.view(torch.int16), dst.view(torch.int16)))
    split = {}
    for v in ("eval_fused", "eval_sliced"):
        d = decs[v]
        d.enable_timing(True)
        steps[v]()
        torch.cuda.synchronize()
        split[v] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    for d in decs.values():
        d.close()
    torch.cuda.empty_cache()
    return {"frames": N, "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in names},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in names},
            "entropy_recon_ms (trimmed: eval_fused, whole C: eval_sliced)": split, "eval_fused_equals_sliced": equal}


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
    assert torch.cuda.is_available(), "resize_box_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): Resize(256) + CenterCrop(224) and thumbnail() chains",
            "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
