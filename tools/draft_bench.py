"""Device time per step of BatchDecoder(reconstruction="libjpeg-turbo", draft=...) (DESIGN §17) against the full-size turbo
reconstruction and the reference path's downscale=k, one GPU:

    python tools/draft_bench.py [--workloads cfg3,cfg2] [--frames 128] [--steps 5] [--warmup 1] [--rounds 3] [--out DIR]

Timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds; the best round is reported next to
all of them. Cases on the same frames:
  packed/k       decode() into the packed output: k = 1 the undrafted turbo batch, k = 2, 4, 8 drafted to 1/k (a request of
                 (H // k, W // k)), and reference/k the reference path's downscale=k (DESIGN §10's box-average IDCT) for scale
  fp16/k         decode_into an fp16 [N, 3, H', W'] tensor with the ImageNet map, turbo at k = 1, 2, 4, 8
  rrc224/turbo   RandomResizedCrop rectangles (seeded) of the full frame, resized to fp16 [N, 3, 224, 224] with the ImageNet map
  rrc224/draft   the same after draft=(224, 224), as a Pillow loader drafts before its RandomResizedCrop: rectangles drawn on the
                 drafted image with the same seed
The entropy / reconstruction split comes from the batch's event timing in a step of its own. With --out, one packed k = 2 and one
packed k = 8 step per workload run again under torch.profiler (CUDA activities) for the times of turbo_idct_draft_kernel (A),
turbo_reconstruct_draft_kernel (B) and turbo_generic_draft_kernel (C), whichever run. Prints one JSON line with the card's name and power limit, read in the same run.
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
from tools.turbo_bench import _timed, rrc_rects  # noqa: E402

T = 224
TURBO = "libjpeg-turbo"
SCALES = (1, 2, 4, 8)


def _drafted_rects(frames, drafts, seed):
    """rrc_rects' rule on the drafted images (their output_size at the draft scale)"""
    import numpy as np
    from libjpeg_b200 import decoder
    rng = np.random.default_rng(seed)
    out = []
    for f, d in zip(frames, drafts):
        h, w = decoder.output_size(f, downscale=decoder.draft_scale(f, d))
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


def run_workload(libjpeg_b200, workload, args):
    import torch
    from libjpeg_b200 import decoder
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    H, W = decoder.output_size(frames[0])
    stream = torch.cuda.Stream()
    decs = {}
    for k in SCALES:
        draft = None if k == 1 else (H // k, W // k)
        decs["packed", k] = libjpeg_b200.BatchDecoder(frames, reconstruction=TURBO, draft=draft)
        decs["fp16", k] = libjpeg_b200.BatchDecoder(frames, reconstruction=TURBO, mode="RGB", draft=draft)
        if k > 1:
            decs["reference", k] = libjpeg_b200.BatchDecoder(frames, downscale=k)
    small_draft = [(T, T)] * N
    decs["rrc224", "turbo"] = libjpeg_b200.BatchDecoder(frames, reconstruction=TURBO, mode="RGB", crop=rrc_rects(frames, 11), resize=(T, T))
    decs["rrc224", "draft"] = libjpeg_b200.BatchDecoder(frames, reconstruction=TURBO, mode="RGB", draft=small_draft,
                                                        crop=_drafted_rects(frames, small_draft, 11), resize=(T, T))
    for d in decs.values():
        d.upload(stream)
    torch.cuda.synchronize()
    outs = {key: decs[key].new_output() for key in decs if key[0] in ("packed", "reference")}
    full = {k: torch.empty(N, 3, *decs["fp16", k].output_shape(0, 0), dtype=torch.float16, device="cuda") for k in SCALES}
    small = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
    steps = {}
    for key in decs:
        if key in outs:
            steps[key] = (lambda key=key: decs[key].decode(outs[key], stream))
        elif key[0] == "fp16":
            steps[key] = (lambda key=key: decs[key].decode_into(full[key[1]], stream, scale=SCALE, bias=BIAS))
        else:
            steps[key] = (lambda key=key: decs[key].decode_into(small, stream, scale=SCALE, bias=BIAS))
    times = {key: [] for key in steps}
    for rnd in range(args.rounds):
        for key in (list(steps) if rnd % 2 == 0 else list(steps)[::-1]):
            times[key].append(_timed(steps[key], args, stream))
    split = {}
    for k in SCALES:
        d = decs["packed", k]
        d.enable_timing(True)
        steps["packed", k]()
        torch.cuda.synchronize()
        split[str(k)] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    name = lambda key: "%s/%s" % key  # noqa: E731
    res = {"frames": N, "size": "%dx%d" % (W, H), "draft_scale_224": decoder.draft_scale(frames[0], (T, T)),
           "ms_per_step": {name(key): [round(t, 3) for t in times[key]] for key in times},
           "ms_per_step_best": {name(key): round(min(times[key]), 3) for key in times},
           "entropy_recon_ms_packed_turbo": split}
    if args.out:
        from torch.profiler import ProfilerActivity, profile
        res["draft_kernel_ms"] = {}
        for k in (2, 8):
            step = steps["packed", k]
            step()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    step()
                torch.cuda.synchronize()
            kt = {}
            for ev in prof.key_averages():
                for kname in ("turbo_idct_draft_kernel", "turbo_reconstruct_draft_kernel", "turbo_generic_draft_kernel"):
                    if kname in ev.key:
                        kt[kname] = round(ev.device_time_total / 1000.0 / args.steps, 3)
            os.makedirs(args.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.out, "draft_%s_k%d.pt.trace.json" % (workload, k)))
            res["draft_kernel_ms"][str(k)] = kt
    for d in decs.values():
        d.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (kernel times are measured only with it)")
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "draft_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): libjpeg-turbo full size vs draft 1/2, 1/4, 1/8, packed / fp16 [N, 3, H', W'] / "
                      "RandomResizedCrop -> fp16 [N, 3, 224, 224], ImageNet map; reference downscale=k for scale",
            "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
