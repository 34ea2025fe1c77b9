"""Device time per step of the output modes (BatchDecoder(mode=...), DESIGN §14) against what a caller does without them, one GPU:

    python tools/mode_bench.py [--workloads cfg3,cfg2] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3] [--grey-every 32]

Timed with CUDA events around `--steps` back-to-back steps, in `--rounds` alternating rounds; the best round is reported next to
all of them. Cases:
  luma            decode_into of BatchDecoder(mode="L") into a uint8 [N, 1, H, W] tensor
  nct_plane0      decode_into of BatchDecoder(color_transform=False) with planes 1 and 2 into a scratch [N, 2, H, W] tensor and
                  plane 0 into the same [N, 1, H, W] tensor: the same bytes as `luma`
  rgb_fused       one batch in which every `--grey-every`-th frame is grey, BatchDecoder(mode="RGB", crop=center, resize=(224,
                  224)) into fp16 [N, 3, 224, 224] with the ImageNet map, one decode_into call
  rgb_split       what is possible without the mode: the colour frames as one batch into their rows of the tensor, the grey frames
                  as a second batch into a [G, 1, 224, 224] fp16 tensor, expanded by torch into the same rows
The entropy / reconstruction split of luma and nct_plane0 comes from the batch's event timing in a step of its own. Prints one
JSON line with the card's name and power limit, read in the same run.
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


def grey_of(data):
    """the grey codestream of a frame's luma: the synthetic encoder on the decoded frame's first channel"""
    from PIL import Image
    import io
    from libjpeg_b200 import synth
    img = np.asarray(Image.open(io.BytesIO(bytes(data))).convert("L"))
    return synth.encode(img, 85, (1, 1), 0).tobytes()


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


def run_workload(libjpeg_b200, workload, args):
    import torch
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [bytes(base[i % len(base)]) for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    grey_base = [grey_of(f) for f in base[:4]]
    grey_idx = list(range(0, N, args.grey_every))
    mixed = [grey_base[i % len(grey_base)] if i in grey_idx else f for i, f in enumerate(frames)]
    colour_idx = [i for i in range(N) if i not in grey_idx]

    luma = libjpeg_b200.BatchDecoder(frames, mode="L")
    nct = libjpeg_b200.BatchDecoder(frames, color_transform=False)
    H, W = luma.output_shape(0, 0)
    rect = lambda h, w: ((w - min(h, w)) // 2, (h - min(h, w)) // 2, min(h, w), min(h, w))  # center square
    rects = [rect(*libjpeg_b200.decoder.output_size(f)) for f in mixed]
    fused = libjpeg_b200.BatchDecoder(mixed, mode="RGB", crop=rects, resize=(T, T))
    split_c = libjpeg_b200.BatchDecoder([mixed[i] for i in colour_idx], crop=[rects[i] for i in colour_idx], resize=(T, T))
    split_g = libjpeg_b200.BatchDecoder([mixed[i] for i in grey_idx], crop=[rects[i] for i in grey_idx], resize=(T, T))
    for d in (luma, nct, fused, split_c, split_g):
        d.upload(stream)
    torch.cuda.synchronize()

    y = torch.empty(N, 1, H, W, dtype=torch.uint8, device="cuda")
    chroma = torch.empty(N, 2, H, W, dtype=torch.uint8, device="cuda")
    nct_dst = [[y[i, 0], chroma[i, 0], chroma[i, 1]] for i in range(N)]
    out = torch.empty(N, 3, T, T, dtype=torch.float16, device="cuda")
    grey_out = torch.empty(len(grey_idx), 1, T, T, dtype=torch.float16, device="cuda")
    rows = [[out[i, 0], out[i, 1], out[i, 2]] for i in colour_idx]
    gi = torch.tensor(grey_idx, device="cuda")
    scale_g = torch.tensor(SCALE, device="cuda").view(1, 3, 1, 1)
    bias_g = torch.tensor(BIAS, device="cuda").view(1, 3, 1, 1)

    def split_step():
        split_c.decode_into(rows, stream, scale=SCALE, bias=BIAS)
        split_g.decode_into(grey_out, stream)  # uint8 values as float16, mapped per output channel below
        with torch.cuda.stream(stream):
            out.index_copy_(0, gi, (grey_out.float().expand(-1, 3, -1, -1) * scale_g + bias_g).half())

    steps = {
        "luma": lambda: luma.decode_into(y, stream),
        "nct_plane0": lambda: nct.decode_into(nct_dst, stream),
        "rgb_fused": lambda: fused.decode_into(out, stream, scale=SCALE, bias=BIAS),
        "rgb_split": split_step,
    }
    times = {v: [] for v in steps}
    for rnd in range(args.rounds):
        for v in (list(steps) if rnd % 2 == 0 else list(steps)[::-1]):
            times[v].append(_timed(steps[v], args, stream))
    steps["luma"]()
    torch.cuda.synchronize()
    y_luma = y.clone()
    steps["nct_plane0"]()
    torch.cuda.synchronize()
    # the two RGB variants write the same tensor up to the float rounding of the split path's map (grey: in float32, then half)
    steps["rgb_fused"]()
    torch.cuda.synchronize()
    a = out.float().clone()
    split_step()
    torch.cuda.synchronize()
    maxdiff = float((a - out.float()).abs().max())
    split = {}
    for v, d in (("luma", luma), ("nct_plane0", nct)):
        d.enable_timing(True)
        steps[v]()
        torch.cuda.synchronize()
        split[v] = [round(t, 3) for t in d.last_timing()]
        d.enable_timing(False)
    for d in (luma, nct, fused, split_c, split_g):
        d.close()
    torch.cuda.empty_cache()
    return {"frames": N, "size": "%dx%d" % (W, H), "grey_frames": len(grey_idx),
            "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in times},
            "ms_per_step_best": {v: round(min(times[v]), 3) for v in times},
            "entropy_recon_ms": split, "max_abs_diff_rgb_fused_vs_split": maxdiff,
            "luma_equals_plane0": bool(torch.equal(y_luma, y))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--grey-every", type=int, default=32, help="every k-th frame of the RGB case is grey (default: 1 in 32, ~3 %%)")
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "mode_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events): mode=L vs color_transform=False keeping plane 0; mode=RGB mixed batch "
                      "resized to fp16 [N, 3, 224, 224] in one call vs two batches and a torch expand",
            "gpu": bench.gpu_facts(0), "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
