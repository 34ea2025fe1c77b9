"""Device time per step of Exif-oriented decoding (BatchDecoder(exif_orientation=True)) against what a user does without it, one
GPU:

    python tools/orientation_bench.py [--workloads cfg3,cfg2] [--frames 256] [--steps 5] [--warmup 1] [--rounds 3]

Every frame of a workload gets an Exif APP1 segment; each batch is uniform in one orientation o of 1, 2, 3 and 6. Per o, timed with
CUDA events around `--steps` back-to-back steps in `--rounds` alternating rounds:
  packed_o   decode() of the flagged batch into its packed slots
  f16_o      decode_into an fp16 [N, 3, H_o, W_o] tensor with an ImageNet-style map, oriented in the store
  rot_o      (o > 1) the same batch without the flag decode_into an fp16 [N, 3, H, W] tensor, then torch.flip / torch.rot90 into a
             preallocated oriented tensor, `CHUNK` frames at a time
f16_o and rot_o must write the same bytes ("agree"); packed_o is compared with packed_1 oriented on the device.
Prints one JSON line with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools import bench_inputs  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SCALE, BIAS = [1 / (255 * s) for s in STD], [-m / s for m, s in zip(MEAN, STD)]
CHUNK = 16
ORIENTS = (1, 2, 3, 6)


def exif_tagged(data, o):
    """data with an APP1 Exif segment of orientation o behind SOI: little-endian TIFF header, IFD0 with one SHORT 0x0112"""
    tiff = b"II*\0" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, o, 0) + struct.pack("<I", 0)
    payload = b"Exif\0\0" + tiff
    return data[:2] + b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload + data[2:]


def _orient_torch(t, o):
    """[.., H, W] -> the oriented [.., H_o, W_o] (the numpy table of tests/orientation_model.py in torch)"""
    import torch
    if o == 2:
        return torch.flip(t, (-1,))
    if o == 3:
        return torch.flip(t, (-2, -1))
    if o == 6:
        return torch.rot90(t, -1, (-2, -1))
    return t


def _digest(chunks):
    """a position-weighted sum of the bytes of a sequence of tensors, on the device"""
    import torch
    total, off = 0, 0
    for t in chunks:
        x = t.contiguous().view(-1).view(torch.uint8).to(torch.int64)
        w = torch.arange(off, off + x.numel(), device=x.device, dtype=torch.int64) % 65521 + 1
        total += int((x * w).sum())
        off += x.numel()
    return total


def _packed_frames(dec, out, o):
    """the [H, W, C] frames of a decode() output, each oriented by o"""
    for i in range(dec.n):
        f = dec.frame_view(out, i)
        yield _orient_torch(f.permute(2, 0, 1), o).permute(1, 2, 0)


def run_workload(libjpeg_b200, workload, args):
    import torch
    base = bench_inputs.make_frames(workload, args.distinct, max(1, min(16, os.cpu_count() or 1)))
    frames = [base[i % len(base)] for i in range(args.frames)]
    N = len(frames)
    stream = torch.cuda.Stream()
    decs = {o: libjpeg_b200.BatchDecoder([exif_tagged(bytes(f), o) for f in frames], exif_orientation=True) for o in ORIENTS}
    plain = libjpeg_b200.BatchDecoder([exif_tagged(bytes(f), 6) for f in frames])  # the user's alternative: the flag off
    for d in list(decs.values()) + [plain]:
        d.upload(stream)
    torch.cuda.synchronize()
    H, W = plain.output_shape(0, 0)
    digests = {}

    def setup(v):
        kind, o = v.split("_")
        o = int(o)
        if kind == "packed":
            out = decs[o].new_output()
            return (lambda: decs[o].decode(out, stream)), out
        h, w = decs[o].output_shape(0, 0)
        if kind == "f16":
            t = torch.empty(N, 3, h, w, dtype=torch.float16, device="cuda")
            return (lambda: decs[o].decode_into(t, stream, scale=SCALE, bias=BIAS)), t
        full = torch.empty(N, 3, H, W, dtype=torch.float16, device="cuda")
        dst = torch.empty(N, 3, h, w, dtype=torch.float16, device="cuda")

        def step():
            plain.decode_into(full, stream, scale=SCALE, bias=BIAS)
            with torch.cuda.stream(stream):
                for a in range(0, N, CHUNK):
                    dst[a:a + CHUNK].copy_(_orient_torch(full[a:a + CHUNK], o))
        return step, dst

    variants = ["packed_%d" % o for o in ORIENTS] + ["f16_%d" % o for o in ORIENTS] + ["rot_%d" % o for o in ORIENTS if o > 1]
    times = {v: [] for v in variants}
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
            if rnd == args.rounds - 1:  # digests of what the variant wrote (packed_1: of its frames under every orientation)
                torch.cuda.synchronize()
                kind, o = v.split("_")
                if kind == "packed":
                    for oo in (ORIENTS if o == "1" else (int(o),)):
                        digests["%s_%d" % (v, oo)] = _digest(_packed_frames(decs[int(o)], keep, oo if o == "1" else 1))
                else:
                    digests[v] = _digest(keep[a] for a in range(N))
            del step, keep
            torch.cuda.empty_cache()
    agree = {}
    for o in ORIENTS:
        agree["packed_%d" % o] = digests["packed_%d_%d" % (o, o)] == digests["packed_1_%d" % o]
        if o > 1:
            agree["f16_%d" % o] = digests["f16_%d" % o] == digests["rot_%d" % o]
    for d in list(decs.values()) + [plain]:
        d.close()
    torch.cuda.empty_cache()
    best = {v: round(min(times[v]), 3) for v in variants}
    return {"frames": N, "size": "%dx%d" % (W, H), "ms_per_step": {v: [round(t, 3) for t in times[v]] for v in variants},
            "ms_per_step_best": best, "frames_per_s_best": {v: round(N / best[v] * 1000.0, 1) for v in variants}, "agree": agree}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg2")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=32)
    args = ap.parse_args()
    import torch
    import libjpeg_b200
    assert torch.cuda.is_available(), "orientation_bench.py needs a CUDA device"
    torch.cuda.set_device(0)
    line = {"metric": "device ms per step (CUDA events), Exif orientation in the store vs decode then flip / rot90", "gpu": bench.gpu_facts(0),
            "steps": args.steps, "rounds": args.rounds}
    for w in args.workloads.split(","):
        line[w] = run_workload(libjpeg_b200, w, args)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
