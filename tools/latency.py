"""Latency of ONE frame through the C ABI (VERDICT r1 weak #3): b200jpg_decode_to_host -- parse, pack, H2D, restart index, kernels,
D2H of every pixel, all inside -- and the device part alone (upload + decode on a resident batch), for a 4K 4:2:0 q75 frame with
one restart interval per MCU row, the same frame without restart markers, and the progressive one.
    python tools/latency.py            prints one JSON line"""
import ctypes
import json
import statistics
import sys
import time

sys.path.insert(0, ".")
import torch

import libjpeg_b200
from libjpeg_b200 import native
from tools import bench_inputs


def main():
    res = {}
    from libjpeg_b200.decoder import Context
    ctx = Context(-1)
    for wl in ("cfg3", "cfg3n", "cfg4", "cfg2"):
        data = bench_inputs.make_frames(wl, 1, 1)[0]
        fi = libjpeg_b200.parse(data)
        out = torch.empty(fi.width * fi.height * fi.ncomp, dtype=torch.uint8).pin_memory()
        buf = (ctypes.c_char * len(data)).from_buffer_copy(data)
        ptrs = (ctypes.c_void_p * 1)(ctypes.addressof(buf))
        lens = (ctypes.c_size_t * 1)(len(data))
        ts = []
        for it in range(12):
            t0 = time.perf_counter()
            rc = native.lib.b200jpg_decode_to_host(ctx.handle, ptrs, lens, 1, ctypes.c_void_p(out.data_ptr()), ctypes.c_uint64(out.numel()))
            ts.append((time.perf_counter() - t0) * 1e3)
            assert rc == 0, rc
        dec = libjpeg_b200.BatchDecoder([data], ctx=ctx)
        dout = dec.new_output()
        td = []
        for it in range(12):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dec.upload()
            dec.decode(dout)
            torch.cuda.synchronize()
            td.append((time.perf_counter() - t0) * 1e3)
        dec.enable_timing(True)
        dec.decode(dout)
        torch.cuda.synchronize()
        e, r = dec.last_timing()
        res[wl] = {"decode_to_host_ms_median": round(statistics.median(ts[2:]), 3), "decode_to_host_ms_min": round(min(ts[2:]), 3),
                   "upload_plus_kernels_ms_median": round(statistics.median(td[2:]), 3), "entropy_ms": round(e, 3), "reconstruction_ms": round(r, 3),
                   "codestream_bytes": len(data)}
        dec.close()
    print(json.dumps({"what": "one frame per call, one GPU; decode_to_host = b200jpg_decode_to_host wall clock (host parse + pack + H2D + "
                              "restart index + kernels + D2H into pinned memory + batch teardown)", "frames": res}))


if __name__ == "__main__":
    main()
