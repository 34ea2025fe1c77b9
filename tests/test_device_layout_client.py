"""GPU: JPEG::DisplayRectangle into device bitmaps of any layout (JPGTAG_B200_DEVICE_BITMAPS, tests/client/device_layout_client.cpp):
per-component device planes, a BGR canvas, bottom-up planes and, without upsampling, each component at its own size, in
8-row stripes. What the client copies back must be the reference's samples where the requests put them and the sentinel
everywhere else (padding columns, rows below the image)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SENT = 0x5A
NAMES = ["c420_96x80_z6_q75", "c420_127x255_z7_q30", "c444_17x9_q95", "g_40x24_z2_q75", "c422_100x60_z5_q80", "c440_100x61_z3_q80",
         "deep12/d12_420_50x38_q60"]


@pytest.fixture(scope="module")
def client(built, tmp_path_factory):
    import subprocess
    lib_dir = os.path.join(ROOT, "libjpeg_b200")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path_factory.mktemp("client") / "device_layout_client")
    subprocess.run(["g++", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                    os.path.join(ROOT, "tests", "client", "device_layout_client.cpp"), "-L" + lib_dir, "-lb200jpg",
                    "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"),
                    "-o", exe], check=True)
    return exe


def _reference(built, name, upsample):
    """per component the samples as [h, w] uint16 arrays: the reference's pixels, or (upsample=False) the batch path's planes"""
    import torch
    path = os.path.join(GOLDEN, name + ".jpg")
    if upsample:
        if name.startswith("deep12/"):
            px = np.load(os.path.join(GOLDEN, "deep12", "deep12_pixels.npz"))[name.split("/")[1]]
        else:
            px = np.load(os.path.join(GOLDEN, "golden_pixels.npz"))[name]
        info = built.parse(open(path, "rb").read())
        px = px.reshape(info.height, info.width, info.ncomp).astype(np.uint16)
        return [px[..., c] for c in range(info.ncomp)]
    dec = built.BatchDecoder([open(path, "rb").read()], upsample=False)
    out = dec.new_output()
    dec.upload()
    dec.decode(out)
    torch.cuda.synchronize()
    return [p.cpu().numpy().view(np.uint16) if p.dtype == torch.int16 else p.cpu().numpy().astype(np.uint16) for p in dec.plane_views(out, 0)]


def _put(buf, at, v, ss):
    buf[at] = (v & 0xFF).astype(np.uint8)
    if ss == 2:
        buf[at + 1] = (v >> 8).astype(np.uint8)


@pytest.mark.parametrize("mode", ["planar", "bgr", "bottomup", "planes"])
@pytest.mark.parametrize("name", NAMES)
def test_device_bitmaps_of_any_layout(built, client, tmp_path, mode, name):
    import subprocess
    raw = str(tmp_path / "o.raw")
    r = subprocess.run([client, mode, os.path.join(GOLDEN, name + ".jpg"), raw], capture_output=True, text=True)
    lines = r.stdout.split("\n")
    assert r.returncode == 0 and "ok=1" in lines[0], (name, mode, r.stdout, r.stderr)
    w, h, d, ss = (int(v) for v in lines[0].split()[:4])
    bufs = [tuple(int(v) for v in ln.split()) for ln in lines[1:] if ln.strip()]
    got = np.fromfile(raw, dtype=np.uint8)
    assert got.size == sum(rows * pitch for _, rows, pitch in bufs)
    want = np.full(got.size, SENT, dtype=np.uint8)
    refs = _reference(built, name, mode != "planes")
    assert len(refs) == d
    starts = np.cumsum([0] + [rows * pitch for _, rows, pitch in bufs])
    for c, ref in enumerate(refs):
        ys, xs = np.mgrid[0:ref.shape[0], 0:ref.shape[1]].astype(np.int64)
        if mode == "bgr":
            at = ys * bufs[0][2] + xs * d * ss + (d - 1 - c) * ss
        else:
            _, rows, pitch = bufs[c]
            at = starts[c] + (rows - 1 - ys if mode == "bottomup" else ys) * pitch + xs * ss
        _put(want, at, ref, ss)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, "%s %s: %d bytes differ, first at %d" % (name, mode, len(bad), bad[0])
