"""Synthetic inputs: the deterministic source images of SURVEY.md 8d and a baseline-JPEG stream generator
(libb200jpg_synth.so, csrc/synth_encoder.cpp).  Benchmark / test inputs only -- not part of the decode path."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "libb200jpg_synth.so")
_lib = None


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError("libb200jpg_synth.so is missing: run `python -m libjpeg_b200.build`")
        _lib = ctypes.CDLL(_PATH)
        _lib.b200jpg_synth_encode.restype = ctypes.c_long
        _lib.b200jpg_synth_encode.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_long]
        _lib.b200jpg_synth_encode_ex.restype = ctypes.c_long
        _lib.b200jpg_synth_encode_ex.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                 ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_long]
    return _lib


def source_image(w, h, seed):
    """S(w,h,seed): per-channel ramps (255x/w, 255y/h, 255(x+y)/(w+h)) + N(0,12), clipped to u8."""
    rng = np.random.default_rng(seed)
    x = np.arange(w, dtype=np.float32)[None, :]
    y = np.arange(h, dtype=np.float32)[:, None]
    img = np.empty((h, w, 3), dtype=np.float32)
    img[..., 0] = 255.0 * x / w
    img[..., 1] = 255.0 * y / h
    img[..., 2] = 255.0 * (x + y) / (w + h)
    img += rng.normal(0.0, 12.0, size=(h, w, 3)).astype(np.float32)
    return np.clip(img, 0, 255).astype(np.uint8)


NON_INTERLEAVED, SOF1, DQT16, SHARED_TABLES = 1, 2, 4, 8


def encode(pixels, quality=75, subsampling=(2, 2), restart_interval=0, flags=0):
    """Baseline JPEG bytes for an [H,W,3] or [H,W] uint8 image. subsampling = (hs, vs) of the luma component.
    flags: NON_INTERLEAVED (one scan per component), SOF1 (extended sequential header), DQT16 (16-bit table entries),
    SHARED_TABLES (every component on Huffman tables 0)."""
    lib = _load()
    px = np.ascontiguousarray(pixels, dtype=np.uint8)
    h, w = px.shape[:2]
    nc = 1 if px.ndim == 2 else px.shape[2]
    cap = w * h * nc * 2 + 65536
    out = np.empty(cap, dtype=np.uint8)
    n = lib.b200jpg_synth_encode_ex(px.ctypes.data, w, h, nc, subsampling[0], subsampling[1], quality, restart_interval, flags,
                                    out.ctypes.data, cap)
    if n <= 0:
        raise RuntimeError("synthetic encoder failed (%d)" % n)
    return out[:n].copy()


def frame(w, h, seed, quality=75, subsampling=(2, 2), restart_interval=None):
    """One synthetic codestream; restart interval defaults to one MCU row (the benchmark's partitioning)."""
    if restart_interval is None:
        restart_interval = (w + 8 * subsampling[0] - 1) // (8 * subsampling[0])
    return encode(source_image(w, h, seed), quality, subsampling, restart_interval)
