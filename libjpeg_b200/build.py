"""Builds libjpeg_b200/libb200jpg.so (CUDA kernels for sm_90a + C ABI + C++ JPEG shim) in-tree with nvcc.

The shared object travels to the GPU box with the repo snapshot; nothing is JIT-compiled at run time.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200jpg.so")
SYNTH_LIB = os.path.join(HERE, "libb200jpg_synth.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
          "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]

CUDA_SOURCES = ["huffman_sm100.cu", "specsync_sm100.cu", "progressive_sm100.cu", "progfused_sm100.cu", "recon_sm100.cu", "bitmap_sm100.cu",
                "microbench_sm100.cu", "resample_sm100.cu", "turbo_sm90.cu"]
HOST_SOURCES = ["abi.cpp", "parse.cpp", "jpeg_shim.cpp"]
# the resample tables are computed on the host in double precision: no contraction into FMA, so every host computes the same bits
EXTRA = {"resample_sm100.cu": ["-Xcompiler", "-ffp-contract=off"]}


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libb200jpg.so cannot be built")
    return nvcc


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build step failed: " + " ".join(cmd))
    if verbose and (r.stdout or r.stderr):
        print(r.stdout + r.stderr)


def build(force=False, verbose=False, ptxas_info=False):
    """Compile every translation unit for sm_90a and link the shared objects. Returns the library path."""
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".hpp", ".cuh"))]
    headers += [os.path.join(ROOT, "include", "b200jpg.h")]
    headers += [os.path.abspath(__file__)]  # the flags (ARCH, COMMON) live here: objects built with other flags are stale
    idir = os.path.join(ROOT, "include", "interface")
    if os.path.isdir(idir):
        headers += [os.path.join(idir, f) for f in os.listdir(idir)]
    objs = []
    for src in CUDA_SOURCES + HOST_SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(OBJ, src + ".o")
        objs.append(obj)
        if force or _newer(obj, [path] + headers):
            cmd = [nvcc] + ARCH + COMMON + EXTRA.get(src, [])
            if src.endswith(".cu") and ptxas_info:
                cmd += ["-Xptxas", "-v"]
            cmd += ["-c", path, "-o", obj]
            _run(cmd, verbose or ptxas_info)
    if force or _newer(LIB, objs):
        _run([nvcc] + ARCH + ["-shared", "-o", LIB] + objs, verbose)
    synth = os.path.join(CSRC, "synth_encoder.cpp")
    if os.path.exists(synth) and (force or _newer(SYNTH_LIB, [synth])):
        _run(["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", SYNTH_LIB, synth], verbose)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True, ptxas_info="--ptxas" in sys.argv)
    print("built", LIB)
