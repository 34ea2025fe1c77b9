"""libjpeg_b200 -- a H100-native (sm_90a) baseline-JPEG decode path behind the thorfdbg/libjpeg interface.

The product is the shared library ``libb200jpg.so`` (hand-written CUDA kernels + C ABI + the C++ ``class JPEG``
shim, see ``include/``).  This Python package is the thin host layer used by the tests and the benchmark:
ctypes bindings of the C ABI, with PyTorch supplying device memory and streams only.
"""
from .native import NativeError, lib, library_path  # noqa: F401
from .decoder import BatchDecoder, FrameInfo, parse, sample_table  # noqa: F401
