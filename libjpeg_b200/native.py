"""ctypes bindings of include/b200jpg.h.  Loading fails loudly when the library has not been built."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("B200JPG_LIB") or os.path.join(_HERE, "libb200jpg.so")  # env override: kernel experiments


class NativeError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("b200jpg error %d: %s" % (code, message))
        self.code = code
        self.message = message


class FrameInfoStruct(ctypes.Structure):
    _fields_ = [
        ("width", ctypes.c_uint32), ("height", ctypes.c_uint32),
        ("ncomp", ctypes.c_uint8), ("precision", ctypes.c_uint8), ("frame_type", ctypes.c_uint8), ("ycbcr", ctypes.c_uint8),
        ("comp_id", ctypes.c_uint8 * 4), ("hs", ctypes.c_uint8 * 4), ("vs", ctypes.c_uint8 * 4),
        ("subx", ctypes.c_uint8 * 4), ("suby", ctypes.c_uint8 * 4), ("tq", ctypes.c_uint8 * 4),
        ("mcu_cols", ctypes.c_uint32), ("mcu_rows", ctypes.c_uint32),
        ("blocks_w", ctypes.c_uint32 * 4), ("blocks_h", ctypes.c_uint32 * 4),
        ("nscans", ctypes.c_uint32), ("restart_interval", ctypes.c_uint32), ("n_intervals", ctypes.c_uint32),
        ("ecs_bytes", ctypes.c_uint64), ("stored_blocks", ctypes.c_uint64),
    ]


class PlaneStruct(ctypes.Structure):
    """b200jpg_plane: the sample (x, y) of a component goes to data + x * bytes_per_pixel + y * bytes_per_row."""
    _fields_ = [("data", ctypes.c_void_p), ("bytes_per_pixel", ctypes.c_int32), ("pad", ctypes.c_int32), ("bytes_per_row", ctypes.c_int64)]


class ConvertStruct(ctypes.Structure):
    """b200jpg_convert: element type (SAMPLE_*) and the per-component map y = v * scale[c] + bias[c] of a float destination."""
    _fields_ = [("type", ctypes.c_int32), ("scale", ctypes.c_float * 4), ("bias", ctypes.c_float * 4)]


class ConvertTableStruct(ctypes.Structure):
    """b200jpg_convert_table: element type (SAMPLE_*) and the per-component sample tables y = table[c][v] of a float destination."""
    _fields_ = [("type", ctypes.c_int32), ("table", (ctypes.c_float * 256) * 4)]


class RectStruct(ctypes.Structure):
    """b200jpg_rect: a crop rectangle of b200jpg_batch_create_crop, in output coordinates; all zero = the whole frame."""
    _fields_ = [("x", ctypes.c_uint32), ("y", ctypes.c_uint32), ("width", ctypes.c_uint32), ("height", ctypes.c_uint32)]


class SizeStruct(ctypes.Structure):
    """b200jpg_size: a target size of b200jpg_batch_create_resize; all zero = not resized."""
    _fields_ = [("width", ctypes.c_uint32), ("height", ctypes.c_uint32)]


class BoxStruct(ctypes.Structure):
    """b200jpg_box: a source box of b200jpg_batch_create_resample, Pillow's (x0, y0, x1, y1); all zero = the default box."""
    _fields_ = [("x0", ctypes.c_double), ("y0", ctypes.c_double), ("x1", ctypes.c_double), ("y1", ctypes.c_double)]


SAMPLE_F32, SAMPLE_F16, SAMPLE_BF16 = 1, 2, 3
FLAG_NO_COLOR_TRANSFORM, FLAG_NO_UPSAMPLE = 1, 2
DOWNSCALE_FLAGS = {1: 0x0, 2: 0x4, 4: 0x8, 8: 0xC}  # B200JPG_FLAG_DOWNSCALE_k
FLAG_EXIF_ORIENTATION = 0x10
MODE_FLAGS = {None: 0x0, "RGB": 0x20, "L": 0x40}  # B200JPG_FLAG_OUTPUT_RGB / _L, named after PIL's Image.convert(mode)
RECONSTRUCTION_FLAGS = {"reference": 0x0, "libjpeg-turbo": 0x80}  # B200JPG_FLAG_LIBJPEG_TURBO
COLORSPACES = [None, "L", "YCbCr", "RGB", "CMYK", "YCCK"]  # B200JPG_COLORSPACE_UNKNOWN .. _YCCK, named after PIL's modes
RESAMPLE = {"lanczos": 1, "bilinear": 2, "bicubic": 3, "box": 4, "hamming": 5}  # B200JPG_RESAMPLE_*, PIL's values
# B200JPG_RESAMPLE_CV_*: OpenCV's cv2.resize, 0x100 | cv2.INTER_LINEAR / cv2.INTER_AREA (DESIGN §20)
RESAMPLE.update({"cv2-linear": 0x101, "cv2-area": 0x103})
FLIP_H, FLIP_V = 1, 2  # B200JPG_FLIP_H / _V of b200jpg_batch_create_flip


def library_path():
    return _LIB_PATH


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            "libjpeg_b200/libb200jpg.so is missing: build it with `python -m libjpeg_b200.build` "
            "(or __graft_entry__.build()). There is no CPU fallback for the decode path.")
    l = ctypes.CDLL(_LIB_PATH)
    vp, u8p, u64, i32 = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint8), ctypes.c_uint64, ctypes.c_int
    sig = {
        "b200jpg_parse": (i32, [vp, ctypes.c_size_t, ctypes.POINTER(FrameInfoStruct)]),
        "b200jpg_exif_orientation": (i32, [vp, ctypes.c_size_t]),
        "b200jpg_colorspace": (i32, [vp, ctypes.c_size_t]),
        "b200jpg_output_size": (i32, [vp, ctypes.c_size_t, ctypes.c_uint, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_build_tables": (u64, [vp, ctypes.c_size_t, i32, vp, u64]),
        "b200jpg_create": (i32, [i32, ctypes.POINTER(vp)]),
        "b200jpg_destroy": (None, [vp]),
        "b200jpg_trim": (None, [vp]),
        "b200jpg_last_error": (i32, [vp, ctypes.POINTER(ctypes.c_char_p)]),
        "b200jpg_batch_create": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.POINTER(vp)]),
        "b200jpg_batch_create_ex": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint, ctypes.POINTER(vp)]),
        "b200jpg_batch_create_crop": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint,
                                            ctypes.POINTER(RectStruct), ctypes.POINTER(vp)]),
        "b200jpg_batch_create_resize": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint,
                                              ctypes.POINTER(RectStruct), ctypes.POINTER(SizeStruct), i32, ctypes.POINTER(vp)]),
        "b200jpg_batch_create_draft": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint,
                                             ctypes.POINTER(SizeStruct), ctypes.POINTER(RectStruct), ctypes.POINTER(SizeStruct), i32,
                                             ctypes.POINTER(vp)]),
        "b200jpg_batch_create_resample": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint,
                                                ctypes.POINTER(SizeStruct), ctypes.POINTER(RectStruct), ctypes.POINTER(SizeStruct),
                                                ctypes.POINTER(BoxStruct), ctypes.POINTER(RectStruct), i32, ctypes.c_double,
                                                ctypes.POINTER(vp)]),
        "b200jpg_batch_create_flip": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, i32, ctypes.c_uint,
                                            ctypes.POINTER(SizeStruct), ctypes.POINTER(RectStruct), ctypes.POINTER(SizeStruct),
                                            ctypes.POINTER(BoxStruct), ctypes.POINTER(RectStruct), i32, ctypes.c_double,
                                            ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(vp)]),
        "b200jpg_draft_scale": (i32, [vp, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32]),
        "b200jpg_resample_coefficients": (i32, [ctypes.c_uint32, ctypes.c_uint32, i32, vp, vp, u64, ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_resample_coefficients_box": (i32, [ctypes.c_uint32, ctypes.c_float, ctypes.c_float, ctypes.c_uint32, i32, vp, vp, u64,
                                                    ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_batch_destroy": (None, [vp]),
        "b200jpg_batch_frame_info": (i32, [vp, i32, ctypes.POINTER(FrameInfoStruct)]),
        "b200jpg_batch_output_extent": (i32, [vp, i32, i32, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_batch_frame_orientation": (i32, [vp, i32]),
        "b200jpg_batch_output_components": (i32, [vp, i32]),
        "b200jpg_batch_out_offset": (u64, [vp, i32]),
        "b200jpg_batch_out_bytes": (u64, [vp, i32]),
        "b200jpg_batch_ecs_bytes": (u64, [vp]),
        "b200jpg_batch_stored_blocks": (u64, [vp]),
        "b200jpg_batch_h2d_bytes": (u64, [vp]),
        "b200jpg_batch_export_tables": (u64, [vp, vp, u64]),
        "b200jpg_batch_import_tables": (i32, [vp, vp, u64]),
        "b200jpg_batch_upload": (i32, [vp, vp]),
        "b200jpg_batch_reindex": (i32, [vp, vp]),
        "b200jpg_batch_decode": (i32, [vp, vp, vp]),
        "b200jpg_batch_decode_into": (i32, [vp, ctypes.POINTER(PlaneStruct), vp]),
        "b200jpg_batch_decode_into_ex": (i32, [vp, ctypes.POINTER(PlaneStruct), ctypes.POINTER(ConvertStruct), vp]),
        "b200jpg_batch_decode_into_table": (i32, [vp, ctypes.POINTER(PlaneStruct), ctypes.POINTER(ConvertTableStruct), vp]),
        "b200jpg_batch_decode_entropy": (i32, [vp, vp]),
        "b200jpg_batch_reconstruct": (i32, [vp, vp, vp]),
        "b200jpg_batch_frame_status": (i32, [vp, i32]),
        "b200jpg_batch_read_coefficients": (i32, [vp, i32, i32, vp, u64]),
        "b200jpg_batch_last_launch_count": (i32, [vp]),
        "b200jpg_batch_enable_timing": (None, [vp, i32]),
        "b200jpg_batch_last_timing": (i32, [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]),
        "b200jpg_batch_last_unstuff_ms": (ctypes.c_float, [vp]),
        "b200jpg_selftest_restartless": (i32, [vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_selftest_restartless_items": (i32, [vp, ctypes.c_size_t, vp, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32),
                                                     ctypes.POINTER(ctypes.c_uint32)]),
        "b200jpg_selftest_table_cache": (i32, [ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32]),
        "b200jpg_decode_to_host": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, vp, u64]),
        "b200jpg_decode_to_host_ex": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, vp, u64, ctypes.c_uint]),
        "b200jpg_decode_to_device_ex": (i32, [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t), i32, ctypes.c_uint, ctypes.POINTER(vp), ctypes.POINTER(u64)]),
        "b200jpg_device_free": (None, [vp, vp]),
        "b200jpg_device_copy_rect": (i32, [vp, vp, ctypes.c_int64, vp, ctypes.c_int64, u64, u64]),
        "b200jpg_microbench_int32": (i32, [i32, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(l, name)  # AttributeError here = the ABI and the header disagree
        fn.restype = res
        fn.argtypes = args
    return l


lib = _load()
ABI_SYMBOLS = [
    "b200jpg_parse", "b200jpg_build_tables", "b200jpg_create", "b200jpg_destroy", "b200jpg_trim", "b200jpg_last_error", "b200jpg_batch_create", "b200jpg_batch_create_ex",
    "b200jpg_batch_destroy", "b200jpg_batch_frame_info", "b200jpg_batch_output_extent", "b200jpg_batch_out_offset", "b200jpg_batch_out_bytes",
    "b200jpg_batch_ecs_bytes", "b200jpg_batch_stored_blocks", "b200jpg_batch_h2d_bytes", "b200jpg_batch_export_tables",
    "b200jpg_batch_import_tables", "b200jpg_batch_upload", "b200jpg_batch_reindex", "b200jpg_batch_decode", "b200jpg_batch_decode_into", "b200jpg_batch_decode_into_ex",
    "b200jpg_batch_decode_entropy",
    "b200jpg_batch_reconstruct", "b200jpg_batch_frame_status", "b200jpg_batch_read_coefficients",
    "b200jpg_batch_last_launch_count", "b200jpg_batch_enable_timing", "b200jpg_batch_last_timing", "b200jpg_batch_last_unstuff_ms", "b200jpg_decode_to_host", "b200jpg_decode_to_host_ex", "b200jpg_decode_to_device_ex",
    "b200jpg_device_free", "b200jpg_device_copy_rect", "b200jpg_selftest_restartless", "b200jpg_selftest_restartless_items",
    "b200jpg_selftest_table_cache", "b200jpg_microbench_int32", "b200jpg_exif_orientation", "b200jpg_batch_frame_orientation",
    "b200jpg_batch_create_crop", "b200jpg_output_size", "b200jpg_batch_create_resize", "b200jpg_resample_coefficients",
    "b200jpg_batch_output_components", "b200jpg_colorspace", "b200jpg_batch_create_draft", "b200jpg_draft_scale",
    "b200jpg_batch_create_resample", "b200jpg_resample_coefficients_box", "b200jpg_batch_create_flip",
    "b200jpg_batch_decode_into_table",
]


def last_error(ctx=None):
    msg = ctypes.c_char_p()
    code = lib.b200jpg_last_error(ctx, ctypes.byref(msg))
    return code, (msg.value or b"").decode("utf-8", "replace")


def check(rc, ctx=None):
    if rc != 0:
        code, msg = last_error(ctx)
        raise NativeError(rc, msg if code == rc else "(no message)")
