"""ctypes binding of libsmap_b200.so (C ABI declared in include/smap_b200.h)."""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# SMAPB_LIB: load another build of the same library (A/B comparisons of kernel changes, tools/ab_hash.py); the default is
# the in-tree build
LIB_PATH = os.environ.get("SMAPB_LIB") or os.path.join(HERE, "lib", "libsmap_b200.so")

NJ, NL, MAXP, NC2D, SCALE_LEN = 15, 14, 127, 43, 9
PREC_BF16X3, PREC_BF16, PREC_FP16 = 3, 1, 16
RECORD_BYTES = MAXP * NJ * 4 * 8 + MAXP * 8 + MAXP * NJ * 4 * 4 + 8

EXPORTS = [
    "smapb_create", "smapb_destroy", "smapb_last_error", "smapb_version", "smapb_load_weight",
    "smapb_finalize_weights", "smapb_backbone_forward", "smapb_merge_scale", "smapb_assoc_extract",
    "smapb_assoc_connect", "smapb_lift3d", "smapb_infer_device", "smapb_infer_host", "smapb_launch_count",
    "smapb_plan_info", "smapb_conv_test", "smapb_profile_begin", "smapb_profile_end", "smapb_submit_host", "smapb_wait",
    "smapb_refine_load_weight", "smapb_refine_finalize", "smapb_refine_mlp", "smapb_refine3d", "smapb_set_refine",
    "smapb_json_open", "smapb_json_append", "smapb_json_close", "smapb_preprocess", "smapb_preprocess_host",
    "smapb_comm_unique_id", "smapb_comm_create", "smapb_comm_attach", "smapb_allgather_records",
    "smapb_infer_device_gather", "smapb_submit_host_gather", "smapb_set_tile_table", "smapb_get_tile_table",
    "smapb_lift3d_gt", "smapb_infer_device_gather_async", "smapb_gather_sync", "smapb_saturation_count",
    "smapb_jpeg_info", "smapb_decode_jpeg", "smapb_jpeg_info_ex", "smapb_decode_jpeg_ex", "smapb_png_info", "smapb_decode_png",
]

_lib = None


class SmapB200Error(RuntimeError):
    pass


def load():
    """Load the shared library (no compute).  Raises if it has not been built: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SmapB200Error(
            "libsmap_b200.so is not built (%s). Run `python -m smap_b200.build` "
            "(needs nvcc with sm_90a support). There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    c = ctypes
    vp, i32, i64 = c.c_void_p, c.c_int, c.c_int64
    lib.smapb_create.argtypes = [c.POINTER(vp), i32, i32, i32, i32]
    lib.smapb_create.restype = i32
    lib.smapb_destroy.argtypes = [vp]
    lib.smapb_destroy.restype = None
    lib.smapb_last_error.argtypes = [vp]
    lib.smapb_last_error.restype = c.c_char_p
    lib.smapb_version.restype = i32
    lib.smapb_load_weight.argtypes = [vp, c.c_char_p, vp, c.POINTER(i64), i32]
    lib.smapb_finalize_weights.argtypes = [vp, i32]
    lib.smapb_backbone_forward.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    lib.smapb_merge_scale.argtypes = [vp, vp, vp, i32, i32, vp]
    lib.smapb_assoc_extract.argtypes = [vp, vp, i32, vp, vp, vp]
    lib.smapb_assoc_connect.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp]
    lib.smapb_lift3d.argtypes = [vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp]
    lib.smapb_lift3d_gt.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.smapb_infer_device.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.smapb_infer_host.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.smapb_submit_host.argtypes = [vp, i32, vp, vp, i32, i32, vp]
    lib.smapb_wait.argtypes = [vp, i32]
    lib.smapb_launch_count.argtypes = [vp]
    lib.smapb_launch_count.restype = i64
    lib.smapb_saturation_count.argtypes = [vp, i32]
    lib.smapb_saturation_count.restype = i64
    lib.smapb_profile_begin.argtypes = [vp]
    lib.smapb_profile_end.argtypes = [vp, c.POINTER(c.c_double), c.POINTER(i32), c.c_char_p]
    lib.smapb_plan_info.argtypes = [vp, i32, c.POINTER(i32), c.POINTER(c.c_double)]
    lib.smapb_conv_test.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp] + [i32] * 14 + [vp, c.POINTER(i32),
                                                                                       c.POINTER(c.c_float), vp]
    lib.smapb_refine_load_weight.argtypes = [vp, c.c_char_p, vp, c.POINTER(i64), i32]
    lib.smapb_refine_finalize.argtypes = [vp]
    lib.smapb_refine_mlp.argtypes = [vp, vp, i32, vp, vp]
    lib.smapb_refine3d.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.smapb_set_refine.argtypes = [vp, i32]
    lib.smapb_preprocess.argtypes = [vp, vp, i32, i32, vp, c.POINTER(c.c_double), vp]
    lib.smapb_preprocess_host.argtypes = [vp, vp, i32, i32, vp, c.POINTER(c.c_double), vp]
    lib.smapb_comm_unique_id.argtypes = [vp]
    lib.smapb_comm_create.argtypes = [vp, vp, i32, i32]
    lib.smapb_comm_attach.argtypes = [vp, vp, i32, i32]
    lib.smapb_allgather_records.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.smapb_infer_device_gather.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.smapb_submit_host_gather.argtypes = [vp, i32, vp, vp, i32, i32, vp]
    lib.smapb_infer_device_gather_async.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    lib.smapb_gather_sync.argtypes = [vp, vp]
    lib.smapb_jpeg_info.argtypes = [c.c_char_p, i64, c.POINTER(i32), c.POINTER(i32), c.POINTER(i32), c.POINTER(i32)]
    lib.smapb_decode_jpeg.argtypes = [vp, i32, c.POINTER(c.c_char_p), c.POINTER(i64), c.POINTER(vp), c.POINTER(i32), vp]
    lib.smapb_jpeg_info_ex.argtypes = [c.c_char_p, i64, i32, c.POINTER(i32), c.POINTER(i32), c.POINTER(i32), c.POINTER(i32)]
    lib.smapb_decode_jpeg_ex.argtypes = [vp, i32, c.POINTER(c.c_char_p), c.POINTER(i64), c.POINTER(vp), i32, c.POINTER(i32), vp]
    lib.smapb_png_info.argtypes = [c.c_char_p, i64, c.POINTER(i32), c.POINTER(i32), c.POINTER(i32), c.POINTER(i32)]
    lib.smapb_decode_png.argtypes = [vp, i32, c.POINTER(c.c_char_p), c.POINTER(i64), c.POINTER(vp), c.POINTER(i32), vp]
    lib.smapb_png_inflate_stats.argtypes = [vp, c.POINTER(i64)]  # include/smap_b200_debug.h
    lib.smapb_set_tile_table.argtypes = [c.c_char_p]
    lib.smapb_get_tile_table.argtypes = [c.c_char_p, i32]
    lib.smapb_json_open.argtypes = [c.POINTER(vp), c.c_char_p, c.c_char_p]
    lib.smapb_json_append.argtypes = [vp, vp, i32, c.POINTER(c.c_char_p)]
    lib.smapb_json_close.argtypes = [vp]
    for name in EXPORTS:
        fn = getattr(lib, name)
        if fn.restype is c.c_int and name not in ("smapb_version",):
            fn.restype = i32
    _lib = lib
    return lib
