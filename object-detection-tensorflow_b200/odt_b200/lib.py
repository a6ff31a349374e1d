"""ctypes binding of libodt_b200.so (the C ABI declared in include/odt_b200.h).

The product path has no CPU fallback: if the CUDA extension is missing the
import fails loudly (build it with `python __graft_entry__.py`).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libodt_b200.so")

ODT_F16, ODT_F32 = 0, 1
ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2
DECODE_SSD, DECODE_YOLO3, DECODE_FCOS = 0, 1, 2
MAX_LEVELS, MAX_PRIORS = 8, 9
ERR_OVERFLOW = -4
ERR_UNSUPPORTED = -3
ABI_VERSION = 5  # odt_abi_version(): bumped whenever a signature in include/odt_b200.h changes


class ConvParams(C.Structure):
    """Mirror of odt_conv_params."""
    _fields_ = [
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("in_ld", C.c_int),
        ("OH", C.c_int), ("OW", C.c_int), ("Cout", C.c_int),
        ("R", C.c_int), ("S", C.c_int), ("stride", C.c_int), ("dil", C.c_int),
        ("pad_t", C.c_int), ("pad_l", C.c_int),
        ("w_ld", C.c_int), ("Cout_pad", C.c_int),
        ("scale", C.c_void_p), ("shift", C.c_void_p), ("act", C.c_int),
        ("residual", C.c_void_p), ("out0", C.c_void_p), ("out0_dtype", C.c_int),
        ("out0_img_stride", C.c_longlong), ("out0_pix_stride", C.c_int),
        ("out0_group", C.c_int), ("out0_group_stride", C.c_int),
        ("scale2", C.c_void_p), ("shift2", C.c_void_p), ("act2", C.c_int),
        ("out1", C.c_void_p), ("out1_img_stride", C.c_longlong), ("out1_pix_stride", C.c_int),
        ("scale3", C.c_void_p), ("shift3", C.c_void_p), ("act3", C.c_int),
        ("out2", C.c_void_p), ("out2_img_stride", C.c_longlong), ("out2_pix_stride", C.c_int),
        ("in_halo", C.c_int), ("out0_halo", C.c_int), ("out0_pool", C.c_int),
        ("out1_halo", C.c_int), ("out2_halo", C.c_int),
    ]


class Level(C.Structure):
    """Mirror of odt_level."""
    _fields_ = [
        ("H", C.c_int), ("W", C.c_int), ("A", C.c_int), ("offset", C.c_int),
        ("cmul_y", C.c_float), ("cdiv_y", C.c_float), ("cmul_x", C.c_float), ("cdiv_x", C.c_float),
        ("out_mul", C.c_float),
        ("prior_h", C.c_float * MAX_PRIORS), ("prior_w", C.c_float * MAX_PRIORS),
    ]


class TailParams(C.Structure):
    """Mirror of odt_tail_params."""
    _fields_ = [
        ("kind", C.c_int), ("num_levels", C.c_int), ("N", C.c_int), ("num_fg", C.c_int),
        ("nms_classes", C.c_int), ("score_thr", C.c_float), ("iou_thr", C.c_float),
        ("max_boxes", C.c_int), ("cap", C.c_int),
        ("level", Level * MAX_LEVELS),
    ]


# every symbol include/odt_b200.h declares: name -> (restype, argtypes)
_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_longlong, C.c_float
SYMBOLS = {
    "odt_abi_version": (_I, []),
    "odt_crc32c": (C.c_uint, [C.c_uint, _P, C.c_ulonglong]),
    "odt_last_error": (C.c_char_p, []),
    "odt_same_pad": (_I, [_I, _I, _I, _I, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "odt_normalize_input": (_I, [_P, _P, _I, _I, _I, _I, _I, C.POINTER(_F), _P]),
    "odt_conv2d_f16_tc": (_I, [_P, _P, C.POINTER(ConvParams), _P]),
    "odt_conv_tc_pick_bn": (_I, [_I, _L, _I]),
    "odt_conv_tc_swap_plan": (_I, [C.POINTER(ConvParams), C.POINTER(_I), C.POINTER(_L), C.POINTER(_I)]),
    "odt_conv2d_direct": (_I, [_P, _P, _I, C.POINTER(ConvParams), _P]),
    "odt_conv2d_stem": (_I, [_P, C.POINTER(_F), _P, _I, C.POINTER(ConvParams), _P]),
    "odt_pack_input_rgbx": (_I, [_P, _P, _I, _I, _I, _I, C.POINTER(_F), _P]),
    "odt_conv2d_stem_rgbx": (_I, [_P, _P, C.POINTER(ConvParams), _P]),
    "odt_maxpool": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "odt_maxpool_affine": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _I, _P, _P, _I, _P, _I, _P]),
    "odt_l2norm_scale": (_I, [_P, _P, _I, _L, _I, _I, _F, _P]),
    "odt_affine_act": (_I, [_P, _P, _I, _L, _I, _I, _P, _P, _I, _P]),
    "odt_upsample_bilinear_add": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P]),
    "odt_upsample_nearest_concat": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "odt_groupnorm_stats": (_I, [_P, _P, _I, _I, _L, _I, _I, _I, _F, _P]),
    "odt_groupnorm_apply": (_I, [_P, _P, _P, _I, _I, _L, _I, _I, _I, _P, _P, _I, _P]),
    "odt_groupnorm_act_workspace_bytes": (_L, [_I, _I, _L, _I, _I]),
    "odt_groupnorm_act": (_I, [_P, _P, _P, _I, _I, _L, _I, _I, _I, _F, _P, _P, _I, _P]),
    "odt_decode_candidates": (_I, [_P, C.POINTER(TailParams), _I, _P, _P, _P]),
    "odt_nms_per_class": (_I, [_P, C.POINTER(TailParams), _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _L, _L, _P]),
    "odt_nms_scratch_bytes": (_L, [C.POINTER(TailParams), _I]),
    "odt_retina_loss_scratch_bytes": (_L, [C.POINTER(TailParams), _I]),
    "odt_retina_loss_fwd": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _F, _F, _P, _P, _P]),
    "odt_ssd_loss_scratch_bytes": (_L, [C.POINTER(TailParams), _I]),
    "odt_ssd_loss_fwd": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _P, _P, _P, _P]),
    "odt_yolo_loss_scratch_bytes": (_L, [C.POINTER(TailParams), _I]),
    "odt_yolo_loss_fwd": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _F, _F, _F, _F, _P, _P, _P]),
    "odt_fcos_loss_scratch_bytes": (_L, [C.POINTER(TailParams), _I]),
    "odt_fcos_loss_fwd": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _P, _P, _P]),
    "odt_retina_loss_grad": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _F, _F, _P, _P, _P, _P]),
    "odt_ssd_loss_grad": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _P, _P, _P, _P, _P]),
    "odt_yolo_loss_grad": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _F, _F, _F, _F, _P, _P, _P, _P]),
    "odt_fcos_loss_grad": (_I, [_P, C.POINTER(TailParams), _I, _P, _I, _P, _P, _P, _P]),
    "odt_pool_classify": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "odt_ctx_unique_id": (_I, [_P]),
    "odt_ctx_create": (_I, [C.POINTER(_P), _I, _I, _P]),
    "odt_ctx_destroy": (_I, [_P]),
    "odt_allgather_dets": (_I, [_P, _P, _P, _L, _P]),
    "odt_bcast_weights": (_I, [_P, _P, _L, _I, _P]),
}


class OdtError(RuntimeError):
    pass


_lib = None


def load():
    """Load the shared library and type every entry point.  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise OdtError(
            "CUDA extension %s is missing: build it (python __graft_entry__.py); "
            "there is no CPU fallback on the product path" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.odt_abi_version() != ABI_VERSION:
        raise OdtError("%s has ABI version %d, this binding expects %d: rebuild it (python __graft_entry__.py)"
                       % (LIB_PATH, lib.odt_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().odt_last_error()
        raise OdtError("%s failed (%d): %s" % (what, rc, msg.decode() if msg else ""))


def same_pad(size, k, stride, dil=1):
    out, pb, pa = C.c_int(), C.c_int(), C.c_int()
    check(load().odt_same_pad(size, k, stride, dil, C.byref(out), C.byref(pb), C.byref(pa)),
          "odt_same_pad")
    return out.value, pb.value, pa.value
