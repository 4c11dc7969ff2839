"""ctypes prototypes of the EnCodec and resampler entry points (include/vcb200_codec.h)."""
import ctypes as C


class enc_config(C.Structure):
    _fields_ = [("n_q", C.c_int32), ("bins", C.c_int32), ("dimension", C.c_int32), ("n_filters", C.c_int32),
                ("n_ratios", C.c_int32), ("ratios", C.c_int32 * 8), ("kernel_size", C.c_int32),
                ("last_kernel_size", C.c_int32), ("residual_kernel_size", C.c_int32), ("dilation_base", C.c_int32),
                ("n_residual_layers", C.c_int32), ("compress", C.c_int32), ("lstm", C.c_int32), ("causal", C.c_int32),
                ("pad_reflect", C.c_int32), ("true_skip", C.c_int32), ("channels", C.c_int32),
                ("trim_right_ratio", C.c_float), ("device", C.c_int32)]


PROTOTYPES = {
    "enc_create": (C.c_int, [C.POINTER(enc_config), C.POINTER(C.c_void_p)]),
    "enc_destroy": (C.c_int, [C.c_void_p]),
    "enc_load_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.c_int32]),
    "enc_finalize": (C.c_int, [C.c_void_p]),
    "enc_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "enc_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "enc_encode_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p,
                                    C.POINTER(C.c_int32), C.c_void_p]),
    "enc_counter": (C.c_int64, [C.c_void_p, C.c_char_p]),
    "enc_debug_tensor": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int32)]),
    "enc_stream_create": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "enc_stream_destroy": (C.c_int, [C.c_void_p]),
    "enc_stream_reset": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]),
    "enc_stream_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "enc_resampler_create": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "enc_resampler_destroy": (C.c_int, [C.c_void_p]),
    "enc_resample": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                               C.POINTER(C.c_int32), C.c_void_p]),
    "enc_resampler_push": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                     C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]),
    "enc_resampler_reset": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]),
}


def attach(lib):
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
