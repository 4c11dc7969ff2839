"""ctypes binding of libvcb200.so (C ABI declared in include/vcb200.h).

The shared library is built in-tree by ``__graft_entry__.build()`` / ``make -C voicecraft_b200/csrc``.
There is deliberately no fallback: if the library is missing or no sm_90 GPU is present, loading or
``vcb_create`` fails loudly (the product path never routes through a CPU implementation).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VCB_LIB") or os.path.join(_HERE, "libvcb200.so")   # VCB_LIB: A/B runs of two builds


class VcbError(RuntimeError):
    pass


class vcb_config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "d_model", "nhead", "num_layers", "n_codebooks", "audio_vocab_size", "n_special", "text_vocab_rows",
        "empty_token", "eog", "audio_pad_token", "eos", "encodec_sr", "max_n_spans", "max_slots", "max_seq_len",
        "max_new_tokens", "kv_dtype", "device", "weight_dtype", "align_text_cap")] + [("kv_pool_bytes", C.c_int64)]


VCB_ERR_KV_FULL = -3        # vcb_decode_step: the KV pool cannot cover the listed slots' next positions; nothing was done
KV_GROW_PAGES = 4           # pages a one-copy utterance's page list grows by (VCB_KV_GROW_PAGES)
ALIGN_MAX_TEXT = 4096       # largest align_text_cap and vcb_align_monotonic X (VCB_ALIGN_MAX_TEXT)


class vcb_sampling(C.Structure):
    _fields_ = [("top_k", C.c_int32), ("top_p", C.c_float), ("temperature", C.c_float),
                ("stop_repetition", C.c_int32), ("n_silence", C.c_int32), ("silence_tokens", C.c_int32 * 8),
                ("ras_window", C.c_int32), ("ras_threshold", C.c_int32), ("min_frames", C.c_int32), ("max_frames", C.c_int32)]


class vcb_prompt(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_copies", C.c_int32), ("mode", C.c_int32), ("x_len", C.c_int32),
                ("text_ids_dev", C.c_void_p), ("y_len", C.c_int32), ("y_tokens_dev", C.c_void_p),
                ("mask_rows_dev", C.c_void_p), ("n_more_spans", C.c_int32), ("more_mask_rows", C.c_int32 * 8),
                ("rng_seed", C.c_uint64), ("rng_offset", C.c_uint64), ("rng_threads", C.c_int32), ("rng_reserved", C.c_int32),
                ("sampling", C.POINTER(vcb_sampling)), ("align_heads", C.POINTER(C.c_uint32))]


class vcb_edit_source(C.Structure):
    _fields_ = [("orig_dev", C.c_void_p), ("T", C.c_int32), ("n_spans", C.c_int32), ("spans", (C.c_int32 * 2) * 8)]


class vcb_status(C.Structure):
    _fields_ = [("done", C.c_int32), ("forced", C.c_int32), ("n_steps", C.c_int32), ("keep", C.c_int32),
                ("n_spans_done", C.c_int32), ("span_ends", C.c_int32 * 8), ("reserved", C.c_int32),
                ("rng_offset", C.c_uint64)]


# every symbol include/vcb200.h (and include/vcb200_codec.h) declares, with its prototype
PROTOTYPES = {
    "vcb_last_error": (C.c_char_p, []),
    "vcb_version": (C.c_int, []),
    "vcb_create": (C.c_int, [C.POINTER(vcb_config), C.POINTER(C.c_void_p)]),
    "vcb_destroy": (C.c_int, [C.c_void_p]),
    "vcb_load_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.c_int32]),
    "vcb_load_pe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "vcb_finalize_weights": (C.c_int, [C.c_void_p]),
    "vcb_prefill": (C.c_int, [C.c_void_p, C.POINTER(vcb_prompt), C.c_int32, C.c_void_p]),
    "vcb_sample": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.POINTER(vcb_sampling), C.c_void_p]),
    "vcb_decode_step": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.POINTER(vcb_sampling), C.c_void_p]),
    "vcb_poll": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(vcb_status), C.c_void_p]),
    "vcb_poll_frames": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int64,
                                  C.c_int64, C.c_void_p, C.POINTER(vcb_status), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                  C.c_void_p]),
    "vcb_poll_frames_ex": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(vcb_edit_source),
                                     C.POINTER(C.c_int32), C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.POINTER(vcb_status),
                                     C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p]),
    "vcb_read_tokens": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_void_p]),
    "vcb_read_logprobs": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_void_p]),
    "vcb_read_alignment": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_align_monotonic": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vcb_debug_align_probe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_uint32, C.c_int32, C.c_void_p]),
    "vcb_release": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "vcb_swap_out": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.c_void_p]),
    "vcb_swap_in": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vcb_snapshot_pages": (C.c_int32, [C.c_void_p]),
    "vcb_snapshot_free": (C.c_int, [C.c_void_p]),
    "vcb_debug_logits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "vcb_debug_exponential": (C.c_int, [C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, C.c_int32, C.c_void_p]),
    "vcb_debug_sampler": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int32, C.POINTER(vcb_sampling)] +
                          [C.c_int32] * 7 + [C.POINTER(C.c_int32)] * 3),
    "vcb_debug_sampler_lp": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int32, C.POINTER(vcb_sampling)] +
                             [C.c_int32] * 7 + [C.POINTER(C.c_int32)] * 3 + [C.POINTER(C.c_float)]),
    "vcb_debug_sampler_ras": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int32,
                                        C.POINTER(vcb_sampling)] + [C.c_int32] * 7 + [C.POINTER(C.c_int32)] * 4 +
                              [C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
    "vcb_debug_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_debug_weight_quantize": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vcb_debug_gemm_w8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_debug_gemm_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "vcb_debug_attention": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 4 + [C.c_int32] * 7 + [C.c_void_p]),
    "vcb_debug_attention_groups": (C.c_int, [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 2 + [C.c_int32] * 7 +
                                   [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32]),
    "vcb_debug_mega_attention": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] + [C.c_void_p] * 2 + [C.c_int32] * 3 +
                                 [C.POINTER(C.c_int32), C.c_int32, C.c_void_p]),
    "vcb_debug_kv_quantize": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "vcb_debug_kv_pages": (C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 2),
    "vcb_debug_stage_read": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int32]),
    "vcb_debug_fold_chain": (C.c_int, [C.c_void_p] * 8 + [C.c_int32] * 7 + [C.c_void_p] * 2),
    "vcb_timeline": (C.c_int, [C.c_int32, C.POINTER(C.c_uint64), C.c_int32, C.POINTER(C.c_int32)]),
    "vcb_bench_gemm": (C.c_int, [C.c_int32] * 8 + [C.POINTER(C.c_float)]),
    "vcb_gemm_launch_shape": (C.c_int, [C.c_int32] * 6 + [C.POINTER(C.c_int32)]),
    "vcb_mega_ring_config": (C.c_int, [C.c_int32] * 3 + [C.POINTER(C.c_int32)]),
    "vcb_debug_mega_timeline": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int32, C.POINTER(C.c_int32)]),
    "vcb_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int32]),
    "vcb_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int32]),
    "vcb_counter": (C.c_int64, [C.c_void_p, C.c_char_p]),
    "vcb_delay_pattern": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_void_p]),
}

_lib = None


def load():
    """dlopen libvcb200.so and attach prototypes.  Raises VcbError if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VcbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU / PyTorch fallback for the hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    try:
        from . import _codec_lib
        _codec_lib.attach(lib)
    except ImportError:
        pass
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise VcbError((load().vcb_last_error() or b"unknown error").decode())
