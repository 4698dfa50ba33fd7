"""ctypes binding of libvlpk.so (C ABI declared in include/vlpk.h).

The library is the product; this module only marshals raw device pointers, sizes and the current
CUDA stream across the C boundary.  There is no fallback path: if the shared library is missing or a
call fails, a RuntimeError is raised (SURVEY.md §8b "Error convention").
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvlpk.so")

c_void_p, c_int, c_i64, c_u64, c_float = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.c_float


class VlpkDropout(C.Structure):
    _fields_ = [("p", c_float), ("seed", c_u64), ("seed_dev", c_void_p)]


class VlpkShape(C.Structure):
    # kv_slots: 0 = the 128-slot layout (Lq, Lkv <= 128); else 128 * ceil(Lkv / 128), see ops.kv_slots.  Left at 0 by the six-field form.
    _fields_ = [("B", C.c_int32), ("Lq", C.c_int32), ("Lkv", C.c_int32), ("H", C.c_int32), ("heads", C.c_int32),
                ("I", C.c_int32), ("kv_slots", C.c_int32)]


WEIGHT_FIELDS = ["wq", "wk", "wv", "bq", "bk", "bv", "wo", "bo", "ln1_g", "ln1_b", "w1", "b1", "w2", "b2", "ln2_g", "ln2_b"]
GRAD_FIELDS = ["wqkv", "bqkv", "wo", "bo", "ln1_g", "ln1_b", "w1", "b1", "w2", "b2", "ln2_g", "ln2_b"]
ACT_FIELDS = ["qkv", "ctx", "t1", "y1", "u", "hmid", "t2", "y", "lse", "stats1", "stats2", "kv", "drop_attn"]
SCRATCH_FIELDS = ["dz2", "dt2", "du", "dy1", "dz1", "dt1", "dctx", "dqkv", "dx"]


class VlpkLayerWeights(C.Structure):
    _fields_ = [(n, c_void_p) for n in WEIGHT_FIELDS]


class VlpkLayerGrads(C.Structure):
    _fields_ = [(n, c_void_p) for n in GRAD_FIELDS]


class VlpkLayerActs(C.Structure):
    _fields_ = [(n, c_void_p) for n in ACT_FIELDS]


class VlpkBwdScratch(C.Structure):
    _fields_ = [(n, c_void_p) for n in SCRATCH_FIELDS]


class VlpkAdamTensor(C.Structure):
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("master", c_void_p), ("m", c_void_p), ("v", c_void_p), ("n", c_i64),
                ("weight_decay", c_float), ("param_dtype", C.c_int32), ("grad_dtype", C.c_int32), ("reserved", C.c_int32)]


class VlpkConstrainedBeamArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("B", "K", "C", "A", "P", "f", "V")] + [("logits", c_void_p), ("ld", c_i64), ("bias", c_void_p)] \
        + [(n, C.c_int32) for n in ("fp32", "eos_id", "block_eos", "T_cap", "n")] \
        + [("hist_in", c_void_p), ("hist_out", c_void_p), ("ignore", c_void_p), ("n_ignore", C.c_int32)] \
        + [(n, c_void_p) for n in ("cons", "prev_wid", "prev_ptr", "prev_score", "prev_eos", "top_w", "top_lp", "top_dest", "wid", "ptr",
                                   "score", "eos")]


class VlpkPromptRows(C.Structure):
    _fields_ = [("hist_off", C.c_int32), ("eos_until", c_void_p)]


# name -> (restype, argtypes); mirrors include/vlpk.h one to one
_P = c_void_p
_SIGS = {
    "vlpk_version": (c_int, []),
    "vlpk_last_error": (C.c_char_p, []),
    "vlpk_debug_set_option": (c_int, [C.c_char_p, c_int]),
    "vlpk_set_reserved_sms": (None, [c_int]),
    "vlpk_set_deterministic": (None, [c_int]),
    "vlpk_debug_plan_gemm": (c_int, [c_int] * 10 + [C.POINTER(c_int)]),
    "vlpk_mask_pack": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_i64, c_i64, _P, _P]),
    "vlpk_mask_synth": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "vlpk_mask_synth_grouped": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P]),
    "vlpk_linear_fwd": (c_int, [c_int, c_int, c_int, _P, c_i64, _P, c_i64, _P, _P, c_i64, c_int, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_linear_bwd": (c_int, [c_int, c_int, c_int, _P, c_i64, _P, c_i64, _P, c_i64, _P, c_i64, _P, _P, c_i64, _P, c_i64, _P,
                                c_int, c_float, _P]),
    "vlpk_embed_fwd": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                               C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_embed_bwd": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                               C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_embed_tables_bwd": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    "vlpk_ln_res_drop_fwd": (c_int, [c_i64, c_int, _P, _P, _P, _P, _P, _P, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_ln_res_drop_bwd": (c_int, [c_i64, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_attn_core_fwd": (c_int, [c_int, c_int, c_int, c_int, _P, c_i64, _P, _P, c_i64, _P, c_int, _P, c_i64, _P,
                                   C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_attn_core_bwd": (c_int, [c_int, c_int, c_int, _P, _P, _P, c_i64, _P, c_int, _P, _P, c_i64, _P, _P, _P, _P, c_i64,
                                   C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_attn_core_fwd_wide": (c_int, [c_int, c_int, c_int, c_int, _P, c_i64, _P, _P, c_i64, _P, c_int, _P, c_i64, _P,
                                        C.POINTER(VlpkDropout), c_u64, c_int, _P]),
    "vlpk_attn_core_bwd_wide": (c_int, [c_int, c_int, c_int, _P, _P, _P, c_i64, _P, c_int, _P, _P, c_i64, _P, _P, _P, _P, c_i64,
                                        C.POINTER(VlpkDropout), c_u64, c_int, _P]),
    "vlpk_attn_core_self_fwd": (c_int, [c_int, c_int, c_int, c_int, _P, c_i64, c_i64, _P, _P, c_i64, c_i64, _P, _P, _P, c_int, _P, c_i64,
                                        c_i64, _P, _P]),
    "vlpk_attn_core_group_self_fwd": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, _P, c_i64, c_i64, _P, c_int, c_i64, _P, c_int,
                                              c_i64, _P, _P, _P, c_int, _P, c_i64, c_i64, _P, _P]),
    "vlpk_attn_probs": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_i64, c_i64, _P, c_i64, c_i64, _P, c_int, c_int, _P, _P, c_i64,
                                c_i64, _P]),
    "vlpk_mha_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, _P, c_int, C.POINTER(VlpkLayerActs),
                             c_float, c_float, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_ffn_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), C.POINTER(VlpkLayerActs), c_float,
                             C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_layer_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, _P, c_int, C.POINTER(VlpkLayerActs),
                               c_float, c_float, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_layer_bwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, c_int, C.POINTER(VlpkLayerActs), _P, _P,
                               C.POINTER(VlpkLayerGrads), C.POINTER(VlpkBwdScratch), c_float, c_float, C.POINTER(VlpkDropout),
                               c_u64, _P]),
    "vlpk_ffn_bwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), C.POINTER(VlpkLayerActs), _P, _P,
                             C.POINTER(VlpkLayerGrads), C.POINTER(VlpkBwdScratch), c_float, C.POINTER(VlpkDropout), c_u64, _P]),
    "vlpk_mha_bwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, c_int, C.POINTER(VlpkLayerActs), _P, _P,
                             C.POINTER(VlpkLayerGrads), C.POINTER(VlpkBwdScratch), c_float, c_float, C.POINTER(VlpkDropout),
                             c_u64, _P]),
    "vlpk_mha_incr_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, _P, c_int,
                                  C.POINTER(VlpkLayerActs), c_u64, _P]),
    "vlpk_layer_cached_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, c_int, c_int, _P, c_int,
                                      C.POINTER(VlpkLayerActs), c_u64, _P]),
    "vlpk_layer_cached_group_fwd": (c_int, [C.POINTER(VlpkShape), C.POINTER(VlpkLayerWeights), _P, _P, c_int, c_int, _P, c_int, _P, c_int,
                                            c_int, _P, c_int, C.POINTER(VlpkLayerActs), c_u64, _P]),
    "vlpk_workspace_bytes": (c_int, [C.POINTER(VlpkShape), C.POINTER(C.c_size_t)]),
    "vlpk_encoder_fwd": (c_int, [C.POINTER(VlpkShape), c_int, C.POINTER(VlpkLayerWeights), _P, _P, c_int,
                                 C.POINTER(VlpkLayerActs), c_float, c_float, C.POINTER(VlpkDropout), _P]),
    "vlpk_encoder_score_fwd": (c_int, [C.POINTER(VlpkShape), c_int, c_int, C.POINTER(VlpkLayerWeights), _P, _P, _P, C.POINTER(VlpkLayerActs),
                                       _P]),
    "vlpk_encoder_score_workspace_bytes": (c_int, [C.POINTER(VlpkShape), c_int, C.POINTER(C.c_size_t)]),
    "vlpk_encoder_score_group_fwd": (c_int, [C.POINTER(VlpkShape), c_int, c_int, c_int, c_int, C.POINTER(VlpkLayerWeights), _P,
                                             C.POINTER(c_void_p), c_int, _P, _P, C.POINTER(VlpkLayerActs), _P]),
    "vlpk_encoder_score_group_workspace_bytes": (c_int, [C.POINTER(VlpkShape), c_int, C.POINTER(C.c_size_t)]),
    "vlpk_encoder_bwd": (c_int, [C.POINTER(VlpkShape), c_int, C.POINTER(VlpkLayerWeights), _P, _P, c_int,
                                 C.POINTER(VlpkLayerActs), C.POINTER(c_void_p), _P, C.POINTER(VlpkLayerGrads),
                                 C.POINTER(VlpkBwdScratch), c_float, c_float, C.POINTER(VlpkDropout), _P]),
    "vlpk_decoder_ce_fwd": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlpk_decoder_ce_bwd": (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlpk_decoder_ce_ls_fwd": (c_int, [c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlpk_decoder_ce_ls_bwd": (c_int, [c_int, c_int, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlpk_bertadam_chunk": (c_int, []),
    "vlpk_bertadam_step": (c_int, [_P, _P, _P, _P, c_int, _P, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _P]),
    "vlpk_profile_enable": (None, [c_int]),
    "vlpk_profile_reset": (None, []),
    "vlpk_profile_get": (c_int, [c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(c_i64)]),
    "vlpk_launch_count": (c_i64, []),
    "vlpk_beam_ngram_block": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_int, _P, c_i64, c_int, _P]),
    "vlpk_sample_tokens": (c_int, [c_int, c_int, _P, c_i64, _P, c_int, c_int, c_int, c_float, c_u64, c_int, _P, c_int, _P, _P, _P, c_int,
                                   c_int, c_int, c_int, _P, c_int, _P]),
    "vlpk_diverse_beam_step": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_i64, _P, c_int, c_float, c_int, c_int, c_int, c_int, _P,
                                       _P, _P, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vlpk_constrained_beam_step": (c_int, [C.POINTER(VlpkConstrainedBeamArgs), _P]),
    "vlpk_sample_tokens_prompt": (c_int, [c_int, c_int, _P, c_i64, _P, c_int, c_int, c_int, c_float, c_u64, c_int, _P, c_int, _P, _P, _P,
                                          c_int, c_int, c_int, _P, c_int, C.POINTER(VlpkPromptRows), _P]),
    "vlpk_diverse_beam_step_prompt": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_i64, _P, c_int, c_float, c_int, c_int, c_int, _P,
                                              _P, _P, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(VlpkPromptRows), _P]),
    "vlpk_constrained_beam_step_prompt": (c_int, [C.POINTER(VlpkConstrainedBeamArgs), C.POINTER(VlpkPromptRows), _P]),
    "vlpk_f32_to_bf16": (c_int, [_P, _P, c_i64, _P]),
    "vlpk_colsum": (c_int, [_P, c_i64, c_i64, c_int, _P, _P]),
    "vlpk_debug_dropout_mask": (c_int, [C.POINTER(VlpkDropout), c_u64, c_i64, _P, _P]),
    "vlpk_add_bf16": (c_int, [_P, _P, _P, c_i64, _P]),
    "vlpk_gemm": (c_int, [c_int, c_int, c_int, c_int, _P, c_i64, c_int, _P, c_i64, _P, _P, c_i64, _P, c_i64, _P, c_i64, c_int,
                          c_int, c_int, _P]),
}
EXPORTED_SYMBOLS = tuple(_SIGS.keys())

_lib = None


def lib():
    """Load libvlpk.so (once).  Raises if it has not been built: there is no fallback implementation."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(vlp_b200 has no CPU / PyTorch fallback path)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().vlpk_last_error()
        raise RuntimeError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


# The library's deterministic mode as last sent (its default is off).  `call` follows torch.use_deterministic_algorithms: the
# switch is read before every library call and forwarded when it has changed since the last one.
_deterministic = False


def call(name, *args):
    global _deterministic
    det = torch.are_deterministic_algorithms_enabled()
    if det != _deterministic:
        invoke("vlpk_set_deterministic", int(det))
        _deterministic = det
    invoke(name, *args)


def invoke(name, *args):
    """One library call, no mode check; raises on a non-zero return code."""
    rc = getattr(lib(), name)(*args)
    if rc is not None:
        check(rc, name)
