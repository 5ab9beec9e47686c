"""ctypes binding of libdprb.so (C ABI declared in include/dprb.h).

The product path has NO CPU or eager fallback: if the shared library is missing or a call fails the
error is raised immediately (``DprbError``).  Build with ``python __graft_entry__.py`` or
``make -C dpr_scale_b200/csrc``.
"""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p, POINTER, Structure

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libdprb.so")


class DprbError(RuntimeError):
    pass


class EncoderWeights(Structure):
    """Mirror of ``dprb_encoder_weights`` (include/dprb.h)."""
    _fields_ = [
        ("hidden", c_int32), ("inter", c_int32), ("layers", c_int32), ("heads", c_int32),
        ("vocab", c_int32), ("max_pos", c_int32), ("type_vocab", c_int32), ("ln_eps", c_float),
        ("master", c_void_p), ("shadow", c_void_p), ("grads", c_void_p),
        ("off_word", c_int64), ("off_pos", c_int64), ("off_type", c_int64),
        ("off_emb_ln_g", c_int64), ("off_emb_ln_b", c_int64),
        ("off_layer0", c_int64), ("layer_stride", c_int64),
        ("rel_wqkv", c_int64), ("rel_bqkv", c_int64), ("rel_wo", c_int64), ("rel_bo", c_int64),
        ("rel_ln1_g", c_int64), ("rel_ln1_b", c_int64), ("rel_w1", c_int64), ("rel_b1", c_int64),
        ("rel_w2", c_int64), ("rel_b2", c_int64), ("rel_ln2_g", c_int64), ("rel_ln2_b", c_int64),
    ]


class EncoderBatch(Structure):
    """Mirror of ``dprb_encoder_batch`` (include/dprb.h)."""
    _fields_ = [
        ("nseq", c_int32), ("S", c_int32),
        ("ids", c_void_p), ("type_ids", c_void_p), ("pos_ids", c_void_p), ("attn_mask", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_int64),
        ("save_for_backward", c_int32),
        ("dropout_p", c_float),
        ("dropout_seed", c_uint64),
    ]


_P = c_void_p
# name -> (restype, argtypes); must list EVERY symbol include/dprb.h declares (tests check this).
SIGNATURES = {
    "dprb_version": (c_int, []),
    "dprb_last_error": (c_char_p, []),
    "dprb_num_sms": (c_int, []),
    "dprb_launch_count": (c_int64, []),
    "dprb_gemm_bf16": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int, c_int, c_int,
                               _P, _P, c_int64, _P, c_float, c_int, _P, c_float, c_uint64, _P]),
    "dprb_gemm_profile_enable": (c_int, [c_int, c_int]),
    "dprb_gemm_profile_read": (c_int, [POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(c_int64)]),
    "dprb_embed_ln_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                  c_float, c_float, c_uint64, _P, _P]),
    "dprb_embed_ln_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_float,
                                  c_uint64, _P]),
    "dprb_dropout_site_seed": (c_uint64, [c_uint64, c_int, c_int]),
    "dprb_dropout_mask": (c_int, [_P, c_int64, c_int, c_float, c_uint64, c_int, c_int, _P]),
    "dprb_ln_fwd": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_float, c_int, _P, _P]),
    "dprb_ln_bwd": (c_int, [_P, _P, c_int, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, _P, c_float, c_uint64, c_int,
                            _P]),
    "dprb_gelu_from_pre": (c_int, [_P, _P, c_int64, _P]),
    "dprb_colsum_bf16": (c_int, [_P, c_int64, _P, c_int, c_int, _P]),
    "dprb_attn_fwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_uint64, _P]),
    "dprb_attn_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_float, c_uint64, _P]),
    "dprb_attn_cls_fwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_uint64, _P]),
    "dprb_attn_cls_bwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_uint64, _P]),
    "dprb_score_tc_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int, c_int]),
    "dprb_score_tc_fwd": (c_int, [_P, _P, _P, _P, _P, c_float, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, c_int64,
                                  _P]),
    "dprb_score_tc_bwd": (c_int, [_P, _P, _P, _P, c_float, c_float, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_int, _P, c_int64, _P]),
    "dprb_sumsq_f32": (c_int, [_P, c_int64, _P, _P]),
    "dprb_adamw_step": (c_int, [_P, _P, _P, _P, _P, c_int64, c_float, c_float, c_float, c_float, c_float, c_int,
                                c_float, _P, c_float, _P]),
    "dprb_lamb_workspace_bytes": (c_int64, [c_int, c_int]),
    "dprb_lamb_step": (c_int, [_P, _P, _P, _P, _P, c_int64, _P, c_int, c_int, c_float, c_float, c_float, c_float,
                               c_float, c_float, c_int, c_int, c_int, c_float, _P, c_float, _P, c_int64, _P]),
    "dprb_madgrad_step": (c_int, [_P, _P, _P, _P, _P, _P, c_int64, c_float, c_float, c_float, c_float, c_int, c_float,
                                  _P, c_float, _P]),
    "dprb_cast_f32_bf16": (c_int, [_P, _P, c_int64, _P]),
    "dprb_cast_bf16_f32": (c_int, [_P, _P, c_int64, _P]),
    "dprb_encoder_workspace_bytes": (c_int64, [POINTER(EncoderWeights), c_int, c_int, c_int]),
    "dprb_encoder_fwd": (c_int, [POINTER(EncoderWeights), POINTER(EncoderBatch), _P, _P]),
    "dprb_encoder_bwd": (c_int, [POINTER(EncoderWeights), POINTER(EncoderBatch), _P, c_int, c_int, _P]),
    "dprb_encoder_fwd_tokens": (c_int, [POINTER(EncoderWeights), POINTER(EncoderBatch), _P, _P]),
    "dprb_maxsim_fwd": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "dprb_maxsim_expert_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                       c_int, c_int, c_int, _P, _P]),
    "dprb_splade_pool_fwd": (c_int, [_P, c_int64, _P, c_int64, _P, _P, c_int64, c_int, c_int, c_int, _P, c_int64, _P]),
    "dprb_expert_group_workspace_bytes": (c_int64, [c_int, c_int, c_int]),
    "dprb_expert_group": (c_int, [_P, _P, _P, _P, _P, c_int64, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P,
                                  _P, _P, _P, _P, _P, c_int64, _P]),
    "dprb_seqcls_head_fwd": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "dprb_seqcls_group_ce_workspace_bytes": (c_int64, [c_int, c_int]),
    "dprb_seqcls_group_ce": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_uint64, _P, _P, _P, _P, _P, _P,
                                     c_int64, _P]),
    "dprb_search_workspace_bytes": (c_int64, [c_int64, c_int]),
    "dprb_search_topk": (c_int, [_P, _P, c_int, c_int64, c_int64, c_int, c_int, c_int64, _P, _P, _P, c_int64, _P]),
    "dprb_topk_merge_workspace_bytes": (c_int64, [c_int64, c_int]),
    "dprb_topk_merge": (c_int, [_P, _P, c_int64, c_int, c_int, _P, _P, _P, c_int64, _P]),
    "dprb_expert_search_block_queries": (c_int, [c_int64]),
    "dprb_expert_search_workspace_bytes": (c_int64, [c_int64, c_int]),
    "dprb_expert_search": (c_int, [_P, _P, _P, c_int64, c_int, c_int, c_int, _P, c_int, c_int, _P, c_int64, _P, _P,
                                   c_int64, _P, c_int, _P, _P, c_int, c_int, c_int, _P, _P, _P, c_int64, _P]),
    "dprb_sparse_search_block_queries": (c_int, [c_int64]),
    "dprb_sparse_search_workspace_bytes": (c_int64, [c_int64, c_int]),
    "dprb_sparse_search": (c_int, [_P, _P, _P, c_int64, c_int, _P, c_int64, _P, _P, _P, _P, c_int, c_int, c_int, c_int,
                                   _P, _P, _P, c_int64, _P]),
    "dprb_sqerr_workspace_bytes": (c_int64, [c_int, c_int]),
    "dprb_sqerr_fwd": (c_int, [_P, c_int64, _P, c_int64, c_int, c_int, _P, _P, c_int64, _P, c_int64, _P]),
}

_lib = None


def load():
    """Load libdprb.so once; raise DprbError (never fall back) if it is missing or incomplete."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DprbError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python __graft_entry__.py` "
            "(or `make -C dpr_scale_b200/csrc`). There is no CPU fallback."
        )
    # PyDLL: keep the GIL across the calls.  Every entry point only enqueues kernels (microseconds); releasing and
    # re-taking the GIL ~10 times per step would make the training thread queue behind the input-pipeline thread
    # (datamodule/dpr.py) for up to a switch interval each time.
    lib = ctypes.PyDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise DprbError(f"libdprb.so does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().dprb_last_error()
        raise DprbError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
