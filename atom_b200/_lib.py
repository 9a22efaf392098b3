"""ctypes loader of libatom_b200.so (the C ABI declared in include/atom_b200.h).

There is no CPU path and no fallback: if the library is missing or a call fails, a RuntimeError is raised
(the reference's pybind module fails the same way at import, punica/ops/__init__.py:3).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libatom_b200.so")

_P, _I, _I64, _U32, _F = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint32, ctypes.c_float

_SIGNATURES = {
    "atom_version": (ctypes.c_int, []),
    "atom_last_error": (ctypes.c_char_p, []),
    "atom_scale_index": (_I, [_I]),
    "atom_scale_size": (_I, [_I]),
    "atom_reorder_fp16_i4": (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "atom_rmsnorm_fp16_i4": (_I, [_P, _P, _F, _P, _I, _I, _P, _P, _P, _P, _P]),
    "atom_add_rmsnorm_fp16_i4": (_I, [_P, _P, _P, _P, _F, _P, _I, _I, _P, _P, _P, _P, _P]),
    "atom_activate_fp16_i4": (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "atom_gemm_i4_o16": (_I, [_P] * 9 + [_I64, _I64, _I64, _U32, _P]),
    "atom_gemm_i4_o4": (_I, [_P] * 10 + [_I64, _I64, _I64, _U32, _P]),
    "atom_gemm_i4_qkv": (_I, [_P] * 13 + [_I64, _I64, _I64, _U32, _P]),
    "atom_gemm_i4_qkv_gqa": (_I, [_P] * 13 + [_I64, _I64, _I64, _I64, _U32, _P]),
    "atom_gemm_i4_gateup_act": (_I, [_P] * 12 + [_I64, _I64, _I64, _U32, _P]),
    "atom_gemm_set_trace": (_I, [_P]),
    "atom_set_pdl": (_I, [_I]),
    "atom_batch_decode_i4": (_I, [_P] * 7 + [_I] * 5 + [_P]),
    "atom_batch_decode_gqa_i4": (_I, [_P] * 7 + [_I] * 6 + [_F, _P]),
    "atom_batch_decode_split_gqa_i4": (_I, [_P] * 7 + [_I] * 6 + [_F, _I, _P]),
    "atom_decode_kv_split": (_I, [_I] * 4),
    "atom_batch_decode_shared_gqa_i4": (_I, [_P] * 7 + [_I] * 6 + [_F] + [_P] * 3 + [_I] * 2 + [_P] * 2 + [_I, _P]),
    "atom_decode_shared_chunks": (_I, [_I] * 5),
    "atom_batch_verify_gqa_i4": (_I, [_P] * 7 + [_I] * 7 + [_F] + [_P] * 2 + [_I, _P]),
    "atom_verify_chunks": (_I, [_I] * 3),
    "atom_prefill_attention_i4": (_I, [_P] * 11 + [_I] * 4 + [_P]),
    "atom_prefill_attention_gqa_i4": (_I, [_P] * 11 + [_I] * 5 + [_P]),
    "atom_prefill_attention_ctx_gqa_i4": (_I, [_P] * 11 + [_I] * 5 + [_P] * 5 + [_I] * 3 + [_P]),
    "atom_allreduce_push_f16": (_I, [_P] * 4 + [_I64, _I64, _I, _I, _P]),
    "atom_allreduce_state_words": (_I, []),
    "atom_gemm_i4_o16_push": (_I, [_P] * 10 + [_I64, _I, _I, _I64, _I64, _I64, _U32, _P]),
    "atom_reduce_add_rmsnorm_fp16_i4": (_I, [_P, _P, _I64, _I, _I, _P, _P, _P, _F, _P, _I, _I, _P, _P, _P, _P, _P]),
    "atom_append_kv_i4": (_I, [_P] * 9 + [_I] * 5 + [_P]),
    "atom_init_kv_i4": (_I, [_P] * 10 + [_I] * 6 + [_P]),
    "atom_moe_route_f16": (_I, [_P, _P, _F, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "atom_moe_plan": (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _P]),
    "atom_moe_gather_i4": (_I, [_P] * 4 + [_I, _I, _I, _P, _I] + [_P] * 5),
    "atom_gemm_i4_gateup_act_grouped": (_I, [_P] * 13 + [_I, _I, _I64, _I64, _I64, _I64, _P]),
    "atom_gemm_i4_o16_grouped": (_I, [_P] * 10 + [_I, _I, _I64, _I64, _I64, _I64, _P]),
    "atom_moe_combine_f16": (_I, [_P] * 4 + [_I, _I, _I, _P, _P]),
    "atom_sample_f16": (_I, [_P, _I64, _I, _I] + [_P] * 7),
    "atom_sample_ex_f16": (_I, [_P, _I64, _I, _I] + [_P] * 11 + [_I64, _P, _P, _I, _P, _P, _P]),
    "atom_sample_slot_init": (_I, [_P, _I64, _I, _I, _P, _I, _P]),
    "atom_sample_draft_f16": (_I, [_P, _I64, _I, _I] + [_P] * 8 + [_I, _P, _P, _P, _P]),
    "atom_spec_commit_propose": (_I, [_P] * 4 + [_I, _P, _P] + [_I] * 5 + [_P, _P]),
    "atom_beam_select_f16": (_I, [_P, _I64, _I, _I, _P, _I, _P, _P, _I, _I] + [_P] * 6),
    "atom_kv_copy_pages_i4": (_I, [_P, _P] + [_I] * 4 + [_P] * 3 + [_I, _P]),
}

_lib = None


def symbols():
    """Names every C-ABI entry point include/atom_b200.h declares."""
    return list(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               f"(make -C atom_b200/csrc). atom_b200 has no CPU fallback.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype, fn.argtypes = res, args
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().atom_last_error()
        raise RuntimeError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")
