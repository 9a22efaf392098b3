"""ctypes front-end of oracle/_ref/libatom_ref.so: the REFERENCE's own CUDA kernels, compiled unmodified from
the reference tree by oracle/Makefile for sm_90a.  TEST / BENCH INFRASTRUCTURE ONLY (live GPU oracle and the
`--impl reference` timing arm); never imported by atom_b200/.

All launches go to the legacy default stream, as in the reference (Reorder.cuh:219, GEMM.cuh:763).
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libatom_ref.so")
_lib = None


def available():
    return os.path.exists(SO)


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(SO)
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _chk(rc, what):
    if rc != 0:
        raise RuntimeError(f"reference kernel {what}: cuda error {rc}")


def scale_size(x):
    return ((x) // 16 * 64 + 64 - (1 - (x % 16) // 8) * (8 - (x % 8)) * 8)


def _quant_out(bs, hidden, dev):
    # zero-filled so that unwritten slots of the scale layout compare equal
    return (torch.zeros((bs, 128), dtype=torch.int8, device=dev), torch.zeros((bs, (hidden - 128) // 2), dtype=torch.int8, device=dev),
            torch.zeros((scale_size(bs),), dtype=torch.float16, device=dev),
            torch.zeros((hidden // 128 - 1, scale_size(bs)), dtype=torch.float16, device=dev))


def reorder_fp16_i4(x, idx, sync=1):
    assert x.shape[1] == 4096
    out = _quant_out(x.shape[0], 4096, x.device)
    _chk(lib().atom_ref_reorder_fp16_i4(_p(x), x.shape[0], _p(idx), *[_p(o) for o in out], sync), "reorder")
    return out


def rmsnorm_fp16_i4(x, w, idx, eps, sync=1):
    assert x.shape[1] == 4096
    out = _quant_out(x.shape[0], 4096, x.device)
    _chk(lib().atom_ref_rmsnorm_fp16_i4(_p(x), _p(w), ctypes.c_float(eps), x.shape[0], _p(idx), *[_p(o) for o in out], sync), "rmsnorm")
    return out


def activate_fp16_i4(a, b, sync=1):
    assert a.shape[1] == 11008
    out = _quant_out(a.shape[0], 11008, a.device)
    _chk(lib().atom_ref_activate_fp16_i4(_p(a), _p(b), a.shape[0], *[_p(o) for o in out], sync), "activate")
    return out


def gemm_i4_o16(a, b, a_s, b_s, ak, bk, aks, bks, d=None, sync=1):
    m, n, k = a.shape[0], b.shape[0], a.shape[1] * 2 + ak.shape[1]
    if d is None:
        d = torch.empty((m, n), dtype=torch.float16, device=a.device)
    _chk(lib().atom_ref_gemm_i4_o16(_p(a), _p(b), _p(a_s), _p(b_s), _p(ak), _p(bk), _p(aks), _p(bks), _p(d),
                                    ctypes.c_size_t(m), ctypes.c_size_t(n), ctypes.c_size_t(k), sync), "gemm_o16")
    return d


def gemm_i4_o4(a, b, a_s, b_s, ak, bk, aks, bks, sync=1):
    m, n, k = a.shape[0], b.shape[0], a.shape[1] * 2 + ak.shape[1]
    d = torch.empty((m, n // 2), dtype=torch.uint8, device=a.device)
    ds = torch.empty((m, n // 128 * 2), dtype=torch.float16, device=a.device)
    _chk(lib().atom_ref_gemm_i4_o4(_p(a), _p(b), _p(a_s), _p(b_s), _p(ak), _p(bk), _p(aks), _p(bks), _p(d), _p(ds),
                                   ctypes.c_size_t(m), ctypes.c_size_t(n), ctypes.c_size_t(k), sync), "gemm_o4")
    return d, ds


def batch_decode_i4(q, data, param, indptr, indices, last, layer, sync=1):
    o = torch.empty_like(q)
    _, L, _, H, P, _ = data.shape
    _chk(lib().atom_ref_batch_decode_i4(_p(o), _p(q), _p(data), _p(param), _p(indptr), _p(indices), _p(last), L, layer, H, P,
                                        q.shape[0], sync), "batch_decode")
    return o


def append_kv_i4(data, param, indptr, indices, last, k, v, kp, vp, layer, sync=1):
    _, L, _, H, P, _ = data.shape
    _chk(lib().atom_ref_append_kv_i4(_p(data), _p(param), _p(indptr), _p(indices), _p(last), _p(k), _p(v), _p(kp), _p(vp), L,
                                     layer, H, P, k.shape[0], sync), "append_kv")


def init_kv_i4(data, param, indptr, indices, last, k, v, kp, vp, seqlen_indptr, layer, sync=1):
    _, L, _, H, P, _ = data.shape
    _chk(lib().atom_ref_init_kv_i4(_p(data), _p(param), _p(indptr), _p(indices), _p(last), _p(k), _p(v), _p(kp), _p(vp),
                                   _p(seqlen_indptr), L, layer, H, P, last.shape[0], sync), "init_kv")
