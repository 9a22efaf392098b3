"""numpy front-end of tests/gqa_oracle.c, the CPU oracle of the grouped-query INT4 paged-KV decode attention.

TEST INFRASTRUCTURE ONLY.  The C file is compiled on first use into a temporary directory (same flags as oracle/Makefile:
no contraction, so the float arithmetic is the multi-head oracle's), never into the source tree.
"""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="atom_gqa_oracle_")
        atexit.register(shutil.rmtree, tmp, ignore_errors=True)
        so = os.path.join(tmp, "libgqa_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-o", so,
                               os.path.join(_HERE, "gqa_oracle.c"), "-lm"])
        _lib = ctypes.CDLL(so)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def batch_decode_gqa_i4(q, data, param, indptr, indices, last_off, layer, theta=1e4):
    """q f16 [B, Hq, 128]; data u8 [pages, L, 2, Hkv, P, 64]; param f16 [pages, L, 2, Hkv, P, 2] -> o f16 [B, Hq, 128]."""
    q = np.ascontiguousarray(q, np.float16)
    B, Hq, D = q.shape
    _, L, _, Hkv, P, _ = data.shape
    assert D == 128 and Hq % Hkv == 0
    data, param = np.ascontiguousarray(data, np.uint8), np.ascontiguousarray(param, np.float16)
    indptr, indices, last_off = (np.ascontiguousarray(a, np.int32) for a in (indptr, indices, last_off))
    o = np.zeros_like(q)
    lib().gqa_oracle_batch_decode_i4(_p(o), _p(q), _p(data), _p(param), _p(indptr), _p(indices), _p(last_off), L, int(layer), Hq, Hkv, P,
                                     B, ctypes.c_float(theta))
    return o


def repeat_heads(data, param, g):
    """The cache a multi-head kernel needs to emulate grouped-query attention: every KV head g times (axis 3)."""
    return np.repeat(data, g, axis=3), np.repeat(param, g, axis=3)
