#!/usr/bin/env python
"""Writes tests/golden/decode_unsplit_h100.npz: SHA-256 digests of the unsplit decode attention's output bytes for the seeded
inputs of tests/test_z_decode_splitkv_gpu.py (UNSPLIT_CASES, one per unsplit batch_decode_kernel instantiation).  Run it with a
library built from a revision whose atom_batch_decode_gqa_i4 never splits -- the revision before split-KV decode -- so that the
suite can check that kv_split = 1 still computes exactly what that kernel computed.  Needs a GPU.

    python tools/decode_unsplit_digests.py --lib /path/to/old/libatom_b200.so --out tests/golden/decode_unsplit_h100.npz
"""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tests.test_z_decode_splitkv_gpu import UNSPLIT_CASES, T, digest, unsplit_case  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True, help="libatom_b200.so whose atom_batch_decode_gqa_i4 is the unsplit kernel")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_unsplit_digests: needs a CUDA device")
    lib = ctypes.CDLL(os.path.abspath(args.lib))
    fn = lib.atom_batch_decode_gqa_i4
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int] * 6 + [ctypes.c_float, ctypes.c_void_p]
    out = {}
    for G, P in UNSPLIT_CASES:
        q, (data, param, indptr, indices, last), theta = unsplit_case(G, P)
        t = [T(x) for x in (q, data, param, indptr, indices, last)]
        o = torch.empty_like(t[0])
        rc = fn(o.data_ptr(), *[x.data_ptr() for x in t], data.shape[1], 1, q.shape[1], data.shape[3], P, q.shape[0], theta,
                torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise SystemExit(f"atom_batch_decode_gqa_i4 failed ({rc}) for G={G} P={P}")
        out[f"g{G}_p{P}"] = np.array(digest(o.cpu().numpy()))
        print(f"g{G}_p{P} {out[f'g{G}_p{P}']}")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, **out)


if __name__ == "__main__":
    main()
