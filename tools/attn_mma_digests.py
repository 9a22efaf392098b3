#!/usr/bin/env python
"""Writes tests/golden/attn_mma_h100.npz: SHA-256 digests of the output bytes of the tensor-core attention kernels (prefill with
and without a cached context, verify, the cascade's shared-prefix pass) for the seeded cases of
tests/test_z_attn_mma_digests_gpu.py.  Run it with a library built before those kernels shared one tile step, so that the suite
can check that they still compute exactly what they computed then.  Needs a GPU; the cases' automatic chunk counts follow the SM
count, so take the digests on the GPU model the test names.

    python tools/attn_mma_digests.py --lib /path/to/old/libatom_b200.so --out tests/golden/attn_mma_h100.npz
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from atom_b200 import _lib  # noqa: E402
from tests.test_z_attn_mma_digests_gpu import CASES, compute, digest  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", required=True, help="libatom_b200.so to take the digests from")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_mma_digests: needs a CUDA device")
    _lib.LIB_PATH = os.path.abspath(args.lib)         # every ops call below goes through this library
    print(f"{torch.cuda.get_device_name()}, {torch.cuda.get_device_properties(0).multi_processor_count} SMs")
    out = {}
    for name in CASES:
        out[name] = np.array(digest(compute(name)))
        print(f"{name} {out[name]}")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, **out)


if __name__ == "__main__":
    main()
