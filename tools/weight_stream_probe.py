"""How fast the decode GEMM's INT4 weight tiles can reach shared memory, by fetch geometry.

python tools/weight_stream_probe.py [--sets 14] [--rounds 4] [--reps 20]

Compiles tools/weight_stream_probe.cu into a temporary directory and times, per fetch variant, a kernel that reproduces the
launch conditions of the headline GEMM (gemm_i4_o16, M = 16, N = K = 4096: 32 channel tiles x a 4-rank K cluster, 384
threads, the GEMM's dynamic shared memory, programmatic dependent launch with every weight request before
griddepcontrol.wait) and moves only rank r's K range of its 128 weight rows (4096 x 1984 B per tensor) into shared memory:

  a     2-D UINT8 map, box 64 B x 128 rows, one request per group (the GEMM's fetch)
  b     (a) with CU_TENSOR_MAP_L2_PROMOTION_L2_256B
  c     2-D UINT8 map, box 128 B x 128 rows, SWIZZLE_128B: two groups per request row
  d256  2-D UINT64 map, box 32 elements (256 B) x 128 rows: four groups per request row
  d512  2-D UINT64 map, box 64 elements (512 B) x 128 rows: eight groups per request row
  d256u8  2-D UINT8 map, box 256 B x 128 rows
  e     3-D map (64 B, row, group), strides (pitch, 64), box {64, 128, 8}: the per-group layout in one request
  f     one 1-D cp.async.bulk per row span (128 x 512 B)
  g     (a) after a cluster-cooperative cp.async.bulk.prefetch.L2 of the cluster's contiguous 128-row block
  read  a plain coalesced 16-byte-vector read of the same tensors (8 CTAs x 256 threads per SM, 4 loads in flight each)

Each variant runs over HBM (one CUDA graph of back-to-back launches rotating over --sets tensors, together larger than the
50 MB L2) and L2-resident (one tensor).  Prints one JSON object: us per launch, GB/s and the share of the data sheet's
3.35 TB/s per variant and residency, with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = ("a", "b", "c", "d256", "d512", "d256u8", "e", "f", "g", "read")
HBM_TBPS = 3.35


def build(out_dir):
    so = os.path.join(out_dir, "weight_stream_probe.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                           "--expt-relaxed-constexpr", "-shared", "-o", so,
                           os.path.join(ROOT, "tools", "weight_stream_probe.cu"), "-lcudart"])
    return so


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"error": "nvidia-smi unavailable"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=14, help="weight tensors the HBM run rotates over (>= 14 exceed L2)")
    ap.add_argument("--rounds", type=int, default=4, help="passes over the sets per graph")
    ap.add_argument("--warm", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("weight_stream_probe.py needs a CUDA device")
    lib = ctypes.CDLL(build(tempfile.mkdtemp(prefix="atom_probe_")))
    lib.probe_last_error.restype = ctypes.c_char_p
    lib.probe_run.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                              ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    assert lib.probe_variants() == len(VARIANTS) - 1
    nbytes = lib.probe_tensor_bytes()
    g = torch.Generator(device="cuda:0").manual_seed(7)
    sets = [torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda:0", generator=g) for _ in range(a.sets)]
    torch.cuda.synchronize()
    res = {}
    for vi, name in enumerate(VARIANTS):
        for where, n in (("hbm", a.sets), ("l2", 1)):
            ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in sets[:n]])
            us = ctypes.c_float(0)
            rc = lib.probe_run(vi, ptrs, n, a.rounds if n > 1 else a.rounds * a.sets, a.warm, a.reps, ctypes.byref(us))
            if rc < 0:                        # a CUDA error: the context may be unusable, stop here
                print(json.dumps({"error": lib.probe_last_error().decode(), "variant": name, "where": where}), flush=True)
                sys.exit(1)
            if rc > 0:                        # cuTensorMapEncodeTiled rejected the variant's map
                res.setdefault(name, {})[where] = {"rejected": lib.probe_last_error().decode()}
                continue
            gbs = nbytes / (us.value * 1e-6) / 1e9
            res.setdefault(name, {})[where] = {"us_per_launch": round(us.value, 3), "GB_s": round(gbs, 1),
                                               "of_3_35_TBs": round(gbs / (HBM_TBPS * 1e3), 3)}
    print(json.dumps({"probe": "weight_stream", "bytes_per_launch": nbytes, "sets": a.sets, "card": card(),
                      "variants": res}), flush=True)


if __name__ == "__main__":
    main()
