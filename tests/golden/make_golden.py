"""Regenerates tests/golden/*.npz from the reference tree (needs the reference tree: ATOM_REFERENCE).

Two sources, both the reference's own code, neither copied into this repo:
  * the CPU golden functions of test_Reorder.cu / test_RMSNorm.cu / test_activate.cu
    (compiled where they lie, see gen_ref_golden.cu);
  * model/quant.py + model/qLinearLayer.py imported from /root/reference/model with
    `bitsandbytes` stubbed (only used for --quant_type fp, quant.py:134-138);
  * generate_request_set of e2e/punica-atom/benchmarks/bench_textgen.py (the serving harness's workload).
Run:  python tests/golden/make_golden.py
"""
import os, subprocess, sys, types, tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("ATOM_REFERENCE", "/root/reference")
CSRC = os.path.join(REF, "e2e/punica-atom/punica/ops/csrc")


def cpp_golden(kind, seq_len, hidden):
    tmp = tempfile.mkdtemp()
    exe, out = os.path.join(tmp, "gen"), os.path.join(tmp, "out.bin")
    subprocess.check_call(["nvcc", "-w", "-O1", "-std=c++17", "-arch=sm_90a", f"-DGEN_{kind.upper()}",
                           f"-I{CSRC}", os.path.join(HERE, "gen_ref_golden.cu"), "-o", exe])
    subprocess.check_call([exe, str(seq_len), str(hidden), out])
    raw = open(out, "rb").read()
    ldm = seq_len // 16 * 64 + 64 - (1 - (seq_len % 16) // 8) * (8 - (seq_len % 8)) * 8
    spec = [("x", np.float16, seq_len * hidden), ("x2", np.float16, seq_len * hidden), ("w", np.float16, hidden),
            ("idx", np.int16, hidden), ("o8", np.int8, seq_len * 128), ("o4", np.uint8, seq_len * (hidden - 128) // 2),
            ("s8", np.float16, ldm), ("s4", np.float16, (hidden // 128 - 1) * ldm)]
    res, off = {}, 0
    for name, dt, n in spec:
        nb = n * np.dtype(dt).itemsize
        res[name] = np.frombuffer(raw[off:off + nb], dtype=dt).copy()
        off += nb
    assert off == len(raw)
    res["x"] = res["x"].reshape(seq_len, hidden)
    res["x2"] = res["x2"].reshape(seq_len, hidden)
    res["o8"] = res["o8"].reshape(seq_len, 128)
    res["o4"] = res["o4"].reshape(seq_len, -1)
    res["s4"] = res["s4"].reshape(hidden // 128 - 1, ldm)
    if kind != "activate":
        res.pop("x2")
    if kind != "rmsnorm":
        res.pop("w")
    if kind == "activate":
        res.pop("idx")
    np.savez_compressed(os.path.join(HERE, f"ref_cpu_{kind}_{seq_len}x{hidden}.npz"), **res)
    print("wrote", kind, seq_len, hidden)


def python_golden():
    import torch
    sys.modules.setdefault("bitsandbytes", types.ModuleType("bitsandbytes"))
    fn = types.ModuleType("bitsandbytes.functional")
    fn.quantize_fp4 = fn.dequantize_fp4 = None
    sys.modules["bitsandbytes.functional"] = fn
    sys.path.insert(0, os.path.join(REF, "model"))
    import quant as rq
    from qLinearLayer import QLinearLayer
    args = types.SimpleNamespace(wbits=4, abits=4, w_sym=True, a_sym=True, weight_group_size=128, act_group_size=128,
                                 weight_channel_group=2, w_clip_ratio=0.85, a_clip_ratio=0.9, keeper=128,
                                 keeper_precision=3, exponential=False, tiling=0, quant_type="int", static=False,
                                 kv_clip_ratio=1.0, reorder=True)
    torch.manual_seed(0)
    lin = torch.nn.Linear(512, 256, bias=False)
    w0 = lin.weight.detach().clone()
    q = QLinearLayer(lin, args)
    q.quant()
    x = torch.randn(5, 512)
    xq = rq.quantize_activation_wrapper(x.clone(), args)
    y = q(xq)
    kv = torch.randn(2, 3, 4, 128)
    kq = rq.quantize_attn_k_wrapper(kv.clone(), args)
    t = torch.randn(6, 256)
    t_sym = rq.quantize_tensor(t.clone(), n_bits=4, group_size=128, tiling=0, sym=True, clip_ratio=0.9)
    t_asym = rq.quantize_tensor(t.clone(), n_bits=4, group_size=128, tiling=0, sym=False, clip_ratio=1.0)
    np.savez_compressed(os.path.join(HERE, "ref_py_fakequant.npz"), w0=w0.numpy(), wq=q.weight.numpy(), x=x.numpy(),
                        xq=xq.numpy(), y=y.numpy(), kv=kv.numpy(), kq=kq.numpy(), t=t.numpy(), t_sym=t_sym.numpy(),
                        t_asym=t_asym.numpy())
    print("wrote python fake-quant golden")


def request_set_golden():
    """generate_request_set of the reference's serving harness (benchmarks/bench_textgen.py:31-47), imported as is."""
    import importlib
    sys.path.insert(0, os.path.join(REF, "e2e/punica-atom"))
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp())          # keep this repo's own top-level modules out of the way
    m = importlib.import_module("benchmarks.bench_textgen")
    os.chdir(cwd)
    a, b = m.generate_request_set(160, 2048), m.generate_request_set(48, 512)
    np.savez_compressed(os.path.join(HERE, "ref_py_request_set.npz"), p160=a.prompt_lens, o160=a.output_lens,
                        p48=b.prompt_lens, o48=b.output_lens)
    print("wrote request-set golden")


if __name__ == "__main__":
    cpp_golden("reorder", 21, 4096)
    # test_RMSNorm.cu does not compile against the reference's own RMSNorm.cu (its perf_gpu() instantiates
    # rmsnorm_fp16_i4_kernel<threads,32,4096> with a stale 3-parameter signature, test_RMSNorm.cu:259), so
    # run_cpu_rmsnorm_fp16_i4 cannot be built; K4 is pinned through its shared tail (reorder golden), a
    # float64 restatement in the tests, and the reference CUDA kernel on the GPU box.
    cpp_golden("activate", 5, 11008)
    python_golden()
    request_set_golden()
