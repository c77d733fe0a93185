#!/usr/bin/env python
"""Where the 3xTF32 GEMM's warps spend their time: builds gemm_tf32x3.cu with -DB200MP_GEMM_TRACE into a temporary
library of its own (the package's library is not touched), runs the layer's three dense products at bench.py's shape
and prints one JSON line with the clock64 totals of each role as shares of that role's time:
  consumers  waiting on bar_full / bar_sfull, in wgmma.wait_group, in the epilogue, and the rest (issuing MMAs, which
             stalls while the tensor pipe is full, splitting A fragments, releasing stages);
  producer   waiting on bar_empty (the ring is full: the consumers are behind);
  B prep     waiting on bar_full (TMA data) and on bar_sempty (prepared slots still in use).
The traced build times the calls too, but clock64 reads and the totals' registers perturb the kernel: take the
products' times from benchmarks/gemm_only.py or bench.py.

    python benchmarks/gemm_stalls.py [--rows 5000000] [--n 256] [--k 256] [--steps 5] [--src DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = ["full_wait", "mma_wait", "epilogue", "consumer", "empty_wait", "producer", "prep_full_wait",
         "prep_slot_wait", "prep"]                       # TraceSlot order in gemm_tf32x3.cu


def build_traced(src_dir, out_dir):
    from pytorch_geometric_b200 import _build
    nvcc = _build._nvcc()
    include = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(src_dir))), "include")
    objs = []
    for name in ("gemm_tf32x3.cu", "core.cu"):
        obj = os.path.join(out_dir, name[:-3] + ".o")
        cmd = [nvcc, *_build.NVCC_FLAGS, "-DB200MP_GEMM_TRACE", "-I", include, "-c", os.path.join(src_dir, name), "-o", obj]
        subprocess.run(cmd, check=True)
        objs.append(obj)
    so = os.path.join(out_dir, "libgemm_trace.so")
    subprocess.run([nvcc, "-shared", *_build.ARCH_FLAGS, "-o", so, *objs], check=True)
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--k", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--src", default=os.path.join(ROOT, "pytorch_geometric_b200", "csrc"),
                    help="directory holding gemm_tf32x3.cu and core.cu (with ../../include/b200mp.h)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_stalls.py needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="gemm_trace_")
    lib = ctypes.CDLL(build_traced(args.src, tmp))
    P, I64, INT = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.b200mp_split_tf32.argtypes = [P, P, P, I64, P]
    lib.b200mp_split_tf32_transposed.argtypes = [P, P, P, I64, I64, P]
    lib.b200mp_linear_tf32x3.argtypes = [P, P, P, P, I64, I64, I64, P]
    lib.b200mp_gemm_pair_tf32x3.argtypes = [P, I64, P, I64, P, P, INT, P, INT, P, I64, P, I64, I64, P]
    lib.b200mp_linear_grad_weight_workspace_bytes.restype = I64
    lib.b200mp_linear_grad_weight_workspace_bytes.argtypes = [I64, I64, I64]
    lib.b200mp_linear_grad_weight_tf32x3.argtypes = [P, P, P, I64, I64, I64, P, I64, P]
    lib.b200mp_gemm_trace_read.argtypes = [P, INT, INT]

    dev = torch.device("cuda", 0)
    m, n, k = args.rows, args.n, args.k
    x = torch.randn(m, k, device=dev)
    g = torch.randn(m, n, device=dev)
    w = torch.randn(n, k, device=dev) / k ** 0.5
    s = torch.cuda.current_stream().cuda_stream
    w_hi, w_lo = torch.empty_like(w), torch.empty_like(w)
    wt_hi, wt_lo = torch.empty(k, n, device=dev), torch.empty(k, n, device=dev)
    y, gx, gw = torch.empty(m, n, device=dev), torch.empty(m, k, device=dev), torch.empty(n, k, device=dev)
    ws = torch.empty(lib.b200mp_linear_grad_weight_workspace_bytes(m, n, k), dtype=torch.uint8, device=dev)

    def check(rc):
        if rc != 0:
            raise RuntimeError(f"library call failed with {rc}")

    check(lib.b200mp_split_tf32(w.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), w.numel(), s))
    check(lib.b200mp_split_tf32_transposed(w.data_ptr(), wt_hi.data_ptr(), wt_lo.data_ptr(), n, k, s))
    products = {   # as the GCN layer runs them (dense.linear_forward, linear_grad_input_w, linear_grad_weight)
        "linear_tf32x3": lambda: lib.b200mp_linear_tf32x3(x.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), y.data_ptr(),
                                                          m, n, k, s),
        "linear_grad_input_tf32x3": lambda: lib.b200mp_gemm_pair_tf32x3(g.data_ptr(), n, None, 0, wt_hi.data_ptr(),
                                                                        wt_lo.data_ptr(), 0, None, 0, gx.data_ptr(), k,
                                                                        None, 0, m, s),
        "linear_grad_weight_tf32x3": lambda: lib.b200mp_linear_grad_weight_tf32x3(g.data_ptr(), x.data_ptr(),
                                                                                  gw.data_ptr(), m, n, k, ws.data_ptr(),
                                                                                  ws.numel(), s),
    }
    buf = (ctypes.c_ulonglong * len(SLOTS))()
    res = {"gpu": torch.cuda.get_device_name(0), "rows": m, "n": n, "k": k, "src": os.path.abspath(args.src)}
    for name, fn in products.items():
        check(fn())
        check(lib.b200mp_gemm_trace_read(buf, len(SLOTS), 1))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            check(fn())
        e1.record()
        check(lib.b200mp_gemm_trace_read(buf, len(SLOTS), 1))
        t = dict(zip(SLOTS, (float(v) for v in buf)))
        cons = max(t["consumer"], 1.0)
        other = cons - t["full_wait"] - t["mma_wait"] - t["epilogue"]
        r = {"ms_traced": e0.elapsed_time(e1) / args.steps,
             "consumer_share": {key: round(t[key] / cons, 4) for key in ("full_wait", "mma_wait", "epilogue")},
             "producer_empty_wait_share": round(t["empty_wait"] / max(t["producer"], 1.0), 4)}
        r["consumer_share"]["issue_split_other"] = round(other / cons, 4)
        if t["prep"] > 0:
            r["prep_share"] = {"full_wait": round(t["prep_full_wait"] / t["prep"], 4),
                               "slot_wait": round(t["prep_slot_wait"] / t["prep"], 4)}
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
