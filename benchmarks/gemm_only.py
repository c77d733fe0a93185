#!/usr/bin/env python
"""The layer's three dense products alone (for ncu captures and A/B timing of the wgmma 3xTF32 GEMMs).

    python benchmarks/gemm_only.py [--rows 10000000] [--n 256] [--k 256] [--steps 5] [--bsplit 0|1] [--mode 0|1]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--k", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--bsplit", type=int, default=0)
    ap.add_argument("--mode", type=int, default=-1)
    ap.add_argument("--prefetch", type=int, default=-1, help="TMA L2-prefetch distance in k-blocks (gemm_prefetch option)")
    args = ap.parse_args()
    from pytorch_geometric_b200 import dense, ops
    if args.mode >= 0:
        ops.set_option("gemm_mode", args.mode)
    if args.prefetch >= 0:
        ops.set_option("gemm_prefetch", args.prefetch)
    dense.set_b_split(bool(args.bsplit))
    dev = torch.device("cuda", 0)
    x = torch.randn(args.rows, args.k, device=dev)
    g = torch.randn(args.rows, args.n, device=dev)
    w = torch.randn(args.n, args.k, device=dev) / args.k ** 0.5
    w_hi, w_lo = dense.prepare_weight(w)
    res = {}
    for name, fn in (("forward", lambda: dense.linear_forward(x, w_hi, w_lo)),
                     ("grad_input", lambda: dense.linear_grad_input(g, w_hi, w_lo)),
                     ("grad_input_kmajor", lambda: dense.linear_grad_input_w(g, w, w_hi, w_lo)),
                     ("grad_weight", lambda: dense.linear_grad_weight(g, x))):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        res[name] = {"ms": ms, "tflops_3x": 3 * 2 * args.rows * args.n * args.k / (ms * 1e-3) / 1e12,
                     "hbm_GBps_min": 2 * args.rows * (args.n if name == "forward" else args.k) * 4 / (ms * 1e-3) / 1e9}
    print(json.dumps({"rows": args.rows, "n": args.n, "k": args.k, "bsplit": args.bsplit, "prefetch": args.prefetch, **res}))


if __name__ == "__main__":
    main()
