"""GINEConv, forward + backward, with the plug-in (fused relu(x_j + e_ji) sweep) against the reference's own CUDA path.

    python benchmarks/gine.py [--nodes 2000000] [--edges 10000000] [--feat 128] [--reps 5] [--warmup 2]

The model is an UNMODIFIED reference `GINEConv(Linear(F, F))` (oracle/_ref) with `edge_attr` requiring grad, so the
step has the three gradients a GINEConv user trains with.  Two arms in one process, alternated rep by rep after
warm-up: "fused" (`plugin.install()`) and "reference" (plug-in uninstalled: index_select, add, relu and scatter as
ATen kernels).  Prints one JSON line: ms for forward / backward / step (median over reps), the peak
`torch.cuda.max_memory_allocated` of a step for each arm, the engine's per-kernel time from `ops.PROFILE` (a separate
profiled step) with the bytes each kernel must move -- computed from shapes -- over that time against the H100 SXM
data sheet's 3.35 TB/s, sampled-row parity of out and grad_x against an fp64 formula, and the card's name and power
limit as nvidia-smi reports them in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))          # the unmodified reference, installed by build()

HBM_BYTES_PER_S = 3.35e12


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _graph(n: int, e: int, f: int, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=dev, generator=g)
    dst = (torch.rand(e, device=dev, generator=g) ** 2 * (n - 1)).long()    # skewed in-degrees, hub rows included
    x = torch.randn(n, f, device=dev, generator=g)
    ea = torch.randn(e, f, device=dev, generator=g)
    gout = torch.randn(n, f, device=dev, generator=g)
    return torch.stack([src, dst]), x, ea, gout


def _step(model, x, ei, ea, gout):
    x.grad = ea.grad = None
    model.zero_grad(set_to_none=True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    out = model(x, ei, ea)
    ev[1].record()
    out.backward(gout)
    ev[2].record()
    torch.cuda.synchronize()
    return out, (ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[2]))


def _parity(model, x, ei, ea, gout, out, gx, rows: int = 64) -> dict:
    """max |err| / max |ref| of out and grad_x on sampled destination / source rows against fp64 (pre-activation rounded
    to fp32 as both arms compute it)."""
    dev = x.device
    n = x.size(0)
    src, dst = ei[0], ei[1]
    g = torch.Generator(device=dev).manual_seed(1)
    pick = torch.unique(torch.cat([torch.randint(0, n, (rows, ), device=dev, generator=g),
                                   torch.tensor([0, 1], device=dev)]))               # + the biggest hubs
    W = model.nn.weight.detach().double()
    b = model.nn.bias.detach().double()
    one_eps = 1.0 + float(model.eps)
    # out rows: nn(sum_{e -> i} relu(x_j + e) + (1 + eps) x_i)
    sel = torch.isin(dst, pick)
    pre = (x.detach()[src[sel]] + ea.detach()[sel]).double()
    loc = torch.searchsorted(pick, dst[sel])
    agg = torch.zeros(pick.numel(), x.size(1), dtype=torch.float64, device=dev).index_add_(0, loc, pre.clamp(min=0))
    want = (agg + one_eps * x.detach()[pick].double()) @ W.T + b
    # grad_x rows: sum_{e: j -> i} [pre > 0] (g W)[i] + (1 + eps) (g W)[j]
    gW = gout.double() @ W
    sel = torch.isin(src, pick)
    pre = (x.detach()[src[sel]] + ea.detach()[sel]).double()
    loc = torch.searchsorted(pick, src[sel])
    gxw = torch.zeros(pick.numel(), x.size(1), dtype=torch.float64, device=dev).index_add_(
        0, loc, torch.where(pre > 0, gW[dst[sel]], 0.0))
    gxw += one_eps * gW[pick]
    rel = lambda a, r: float((a.double() - r).abs().max() / r.abs().max().clamp(min=1e-30))   # noqa: E731
    return {"rows": int(pick.numel()), "out_rel_err": rel(out.detach()[pick], want), "grad_x_rel_err": rel(gx[pick], gxw)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=2_000_000)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--feat", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gine.py measures on a CUDA GPU; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200 import plugin as P

    dev = torch.device("cuda")
    n, e, f = args.nodes, args.edges, args.feat
    ei, x0, ea0, gout = _graph(n, e, f, dev)
    torch.manual_seed(0)
    model = tg.nn.GINEConv(torch.nn.Linear(f, f)).to(dev)
    x = x0.clone().requires_grad_()
    ea = ea0.clone().requires_grad_()

    def arm(name):
        if name == "fused":
            if not P.installed():
                P.install()
        else:
            P.uninstall()

    arms = ("fused", "reference")
    times = {a: [] for a in arms}
    peak = {}
    parity = {}
    for a in arms:                                    # warm-up (graph build, allocator, library algorithms)
        arm(a)
        for _ in range(args.warmup):
            _step(model, x, ei, ea, gout)
    for _ in range(args.reps):
        for a in arms:
            arm(a)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out, t = _step(model, x, ei, ea, gout)
            peak[a] = max(peak.get(a, 0), torch.cuda.max_memory_allocated() - base)
            times[a].append(t)
            if a not in parity:
                parity[a] = _parity(model, x, ei, ea, gout, out, x.grad)
            del out

    # per-kernel time of the fused arm, in a profiled step of its own
    arm("fused")
    ops.PROFILE.reset(enabled=True)
    _step(model, x, ei, ea, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    P.uninstall()
    s = x.element_size()
    bytes_needed = {                                  # per edge (int32 indices; perm read: the graph is sorted here)
        "edge_relu_csr": e * (2 * f * s + 4 + 4 + f / 8) + n * f * s,
        "edge_relu_backward_x": e * (f * s + f / 8 + 8) + n * f * s,
        "edge_relu_backward_edge": e * (f * s + f / 8 + 4) + n * f * s,
    }
    kernels = {}
    for k, nbytes in bytes_needed.items():
        ms = prof.get(k, {}).get("ms_total")
        kernels[k] = {"ms": ms, "bytes": nbytes,
                      "bytes_per_s": None if not ms else nbytes / (ms * 1e-3),
                      "share_of_3.35TBps": None if not ms else nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    med = {a: {k: statistics.median(t[i] for t in times[a]) for i, k in enumerate(("fwd_ms", "bwd_ms", "step_ms"))}
           for a in arms}
    res = {"bench": "gine", "N": n, "E": e, "F": f, "dtype": "float32", "reps": args.reps, "warmup": args.warmup,
           "ms": med, "ms_all": times, "max_memory_allocated_bytes": peak,
           "speedup_step": med["reference"]["step_ms"] / med["fused"]["step_ms"], "kernels": kernels,
           "other_engine_ops_ms": {k: v["ms_total"] for k, v in prof.items() if k not in bytes_needed},
           "parity": parity, "gpu": _card()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
