"""ResGatedGraphConv, forward + backward, with the plug-in (fused sigmoid(k_i + q_j) * v_j sweep) against the
reference's own CUDA path.

    python benchmarks/res_gated.py [--nodes 2000000] [--edges 10000000] [--feat 128] [--reps 5] [--warmup 2]

The model is an UNMODIFIED reference `ResGatedGraphConv(F, F)` (oracle/_ref), trained with x requiring grad.  Two arms
in one process, alternated rep by rep after warm-up: "fused" (`plugin.install()`) and "reference" (plug-in
uninstalled: three index_selects, add, sigmoid, mul and scatter as ATen kernels).  Prints one JSON line: ms for
forward / backward / step (median over reps), the peak `torch.cuda.max_memory_allocated` growth of a step for each
arm, the engine's per-kernel time from `ops.PROFILE` (a separate profiled step) with the bytes each kernel must move --
computed from shapes -- over that time against the H100 SXM data sheet's 3.35 TB/s, sampled-row parity of out against
an fp64 formula for both arms, and the card's name and power limit as nvidia-smi reports them in the same run.
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
    gout = torch.randn(n, f, device=dev, generator=g)
    return torch.stack([src, dst]), x, gout


def _step(model, x, ei, gout):
    x.grad = None
    model.zero_grad(set_to_none=True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    out = model(x, ei)
    ev[1].record()
    out.backward(gout)
    ev[2].record()
    torch.cuda.synchronize()
    return out, (ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[2]))


def _parity(model, x, ei, out, rows: int = 64) -> dict:
    """max |err| / max |ref| of out on sampled destination rows (plus the biggest hubs) against fp64:
    out_i = sum_{e: j -> i} sigmoid(k_i + q_j) * v_j + W_skip x_i + bias."""
    dev = x.device
    n = x.size(0)
    src, dst = ei[0], ei[1]
    g = torch.Generator(device=dev).manual_seed(1)
    pick = torch.unique(torch.cat([torch.randint(0, n, (rows, ), device=dev, generator=g),
                                   torch.tensor([0, 1], device=dev)]))
    xd = x.detach().double()
    lin = lambda m, t: t @ m.weight.detach().double().T + (0 if m.bias is None else m.bias.detach().double())  # noqa: E731
    sel = torch.isin(dst, pick)
    s_, d_ = src[sel], dst[sel]
    gate = torch.sigmoid(lin(model.lin_key, xd[d_]) + lin(model.lin_query, xd[s_]))
    loc = torch.searchsorted(pick, d_)
    agg = torch.zeros(pick.numel(), x.size(1), dtype=torch.float64, device=dev).index_add_(
        0, loc, gate * lin(model.lin_value, xd[s_]))
    want = agg + lin(model.lin_skip, xd[pick]) + model.bias.detach().double()
    return {"rows": int(pick.numel()),
            "out_rel_err": float((out.detach()[pick].double() - want).abs().max() / want.abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=2_000_000)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--feat", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/res_gated.py measures on a CUDA GPU; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200 import plugin as P

    dev = torch.device("cuda")
    n, e, f = args.nodes, args.edges, args.feat
    ei, x0, gout = _graph(n, e, f, dev)
    torch.manual_seed(0)
    model = tg.nn.ResGatedGraphConv(f, f).to(dev)
    with torch.no_grad():
        model.bias.normal_(0, 0.1)
    x = x0.clone().requires_grad_()

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
            _step(model, x, ei, gout)
    for _ in range(args.reps):
        for a in arms:
            arm(a)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out, t = _step(model, x, ei, gout)
            peak[a] = max(peak.get(a, 0), torch.cuda.max_memory_allocated() - base)
            times[a].append(t)
            if a not in parity:
                parity[a] = _parity(model, x, ei, out)
            del out

    # per-kernel time of the fused arm, in a profiled step of its own
    arm("fused")
    ops.PROFILE.reset(enabled=True)
    _step(model, x, ei, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    P.uninstall()
    r = f * x.element_size()                          # bytes per feature row; int32 indices
    bytes_needed = {
        "gated_csr": e * (2 * r + 4) + n * 2 * r,             # q, v, col per edge; k read, out written per row
        "gated_backward_dst": e * (2 * r + 4) + n * 3 * r,    # q, v, col per edge; k, g read, grad_k written
        "gated_backward_src": e * (2 * r + 4) + n * 4 * r,    # k, g, col_t per edge; q, v read, grad_q, grad_v written
    }
    kernels = {}
    for k, nbytes in bytes_needed.items():
        ms = prof.get(k, {}).get("ms_total")
        kernels[k] = {"ms": ms, "bytes": nbytes,
                      "bytes_per_s": None if not ms else nbytes / (ms * 1e-3),
                      "share_of_3.35TBps": None if not ms else nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    med = {a: {k: statistics.median(t[i] for t in times[a]) for i, k in enumerate(("fwd_ms", "bwd_ms", "step_ms"))}
           for a in arms}
    res = {"bench": "res_gated", "N": n, "E": e, "F": f, "dtype": "float32", "reps": args.reps,
           "warmup": args.warmup, "ms": med, "ms_all": times, "max_memory_allocated_bytes": peak,
           "speedup_step": med["reference"]["step_ms"] / med["fused"]["step_ms"], "kernels": kernels,
           "other_engine_ops_ms": {k: v["ms_total"] for k, v in prof.items() if k not in bytes_needed},
           "parity": parity, "gpu": _card()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
