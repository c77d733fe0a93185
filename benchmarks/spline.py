"""SplineConv, forward + backward, fused (`plugin.conv.B200SplineConv`) against the unmodified reference layer running
through the engine's standalone `spline_basis` / `spline_weighting` shim ops (the only other path: pyg-lib is not
installed, and the reference has no spline code of its own).

    python benchmarks/spline.py [--workload faust|mnist|power_law_d2|power_law_d3|all] [--reps 3] [--warmup 1]

Workloads:
  * faust: N = 6890, E = 41328 (in-degree 6), dim 3, kernel 5 (K = 125), 64 -> 64, add (examples/faust.py's layers);
  * mnist: 64 graphs x 75 superpixels, 8 nearest neighbours each, dim 2, kernel 5 (K = 25), 32 -> 64, mean
    (examples/mnist_graclus.py's second conv);
  * power_law_d2 / power_law_d3: N = 1M, E = 10M with skewed in-degrees (hub rows split by the long-row plan),
    64 -> 64, add, at dim 2 (K = 25) and dim 3 (K = 125).  At dim 3 the fused path writes and reads back
    P = N K F_in fp32 (32 GB each way), which can cost more than the unfused path's E S F_in F_out FMAs.

One process, both arms on the same module and inputs, alternated rep by rep after warm-up.  Prints one JSON line per
workload: median ms of a forward + backward step per arm, the peak `torch.cuda.max_memory_allocated` growth of a step,
the engine's per-op time from `ops.PROFILE` in a separate profiled step (the fused arm's sweep `spline_csr` /
`spline_backward_dst` and its GEMMs, the other arm's `spline_weighting*`), the max relative difference of the two
arms' outputs, and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.  An arm
that runs out of memory is recorded as such.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))          # the unmodified reference, installed by build()

WORKLOADS = {"faust": dict(n=6890, deg=6, dim=3, ks=5, fi=64, fo=64, aggr="add"),
             "mnist": dict(graphs=64, nodes=75, deg=8, dim=2, ks=5, fi=32, fo=64, aggr="mean"),
             "power_law_d2": dict(n=1_000_000, e=10_000_000, dim=2, ks=5, fi=64, fo=64, aggr="add"),
             "power_law_d3": dict(n=1_000_000, e=10_000_000, dim=3, ks=5, fi=64, fo=64, aggr="add")}


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _inputs(w: dict, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    if "graphs" in w:                                 # per graph: every node takes `deg` random in-neighbours
        n = w["graphs"] * w["nodes"]
        dst = torch.arange(n, device=dev).repeat_interleave(w["deg"])
        src = dst // w["nodes"] * w["nodes"] + torch.randint(0, w["nodes"], (dst.numel(), ), device=dev, generator=g)
    elif "deg" in w:                                  # mesh-like: constant in-degree, nearby sources
        n = w["n"]
        dst = torch.arange(n, device=dev).repeat_interleave(w["deg"])
        src = (dst + torch.randint(-50, 51, (dst.numel(), ), device=dev, generator=g)).clamp(0, n - 1)
    else:
        n, e = w["n"], w["e"]
        src = torch.randint(0, n, (e, ), device=dev, generator=g)
        dst = (torch.rand(e, device=dev, generator=g) ** 3 * (n - 1)).long()
    ei = torch.stack([src, dst])
    x = torch.randn(n, w["fi"], device=dev, generator=g)
    ea = torch.rand(ei.size(1), w["dim"], device=dev, generator=g)
    return ei, x, ea


def _step(conv, ei, x, ea):
    xg = x.detach().requires_grad_()
    out = conv(xg, ei, ea)
    out.backward(torch.ones_like(out))
    return out.detach()


def _timed(conv, ei, x, ea):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = _step(conv, ei, x, ea)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), (torch.cuda.max_memory_allocated() - base) / 1e9, out


def run(name: str, reps: int, warmup: int) -> dict:
    import torch_geometric.nn as tgnn

    from pytorch_geometric_b200 import ops, plugin
    from pytorch_geometric_b200.plugin import conv as PC
    dev = torch.device("cuda")
    w = WORKLOADS[name]
    plugin.install(layers=True)
    torch.manual_seed(0)
    fused = tgnn.SplineConv(w["fi"], w["fo"], w["dim"], kernel_size=w["ks"], aggr=w["aggr"]).to(dev)
    assert type(fused) is PC.B200SplineConv
    unfused = copy.deepcopy(fused)
    unfused.__class__ = PC.B200SplineConv.__mro__[1]            # the reference's forward: message = the shim ops
    ei, x, ea = _inputs(w, dev)
    arms = {"fused": fused, "shim_ops": unfused}
    res = {"workload": name, **{k: v for k, v in w.items()}, "E": ei.size(1), "K": w["ks"] ** w["dim"],
           "card": _card()}
    times = {k: [] for k in arms}
    mem, outs, oom = {}, {}, {}
    for it in range(warmup + reps):
        for k, conv in arms.items():
            if k in oom:
                continue
            try:
                ms, gb, out = _timed(conv, ei, x, ea)
            except torch.cuda.OutOfMemoryError:
                oom[k] = f"out of memory at N = {x.size(0)}, E = {ei.size(1)}"
                torch.cuda.empty_cache()
                continue
            if it >= warmup:
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0.0), gb)
            outs[k] = out
    for k in arms:
        if k in oom:
            res[k] = {"oom": oom[k]}
            continue
        ops.PROFILE.reset(enabled=True)
        _step(arms[k], ei, x, ea)
        torch.cuda.synchronize()
        prof = {op: round(v["ms_total"], 3) for op, v in ops.PROFILE.summary().items()}
        ops.PROFILE.reset(enabled=False)
        res[k] = {"step_ms": round(statistics.median(times[k]), 3), "step_ms_all": [round(t, 3) for t in times[k]],
                  "peak_mem_growth_gb": round(mem[k], 3), "profile_ms": prof}
    if len(outs) == 2:
        a, b = outs["fused"].double(), outs["shim_ops"].double()
        res["max_rel_diff"] = ((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()
    if "fused" in times and "shim_ops" in times and times["fused"] and times["shim_ops"]:
        res["speedup"] = round(statistics.median(times["shim_ops"]) / statistics.median(times["fused"]), 3)
    plugin.uninstall()
    del arms, fused, unfused, ei, x, ea, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=[*WORKLOADS, "all"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    for name in (WORKLOADS if args.workload == "all" else [args.workload]):
        print(json.dumps(run(name, args.reps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
