"""QuantileAggregation / MedianAggregation: the reference against the engine's selection sweep (csrc/quantile.cu).

    python benchmarks/quantile.py [--size small|large|both] [--reps 5] [--warmup 2]

Two cases on the power-law generator of benchmarks/gen.py (uniform sources, destinations skewed towards low ids, so
hub rows and short rows both occur):
  * sage: the reference SAGEConv(F, F, aggr='median'), unpatched and under plugin.install() (lazy x_j, never gathered);
  * aggr: the standalone QuantileAggregation([0.25, 0.5, 0.75], 'linear') over [E, F] messages in caller order, the
    reference module against nn.QuantileAggregation.
Sizes: small N = 500k, E = 5M, F = 64 (the reference fits); large N = 2M, E = 20M, F = 128 (by quantile.py's ~40
bytes per message element the reference needs more than 80 GB).  Printed per arm: forward and backward ms (median of
--reps after --warmup), peak memory growth, per-kernel CUDA times of one engine step from torch.profiler
(quantile_kernel: rows up to the plan's chunk; quantile_hub_kernel: hub rows), the time of the engine's max over the
same CSR as the one-pass floor, sampled-row parity against tests/quantile_oracle.py, and the card's name, power limit
and max SM clock from nvidia-smi in the same run.  A third line per size splits the forward by in-degree tier (each
tier's rows alone; hub rows are those above the plan's chunk of 512).  One JSON line per case."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))          # the unmodified reference, installed by build()

SIZES = {"small": dict(n=500_000, e=5_000_000, f=64), "large": dict(n=2_000_000, e=20_000_000, f=128)}
Q = [0.25, 0.5, 0.75]


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _inputs(s: dict, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    n, e, f = s["n"], s["e"], s["f"]
    src = torch.randint(0, n, (e, ), device=dev, generator=g)
    dst = (torch.rand(e, device=dev, generator=g) ** 2 * (n - 1)).long()
    return torch.stack([src, dst]), torch.randn(n, f, device=dev, generator=g)


def _time(fn, reps: int, warmup: int):
    """(forward ms, backward ms, peak growth bytes) of fn() -> (output, backward closure); None when it does not fit."""
    try:
        for _ in range(warmup):
            out, bwd = fn()
            bwd(out)
        fw, bw = [], []
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        for _ in range(reps):
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            out, bwd = fn()
            e1.record()
            bwd(out)
            e2.record()
            torch.cuda.synchronize()
            fw.append(e0.elapsed_time(e1))
            bw.append(e1.elapsed_time(e2))
            del out
        return dict(fwd_ms=round(statistics.median(fw), 3), bwd_ms=round(statistics.median(bw), 3),
                    peak_growth_gib=round((torch.cuda.max_memory_allocated() - base) / 2**30, 3))
    except torch.OutOfMemoryError as exc:
        torch.cuda.empty_cache()
        return dict(error="out of memory", detail=str(exc).splitlines()[0][:160])


def _kernels(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile
    out, bwd = fn()
    bwd(out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out, bwd = fn()
        bwd(out)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t > 0:
            rows[ev.key[:60]] = round(t / 1e3, 3)
    return dict(sorted(rows.items(), key=lambda kv: -kv[1])[:10])


def _parity(out, msgs_of_row, rowptr, interp, rows: int = 64) -> dict:
    """out[i] against the oracle over sampled rows (messages in CSR slot order, ranks at the global offsets)."""
    import quantile_oracle as O
    rng = np.random.default_rng(0)
    rp = rowptr.cpu().numpy()
    deg = np.diff(rp)
    pick = np.concatenate([np.argsort(-deg)[:4], rng.choice(rp.size - 1, rows - 4, replace=False)])
    V, lens = zip(*(msgs_of_row(int(i)) for i in pick))
    sub = np.concatenate([[0], np.cumsum(lens)])
    want, _ = O.forward(sub, np.concatenate(V), np.array(Q if interp == "linear" else [0.5], np.float32), interp, 0.0,
                        False, offsets=rp[pick])
    got = out[torch.from_numpy(pick).to(out.device)].float().cpu().numpy()
    nan = np.isnan(want)
    return dict(rows=int(pick.size), max_deg=int(deg.max()), exact=bool((got[~nan] == want[~nan]).all()
                                                                         and (np.isnan(got) == nan).all()))


def _sage(s, reps, warmup, P, dev) -> dict:
    from torch_geometric.nn import SAGEConv

    import pytorch_geometric_b200.functional as Fn
    from pytorch_geometric_b200.plugin import graphs
    ei, x = _inputs(s, dev)
    f = s["f"]
    torch.manual_seed(0)
    conv = SAGEConv(f, f, aggr="median").to(dev)
    xg = x.clone().requires_grad_()

    def step():
        out = conv(xg, ei)
        return out, lambda o: o.sum().backward()
    res = {"reference": _time(step, reps, warmup)}
    P.install()
    try:
        res["engine"] = _time(step, reps, warmup)
        res["engine_kernels_ms"] = _kernels(step)
        g = graphs.graph_from_pair(ei[0], ei[1], s["n"], s["n"])
        res["floor_max_fwd_ms"] = _time(lambda: (Fn.aggregate(g, x, "max"), lambda o: None), reps, warmup)["fwd_ms"]
        aggr = conv.aggr_module
        with torch.no_grad():
            med = aggr(x[ei[0]], ei[1], dim_size=s["n"]) if s["e"] <= 5_000_000 else None
        if med is not None:
            rp, col = g.rowptr.long(), g.col.long()
            res["parity"] = _parity(med, lambda i: (x[col[rp[i]:rp[i + 1]]].cpu().numpy(), int(rp[i + 1] - rp[i])),
                                    g.rowptr, "lower")
    finally:
        P.uninstall()
    return res


def _aggr(s, reps, warmup, dev) -> dict:
    from torch_geometric.nn.aggr import QuantileAggregation as TQ

    import pytorch_geometric_b200.functional as Fn
    from pytorch_geometric_b200.graph import CSRGraph
    from pytorch_geometric_b200.nn import QuantileAggregation
    ei, _ = _inputs(s, dev)
    n, e, f = s["n"], s["e"], s["f"]
    msgs = torch.randn(e, f, device=dev, generator=torch.Generator(device=dev).manual_seed(1)).requires_grad_()
    idx = ei[1]
    res = {}
    for name, mod in (("reference", TQ(Q, "linear").to(dev)), ("engine", QuantileAggregation(Q, "linear").to(dev))):
        def step(mod=mod):
            out = mod(msgs, idx, dim_size=n)
            return out, lambda o: o.sum().backward()
        res[name] = _time(step, reps, warmup)
        if name == "engine":
            res["engine_kernels_ms"] = _kernels(step)
    g = CSRGraph(torch.arange(e, device=dev), idx, e, n)
    res["floor_max_fwd_ms"] = _time(lambda: (Fn.aggregate(g, msgs.detach(), "max"), lambda o: None), reps,
                                    warmup)["fwd_ms"]
    with torch.no_grad():
        out = QuantileAggregation(Q, "linear").to(dev)(msgs.detach(), idx, dim_size=n)
    rp, perm = g.rowptr.long(), g.perm.long()
    res["parity"] = _parity(out, lambda i: (msgs.detach()[perm[rp[i]:rp[i + 1]]].cpu().numpy(),
                                            int(rp[i + 1] - rp[i])), g.rowptr, "linear")
    return res


TIERS = ((1, 4), (5, 16), (17, 64), (65, 512), (513, None))     # in-degree tiers; above 512 the hub kernel


def _tiers(s, reps, warmup, dev) -> list:
    """Forward time per in-degree tier: each tier's rows and their messages alone, as a ptr-grouped [E_t, F] matrix,
    for the median (one selection per channel) and the three-q linear case (six), against the engine's max over the
    same rows."""
    import pytorch_geometric_b200.functional as Fn
    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200.graph import DEFAULT_CHUNK
    ei, _ = _inputs(s, dev)
    n, e, f = s["n"], s["e"], s["f"]
    deg = torch.bincount(ei[1], minlength=n)
    order = torch.argsort(ei[1], stable=True)
    dst = ei[1][order]
    msgs = torch.randn(e, f, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    out = []
    for lo, hi in TIERS:
        keep_row = (deg >= lo) & (deg <= hi if hi is not None else torch.ones_like(deg, dtype=torch.bool))
        keep = keep_row[dst]
        m = msgs[keep].contiguous()
        ptr = torch.cat([deg.new_zeros(1), torch.cumsum(deg[keep_row], 0)])
        plan = ops.LongRowPlan(ptr, DEFAULT_CHUNK)
        row = dict(tier=f"{lo}-{hi if hi is not None else 'max'}", rows=int(keep_row.sum()), edges=int(m.size(0)))
        for name, q, interp in (("median", 0.5, "lower"), ("q3_linear", Q, "linear")):
            qt = torch.tensor(q if isinstance(q, list) else [q], device=dev)
            row[f"{name}_fwd_ms"] = _time(lambda: (Fn.quantile_aggregate((ptr, plan), None, m, qt, interp),
                                                   lambda o: None), reps, warmup)["fwd_ms"]
        row["max_fwd_ms"] = _time(lambda: (Fn.segment(m, ptr, "max"), lambda o: None), reps, warmup)["fwd_ms"]
        out.append(row)
        del m
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", choices=["small", "large", "both"], default="both")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from pytorch_geometric_b200 import plugin as P
    dev = torch.device("cuda")
    card = _card()
    for size in (("small", "large") if args.size == "both" else (args.size, )):
        s = SIZES[size]
        for case in ("sage", "aggr"):
            res = _sage(s, args.reps, args.warmup, P, dev) if case == "sage" else _aggr(s, args.reps, args.warmup,
                                                                                         dev)
            print(json.dumps(dict(case=case, size=size, **s, card=card, **res)), flush=True)
            torch.cuda.empty_cache()
        print(json.dumps(dict(case="tiers", size=size, **s, card=card,
                              tiers=_tiers(s, args.reps, args.warmup, dev))), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
