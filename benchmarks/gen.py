"""GENConv, forward + backward, fused (`plugin.conv.B200GENConv`) against the reference's own CUDA path.

    python benchmarks/gen.py [--workload proteins|power_law|both] [--reps 5] [--warmup 2]

Two workloads:
  * proteins: a synthetic graph at ogbn-proteins' size (N = 132,534 nodes, E = 79.1M directed edges with skewed
    in-degrees), F = 64, the DeeperGCN example's layer: aggr='softmax', learn_t=True, num_layers=2, norm='layer'.  x and
    a leaf edge_attr [E, 64] (standing in for the shared edge encoder's output) both require grad;
  * power_law: N = 2M, E = 10M skewed in-degrees, F = 128, aggr='powermean', learn_p=True, no edge features.

The model is an UNMODIFIED reference `GENConv` (oracle/_ref).  The fused arm first runs alone at full size (its step
time and peak memory growth).  Then both arms run in one process, alternated rep by rep after warm-up: "fused" is the
same module with its class switched to `B200GENConv` (plug-in installed), "reference" the reference class with the
plug-in uninstalled.  If the reference arm runs out of memory, that size is recorded and both arms run again at half
the nodes and edges until the reference fits.  Prints one JSON line per workload: ms for forward / backward / step
(median over reps), the peak `torch.cuda.max_memory_allocated` growth of a step per arm, the engine's per-kernel time
from `ops.PROFILE` (a separate profiled step) with the bytes each kernel must move -- computed from shapes -- over
that time against the H100 SXM data sheet's 3.35 TB/s, sampled-row parity of the aggregation against an fp64 formula
for both arms, and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
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

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {"proteins": dict(n=132_534, e=79_122_504, f=64, edge=True,
                              kw=dict(aggr="softmax", learn_t=True, num_layers=2, norm="layer")),
             "power_law": dict(n=2_000_000, e=10_000_000, f=128, edge=False,
                               kw=dict(aggr="powermean", learn_p=True))}


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _inputs(w: dict, n: int, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    e = w["e"] * n // w["n"]
    src = torch.randint(0, n, (e, ), device=dev, generator=g)
    dst = (torch.rand(e, device=dev, generator=g) ** 2 * (n - 1)).long()       # skewed in-degrees, hub rows included
    x = torch.randn(n, w["f"], device=dev, generator=g)
    ea = torch.randn(e, w["f"], device=dev, generator=g) if w["edge"] else None
    gout = torch.randn(n, w["f"], device=dev, generator=g)
    return torch.stack([src, dst]), x, ea, gout


class _Capture:
    """The MLP's input of the last forward: the aggregation plus the residual x."""

    def __init__(self, model):
        self.mlp_in = None
        model.mlp.register_forward_pre_hook(lambda mod, inp: setattr(self, "mlp_in", inp[0].detach()))


def _clear(model, x, ea):
    """Drop the last step's gradients, so that a step's peak growth counts the ones it allocates."""
    x.grad = None
    if ea is not None:
        ea.grad = None
    model.zero_grad(set_to_none=True)


def _step(model, x, ei, ea, gout):
    _clear(model, x, ea)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    out = model(x, ei, ea)
    ev[1].record()
    out.backward(gout)
    ev[2].record()
    torch.cuda.synchronize()
    return out, (ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[2]))


def _parity(model, x, ei, ea, agg, rows: int = 64) -> dict:
    """max |err| / max |ref| of the aggregation on sampled destination rows against fp64: m = relu(x_j (+ e_ji)) + eps,
    then sum softmax(t m) m, or clamp(mean clamp(m)^p)^(1/p)."""
    dev = x.device
    n = x.size(0)
    src, dst = ei[0], ei[1]
    g = torch.Generator(device=dev).manual_seed(1)
    pick = torch.unique(torch.cat([torch.randint(0, n, (rows, ), device=dev, generator=g),
                                   torch.tensor([0, 1], device=dev)]))
    sel = torch.isin(dst, pick)
    s_, d_ = src[sel], dst[sel]
    m = x.detach().double()[s_]
    if ea is not None:
        m = m + ea.detach().double()[sel]
    m = m.relu() + model.eps
    loc = torch.searchsorted(pick, d_)
    k = pick.numel()
    idx = loc.view(-1, 1).expand_as(m)
    a = model.aggr_module
    if hasattr(a, "t"):
        z = m * a.t.detach().double() if hasattr(a.t, "detach") else m * a.t
        mx = torch.full((k, m.size(1)), -float("inf"), dtype=torch.float64, device=dev).scatter_reduce(0, idx, z, "amax")
        ex = (z - mx[loc]).exp()
        den = torch.zeros(k, m.size(1), dtype=torch.float64, device=dev).index_add_(0, loc, ex)
        want = torch.zeros_like(den).index_add_(0, loc, ex * m) / den.clamp(min=1e-300)
    else:
        p = a.p.detach().double() if hasattr(a.p, "detach") else float(a.p)
        y = m.clamp(min=a.min_value, max=a.max_value).pow(p)
        cnt = torch.bincount(loc, minlength=k).clamp(min=1).double().view(-1, 1)
        mean = torch.zeros(k, m.size(1), dtype=torch.float64, device=dev).index_add_(0, loc, y) / cnt
        want = mean.clamp(min=a.min_value, max=a.max_value).pow(1.0 / p)
    return {"rows": int(k), "agg_rel_err": float((agg[pick].double() - want).abs().max() / want.abs().max())}


def _bytes(kernel_names, n: int, e: int, f: int, s: int, edge: bool) -> dict:
    """Bytes each engine kernel must move, from shapes: R = F s per feature row, int32 indices, a sorted CSR (perm)."""
    r = f * s
    er = r + 4 if edge else 0                                        # edge row and its perm entry
    table = {
        "softmax_aggr_csr": e * (r + 4 + er) + n * (r + 4 * f),      # x row, col (+ edge row) per edge; out, lse
        "softmax_aggr_backward_dst": e * (r + 4 + 2 * er) + n * (2 * r + 4 * f),   # (+ grad_a written); g, out, lse
        "power_mean_csr": e * (r + 4 + er) + n * (r + 4 * f),        # x row, col (+ edge row) per edge; out, M
        "power_mean_backward_dst": e * (r + 4 + 2 * er) + n * (2 * r + 4 * f),
        "power_mean_backward_src": e * (4 * f + 4 + er) + n * (2 * r + 8 * f) + n * 2 * r,   # G row, col_t per edge;
        "spmm_csr": e * (r + 4) + n * r,                             # node plane; x read, grad_x written
    }
    return {k: table[k] for k in kernel_names if k in table}


def _model(tg, w, dev):
    torch.manual_seed(0)
    ref = tg.nn.GENConv(w["f"], w["f"], **w["kw"]).to(dev)
    with torch.no_grad():
        for name, prm in ref.named_parameters():
            if name in ("aggr_module.t", "aggr_module.p"):
                prm.fill_(1.5)
    return ref


def _fused_alone(w, n, reps, warmup, tg, P, dev) -> dict:
    from pytorch_geometric_b200.plugin import conv as PC
    ei, x0, ea, gout = _inputs(w, n, dev)
    fused = _model(tg, w, dev)
    fused.__class__ = PC.B200GENConv
    P.install()
    x = x0.clone().requires_grad_()
    if ea is not None:
        ea.requires_grad_()
    for _ in range(warmup):
        _step(fused, x, ei, ea, gout)
    times, peak = [], 0
    for _ in range(reps):
        _clear(fused, x, ea)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out, t = _step(fused, x, ei, ea, gout)
        peak = max(peak, torch.cuda.max_memory_allocated() - base)
        times.append(t)
        del out
    P.uninstall()
    return {"N": n, "E": ei.size(1), "step_ms": statistics.median(t[2] for t in times),
            "fwd_ms": statistics.median(t[0] for t in times), "bwd_ms": statistics.median(t[1] for t in times),
            "max_memory_allocated_bytes": peak}


def _run(wname: str, w: dict, n: int, reps: int, warmup: int, tg, P, ops, dev) -> dict:
    from pytorch_geometric_b200.plugin import conv as PC
    ei, x0, ea, gout = _inputs(w, n, dev)
    ref = _model(tg, w, dev)
    fused = copy.deepcopy(ref)
    fused.__class__ = PC.B200GENConv
    models = {"fused": fused, "reference": ref}
    caps = {a: _Capture(m) for a, m in models.items()}
    x = x0.clone().requires_grad_()
    if ea is not None:
        ea.requires_grad_()

    def arm(name):
        if name == "fused":
            if not P.installed():
                P.install()
        else:
            P.uninstall()

    arms = ("fused", "reference")
    times = {a: [] for a in arms}
    peak, parity = {}, {}
    for a in arms:                                    # warm-up (graph build, allocator, library algorithms)
        arm(a)
        for _ in range(warmup):
            _step(models[a], x, ei, ea, gout)
    for _ in range(reps):
        for a in arms:
            arm(a)
            _clear(models[a], x, ea)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out, t = _step(models[a], x, ei, ea, gout)
            peak[a] = max(peak.get(a, 0), torch.cuda.max_memory_allocated() - base)
            times[a].append(t)
            if a not in parity:
                parity[a] = _parity(models[a], x, ei, ea, caps[a].mlp_in - x.detach())
            del out
    arm("fused")
    ops.PROFILE.reset(enabled=True)
    _step(fused, x, ei, ea, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    P.uninstall()
    e = ei.size(1)
    bytes_needed = _bytes(prof.keys(), n, e, w["f"], x.element_size(), w["edge"])
    kernels = {}
    for k, nbytes in bytes_needed.items():
        ms = prof[k]["ms_total"]
        kernels[k] = {"ms": ms, "bytes": nbytes, "bytes_per_s": nbytes / (ms * 1e-3),
                      "share_of_3.35TBps": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    med = {a: {k: statistics.median(t[i] for t in times[a]) for i, k in enumerate(("fwd_ms", "bwd_ms", "step_ms"))}
           for a in arms}
    return {"bench": "gen", "workload": wname, "N": n, "E": e, "F": w["f"], "layer": w["kw"], "dtype": "float32",
            "reps": reps, "warmup": warmup, "ms": med, "ms_all": times, "max_memory_allocated_bytes": peak,
            "speedup_step": med["reference"]["step_ms"] / med["fused"]["step_ms"], "kernels": kernels,
            "other_engine_ops_ms": {k: v["ms_total"] for k, v in prof.items() if k not in bytes_needed},
            "parity": parity}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["proteins", "power_law", "both"], default="both")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gen.py measures on a CUDA GPU; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200 import plugin as P

    dev = torch.device("cuda")
    card = _card()
    for wname in (("proteins", "power_law") if args.workload == "both" else (args.workload, )):
        w = WORKLOADS[wname]
        full = _fused_alone(w, w["n"], args.reps, args.warmup, tg, P, dev)
        torch.cuda.empty_cache()
        n, oom_at = w["n"], []
        while True:
            try:
                res = _run(wname, w, n, args.reps, args.warmup, tg, P, ops, dev)
                break
            except torch.cuda.OutOfMemoryError:
                P.uninstall()
                oom_at.append(n)
                n //= 2
                torch.cuda.empty_cache()
        res["fused_alone_full_size"] = full
        res["reference_out_of_memory_at_N"] = oom_at
        res["gpu"] = card
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
