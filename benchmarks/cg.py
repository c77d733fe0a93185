"""CGConv, forward + backward, fused (`plugin.conv.B200CGConv`) against the reference's own CUDA path.

    python benchmarks/cg.py [--workload crystal|power_law|both] [--reps 5] [--warmup 2]

Two workloads:
  * crystal: N = 1M atoms, 12 in-edges each, F = 64, dim = 41 (CGCNN's Gaussian distance expansion), sum,
    batch_norm=True; x requires grad, edge_attr does not (its weight block does, so c and grad_c exist);
  * power_law: N = 2M, E = 10M skewed in-degrees, F = 128, dim = 0, mean.

The model is an UNMODIFIED reference `CGConv` (oracle/_ref).  Two arms in one process, alternated rep by rep after
warm-up: "fused" is the same module with its class switched to `B200CGConv` (plug-in installed), "reference" the
reference class with the plug-in uninstalled (x_i / x_j gathers, cat, two Linears over E rows, sigmoid, softplus, mul and
scatter as ATen kernels).  If the reference arm runs out of memory, that is recorded and both arms are run again at
half the nodes and edges until the reference fits.  Prints one JSON line per workload: ms for forward / backward / step
(median over reps), the peak `torch.cuda.max_memory_allocated` growth of a step for each arm, the engine's per-kernel
time from `ops.PROFILE` (a separate profiled step) with the bytes each kernel must move -- computed from shapes -- over
that time against the H100 SXM data sheet's 3.35 TB/s, sampled-row parity of the aggregated message against an fp64
formula for both arms, and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))          # the unmodified reference, installed by build()

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {"crystal": dict(n=1_000_000, deg=12, f=64, dim=41, aggr="add", batch_norm=True),
             "power_law": dict(n=2_000_000, e=10_000_000, f=128, dim=0, aggr="mean", batch_norm=False)}


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _inputs(w: dict, n: int, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    f, dim = w["f"], w["dim"]
    if "deg" in w:                                    # every atom has exactly `deg` neighbours
        dst = torch.arange(n, device=dev).repeat_interleave(w["deg"])
        src = torch.randint(0, n, (dst.numel(), ), device=dev, generator=g)
    else:
        e = w["e"] * n // w["n"]
        src = torch.randint(0, n, (e, ), device=dev, generator=g)
        dst = (torch.rand(e, device=dev, generator=g) ** 2 * (n - 1)).long()  # skewed in-degrees, hub rows included
    x = torch.randn(n, f, device=dev, generator=g)
    ea = torch.rand(src.numel(), dim, device=dev, generator=g) if dim else None
    gout = torch.randn(n, f, device=dev, generator=g)
    return torch.stack([src, dst]), x, ea, gout


class _Capture:
    """The aggregated message of the last forward: BatchNorm's input, or out - x without BatchNorm."""

    def __init__(self, model):
        self.agg = None
        if model.bn is not None:
            model.bn.register_forward_pre_hook(lambda mod, inp: setattr(self, "agg", inp[0].detach()))


def _step(model, x, ei, ea, gout):
    x.grad = None
    model.zero_grad(set_to_none=True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    out = model(x, ei, ea)
    ev[1].record()
    out.backward(gout)
    ev[2].record()
    torch.cuda.synchronize()
    return out, (ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[2]))


def _parity(model, x, ei, ea, agg, mean: bool, rows: int = 64) -> dict:
    """max |err| / max |ref| of the aggregated message on sampled destination rows against fp64:
    agg_i = REDUCE_{e: j -> i} sigmoid(z W_f^T + b_f) * softplus(z W_s^T + b_s), z = [x_i, x_j, e_ji]."""
    dev = x.device
    n = x.size(0)
    src, dst = ei[0], ei[1]
    g = torch.Generator(device=dev).manual_seed(1)
    pick = torch.unique(torch.cat([torch.randint(0, n, (rows, ), device=dev, generator=g),
                                   torch.tensor([0, 1], device=dev)]))
    xd = x.detach().double()
    sel = torch.isin(dst, pick)
    s_, d_ = src[sel], dst[sel]
    z = torch.cat([xd[d_], xd[s_]] + ([ea[sel].double()] if ea is not None else []), 1)
    lin = lambda m: z @ m.weight.detach().double().T + (0 if m.bias is None else m.bias.detach().double())  # noqa: E731
    m = torch.sigmoid(lin(model.lin_f)) * F.softplus(lin(model.lin_s))
    loc = torch.searchsorted(pick, d_)
    want = torch.zeros(pick.numel(), x.size(1), dtype=torch.float64, device=dev).index_add_(0, loc, m)
    if mean:
        want = want / torch.bincount(loc, minlength=pick.numel()).clamp(min=1).double().view(-1, 1)
    return {"rows": int(pick.numel()),
            "agg_rel_err": float((agg[pick].double() - want).abs().max() / want.abs().max())}


def _bytes(kernel_names, n: int, e: int, f: int, s: int, has_c: bool, mean: bool) -> dict:
    """Bytes each engine kernel must move, from shapes: R = F s per feature row, int32 indices, a sorted CSR (perm)."""
    r = f * s
    ce = 2 * r + 4 if has_c else 0                              # c row and its perm entry
    table = {
        "cg_csr": e * (2 * r + 4 + ce) + n * 3 * r,             # v, col (+ c) per edge; u read, out written per row
        "cg_backward_dst": e * (2 * r + 4 + ce + (2 * r if has_c else 0)) + n * 5 * r,   # (+ grad_c written); u, g, grad_u
        "cg_backward_src": e * (3 * r + 4 + (4 if mean else 0) + ce) + n * 4 * r,       # u, g, col_t (val_t, c); v, grad_v
        "spmm_csr": e * (2 * r + 4) + n * 2 * r,                # grad_c rows and perm_t per edge; grad_v written
    }
    return {k: table[k] for k in kernel_names if k in table}


def _run(wname: str, w: dict, n: int, reps: int, warmup: int, tg, P, ops, dev) -> dict:
    ei, x0, ea, gout = _inputs(w, n, dev)
    torch.manual_seed(0)
    ref = tg.nn.CGConv(w["f"], dim=w["dim"], aggr=w["aggr"], batch_norm=w["batch_norm"]).to(dev)
    from pytorch_geometric_b200.plugin import conv as PC
    fused = copy.deepcopy(ref)
    fused.__class__ = PC.B200CGConv
    models = {"fused": fused, "reference": ref}
    caps = {a: _Capture(m) for a, m in models.items()}
    x = x0.clone().requires_grad_()

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
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out, t = _step(models[a], x, ei, ea, gout)
            peak[a] = max(peak.get(a, 0), torch.cuda.max_memory_allocated() - base)
            times[a].append(t)
            if a not in parity:
                agg = caps[a].agg if models[a].bn is not None else (out.detach() - x.detach())
                parity[a] = _parity(models[a], x, ei, ea, agg, w["aggr"] == "mean")
            del out
    arm("fused")
    ops.PROFILE.reset(enabled=True)
    _step(fused, x, ei, ea, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    P.uninstall()
    e = ei.size(1)
    bytes_needed = _bytes(prof.keys(), n, e, w["f"], x.element_size(), w["dim"] > 0, w["aggr"] == "mean")
    kernels = {}
    for k, nbytes in bytes_needed.items():
        ms = prof[k]["ms_total"]
        kernels[k] = {"ms": ms, "bytes": nbytes, "bytes_per_s": nbytes / (ms * 1e-3),
                      "share_of_3.35TBps": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    med = {a: {k: statistics.median(t[i] for t in times[a]) for i, k in enumerate(("fwd_ms", "bwd_ms", "step_ms"))}
           for a in arms}
    return {"bench": "cg", "workload": wname, "N": n, "E": e, "F": w["f"], "dim": w["dim"], "aggr": w["aggr"],
            "batch_norm": w["batch_norm"], "dtype": "float32", "reps": reps, "warmup": warmup, "ms": med,
            "ms_all": times, "max_memory_allocated_bytes": peak,
            "speedup_step": med["reference"]["step_ms"] / med["fused"]["step_ms"], "kernels": kernels,
            "other_engine_ops_ms": {k: v["ms_total"] for k, v in prof.items() if k not in bytes_needed},
            "parity": parity}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["crystal", "power_law", "both"], default="both")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/cg.py measures on a CUDA GPU; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200 import plugin as P

    dev = torch.device("cuda")
    card = _card()
    for wname in (("crystal", "power_law") if args.workload == "both" else (args.workload, )):
        w = WORKLOADS[wname]
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
        res["reference_out_of_memory_at_N"] = oom_at
        res["gpu"] = card
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
