"""NNConv (ECConv), forward + backward, fused (`plugin.conv.B200NNConv`) against the reference's own CUDA path.

    python benchmarks/nn_conv.py [--workload qm9|power_law|both] [--reps 5] [--warmup 2]

Two workloads, chosen for the two regimes of the sweep:
  * qm9: 128 complete 18-atom graphs (N = 2304, E = 39168, in-degree 17), D = 5 edge features, edge network
    Linear(5, 128) -> ReLU -> Linear(128, 64 * 64), F = 64, mean: many short rows, (K+1) F_in = 8256 (the layer of the
    reference's examples/qm9_nn_conv.py);
  * power_law: N = 200k, E = 4M with skewed in-degrees (hub rows split by the long-row plan), D = 8, edge network
    Linear(8, 64) -> ReLU -> Linear(64, 64 * 64), F = 64, sum.

The model is an UNMODIFIED reference `NNConv` (oracle/_ref).  Two arms in one process, alternated rep by rep after
warm-up: "fused" is the same module with its class switched to `B200NNConv` (plug-in installed), "reference" the
reference class with the plug-in uninstalled (the edge network's [E, F_in F_out] output, the gathered x_j, a batched
matmul and scatter as ATen kernels).  Whenever an arm runs out of memory, the arm and the N and E it ran at are recorded
and both arms are run again at half the nodes and edges.  Prints one JSON line per workload: ms for forward / backward / step (median over
reps), the peak `torch.cuda.max_memory_allocated` growth of a step for each arm, the engine's per-kernel time from
`ops.PROFILE` (a separate profiled step) with the FLOPs and bytes each kernel must handle -- computed from shapes -- over
that time against the H100 SXM data sheet's 67 TFLOP/s FP32 and 3.35 TB/s, sampled-row parity of each arm's output
against an fp64 formula, and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
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
FP32_FLOP_PER_S = 67e12
WORKLOADS = {"qm9": dict(graphs=128, atoms=18, d=5, k=128, f=64, aggr="mean"),
             "power_law": dict(n=200_000, e=4_000_000, d=8, k=64, f=64, aggr="add")}


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _inputs(w: dict, scale: int, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    if "graphs" in w:                                 # complete directed graphs without self-loops
        a = w["atoms"]
        loc = torch.cartesian_prod(torch.arange(a), torch.arange(a)).to(dev)
        loc = loc[loc[:, 0] != loc[:, 1]]
        off = (torch.arange(w["graphs"] // scale, device=dev) * a).repeat_interleave(loc.size(0))
        ei = (loc.repeat(w["graphs"] // scale, 1) + off[:, None]).T.contiguous()
        n = a * (w["graphs"] // scale)
    else:
        n, e = w["n"] // scale, w["e"] // scale
        src = torch.randint(0, n, (e, ), device=dev, generator=g)
        dst = (torch.rand(e, device=dev, generator=g) ** 2 * (n - 1)).long()   # skewed in-degrees, hub rows included
        ei = torch.stack([src, dst])
    x = torch.randn(n, w["f"], device=dev, generator=g)
    ea = torch.rand(ei.size(1), w["d"], device=dev, generator=g)
    gout = torch.randn(n, w["f"], device=dev, generator=g)
    return ei, x, ea, gout


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


def _parity(model, x, ei, ea, out, mean: bool, rows: int = 64) -> dict:
    """max |err| / max |ref| of the layer output on sampled destination rows against fp64:
    out_i = x_i Theta + REDUCE_{e: j -> i} x_j reshape(nn(e_ji), [F_in, F_out]) + bias."""
    dev = x.device
    n = x.size(0)
    src, dst = ei[0], ei[1]
    g = torch.Generator(device=dev).manual_seed(1)
    pick = torch.unique(torch.cat([torch.randint(0, n, (rows, ), device=dev, generator=g),
                                   torch.tensor([0, 1], device=dev)]))
    sel = torch.isin(dst, pick)
    s_, d_ = src[sel], dst[sel]
    net = copy.deepcopy(model.nn).double()
    xd = x.detach().double()
    with torch.no_grad():
        w_e = net(ea[sel].double()).view(-1, model.in_channels_l, model.out_channels)
        msg = torch.bmm(xd[s_].unsqueeze(1), w_e).squeeze(1)
        loc = torch.searchsorted(pick, d_)
        want = torch.zeros(pick.numel(), model.out_channels, dtype=torch.float64, device=dev).index_add_(0, loc, msg)
        if mean:
            want = want / torch.bincount(loc, minlength=pick.numel()).clamp(min=1).double().view(-1, 1)
        want = want + xd[pick] @ model.lin.weight.detach().double().T + model.bias.detach().double()
    return {"rows": int(pick.numel()), "out_rel_err": float((out[pick].double() - want).abs().max() / want.abs().max())}


def _work(kernel_names, n: int, e: int, k: int, f: int, f_out: int, s: int) -> dict:
    """(FLOPs, bytes) each engine kernel must handle in one step, summed over its calls, from shapes: M = (K+1) F_in fp32
    columns of P, int32 indices and a sorted CSR (perm).  The forward sweep runs twice per step (forward, and the
    backward's recompute of P for dW'); each GEMM runs once per step over all destination rows."""
    m = (k + 1) * f
    gemm = (2 * n * m * f_out, 4 * (n * m + n * f_out + m * f_out))
    table = {
        "nn_conv_csr": (2 * 2 * e * m, 2 * (e * ((f + k) * s + 8) + 4 * n * m)),           # x_j, h_e, col, perm; P
        "nn_conv_backward_dst": (4 * e * m, e * (2 * (f + k) * s + 8) + 4 * n * m),       # + grad_h, q; dP
        "spmm_csr": (e * f, e * (f * s + 4) + n * f * s),                                 # q rows, perm_t; grad_x
        "linear_grad_input_tf32x3": gemm, "linear_tf32x3": gemm, "linear_grad_weight_tf32x3": gemm,
    }
    return {name: table[name] for name in kernel_names if name in table}


class _ArmOutOfMemory(Exception):
    def __init__(self, arm: str, n: int, e: int):
        super().__init__(f"{arm} arm out of memory at N = {n}, E = {e}")
        self.record = {"arm": arm, "N": n, "E": e}


def _run(wname: str, w: dict, scale: int, reps: int, warmup: int, tg, P, ops, dev) -> dict:
    ei, x0, ea, gout = _inputs(w, scale, dev)
    n, e, f, k = x0.size(0), ei.size(1), w["f"], w["k"]
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(w["d"], k), torch.nn.ReLU(), torch.nn.Linear(k, f * f))
    ref = tg.nn.NNConv(f, f, net, aggr=w["aggr"]).to(dev)
    with torch.no_grad():
        ref.bias.normal_()
    from pytorch_geometric_b200.plugin import conv as PC
    fused = copy.deepcopy(ref)
    fused.__class__ = PC.B200NNConv
    models = {"fused": fused, "reference": ref}
    x = x0.clone().requires_grad_()
    current = {}

    def arm(name):
        current["arm"] = name
        if name == "fused":
            if not P.installed():
                P.install()
        else:
            P.uninstall()

    try:
        return _measure(wname, w, n, e, k, f, models, x, ei, ea, gout, reps, warmup, arm, P, ops)
    except torch.cuda.OutOfMemoryError:
        raise _ArmOutOfMemory(current.get("arm"), n, e) from None


def _measure(wname, w, n, e, k, f, models, x, ei, ea, gout, reps, warmup, arm, P, ops) -> dict:
    fused = models["fused"]
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
                parity[a] = _parity(models[a], x, ei, ea, out.detach(), w["aggr"] == "mean")
            del out
    arm("fused")
    ops.PROFILE.reset(enabled=True)
    _step(fused, x, ei, ea, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    P.uninstall()
    work = _work(prof.keys(), n, e, k, f, f, x.element_size())
    kernels = {}
    for name, (flops, nbytes) in work.items():
        sec = prof[name]["ms_total"] * 1e-3
        t_flop, t_byte = flops / FP32_FLOP_PER_S, nbytes / HBM_BYTES_PER_S
        kernels[name] = {"ms": prof[name]["ms_total"], "calls": prof[name]["calls"], "flops": flops, "bytes": nbytes,
                         "flop_per_s": flops / sec, "bytes_per_s": nbytes / sec,
                         "bound": "fp32" if t_flop >= t_byte else "hbm", "share_of_bound": max(t_flop, t_byte) / sec}
    med = {a: {key: statistics.median(t[i] for t in times[a]) for i, key in enumerate(("fwd_ms", "bwd_ms", "step_ms"))}
           for a in arms}
    return {"bench": "nn_conv", "workload": wname, "N": n, "E": e, "D": w["d"], "K": k, "F": f, "aggr": w["aggr"],
            "dtype": "float32", "reps": reps, "warmup": warmup, "ms": med, "ms_all": times,
            "max_memory_allocated_bytes": peak,
            "reference_edge_weight_bytes": e * f * f * 4,
            "speedup_step": med["reference"]["step_ms"] / med["fused"]["step_ms"], "kernels": kernels,
            "other_engine_ops_ms": {key: v["ms_total"] for key, v in prof.items() if key not in work},
            "parity": parity}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["qm9", "power_law", "both"], default="both")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/nn_conv.py measures on a CUDA GPU; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200 import plugin as P

    dev = torch.device("cuda")
    card = _card()
    for wname in (("qm9", "power_law") if args.workload == "both" else (args.workload, )):
        w = WORKLOADS[wname]
        scale, oom_at = 1, []
        while True:
            try:
                res = _run(wname, w, scale, args.reps, args.warmup, tg, P, ops, dev)
                break
            except _ArmOutOfMemory as oom:
                P.uninstall()
                oom_at.append(oom.record)
                scale *= 2
                torch.cuda.empty_cache()
        res["out_of_memory_at"] = oom_at
        res["gpu"] = card
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
