"""PNAConv (the layer of examples/pna.py), forward + backward, fused against the reference's own CUDA path.

    python benchmarks/pna.py [--mol-nodes 250000] [--pl-nodes 1000000] [--pl-edges 5000000] [--reps 5] [--warmup 2]

The layer is an UNMODIFIED reference `PNAConv(75, 75, [mean, min, max, std], [identity, amplification, attenuation],
deg, edge_dim=50, towers=5, pre_layers=1, post_layers=1, divide_input=False)` (oracle/_ref) with x and edge_attr
requiring grad.  Two graphs:
  (a) molecule-like: in-degree 1-4 per node, 250k nodes by default: at 1M nodes the reference arm runs out of memory
      on an 80 GB H100 (reported as "out of memory"; the fused arm fits).  Two arms alternated rep by rep after warm-up: "fused" (the same module
      with its class set to `plugin.conv.B200PNAConv`) and "reference" (its own forward).  Step time (median) and the
      peak `max_memory_allocated` growth of a step for each arm, and the max |fused - reference| of the output.
  (b) power-law: N nodes, E edges with skewed in-degrees (1M / 5M by default: at 10M edges the fused step itself needs
      more than 80 GB -- the [E, T F] edge products c and grad_c, the edge encoder's [E, F] rows and their gradients); fused only, with the engine's per-kernel time from
      `ops.PROFILE` (a separate profiled step), the bytes each kernel must move -- computed from shapes -- and their
      ratio to the H100 SXM data sheet's 3.35 TB/s.
Prints one JSON line with the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
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
AGGRS = ["mean", "min", "max", "std"]
SCALERS = ["identity", "amplification", "attenuation"]
F, T, EDGE_DIM = 75, 5, 50


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _molecule(n: int, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    k = torch.randint(1, 5, (n, ), device=dev, generator=g)                    # in-degree 1..4
    dst = torch.repeat_interleave(torch.arange(n, device=dev), k)
    src = (dst + torch.randint(1, 30, dst.shape, device=dev, generator=g)) % n  # nearby atoms
    return torch.stack([src, dst])


def _power_law(n: int, e: int, dev):
    g = torch.Generator(device=dev).manual_seed(1)
    src = torch.randint(0, n, (e, ), device=dev, generator=g)
    dst = (torch.rand(e, device=dev, generator=g) ** 3 * (n - 1)).long()
    return torch.stack([src, dst])


def _layer(tg, ei, n, dev):
    deg = torch.bincount(torch.bincount(ei[1], minlength=n)).cpu()
    torch.manual_seed(0)
    return tg.nn.PNAConv(F, F, AGGRS, SCALERS, deg, edge_dim=EDGE_DIM, towers=T, pre_layers=1, post_layers=1,
                         divide_input=False).to(dev)


def _step(model, x, ei, ea, gout):
    x.grad = ea.grad = None
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = model(x, ei, ea)
    out.backward(gout)
    e1.record()
    torch.cuda.synchronize()
    return out.detach(), e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def _bytes(name: str, n: int, e: int) -> float:
    """Bytes a kernel must move at least, from shapes (fp32, int32 indices, W = T F): every distinct row once -- the
    per-edge c rows and indices, and each node's rows a single time however many edges revisit them."""
    W = T * F
    A, S = len(AGGRS), len(SCALERS)
    blk = n * T * (1 + A * S) * F * 4
    if name == "pna_edge_stats":          # col + perm and a c row per edge; v rows; 6 statistic planes written
        return e * (8 + W * 4) + n * W * 4 + n * 6 * W * 4
    if name == "pna_edge_backward":       # col_t + perm_t, a c row read and a grad_c row written per edge; v read and
        return e * (8 + 2 * W * 4) + n * 2 * W * 4 + n * 6 * W * 4   # grad_v written per source; 6 destination rows
    if name == "pna_epilogue":            # 4 stat planes + u + x in, the block out
        return n * 6 * W * 4 + blk
    if name == "pna_prologue":            # block gradient + 6 stat planes + u in, 4 term rows + grad_u + grad_x out
        return blk + n * 7 * W * 4 + n * 6 * W * 4
    return 0.0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--mol-nodes", type=int, default=250_000)
    ap.add_argument("--pl-nodes", type=int, default=1_000_000)
    ap.add_argument("--pl-edges", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/pna.py measures on a CUDA device; none is visible")
    import torch_geometric as tg

    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200.plugin import conv as PC
    dev = torch.device("cuda")
    res = {"card": _card(), "layer": f"PNAConv({F}, {F}, towers={T}, edge_dim={EDGE_DIM}) {AGGRS} x {SCALERS}"}

    # (a) molecule-like batch, fused against the reference's CUDA path
    n = args.mol_nodes
    ei = _molecule(n, dev)
    ref = _layer(tg, ei, n, dev)
    fused = copy.deepcopy(ref)
    fused.__class__ = PC.B200PNAConv
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(n, F, device=dev, generator=g).requires_grad_()
    ea = torch.randn(ei.size(1), EDGE_DIM, device=dev, generator=g).requires_grad_()
    gout = torch.randn(n, F, device=dev, generator=g)
    arms = {"fused": fused, "reference": ref}
    times = {k: [] for k in arms}
    mem = {}
    outs = {}
    oom = set()
    for rep in range(args.warmup + args.reps):
        for k, mod in arms.items():
            if k in oom:
                continue
            try:
                out, ms, grow = _step(mod, x, ei, ea, gout)
            except torch.OutOfMemoryError:           # an arm that does not fit on the card is reported as such
                oom.add(k)
                x.grad = ea.grad = None
                mod.zero_grad(set_to_none=True)
                torch.cuda.empty_cache()
                continue
            if rep >= args.warmup:
                times[k].append(ms)
                mem[k] = max(mem.get(k, 0), grow)
            outs[k] = out
    res["molecule"] = {"nodes": n, "edges": ei.size(1)}
    for k in arms:
        res["molecule"][f"{k}_step_ms"] = "out of memory" if k in oom else statistics.median(times[k])
        res["molecule"][f"{k}_peak_growth_gb"] = "out of memory" if k in oom else mem[k] / 1e9
    if not oom:
        res["molecule"]["max_abs_diff_out"] = (outs["fused"] - outs["reference"]).abs().max().item()
        res["molecule"]["speedup"] = res["molecule"]["reference_step_ms"] / res["molecule"]["fused_step_ms"]
    del arms, ref, fused, x, ea, gout, outs
    torch.cuda.empty_cache()

    # (b) power-law graph, engine only, per-kernel time and bandwidth
    n, e = args.pl_nodes, args.pl_edges
    ei = _power_law(n, e, dev)
    mod = _layer(tg, ei, n, dev)
    mod.__class__ = PC.B200PNAConv
    x = torch.randn(n, F, device=dev, generator=g).requires_grad_()
    ea = torch.randn(e, EDGE_DIM, device=dev, generator=g).requires_grad_()
    gout = torch.randn(n, F, device=dev, generator=g)
    steps = []
    try:
        for rep in range(args.warmup + args.reps):
            _, ms, grow = _step(mod, x, ei, ea, gout)
            if rep >= args.warmup:
                steps.append(ms)
    except torch.OutOfMemoryError:
        res["power_law"] = {"nodes": n, "edges": e, "fused_step_ms": "out of memory"}
        print(json.dumps(res))
        return
    ops.PROFILE.reset(enabled=True)
    _step(mod, x, ei, ea, gout)
    prof = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    kernels = {}
    for name in ("pna_edge_stats", "pna_epilogue", "pna_prologue", "pna_edge_backward"):
        if name in prof:
            ms = prof[name]["ms_total"]
            b = _bytes(name, n, e)
            kernels[name] = {"ms": ms, "min_bytes": b, "frac_of_3.35TBps": b / (ms * 1e-3) / HBM_BYTES_PER_S}
    res["power_law"] = {"nodes": n, "edges": e, "fused_step_ms": statistics.median(steps), "peak_growth_gb": grow / 1e9,
                        "kernels": kernels}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
