"""Clustering for pooling on the engine (csrc/cluster.cu) against a torch composite of the same contract on the same
GPU.  One JSON line per workload:

    python benchmarks/cluster.py [--workload mnist_graclus|mnist_voxel_grid|graclus_large|grid_large|all] [--reps 5]
                                 [--warmup 2]

Workloads:
  * mnist_graclus / mnist_voxel_grid: one training step of each MNIST-superpixel example network (the unmodified
    reference under plugin.install(layers=True, flip_flags=True); tests/cluster_nets.py restates the examples' Net) on
    64 x 75 synthetic superpixels, with the engine's per-op times inside the step; the arms time the network's first
    cluster op on its own inputs
  * graclus_large: a symmetric power-law graph with N = 5 M and E = 50 M, unweighted and with normalized-cut weights
  * grid_large: voxel_grid on 20 M 3-D points in 16 examples, start and end from the data

Composite arm: graclus = the same rounds, colours and choice rules as torch gathers and scatter_reduce per phase, with
one host read per round (the done test); grid = the elementwise formula.  Because both arms implement one contract,
their cluster vectors must be identical ("equal").  Each line has the medians of alternated reps, graclus's rounds,
and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.nn import pool  # noqa: E402

DEV = "cuda"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def alternate(arms, reps, warmup):
    """Median ms of each arm, the arms interleaved rep by rep."""
    times = {k: [] for k in arms}
    for k, fn in arms.items():
        timed(fn, 0, warmup)
    for _ in range(reps):
        for k, fn in arms.items():
            times[k] += timed(fn, 1, 0)
    return {k: statistics.median(v) for k, v in times.items()}


def profiled(fn):
    ops.PROFILE.reset(enabled=True)
    fn()
    s = ops.PROFILE.summary()
    ops.PROFILE.reset(enabled=False)
    return {k: round(v["ms_total"], 4) for k, v in s.items()}


# ---------------------------------------------------------------------------------------------- composite arm
def _i64(c):
    return c - (1 << 64) if c >= 1 << 63 else c


def _shr(z, k):
    return (z >> k) & ((1 << (64 - k)) - 1)                       # logical shift of the int64 bit pattern


def composite_blue(seed, rnd, n, nodes):
    z = _i64(seed & ((1 << 64) - 1)) + (rnd * n + nodes) * _i64(0x9E3779B97F4A7C15)
    z = (z ^ _shr(z, 30)) * _i64(0xBF58476D1CE4E5B9)
    z = (z ^ _shr(z, 27)) * _i64(0x94D049BB133111EB)
    z = z ^ _shr(z, 31)
    return z < 0


def _pick(s, p, w, n, weighted):
    """Per node, the CSR position of the largest w among its edges (s, p, w), ties to the lowest position; -1 if none."""
    big = torch.iinfo(torch.int64).max
    if weighted:
        best = torch.full((n, ), -float("inf"), dtype=torch.float64, device=s.device)
        best.scatter_reduce_(0, s, w, "amax", include_self=True)
        top = w == best[s]
        s, p = s[top], p[top]
    out = torch.full((n, ), big, dtype=torch.int64, device=s.device)
    out.scatter_reduce_(0, s, p, "amin", include_self=True)
    return torch.where(out == big, -1, out)


def composite_graclus(rowptr, col, weight, seed):
    n = rowptr.numel() - 1
    col = col.long()
    src = torch.repeat_interleave(torch.arange(n, device=col.device), rowptr.diff().long())
    pos = torch.arange(col.numel(), device=col.device)
    w = torch.zeros(col.numel(), dtype=torch.float64, device=col.device) if weight is None else weight.double()
    keep = (col != src) & ~torch.isnan(w)
    src, dst, pos, w = src[keep], col[keep], pos[keep], w[keep]
    nodes = torch.arange(n, device=col.device)
    cluster = torch.full((n, ), -1, dtype=torch.int64, device=col.device)
    proposal, accept = cluster.clone(), cluster.clone()
    rnd = 0
    while rnd < ops.GRACLUS_MAX_ROUNDS:
        blue = composite_blue(seed, rnd, n, nodes)
        free = cluster == -1
        cand = free[src] & free[dst]
        s, d, p, ww = src[cand], dst[cand], pos[cand], w[cand]
        has = torch.zeros(n, dtype=torch.int64, device=col.device).index_add_(0, s, torch.ones_like(s)) > 0
        m = blue[s] & ~blue[d]
        pick = _pick(s[m], p[m], ww[m], n, weight is not None)
        bf = free & blue
        prop = torch.where(has, torch.where(pick >= 0, col[pick.clamp(min=0)], -1), -2)
        proposal = torch.where(bf, prop, proposal)
        m = ~blue[s] & blue[d] & (proposal[d] == s)
        pick = _pick(s[m], p[m], ww[m], n, weight is not None)
        rf = free & ~blue
        acc = torch.where(has, torch.where(pick >= 0, col[pick.clamp(min=0)], -1), -2)
        accept = torch.where(rf, acc, accept)
        pu = proposal.clamp(min=0)
        matched_b = bf & (proposal >= 0) & (accept[pu] == nodes)
        new = torch.where(bf & (proposal == -2), nodes, cluster)
        new = torch.where(matched_b, torch.minimum(nodes, proposal), new)
        new = torch.where(rf & (accept == -2), nodes, new)
        new = torch.where(rf & (accept >= 0), torch.minimum(nodes, accept), new)
        cluster = new
        rnd += 1
        if not bool((cluster == -1).any()):                      # the one host read of the round
            break
    return torch.where(cluster == -1, nodes, cluster), rnd


def composite_grid(pos, size, start=None, end=None):
    start = pos.min(0)[0] if start is None else start
    end = pos.max(0)[0] if end is None else end
    voxels = ((end - start) / size).to(torch.int64) + 1
    stride = torch.cat([voxels.new_ones(1), voxels[:-1].cumprod(0)])
    return (((pos - start) / size).to(torch.int64) * stride).sum(1)


def composite_voxel_grid(pos, size, batch):
    pos = torch.cat([pos, batch.view(-1, 1).to(pos.dtype)], dim=-1)
    size = torch.cat([torch.full((pos.size(1) - 1, ), size, dtype=pos.dtype, device=pos.device), pos.new_ones(1)])
    return composite_grid(pos, size)


# ---------------------------------------------------------------------------------------------- workloads
def power_law_csr(n, e, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randint(0, n, (e // 2, ), device=DEV, generator=g)
    u = torch.rand(e // 2, device=DEV, generator=g).clamp(min=1e-7)
    b = (8.0 * (u.pow(-1.0 / 1.2) - 1.0)).long() % n              # Pareto(1.2) targets over the node ids
    row, col = torch.cat([a, b]), torch.cat([b, a])
    perm = torch.sort(row * n + col)[1]
    row, col = row[perm], col[perm]
    return ops.index2ptr(row, n), col, row


def wl_graclus_large(reps, warmup):
    n, e = 5_000_000, 50_000_000
    rowptr, col, row = power_law_csr(n, e, 0)
    deg = rowptr.diff().float()
    xy = torch.rand(n, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    ncut = torch.norm(xy[row] - xy[col], dim=1) * (1.0 / deg[row] + 1.0 / deg[col])
    del row
    lines = []
    for tag, w in (("graclus_large", None), ("graclus_large_ncut", ncut)):
        seed = 12345

        def eng():
            return ops.graclus(rowptr, col, w, seed=seed, return_rounds=True)

        def comp():
            return composite_graclus(rowptr, col, w, seed)

        t = alternate({"engine": eng, "composite": comp}, reps, warmup)
        (a, rounds), (b, c_rounds) = eng(), comp()
        lines.append({"workload": tag, "n": n, "e": e, "engine_ms": t["engine"], "composite_ms": t["composite"],
                      "rounds": int(rounds), "composite_rounds": c_rounds, "equal": bool(torch.equal(a, b))})
    return lines


def wl_grid_large(reps, warmup):
    g = torch.Generator(device=DEV).manual_seed(2)
    pos = torch.rand(20_000_000, 3, device=DEV, generator=g) * 10.0
    batch = torch.arange(16, device=DEV).repeat_interleave(20_000_000 // 16)

    def eng():
        return pool.voxel_grid(pos, 0.05, batch)

    def comp():
        return composite_voxel_grid(pos, 0.05, batch)

    t = alternate({"engine": eng, "composite": comp}, reps, warmup)
    return {"workload": "grid_large", "n": pos.size(0), "engine_ms": t["engine"], "composite_ms": t["composite"],
            "engine_ops_ms": profiled(eng), "equal": bool(torch.equal(eng(), comp()))}


def wl_mnist(tag, reps, warmup):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import cluster_nets as CN
    from pytorch_geometric_b200 import plugin
    from torch_geometric.utils import normalized_cut
    plugin.install(layers=True, flip_flags=True)
    try:
        torch.manual_seed(0)
        model = (CN.graclus_net() if tag == "mnist_graclus" else CN.voxel_grid_net()).to(DEV).train()
        opt = torch.optim.Adam(model.parameters(), lr=0.01)
        arrays = CN.superpixel_arrays(64, seed=0)
        data0 = CN.superpixel_batch(arrays, DEV)

        def step():
            opt.zero_grad()
            data = data0.clone()
            loss = torch.nn.functional.nll_loss(model(data), data.y)
            loss.backward()
            opt.step()

        step_ms = statistics.median(timed(step, reps, warmup))
        per_op = profiled(step)
        if tag == "mnist_graclus":
            n = data0.num_nodes
            ei = data0.edge_index
            w = normalized_cut(ei, torch.norm(data0.pos[ei[0]] - data0.pos[ei[1]], dim=1), num_nodes=n)
            rowptr = ops.index2ptr(ei[0], n)

            def eng():
                return ops.graclus(rowptr, ei[1], w, seed=7, return_rounds=True)

            def comp():
                return composite_graclus(rowptr, ei[1], w, 7)

            t = alternate({"engine": eng, "composite": comp}, reps, warmup)
            (a, rounds), (b, _) = eng(), comp()
            extra = {"rounds": int(rounds)}
        else:
            def eng():
                return pool.voxel_grid(data0.pos, 5, data0.batch, start=0, end=28)

            def comp():
                p = torch.cat([data0.pos, data0.batch.view(-1, 1).float()], 1)
                size = torch.tensor([5.0, 5.0, 1.0], device=DEV)
                start = torch.zeros(3, device=DEV)
                end = torch.tensor([28.0, 28.0, float(data0.batch.max())], device=DEV)
                return composite_grid(p, size, start, end)

            t = alternate({"engine": eng, "composite": comp}, reps, warmup)
            a, b = eng(), comp()
            extra = {}
        cluster_ms = sum(v for k, v in per_op.items() if k in ("graclus", "grid_cluster"))
        return {"workload": tag, "graphs": 64, "nodes_per_graph": 75, "step_ms": step_ms,
                "step_cluster_ops_ms": round(cluster_ms, 4), "step_engine_ops_ms": per_op,
                "engine_ms": t["engine"], "composite_ms": t["composite"], **extra, "equal": bool(torch.equal(a, b))}
    finally:
        plugin.uninstall()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all",
                    choices=["mnist_graclus", "mnist_voxel_grid", "graclus_large", "grid_large", "all"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    info = card()
    runs = []
    for tag in ("mnist_graclus", "mnist_voxel_grid"):
        if a.workload in (tag, "all"):
            runs.append(lambda tag=tag: wl_mnist(tag, a.reps, a.warmup))
    if a.workload in ("graclus_large", "all"):
        runs.append(lambda: wl_graclus_large(a.reps, a.warmup))
    if a.workload in ("grid_large", "all"):
        runs.append(lambda: wl_grid_large(a.reps, a.warmup))
    for run in runs:
        res = run()
        for line in (res if isinstance(res, list) else [res]):
            line["card"] = info
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
