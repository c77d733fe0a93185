"""Random walks on the engine (csrc/random_walk.cu) against a torch composite of the same contract on the same GPU.
One JSON line per workload:

    python benchmarks/random_walk.py [--workload node2vec_cora|corpus|row_order|dropout_path|rooted_rw|all]
                                     [--reps 5] [--warmup 2]

Workloads:
  * node2vec_cora: Node2Vec with examples/node2vec.py's settings (batch 128, 10 walks per node, walk_length 20,
    context 10, p = q = 1, SparseAdam) on a seeded Cora-sized graph (2,708 nodes, 10,556 edges), the unmodified
    reference model under plugin.install(layers=True, flip_flags=True): one sample() of each arm and one whole
    training step (sample, loss, backward, optimiser step) on the engine
  * corpus: a DeepWalk / node2vec corpus, one walk of length 80 from every node of an ogbn-products-sized power-law
    graph (2.4 M nodes, 62 M undirected edges from bench.py's generator, both directions, rows sorted), at p = q = 1
    and at p = 0.25, q = 4; walks/s and steps/s
  * row_order: node2vec (p = 0.25, q = 4, length 20, one walk per node) on a 1 M-node graph of uniform random edges
    (average degree 20) with sorted rows (binary search), with each row shuffled (linear scan), and with the trial cap
    at 64 and at 0 (every step the exact draw), so that both sides of each selection and the cap are measured
  * dropout_path: utils.dropout_path(p = 0.2, walk_length = 3) on bench.py's 5 M-node / 50 M-edge graph
  * rooted_rw: RootedRWSubgraph(walk_length = 3, repeat = 4) over 128 small molecules (20-40 atoms, ring-and-chain
    bonds)

Composite arm: the contract of csrc/random_walk.cu in torch ops: per-step vectorised gathers, the splitmix64 stream in
int64 ops, rejection rounds with the neighbour test as a searchsorted of row * N + col keys, and the exact draw as a
padded per-row running sum.  Both arms must produce identical walks ("equal").  Each line has the medians of
alternated reps, and the card's name, power limit and max SM clock as nvidia-smi reports them in the same run.
"""
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
from bench import synth_graph  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200 import utils as U  # noqa: E402

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
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


# ---------------------------------------------------------------------------------------------- composite arm
def _i64(c):
    c &= (1 << 64) - 1
    return c - (1 << 64) if c >= 1 << 63 else c


def _shr(z, k):
    return (z >> k) & ((1 << (64 - k)) - 1)                       # logical shift of the int64 bit pattern


def _mix(seed, key):
    z = seed + key * _i64(0x9E3779B97F4A7C15)
    z = (z ^ _shr(z, 30)) * _i64(0xBF58476D1CE4E5B9)
    z = (z ^ _shr(z, 27)) * _i64(0x94D049BB133111EB)
    return z ^ _shr(z, 31)


def _umulhi(r, d):
    """High 64 bits of r * d for the int64 bit pattern r (unsigned) and 0 <= d < 2^31."""
    return (_shr(r, 32) * d + _shr((r & 0xFFFFFFFF) * d, 32)) >> 32


def _uniform(r):
    return _shr(r, 11).double() * 2.0**-53


def composite_walk(rowptr, col, start, L, p=1.0, q=1.0, seed=0, max_trials=ops.RANDOM_WALK_MAX_TRIALS, keys=None):
    """The walks of ops.random_walk for a well-formed int64 CSR (values in range), in torch ops.  keys: the sorted
    row * N + col keys (the neighbour test), built here when not given."""
    n, S = rowptr.numel() - 1, start.numel()
    biased = p != 1.0 or q != 1.0
    w_t, w_q = 1.0 / p, 1.0 / q
    m = max(max(w_t, 1.0), w_q)
    acc = torch.tensor([w_t / m, 1.0 / m, w_q / m], dtype=torch.float64, device=DEV)
    wts = torch.tensor([w_t, 1.0, w_q], dtype=torch.float64, device=DEV)
    if biased and keys is None:
        row = torch.repeat_interleave(torch.arange(n, device=DEV), rowptr.diff())
        keys = torch.sort(row * n + col)[0]
    key = _mix(_i64(seed), torch.arange(S, device=DEV))
    draws = torch.zeros(S, dtype=torch.int64, device=DEV)
    out = torch.empty(S, L + 1, dtype=torch.int64, device=DEV)
    v = start.clone()
    out[:, 0] = v
    t = torch.full_like(v, -1)

    def draw(sel):
        draws[sel] += 1
        return _mix(key[sel], draws[sel])

    def cls(tt, x):
        k = tt * n + x
        nb = keys[torch.searchsorted(keys, k).clamp_(max=keys.numel() - 1)] == k
        return torch.where(x == tt, 0, torch.where(nb, 1, 2))

    for k in range(1, L + 1):
        s, e = rowptr[v], rowptr[v + 1]
        deg = e - s
        x = v.clone()                                              # dead ends stay, without a draw
        if not biased or k == 1:
            mv = (deg > 0).nonzero().squeeze(1)
            x[mv] = col[s[mv] + _umulhi(draw(mv), deg[mv])]
        else:
            pending = (deg > 0).nonzero().squeeze(1)
            for _ in range(max_trials):
                if pending.numel() == 0:
                    break
                cand = col[s[pending] + _umulhi(draw(pending), deg[pending])]
                x[pending] = cand
                take = _uniform(draw(pending)) < acc[cls(t[pending], cand)]
                pending = pending[~take]
            if pending.numel():                                   # the exact draw: a padded per-row running sum
                u = _uniform(draw(pending))
                ps, pd, pt = s[pending], deg[pending], t[pending]
                D = int(pd.max())
                total = torch.zeros(pending.numel(), dtype=torch.float64, device=DEV)
                for j in range(D):
                    on = j < pd
                    y = col[torch.where(on, ps + j, ps)]
                    total += torch.where(on, wts[cls(pt, y)], 0.0)
                target, run = u * total, torch.zeros_like(total)
                pick = ps + pd - 1
                found = torch.zeros(pending.numel(), dtype=torch.bool, device=DEV)
                for j in range(D):
                    on = j < pd
                    y = col[torch.where(on, ps + j, ps)]
                    run += torch.where(on, wts[cls(pt, y)], 0.0)
                    hit = on & ~found & (run > target)
                    pick = torch.where(hit, ps + j, pick)
                    found |= hit
                x[pending] = col[pick]
        t, v = v, x
        out[:, k] = v
    return out


# ---------------------------------------------------------------------------------------------- graphs
def csr_from_edges(ei, n):
    row, col = ei[0].long(), ei[1].long()
    kk = torch.sort(row * n + col)[0]
    return torch.ops.aten._convert_indices_from_coo_to_csr(kk // n, n, out_int32=False), kk % n, kk


def symmetric(ei):
    return torch.cat([ei, ei.flip(0)], 1)


def line(tag, t, walks_equal, n_walks, steps, **extra):
    res = {"workload": tag, "engine_ms": t["engine"], "composite_ms": t["composite"], "equal": bool(walks_equal)}
    if n_walks:
        res.update({"walks": n_walks, "walk_length": steps,
                    "engine_walks_per_s": round(n_walks / t["engine"] * 1e3),
                    "engine_steps_per_s": round(n_walks * steps / t["engine"] * 1e3),
                    "composite_steps_per_s": round(n_walks * steps / t["composite"] * 1e3)})
    res.update(extra)
    return res


def wl_corpus(reps, warmup):
    n = 2_400_000
    rowptr, col, keys = csr_from_edges(symmetric(synth_graph(n, 62_000_000, 11, DEV)), n)
    start = torch.arange(n, device=DEV)
    out = []
    for p, q in ((1.0, 1.0), (0.25, 4.0)):
        t = alternate({"engine": lambda: ops.random_walk(rowptr, col, start, 80, p, q, seed=3),
                       "composite": lambda: composite_walk(rowptr, col, start, 80, p, q, 3, keys=keys)}, reps, warmup)
        eq = torch.equal(ops.random_walk(rowptr, col, start, 80, p, q, seed=3),
                         composite_walk(rowptr, col, start, 80, p, q, 3, keys=keys))
        extra = {"nodes": n, "csr_entries": col.numel(), "max_degree": int(rowptr.diff().max()), "p": p, "q": q}
        out.append(line(f"corpus_p{p}_q{q}", t, eq, n, 80, **extra))
    return out


def wl_row_order(reps, warmup):
    n = 1_000_000
    g = torch.Generator(device=DEV).manual_seed(5)
    ei = symmetric(torch.randint(0, n, (2, n * 10), device=DEV, generator=g))
    rowptr, col, keys = csr_from_edges(ei, n)
    row = torch.repeat_interleave(torch.arange(n, device=DEV), rowptr.diff())
    shuffled = col[torch.sort(row * 4 + torch.randint(0, 4, row.shape, device=DEV, generator=g), stable=True)[1]]
    start = torch.arange(n, device=DEV)
    out = []
    cap = ops.RANDOM_WALK_MAX_TRIALS
    for tag, c, cap in (("row_order_sorted", col, cap), ("row_order_unsorted", shuffled, cap),
                        ("row_order_sorted_cap_64", col, 64), ("row_order_fallback_only", col, 0)):
        t = alternate({"engine": lambda: ops.random_walk(rowptr, c, start, 20, 0.25, 4.0, seed=4, max_trials=cap),
                       "composite": lambda: composite_walk(rowptr, c, start, 20, 0.25, 4.0, 4, cap, keys)}, reps, warmup)
        eq = torch.equal(ops.random_walk(rowptr, c, start, 20, 0.25, 4.0, seed=4, max_trials=cap),
                         composite_walk(rowptr, c, start, 20, 0.25, 4.0, 4, cap, keys))
        out.append(line(tag, t, eq, n, 20, max_trials=cap, csr_entries=c.numel()))
    return out


def _plugin():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from pytorch_geometric_b200 import plugin
    plugin.install(layers=True, flip_flags=True)
    return plugin


def _cora_like():
    """2,708 nodes and 10,556 directed edges (5,278 undirected pairs) in seven communities, seeded."""
    rng = np.random.default_rng(0)
    n, y = 2708, np.random.default_rng(1).integers(0, 7, 2708)
    pairs = set()
    while len(pairs) < 5278:
        a = int(rng.integers(0, n))
        same = np.nonzero(y == y[a])[0] if rng.random() < 0.8 else np.arange(n)
        b = int(rng.choice(same))
        if a != b:
            pairs.add((min(a, b), max(a, b)))
    e = np.array(sorted(pairs)).T
    return torch.from_numpy(np.concatenate([e, e[::-1]], 1).copy())


def wl_node2vec_cora(reps, warmup):
    plugin = _plugin()
    try:
        import torch_geometric.nn as tgnn
        ei = _cora_like()
        model = tgnn.Node2Vec(ei, embedding_dim=128, walk_length=20, context_size=10, walks_per_node=10,
                              num_negative_samples=1, p=1.0, q=1.0, sparse=True).to(DEV)
        opt = torch.optim.SparseAdam(list(model.parameters()), lr=0.01)
        batch = torch.arange(128, device=DEV)

        def comp_sample():
            rw = composite_walk(model.rowptr, model.col, batch.repeat(10), 19, seed=int(torch.randint(0, 2**63 - 1, ())))
            pos = torch.cat([rw[:, j:j + 10] for j in range(11)])
            return pos, model.neg_sample(batch)

        def step():
            pos, neg = model.sample(batch)
            opt.zero_grad()
            loss = model.loss(pos, neg)
            loss.backward()
            opt.step()

        t = alternate({"engine": lambda: model.sample(batch), "composite": comp_sample}, reps, warmup)
        torch.manual_seed(9)
        a = model.sample(batch)[0]
        torch.manual_seed(9)
        b = comp_sample()[0]
        step_ms = round(statistics.median(timed(step, reps, warmup)), 3)
        return line("node2vec_cora_sample", t, torch.equal(a, b), 1280, 19, train_step_ms=step_ms,
                    nodes=2708, edges=ei.size(1))
    finally:
        plugin.uninstall()


def wl_dropout_path(reps, warmup):
    plugin = _plugin()
    try:
        from torch_geometric.utils import dropout_path
        n = 5_000_000
        ei = synth_graph(n, 50_000_000, 0, DEV)

        def comp():
            num_edges = ei.size(1)
            row, col, order = U.sort_edge_index_by_row_col(ei, n)
            sample = torch.rand(num_edges, device=DEV) <= 0.2
            start = row[sample]
            rowptr = ops.index2ptr(row, n)
            walk = composite_walk(rowptr, col, start, 3, seed=int(torch.randint(0, 2**63 - 1, ())))
            wk = walk[:, :-1].reshape(-1) * n + walk[:, 1:].reshape(-1)
            hit = torch.isin(row * n + col, wk).nonzero().view(-1)
            mask = torch.ones(num_edges, dtype=torch.bool, device=DEV)
            mask[order[hit]] = False
            return ei[:, mask], mask

        t = alternate({"engine": lambda: dropout_path(ei, 0.2, 1, 3), "composite": comp}, reps, warmup)
        torch.manual_seed(2)
        a = dropout_path(ei, 0.2, 1, 3)[1]
        torch.manual_seed(2)
        b = comp()[1]
        ops.PROFILE.reset(enabled=True)
        dropout_path(ei, 0.2, 1, 3)
        walk_ms = round(ops.PROFILE.summary()["random_walk"]["ms_total"], 3)
        ops.PROFILE.reset(enabled=False)
        return line("dropout_path", t, torch.equal(a, b), 0, 3, nodes=n, edges=ei.size(1), engine_walk_kernel_ms=walk_ms)
    finally:
        plugin.uninstall()


def _molecules(count=128, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        n = int(rng.integers(20, 41))
        chain = [(i, i + 1) for i in range(n - 1)]
        rings = [(i, i + 5) for i in range(0, n - 5, 7)]
        e = np.array(chain + rings).T
        out.append((torch.from_numpy(np.concatenate([e, e[::-1]], 1).copy()).to(DEV), n))
    return out


def wl_rooted_rw(reps, warmup):
    plugin = _plugin()
    try:
        from torch_geometric.data import Data
        from torch_geometric.transforms import RootedRWSubgraph
        mols = [Data(edge_index=e, num_nodes=n) for e, n in _molecules()]
        tr = RootedRWSubgraph(3, 4)

        def comp_one(data):
            n = data.num_nodes
            start = torch.arange(n, device=DEV).view(-1, 1).repeat(1, 4).view(-1)
            row, col, _ = U.sort_edge_index_by_row_col(data.edge_index, n)
            walk = composite_walk(ops.index2ptr(row, n), col, start, 3, seed=int(torch.randint(0, 2**63 - 1, ())))
            mask = torch.zeros((n, n), dtype=torch.bool, device=DEV)
            mask[start.view(-1, 1).repeat(1, 4).view(-1), walk.view(-1)] = True
            return tr.map(data, mask)

        t = alternate({"engine": lambda: [tr(d) for d in mols], "composite": lambda: [comp_one(d) for d in mols]},
                      reps, warmup)
        torch.manual_seed(5)
        a = [tr(d).n_id for d in mols]
        torch.manual_seed(5)
        b = [comp_one(d)[1] for d in mols]                          # map gives (sub_edge_index, n_id, ...)
        eq = all(torch.equal(x, y) for x, y in zip(a, b))
        return line("rooted_rw_subgraph", t, eq, 0, 3, molecules=len(mols), atoms=sum(d.num_nodes for d in mols))
    finally:
        plugin.uninstall()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all",
                    choices=["node2vec_cora", "corpus", "row_order", "dropout_path", "rooted_rw", "all"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    info = card()
    runs = {"node2vec_cora": wl_node2vec_cora, "corpus": wl_corpus, "row_order": wl_row_order,
            "dropout_path": wl_dropout_path, "rooted_rw": wl_rooted_rw}
    for tag, run in runs.items():
        if a.workload not in (tag, "all"):
            continue
        print(json.dumps({"running": tag}), flush=True)
        res = run(a.reps, a.warmup)
        for ln in (res if isinstance(res, list) else [res]):
            ln["card"] = info
            print(json.dumps(ln), flush=True)
            assert ln["equal"], f"{ln['workload']}: the two arms' walks differ"


if __name__ == "__main__":
    main()
