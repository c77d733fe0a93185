"""Point-cloud graph construction on the engine (csrc/point.cu) against the torch composite users fall back to without
pyg-lib, on the same GPU.  One JSON line per workload:

    python benchmarks/point.py [--workload dgcnn|dgcnn_step|pointnet2|schnet|cloud200k|all] [--reps 5] [--warmup 2]

Workloads (sizes of the reference's examples):
  * dgcnn_f3 / f64 / f128: knn_graph with k = 20 on 32 clouds x 1024 points (DGCNN's shapes, examples/dgcnn_*.py)
  * dgcnn_step: one training step of DGCNN's classification Net (two DynamicEdgeConv layers on 32 x 1024 points), the
    unmodified reference on the engine; no composite arm (the reference layer cannot take one without patching)
  * pointnet2: set abstraction -- fps 0.5 then radius 0.2 (max 64), fps 0.25 then radius 0.4 (max 64)
  * schnet: radius_graph with cutoff 10 on 128 molecules of about 18 atoms
  * cloud200k_knn / cloud200k_radius: one 200k-point cloud, knn with k = 16 and radius 0.02 (max 64); fps on one such
    cloud runs in one CTA (a known follow-up) and is timed as cloud200k_fps without a composite arm

Composite arm: knn = torch.cdist + topk, chunked by queries; radius = cdist + mask (capped by a running count) +
nonzero; fps = a per-step torch loop (smaller sizes only).  The two arms alternate; each line has both medians, the
engine's per-op time from ops.PROFILE (a separate profiled pass), the fraction of queries whose neighbour set equals the composite's (cdist's
matmul form rounds differently, so near-ties may differ), and the card's name, power limit and max SM clock as
nvidia-smi reports them in the same run.
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
def composite_knn(x, y, k, bx, by, chunk=1024):
    rows, cols = [], []
    for b in torch.unique(by).tolist():
        xi, yi = (bx == b).nonzero().view(-1), (by == b).nonzero().view(-1)
        for s in range(0, yi.numel(), chunk):
            q = yi[s:s + chunk]
            d = torch.cdist(y[q].float(), x[xi].float())
            kk = min(k, xi.numel())
            j = d.topk(kk, dim=1, largest=False).indices
            rows.append(q.repeat_interleave(kk))
            cols.append(xi[j.reshape(-1)])
    return torch.stack([torch.cat(rows), torch.cat(cols)])


def composite_radius(x, y, r, bx, by, cap, chunk=1024):
    """Each query's first `cap` x points (ascending index) within r, as max_num_neighbors keeps them."""
    rows, cols = [], []
    for s in range(0, y.size(0), chunk):
        d = torch.cdist(y[s:s + chunk].float(), x.float())
        m = (d < r) & (by[s:s + chunk, None] == bx[None, :])
        m &= m.cumsum(1) <= cap
        i, j = m.nonzero(as_tuple=True)
        rows.append(i + s)
        cols.append(j)
    return torch.stack([torch.cat(rows), torch.cat(cols)])


def composite_fps(x, n_clouds, ratio):
    """Equal-size clouds [B, n, F]: per-step loop, first point as start."""
    p = x.view(n_clouds, -1, x.size(-1)).float()
    B, n, _ = p.shape
    m = int(-(-n * ratio // 1))
    idx = torch.zeros(B, m, dtype=torch.long, device=x.device)
    mind = torch.full((B, n), float("inf"), device=x.device)
    ar = torch.arange(B, device=x.device)
    for s in range(1, m):
        last = p[ar, idx[:, s - 1]]
        mind = torch.minimum(mind, ((p - last[:, None]) ** 2).sum(-1))
        idx[:, s] = mind.argmax(1)
    return (idx + ar[:, None] * n).view(-1)


def match_fraction(a, b, n_q):
    """Fraction of queries 0..n_q-1 whose neighbour sets agree (row 0 = query, row 1 = neighbour)."""
    def sets(e):
        e = e.cpu()
        o = torch.argsort(e[0] * (1 << 32) + e[1])
        e = e[:, o]
        cnt = torch.bincount(e[0], minlength=n_q)
        return torch.split(e[1], cnt.tolist())
    sa, sb = sets(a), sets(b)
    return sum(torch.equal(u, v) for u, v in zip(sa, sb)) / max(n_q, 1)


# ---------------------------------------------------------------------------------------------- workloads
def wl_dgcnn(f, reps, warmup):
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.rand(32 * 1024, f, device=DEV, generator=g)
    batch = torch.arange(32, device=DEV).repeat_interleave(1024)
    ptr = ops.index2ptr(batch, 32)

    def eng():
        return ops.knn(x, x, 20, ptr, ptr)

    def comp():
        return composite_knn(x, x, 20, batch, batch)

    t = alternate({"engine": eng, "composite": comp}, reps, warmup)
    return {"workload": f"dgcnn_f{f}", "engine_ms": t["engine"], "composite_ms": t["composite"],
            "engine_ops_ms": profiled(eng), "match": match_fraction(eng(), comp(), x.size(0))}


def wl_dgcnn_step(reps, warmup):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import torch_geometric.nn as tgnn
    from torch_geometric.nn import MLP
    from pytorch_geometric_b200 import plugin
    plugin.install(flip_flags=True)
    try:
        class Net(torch.nn.Module):
            def __init__(self, out_channels, k=20, aggr="max"):
                super().__init__()
                self.conv1 = tgnn.DynamicEdgeConv(MLP([2 * 3, 64, 64, 64]), k, aggr)
                self.conv2 = tgnn.DynamicEdgeConv(MLP([2 * 64, 128]), k, aggr)
                self.lin1 = torch.nn.Linear(128 + 64, 1024)
                self.mlp = MLP([1024, 512, 256, out_channels], dropout=0.5, norm=None)

            def forward(self, pos, batch):
                x1 = self.conv1(pos, batch)
                x2 = self.conv2(x1, batch)
                out = self.lin1(torch.cat([x1, x2], dim=1))
                out = tgnn.global_max_pool(out, batch)
                return self.mlp(out).log_softmax(dim=1)

        torch.manual_seed(0)
        model = Net(40).to(DEV)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        pos = torch.rand(32 * 1024, 3, device=DEV)
        batch = torch.arange(32, device=DEV).repeat_interleave(1024)
        y = torch.randint(0, 40, (32, ), device=DEV)

        def step():
            opt.zero_grad()
            loss = torch.nn.functional.nll_loss(model(pos, batch), y)
            loss.backward()
            opt.step()

        t = statistics.median(timed(step, reps, warmup))
        return {"workload": "dgcnn_step", "engine_ms": t, "composite_ms": None, "engine_ops_ms": profiled(step),
                "match": None}
    finally:
        plugin.uninstall()


def wl_pointnet2(reps, warmup):
    g = torch.Generator(device=DEV).manual_seed(1)
    pos = torch.rand(32 * 1024, 3, device=DEV, generator=g)
    batch = torch.arange(32, device=DEV).repeat_interleave(1024)

    def eng():
        i1 = pool.fps(pos, batch, 0.5, random_start=False)
        e1 = pool.radius(pos, pos[i1], 0.2, batch, batch[i1], 64)
        p2, b2 = pos[i1], batch[i1]
        i2 = pool.fps(p2, b2, 0.25, random_start=False)
        e2 = pool.radius(p2, p2[i2], 0.4, b2, b2[i2], 64)
        return i1, e1, i2, e2

    def comp():
        i1 = composite_fps(pos, 32, 0.5)
        e1 = composite_radius(pos, pos[i1], 0.2, batch, batch[i1], 64)
        p2, b2 = pos[i1], batch[i1]
        i2 = composite_fps(p2, 32, 0.25)
        e2 = composite_radius(p2, p2[i2], 0.4, b2, b2[i2], 64)
        return i1, e1, i2, e2

    t = alternate({"engine": eng, "composite": comp}, reps, warmup)
    a, b = eng(), comp()
    return {"workload": "pointnet2", "engine_ms": t["engine"], "composite_ms": t["composite"],
            "engine_ops_ms": profiled(eng), "fps_equal": bool(torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])),
            "match": match_fraction(a[1], b[1], a[0].numel()),
            "match_level2": match_fraction(a[3], b[3], a[2].numel())}


def wl_schnet(reps, warmup):
    g = torch.Generator().manual_seed(2)
    sizes = torch.randint(12, 25, (128, ), generator=g)
    batch = torch.arange(128).repeat_interleave(sizes).to(DEV)
    pos = (torch.rand(int(sizes.sum()), 3, generator=g) * 6.0).to(DEV)

    def eng():
        return pool.radius_graph(pos, 10.0, batch, max_num_neighbors=32, flow="target_to_source")

    def comp():
        e = composite_radius(pos, pos, 10.0, batch, batch, 32)
        return e[:, e[0] != e[1]]

    t = alternate({"engine": eng, "composite": comp}, reps, warmup)
    return {"workload": "schnet", "engine_ms": t["engine"], "composite_ms": t["composite"],
            "engine_ops_ms": profiled(eng), "match": match_fraction(eng(), comp(), pos.size(0))}


def wl_cloud200k(reps, warmup):
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.rand(200_000, 3, device=DEV, generator=g)
    zero = torch.zeros(x.size(0), dtype=torch.long, device=DEV)
    lines = []

    def eng_knn():
        return ops.knn(x, x, 16)

    def comp_knn():
        return composite_knn(x, x, 16, zero, zero)

    t = alternate({"engine": eng_knn, "composite": comp_knn}, reps, warmup)
    lines.append({"workload": "cloud200k_knn", "engine_ms": t["engine"], "composite_ms": t["composite"],
                  "engine_ops_ms": profiled(eng_knn), "match": match_fraction(eng_knn(), comp_knn(), x.size(0))})

    def eng_rad():
        return ops.radius(x, x, 0.02, None, None, 64)

    def comp_rad():
        return composite_radius(x, x, 0.02, zero, zero, 64)

    t = alternate({"engine": eng_rad, "composite": comp_rad}, reps, warmup)
    lines.append({"workload": "cloud200k_radius", "engine_ms": t["engine"], "composite_ms": t["composite"],
                  "engine_ops_ms": profiled(eng_rad), "match": match_fraction(eng_rad(), comp_rad(), x.size(0))})

    def eng_fps():
        return ops.fps(x, None, 0.05, False)

    lines.append({"workload": "cloud200k_fps", "engine_ms": statistics.median(timed(eng_fps, max(reps // 2, 1), 1)),
                  "composite_ms": None, "engine_ops_ms": profiled(eng_fps), "match": None})
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all",
                    choices=["dgcnn", "dgcnn_step", "pointnet2", "schnet", "cloud200k", "all"])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    info = card()
    runs = []
    if a.workload in ("dgcnn", "all"):
        runs += [lambda f=f: wl_dgcnn(f, a.reps, a.warmup) for f in (3, 64, 128)]
    if a.workload in ("dgcnn_step", "all"):
        runs.append(lambda: wl_dgcnn_step(a.reps, a.warmup))
    if a.workload in ("pointnet2", "all"):
        runs.append(lambda: wl_pointnet2(a.reps, a.warmup))
    if a.workload in ("schnet", "all"):
        runs.append(lambda: wl_schnet(a.reps, a.warmup))
    if a.workload in ("cloud200k", "all"):
        runs.append(lambda: wl_cloud200k(a.reps, a.warmup))
    for run in runs:
        res = run()
        for line in (res if isinstance(res, list) else [res]):
            line["card"] = info
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
