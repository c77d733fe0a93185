"""Clustering ops on the GPU (csrc/cluster.cu): grid_cluster and graclus equal the numpy oracle of
tests/cluster_oracle.py bit for bit -- fp32 / fp64 grids with and without start / end, negative offsets, non-finite
coordinates and D = 1..4; graclus with int32 / int64 indices, unweighted and fp32 / bf16 / fp64 weights, self-loops,
NaN weights, isolated nodes, duplicate edges, tiny graphs and a directed 3-cycle that reaches the round cap -- give the
same vector for the same seed, handle a 1M-node power-law graph, never synchronise, and the unmodified reference's
graclus, voxel_grid, pooling functions and both MNIST-superpixel example networks reproduce tests/golden/cluster.npz
after plugin.install(layers=True, flip_flags=True)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cluster_nets as CN  # noqa: E402
import cluster_oracle as CO  # noqa: E402

from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.nn import pool  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _eq(a, b, what=""):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = np.asarray(b)
    assert a.dtype == np.int64, what
    assert a.shape == b.shape and np.array_equal(a, b), f"{what}: {int((a != b).sum())} differ, {a[:8]} vs {b[:8]}"


def _csr(n, row, col, w=None):
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    o = np.lexsort((col, row))
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))]).astype(np.int64)
    return rowptr, col[o], (None if w is None else np.asarray(w)[o])


def _power_law(n, avg, seed):
    """Symmetric graph, no self-loops: sources uniform, targets Pareto-distributed over the node ids."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, n, n * avg // 2)
    b = (rng.pareto(1.2, a.size) * 8).astype(np.int64) % n
    keep = a != b
    a, b = a[keep], b[keep]
    return np.concatenate([a, b]), np.concatenate([b, a])


def _graclus(rowptr, col, w, seed, idx=torch.int64):
    cl, rounds = ops.graclus(torch.from_numpy(rowptr).to(DEV, idx), torch.from_numpy(col).to(DEV, idx), w, seed=seed,
                             return_rounds=True)
    return cl, int(rounds)


# ---------------------------------------------------------------------------------------------- grid_cluster
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("given", ["none", "start", "end", "both"])
def test_grid_cluster_equals_the_oracle(dtype, d, given):
    g = torch.Generator().manual_seed(d)
    pos = (torch.randn(5000, d, generator=g) * 3.0).to(dtype)
    size = (torch.rand(d, generator=g) * 0.5 + 0.05).to(dtype)
    start = (torch.rand(d, generator=g) * 2 - 12).to(dtype) if given in ("start", "both") else None   # negative offsets
    end = (torch.rand(d, generator=g) + 12).to(dtype) if given in ("end", "both") else None
    cuda = (lambda t: None if t is None else t.to(DEV))
    got = ops.grid_cluster(pos.to(DEV), size.to(DEV), cuda(start), cuda(end))
    npy = (lambda t: None if t is None else t.numpy())
    _eq(got, CO.grid_cluster(pos.numpy(), size.numpy(), npy(start), npy(end)), f"grid {dtype} d={d} {given}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_grid_cluster_non_finite_coordinates_and_empty_input(dtype):
    pos = torch.randn(300, 3, dtype=dtype)
    pos[5, 0], pos[17, 2], pos[40, 1] = float("nan"), float("inf"), -float("inf")
    size = torch.tensor([0.25, 0.5, 1.0], dtype=dtype)
    start, end = torch.full((3, ), -4.0, dtype=dtype), torch.full((3, ), 4.0, dtype=dtype)
    _eq(ops.grid_cluster(pos.to(DEV), size.to(DEV), start.to(DEV), end.to(DEV)),
        CO.grid_cluster(pos.numpy(), size.numpy(), start.numpy(), end.numpy()), "non-finite, start / end given")
    _eq(ops.grid_cluster(pos.to(DEV), size.to(DEV)), CO.grid_cluster(pos.numpy(), size.numpy()), "NaN min / max")
    assert ops.grid_cluster(torch.empty(0, 3, dtype=dtype, device=DEV), size.to(DEV)).shape == (0, )


def test_voxel_grid_mirror_is_the_reference_composition():
    pos = torch.tensor([[0.0, 0.0], [11.0, 9.0], [2.0, 8.0], [2.0, 2.0], [8.0, 3.0]], device=DEV)
    batch = torch.tensor([0, 0, 0, 1, 1], device=DEV)
    assert pool.voxel_grid(pos, 5, batch).tolist() == [0, 5, 3, 6, 7]
    assert pool.voxel_grid(pos, 5).tolist() == [0, 5, 3, 0, 1]
    assert pool.voxel_grid(pos, 5, batch, start=-1, end=[18, 14]).tolist() == [0, 10, 4, 16, 17]
    assert pool.voxel_grid(pos, 5, None, start=-1, end=[18, 14]).tolist() == [0, 10, 4, 0, 1]
    assert pool.voxel_grid(pos.double(), 5, batch).tolist() == [0, 5, 3, 6, 7]


# ---------------------------------------------------------------------------------------------- graclus
@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
@pytest.mark.parametrize("wdt", [None, torch.float32, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("seed", [0, 1, 2**63 + 5])
def test_graclus_equals_the_oracle(idx, wdt, seed):
    n = 3000
    row, col = _power_law(n, 6, 1)
    # extra edge cases: self-loops, duplicate edges, isolated nodes (the ids the generator never reaches stay alone)
    row = np.concatenate([row, np.arange(0, n, 97), row[:50]])
    col = np.concatenate([col, np.arange(0, n, 97), col[:50]])
    w = None
    if wdt is not None:
        w = torch.rand(row.size, generator=torch.Generator().manual_seed(2)).to(wdt)
        w[::41] = float("nan")
    rowptr, c, wo = _csr(n, row, col, None if w is None else w.double().numpy())
    wt = None if w is None else torch.from_numpy(wo).to(wdt).to(DEV)
    got, rounds = _graclus(rowptr, c, wt, seed, idx)
    want, want_rounds = CO.graclus(rowptr, c, wo, seed)
    _eq(got, want, f"graclus idx={idx} w={wdt} seed={seed}")
    assert rounds == want_rounds < ops.GRACLUS_MAX_ROUNDS


def test_graclus_tiny_graphs_and_the_directed_three_cycle():
    for rowptr, col in (([0], []), ([0, 0], []), ([0, 1], [0]), ([0, 1, 2], [1, 0])):
        rp, c = np.asarray(rowptr, np.int64), np.asarray(col, np.int64)
        for seed in range(4):
            got, rounds = _graclus(rp, c, None, seed)
            want, want_rounds = CO.graclus(rp, c, None, seed)
            _eq(got, want, f"tiny {rowptr} {col}")
            assert rounds == want_rounds
    got, rounds = _graclus(np.array([0, 1, 2, 3]), np.array([1, 2, 0]), None, 9)
    assert got.tolist() == [0, 1, 2] and rounds == ops.GRACLUS_MAX_ROUNDS == CO.MAX_ROUNDS


def test_graclus_is_deterministic_and_seeded_by_the_cpu_generator():
    rowptr, col, _ = _csr(20000, *_power_law(20000, 8, 3))
    rp, c = torch.from_numpy(rowptr).to(DEV), torch.from_numpy(col).to(DEV)
    w = torch.rand(c.numel(), device=DEV)
    assert torch.equal(ops.graclus(rp, c, w, seed=5), ops.graclus(rp, c, w, seed=5))
    torch.manual_seed(4)
    a = ops.graclus(rp, c)
    torch.manual_seed(4)
    b = ops.graclus(rp, c)
    torch.manual_seed(4)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    assert torch.equal(a, b) and torch.equal(a, ops.graclus(rp, c, seed=seed))


def test_a_1m_node_power_law_graph():
    n = 1_000_000
    rowptr, col, _ = _csr(n, *_power_law(n, 10, 4))
    got, rounds = _graclus(rowptr, col, None, 77)
    assert rounds < CO.MAX_ROUNDS // 4, rounds
    want, want_rounds = CO.graclus(rowptr, col, None, 77)
    _eq(got, want, "1M graclus")
    assert rounds == want_rounds
    cl = got.cpu().numpy()
    counts = np.bincount(cl, minlength=n)
    assert counts.max() <= 2 and (cl <= np.arange(n)).all() and (cl[cl] == cl).all()
    src = np.repeat(np.arange(n), np.diff(rowptr))
    single = counts[cl] == 1
    assert not (single[src] & single[col]).any()                     # no edge joins two singletons
    pair = cl[src] == cl[col]                                        # pairs are joined by an edge
    assert np.unique(cl[src[pair]]).size == (counts == 2).sum()


def test_no_synchronisation():
    rowptr, col, _ = _csr(5000, *_power_law(5000, 6, 5))
    rp, c = torch.from_numpy(rowptr).to(DEV), torch.from_numpy(col).to(DEV)
    w = torch.rand(c.numel(), device=DEV, dtype=torch.float64)
    pos, size = torch.rand(5000, 3, device=DEV), torch.full((3, ), 0.1, device=DEV)
    ops.graclus(rp, c, w)
    ops.grid_cluster(pos, size)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ops.graclus(rp, c)
        ops.graclus(rp, c, w)
        ops.grid_cluster(pos, size)
        ops.grid_cluster(pos, size, torch.zeros(3, device=DEV), torch.ones(3, device=DEV))
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---------------------------------------------------------------------------------------------- the reference
@pytest.fixture
def tg_cluster(tg):
    from pytorch_geometric_b200 import plugin
    plugin.install(layers=True, flip_flags=True)
    yield tg
    plugin.uninstall()


def _t(z, key):
    return torch.from_numpy(np.asarray(z[key])).to(DEV)


def _close(a, b, tol, what):
    a, b = a.detach().double().cpu(), torch.as_tensor(np.asarray(b)).double()
    assert a.shape == b.shape, what
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= tol * max(scale, 1e-3), f"{what}: max err {err:.3e} vs scale {scale:.3e}"


def test_reference_graclus_and_voxel_grid_match_golden(tg_cluster, golden):
    z = golden("cluster")
    nn = tg_cluster.nn
    assert nn.graclus(torch.tensor([[0, 1], [1, 0]], device=DEV)).tolist() == z["anchor_graclus"].tolist()
    pos = torch.tensor([[0.0, 0.0], [11.0, 9.0], [2.0, 8.0], [2.0, 2.0], [8.0, 3.0]], device=DEV)
    batch = torch.tensor([0, 0, 0, 1, 1], device=DEV)
    got = [nn.voxel_grid(pos, size=5, batch=batch), nn.voxel_grid(pos, size=5),
           nn.voxel_grid(pos, size=5, batch=batch, start=-1, end=[18, 14]),
           nn.voxel_grid(pos, size=5, start=-1, end=[18, 14])]
    _eq(torch.stack(got), z["anchor_voxel_want"], "voxel anchors")
    ei = _t(z, "gr_ei")
    torch.manual_seed(21)
    _eq(nn.graclus(ei, num_nodes=60), z["gr_cluster"], "graclus")
    torch.manual_seed(22)
    _eq(nn.graclus(ei, _t(z, "gr_w"), 60), z["grw_cluster"], "graclus weighted")
    pos, batch = _t(z, "vg_pos"), _t(z, "vg_batch")
    _eq(nn.voxel_grid(pos, 0.7, batch), z["vg_b"], "voxel_grid")
    _eq(nn.voxel_grid(pos, [0.7, 0.5, 1.1]), z["vg_nob"], "voxel_grid without batch")
    _eq(nn.voxel_grid(pos, 0.6, batch, start=-1.5, end=[3.2, 3.0, 3.5]), z["vg_b_se"], "voxel_grid start / end")
    _eq(nn.voxel_grid(pos, 0.6, None, start=[-1.0, -1.2, -1.1], end=3.0), z["vg_nob_se"], "voxel_grid no batch")


def test_reference_pooling_on_the_clusters_matches_golden(tg_cluster, golden):
    z = golden("cluster")
    nn = tg_cluster.nn
    from torch_geometric.data import Batch
    for tag in ("gr", "grw", "vg"):
        cluster = _t(z, f"{tag}_cluster" if tag != "vg" else "vg_b")
        x, ei, pos, b = (_t(z, f"pool_{tag}_{k}") for k in ("x", "ei", "pos", "batch"))
        mp = nn.max_pool(cluster, Batch(x=x, edge_index=ei, pos=pos, batch=b))
        _close(mp.x, z[f"pool_{tag}_max_x"], 0.0, f"{tag} max_pool x")
        _eq(mp.edge_index, z[f"pool_{tag}_max_ei"], f"{tag} max_pool edges")
        _eq(mp.batch, z[f"pool_{tag}_max_batch"], f"{tag} max_pool batch")
        _close(mp.pos, z[f"pool_{tag}_max_pos"], 1e-5, f"{tag} max_pool pos")
        ap = nn.avg_pool(cluster, Batch(x=x, edge_index=ei, pos=pos, batch=b))
        _close(ap.x, z[f"pool_{tag}_avg_x"], 1e-5, f"{tag} avg_pool x")
        _close(ap.pos, z[f"pool_{tag}_avg_pos"], 1e-5, f"{tag} avg_pool pos")
        _eq(ap.edge_index, z[f"pool_{tag}_avg_ei"], f"{tag} avg_pool edges")
        mx, mb = nn.max_pool_x(cluster, x, b)
        _close(mx, z[f"pool_{tag}_maxx_x"], 0.0, f"{tag} max_pool_x")
        _eq(mb, z[f"pool_{tag}_maxx_batch"], f"{tag} max_pool_x batch")
    mx, _ = nn.max_pool_x(_t(z, "vg_b_se"), _t(z, "pool_vg_x"), _t(z, "vg_batch"), size=8 * 8 * 9)
    _close(mx, z["pool_vg_maxx_size"], 0.0, "max_pool_x size=")


@pytest.mark.parametrize("tag,make,n_clusters", [("mnist_graclus", CN.graclus_net, 2),
                                                  ("mnist_voxel_grid", CN.voxel_grid_net, 3)])
def test_example_networks_match_golden(tg_cluster, golden, tag, make, n_clusters):
    z = golden("cluster")
    model = CN.seed_parameters(make(), 7).to(DEV).eval()
    from pytorch_geometric_b200.plugin import conv as ours
    assert isinstance(model.conv1, ours.B200SplineConv)
    data = CN.superpixel_batch(tuple(z[f"sp_{k}"] for k in ("x", "pos", "ei", "batch", "y")), DEV)
    torch.manual_seed(11)                                          # as the generator seeded it before the forward
    out = model(data)
    for i in range(n_clusters):
        _eq(model.clusters[i], z[f"{tag}_cluster{i}"], f"{tag} cluster {i}")
    out.backward(_t(z, f"{tag}_gout"))
    _close(out, z[f"{tag}_out"], 1e-5, f"{tag} out")
    # the parameter gradients pass back through two or three SplineConvs and max-pools whose fp32 summation orders
    # differ between the two devices
    # the golden data keeps the larger gradients at sampled entries (cluster_nets.grad_entries)
    for name, p in model.named_parameters():
        got = p.grad.reshape(-1)[torch.from_numpy(CN.grad_entries(p.numel())).to(DEV)]
        _close(got, z[f"{tag}_g_{name}"], 1e-4, f"{tag} grad {name}")


def test_example_network_training_step_on_cuda(tg_cluster):
    """A whole training step (dropout on, optimiser step) of both networks on CUDA tensors."""
    data_arrays = CN.superpixel_arrays(8, seed=1)
    for make in (CN.graclus_net, CN.voxel_grid_net):
        model = make().to(DEV).train()
        opt = torch.optim.Adam(model.parameters(), lr=0.01)
        data = CN.superpixel_batch(data_arrays, DEV)
        opt.zero_grad()
        loss = torch.nn.functional.nll_loss(model(data), data.y)
        loss.backward()
        opt.step()
        assert torch.isfinite(loss) and all(torch.isfinite(p).all() for p in model.parameters())
