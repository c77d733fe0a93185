"""Golden vectors for the consumers of torch.ops.pyg.{graclus_cluster, grid_cluster}: the UNMODIFIED reference on the
CPU with the numpy restatement of both ops from tests/cluster_oracle.py registered as their CPU implementations and
WITH_GRACLUS / WITH_GRID_CLUSTER set (pyg-lib is not installed, so graclus and voxel_grid raise ImportError without
them), and tests/spline_oracle.py bound into SplineConv.  Cases: graclus unweighted and weighted, voxel_grid with and
without batch, start and end, max_pool / avg_pool / max_pool_x (with and without size=) on those clusters, both
MNIST-superpixel example networks (tests/cluster_nets.py: parameters from cluster_nets.seed_parameters, so they are
not stored; eval mode; a synthetic batch of 4 x 75 superpixels) forward and backward, with each parameter gradient kept
whole up to 16384 entries and at 4096 entries spread over it beyond (cluster_nets.grad_entries), and the anchors the
reference's own tests state.  The CPU generator is seeded
immediately before each graclus-bearing call.  Inputs are chosen so that every node's candidate weights differ by more
than 1e-5 relative, so the matching does not depend on the device that computes the normalized-cut weights.  Same
provenance rules as make_golden.py (needs the reference in oracle/_ref; writes tests/golden/cluster.npz).

    python tests/golden/make_golden_cluster.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))             # oracle/install_ref.sh
sys.path.insert(0, os.path.join(HERE, ".."))
import cluster_nets as CN  # noqa: E402
import cluster_oracle as CO  # noqa: E402
import spline_oracle as SO  # noqa: E402
import torch_geometric.nn.conv.spline_conv as tg_spline  # noqa: E402
import torch_geometric.typing as tgt  # noqa: E402

OUT = HERE
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)
SCHEMAS = {
    "graclus_cluster": "graclus_cluster(Tensor rowptr, Tensor col, Tensor? weight) -> Tensor",
    "grid_cluster": "grid_cluster(Tensor pos, Tensor size, Tensor? start, Tensor? end) -> Tensor",
}
MIN_GAP = 1e-5
_GAPS = []


def weight_gap(rowptr, col, weight):
    """Smallest relative gap between two weights of one node's adjacency (self-loops excluded)."""
    worst = np.inf
    for u in range(rowptr.size - 1):
        s, e = rowptr[u], rowptr[u + 1]
        w = np.sort(weight[s:e][col[s:e] != u])
        if w.size > 1:
            worst = min(worst, float(((w[1:] - w[:-1]) / np.maximum(np.abs(w[1:]), 1e-30)).min()))
    return worst


def bind_oracle():
    impls = CO.torch_ops()
    graclus = impls["graclus_cluster"]

    def checked(rowptr, col, weight=None):
        if weight is not None:
            _GAPS.append(weight_gap(rowptr.numpy(), col.numpy(), weight.double().numpy()))
        return graclus(rowptr, col, weight)

    impls["graclus_cluster"] = checked
    lib = torch.library.Library("pyg", "FRAGMENT")
    for name, fn in impls.items():
        lib.define(SCHEMAS[name])
        lib.impl(name, fn, "CPU")
    tgt.WITH_GRACLUS = tgt.WITH_GRID_CLUSTER = True
    tg_spline.spline_basis, tg_spline.spline_weighting = SO.torch_spline_basis, SO.torch_spline_weighting
    return lib


def random_graph(n, k, g):
    """A symmetric graph without self-loops: each node joined to k random others."""
    row = torch.arange(n).repeat_interleave(k)
    col = (row + torch.randint(1, n, (n * k, ), generator=g)) % n
    key = torch.unique(torch.cat([row * n + col, col * n + row]))
    return torch.stack([key // n, key % n])


def run_net(arrs, tag, make, data_arrays, g):
    model = CN.seed_parameters(make(), 7)
    model.eval()                                              # dropout off: its mask depends on the device
    data = CN.superpixel_batch(data_arrays)
    torch.manual_seed(11)                                     # immediately before the forward
    out = model(data)
    gout = torch.randn(out.shape, generator=g)
    out.backward(gout)
    arrs[f"{tag}_out"], arrs[f"{tag}_gout"] = out, gout
    for i, c in enumerate(model.clusters):
        arrs[f"{tag}_cluster{i}"] = c
    for name, p in model.named_parameters():
        arrs[f"{tag}_g_{name}"] = p.grad.reshape(-1)[torch.from_numpy(CN.grad_entries(p.numel()))]


def main():
    lib = bind_oracle()  # noqa: F841  (kept alive while the reference runs)
    import torch_geometric.nn as tgnn
    from torch_geometric.data import Batch

    arrs = {}
    g = torch.Generator().manual_seed(3030)

    # the anchors the reference's tests state
    arrs["anchor_graclus"] = tgnn.graclus(torch.tensor([[0, 1], [1, 0]]))
    pos = torch.tensor([[0.0, 0.0], [11.0, 9.0], [2.0, 8.0], [2.0, 2.0], [8.0, 3.0]])
    batch = torch.tensor([0, 0, 0, 1, 1])
    arrs["anchor_voxel"] = torch.stack([tgnn.voxel_grid(pos, size=5, batch=batch), tgnn.voxel_grid(pos, size=5),
                                        tgnn.voxel_grid(pos, size=5, batch=batch, start=-1, end=[18, 14]),
                                        tgnn.voxel_grid(pos, size=5, start=-1, end=[18, 14])])
    arrs["anchor_voxel_want"] = torch.tensor([[0, 5, 3, 6, 7], [0, 5, 3, 0, 1], [0, 10, 4, 16, 17], [0, 10, 4, 0, 1]])
    diag = torch.arange(5.0).view(-1, 1).repeat(1, 2)
    arrs["anchor_single"] = torch.stack([tgnn.voxel_grid(diag, size=5, batch=batch), tgnn.voxel_grid(diag, size=5)])
    arrs["anchor_single_want"] = torch.tensor([[0, 0, 0, 1, 1], [0, 0, 0, 0, 0]])

    # graclus on a random symmetric graph, unweighted and weighted (symmetric distinct weights)
    ei = random_graph(60, 3, g)
    key = torch.minimum(ei[0], ei[1]) * 60 + torch.maximum(ei[0], ei[1])
    w = (torch.rand(3600, generator=g) + 0.5)[key]
    x = torch.randn(60, 8, generator=g)
    arrs.update(gr_ei=ei, gr_w=w, gr_x=x)
    torch.manual_seed(21)
    arrs["gr_cluster"] = c_u = tgnn.graclus(ei, num_nodes=60)
    torch.manual_seed(22)
    arrs["grw_cluster"] = c_w = tgnn.graclus(ei, w, 60)

    # voxel_grid: 3 clouds of 20 points in 3-D
    pos = torch.rand(60, 3, generator=g) * 4.0 - 1.0
    batch = torch.arange(3).repeat_interleave(20)
    arrs.update(vg_pos=pos, vg_batch=batch,
                vg_b=tgnn.voxel_grid(pos, 0.7, batch), vg_nob=tgnn.voxel_grid(pos, [0.7, 0.5, 1.1]),
                vg_b_se=tgnn.voxel_grid(pos, 0.6, batch, start=-1.5, end=[3.2, 3.0, 3.5]),
                vg_nob_se=tgnn.voxel_grid(pos, 0.6, None, start=[-1.0, -1.2, -1.1], end=3.0))

    # pooling on those clusters
    for tag, cluster in (("gr", c_u), ("grw", c_w), ("vg", arrs["vg_b"])):
        n = cluster.numel()
        ei_p = ei if tag != "vg" else random_graph(60, 3, g)
        xp = torch.randn(n, 8, generator=g)
        posp = pos if tag == "vg" else torch.rand(n, 2, generator=g)
        bp = batch if tag == "vg" else torch.zeros(n, dtype=torch.long)
        arrs.update({f"pool_{tag}_ei": ei_p, f"pool_{tag}_x": xp, f"pool_{tag}_pos": posp, f"pool_{tag}_batch": bp})
        data = Batch(x=xp, edge_index=ei_p, pos=posp, batch=bp)
        mp = tgnn.max_pool(cluster, data)
        ap = tgnn.avg_pool(cluster, Batch(x=xp, edge_index=ei_p, pos=posp, batch=bp))
        arrs.update({f"pool_{tag}_max_x": mp.x, f"pool_{tag}_max_ei": mp.edge_index, f"pool_{tag}_max_pos": mp.pos,
                     f"pool_{tag}_max_batch": mp.batch, f"pool_{tag}_avg_x": ap.x, f"pool_{tag}_avg_ei": ap.edge_index,
                     f"pool_{tag}_avg_pos": ap.pos})
        mx, mb = tgnn.max_pool_x(cluster, xp, bp)
        arrs.update({f"pool_{tag}_maxx_x": mx, f"pool_{tag}_maxx_batch": mb})
    # size=: the cluster is the voxel index itself, one block of 8 * 8 * 9 voxels per example
    arrs["pool_vg_maxx_size"] = tgnn.max_pool_x(arrs["vg_b_se"], arrs["pool_vg_x"], batch, size=8 * 8 * 9)[0]

    # both example networks on a synthetic batch; the data seed keeps every node's cut weights apart
    for seed in range(100):
        data_arrays = CN.superpixel_arrays(4, seed=seed)
        _GAPS.clear()
        tmp = {}
        run_net(tmp, "mnist_graclus", CN.graclus_net, data_arrays, torch.Generator().manual_seed(1))
        if min(_GAPS) > MIN_GAP:
            break
    else:
        raise RuntimeError("no superpixel seed with well-separated cut weights")
    x, p, e, b, y = data_arrays
    arrs.update(sp_seed=np.asarray(seed), sp_x=x, sp_pos=p, sp_ei=e, sp_batch=b, sp_y=y,
                mnist_graclus_min_gap=np.asarray(min(_GAPS)))
    run_net(arrs, "mnist_graclus", CN.graclus_net, data_arrays, g)
    assert min(_GAPS) > MIN_GAP
    run_net(arrs, "mnist_voxel_grid", CN.voxel_grid_net, data_arrays, g)

    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "cluster.npz"), **np_arrs)
    print("wrote cluster", len(np_arrs), "arrays; data seed", seed, "min cut-weight gap", min(_GAPS))


if __name__ == "__main__":
    main()
