"""Golden vectors for the point-cloud consumers of torch.ops.pyg.{knn, radius, fps, nearest}: the UNMODIFIED reference
on the CPU with the float32 restatement of pyg-lib's ops from tests/point_oracle.py registered as CPU implementations
of torch.ops.pyg.* and WITH_KNN / WITH_RADIUS / WITH_FPS / WITH_NEAREST set (pyg-lib is not installed, so the
constructors and functions raise ImportError without them).  Cases: DynamicEdgeConv (batched, and bipartite with
batches), GravNetConv, XConv with dilation 2, knn_interpolate, one PointNet++ set-abstraction step (fps with
random_start=False, radius, PointNetConv), SchNet's forward, the KNNGraph and RadiusGraph transforms, and the anchors
the reference's own tests state.  Weights are seeded; the seeds are chosen so that every k-th / (k+1)-th distance gap
of a k-NN in a learned space (GravNetConv's s) is above 1e-3 relative, far above fp32 rounding, so the neighbour sets
do not depend on the device that computes s.  Same provenance rules as make_golden.py (needs the reference in
oracle/_ref; writes tests/golden/point.npz).

    python tests/golden/make_golden_point.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))             # oracle/install_ref.sh
sys.path.insert(0, os.path.join(HERE, ".."))
import point_oracle as PO  # noqa: E402
import torch_geometric.typing as tgt  # noqa: E402

OUT = HERE
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)
SCHEMAS = {
    "knn": "knn(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y, int k, bool cosine, int num_workers) -> Tensor",
    "radius": "radius(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y, float r, int max_num_neighbors, "
              "int num_workers, bool ignore_same_index) -> Tensor",
    "fps": "fps(Tensor src, Tensor ptr, float ratio, bool random_start) -> Tensor",
    "nearest": "nearest(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y) -> Tensor",
}
SIX = [[0.0, 0.0], [1.0, 0.0], [2.0, 0.0], [0.0, 1.0], [-2.0, 0.0], [0.0, -2.0]]


def bind_oracle():
    lib = torch.library.Library("pyg", "FRAGMENT")
    for name, fn in PO.torch_ops().items():
        lib.define(SCHEMAS[name])
        lib.impl(name, fn, "CPU")
    for flag in ("WITH_KNN", "WITH_RADIUS", "WITH_FPS", "WITH_NEAREST"):
        setattr(tgt, flag, True)
    return lib


def min_gap(space, batch, k):
    """Smallest relative gap between consecutive sorted distances among each query's k + 1 nearest."""
    s = space.detach().double().numpy()
    b = batch.numpy()
    worst = np.inf
    for g in np.unique(b):
        p = s[b == g]
        d = ((p[:, None, :] - p[None, :, :]) ** 2).sum(-1)
        for row in d:
            r = np.sort(row)[:k + 2]
            worst = min(worst, float(((r[1:] - r[:-1]) / np.maximum(r[1:], 1e-30)).min()))
    return worst


def main():
    lib = bind_oracle()  # noqa: F841  (kept alive while the reference runs)
    import torch_geometric.nn as tgnn
    import torch_geometric.transforms as T
    from torch_geometric.data import Data
    from torch_geometric.nn import knn_interpolate
    from torch_geometric.nn.models import SchNet

    arrs = {}
    g = torch.Generator().manual_seed(20260)

    def lin_mlp(*ch):
        layers = []
        for a, b in zip(ch[:-1], ch[1:]):
            layers += [torch.nn.Linear(a, b), torch.nn.ReLU()]
        return torch.nn.Sequential(*layers[:-1])

    def run(tag, module, args, grads=()):
        for name, p in module.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p.clone()
        out = module(*args)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs[f"{tag}_out"], arrs[f"{tag}_gout"] = out, gout
        for name, t in grads:
            arrs[f"{tag}_g{name}"] = t.grad
        for name, p in module.named_parameters():
            arrs[f"{tag}_g_{name}"] = p.grad

    # DynamicEdgeConv, batched: 2 clouds x 16 points, F = 5, k = 6
    batch = torch.arange(2).repeat_interleave(16)
    x = torch.randn(32, 5, generator=g)
    torch.manual_seed(1)
    conv = tgnn.DynamicEdgeConv(lin_mlp(10, 16, 8), k=6, aggr="max")
    xr = x.clone().requires_grad_()
    arrs.update(dec_x=x, dec_batch=batch)
    run("dec", conv, (xr, batch), [("x", xr)])

    # DynamicEdgeConv, bipartite: 2 x 16 sources, 2 x 8 targets
    xl, xrt = torch.randn(32, 5, generator=g), torch.randn(16, 5, generator=g)
    bl, br = torch.arange(2).repeat_interleave(16), torch.arange(2).repeat_interleave(8)
    torch.manual_seed(2)
    conv = tgnn.DynamicEdgeConv(lin_mlp(10, 16, 8), k=5, aggr="add")
    a, b_ = xl.clone().requires_grad_(), xrt.clone().requires_grad_()
    arrs.update(decb_xl=xl, decb_xr=xrt, decb_bl=bl, decb_br=br)
    run("decb", conv, ((a, b_), (bl, br)), [("xl", a), ("xr", b_)])

    # GravNetConv: 2 x 20 points, k = 4, s = lin_s(x) of 3 dimensions; seed chosen for well-separated neighbours
    batch = torch.arange(2).repeat_interleave(20)
    for seed in range(100, 400):
        torch.manual_seed(seed)
        x = torch.randn(40, 6)
        conv = tgnn.GravNetConv(6, 8, space_dimensions=3, propagate_dimensions=4, k=4)
        if min_gap(conv.lin_s(x), batch, 4) > 1e-3:
            break
    else:
        raise RuntimeError("no GravNetConv seed with well-separated neighbours")
    arrs.update(grav_x=x, grav_batch=batch, grav_seed=np.asarray(seed))
    xr = x.clone().requires_grad_()
    run("grav", conv, (xr, batch), [("x", xr)])

    # XConv, dilation 2: 2 clouds x 24 points in 3-D, kernel_size 4
    batch = torch.arange(2).repeat_interleave(24)
    pos, x = torch.rand(48, 3, generator=g), torch.randn(48, 4, generator=g)
    torch.manual_seed(3)
    conv = tgnn.XConv(4, 8, dim=3, kernel_size=4, hidden_channels=6, dilation=2)
    xr = x.clone().requires_grad_()
    arrs.update(xconv_x=x, xconv_pos=pos, xconv_batch=batch)
    run("xconv", conv, (xr, pos, batch), [("x", xr)])

    # knn_interpolate: the reference test's case, and a random one
    xi = torch.tensor([[1.0], [10.0], [100.0], [-1.0], [-10.0], [-100.0]])
    px = torch.tensor([[-1.0, 0.0], [0.0, 0.0], [1.0, 0.0], [-2.0, 0.0], [0.0, 0.0], [2.0, 0.0]])
    py = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [-2.0, -2.0], [2.0, 2.0]])
    bx, by = torch.tensor([0, 0, 0, 1, 1, 1]), torch.tensor([0, 0, 1, 1])
    arrs["interp_anchor_out"] = knn_interpolate(xi, px, py, bx, by, k=2)
    arrs["interp_anchor_want"] = torch.tensor([[4.0], [70.0], [-4.0], [-70.0]])
    x, px, py = torch.randn(40, 3, generator=g), torch.rand(40, 3, generator=g), torch.rand(24, 3, generator=g)
    bx, by = torch.arange(2).repeat_interleave(20), torch.arange(2).repeat_interleave(12)
    arrs.update(interp_x=x, interp_px=px, interp_py=py, interp_bx=bx, interp_by=by,
                interp_out=knn_interpolate(x, px, py, bx, by, k=3))

    # PointNet++ set abstraction (examples/pointnet2_classification.py's SAModule, random_start=False)
    pos, x = torch.rand(64, 3, generator=g), torch.randn(64, 4, generator=g)
    batch = torch.arange(2).repeat_interleave(32)
    idx = tgnn.fps(pos, batch, ratio=0.5, random_start=False)
    row, col = tgnn.radius(pos, pos[idx], 0.4, batch, batch[idx], max_num_neighbors=16)
    torch.manual_seed(4)
    conv = tgnn.PointNetConv(lin_mlp(3 + 4, 16, 16), add_self_loops=True)
    xr = x.clone().requires_grad_()
    out = conv((xr, None), (pos, pos[idx]), torch.stack([col, row], dim=0))
    arrs.update(sa_pos=pos, sa_x=x, sa_batch=batch, sa_idx=idx, sa_row=row, sa_col=col)
    for name, p in conv.state_dict().items():
        arrs[f"sa_p_{name}"] = p.clone()
    arrs["sa_out"] = out

    # SchNet: 3 molecules of 7 atoms, cutoff 10
    z = torch.randint(1, 10, (21, ), generator=g)
    pos = torch.rand(21, 3, generator=g) * 3.0
    batch = torch.arange(3).repeat_interleave(7)
    torch.manual_seed(5)
    model = SchNet(hidden_channels=16, num_filters=16, num_interactions=2, num_gaussians=10, cutoff=10.0)
    for name, p in model.state_dict().items():
        arrs[f"schnet_p_{name}"] = p.clone()
    arrs.update(schnet_z=z, schnet_pos=pos, schnet_batch=batch, schnet_out=model(z, pos, batch))

    # transforms: the reference tests' six-point set, and a random cloud
    six = torch.tensor(SIX)
    arrs["knngraph_six"] = T.KNNGraph(k=2, force_undirected=True)(Data(pos=six)).edge_index
    arrs["radiusgraph_six"] = T.RadiusGraph(r=1.5)(Data(pos=six)).edge_index
    cloud = torch.rand(50, 3, generator=g)
    arrs.update(cloud=cloud, knngraph_cloud=T.KNNGraph(k=6)(Data(pos=cloud)).edge_index,
                radiusgraph_cloud=T.RadiusGraph(r=0.3, max_num_neighbors=8)(Data(pos=cloud)).edge_index)

    # the anchors the reference's tests and docstrings state
    arrs["knngraph_six_want"] = torch.tensor([[0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 3, 4, 4, 5, 5],
                                              [1, 2, 3, 4, 5, 0, 2, 3, 5, 0, 1, 0, 1, 4, 0, 3, 0, 1]])
    arrs["radiusgraph_six_want"] = torch.tensor([[0, 0, 1, 1, 1, 2, 3, 3], [1, 3, 0, 2, 3, 1, 0, 1]])
    nx = torch.tensor([[-1.0, -1.0], [-1.0, 1.0], [1.0, -1.0], [1.0, 1.0]])
    ny = torch.tensor([[-1.0, 0.0], [1.0, 0.0]])
    arrs["nearest_x"], arrs["nearest_y"] = nx, ny
    arrs["nearest_out"] = tgnn.nearest(nx, ny, torch.zeros(4, dtype=torch.long), torch.zeros(2, dtype=torch.long))
    arrs["nearest_want"] = torch.tensor([0, 0, 1, 1])

    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "point.npz"), **np_arrs)
    print("wrote point", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
