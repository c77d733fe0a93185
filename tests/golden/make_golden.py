"""Generates tests/golden/*.npz by running the UNMODIFIED reference (pyg-team/pytorch_geometric
v2.9.0, installed into oracle/_ref by oracle/install_ref.sh, pure Python over ATen, all WITH_*
extension flags False) on seeded inputs.  Needs that installed reference; the .npz files are committed
and are what pins the oracle (tests/test_oracle_golden.py) and, through it, the CUDA path.

    python tests/golden/make_golden.py

Every case stores its inputs and the reference outputs.  Sizes are tiny (a few kB each).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric  # noqa: E402
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric import EdgeIndex  # noqa: E402
from torch_geometric.nn import GATConv, GCNConv, GINConv, RGCNConv, SAGEConv  # noqa: E402
from torch_geometric.nn.aggr import (MaxAggregation, MeanAggregation, MinAggregation,  # noqa: E402
                                     SoftmaxAggregation, SumAggregation)
from torch_geometric.nn.conv.gcn_conv import gcn_norm  # noqa: E402
from torch_geometric.utils import (add_remaining_self_loops, degree, scatter, segment,  # noqa: E402
                                   softmax, spmm)
from torch_geometric.index import index2ptr, ptr2index  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)


def save(name, **arrs):
    conv = {}
    for k, v in arrs.items():
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()
        conv[k] = np.asarray(v)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **conv)
    print("wrote", name, {k: v.shape for k, v in conv.items()})


def rand_graph(g, N, E, self_loops=True):
    row = torch.randint(0, N, (E, ), generator=g)
    col = torch.randint(0, N, (E, ), generator=g)
    if self_loops:  # force a few existing (and duplicated) self loops
        row[:3] = torch.tensor([1, 1, 4]) % N
        col[:3] = torch.tensor([1, 1, 4]) % N
    return torch.stack([row, col])


def main():
    g = torch.Generator().manual_seed(1234)

    # ---- scatter: every reduce, empty groups (ids N-1, 3 unused), ties for min/max, fwd + bwd
    for F in (1, 5):
        N, E = 9, 40
        index = torch.randint(0, N - 1, (E, ), generator=g)
        index[index == 3] = 2
        src = torch.randn(E, F, generator=g)
        src[5] = src[7]  # a tie candidate
        index[5] = index[7]
        src = torch.round(src * 4) / 4  # coarse grid => real ties for max/min
        out = {}
        for red in ("sum", "mean", "min", "max", "mul"):
            s = src.clone().requires_grad_(red != "mul")
            o = scatter(s, index, 0, dim_size=N, reduce=red)
            out["out_" + red] = o
            if red != "mul":
                go = torch.randn(o.shape, generator=torch.Generator().manual_seed(7))
                o.backward(go)
                out["gout_" + red] = go
                out["gsrc_" + red] = s.grad
        save(f"scatter_F{F}", src=src, index=index, N=N, **out)

    # ---- segment (empty first segment, like test/utils/test_segment.py:13-31)
    src = torch.randn(20, 3, generator=g)
    ptr = torch.tensor([0, 0, 5, 10, 15, 20])
    save("segment", src=src, ptr=ptr,
         **{"out_" + r: segment(src, ptr, reduce=r) for r in ("sum", "mean", "min", "max")})

    # ---- softmax: known answer (test/utils/test_softmax.py:12-27) and random, index + ptr path
    src1 = torch.tensor([1., 1., 1., 1.])
    index1 = torch.tensor([0, 0, 1, 2])
    ptr1 = torch.tensor([0, 2, 3, 4])
    N, E, H = 7, 30, 4
    index = torch.sort(torch.randint(0, N, (E, ), generator=g))[0]
    srcs = torch.randn(E, H, generator=g).requires_grad_()
    o = softmax(srcs, index, num_nodes=N)
    go = torch.randn(E, H, generator=g)
    o.backward(go)
    ptr = index2ptr(index, N)
    save("softmax", src1=src1, index1=index1, ptr1=ptr1, out1=softmax(src1, index1),
         out1_ptr=softmax(src1, None, ptr1), src=srcs, index=index, ptr=ptr, N=N, out=o,
         out_ptr=softmax(srcs.detach(), None, ptr), gout=go, gsrc=srcs.grad)

    # ---- integer work: degree, index2ptr, ptr2index, add_remaining_self_loops, gcn_norm
    row = torch.tensor([0, 0, 0, 1, 2, 2])
    col = torch.tensor([0, 0, 1, 0, 2, 1])
    w = torch.tensor([1., 2., 3., 4., 5., 6.])
    ei2, w2 = add_remaining_self_loops(torch.stack([row, col]), w, fill_value=1.0, num_nodes=3)
    ei3, _ = add_remaining_self_loops(torch.stack([row, col]), None, num_nodes=3)
    ei = rand_graph(g, 11, 50)
    wr = torch.rand(50, generator=g) + 0.1
    eiR, wR = add_remaining_self_loops(ei, wr, fill_value=2.0, num_nodes=11)
    idx_sorted = torch.sort(ei[1])[0]
    save("structure", row=row, col=col, w=w, asl_ei=ei2, asl_w=w2, asl_ei_now=ei3,
         deg=degree(torch.tensor([0, 1, 0, 2, 0]), dtype=torch.long),
         deg_index=torch.tensor([0, 1, 0, 2, 0]), ei=ei, wr=wr, asl_eiR=eiR, asl_wR=wR,
         idx_sorted=idx_sorted, ptr=index2ptr(idx_sorted, 11), ptr2idx=ptr2index(index2ptr(idx_sorted, 11)),
         stable_perm=torch.sort(ei[1], stable=True)[1])
    outs = {}
    for tag, ww, improved, asl in (("a", None, False, True), ("b", wr, False, True),
                                   ("c", wr, True, True), ("d", wr, False, False)):
        e2, w2 = gcn_norm(ei, ww, 11, improved, asl, "source_to_target", torch.float32)
        outs["ei_" + tag], outs["w_" + tag] = e2, w2
    save("gcn_norm", ei=ei, wr=wr, N=11, **outs)

    # ---- gather + aggregate == EdgeIndex.matmul / spmm, all reduces, fwd + grads
    N, E, F = 13, 60, 6
    ei = rand_graph(g, N, E)
    x = torch.randn(N, F, generator=g)
    x = torch.round(x * 8) / 8
    val = torch.rand(E, generator=g) + 0.5
    outs = {}
    perm = torch.sort(ei[0] * N + ei[1], stable=True)[1]  # row-major sorted for EdgeIndex
    eis = ei[:, perm]
    adj = EdgeIndex(eis, sparse_size=(N, N), sort_order="row")
    for red in ("sum", "mean", "min", "max"):
        xs = x.clone().requires_grad_()
        o = adj.matmul(xs, reduce=red)  # out[row] = reduce_{col} x[col]
        go = torch.randn(o.shape, generator=torch.Generator().manual_seed(3))
        o.backward(go)
        outs["out_" + red], outs["gout_" + red], outs["gx_" + red] = o, go, xs.grad
    xs = x.clone().requires_grad_()
    vs = val[perm].clone().requires_grad_()
    o = adj.matmul(xs, input_value=vs, reduce="sum")
    go = torch.randn(o.shape, generator=torch.Generator().manual_seed(4))
    o.backward(go)
    csr = torch.sparse_csr_tensor(index2ptr(eis[0], N), eis[1], val[perm], (N, N))
    outs.update(out_wsum=o, gout_wsum=go, gx_wsum=xs.grad, gval_wsum=vs.grad,
                out_spmm_wsum=spmm(csr, x, "sum"), out_spmm_wmean=spmm(csr, x, "mean"))
    save("spmm", ei_sorted=eis, val_sorted=val[perm], x=x, N=N, **outs)

    # ---- aggregation modules (index path == ptr path, test/nn/aggr/test_basic.py:35-63)
    N, E, F = 6, 24, 4
    index = torch.sort(torch.randint(0, N - 1, (E, ), generator=g))[0]
    xa = torch.randn(E, F, generator=g)
    outs = {}
    for name, mod in (("sum", SumAggregation()), ("mean", MeanAggregation()),
                      ("max", MaxAggregation()), ("min", MinAggregation()),
                      ("softmax", SoftmaxAggregation(t=1.0))):
        outs["out_" + name] = mod(xa, index, dim_size=N)
    save("aggr", x=xa, index=index, ptr=index2ptr(index, N), N=N, **outs)

    # ---- GCNConv: Cora-shaped config 1 (2708 nodes / 10556 edges / h=16), 2 layers, fwd + bwd
    torch.manual_seed(11)
    N, E, F = 2708, 10556, 16
    ei = rand_graph(g, N, E)
    x = torch.randn(N, F, generator=g)
    c1, c2 = GCNConv(F, F), GCNConv(F, F)
    with torch.no_grad():
        c1.bias.copy_(torch.randn(F, generator=g) * 0.1)
        c2.bias.copy_(torch.randn(F, generator=g) * 0.1)
    xs = x.clone().requires_grad_()
    h1 = c1(xs, ei)
    o = c2(h1.relu(), ei)
    go = torch.randn(o.shape, generator=g)
    o.backward(go)
    save("gcn_cora", ei=ei, x=x, w1=c1.lin.weight, b1=c1.bias, w2=c2.lin.weight, b2=c2.bias,
         h1=h1, out=o, gout=go, gx=xs.grad, gw1=c1.lin.weight.grad, gb1=c1.bias.grad,
         gw2=c2.lin.weight.grad, gb2=c2.bias.grad)

    # ---- GCNConv small with edge weights + improved
    N, E, Fi, Fo = 17, 70, 5, 7
    ei = rand_graph(g, N, E)
    w = torch.rand(E, generator=g) + 0.2
    x = torch.randn(N, Fi, generator=g)
    conv = GCNConv(Fi, Fo, improved=True)
    xs = x.clone().requires_grad_()
    o = conv(xs, ei, w)
    go = torch.randn(o.shape, generator=g)
    o.backward(go)
    save("gcn_small", ei=ei, w=w, x=x, weight=conv.lin.weight, bias=conv.bias, out=o, gout=go,
         gx=xs.grad, gweight=conv.lin.weight.grad, gbias=conv.bias.grad)

    # ---- SAGEConv (mean + max), GIN aggregation
    N, E, Fi, Fo = 19, 80, 6, 5
    ei = rand_graph(g, N, E)
    x = torch.randn(N, Fi, generator=g)
    outs = {}
    for aggr in ("mean", "max", "sum"):
        conv = SAGEConv(Fi, Fo, aggr=aggr)
        xs = x.clone().requires_grad_()
        o = conv(xs, ei)
        go = torch.randn(o.shape, generator=torch.Generator().manual_seed(5))
        o.backward(go)
        outs.update({f"wl_{aggr}": conv.lin_l.weight, f"bl_{aggr}": conv.lin_l.bias,
                     f"wr_{aggr}": conv.lin_r.weight, f"out_{aggr}": o, f"gout_{aggr}": go,
                     f"gx_{aggr}": xs.grad, f"gwl_{aggr}": conv.lin_l.weight.grad,
                     f"gwr_{aggr}": conv.lin_r.weight.grad})
    gin = GINConv(torch.nn.Identity(), eps=0.25)
    outs["gin_out"] = gin(x, ei)
    save("sage_gin", ei=ei, x=x, **outs)

    # ---- GATConv 4 heads x 3 channels, fwd (out + attention) + bwd
    N, E, Fi, H, C = 15, 64, 6, 4, 3
    ei = rand_graph(g, N, E)
    x = torch.randn(N, Fi, generator=g)
    conv = GATConv(Fi, C, heads=H)
    xs = x.clone().requires_grad_()
    o, (ei2, alpha) = conv(xs, ei, return_attention_weights=True)
    go = torch.randn(o.shape, generator=g)
    o.backward(go)
    save("gat", ei=ei, x=x, lin=conv.lin.weight, att_src=conv.att_src, att_dst=conv.att_dst,
         bias=conv.bias, out=o, ei2=ei2, alpha=alpha, gout=go, gx=xs.grad, glin=conv.lin.weight.grad,
         gatt_src=conv.att_src.grad, gatt_dst=conv.att_dst.grad, slope=conv.negative_slope)

    # ---- RGCNConv 4 relations, default aggr='mean', per-relation loop (rgcn_conv.py:257-280)
    N, E, Fi, Fo, R = 14, 90, 5, 4, 4
    ei = rand_graph(g, N, E)
    et = torch.randint(0, R, (E, ), generator=g)
    x = torch.randn(N, Fi, generator=g)
    outs = {}
    for aggr in ("mean", "sum"):
        conv = RGCNConv(Fi, Fo, R, aggr=aggr)
        with torch.no_grad():
            conv.bias.copy_(torch.randn(Fo, generator=g) * 0.1)
        xs = x.clone().requires_grad_()
        o = conv(xs, ei, et)
        go = torch.randn(o.shape, generator=torch.Generator().manual_seed(6))
        o.backward(go)
        outs.update({f"weight_{aggr}": conv.weight, f"root_{aggr}": conv.root,
                     f"bias_{aggr}": conv.bias, f"out_{aggr}": o, f"gout_{aggr}": go,
                     f"gx_{aggr}": xs.grad, f"gweight_{aggr}": conv.weight.grad,
                     f"groot_{aggr}": conv.root.grad})
    save("rgcn", ei=ei, et=et, x=x, R=R, **outs)

    with open(os.path.join(OUT, "PROVENANCE.txt"), "w") as f:
        f.write(f"reference: torch_geometric {torch_geometric.__version__} (unmodified, oracle/install_ref.sh)\n"
                f"torch: {torch.__version__}\n"
                f"extensions: WITH_TORCH_SCATTER={tgt.WITH_TORCH_SCATTER} "
                f"WITH_TORCH_SPARSE={tgt.WITH_TORCH_SPARSE} WITH_PYG_LIB={tgt.WITH_PYG_LIB}\n"
                "generator: tests/golden/make_golden.py\n")


if __name__ == "__main__":
    main()
