"""Golden vectors for the mini-batch side (SURVEY section 8(f) rank 4) from the UNMODIFIED reference:
`trim_to_layer` driving a 3-layer SAGE model over a BFS-ordered sampled subgraph (the layout NeighborLoader emits:
hops concatenated, each hop grouped by destination), and `coalesce` with duplicates and every reduce.
Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes tests/golden/minibatch.npz).

    python tests/golden/make_golden_minibatch.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import SAGEConv  # noqa: E402
from torch_geometric.utils import coalesce, trim_to_layer  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)


def bfs_sample(g, n_seed=6, fanouts=(4, 3, 2), n_pool=200):
    """Edges (src = sampled neighbour, dst = frontier node) hop by hop; node ids in order of first appearance."""
    nodes = list(range(n_seed))
    frontier = list(range(n_seed))
    src, dst, nodes_per_hop, edges_per_hop = [], [], [n_seed], []
    next_id = n_seed
    for f in fanouts:
        new_frontier, e0 = [], len(src)
        for d in frontier:
            k = int(torch.randint(0, f + 1, (1, ), generator=g))
            for _ in range(k):
                if float(torch.rand(1, generator=g)) < 0.25 and next_id > 0:      # sometimes an already-sampled node
                    s = int(torch.randint(0, next_id, (1, ), generator=g))
                else:
                    s = next_id
                    next_id += 1
                    new_frontier.append(s)
                src.append(s)
                dst.append(d)
        nodes_per_hop.append(len(new_frontier))
        edges_per_hop.append(len(src) - e0)
        frontier = new_frontier
    return torch.tensor([src, dst]), nodes_per_hop, edges_per_hop, next_id


def main():
    g = torch.Generator().manual_seed(4242)
    ei, nodes_per_hop, edges_per_hop, n = bfs_sample(g)
    assert bool((ei[1][1:] >= ei[1][:-1]).all())                                  # destination-sorted, as the loader emits
    F = 8
    x = torch.randn(n, F, generator=g)
    torch.manual_seed(9)
    convs = [SAGEConv(F, F) for _ in range(3)]
    h = x.clone().requires_grad_()
    xr = h
    arrs = {"ei": ei.numpy(), "x": x.numpy(), "nodes_per_hop": np.asarray(nodes_per_hop), "edges_per_hop": np.asarray(edges_per_hop)}
    e = ei
    for i, conv in enumerate(convs):
        h, e, _ = trim_to_layer(i, nodes_per_hop, edges_per_hop, h, e)
        arrs[f"trim{i}_ei"] = e.numpy().copy()
        arrs[f"trim{i}_n"] = np.asarray(h.size(0))
        h = conv(h, e)
        if i < 2:
            h = h.relu()
        arrs[f"h{i}"] = h.detach().numpy().copy()
        arrs[f"conv{i}_lin_l_w"] = conv.lin_l.weight.detach().numpy()
        arrs[f"conv{i}_lin_l_b"] = conv.lin_l.bias.detach().numpy()
        arrs[f"conv{i}_lin_r_w"] = conv.lin_r.weight.detach().numpy()
    out = h[:nodes_per_hop[0]]
    gout = torch.randn(out.shape, generator=g)
    out.backward(gout)
    arrs.update({"out": out.detach().numpy(), "gout": gout.numpy(), "gx": xr.grad.numpy()})
    # ---- coalesce
    ce = torch.randint(0, 7, (2, 60), generator=g)
    ca = torch.randn(60, 3, generator=g)
    arrs.update({"c_ei": ce.numpy(), "c_attr": ca.numpy()})
    for reduce in ("sum", "mean", "min", "max"):
        for by_row in (True, False):
            oe, oa = coalesce(ce, ca, num_nodes=7, reduce=reduce, sort_by_row=by_row)
            arrs[f"c_{reduce}_{int(by_row)}_ei"] = oe.numpy()
            arrs[f"c_{reduce}_{int(by_row)}_attr"] = oa.numpy()
    np.savez_compressed(os.path.join(OUT, "minibatch.npz"), **arrs)
    print("wrote minibatch", len(arrs), "arrays; nodes/hop", nodes_per_hop, "edges/hop", edges_per_hop)


if __name__ == "__main__":
    main()
