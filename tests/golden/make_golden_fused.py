"""Golden vectors for the multi-aggregation sweep: the UNMODIFIED reference's FusedAggregation
(torch_geometric/nn/aggr/fused.py) and MultiAggregation (multi.py), forward and backward, on seeded
inputs with empty groups, ties and constant groups (std mask).  Same provenance rules as make_golden.py
(needs the reference in oracle/_ref; writes tests/golden/fused_aggr.npz).

    python tests/golden/make_golden_fused.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn.aggr import MultiAggregation  # noqa: E402
from torch_geometric.nn.aggr.fused import FusedAggregation  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

CASES = {
    "all": ["sum", "mean", "min", "max", "var", "std"],
    "pna": ["mean", "min", "max", "std"],          # the PNAConv default aggregator set
    "sumstd": ["sum", "std"],
    "var": ["var"],
    "minmax": ["min", "max"],
}


def main():
    g = torch.Generator().manual_seed(4321)
    N, E, F = 12, 90, 5
    index = torch.randint(0, N - 2, (E, ), generator=g)
    index[index == 4] = 5                          # groups 4, 10, 11 are empty
    x = torch.randn(E, F, generator=g)
    x[index == 2] = x[index == 2][0]               # a constant group: var = 0, std masked to 0
    x[5, :] = x[7, :] = 0.0                        # zeros
    x[index == 6, 1] = torch.relu(x[index == 6, 1])    # ties at 0 for min (post-ReLU pattern)
    x[index == 7, 2] = x[index == 7, 2].round()         # integer ties for min / max
    arrs = {"x": x.numpy(), "index": index.numpy(), "N": np.asarray(N)}
    for name, aggrs in CASES.items():
        xr = x.clone().requires_grad_()
        outs = FusedAggregation(aggrs)(xr, index, dim_size=N)
        gouts = [torch.randn(o.shape, generator=g) for o in outs]
        torch.autograd.backward(outs, gouts)
        for a, o, go in zip(aggrs, outs, gouts):
            arrs[f"{name}_out_{a}"] = o.detach().numpy()
            arrs[f"{name}_gout_{a}"] = go.numpy()
        arrs[f"{name}_gx"] = xr.grad.numpy()
    # MultiAggregation(mode='cat') through the fused path
    xr = x.clone().requires_grad_()
    out = MultiAggregation(CASES["pna"], mode="cat")(xr, index, dim_size=N)
    go = torch.randn(out.shape, generator=g)
    out.backward(go)
    arrs.update(multi_cat_out=out.detach().numpy(), multi_cat_gout=go.numpy(), multi_cat_gx=xr.grad.numpy())
    np.savez_compressed(os.path.join(OUT, "fused_aggr.npz"), **arrs)
    print("wrote fused_aggr", len(arrs), "arrays")


if __name__ == "__main__":
    main()
