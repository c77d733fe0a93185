"""Writes quantile.npz and PROVENANCE_quantile.txt from the UNMODIFIED reference QuantileAggregation /
MedianAggregation (torch_geometric/nn/aggr/quantile.py) on the CPU:

    PYTHONPATH=<pytorch_geometric 2.9.0 source tree> python tests/golden/make_golden_quantile.py

Each case stores x (float32 values; bf16 cases hold bf16 values), index, the module's arguments, the forward output
and the gradient of (out * w).sum() for a seeded w.  Cases: every interpolation with q = 0.5 and q = [0, 0.1, 0.5,
0.9, 1]; fill_value 0 and 10 with dim_size larger than needed; an unsorted index; 3-D x aggregated along dim 0 and
dim 1; bf16; ties, +-0, NaN and +-inf; a 'nearest' group at an odd offset with frac 0.5; MedianAggregation.  No group
0 is empty: there the reference raises IndexError for floor-based ranks (floor(-q) = -1)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
INTERP = ("linear", "lower", "higher", "nearest", "midpoint")
Q5 = [0.0, 0.1, 0.5, 0.9, 1.0]


def _groups(rng, sizes):
    return np.repeat(np.arange(len(sizes)), sizes)


def _values(rng, E, W, kind):
    if kind == "ties":
        return rng.integers(-3, 4, size=(E, W)).astype(np.float32)
    if kind == "special":
        pool = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.0, -1.0, 2.5], dtype=np.float32)
        return pool[rng.integers(0, len(pool), size=(E, W))]
    return rng.standard_normal((E, W)).astype(np.float32)


def main():
    from torch_geometric.nn.aggr import MedianAggregation, QuantileAggregation
    import torch_geometric
    rng = np.random.default_rng(20261018)
    sizes = [3, 1, 2, 0, 7, 4, 12, 5, 1, 9]                  # group 3 is empty
    cases = {}

    def add(name, x, index, kwargs, dim_size=None, dim=-2, bf16=False, median=False):
        xt = torch.from_numpy(x)
        if bf16:
            xt = xt.to(torch.bfloat16)
        xt.requires_grad_(True)
        it = torch.from_numpy(index)
        mod = MedianAggregation(**kwargs) if median else QuantileAggregation(**kwargs)
        out = mod(xt, it, dim_size=dim_size, dim=dim)
        w = torch.from_numpy(rng.standard_normal(tuple(out.shape)).astype(np.float32))
        (out.float() * w).sum().backward()
        cases[name] = dict(x=xt.detach().float().numpy(), index=index, w=w.numpy(), out=out.detach().float().numpy(),
                           grad=xt.grad.float().numpy(), bf16=np.array(bf16), median=np.array(median),
                           q=np.array(kwargs.get("q", 0.5), dtype=np.float64).reshape(-1),
                           interpolation=np.array(kwargs.get("interpolation", "lower")),
                           fill=np.array(kwargs.get("fill_value", 0.0), dtype=np.float64),
                           dim_size=np.array(-1 if dim_size is None else dim_size), dim=np.array(dim),
                           out_dtype=np.array(str(out.dtype)))

    idx = _groups(rng, sizes)
    E = idx.size
    for interp in INTERP:
        for qn, q in (("q05", 0.5), ("q5", Q5)):
            add(f"{interp}_{qn}", _values(rng, E, 4, "normal"), idx, dict(q=q, interpolation=interp))
            add(f"{interp}_{qn}_ties", _values(rng, E, 4, "ties"), idx, dict(q=q, interpolation=interp))
            add(f"{interp}_{qn}_bf16", _values(rng, E, 8, "ties" if qn == "q5" else "normal"), idx,
                dict(q=q, interpolation=interp), bf16=True)
        add(f"{interp}_special", _values(rng, E, 5, "special"), idx, dict(q=Q5, interpolation=interp))
        add(f"{interp}_fill10_dimsize", _values(rng, E, 3, "normal"), idx,
            dict(q=[0.25, 0.75], interpolation=interp, fill_value=10.0), dim_size=len(sizes) + 3)
        perm = rng.permutation(E)
        add(f"{interp}_unsorted", _values(rng, E, 3, "ties"), idx[perm], dict(q=Q5, interpolation=interp))
        x3 = _values(rng, E * 2 * 3, 1, "normal").reshape(E, 2, 3)
        add(f"{interp}_3d_dim0", x3, idx, dict(q=[0.3, 0.6], interpolation=interp), dim=0)
        x3b = _values(rng, 2 * E * 3, 1, "normal").reshape(2, E, 3)
        add(f"{interp}_3d_dim1", x3b, idx, dict(q=[0.3, 0.6], interpolation=interp), dim=1)
        add(f"{interp}_lastdim", _values(rng, 2, E, "normal"), idx, dict(q=Q5, interpolation=interp), dim=-1)
    # 'nearest' with frac 0.5: groups of 3 at q = 0.25 give P = ptr + 0.5, so an odd offset rounds up, an even one down
    idx_n = _groups(rng, [3, 3, 2, 3, 3])
    add("nearest_half_offsets", _values(rng, idx_n.size, 4, "normal"), idx_n, dict(q=0.25, interpolation="nearest"))
    add("median", _values(rng, E, 4, "normal"), idx, dict(fill_value=-1.0), median=True)
    add("median_bf16", _values(rng, E, 8, "ties"), idx, dict(), bf16=True, median=True)

    flat = {f"{name}/{k}": v for name, c in cases.items() for k, v in c.items()}
    np.savez_compressed(os.path.join(HERE, "quantile.npz"), **flat)
    with open(os.path.join(HERE, "PROVENANCE_quantile.txt"), "w") as fh:
        fh.write("quantile.npz: written by tests/golden/make_golden_quantile.py from the unmodified reference\n"
                 f"torch_geometric {torch_geometric.__version__} (nn/aggr/quantile.py) on the CPU with torch "
                 f"{torch.__version__.split('+')[0]}, numpy seed 20261018; {len(cases)} cases:\n")
        for name in cases:
            fh.write(f"  {name}\n")


if __name__ == "__main__":
    sys.exit(main())
