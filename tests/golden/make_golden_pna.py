"""Golden vectors for PNAConv (pna_conv.py:20-209): the UNMODIFIED reference's layer on the CPU, forward and backward,
for three cases -- `PNAConv(16, 32)` with all six aggregators, all five scalers, `towers=4`, `edge_dim=3`; `towers=2`,
`divide_input=True`, `post_layers=2` without edge features; `towers=1`, `edge_dim=5`, `train_norm=True` with
[mean, min, max, std] x [identity, amplification, attenuation] (the examples/pna.py choice) -- plus the `state_dict`
shapes and the repr of each.  Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes
tests/golden/pna.npz).

    python tests/golden/make_golden_pna.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import PNAConv  # noqa: E402
from torch_geometric.utils import degree  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

ALL_AGGRS = ["mean", "min", "max", "std", "sum", "var"]
ALL_SCALERS = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
# (tag, in_channels, out_channels, constructor kwargs)
CASES = [("all", 16, 32, dict(aggregators=ALL_AGGRS, scalers=ALL_SCALERS, towers=4, edge_dim=3)),
         ("divide", 16, 32, dict(aggregators=["sum", "max", "var"], scalers=["identity", "linear"], towers=2,
                                 divide_input=True, post_layers=2)),
         ("train_norm", 12, 8, dict(aggregators=["mean", "min", "max", "std"],
                                    scalers=["identity", "amplification", "attenuation"], edge_dim=5, train_norm=True))]


def main():
    g = torch.Generator().manual_seed(6262)
    N, E = 13, 70
    arrs = {}
    for k, (tag, ic, oc, kw) in enumerate(CASES):
        ei = torch.stack([torch.randint(0, N, (E, ), generator=g), torch.randint(0, N - 1, (E, ), generator=g)])
        ei[:, 1] = ei[:, 0]                                    # a duplicated edge; destination N-1 has no in-edge
        ei[1, 2:40] = 3                                        # one row far above the others
        deg = torch.bincount(degree(ei[1], N, dtype=torch.long))
        x = torch.randint(-3, 4, (N, ic), generator=g).float()  # small integers: exact min / max ties
        ea = torch.randn(E, kw["edge_dim"], generator=g) if kw.get("edge_dim") else None
        torch.manual_seed(31 + k)
        conv = PNAConv(ic, oc, deg=deg, **kw)
        xr = x.clone().requires_grad_()
        ear = ea.clone().requires_grad_() if ea is not None else None
        out = conv(xr, ei, ear)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_deg": deg, f"{tag}_x": x, f"{tag}_out": out, f"{tag}_gout": gout,
                     f"{tag}_gx": xr.grad})
        if ea is not None:
            arrs.update({f"{tag}_ea": ea, f"{tag}_gea": ear.grad})
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p
        for name, p in conv.named_parameters():
            if p.grad is not None:                             # avg_deg_lin is unused without a linear scaler
                arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({n: list(p.shape) for n, p in conv.state_dict().items()}))
        arrs[f"{tag}_repr"] = np.asarray(repr(conv))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "pna.npz"), **np_arrs)
    print("wrote pna", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
