"""Golden vectors for GENConv (gen_conv.py:45-243): the UNMODIFIED reference's layer on the CPU, forward and backward
in training mode, for seven cases -- softmax with a learnable t; softmax_sg; powermean with a fixed p = 2.5; powermean
with a learnable per-channel p; edge_dim with lin_edge; a bipartite layer with lin_src and lin_dst; msg_norm with a
learnable scale -- plus the state_dict shapes and the repr of each.  The graph has a duplicated edge and a destination
without in-edges.  Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes
tests/golden/gen.npz).

    python tests/golden/make_golden_gen.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import GENConv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

# (tag, in_channels, constructor kwargs, edge_dim of the input edge features or None, bipartite)
CASES = [("softmax_learn", 16, {"aggr": "softmax", "learn_t": True}, None, False),
         ("softmax_sg", 16, {"aggr": "softmax_sg", "t": 0.5}, None, False),
         ("pm_fixed", 16, {"aggr": "powermean", "p": 2.5}, None, False),
         ("pm_learn_channels", 16, {"aggr": "powermean", "aggr_kwargs": {"p": 1.5, "learn": True, "channels": 16}},
          None, False),
         ("edge", 16, {"aggr": "softmax", "learn_t": True, "edge_dim": 4}, 4, False),
         ("bipartite", (8, 12), {"aggr": "powermean", "learn_p": True, "norm": None}, None, True),
         ("msg_norm", 16, {"aggr": "softmax", "msg_norm": True, "learn_msg_scale": True}, None, False)]
OUT_CH = 16


def main():
    g = torch.Generator().manual_seed(9090)
    N_src, N_dst, E = 13, 9, 70
    arrs = {}
    for k, (tag, ch, kw, edim, bip) in enumerate(CASES):
        n_dst = N_dst if bip else N_src
        f_src, f_dst = (ch, ch) if isinstance(ch, int) else ch
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(0, n_dst - 1, (E, ), generator=g)])
        ei[:, 1] = ei[:, 0]                                    # a duplicated edge; destination n_dst-1 has no in-edge
        x = torch.randn(N_src, f_src, generator=g)
        x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
        ea = torch.randn(E, edim, generator=g) if edim else None
        torch.manual_seed(41 + k)
        conv = GENConv(ch, OUT_CH, **kw)
        with torch.no_grad():
            for name, p in conv.named_parameters():
                if name in ("aggr_module.t", "aggr_module.p"):   # learnable t / p away from their initial value
                    p.copy_(torch.rand(p.shape, generator=g) + 0.75)
                elif name.startswith("mlp.1."):                  # the reference initialises BatchNorm to 1 and 0
                    p.normal_(generator=g)
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p.clone()
        conv.train()
        xr = x.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        ear = ea.clone().requires_grad_() if edim else None
        out = conv((xr, xdr) if bip else xr, ei, ear)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_x": x, f"{tag}_out": out, f"{tag}_gout": gout, f"{tag}_gx": xr.grad})
        if bip:
            arrs.update({f"{tag}_x_dst": x_dst, f"{tag}_gx_dst": xdr.grad})
        if edim:
            arrs.update({f"{tag}_ea": ea, f"{tag}_gea": ear.grad})
        for name, p in conv.named_parameters():
            if p.grad is not None:
                arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({n: list(p.shape) for n, p in conv.state_dict().items()}))
        arrs[f"{tag}_repr"] = np.asarray(repr(conv))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "gen.npz"), **np_arrs)
    print("wrote gen", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
