"""Golden vectors for the next attention row (SURVEY section 8(f) rank 2): the UNMODIFIED reference's GATv2Conv,
forward and backward, with and without shared weights.  Same provenance rules as make_golden.py (needs the
reference in oracle/_ref; writes tests/golden/gatv2.npz).

    python tests/golden/make_golden_gatv2.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import GATv2Conv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)


def main():
    g = torch.Generator().manual_seed(777)
    N, E, Fin, H, C = 11, 60, 6, 4, 3
    ei = torch.stack([torch.randint(0, N, (E, ), generator=g), torch.randint(0, N - 1, (E, ), generator=g)])
    ei[:, :3] = torch.tensor([[1, 1, 4], [1, 1, 4]])          # existing (duplicated) self loops; node N-1 has no in-edge
    x = torch.randn(N, Fin, generator=g)
    arrs = {"ei": ei.numpy(), "x": x.numpy(), "H": np.asarray(H), "C": np.asarray(C)}
    for tag, share in (("sep", False), ("shared", True)):
        torch.manual_seed(5 + int(share))
        conv = GATv2Conv(Fin, C, heads=H, share_weights=share)
        with torch.no_grad():
            conv.bias.normal_(0, 0.1)
        xr = x.clone().requires_grad_()
        out, (ei2, alpha) = conv(xr, ei, return_attention_weights=True)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_lin_l_w": conv.lin_l.weight, f"{tag}_lin_l_b": conv.lin_l.bias,
                     f"{tag}_lin_r_w": conv.lin_r.weight, f"{tag}_lin_r_b": conv.lin_r.bias,
                     f"{tag}_att": conv.att.view(H, C), f"{tag}_bias": conv.bias, f"{tag}_out": out, f"{tag}_ei2": ei2,
                     f"{tag}_alpha": alpha, f"{tag}_gout": gout, f"{tag}_gx": xr.grad,
                     f"{tag}_g_att": conv.att.grad.view(H, C), f"{tag}_g_lin_l_w": conv.lin_l.weight.grad})
    conv_np = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "gatv2.npz"), **conv_np)
    print("wrote gatv2", len(conv_np), "arrays")


if __name__ == "__main__":
    main()
