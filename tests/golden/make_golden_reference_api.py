"""Golden data for the two comparisons with the reference's Python API that need no engine on the reference side:
  * state_dict_layout.json -- keys and shapes of the reference layers' state_dicts for every case of
    tests/test_cabi_cpu.py::STATE_DICT_CASES (checkpoint interchangeability);
  * index_bookkeeping.npz  -- the reference's scatter_argmax / group_argsort / group_cat (utils/_scatter.py:145-300) on
    seeded, tie-free inputs (tests/test_gpu_plugin.py::test_index_bookkeeping_mirrors_match_the_reference).
Same provenance rules as make_golden.py (needs the reference in oracle/_ref).

    python tests/golden/make_golden_reference_api.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))
import torch_geometric  # noqa: E402
from torch_geometric.utils._scatter import scatter_argmax  # noqa: E402  (not re-exported by utils/__init__)

from test_cabi_cpu import STATE_DICT_CASES  # noqa: E402
from test_gpu_plugin import GROUP_ARGSORT_KW  # noqa: E402


def layouts():
    out = []
    for name, args, kw in STATE_DICT_CASES():
        sd = getattr(torch_geometric.nn, name)(*args, **kw).state_dict()
        out.append({"layer": name, "shapes": {k: list(v.shape) for k, v in sd.items()}})
    with open(os.path.join(HERE, "state_dict_layout.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


def bookkeeping():
    g = torch.Generator().manual_seed(12)
    N, E = 70, 900
    index = torch.randint(0, N - 5, (E, ), generator=g)
    src = torch.randperm(E, generator=g).float() * 0.37 - 100.0          # tie-free: the reference leaves ties to scatter order
    x1, x2 = torch.randn(40, 3, generator=g), torch.randn(25, 3, generator=g)
    i1, i2 = torch.sort(torch.randint(0, 9, (40, ), generator=g))[0], torch.sort(torch.randint(0, 9, (25, ), generator=g))[0]
    arrs = {"N": np.asarray(N), "index": index.numpy(), "src": src.numpy(), "x1": x1.numpy(), "x2": x2.numpy(),
            "i1": i1.numpy(), "i2": i2.numpy(),
            "argmax": scatter_argmax(src, index, dim_size=N).numpy(), "argmax_nodim": scatter_argmax(src, index).numpy()}
    for i, kw in enumerate(GROUP_ARGSORT_KW):
        arrs[f"argsort_{i}"] = torch_geometric.utils.group_argsort(src, index, **kw).numpy()
    cat, cat_index = torch_geometric.utils.group_cat([x1, x2], [i1, i2], return_index=True)
    arrs.update(cat=cat.numpy(), cat_index=cat_index.numpy())
    np.savez_compressed(os.path.join(HERE, "index_bookkeeping.npz"), **arrs)


if __name__ == "__main__":
    layouts()
    bookkeeping()
    print("wrote state_dict_layout.json and index_bookkeeping.npz")
