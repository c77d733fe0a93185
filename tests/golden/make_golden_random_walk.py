"""Golden vectors for RootedRWSubgraph, the consumer of torch.ops.pyg.random_walk that the engine must reproduce bit for
bit: the UNMODIFIED reference transform on the CPU, with the numpy restatement of the walk contract from
tests/random_walk_oracle.py registered as the CPU implementation of torch.ops.pyg.random_walk in this script only
(pyg-lib is not installed, so the transform has no such operator otherwise).  The stand-in draws the walks' seed from
torch's CPU generator as ops.random_walk does, and the generator is seeded immediately before each call, so the CUDA
run of the test makes the same walks.  Cases: seeded random graphs (undirected, with self-loops, duplicate edges and a
node without out-edges) at two walk lengths and repeats.  Same provenance rules as make_golden.py (needs the reference
in oracle/_ref; writes tests/golden/random_walk.npz).

    python tests/golden/make_golden_random_walk.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))             # oracle/install_ref.sh
sys.path.insert(0, os.path.join(HERE, ".."))
import random_walk_oracle as RO  # noqa: E402
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.data import Data  # noqa: E402
from torch_geometric.transforms import RootedRWSubgraph  # noqa: E402

assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)
SCHEMA = "random_walk(Tensor rowptr, Tensor col, Tensor seed, int walk_length, float p=1.0, float q=1.0) -> Tensor"
# (graph seed, nodes, undirected edges, walk_length, repeat, torch seed)
CASES = [(1, 12, 20, 3, 1, 31), (2, 30, 70, 4, 3, 32), (3, 60, 90, 6, 2, 33)]


def graph(seed, n, m):
    """Undirected random graph plus two self-loops, a duplicate edge and one directed edge into the last node, which has
    no out-edges."""
    rng = np.random.default_rng(seed)
    a, b = rng.integers(0, n - 1, m), rng.integers(0, n - 1, m)
    row = np.concatenate([a, b, [0, 3, a[0], n - 2]])
    col = np.concatenate([b, a, [0, 3, b[0], n - 1]])
    return torch.from_numpy(np.stack([row, col]).astype(np.int64))


def main():
    lib = torch.library.Library("pyg", "FRAGMENT")
    lib.define(SCHEMA)
    lib.impl("random_walk", RO.torch_op(), "CPU")
    out = {}
    for i, (gseed, n, m, walk_length, repeat, tseed) in enumerate(CASES):
        data = Data(edge_index=graph(gseed, n, m), num_nodes=n)
        torch.manual_seed(tseed)
        sub = RootedRWSubgraph(walk_length, repeat)(data)
        out[f"c{i}_edge_index"] = data.edge_index.numpy()
        for k in ("sub_edge_index", "n_id", "e_id", "n_sub_batch", "e_sub_batch"):
            out[f"c{i}_{k}"] = getattr(sub, k).numpy()
    out["cases"] = np.array(CASES, np.int64)
    np.savez_compressed(os.path.join(HERE, "random_walk.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
