"""Random walks on the GPU (csrc/random_walk.cu): ops.random_walk equals the numpy oracle of tests/random_walk_oracle.py
bit for bit -- int32 / int64 indices, uniform and node2vec walks (p = 10^-3 and q = 10^3 included), sorted and
unsorted rows, the exact fallback forced (max_trials 0 and 1), self-loops, duplicate edges, dead ends, L = 0, S = 0,
repeated starts and a 1M-node power-law graph with hubs; out-of-range starts and column values give -1 rows and raise
in debug mode; nothing synchronises, the cached row-order flag included; and the unmodified reference's
RootedRWSubgraph, dropout_path and Node2Vec run on CUDA tensors after plugin.install(layers=True, flip_flags=True)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random_walk_oracle as RO  # noqa: E402

import pytorch_geometric_b200 as pgb  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200 import utils as U  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _eq(got, want, what=""):
    got = got.cpu().numpy().astype(np.int64)
    want = np.asarray(want)
    assert got.shape == want.shape, f"{what}: {got.shape} vs {want.shape}"
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} differ, first at {bad[:3].tolist()}: {got[tuple(bad[0])]} vs " \
                          f"{want[tuple(bad[0])]}"


def _power_law(n, avg, seed):
    """Symmetric graph: sources uniform, targets Pareto-distributed over the node ids (hubs at the low ids)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, n, n * avg // 2)
    b = (rng.pareto(1.2, a.size) * 8).astype(np.int64) % n
    return np.concatenate([a, b]), np.concatenate([b, a])


def _csr(n, row, col, shuffle_rows=None):
    """CSR with rows non-decreasing, or (shuffle_rows = a seed) each row's entries in random order."""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    inner = col if shuffle_rows is None else np.random.default_rng(shuffle_rows).random(col.size)
    o = np.lexsort((inner, row))
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))]).astype(np.int64)
    return rowptr, col[o]


def _graph(n=3000, seed=1, shuffle_rows=None):
    """Power law plus self-loops and duplicate edges; every node with id % 50 == 7 loses its out-edges (dead ends)."""
    row, col = _power_law(n, 6, seed)
    row = np.concatenate([row, np.arange(0, n, 97), row[:80]])
    col = np.concatenate([col, np.arange(0, n, 97), col[:80]])
    keep = row % 50 != 7
    return _csr(n, row[keep], col[keep], shuffle_rows)


def _walk(rowptr, col, start, L, p=1.0, q=1.0, seed=0, max_trials=ops.RANDOM_WALK_MAX_TRIALS, idx=torch.int64):
    t = (lambda a: torch.from_numpy(np.asarray(a, np.int64)).to(DEV, idx))
    out = ops.random_walk(t(rowptr), t(col), t(start), L, p, q, seed=seed, max_trials=max_trials)
    assert out.dtype == idx and out.shape == (len(start), L + 1)
    return out


PQ = [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25), (1e-3, 1e3)]


@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
@pytest.mark.parametrize("p,q", PQ)
@pytest.mark.parametrize("sorted_rows", [True, False])
def test_walks_equal_the_oracle(idx, p, q, sorted_rows):
    n = 3000
    rowptr, col = _graph(n, 1, None if sorted_rows else 5)
    assert RO.rows_sorted(rowptr, col) == sorted_rows
    start = np.concatenate([np.arange(n), np.arange(0, n, 7)])            # repeated starts: one stream each
    for L, seed in ((37, 11), (5, 2**64 - 3)):                           # 37: two staging passes
        _eq(_walk(rowptr, col, start, L, p, q, seed, idx=idx), RO.random_walk(rowptr, col, start, L, p, q, seed),
            f"idx={idx} p={p} q={q} sorted={sorted_rows} L={L}")


@pytest.mark.parametrize("max_trials", [0, 1])
@pytest.mark.parametrize("p,q", PQ[1:])
@pytest.mark.parametrize("sorted_rows", [True, False])
def test_the_exact_fallback_equals_the_oracle(max_trials, p, q, sorted_rows):
    n = 2000
    rowptr, col = _graph(n, 2, None if sorted_rows else 6)
    start = np.arange(n)
    _eq(_walk(rowptr, col, start, 9, p, q, 3, max_trials),
        RO.random_walk(rowptr, col, start, 9, p, q, 3, max_trials), f"max_trials={max_trials} p={p} q={q}")


def test_lengths_sizes_and_tiny_graphs():
    rowptr, col = _graph(500, 3)
    start = np.array([4, 4, 4, 9, 7, 57])                                 # 7 and 57 are dead ends
    w = _walk(rowptr, col, start, 0, 0.5, 2.0, 1)
    _eq(w, start[:, None], "L = 0")
    assert _walk(rowptr, col, np.array([], np.int64), 6).shape == (0, 7)
    w = _walk(rowptr, col, start, 6, 0.5, 2.0, 1).cpu().numpy()
    assert len({tuple(r) for r in w[:3]}) > 1                             # repeated starts draw their own streams
    assert (w[4] == 7).all() and (w[5] == 57).all()
    _eq(_walk([0], [], [0, -1], 3), np.full((2, 4), -1), "no nodes")
    _eq(_walk([0, 0], [], [0], 3, 2.0, 0.5), np.zeros((1, 4)), "one node, no edges")
    _eq(_walk([0, 1], [0], [0, 0], 4, 0.3, 3.0, 5), np.zeros((2, 5)), "one self-loop")


def test_a_1m_node_power_law_graph_with_hubs():
    n = 1_000_000
    rowptr, col = _csr(n, *_power_law(n, 10, 4))
    assert np.diff(rowptr).max() > 10_000
    start = np.random.default_rng(0).integers(0, n, 200_000)
    for p, q in ((1.0, 1.0), (0.25, 4.0)):
        _eq(_walk(rowptr, col, start, 10, p, q, 77), RO.random_walk(rowptr, col, start, 10, p, q, 77),
            f"1M p={p} q={q}")


def test_out_of_range_starts_and_columns():
    rowptr, col = _graph(400, 4)
    col = col.copy()
    deg = np.diff(rowptr)
    a, b = np.nonzero((deg >= 1) & (deg <= 3))[0][:2]                     # rows of one to three entries
    col[rowptr[a]], col[rowptr[b]] = 403, -5                              # one entry of each out of range
    start = np.array([-1, 400, a, b, 0, 1, 2] * 20)
    for p, q in ((1.0, 1.0), (0.5, 2.0)):
        got = _walk(rowptr, col, start, 8, p, q, 9)
        want = RO.random_walk(rowptr, col, start, 8, p, q, 9)
        _eq(got, want, f"out of range p={p}")
        g = got.cpu().numpy()
        assert (g[0] == -1).all() and (g[1] == -1).all()
        ended = (g == -1).any(1) & (g[:, 0] >= 0)
        assert ended.any()                                                # some walk met a stray column value
        for r in g[ended]:                                                # ... and is -1 from there on
            k = np.argmax(r == -1)
            assert (r[k:] == -1).all()
    t = (lambda a: torch.from_numpy(np.asarray(a, np.int64)).to(DEV))
    with pgb.debug():
        with pytest.raises(IndexError, match="start"):
            ops.random_walk(t(rowptr), t(_graph(400, 4)[1]), t([0, 400]), 3)
        with pytest.raises(IndexError, match="col"):
            ops.random_walk(t(rowptr), t(col), t([0, 1]), 3)


def test_deterministic_and_seeded_by_the_cpu_generator():
    rowptr, col = _graph(5000, 5)
    rp, c = torch.from_numpy(rowptr).to(DEV), torch.from_numpy(col).to(DEV)
    s = torch.arange(5000, device=DEV)
    assert torch.equal(ops.random_walk(rp, c, s, 12, 0.5, 2.0, seed=5), ops.random_walk(rp, c, s, 12, 0.5, 2.0, seed=5))
    torch.manual_seed(4)
    a = ops.random_walk(rp, c, s, 12, 0.5, 2.0)
    torch.manual_seed(4)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    assert torch.equal(a, ops.random_walk(rp, c, s, 12, 0.5, 2.0, seed=seed))


def test_the_row_order_flag_follows_in_place_changes():
    n = 1500
    rowptr, col = _graph(n, 7)
    rp, c = torch.from_numpy(rowptr).to(DEV), torch.from_numpy(col).to(DEV)
    start = np.arange(n)
    s = torch.from_numpy(start).to(DEV)
    _eq(ops.random_walk(rp, c, s, 7, 0.25, 4.0, seed=1), RO.random_walk(rowptr, col, start, 7, 0.25, 4.0, 1), "sorted")
    shuffled = _graph(n, 7, shuffle_rows=8)[1]
    c.copy_(torch.from_numpy(shuffled))                                  # same tensor, new version: the flag is redone
    _eq(ops.random_walk(rp, c, s, 7, 0.25, 4.0, seed=1), RO.random_walk(rowptr, shuffled, start, 7, 0.25, 4.0, 1),
        "shuffled in place")


def test_no_synchronisation():
    rowptr, col = _graph(5000, 8)
    rp, c = torch.from_numpy(rowptr).to(DEV), torch.from_numpy(col).to(DEV)
    c2 = c.clone()
    s = torch.arange(5000, device=DEV)
    ops.random_walk(rp, c, s, 10)
    ops.random_walk(rp, c, s, 10, 0.5, 2.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ops.random_walk(rp, c, s, 10)
        ops.random_walk(rp, c, s, 10, 0.5, 2.0)                          # the cached row-order flag
        ops.random_walk(rp, c2, s, 10, 2.0, 0.5)                         # a new graph: the flag is computed on the device
        ops.random_walk(rp, c2, s, 10, 2.0, 0.5, max_trials=0)
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---------------------------------------------------------------------------------------------- the reference
@pytest.fixture
def tg_walk(tg):
    from pytorch_geometric_b200 import plugin
    plugin.install(layers=True, flip_flags=True)
    yield tg
    plugin.uninstall()


def test_reference_rooted_rw_subgraph_matches_golden(tg_walk, golden):
    from torch_geometric.data import Data
    from torch_geometric.transforms import RootedRWSubgraph
    z = golden("random_walk")
    for i, (_, n, _, walk_length, repeat, tseed) in enumerate(z["cases"].tolist()):
        data = Data(edge_index=torch.from_numpy(z[f"c{i}_edge_index"]).to(DEV), num_nodes=n)
        torch.manual_seed(tseed)
        sub = RootedRWSubgraph(walk_length, repeat)(data)
        for k in ("sub_edge_index", "n_id", "e_id", "n_sub_batch", "e_sub_batch"):
            got = getattr(sub, k)
            assert got.is_cuda
            _eq(got, z[f"c{i}_{k}"], f"case {i} {k}")


def _replay_dropout_path(edge_index, p, walks_per_node, walk_length, tseed):
    """dropout_path's draws replayed: the start mask from torch's CUDA generator, the walks' seed from its CPU
    generator, the walks from the oracle and the composition in numpy."""
    row, col = edge_index.cpu().numpy()
    n = int(edge_index.max()) + 1
    torch.manual_seed(tseed)
    sample = (torch.rand(row.size, device=DEV) <= p).cpu().numpy()
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    order = np.lexsort((col, row))
    rs, cs = row[order], col[order]
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(rs, minlength=n))])
    walk = RO.random_walk(rowptr, cs, np.tile(rs[sample], walks_per_node), walk_length, seed=seed)
    keys = walk[:, :-1].reshape(-1) * n + walk[:, 1:].reshape(-1)
    hit = np.isin(rs * n + cs, keys)
    mask = np.ones(row.size, bool)
    mask[order[hit]] = False
    return mask


def test_reference_dropout_path_replays_exactly(tg_walk):
    from torch_geometric.utils import dropout_path
    row, col = _power_law(3000, 6, 9)
    row, col = np.concatenate([row, row[:40]]), np.concatenate([col, col[:40]])     # duplicate edges
    ei = torch.from_numpy(np.stack([row, col])).to(DEV)
    for p, wpn, L, tseed in ((0.2, 1, 3, 1), (0.5, 2, 5, 2)):
        torch.manual_seed(tseed)
        kept, mask = dropout_path(ei, p, wpn, L)
        assert kept.is_cuda and mask.is_cuda
        assert torch.equal(ei[:, mask], kept)
        want = _replay_dropout_path(ei, p, wpn, L, tseed)
        assert np.array_equal(mask.cpu().numpy(), want) and (~want).any()
        torch.manual_seed(tseed)
        kept2, mask2 = U.dropout_path(ei, p, wpn, L)                     # the standalone mirror
        assert torch.equal(mask2, mask) and torch.equal(kept2, kept)
    for kw in ({"p": 0.0}, {"training": False}):
        kept, mask = dropout_path(ei, **kw)
        assert kept is ei and bool(mask.all())
    import torch_geometric.typing as T
    assert T.WITH_PYG_LIB is False


def _sbm(blocks=4, size=100, p_in=0.08, p_out=0.002, seed=0):
    rng = np.random.default_rng(seed)
    n = blocks * size
    y = np.repeat(np.arange(blocks), size)
    prob = np.where(y[:, None] == y[None, :], p_in, p_out)
    a = np.triu(rng.random((n, n)) < prob, 1)
    r, c = np.nonzero(a | a.T)
    return torch.from_numpy(np.stack([r, c])), torch.from_numpy(y)


def test_reference_node2vec_walks_and_training(tg_walk):
    from pytorch_geometric_b200.nn import Node2Vec as Mirror
    from pytorch_geometric_b200.plugin.models import B200Node2Vec
    ei, y = _sbm()
    ei = torch.cat([ei, torch.tensor([[0], [399]])], 1)                  # node 399 keeps an in-edge
    ei = ei[:, ei[0] != 399]                                             # ... and has no out-edge: a dead end
    torch.manual_seed(0)
    model = tg_walk.nn.Node2Vec(ei, embedding_dim=32, walk_length=10, context_size=5, walks_per_node=5,
                                num_negative_samples=1, p=0.5, q=2.0, sparse=True).to(DEV)
    assert isinstance(model, B200Node2Vec) and model.rowptr.is_cuda
    assert set(model.state_dict()) == {"embedding.weight"}
    edges = set(map(tuple, ei.t().tolist()))
    torch.manual_seed(1)
    pos, neg = model.sample(list(range(400)))
    assert pos.is_cuda and neg.is_cuda and pos.shape == (400 * 5 * 6, 5)
    pr = pos.cpu().numpy()
    for a, b in zip(pr[:, :-1].reshape(-1), pr[:, 1:].reshape(-1)):
        assert (int(a), int(b)) in edges or (a == b == 399), (a, b)
    mirror = Mirror(ei.to(DEV), embedding_dim=32, walk_length=10, context_size=5, walks_per_node=5, p=0.5, q=2.0)
    assert set(mirror.state_dict()) == {"embedding.weight"}
    torch.manual_seed(1)
    assert torch.equal(mirror.pos_sample(torch.arange(400, device=DEV)), pos)

    # examples/node2vec.py's loop: its loader asks for 4 workers; a CUDA model samples in the main process
    loader = model.loader(batch_size=32, shuffle=True, num_workers=4)
    assert loader.num_workers == 0
    opt = torch.optim.SparseAdam(list(model.parameters()), lr=0.05)
    losses = []
    for _ in range(20):
        total = 0.0
        for pos_rw, neg_rw in loader:
            opt.zero_grad()
            loss = model.loss(pos_rw.to(DEV), neg_rw.to(DEV))
            loss.backward()
            opt.step()
            total += loss.item()
        losses.append(total / len(loader))
    assert losses[-1] < 0.8 * losses[0], losses
    z = model().detach()
    perm = torch.from_numpy(np.random.default_rng(3).permutation(400))
    train, test = perm[:200], perm[200:]
    acc = model.test(z[train], y[train], z[test], y[test], max_iter=300)
    # four blocks of 100 nodes with 8 % edges inside a block and 0.2 % across: the embedding separates them
    assert acc > 0.9, acc
