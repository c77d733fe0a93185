"""Random walks without a GPU: the numpy oracle (tests/random_walk_oracle.py) against node2vec's analytic first- and
second-order transition probabilities (chi-square bounds on fixed seeds, so deterministic), with the default trial cap
and with the exact fallback alone; its vectorised form against its one-walk-at-a-time rule book with both neighbour
searches; the binding of the plug-in (torch.ops.pyg.random_walk, node2vec's flag, the dropout_path rebinds, the
global WITH_PYG_LIB left alone, uninstall); B200Node2Vec's state_dict; and the argument errors of ops.random_walk."""
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch
from scipy.stats import chi2

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random_walk_oracle as RO  # noqa: E402

from pytorch_geometric_b200 import ops  # noqa: E402


def _csr(n, row, col):
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    o = np.lexsort((col, row))
    return np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))]), col[o]


def _small_graph():
    """Undirected: a triangle 0-1-2, a path 2-3-4, a square 4-5-6-7 with the chord 5-7, node 8 hanging off 6, plus a
    self-loop at 3 and a duplicate of edge 0-1."""
    und = [(0, 1), (1, 2), (0, 2), (2, 3), (3, 4), (4, 5), (5, 6), (6, 7), (7, 4), (5, 7), (6, 8), (0, 1)]
    row = [a for a, b in und] + [b for a, b in und] + [3]
    col = [b for a, b in und] + [a for a, b in und] + [3]
    return _csr(9, row, col)


def _chi2_ok(counts, probs, what):
    """Pearson's statistic over every context (sum of (O - E)^2 / E) below the 0.9999 quantile of its degrees of
    freedom; contexts with fewer than 50 samples are skipped."""
    stat, dof = 0.0, 0
    for ctx, cnt in counts.items():
        total = sum(cnt.values())
        if total < 50:
            continue
        pr = probs(ctx)
        assert set(cnt) <= set(pr), (what, ctx, cnt, pr)
        for x, px in pr.items():
            e = total * px
            stat += (cnt.get(x, 0) - e) ** 2 / e
        dof += len(pr) - 1
    assert dof > 0
    assert stat < chi2.ppf(0.9999, dof), f"{what}: chi2 {stat:.1f} with {dof} dof"


def _transition_probs(rowptr, col, p, q):
    rows = {v: [int(c) for c in col[rowptr[v]:rowptr[v + 1]]] for v in range(rowptr.size - 1)}

    def first(v):
        out = Counter(rows[v])
        return {x: c / len(rows[v]) for x, c in out.items()}

    def second(ctx):
        t, v = ctx
        w = Counter()
        for x in rows[v]:                                              # one weight per CSR entry (duplicates count)
            w[x] += 1 / p if x == t else (1.0 if x in rows[t] else 1 / q)
        total = sum(w.values())
        return {x: wx / total for x, wx in w.items()}
    return first, second


@pytest.mark.parametrize("p,q", [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25)])
@pytest.mark.parametrize("max_trials", [RO.MAX_TRIALS, 0])
def test_oracle_transitions_follow_node2vec(p, q, max_trials):
    rowptr, col = _small_graph()
    start = np.tile(np.arange(9), 3000)
    walks = RO.random_walk(rowptr, col, start, 3, p, q, seed=12345, max_trials=max_trials)
    first, second = _transition_probs(rowptr, col, p, q)
    c1 = {}
    for v, x in zip(walks[:, 0], walks[:, 1]):
        c1.setdefault(int(v), Counter())[int(x)] += 1
    _chi2_ok(c1, first, f"first order p={p} q={q}")
    c2 = {}
    for k in (2, 3):
        for t, v, x in zip(walks[:, k - 2], walks[:, k - 1], walks[:, k]):
            c2.setdefault((int(t), int(v)), Counter())[int(x)] += 1
    _chi2_ok(c2, second if (p, q) != (1.0, 1.0) else (lambda ctx: first(ctx[1])), f"second order p={p} q={q}")


@pytest.mark.parametrize("p,q", [(0.25, 4.0), (4.0, 0.25), (1e-3, 1e3)])
def test_the_exact_fallback_and_the_trials_agree_on_the_distribution(p, q):
    """With max_trials = 0 every node2vec step is the exact draw; with the default cap nearly every step is a trial.
    Both histograms of the second-order transitions out of one context match each other and node2vec's weights."""
    rowptr, col = _small_graph()
    first, second = _transition_probs(rowptr, col, p, q)
    hist = []
    for mt in (0, RO.MAX_TRIALS):
        walks = RO.random_walk(rowptr, col, np.full(40000, 4), 2, p, q, seed=7, max_trials=mt)
        sel = walks[:, 1] == 5                                        # context (t, v) = (4, 5)
        hist.append(Counter(walks[sel, 2].tolist()))
    pr = second((4, 5))
    for h in hist:
        _chi2_ok({(4, 5): h}, lambda ctx: pr, f"p={p} q={q}")
    # the two samples against each other: a two-sample chi-square on the pooled counts
    keys = sorted(set(hist[0]) | set(hist[1]))
    table = np.array([[h.get(k, 0) for k in keys] for h in hist], float)
    exp = table.sum(1, keepdims=True) * table.sum(0, keepdims=True) / table.sum()
    ok = exp > 0
    stat = ((table - exp)[ok] ** 2 / exp[ok]).sum()
    assert stat < chi2.ppf(0.9999, max(len(keys) - 1, 1)), stat


def test_the_vectorised_oracle_is_the_rule_book():
    """Random small graphs, sorted and unsorted rows, self-loops, duplicates, dead ends, stray column values and
    out-of-range starts: the vectorised oracle equals the one-walk-at-a-time rule book, whose neighbour test is the
    binary search or the linear scan the row order selects."""
    rng = np.random.default_rng(0)
    seen_unsorted = seen_sorted = False
    for trial in range(24):
        n = int(rng.integers(1, 30))
        E = int(rng.integers(0, 120))
        row, col = rng.integers(0, n, E), rng.integers(0, n, E)
        o = np.argsort(row, kind="stable") if trial % 2 else np.lexsort((col, row))
        row, col = row[o], col[o]
        if trial % 5 == 0 and E:
            col[rng.integers(0, E)] = n + 2
        rowptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))])
        srt = RO.rows_sorted(rowptr, col)
        seen_sorted |= srt
        seen_unsorted |= not srt
        start = rng.integers(-1, n + 1, 20)
        for p, q in ((1.0, 1.0), (0.25, 4.0), (1e-3, 1e3)):
            for mt in (0, 1, RO.MAX_TRIALS):
                a = RO.random_walk(rowptr, col, start, 6, p, q, trial, mt)
                b = RO.random_walk_scalar(rowptr, col, start, 6, p, q, trial, mt)
                assert np.array_equal(a, b), (trial, p, q, mt)
    assert seen_sorted and seen_unsorted


def test_oracle_rng_and_rules_by_hand():
    # splitmix64's published first output for state 0 (the finaliser of 0 + golden ratio)
    assert int(RO.splitmix64(np.uint64(0), np.uint64(1))) == 0xE220A8397B1DCDAF
    assert int(RO.umulhi(np.uint64(2**63), np.uint64(6))) == 3
    assert RO.probabilities(0.25, 4.0) == (4.0, 0.25, 1.0, 0.25, 0.0625)
    # a dead end keeps the walk in place; a start outside [0, N) gives -1
    w = RO.random_walk([0, 1, 1], [1], [0, 1, 2, -1], 3, 0.5, 2.0, seed=1)
    assert w.tolist() == [[0, 1, 1, 1], [1, 1, 1, 1], [-1] * 4, [-1] * 4]
    assert RO.rows_sorted([0, 2, 4], [0, 1, 0, 1]) and not RO.rows_sorted([0, 2, 4], [1, 0, 0, 1])   # per row


# ---------------------------------------------------------------------------------------------- the plug-in
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def test_install_binds_the_walk_op_and_flags_and_uninstall_restores(tg, plugin):
    import torch_geometric.nn.models.node2vec as n2v
    import torch_geometric.typing as T
    import torch_geometric.utils as tgu
    import torch_geometric.utils.dropout as tgd
    orig = (tgu.dropout_path, tgd.dropout_path, n2v.WITH_PYG_LIB, tg.nn.Node2Vec, tg.nn.models.Node2Vec)
    assert T.WITH_PYG_LIB is False and n2v.WITH_PYG_LIB is False
    c = plugin.install(layers=True, flip_flags=True)
    assert c["walk_ops"] in (0, 1) and c["walk_flags"] >= 3 and c["models"] == 2
    assert T.WITH_PYG_LIB is False                                     # NeighborLoader keeps its pyg-lib-free path
    assert n2v.WITH_PYG_LIB is True
    assert tgu.dropout_path is not orig[0] and tgu.dropout_path.__wrapped__ is orig[0] and tgd.dropout_path is tgu.dropout_path
    from pytorch_geometric_b200.plugin.models import B200Node2Vec
    assert tg.nn.Node2Vec is B200Node2Vec and tg.nn.models.Node2Vec is B200Node2Vec
    assert str(torch.ops.pyg.random_walk.default._schema) == \
        "pyg::random_walk(Tensor rowptr, Tensor col, Tensor seed, int walk_length, float p=1., float q=1.) -> Tensor"
    from pytorch_geometric_b200.plugin import shims
    assert callable(shims.pyg_lib_module().ops.random_walk)
    # CPU input: the reference's own ImportError, with the global flag still off
    with pytest.raises(ImportError, match="pyg-lib"):
        tgu.dropout_path(torch.tensor([[0, 1], [1, 0]]))
    assert tgu.dropout_path(torch.tensor([[0, 1], [1, 0]]), p=0.0)[1].all()
    with pytest.raises(NotImplementedError):
        torch.ops.pyg.random_walk(torch.tensor([0, 1, 2]), torch.tensor([1, 0]), torch.tensor([0]), 3)
    plugin.uninstall()
    now = (tgu.dropout_path, tgd.dropout_path, n2v.WITH_PYG_LIB, tg.nn.Node2Vec, tg.nn.models.Node2Vec)
    assert all(a is b for a, b in zip(orig, now))
    with pytest.raises(ImportError, match="pyg-lib"):
        tg.nn.Node2Vec(torch.tensor([[0, 1], [1, 0]]), 8, 4, 2)
    c = plugin.install()
    assert "walk_flags" not in c and "models" not in c and n2v.WITH_PYG_LIB is False


def test_b200_node2vec_keeps_the_reference_state_dict(tg, plugin):
    from pytorch_geometric_b200.plugin.models import B200Node2Vec
    ei = torch.tensor([[0, 1, 1, 2, 2, 3], [1, 0, 2, 1, 3, 2]])
    torch.manual_seed(0)
    ref = tg.nn.models.node2vec.Node2Vec.__new__(tg.nn.models.node2vec.Node2Vec)
    import torch_geometric.nn.models.node2vec as n2v
    n2v.WITH_PYG_LIB, had = True, n2v.WITH_PYG_LIB
    try:
        from pytorch_geometric_b200.plugin import shims
        shims.register_walk_ops()
        ref.__init__(ei, 16, 5, 3, walks_per_node=2, p=0.5, q=2.0)
    finally:
        n2v.WITH_PYG_LIB = had
    torch.manual_seed(0)
    ours = B200Node2Vec(ei, 16, 5, 3, walks_per_node=2, p=0.5, q=2.0)
    assert n2v.WITH_PYG_LIB is had
    assert list(ours.state_dict()) == list(ref.state_dict()) == ["embedding.weight"]
    assert torch.equal(ours.state_dict()["embedding.weight"], ref.state_dict()["embedding.weight"])
    assert torch.equal(ours.rowptr, ref.rowptr) and torch.equal(ours.col, ref.col)
    assert dict(ours.named_buffers()).keys() == {"rowptr", "col"}
    ours.load_state_dict(ref.state_dict())
    loader = ours.loader(batch_size=2, num_workers=2)                 # a CPU model keeps the reference's workers
    assert loader.num_workers == 2


# ---------------------------------------------------------------------------------------------- argument errors
def test_random_walk_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.random_walk(torch.tensor([0, 1, 2]), torch.tensor([1, 0]), torch.tensor([0]), 3)


def test_random_walk_argument_errors(monkeypatch):
    monkeypatch.setattr(ops, "_cuda", lambda *ts: None)                  # reach the checks that precede any launch
    rowptr, col, start = torch.tensor([0, 1, 2]), torch.tensor([1, 0]), torch.tensor([0, 1])
    with pytest.raises(TypeError, match="share a dtype"):
        ops.random_walk(rowptr, col, start.int(), 3)
    with pytest.raises(ValueError, match="walk_length"):
        ops.random_walk(rowptr, col, start, -1)
    for p, q in ((0.0, 1.0), (1.0, -2.0), (float("nan"), 1.0), (1.0, float("inf"))):
        with pytest.raises(ValueError, match="finite"):
            ops.random_walk(rowptr, col, start, 3, p, q)
    with pytest.raises(ValueError, match="max_trials"):
        ops.random_walk(rowptr, col, start, 3, 0.5, 2.0, max_trials=-1)
    with pytest.raises(ValueError, match=r"\[N \+ 1\]"):
        ops.random_walk(torch.tensor([], dtype=torch.long), col, start, 3)
