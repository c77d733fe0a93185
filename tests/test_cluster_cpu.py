"""Clustering ops without a GPU: the numpy oracle (tests/cluster_oracle.py) against the expected values the reference's
own tests state and against the golden data the unmodified reference produced with it, properties of its matching,
the torch.ops.pyg binding of the plug-in (flags, operators, schemas, uninstall), and the argument errors of the
mirrors."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cluster_oracle as CO  # noqa: E402

from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.nn import pool  # noqa: E402


def _csr(n, row, col, w=None):
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    o = np.lexsort((col, row))
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))])
    return rowptr, col[o], (None if w is None else np.asarray(w)[o])


def _symmetric(n, k, seed):
    rng = np.random.default_rng(seed)
    row = np.repeat(np.arange(n), k)
    col = (row + rng.integers(1, n, n * k)) % n
    key = np.unique(np.concatenate([row * n + col, col * n + row]))
    return key // n, key % n


def _voxel(pos, size, batch=None, start=None, end=None):
    """voxel_grid's composition on the oracle: the batch index appended as a coordinate of voxel size 1."""
    pos = np.asarray(pos, np.float32)
    dim = pos.shape[1]
    batch = np.zeros(len(pos), np.int64) if batch is None else np.asarray(batch)
    rep = (lambda v: np.broadcast_to(np.asarray(v, np.float32), (dim, )))
    p = np.concatenate([pos, batch[:, None].astype(np.float32)], 1)
    st = None if start is None else np.concatenate([rep(start), [0]])
    en = None if end is None else np.concatenate([rep(end), [batch.max()]])
    return CO.grid_cluster(p, np.concatenate([rep(size), [1]]).astype(np.float32), st, en).tolist()


def check_matching(rowptr, col, cluster):
    """Pairs are mutually adjacent, clusters have at most two members, and each id is the minimum member."""
    n = rowptr.size - 1
    adj = {(u, int(v)) for u in range(n) for v in col[rowptr[u]:rowptr[u + 1]]}
    counts = np.bincount(cluster, minlength=n)
    assert counts.max() <= 2
    for u in range(n):
        c = cluster[u]
        assert c <= u
        if c != u:
            assert cluster[c] == c and (u, c) in adj and (c, u) in adj
    return counts


# ---------------------------------------------------------------------------------------------- the oracle
def test_oracle_reproduces_the_reference_tests_anchors(golden):
    z = golden("cluster")
    for seed in range(8):
        assert CO.graclus([0, 1, 2], [1, 0], None, seed)[0].tolist() == [0, 0]
    assert z["anchor_graclus"].tolist() == [0, 0]
    pos = [[0.0, 0.0], [11.0, 9.0], [2.0, 8.0], [2.0, 2.0], [8.0, 3.0]]
    batch = [0, 0, 0, 1, 1]
    got = [_voxel(pos, 5, batch), _voxel(pos, 5), _voxel(pos, 5, batch, -1, [18, 14]), _voxel(pos, 5, None, -1, [18, 14])]
    assert got == z["anchor_voxel_want"].tolist() == z["anchor_voxel"].tolist()
    diag = np.repeat(np.arange(5.0)[:, None], 2, 1)
    got = [_voxel(diag, 5, batch), _voxel(diag, 5)]
    assert got == z["anchor_single_want"].tolist() == z["anchor_single"].tolist()


def test_oracle_reproduces_the_golden_clusters(golden):
    z = golden("cluster")
    ei = z["gr_ei"]
    rowptr, col, w = _csr(60, ei[0], ei[1], z["gr_w"])
    torch.manual_seed(21)
    assert np.array_equal(CO.torch_ops()["graclus_cluster"](torch.from_numpy(rowptr), torch.from_numpy(col)),
                          z["gr_cluster"])
    torch.manual_seed(22)
    got = CO.torch_ops()["graclus_cluster"](torch.from_numpy(rowptr), torch.from_numpy(col), torch.from_numpy(w))
    assert np.array_equal(got, z["grw_cluster"])
    pos, batch = z["vg_pos"], z["vg_batch"]
    assert _voxel(pos, 0.7, batch) == z["vg_b"].tolist()
    assert _voxel(pos, 0.6, batch, -1.5, [3.2, 3.0, 3.5]) == z["vg_b_se"].tolist()


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matching_properties(weighted, seed):
    n = 300
    row, col = _symmetric(n, 3, seed)
    w = None
    if weighted:
        key = np.minimum(row, col) * n + np.maximum(row, col)
        w = np.random.default_rng(seed).random(n * n)[key]
    rowptr, col, w = _csr(n, row, col, w)
    cluster, rounds = CO.graclus(rowptr, col, w, seed)
    assert rounds < CO.MAX_ROUNDS
    counts = check_matching(rowptr, col, cluster)
    # no edge joins two singletons when the cap is not reached
    single = (counts[cluster] == 1)
    src = np.repeat(np.arange(n), np.diff(rowptr))
    assert not (single[src] & single[col]).any()


def test_oracle_weighted_choice_and_the_directed_three_cycle():
    # a star: the centre takes its heaviest neighbour whenever the colours allow it
    rowptr, col, w = _csr(4, [0, 0, 0, 1, 2, 3], [1, 2, 3, 0, 0, 0], [1.0, 3.0, 2.0, 1.0, 3.0, 2.0])
    for seed in range(16):
        c, _ = CO.graclus(rowptr, col, w, seed)
        assert c[0] == 0 and c.tolist().count(0) == 2
    cluster, rounds = CO.graclus([0, 1, 2, 3], [1, 2, 0], None, 3)
    assert rounds == CO.MAX_ROUNDS and cluster.tolist() == [0, 1, 2]
    # self-loops and NaN weights are never candidates: node 1's only other entry is NaN, so it stays alone
    cluster, _ = CO.graclus([0, 2, 4], [0, 1, 0, 1], [1.0, np.nan, np.nan, 1.0], 0)
    assert cluster.tolist() == [0, 1]


def test_oracle_grid_is_float32_one_operation_at_a_time():
    rng = np.random.default_rng(0)
    pos = rng.standard_normal((50, 3)).astype(np.float32)
    size = np.array([0.3, 0.7, 0.11], np.float32)
    got = CO.grid_cluster(pos, size)
    lo, hi = pos.min(0), pos.max(0)
    for i in range(50):
        c, stride = 0, 1
        for k in range(3):
            c += int(np.float32(np.float32(pos[i, k] - lo[k]) / size[k])) * stride
            stride *= int(np.float32(np.float32(hi[k] - lo[k]) / size[k])) + 1
        assert got[i] == c
    nan = pos.copy()
    nan[3, 1] = np.nan
    assert CO.grid_cluster(nan[:, 1:2], size[1:2])[3] == np.iinfo(np.int64).min


# ---------------------------------------------------------------------------------------------- the plug-in
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def test_install_defines_the_pyg_ops_and_flags_and_uninstall_restores(tg, plugin):
    import torch_geometric.typing as T
    flags = ("WITH_GRACLUS", "WITH_GRID_CLUSTER")
    assert not any(getattr(T, f) for f in flags)
    c = plugin.install(flip_flags=True)
    assert c["cluster_flags"] == 2 and c["cluster_ops"] in (0, 2) and c["point_ops"] in (0, 4)
    assert all(getattr(T, f) for f in flags)
    assert str(torch.ops.pyg.graclus_cluster.default._schema) == \
        "pyg::graclus_cluster(Tensor rowptr, Tensor col, Tensor? weight) -> Tensor"
    assert str(torch.ops.pyg.grid_cluster.default._schema) == \
        "pyg::grid_cluster(Tensor pos, Tensor size, Tensor? start, Tensor? end) -> Tensor"
    from pytorch_geometric_b200.plugin import shims
    m = shims.pyg_lib_module()
    assert callable(m.ops.graclus_cluster) and callable(m.ops.grid_cluster)
    plugin.uninstall()
    assert not any(getattr(T, f) for f in flags)
    with pytest.raises(ImportError, match="pyg-lib"):
        tg.nn.graclus(torch.tensor([[0, 1], [1, 0]]))
    with pytest.raises(ImportError, match="pyg-lib"):
        tg.nn.voxel_grid(torch.rand(4, 2), 0.5)
    c = plugin.install()
    assert "cluster_flags" not in c and not any(getattr(T, f) for f in flags)


def test_pyg_ops_have_no_cpu_implementation(tg, plugin):
    plugin.install(flip_flags=True)
    with pytest.raises(NotImplementedError):
        torch.ops.pyg.graclus_cluster(torch.tensor([0, 1, 2]), torch.tensor([1, 0]), None)
    with pytest.raises(NotImplementedError):
        torch.ops.pyg.grid_cluster(torch.rand(4, 2), torch.ones(2), None, None)


# ---------------------------------------------------------------------------------------------- argument errors
def test_mirrors_refuse_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        pool.graclus(torch.tensor([[0, 1], [1, 0]]))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.graclus(torch.tensor([0, 1, 2]), torch.tensor([1, 0]))
    with pytest.raises(RuntimeError, match="CUDA"):
        pool.voxel_grid(torch.rand(4, 2), 0.5)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.grid_cluster(torch.rand(4, 2), torch.ones(2))


def test_argument_and_dtype_errors(monkeypatch):
    monkeypatch.setattr(ops, "_cuda", lambda *ts: None)                  # reach the checks that precede any launch
    rowptr, col = torch.tensor([0, 1, 2]), torch.tensor([1, 0])
    with pytest.raises(TypeError, match="share a dtype"):
        ops.graclus(rowptr, col.int())
    with pytest.raises(TypeError, match="float32, bfloat16 or float64"):
        ops.graclus(rowptr, col, torch.ones(2, dtype=torch.float16))
    with pytest.raises(ValueError, match="one value per edge"):
        ops.graclus(rowptr, col, torch.ones(3))
    with pytest.raises(ValueError, match=r"\[N \+ 1\]"):
        ops.graclus(torch.tensor([], dtype=torch.long), col)
    for dt, limit in ((torch.float16, "2048"), (torch.bfloat16, "256")):
        with pytest.raises(TypeError, match=limit):
            ops.grid_cluster(torch.rand(4, 2).to(dt), torch.ones(2))
    with pytest.raises(TypeError, match="float32 or float64"):
        ops.grid_cluster(torch.ones(4, 2, dtype=torch.long), torch.ones(2))
    with pytest.raises(ValueError, match="one value per coordinate"):
        ops.grid_cluster(torch.rand(4, 2), torch.ones(3))
    with pytest.raises(ValueError, match="one value per coordinate"):
        ops.grid_cluster(torch.rand(4, 3), torch.ones(3), torch.zeros(2))
