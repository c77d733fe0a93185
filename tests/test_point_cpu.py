"""Point-cloud ops without a GPU: the float32 oracle (tests/point_oracle.py) against the expected values the
reference's own tests state and against the golden data the unmodified reference produced with it, the torch.ops.pyg
binding of the plug-in (flags, operators, counts, uninstall), and the argument errors of the nn.pool mirrors."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import point_oracle as PO  # noqa: E402

from pytorch_geometric_b200.nn import pool  # noqa: E402

SIX = np.array([[0.0, 0.0], [1.0, 0.0], [2.0, 0.0], [0.0, 1.0], [-2.0, 0.0], [0.0, -2.0]], dtype=np.float32)


# ---------------------------------------------------------------------------------------------- the oracle
def test_oracle_knn_graph_of_the_six_point_set(golden):
    """KNNGraph(k=2, force_undirected=True): k + 1 neighbours, drop self, flip, make undirected, coalesce."""
    z = golden("point")
    e = PO.knn(SIX, SIX, 3)
    e = e[:, e[0] != e[1]][::-1]
    e = np.concatenate([e, e[::-1]], axis=1)
    e = np.unique(e[0] * 6 + e[1])
    assert np.array_equal(np.stack([e // 6, e % 6]), z["knngraph_six_want"])
    assert np.array_equal(z["knngraph_six"], z["knngraph_six_want"])


def test_oracle_radius_graph_of_the_six_point_set(golden):
    z = golden("point")
    e = PO.radius(SIX, SIX, 1.5, ignore_same_index=True)[::-1]
    o = np.lexsort((e[1], e[0]))
    assert np.array_equal(e[:, o], z["radiusgraph_six_want"])


def test_oracle_knn_interpolate_anchor(golden):
    z = golden("point")
    xi = np.array([[1.0], [10.0], [100.0], [-1.0], [-10.0], [-100.0]], dtype=np.float32)
    px = np.array([[-1, 0], [0, 0], [1, 0], [-2, 0], [0, 0], [2, 0]], dtype=np.float32)
    py = np.array([[-1, -1], [1, 1], [-2, -2], [2, 2]], dtype=np.float32)
    yi, xj = PO.knn(px, py, 2, [0, 3, 6], [0, 2, 4])
    w = 1.0 / np.maximum(((px[xj] - py[yi]) ** 2).sum(-1, keepdims=True), 1e-16)
    num, den = np.zeros((4, 1)), np.zeros((4, 1))
    np.add.at(num, yi, xi[xj] * w)
    np.add.at(den, yi, w)
    assert (num / den).tolist() == z["interp_anchor_want"].tolist() == z["interp_anchor_out"].tolist()


def test_oracle_nearest_anchor(golden):
    z = golden("point")
    assert PO.nearest(z["nearest_x"], z["nearest_y"], [0, 4], [0, 2]).tolist() == z["nearest_want"].tolist()
    assert z["nearest_out"].tolist() == [0, 0, 1, 1]
    with pytest.raises(ValueError):
        PO.nearest(z["nearest_x"], z["nearest_y"], [0, 2, 4], [0, 2, 2])


def test_oracle_reproduces_the_golden_graphs(golden):
    z = golden("point")
    idx = PO.fps(z["sa_pos"], [0, 32, 64], 0.5)
    assert np.array_equal(idx, z["sa_idx"])
    row, col = PO.radius(z["sa_pos"], z["sa_pos"][idx], 0.4, [0, 32, 64], [0, 16, 32], 16)
    assert np.array_equal(row, z["sa_row"]) and np.array_equal(col, z["sa_col"])
    e = PO.knn(z["cloud"], z["cloud"], 7)
    e = e[:, e[0] != e[1]][::-1]
    assert np.array_equal(e, z["knngraph_cloud"])


def test_oracle_distances_are_float32_one_operation_at_a_time():
    rng = np.random.default_rng(0)
    x, y = rng.standard_normal((7, 5)).astype(np.float32), rng.standard_normal((3, 5)).astype(np.float32)
    d = PO.distances(x, y)
    for i in range(3):
        for j in range(7):
            acc = np.float32(0)
            for f in range(5):
                t = np.float32(x[j, f] - y[i, f])
                acc = np.float32(acc + np.float32(t * t))
            assert d[i, j] == acc
    c = PO.distances(np.zeros((1, 3), np.float32), y, cosine=True)
    assert np.isnan(c).all() and PO.knn(np.zeros((1, 3), np.float32), y, 1, cosine=True).shape == (2, 0)


def test_oracle_ties_go_to_the_lower_index_and_fps_uses_ceil():
    x = np.array([[1.0], [-1.0], [1.0], [0.0]], dtype=np.float32)
    assert PO.knn(x, np.zeros((1, 1), np.float32), 3).tolist() == [[0, 0, 0], [3, 0, 1]]
    assert PO.fps_counts([0, 3, 3, 10], 10, 0.5) == [2, 0, 4]
    # duplicates: once every running min-distance is 0, the argmax is the lowest index again
    assert PO.fps(np.array([[0.0], [0.0], [1.0]], np.float32), None, 1.0).tolist() == [0, 2, 0]


# ---------------------------------------------------------------------------------------------- the plug-in
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def test_install_defines_the_pyg_ops_and_flags_and_uninstall_restores(tg, plugin):
    import torch_geometric.typing as T
    flags = ("WITH_KNN", "WITH_RADIUS", "WITH_FPS", "WITH_NEAREST")
    assert not any(getattr(T, f) for f in flags)
    c = plugin.install(flip_flags=True)
    assert c["flags"] == 5 and c["point_flags"] == 4 and c["point_ops"] in (0, 4)
    assert all(getattr(T, f) for f in flags)
    for name in ("knn", "radius", "fps", "nearest"):
        assert hasattr(torch.ops.pyg, name)
    from pytorch_geometric_b200.plugin import shims
    m = shims.pyg_lib_module()
    assert all(callable(getattr(m.ops, n)) for n in ("knn", "radius", "fps", "nearest"))
    assert str(torch.ops.pyg.knn.default._schema).startswith("pyg::knn(Tensor x, Tensor y, Tensor? ptr_x")
    mlp = torch.nn.Linear(4, 4)
    tg.nn.DynamicEdgeConv(mlp, k=3)                                       # the constructors no longer raise
    tg.nn.GravNetConv(4, 4, 2, 2, k=3)
    tg.nn.XConv(2, 4, dim=3, kernel_size=3, hidden_channels=2)
    plugin.uninstall()
    assert not any(getattr(T, f) for f in flags)
    for ctor in (lambda: tg.nn.DynamicEdgeConv(mlp, k=3), lambda: tg.nn.GravNetConv(4, 4, 2, 2, k=3),
                 lambda: tg.nn.XConv(2, 4, dim=3, kernel_size=3, hidden_channels=2)):
        with pytest.raises(ImportError, match="pyg-lib"):
            ctor()
    with pytest.raises(ImportError, match="pyg-lib"):
        tg.nn.knn_graph(torch.rand(4, 2), 2)
    c = plugin.install()
    assert "point_flags" not in c and not any(getattr(T, f) for f in flags)


def test_pyg_ops_have_no_cpu_implementation(tg, plugin):
    plugin.install(flip_flags=True)
    with pytest.raises(NotImplementedError):
        torch.ops.pyg.knn(torch.rand(4, 2), torch.rand(4, 2), None, None, 2, False, 1)


# ---------------------------------------------------------------------------------------------- argument errors
def test_mirrors_refuse_cpu_and_unsupported_dtypes():
    for dt in (torch.float32, torch.float64, torch.float16):
        x = torch.rand(6, 3, dtype=dt)
        with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
            pool.knn(x, x, 2)
        with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
            pool.radius_graph(x, 0.5)
        with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
            pool.fps(x)
        with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
            pool.nearest(x, x)


def test_mirrors_refuse_k_above_the_limit_and_ratio_outside_the_unit_interval(monkeypatch):
    from pytorch_geometric_b200 import ops
    monkeypatch.setattr(ops, "_point_values", lambda *ts: None)          # reach the checks that precede any launch
    x = torch.rand(6, 3)
    with pytest.raises(ValueError, match="k <= 128"):
        pool.knn(x, x, 129)
    with pytest.raises(ValueError, match="k <= 128"):
        pool.knn_graph(x, 128)                                            # k + 1 neighbours are asked for
    for ratio in (0.0, -0.5, 1.5):
        with pytest.raises(ValueError, match=r"\(0, 1\]"):
            pool.fps(x, ratio=ratio)
