"""Point-cloud ops on the GPU (csrc/point.cu): knn, radius, fps and nearest equal the float32 oracle of
tests/point_oracle.py bit for bit -- on integer grids full of exact ties, on random fp32 / bf16 coordinates, with empty
examples, examples smaller than k, bipartite inputs with ptrs of different lengths or None, cosine with zero vectors,
non-contiguous inputs and int32 ptrs -- give identical output on two runs, handle a 200k-point cloud, and the
unmodified reference layers reproduce tests/golden/point.npz after plugin.install(flip_flags=True)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import point_oracle as PO  # noqa: E402

from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.nn import pool  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _np(t):
    return None if t is None else t.detach().float().cpu().numpy()


def _ptr(sizes, dtype=torch.int64):
    return torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=dtype, device=DEV)


def _points(n, f, kind, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "grid":
        x = torch.randint(-3, 4, (n, f), generator=g).float()
    else:
        x = torch.randn(n, f, generator=g)
    return x.to(dtype).to(DEV)


def _eq(a, b, what=""):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    assert a.dtype == np.int64, what
    assert a.shape == np.asarray(b).shape and np.array_equal(a, b), f"{what}: {a.tolist()[:3]} vs {np.asarray(b).tolist()[:3]}"


SIZES_X = [0, 7, 150, 3, 41]
SIZES_Y = [5, 9, 60, 0, 33]


# ---------------------------------------------------------------------------------------------- knn
@pytest.mark.parametrize("f", [1, 3, 64, 130])
@pytest.mark.parametrize("k", [1, 20, 32, 33, 128])
@pytest.mark.parametrize("kind,dtype", [("grid", torch.float32), ("randn", torch.float32), ("randn", torch.bfloat16)])
def test_knn_equals_the_oracle(f, k, kind, dtype):
    x = _points(sum(SIZES_X), f, kind, dtype, 1)
    y = _points(sum(SIZES_Y), f, kind, dtype, 2)
    px, py = _ptr(SIZES_X), _ptr(SIZES_Y)
    out = ops.knn(x, y, k, px, py)
    _eq(out, PO.knn(_np(x), _np(y), k, _np(px), _np(py)), "knn")


@pytest.mark.parametrize("k", [4, 40])
def test_knn_bipartite_ptrs_of_different_lengths_and_none(k):
    x, y = _points(60, 3, "grid", torch.float32, 3), _points(50, 3, "grid", torch.float32, 4)
    px, py = _ptr([20, 40]), _ptr([10, 10, 30])                 # y's third example has no x points
    _eq(ops.knn(x, y, k, px, py), PO.knn(_np(x), _np(y), k, _np(px), _np(py)), "longer ptr_y")
    px2 = _ptr([25, 25, 10])
    _eq(ops.knn(x, y, k, px2, _ptr([50])), PO.knn(_np(x), _np(y), k, _np(px2), [0, 50]), "longer ptr_x")
    _eq(ops.knn(x, y, k, None, None), PO.knn(_np(x), _np(y), k), "no ptr")
    _eq(ops.knn(x, y, k, None, py), PO.knn(_np(x), _np(y), k, None, _np(py)), "ptr_x None")


@pytest.mark.parametrize("f", [3, 64])
@pytest.mark.parametrize("k", [5, 40])
def test_knn_cosine_with_zero_vectors(f, k):
    x, y = _points(120, f, "grid", torch.float32, 5), _points(70, f, "randn", torch.float32, 6)
    x[::7] = 0
    y[::5] = 0
    px, py = _ptr([60, 60]), _ptr([30, 40])
    _eq(ops.knn(x, y, k, px, py, cosine=True), PO.knn(_np(x), _np(y), k, _np(px), _np(py), cosine=True), "cosine")


def test_knn_non_finite_coordinates_are_never_selected():
    x, y = _points(40, 3, "randn", torch.float32, 7), _points(10, 3, "randn", torch.float32, 8)
    x[3, 1], x[9, 0], y[2, 2] = float("nan"), float("inf"), float("nan")
    _eq(ops.knn(x, y, 8), PO.knn(_np(x), _np(y), 8), "non-finite")


def test_knn_non_contiguous_inputs_and_int32_ptr():
    base = _points(300, 8, "grid", torch.float32, 9)
    x, y = base[::2, ::2], base[1::3, 1::2]                       # [150, 4] and [100, 4], both strided
    px, py = _ptr([50, 100], torch.int32), _ptr([40, 60], torch.int32)
    _eq(ops.knn(x, y, 12, px, py), PO.knn(_np(x), _np(y), 12, _np(px), _np(py)), "strided")
    _eq(ops.radius(x, y, 2.5, px, py, 7), PO.radius(_np(x), _np(y), 2.5, _np(px), _np(py), 7), "strided radius")


def test_knn_graph_mirror_is_the_reference_composition():
    x = _points(90, 3, "grid", torch.float32, 10)
    batch = torch.arange(3, device=DEV).repeat_interleave(30)
    e = pool.knn_graph(x, 6, batch)
    ref = PO.knn(_np(x), _np(x), 7, [0, 30, 60, 90], [0, 30, 60, 90])
    ref = ref[:, ref[0] != ref[1]][::-1]
    _eq(e, ref, "knn_graph")
    _eq(pool.knn_graph(x, 6, batch, loop=True, flow="target_to_source"),
        PO.knn(_np(x), _np(x), 6, [0, 30, 60, 90], [0, 30, 60, 90]), "knn_graph loop")


def test_requires_grad_inputs_give_integer_outputs():
    x = _points(40, 3, "randn", torch.float32, 11).requires_grad_()
    for e in (pool.knn(x, x, 4), pool.radius_graph(x, 1.0), pool.fps(x), pool.nearest(x, x[:5].detach())):
        assert e.dtype == torch.int64 and not e.requires_grad


# ---------------------------------------------------------------------------------------------- radius
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("f", [1, 3, 64, 130])
def test_radius_equals_the_oracle(dtype, f):
    x = _points(sum(SIZES_X), f, "randn", dtype, 12)
    y = _points(sum(SIZES_Y), f, "randn", dtype, 13)
    px, py = _ptr(SIZES_X), _ptr(SIZES_Y)
    r = float(np.sqrt(2.0 * f))                                    # about half the pairs
    for cap in (1, 32, 1000):
        _eq(ops.radius(x, y, r, px, py, cap), PO.radius(_np(x), _np(y), r, _np(px), _np(py), cap), f"cap {cap}")


@pytest.mark.parametrize("r", [1.0, 2.0 ** 0.5, 2.0, 1.0 + 1e-7])
def test_radius_at_the_boundary_on_a_grid(r):
    """Grid distances are exact integers: d == r^2 is excluded (strict <), and r^2 is formed in fp64 and rounded once."""
    x = _points(200, 2, "grid", torch.float32, 14)
    for same in (False, True):
        for cap in (3, 64):
            _eq(ops.radius(x, x, r, None, None, cap, same), PO.radius(_np(x), _np(x), r, None, None, cap, same),
                f"r {r} cap {cap} ignore_same {same}")
    batch = torch.arange(4, device=DEV).repeat_interleave(50)
    e = pool.radius_graph(x, r, batch, max_num_neighbors=10)
    ref = PO.radius(_np(x), _np(x), r, [0, 50, 100, 150, 200], [0, 50, 100, 150, 200], 10, True)[::-1]
    _eq(e, ref, "radius_graph")


# ---------------------------------------------------------------------------------------------- fps
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("f", [1, 3, 64])
@pytest.mark.parametrize("ratio", [0.25, 0.5, 1.0])
def test_fps_equals_the_oracle(dtype, f, ratio):
    sizes = [0, 1, 17, 300, 64, 0, 5]
    src = _points(sum(sizes), f, "randn", dtype, 15)
    ptr = _ptr(sizes)
    _eq(ops.fps(src, ptr, ratio, False), PO.fps(_np(src), _np(ptr), ratio), "fps")


def test_fps_duplicate_points_grid_ties_and_int32_ptr():
    src = _points(180, 3, "grid", torch.float32, 16)
    src[50:60] = src[40]
    ptr = _ptr([90, 90], torch.int32)
    for ratio in (0.3, 1.0):
        _eq(ops.fps(src, ptr, ratio, False), PO.fps(_np(src), _np(ptr), ratio), f"ratio {ratio}")
    _eq(ops.fps(src, None, 0.5, False), PO.fps(_np(src), None, 0.5), "no ptr")


def test_fps_large_example_streams_from_global_memory():
    src = _points(30000, 3, "randn", torch.float32, 17)            # 30000 * 4 floats exceed the shared-memory budget
    ptr = _ptr([30000])
    _eq(ops.fps(src, ptr, 0.01, False), PO.fps(_np(src), _np(ptr), 0.01), "streamed")


def test_fps_random_start():
    sizes = [40, 0, 25, 70]
    src = _points(sum(sizes), 3, "randn", torch.float32, 18)
    ptr = _ptr(sizes)
    torch.manual_seed(0)
    out = ops.fps(src, ptr, 0.5, True).cpu().numpy()
    counts = PO.fps_counts(_np(ptr), sum(sizes), 0.5)
    offs = np.concatenate([[0], np.cumsum(counts)])
    p = _np(ptr).astype(np.int64)
    starts = []
    for b in range(len(sizes)):
        if counts[b]:
            first = out[offs[b]]
            assert p[b] <= first < p[b + 1]
            starts.append(first - p[b])
        else:
            starts.append(0)
    assert np.array_equal(out, PO.fps(_np(src), _np(ptr), 0.5, starts))
    torch.manual_seed(0)
    assert np.array_equal(ops.fps(src, ptr, 0.5, True).cpu().numpy(), out)   # the draw follows torch's generator


# ---------------------------------------------------------------------------------------------- nearest
@pytest.mark.parametrize("kind,dtype", [("grid", torch.float32), ("randn", torch.float32), ("randn", torch.bfloat16)])
def test_nearest_equals_the_oracle(kind, dtype):
    x, y = _points(300, 3, kind, dtype, 19), _points(40, 3, kind, dtype, 20)
    bx, by = torch.arange(3, device=DEV).repeat_interleave(100), torch.arange(3, device=DEV).repeat_interleave(torch.tensor([10, 20, 10], device=DEV))
    out = pool.nearest(x, y, bx, by)
    _eq(out, PO.nearest(_np(x), _np(y), [0, 100, 200, 300], [0, 10, 30, 40]), "nearest")
    with pytest.raises(ValueError, match="no y point"):
        ops.nearest(x, y, _ptr([100, 100, 100]), _ptr([20, 20, 0]))


# ---------------------------------------------------------------------------------------------- determinism, scale
def test_every_op_is_deterministic():
    x, y = _points(3000, 16, "randn", torch.float32, 21), _points(2000, 16, "randn", torch.float32, 22)
    px, py = _ptr([1000, 2000]), _ptr([500, 1500])
    runs = [(ops.knn(x, y, 20, px, py), ops.knn(x, y, 50, px, py, cosine=True), ops.radius(x, y, 5.0, px, py, 40),
             ops.fps(x, px, 0.3, False), ops.nearest(y, x, py, px)) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_a_200k_point_cloud_on_sampled_queries():
    n = 200_000
    x = torch.rand(n, 3, device=DEV)
    e = ops.knn(x, x, 16)
    assert e.shape == (2, n * 16)
    q = np.random.default_rng(0).choice(n, 48, replace=False)
    xn = _np(x)
    ref = PO.knn(xn, xn[q], 16)
    got = e[1].view(n, 16)[torch.as_tensor(q, device=DEV)].cpu().numpy().ravel()
    assert np.array_equal(got, ref[1])
    r = ops.radius(x, x, 0.03, None, None, 64)
    rows = r[0].cpu().numpy()
    for i in q[:16]:
        want = PO.radius(xn, xn[i:i + 1], 0.03, None, None, 64)[1]
        assert np.array_equal(r[1].cpu().numpy()[rows == i], want)


# ---------------------------------------------------------------------------------------------- the reference layers
@pytest.fixture
def tg_point(tg):
    from pytorch_geometric_b200 import plugin
    plugin.install(flip_flags=True)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                        # XConv's Conv1d: compare in plain fp32
    yield tg
    torch.backends.cudnn.allow_tf32 = prev
    plugin.uninstall()


def _close(a, b, tol, what):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    assert a.shape == b.shape, what
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= tol * max(scale, 1e-3), f"{what}: max err {err:.3e} vs scale {scale:.3e}"


def _t(z, key, grad=False):
    t = torch.from_numpy(z[key]).to(DEV)
    return t.requires_grad_() if grad else t


def _load(module, z, tag):
    module.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
    return module.to(DEV)


def _mlp(*ch):
    layers = []
    for a, b in zip(ch[:-1], ch[1:]):
        layers += [torch.nn.Linear(a, b), torch.nn.ReLU()]
    return torch.nn.Sequential(*layers[:-1])


def _check_step(z, tag, module, out, grads, grad_tol=1e-5):
    out.backward(_t(z, f"{tag}_gout"))
    _close(out, z[f"{tag}_out"], 1e-5, f"{tag} out")
    for name, t in grads:
        _close(t.grad, z[f"{tag}_g{name}"], grad_tol, f"{tag} grad {name}")
    for name, p in module.named_parameters():
        want = z[f"{tag}_g_{name}"]
        if np.abs(want).max() < 1e-5:
            # zero in exact arithmetic (GravNetConv's distances do not move with lin_s's bias): rounding noise only
            assert p.grad.abs().max().item() < 1e-5, f"{tag} grad {name}"
        else:
            _close(p.grad, want, grad_tol, f"{tag} grad {name}")


def test_dynamic_edge_conv_matches_golden(tg_point, golden):
    z = golden("point")
    conv = _load(tg_point.nn.DynamicEdgeConv(_mlp(10, 16, 8), k=6, aggr="max"), z, "dec")
    x = _t(z, "dec_x", True)
    _check_step(z, "dec", conv, conv(x, _t(z, "dec_batch")), [("x", x)])
    conv = _load(tg_point.nn.DynamicEdgeConv(_mlp(10, 16, 8), k=5, aggr="add"), z, "decb")
    xl, xr = _t(z, "decb_xl", True), _t(z, "decb_xr", True)
    _check_step(z, "decb", conv, conv((xl, xr), (_t(z, "decb_bl"), _t(z, "decb_br"))), [("xl", xl), ("xr", xr)])


def test_gravnet_conv_matches_golden(tg_point, golden):
    z = golden("point")
    conv = _load(tg_point.nn.GravNetConv(6, 8, space_dimensions=3, propagate_dimensions=4, k=4), z, "grav")
    x = _t(z, "grav_x", True)
    _check_step(z, "grav", conv, conv(x, _t(z, "grav_batch")), [("x", x)])


def test_xconv_matches_golden(tg_point, golden):
    z = golden("point")
    conv = _load(tg_point.nn.XConv(4, 8, dim=3, kernel_size=4, hidden_channels=6, dilation=2), z, "xconv")
    x = _t(z, "xconv_x", True)
    # the gradients pass through train-mode BatchNorms, whose backward subtracts batch means: the CPU's and the
    # GPU's reduction orders leave about 2e-5 of the largest gradient
    _check_step(z, "xconv", conv, conv(x, _t(z, "xconv_pos"), _t(z, "xconv_batch")), [("x", x)], grad_tol=1e-4)


def test_knn_interpolate_and_nearest_match_golden(tg_point, golden):
    z = golden("point")
    from torch_geometric.nn import knn_interpolate, nearest
    xi = torch.tensor([[1.0], [10.0], [100.0], [-1.0], [-10.0], [-100.0]], device=DEV)
    px = torch.tensor([[-1.0, 0.0], [0.0, 0.0], [1.0, 0.0], [-2.0, 0.0], [0.0, 0.0], [2.0, 0.0]], device=DEV)
    py = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [-2.0, -2.0], [2.0, 2.0]], device=DEV)
    bx, by = torch.tensor([0, 0, 0, 1, 1, 1], device=DEV), torch.tensor([0, 0, 1, 1], device=DEV)
    assert knn_interpolate(xi, px, py, bx, by, k=2).tolist() == z["interp_anchor_want"].tolist()
    out = knn_interpolate(_t(z, "interp_x"), _t(z, "interp_px"), _t(z, "interp_py"), _t(z, "interp_bx"),
                          _t(z, "interp_by"), k=3)
    _close(out, z["interp_out"], 1e-5, "knn_interpolate")
    zero = torch.zeros(4, dtype=torch.long, device=DEV)
    _eq(nearest(_t(z, "nearest_x"), _t(z, "nearest_y"), zero, zero[:2]), z["nearest_want"], "nearest")


def test_pointnet2_set_abstraction_matches_golden(tg_point, golden):
    z = golden("point")
    from torch_geometric.nn import PointNetConv, fps, radius
    pos, x, batch = _t(z, "sa_pos"), _t(z, "sa_x"), _t(z, "sa_batch")
    idx = fps(pos, batch, ratio=0.5, random_start=False)
    row, col = radius(pos, pos[idx], 0.4, batch, batch[idx], max_num_neighbors=16)
    _eq(idx, z["sa_idx"], "fps")
    _eq(row, z["sa_row"], "radius row")
    _eq(col, z["sa_col"], "radius col")
    conv = _load(PointNetConv(_mlp(3 + 4, 16, 16), add_self_loops=True), z, "sa")
    out = conv((x, None), (pos, pos[idx]), torch.stack([col, row], dim=0))
    _close(out, z["sa_out"], 1e-5, "PointNetConv")


def test_schnet_matches_golden(tg_point, golden):
    z = golden("point")
    from torch_geometric.nn.models import SchNet
    model = _load(SchNet(hidden_channels=16, num_filters=16, num_interactions=2, num_gaussians=10, cutoff=10.0), z,
                  "schnet")
    out = model(_t(z, "schnet_z"), _t(z, "schnet_pos"), _t(z, "schnet_batch"))
    _close(out, z["schnet_out"], 1e-5, "SchNet")


def test_transforms_match_golden(tg_point, golden):
    z = golden("point")
    import torch_geometric.transforms as T
    from torch_geometric.data import Data
    six = torch.tensor([[0.0, 0.0], [1.0, 0.0], [2.0, 0.0], [0.0, 1.0], [-2.0, 0.0], [0.0, -2.0]], device=DEV)
    _eq(T.KNNGraph(k=2, force_undirected=True)(Data(pos=six)).edge_index, z["knngraph_six"], "KNNGraph six")
    _eq(T.RadiusGraph(r=1.5)(Data(pos=six)).edge_index, z["radiusgraph_six"], "RadiusGraph six")
    cloud = _t(z, "cloud")
    _eq(T.KNNGraph(k=6)(Data(pos=cloud)).edge_index, z["knngraph_cloud"], "KNNGraph cloud")
    _eq(T.RadiusGraph(r=0.3, max_num_neighbors=8)(Data(pos=cloud)).edge_index, z["radiusgraph_cloud"], "RadiusGraph")
