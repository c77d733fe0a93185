"""The optional-extension operator signatures the reference binds to (SURVEY.md section 8(b), row 2), served by the
engine: flipping `torch_geometric.typing.WITH_*` to True with these modules bound makes every `torch_scatter.*`,
`pyg_lib.ops.*` and `torch.ops.torch_sparse.*` call site of the reference land in the sm_90a kernels.

  torch_scatter.scatter(src, index, dim, out=None, dim_size=None, reduce=...)      utils/_scatter.py:115,135
  torch_scatter.scatter_max / scatter_min(...) -> (out, arg)                       utils/_scatter.py:156
  torch_scatter.segment_csr(src, indptr, out=None, reduce=...)                     utils/_segment.py:34
  torch.ops.torch_sparse.spmm_sum(row, rowptr, col, value, colptr, csr2csc, mat)   edge_index.py:1798-1800
  torch.ops.torch_sparse.spmm_mean(row, rowptr, col, value, rowcount, colptr, csr2csc, mat)          :1802-1805
  torch.ops.torch_sparse.spmm_min / spmm_max(rowptr, col, value, mat) -> (out, arg)                  :1807-1810
  pyg_lib.ops.softmax_csr(src, ptr, dim)                                           utils/_softmax.py:58
  pyg_lib.ops.index_sort(inputs, max_value) -> (values, perm)                      utils/_index_sort.py:32
  pyg_lib.ops.segment_matmul(inputs, ptr, other) / grouped_matmul(inputs, others, biases)   nn/dense/linear.py:255,304-330
  pyg_lib.ops.spline_basis(pseudo, kernel_size, is_open_spline, degree) -> (basis, weight_index)  nn/conv/spline_conv.py:151
  pyg_lib.ops.spline_weighting(x, weight, basis, weight_index)                     nn/conv/spline_conv.py:153
  torch.ops.pyg.knn / radius / fps / nearest (also pyg_lib.ops.*)                  nn/pool/__init__.py:85-375,
                                                                                   nn/conv/{edge,gravnet,x}_conv.py
  torch.ops.pyg.graclus_cluster / grid_cluster (also pyg_lib.ops.*)               nn/pool/graclus.py:39,
                                                                                   nn/pool/voxel_grid.py:66
  torch.ops.pyg.random_walk(rowptr, col, seed, walk_length, p, q) (also pyg_lib.ops.*)   nn/models/node2vec.py:64,103,
                                                                                   utils/dropout.py:285,
                                                                                   transforms/rooted_subgraph.py:171

CUDA fp32 / bf16 operands run in the engine.  The spline and point-cloud ops have no reference fall-back (the reference has no
ATen branch for them), so CPU, float16 and float64 operands raise RuntimeError; neither have the clustering ops, which
take CUDA tensors only (graclus: float32 / bfloat16 / float64 weights; grid_cluster: float32 / float64 positions), nor
has random_walk (int32 or int64 indices).  Other CPU operands fall through to the reference's own ATen branch (the
shim calls the reference function with the extension flag switched off for the duration of the call) -- the engine
itself never computes on the CPU.  torch.ops.torch_sparse.* are `torch.library` operators with a CUDA implementation,
a Meta (shape) implementation so tracing stays legal, and autograd formulas that use the transposed structure the
reference passes (colptr, csr2csc), exactly like torch_sparse's own.

Semantics note: real torch_scatter / torch_sparse route the min / max gradient to ONE arg element; the reference
without extensions (ATen `scatter_reduce`) splits it evenly among ties.  `scatter(..., reduce='max')` here keeps the
ATen rule (the pinned oracle); the explicit `(out, arg)` operators return the first extremum like the originals.
"""
from __future__ import annotations

import contextlib
import types
from typing import List, Optional, Tuple

import torch
from torch import Tensor

from .. import dense
from .. import functional as Fn
from .. import ops
from .. import utils as U

_ENGINE = (torch.float32, torch.bfloat16)


def _ok(t) -> bool:
    return isinstance(t, Tensor) and t.is_cuda and t.dtype in _ENGINE


@contextlib.contextmanager
def _flags_set(value: bool, *names):
    import torch_geometric.typing as T
    old = {n: getattr(T, n) for n in names}
    try:
        for n in names:
            setattr(T, n, value)
        yield
    finally:
        for n, v in old.items():
            setattr(T, n, v)


def _flags_off(*names):
    return _flags_set(False, *names)


def _flags_on(*names):
    return _flags_set(True, *names)


# ================================================================================================ torch_scatter
def _ts_scatter(src: Tensor, index: Tensor, dim: int = -1, out: Optional[Tensor] = None, dim_size: Optional[int] = None,
                reduce: str = "sum") -> Tensor:
    if out is not None:
        raise NotImplementedError("torch_scatter.scatter(out=...) is not used by the reference and not provided")
    d = dim + src.dim() if dim < 0 else dim
    if index.dim() != 1:                                    # torch_scatter broadcasts the index; the reference passes 1-D
        index = index.movedim(d, 0).reshape(index.size(d), -1)[:, 0] if index.dim() == src.dim() else index.reshape(-1)
    if _ok(src):
        return U.scatter(src, index, d, dim_size, reduce)
    from torch_geometric.utils import _scatter as S
    with _flags_off("WITH_TORCH_SCATTER"):
        return getattr(S.scatter, "__wrapped__", S.scatter)(src, index, d, dim_size, reduce)


def _ts_scatter_arg(which: str):
    def fn(src: Tensor, index: Tensor, dim: int = -1, out: Optional[Tensor] = None,
           dim_size: Optional[int] = None) -> Tuple[Tensor, Tensor]:
        if out is not None:
            raise NotImplementedError("out= is not provided")
        d = dim + src.dim() if dim < 0 else dim
        if dim_size is None:
            dim_size = int(index.max()) + 1 if index.numel() else 0
        if not (isinstance(src, Tensor) and src.is_cuda):
            raise NotImplementedError(f"torch_scatter.scatter_{which} shim: CUDA tensors only (the reference itself only "
                                      "calls it when the real extension is installed)")
        x = src if d == 0 else src.movedim(d, 0)
        x32 = x.contiguous().float()
        o = ops.scatter_coo(x32, index.contiguous(), dim_size, which)
        arg = ops.scatter_arg(x32, index.contiguous(), o)
        o = o.to(src.dtype)
        return (o, arg) if d == 0 else (o.movedim(0, d), arg.movedim(0, d))
    fn.__name__ = f"scatter_{which}"
    return fn


def _ts_segment_csr(src: Tensor, indptr: Tensor, out: Optional[Tensor] = None, reduce: str = "sum") -> Tensor:
    if out is not None:
        raise NotImplementedError("out= is not provided")
    if indptr.dim() != 1:                                   # expand_left'ed ptr of Aggregation.reduce: [1, ..., N+1]
        d = indptr.dim() - 1
        x = src if d == 0 else src.movedim(d, 0)
        res = _ts_segment_csr(x.contiguous(), indptr.reshape(-1), None, reduce)
        return res if d == 0 else res.movedim(0, d)
    if _ok(src):
        return U.segment(src, indptr, reduce)
    from torch_geometric.utils import _segment as S
    with _flags_off("WITH_TORCH_SCATTER"):
        return getattr(S.segment, "__wrapped__", S.segment)(src, indptr, reduce)


def torch_scatter_module() -> types.ModuleType:
    m = types.ModuleType("torch_scatter")
    m.__doc__ = "pytorch_geometric_b200 shim of the torch_scatter operators the reference calls"
    m.scatter = _ts_scatter
    for r in ("sum", "add", "mean", "mul", "min", "max"):
        if r in ("min", "max"):
            setattr(m, f"scatter_{r}", _ts_scatter_arg(r))
        else:
            setattr(m, f"scatter_{r}", (lambda rr: lambda src, index, dim=-1, out=None, dim_size=None:
                                        _ts_scatter(src, index, dim, out, dim_size, rr))(r))
    m.segment_csr = _ts_segment_csr
    m.__version__ = "b200mp-shim"
    return m


# ================================================================================================ torch.ops.torch_sparse
_SPARSE_LIB = None


def _mean_rowcount(rowptr: Tensor) -> Tensor:
    return (rowptr[1:] - rowptr[:-1]).clamp(min=1).to(torch.float32)


def register_torch_sparse_ops() -> bool:
    """Defines torch.ops.torch_sparse.spmm_{sum,mean,min,max} with torch_sparse's schemas (CUDA + Meta + autograd).
    Returns False when the namespace already has them (the real extension is installed)."""
    global _SPARSE_LIB
    if _SPARSE_LIB is not None:
        return True
    try:
        torch.ops.torch_sparse.spmm_sum                                            # noqa: B018
        return False
    except (AttributeError, RuntimeError):
        pass
    lib = torch.library.Library("torch_sparse", "DEF")
    lib.define("spmm_sum(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? colptr, Tensor? csr2csc, Tensor mat) -> Tensor")
    lib.define("spmm_mean(Tensor? row, Tensor rowptr, Tensor col, Tensor? value, Tensor? rowcount, Tensor? colptr, Tensor? csr2csc, Tensor mat) -> Tensor")
    lib.define("spmm_min(Tensor rowptr, Tensor col, Tensor? value, Tensor mat) -> (Tensor, Tensor)")
    lib.define("spmm_max(Tensor rowptr, Tensor col, Tensor? value, Tensor mat) -> (Tensor, Tensor)")

    def fwd(rowptr, col, value, mat, reduce):
        if mat.dtype not in _ENGINE:
            raise TypeError("torch_sparse.spmm_* (b200mp): float32 / bfloat16 only")
        v = None if value is None else value.detach().float()
        return ops.spmm_csr(rowptr, col, v, mat.detach(), rowptr.numel() - 1, reduce)

    def sum_cuda(row, rowptr, col, value, colptr, csr2csc, mat):
        return fwd(rowptr, col, value, mat, "sum")

    def mean_cuda(row, rowptr, col, value, rowcount, colptr, csr2csc, mat):
        return fwd(rowptr, col, value, mat, "mean")

    def arg_cuda(reduce):
        def f(rowptr, col, value, mat):
            m32 = mat.detach().float().contiguous()
            v = None if value is None else value.detach().float()
            out = ops.spmm_csr(rowptr, col, v, m32, rowptr.numel() - 1, reduce)
            arg = ops.spmm_csr_arg(rowptr, col, v, m32, out)
            return out.to(mat.dtype), arg
        return f

    def meta1(*args):
        rowptr, mat = (args[1], args[-1])
        return mat.new_empty((rowptr.numel() - 1, mat.size(1)))

    def meta2(rowptr, col, value, mat):
        n = rowptr.numel() - 1
        return mat.new_empty((n, mat.size(1))), mat.new_empty((n, mat.size(1)), dtype=torch.long)

    lib.impl("spmm_sum", sum_cuda, "CUDA")
    lib.impl("spmm_mean", mean_cuda, "CUDA")
    lib.impl("spmm_min", arg_cuda("min"), "CUDA")
    lib.impl("spmm_max", arg_cuda("max"), "CUDA")
    lib.impl("spmm_sum", meta1, "Meta")
    lib.impl("spmm_mean", meta1, "Meta")
    lib.impl("spmm_min", meta2, "Meta")
    lib.impl("spmm_max", meta2, "Meta")

    # ---- autograd (torch_sparse/csrc/spmm.cpp: grad_mat = A^T grad through (colptr, csr2csc); grad_value = SDDMM)
    def make_backward(is_mean):
        def setup(ctx, inputs, output):
            if is_mean:
                row, rowptr, col, value, rowcount, colptr, csr2csc, mat = inputs
            else:
                row, rowptr, col, value, colptr, csr2csc, mat = inputs
            ctx.save_for_backward(row, rowptr, col, value, colptr, csr2csc, mat)

        def backward(ctx, grad):
            row, rowptr, col, value, colptr, csr2csc, mat = ctx.saved_tensors
            grad = grad.contiguous()
            need_mat = ctx.needs_input_grad[-1]
            need_val = value is not None and ctx.needs_input_grad[3]
            g_mat = g_val = None
            scale = None
            if is_mean:
                scale = 1.0 / _mean_rowcount(rowptr)                         # per destination row
            if need_mat:
                if colptr is None or csr2csc is None or row is None:
                    raise RuntimeError("spmm backward needs row / colptr / csr2csc (the reference passes them when "
                                       "`other.requires_grad`, edge_index.py:1789-1796)")
                row_t = row.index_select(0, csr2csc)
                w = None if value is None else value.detach().float().index_select(0, csr2csc)
                if scale is not None:
                    s_t = scale.index_select(0, row_t)
                    w = s_t if w is None else w * s_t
                g_mat = ops.spmm_csr(colptr, row_t, w, grad, mat.size(0), "sum")
            if need_val:
                dot = ops.sddmm_csr(rowptr, col, grad, mat.detach())         # <grad[row(e)], mat[col[e]]> in CSR order
                if scale is not None:
                    dot = dot * scale.index_select(0, ops.ptr2index(rowptr, col.numel()))
                g_val = dot.to(value.dtype)
            n_in = 8 if is_mean else 7
            res = [None] * n_in
            res[3], res[-1] = g_val, g_mat
            return tuple(res)
        return setup, backward

    for name, is_mean in (("spmm_sum", False), ("spmm_mean", True)):
        setup, backward = make_backward(is_mean)
        torch.library.register_autograd(f"torch_sparse::{name}", backward, setup_context=setup, lib=lib)

    def arg_setup(ctx, inputs, output):
        rowptr, col, value, mat = inputs
        ctx.save_for_backward(col, value, output[1], mat)

    def arg_backward(ctx, grad, _grad_arg):
        col, value, arg, mat = ctx.saved_tensors
        nnz = col.numel()
        if nnz == 0:
            return None, None, (None if value is None else torch.zeros_like(value)), torch.zeros_like(mat)
        valid = arg < nnz
        a = arg.clamp(max=nnz - 1)
        g = torch.where(valid, grad, torch.zeros_like(grad))
        src_row = col.long()[a]                                              # [n_rows, F]: the producing source row
        g_mat = g_val = None
        # one producer per output element (torch_sparse semantics): element-wise scatters, done by ATen
        if ctx.needs_input_grad[3]:
            gm = g if value is None else g * value.detach().to(g.dtype)[a]
            g_mat = torch.zeros_like(mat).scatter_add_(0, src_row, gm)
        if value is not None and ctx.needs_input_grad[2]:
            contrib = g * mat.detach().gather(0, src_row)
            g_val = torch.zeros(nnz, dtype=contrib.dtype, device=contrib.device).scatter_add_(0, a.reshape(-1), contrib.reshape(-1))
            g_val = g_val.to(value.dtype)
        return None, None, g_val, g_mat

    for name in ("spmm_min", "spmm_max"):
        torch.library.register_autograd(f"torch_sparse::{name}", arg_backward, setup_context=arg_setup, lib=lib)
    _SPARSE_LIB = lib
    return True


# ================================================================================================ pyg_lib.ops
def _pl_softmax_csr(src: Tensor, ptr: Tensor, dim: int = 0) -> Tensor:
    if _ok(src):
        return U.softmax(src, None, ptr, None, dim).to(src.dtype)
    from torch_geometric.utils import _softmax as S
    with _flags_off("WITH_SOFTMAX", "WITH_TORCH_SCATTER"):
        return getattr(S.softmax, "__wrapped__", S.softmax)(src, None, ptr, None, dim)


def _pl_index_sort(inputs: Tensor, max_value: Optional[int] = None) -> Tuple[Tensor, Tensor]:
    if isinstance(inputs, Tensor) and inputs.is_cuda and inputs.dtype in (torch.int32, torch.int64) and inputs.dim() == 1:
        return U.index_sort(inputs, max_value)
    return inputs.sort(stable=True)


def _pl_segment_matmul(inputs: Tensor, ptr: Tensor, other: Tensor) -> Tensor:
    """out[ptr[r]:ptr[r+1]] = inputs[ptr[r]:ptr[r+1]] @ other[r]   (nn/dense/linear.py:248-255, rgcn_conv.py:288)."""
    return dense.segment_matmul(inputs, ptr, other)


def _pl_grouped_matmul(inputs: List[Tensor], others: List[Tensor], biases: Optional[List[Tensor]] = None) -> List[Tensor]:
    return dense.grouped_matmul(inputs, others, biases)


def _pl_spline_basis(pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor, degree: int) -> Tuple[Tensor, Tensor]:
    return Fn.spline_basis(pseudo, kernel_size, is_open_spline, degree)


def _pl_spline_weighting(x: Tensor, weight: Tensor, basis: Tensor, weight_index: Tensor) -> Tensor:
    return Fn.spline_weighting(x, weight, basis, weight_index)


# ================================================================================================ torch.ops.pyg (point clouds)
_POINT_LIB = None
POINT_SCHEMAS = {
    "knn": "knn(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y, int k, bool cosine, int num_workers) -> Tensor",
    "radius": "radius(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y, float r, int max_num_neighbors, "
              "int num_workers, bool ignore_same_index) -> Tensor",
    "fps": "fps(Tensor src, Tensor ptr, float ratio, bool random_start) -> Tensor",
    "nearest": "nearest(Tensor x, Tensor y, Tensor? ptr_x, Tensor? ptr_y) -> Tensor",
}


def _pyg_knn(x: Tensor, y: Tensor, ptr_x: Optional[Tensor], ptr_y: Optional[Tensor], k: int, cosine: bool = False,
             num_workers: int = 1) -> Tensor:
    return ops.knn(x, y, k, ptr_x, ptr_y, cosine)


def _pyg_radius(x: Tensor, y: Tensor, ptr_x: Optional[Tensor], ptr_y: Optional[Tensor], r: float,
                max_num_neighbors: int = 32, num_workers: int = 1, ignore_same_index: bool = False) -> Tensor:
    return ops.radius(x, y, r, ptr_x, ptr_y, max_num_neighbors, ignore_same_index)


def _pyg_fps(src: Tensor, ptr: Tensor, ratio: float = 0.5, random_start: bool = True) -> Tensor:
    return ops.fps(src, ptr, ratio, random_start)


def _pyg_nearest(x: Tensor, y: Tensor, ptr_x: Optional[Tensor] = None, ptr_y: Optional[Tensor] = None) -> Tensor:
    return ops.nearest(x, y, ptr_x, ptr_y)


POINT_OPS = {"knn": _pyg_knn, "radius": _pyg_radius, "fps": _pyg_fps, "nearest": _pyg_nearest}


def _define_pyg_ops(schemas: dict, impls: dict) -> tuple:
    """Defines the torch.ops.pyg operators of `schemas` that the namespace lacks, with CUDA implementations only (an
    operator it already has -- the real pyg-lib is installed -- is left alone).  Returns (library, number defined)."""
    missing = []
    for name in schemas:
        try:
            getattr(torch.ops.pyg, name)
        except (AttributeError, RuntimeError):
            missing.append(name)
    lib = torch.library.Library("pyg", "FRAGMENT")
    for name in missing:
        lib.define(schemas[name])
        lib.impl(name, impls[name], "CUDA")
    return lib, len(missing)


def register_point_ops() -> int:
    """Defines torch.ops.pyg.{knn, radius, fps, nearest} with pyg-lib's schemas and CUDA implementations only.  Returns
    the number of operators this call or an earlier one defined; an operator the namespace already has (the real
    pyg-lib is installed) is left alone."""
    global _POINT_LIB
    if _POINT_LIB is None:
        _POINT_LIB = _define_pyg_ops(POINT_SCHEMAS, POINT_OPS)
    return _POINT_LIB[1]


# ================================================================================================ torch.ops.pyg (clustering)
_CLUSTER_LIB = None
CLUSTER_SCHEMAS = {
    "graclus_cluster": "graclus_cluster(Tensor rowptr, Tensor col, Tensor? weight) -> Tensor",
    "grid_cluster": "grid_cluster(Tensor pos, Tensor size, Tensor? start, Tensor? end) -> Tensor",
}


def _pyg_graclus_cluster(rowptr: Tensor, col: Tensor, weight: Optional[Tensor] = None) -> Tensor:
    return ops.graclus(rowptr, col, weight)


def _pyg_grid_cluster(pos: Tensor, size: Tensor, start: Optional[Tensor] = None,
                      end: Optional[Tensor] = None) -> Tensor:
    return ops.grid_cluster(pos, size, start, end)


CLUSTER_OPS = {"graclus_cluster": _pyg_graclus_cluster, "grid_cluster": _pyg_grid_cluster}


def register_cluster_ops() -> int:
    """Defines torch.ops.pyg.{graclus_cluster, grid_cluster} with pyg-lib's schemas and CUDA implementations only, as
    register_point_ops does for the point-cloud operators."""
    global _CLUSTER_LIB
    if _CLUSTER_LIB is None:
        _CLUSTER_LIB = _define_pyg_ops(CLUSTER_SCHEMAS, CLUSTER_OPS)
    return _CLUSTER_LIB[1]


# ================================================================================================ torch.ops.pyg (random walks)
_WALK_LIB = None
WALK_SCHEMAS = {
    "random_walk": "random_walk(Tensor rowptr, Tensor col, Tensor seed, int walk_length, float p=1.0, "
                   "float q=1.0) -> Tensor",
}


def _pyg_random_walk(rowptr: Tensor, col: Tensor, seed: Tensor, walk_length: int, p: float = 1.0,
                     q: float = 1.0) -> Tensor:
    # pyg-lib names the start nodes `seed`; the walks' random seed comes from torch's CPU generator
    return ops.random_walk(rowptr, col, seed, walk_length, p, q)


WALK_OPS = {"random_walk": _pyg_random_walk}


def register_walk_ops() -> int:
    """Defines torch.ops.pyg.random_walk with pyg-lib's schema and a CUDA implementation only, as register_point_ops
    does for the point-cloud operators."""
    global _WALK_LIB
    if _WALK_LIB is None:
        _WALK_LIB = _define_pyg_ops(WALK_SCHEMAS, WALK_OPS)
    return _WALK_LIB[1]


def make_dropout_path(theirs):
    """utils.dropout_path (utils/dropout.py:221-298) for CUDA edge_index: the unmodified reference function with the
    global WITH_PYG_LIB switched on for this call only, so it reaches torch.ops.pyg.random_walk.  The flag itself stays
    off: NeighborLoader and to_hetero read it too, and the engine has no neighbour sampler.  CPU input goes to the
    reference unchanged (and raises its own ImportError)."""
    import functools

    @functools.wraps(theirs)
    def dropout_path(edge_index: Tensor, p: float = 0.2, walks_per_node: int = 1, walk_length: int = 3,
                     num_nodes: Optional[int] = None, is_sorted: bool = False, training: bool = True):
        if isinstance(edge_index, Tensor) and edge_index.is_cuda:
            with _flags_on("WITH_PYG_LIB"):
                return theirs(edge_index, p, walks_per_node, walk_length, num_nodes, is_sorted, training)
        return theirs(edge_index, p, walks_per_node, walk_length, num_nodes, is_sorted, training)
    return dropout_path


def pyg_lib_module() -> types.ModuleType:
    m = types.ModuleType("pyg_lib")
    m.__doc__ = "pytorch_geometric_b200 shim of the pyg_lib.ops operators on the aggregation path"
    m.ops = types.ModuleType("pyg_lib.ops")
    m.ops.softmax_csr = _pl_softmax_csr
    m.ops.index_sort = _pl_index_sort
    m.ops.segment_matmul = _pl_segment_matmul
    m.ops.grouped_matmul = _pl_grouped_matmul
    m.ops.spline_basis = _pl_spline_basis
    m.ops.spline_weighting = _pl_spline_weighting
    m.ops.knn = _pyg_knn
    m.ops.radius = _pyg_radius
    m.ops.fps = _pyg_fps
    m.ops.nearest = _pyg_nearest
    m.ops.graclus_cluster = _pyg_graclus_cluster
    m.ops.grid_cluster = _pyg_grid_cluster
    m.ops.random_walk = _pyg_random_walk
    m.__version__ = "b200mp-shim"
    return m
