"""Call-time routing of the reference's functional seams to the engine (SURVEY.md section 8(b)).

Every routed function keeps the reference's signature, validation and error messages.  Routing rule: the engine takes
a call iff the feature tensor is a CUDA tensor of dtype float32 / bfloat16 and the reduction is one it implements with
the reference's semantics; everything else -- CPU tensors, float64 / half / integer data, reduce='any' (whose CUDA result is unspecified in the reference itself) -- falls through to the UNTOUCHED reference function (`__wrapped__`), which is also how the parity oracle
keeps working next to the engine.  Nothing is ever silently computed on the CPU by the engine.

A `LazyRows` message (lazy.py) meets its destination index in `fused_lazy_reduce`: `x_j` or `w * x_j` becomes one CSR
gather-reduce (`Fn.aggregate`), `relu(x_j + t)` reduced by sum or mean one edge-feature sweep (`Fn.aggregate_edge_relu`,
GINEConv's message), `sigmoid(k_i + q_j) * v_j` reduced by sum or mean one gated sweep (`Fn.aggregate_gated`,
ResGatedGraphConv's message); any other lazy is materialised by the caller, as the reference would have computed it.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from .. import functional as Fn
from .. import ops
from .. import utils as U
from ..graph import CSRGraph
from . import graphs
from ._util import plain
from .lazy import GatedRows, LazyRows

_ENGINE_DTYPES = (torch.float32, torch.bfloat16)
_REDUCE = {"sum": "sum", "add": "sum", "mean": "mean", "min": "min", "amin": "min", "max": "max", "amax": "max",
           "mul": "mul"}


def engine_ok(t) -> bool:
    return isinstance(t, Tensor) and t.is_cuda and t.dtype in _ENGINE_DTYPES


def _compiling() -> bool:
    try:
        return torch.compiler.is_compiling()
    except Exception:
        return False


_plain = plain


def _sorted_ptr(index, dim_size: Optional[int]):
    """indptr of a sorted `Index` (index.py:244-299), or None: the only sortedness evidence the reference carries."""
    if not getattr(index, "is_sorted", False):
        return None
    try:
        ptr = index.get_indptr()
    except Exception:
        return None
    if dim_size is not None and ptr.numel() != dim_size + 1:
        return None
    return _plain(ptr)


# ------------------------------------------------------------------------------------------------ fused gather + reduce
def fused_lazy_reduce(lazy: LazyRows, index: Tensor, ptr: Optional[Tensor], dim_size: Optional[int], reduce: str):
    """aggregate(LazyRows(x, index_j[, w]), index_i) == one CSR gather-reduce, and
    aggregate(LazyRows(x, index_j, add=t, relu=True), index_i) == one `relu(x_j + t)` gather-reduce for sum / mean;
    None when not applicable (the caller then materialises)."""
    r = _REDUCE.get(reduce)
    if isinstance(lazy, GatedRows):
        return _fused_gated(lazy, index, ptr, dim_size, r)
    src = lazy._src
    if r is None or r == "mul" or not engine_ok(src) or index is None:
        return None
    if lazy._add is not None and (not lazy._relu or r not in ("sum", "mean")):
        return None
    if lazy._scale is not None and r in ("min", "max") and lazy._scale.requires_grad:
        return None
    if dim_size is None:
        dim_size = getattr(index, "dim_size", None)
        if dim_size is None:
            return None
    g = graphs.graph_from_pair(lazy._index, index, src.size(0), int(dim_size), ptr=ptr)
    if lazy._add is not None:
        return Fn.aggregate_edge_relu(g, src, lazy._add, r)
    x2 = src if src.dim() == 2 else src.reshape(src.size(0), -1)
    w = lazy._scale
    if w is not None and w.dtype != torch.float32:
        w = w.float()
    out = Fn.aggregate(g, x2, r, w)
    return out if src.dim() == 2 else out.view((int(dim_size), ) + tuple(src.shape[1:]))


def _same_index(a, b) -> bool:
    """The same index vector: one object, or one data pointer, dtype, shape and stride (`_lift` indexes
    `edge_index[dim]` afresh for every operand, message_passing.py:321)."""
    if a is b:
        return True
    a, b = _plain(a), _plain(b)
    return (a.device == b.device and a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride()
            and a.data_ptr() == b.data_ptr())


def _fused_gated(lazy: GatedRows, index: Tensor, ptr: Optional[Tensor], dim_size: Optional[int], r: Optional[str]):
    """aggregate(sigmoid(k_i + q_j) * v_j, index_i) == one gated sweep for sum / mean: the summand gathered by the
    aggregate's own index is k, the other q, and v must be gathered by q's index.  None otherwise."""
    if lazy._stage != "message" or r not in ("sum", "mean") or index is None:
        return None
    a, b, v = lazy._a, lazy._b, lazy._v
    a_dst, b_dst = _same_index(a._index, index), _same_index(b._index, index)
    if a_dst == b_dst:
        return None
    k, q = (a, b) if a_dst else (b, a)
    if not _same_index(v._index, q._index) or not all(engine_ok(t._src) for t in (k, q, v)):
        return None
    if dim_size is None:
        dim_size = getattr(index, "dim_size", None)
        if dim_size is None:
            return None
    if k._src.size(0) != int(dim_size) or v._src.size(0) != q._src.size(0):
        return None
    g = graphs.graph_from_pair(q._index, index, q._src.size(0), int(dim_size), ptr=ptr)
    return Fn.aggregate_gated(g, k._src, q._src, v._src, r)


# ------------------------------------------------------------------------------------------------ utils.scatter
def make_scatter(theirs):
    def scatter(src: Tensor, index: Tensor, dim: int = 0, dim_size: Optional[int] = None, reduce: str = "sum") -> Tensor:
        if isinstance(src, LazyRows):
            d = dim + src.dim() if dim < 0 else dim
            if d == 0 and not _compiling():
                out = fused_lazy_reduce(src, index, None, dim_size, reduce)
                if out is not None:
                    return out
            src = src.materialise()
        r = _REDUCE.get(reduce)
        if (not engine_ok(src) or _compiling() or r is None
                or not isinstance(index, Tensor) or index.dim() != 1):
            return theirs(src, index, dim, dim_size, reduce)           # incl. every argument error of the reference
        d = src.dim() + dim if dim < 0 else dim
        if d < 0 or d >= src.dim():
            return theirs(src, index, dim, dim_size, reduce)
        ptr = _sorted_ptr(index, dim_size) if r != "mul" else None
        if ptr is not None:                                            # sorted Index: deterministic CSR kernel, no atomics
            x = src if d == 0 else src.movedim(d, 0).contiguous()
            out = Fn.segment(x, ptr, r)
            return out if d == 0 else out.movedim(0, d)
        return U.scatter(src, _plain(index), d, dim_size, r)
    scatter.__wrapped__ = theirs
    scatter.__name__, scatter.__doc__ = "scatter", theirs.__doc__
    return scatter


def make_segment(theirs):
    def segment(src: Tensor, ptr: Tensor, reduce: str = "sum") -> Tensor:
        if isinstance(src, LazyRows):
            src = src.materialise()
        if not engine_ok(src) or _compiling() or ptr.dim() != 1 or reduce not in ("sum", "mean", "min", "max"):
            return theirs(src, ptr, reduce)
        return Fn.segment(src, _plain(ptr), reduce)
    segment.__wrapped__ = theirs
    segment.__name__, segment.__doc__ = "segment", theirs.__doc__
    return segment


def make_softmax(theirs):
    def softmax(src: Tensor, index: Optional[Tensor] = None, ptr: Optional[Tensor] = None,
                num_nodes: Optional[int] = None, dim: int = 0) -> Tensor:
        if isinstance(src, LazyRows):
            src = src.materialise()
        if not engine_ok(src) or _compiling() or (index is None and ptr is None) or (ptr is not None and ptr.dim() != 1):
            return theirs(src, index, ptr, num_nodes, dim)
        if ptr is None:
            ptr = _sorted_ptr(index, num_nodes)
        out = U.softmax(src, None if ptr is not None else _plain(index), None if ptr is None else _plain(ptr), num_nodes, dim)
        return out.to(src.dtype)                                       # the reference returns src's dtype
    softmax.__wrapped__ = theirs
    softmax.__name__, softmax.__doc__ = "softmax", theirs.__doc__
    return softmax


# ------------------------------------------------------------------------------------------------ spmm / EdgeIndex.matmul
def make_spmm(theirs):
    def spmm(src, other: Tensor, reduce: str = "sum") -> Tensor:
        r = "sum" if reduce == "add" else reduce
        if isinstance(src, CSRGraph):
            return U.spmm(src, other, reduce)
        if (engine_ok(other) and not _compiling() and isinstance(src, Tensor) and src.layout == torch.sparse_csr
                and r in ("sum", "mean", "min", "max") and other.dim() == 2 and src.dim() == 2):
            val = src.values()
            if val.dim() == 1 and val.dtype in _ENGINE_DTYPES + (torch.float64, ) and not val.requires_grad:
                g = graphs.graph_from_sparse_csr(src)
                return Fn.aggregate(g, other, r, val.float())          # differentiable wrt `other` (training included)
        return theirs(src, other, reduce)                              # EdgeIndex inputs reach edge_index._spmm below
    spmm.__wrapped__ = theirs
    spmm.__name__, spmm.__doc__ = "spmm", theirs.__doc__
    return spmm


def make_edge_index_spmm(theirs):
    """edge_index._spmm (edge_index.py:1925-1970): CUDA operands go to the CSR kernel with the EdgeIndex's own cached
    structure (no re-sort), forward and backward, all four reductions, value gradients included."""
    def _spmm(input, other: Tensor, value: Optional[Tensor] = None, reduce: str = "sum", transpose: bool = False) -> Tensor:
        r = "sum" if reduce == "add" else reduce
        if (not engine_ok(other) or _compiling() or other.dim() != 2 or r not in ("sum", "mean", "min", "max")
                or (value is not None and (value.dim() != 1 or not value.is_floating_point()))
                or (value is not None and value.requires_grad and r not in ("sum", "mean"))):
            return theirs(input, other, value, reduce, transpose)
        if (not transpose and not input.is_sorted_by_row) or (transpose and not input.is_sorted_by_col):
            return theirs(input, other, value, reduce, transpose)      # raises the reference's ValueError
        g = graphs.graph_from_edge_index(input, transpose)
        return Fn.aggregate(g, other, r, value)
    _spmm.__wrapped__ = theirs
    return _spmm


# ------------------------------------------------------------------------------------------------ Aggregation.reduce
def make_aggr_reduce(theirs):
    """nn/aggr/base.py:173-185.  The reference ignores `ptr` unless deterministic mode is on; the engine uses it
    whenever it is there (same result, test/nn/aggr/test_basic.py:63) because the CSR kernel is the deterministic,
    atomics-free path -- and this is where a LazyRows message meets its destination index."""
    def reduce(self, x: Tensor, index: Optional[Tensor] = None, ptr: Optional[Tensor] = None,
               dim_size: Optional[int] = None, dim: int = -2, reduce: str = "sum") -> Tensor:
        d = dim + x.dim() if dim < 0 else dim
        if isinstance(x, LazyRows):
            if d == 0 and not _compiling() and index is not None:
                out = fused_lazy_reduce(x, index, None if ptr is None else _plain(ptr), dim_size, reduce)
                if out is not None:
                    return out
            x = x.materialise()
        if engine_ok(x) and not _compiling() and ptr is not None and ptr.dim() == 1 and reduce in ("sum", "mean", "min", "max"):
            xm = x if d == 0 else x.movedim(d, 0).contiguous()
            out = Fn.segment(xm, _plain(ptr), reduce)
            return out if d == 0 else out.movedim(0, d)
        return theirs(self, x, index, ptr, dim_size, dim, reduce)
    reduce.__wrapped__ = theirs
    return reduce


# ------------------------------------------------------------------------------------------------ QuantileAggregation
def make_quantile_forward(theirs):
    """QuantileAggregation.forward (nn/aggr/quantile.py:71-131; MedianAggregation inherits it): CUDA float32 / bfloat16
    messages with a float32 `q` buffer take one selection sweep (functional.quantile_aggregate) instead of two sorts
    of the [E, F] matrix.  A lazy `x_j` without a scale is never gathered: its CSR comes from the layer's index pair,
    as in fused_lazy_reduce.  A scaled one (`w * x_j`) is materialised and read as edge rows.  Everything else --
    CPU tensors, other dtypes, compiling or scripting, no index -- runs the reference's forward."""
    def forward(self, x, index: Optional[Tensor] = None, ptr: Optional[Tensor] = None, dim_size: Optional[int] = None,
                dim: int = -2) -> Tensor:
        from ..nn.aggr import quantile_layout
        lazy = isinstance(x, LazyRows) and not isinstance(x, GatedRows)
        src = x._src if lazy else x
        d = dim + x.dim() if dim < 0 else dim
        if (index is None or not engine_ok(src) or _compiling() or torch.jit.is_scripting()
                or not isinstance(self.q, Tensor) or self.q.dtype != torch.float32 or self.q.device != src.device
                or self.interpolation not in ops.QUANTILE_INTERPOLATIONS or (lazy and x._add is not None)):
            if isinstance(x, LazyRows):
                x = x.materialise()
            return theirs(self, x, index, ptr, dim_size, dim)
        index = _plain(index)
        if dim_size is None:
            dim_size = int(index.max()) + 1 if index.numel() > 0 else 0        # the reference's bincount length
        if lazy and d == 0 and x._scale is None:
            g = graphs.graph_from_pair(x._index, index, src.size(0), int(dim_size), ptr=None if ptr is None else _plain(ptr))
            out = Fn.quantile_aggregate(g, src.reshape(src.size(0), -1), None, self.q, self.interpolation,
                                        self.fill_value)
            return quantile_layout(out, self.q.numel(), tuple(x.shape), 0)
        if isinstance(x, LazyRows):
            x = x.materialise()
        xm = x.movedim(d, 0)
        x2 = xm.reshape(xm.size(0), -1)
        if x2.size(0) == 0:
            return theirs(self, x, index, ptr, dim_size, dim)
        sptr = _sorted_ptr(index, dim_size)
        if sptr is not None:
            out = Fn.quantile_aggregate((sptr, ops.segment_plan(sptr, x2.size(0))), None, x2, self.q,
                                        self.interpolation, self.fill_value)
        else:
            e = torch.arange(index.numel(), device=index.device, dtype=index.dtype)
            out = Fn.quantile_aggregate(CSRGraph(e, index, index.numel(), int(dim_size)), None, x2, self.q,
                                        self.interpolation, self.fill_value)
        return quantile_layout(out, self.q.numel(), tuple(x.shape), d)
    forward.__wrapped__ = theirs
    forward.__name__, forward.__doc__ = "forward", theirs.__doc__
    return forward


# ------------------------------------------------------------------------------------------------ MessagePassing._index_select
def make_index_select(theirs):
    """nn/conv/message_passing.py:263-267: the gather of `_collect` / `_lift` becomes lazy (see lazy.py)."""
    def _index_select(self, src: Tensor, index) -> Tensor:
        if (engine_ok(src) and not _compiling() and not torch.jit.is_scripting() and isinstance(index, Tensor)
                and index.dim() == 1 and src.dim() >= 2 and (self.node_dim == 0 or self.node_dim == -src.dim())
                and not isinstance(src, LazyRows) and not getattr(self, "explain", False)):
            return LazyRows(src, index)
        return theirs(self, src, index)
    _index_select.__wrapped__ = theirs
    return _index_select
