"""Host-side mirror of the reference's functional API for the aggregation path: same names,
argument meaning and error behaviour as torch_geometric.utils.{scatter, segment, softmax, spmm,
degree, index_sort, add_remaining_self_loops, ...}, routed to the sm_90a kernels.

Differences from the reference, all deliberate:
 * CUDA tensors only -- a CPU tensor raises instead of silently running somewhere else.
 * `scatter` uses the deterministic CSR kernel whenever the index is known to be sorted (pass
   `sorted=True`, or an index produced by `ptr2index`) and the atomic COO kernel otherwise.
 * `dim_size=None` costs the same device->host read as the reference's `int(index.max()) + 1`
   (_scatter.py:48); pass it to stay asynchronous.
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch
from torch import Tensor

from . import functional as Fn
from . import ops
from .graph import CSRGraph


def _move_dim0(src: Tensor, dim: int) -> Tuple[Tensor, bool]:
    if dim == 0:
        return src, False
    return src.movedim(dim, 0).contiguous(), True


def scatter(src: Tensor, index: Tensor, dim: int = 0, dim_size: Optional[int] = None, reduce: str = "sum",
            sorted: Optional[bool] = None) -> Tensor:
    """Mirror of torch_geometric.utils.scatter (utils/_scatter.py:14-138)."""
    if isinstance(index, Tensor) and index.dim() != 1:
        raise ValueError(f"The `index` argument must be one-dimensional (got {index.dim()} dimensions)")
    dim = src.dim() + dim if dim < 0 else dim
    if dim < 0 or dim >= src.dim():
        raise ValueError(f"The `dim` argument must lay between 0 and {src.dim() - 1} (got {dim})")
    if reduce not in ("sum", "add", "mean", "min", "max", "amin", "amax", "mul", "any"):
        raise ValueError(f"Encountered invalid `reduce` argument '{reduce}'")
    reduce = {"add": "sum", "amin": "min", "amax": "max"}.get(reduce, reduce)
    if dim_size is None:
        dim_size = (ops.index_stats(index)[1] + 1) if index.numel() > 0 else 0
    x, moved = _move_dim0(src, dim)
    if reduce == "any":
        out = Fn.scatter_any(x if x.dtype in (torch.float32, torch.bfloat16) else x.float(), index, dim_size).to(x.dtype)
        return out.movedim(0, dim) if moved else out
    if sorted and reduce != "mul" and x.dtype in (torch.float32, torch.bfloat16):
        out = Fn.segment(x, ops.index2ptr(index, dim_size), reduce)
    else:
        if x.dtype != torch.float32:
            out = Fn.scatter_coo(x.float(), index, dim_size, reduce).to(x.dtype)
        else:
            out = Fn.scatter_coo(x, index, dim_size, reduce)
    return out.movedim(0, dim) if moved else out


def scatter_argmax(src: Tensor, index: Tensor, dim: int = 0, dim_size: Optional[int] = None) -> Tensor:
    """Mirror of torch_geometric.utils.scatter_argmax (utils/_scatter.py:145-182) for the 1-D case it implements: the position
    of a maximal member of every group; empty groups give dim_size - 1 (the reference's fill value).  The maximum comes from
    the atomic COO kernel, the position from b200mp_scatter_arg (the smallest tied position; the reference leaves ties to
    the order of a duplicate-index assignment)."""
    assert src.dim() == 1 and index.dim() == 1
    assert dim == 0 or dim == -1
    assert src.numel() == index.numel()
    if dim_size is None:
        dim_size = (ops.index_stats(index)[1] + 1) if index.numel() > 0 else 0
    x = src.detach().float().view(-1, 1)
    res = ops.scatter_coo(x, index, dim_size, "max")
    arg = ops.scatter_arg(x, index, res).view(-1)
    return torch.where(arg >= src.numel(), arg.new_full((), dim_size - 1), arg).to(index.dtype)


def group_argsort(src: Tensor, index: Tensor, dim: int = 0, num_groups: Optional[int] = None, descending: bool = False,
                  return_consecutive: bool = False, stable: bool = False) -> Tensor:
    """Rank of every value inside its group -- the contract of torch_geometric.utils.group_argsort (utils/_scatter.py:185-246).
    Two stable sorts: the values (torch's float sort), then the group ids with the engine's stable radix sort
    (`b200mp_sort_by_key`), which also returns the group offsets -- no value normalisation, so large group ids cannot
    collide in float arithmetic.  Index bookkeeping, not a hot path."""
    if src.dim() != 1 or index.dim() != 1 or src.numel() != index.numel() or dim not in (0, -1):
        raise AssertionError("group_argsort is defined for 1-D `src` / `index` of equal length along dim 0")
    n = src.numel()
    if n == 0:
        return torch.zeros_like(src)
    if num_groups is None:
        num_groups = ops.index_stats(index)[1] + 1
    by_value = torch.argsort(src, descending=descending, stable=True).to(index.dtype)
    _, by_group, ptr = ops.sort_by_key(ops.permute(index, by_value), num_groups, want_sorted=False)
    order = ops.permute(by_value, by_group)                         # order[r] = the element at position r of the grouped order
    rank = torch.empty_like(index)
    rank[order.long()] = torch.arange(n, device=index.device, dtype=index.dtype)
    if return_consecutive:
        return rank
    return rank - ptr[index.long()]


def group_cat(tensors, indices, dim: int = 0, return_index: bool = False):
    """Concatenation grouped by the index tensors -- the contract of torch_geometric.utils.group_cat
    (utils/_scatter.py:249-300): one stable radix sort of the concatenated group ids, one row gather."""
    if len(tensors) != len(indices):
        raise AssertionError("group_cat needs one index tensor per tensor")
    index = torch.cat(list(indices))
    n_groups = (ops.index_stats(index)[1] + 1) if index.numel() else 0
    sorted_index, perm, _ = ops.sort_by_key(index, n_groups, want_ptr=False)
    stacked = torch.cat(list(tensors), dim=dim)
    d = dim + stacked.dim() if dim < 0 else dim
    if d == 0 and stacked.dtype in (torch.float32, torch.bfloat16):
        out = ops.gather_rows(stacked, perm)
    else:
        out = stacked.index_select(d, perm.long())
    return (out, sorted_index) if return_index else out


def segment(src: Tensor, ptr: Tensor, reduce: str = "sum") -> Tensor:
    """Mirror of torch_geometric.utils.segment (utils/_segment.py:11-50); ptr must be 1-D."""
    if ptr.dim() != 1:
        raise ImportError("'segment' in an arbitrary dimension requires the 'torch-scatter' package")
    if reduce not in ("sum", "mean", "min", "max"):
        raise ValueError(f"Encountered invalid `reduce` argument '{reduce}'")
    return Fn.segment(src, ptr, reduce)


def softmax(src: Tensor, index: Optional[Tensor] = None, ptr: Optional[Tensor] = None,
            num_nodes: Optional[int] = None, dim: int = 0) -> Tensor:
    """Mirror of torch_geometric.utils.softmax (utils/_softmax.py:12-92).  The ptr path runs the
    CSR kernel directly; the index path sorts once (stable) and un-permutes the result."""
    dim = dim + src.dim() if dim < 0 else dim
    x, moved = _move_dim0(src, dim)
    if ptr is not None:
        out = Fn.softmax_csr(x, ptr)
    elif index is not None:
        N = num_nodes if num_nodes is not None else ((ops.index_stats(index)[1] + 1) if index.numel() else 0)
        _, perm, p = ops.sort_by_key(index, N, want_sorted=False)
        inv = torch.empty_like(perm)
        inv[perm.long()] = torch.arange(perm.numel(), device=perm.device, dtype=perm.dtype)
        out = Fn.softmax_csr(x.index_select(0, perm.long()), p).index_select(0, inv.long())
    else:
        raise NotImplementedError("'softmax' requires 'index' to be specified")
    return out.movedim(0, dim) if moved else out


def degree(index: Tensor, num_nodes: Optional[int] = None, dtype: Optional[torch.dtype] = None) -> Tensor:
    """Mirror of torch_geometric.utils.degree (utils/_degree.py:9-31)."""
    N = num_nodes if num_nodes is not None else ((ops.index_stats(index)[1] + 1) if index.numel() else 0)
    deg = ops.degree(index, N)
    return deg.to(dtype if dtype is not None else torch.get_default_dtype())


def index2ptr(index: Tensor, size: Optional[int] = None) -> Tensor:
    """torch_geometric.index.index2ptr (index.py:32-37)."""
    if size is None:
        size = int(index.max()) + 1 if index.numel() > 0 else 0
    return ops.index2ptr(index, size)


def ptr2index(ptr: Tensor, output_size: Optional[int] = None) -> Tensor:
    """torch_geometric.index.ptr2index (index.py:27-30)."""
    return ops.ptr2index(ptr, output_size)


def index_sort(inputs: Tensor, max_value: Optional[int] = None, stable: bool = False) -> Tuple[Tensor, Tensor]:
    """Mirror of torch_geometric.utils.index_sort (utils/_index_sort.py:10-32): always stable
    (a member of the set of permutations the reference accepts)."""
    if max_value is None:
        max_value = ops.index_stats(inputs)[1] if inputs.numel() else 0
    ks, perm, _ = ops.sort_by_key(inputs, int(max_value) + 1, want_sorted=True, want_ptr=False)
    return ks, perm.to(torch.int64)


def sort_edge_index_by_row_col(edge_index: Tensor, num_nodes: int) -> Tuple[Tensor, Tensor, Tensor]:
    """(row, col, perm): the edges ordered by row, then column, as torch_geometric.utils.sort_edge_index orders them
    (utils/_sort_edge_index.py: the key row * N + col), by two stable passes of the engine's sort with keys in [0, N)."""
    row, col = edge_index[0].contiguous(), edge_index[1].contiguous()
    _, by_col, _ = ops.sort_by_key(col, num_nodes, want_sorted=False, want_ptr=False)
    _, by_row, _ = ops.sort_by_key(row[by_col], num_nodes, want_sorted=False, want_ptr=False)
    perm = by_col[by_row]
    return row[perm], col[perm], perm


def dropout_path(edge_index: Tensor, p: float = 0.2, walks_per_node: int = 1, walk_length: int = 3,
                 num_nodes: Optional[int] = None, is_sorted: bool = False, training: bool = True) -> Tuple[Tensor, Tensor]:
    """Mirror of torch_geometric.utils.dropout_path (utils/dropout.py:221-298): every edge that a uniform random walk
    of walk_length steps traverses is dropped, the walks starting walks_per_node times at the source of each edge
    kept by a Bernoulli(p) draw.  Returns (kept edge_index, edge mask).  The draws are the reference's: the start mask
    from torch.rand on edge_index's device, then the walks' seed from torch's CPU generator (ops.random_walk)."""
    if p < 0.0 or p > 1.0:
        raise ValueError(f"Sample probability has to be between 0 and 1 (got {p}")
    num_edges = edge_index.size(1)
    edge_mask = edge_index.new_ones(num_edges, dtype=torch.bool)
    if not training or p == 0.0:
        return edge_index, edge_mask
    if num_nodes is None:
        num_nodes = int(edge_index.max()) + 1 if edge_index.numel() > 0 else 0
    if is_sorted:
        row, col, order = edge_index[0], edge_index[1], None
    else:
        row, col, order = sort_edge_index_by_row_col(edge_index, num_nodes)
    sample_mask = torch.rand(num_edges, device=edge_index.device) <= p
    start = row[sample_mask].repeat(walks_per_node)
    walk = ops.random_walk(ops.index2ptr(row.contiguous(), num_nodes), col.contiguous(), start, walk_length)
    walk_keys = walk[:, :-1].reshape(-1).long() * num_nodes + walk[:, 1:].reshape(-1).long()
    hit = torch.isin(row.long() * num_nodes + col.long(), walk_keys).nonzero().view(-1)
    edge_mask[hit if order is None else order[hit]] = False
    return edge_index[:, edge_mask], edge_mask


def add_remaining_self_loops(edge_index: Tensor, edge_attr: Optional[Tensor] = None,
                             fill_value: Optional[float] = None,
                             num_nodes: Optional[int] = None) -> Tuple[Tensor, Optional[Tensor]]:
    """Mirror of utils/loop.py:585-657 for 1-D edge weights and a scalar fill_value."""
    if edge_attr is not None and edge_attr.dim() != 1:
        raise NotImplementedError("multi-dimensional edge_attr is not on the aggregation path")
    if isinstance(fill_value, (str, Tensor)):
        raise NotImplementedError("only scalar fill_value is supported")
    N = num_nodes if num_nodes is not None else ((ops.index_stats(edge_index.reshape(-1))[1] + 1)
                                                  if edge_index.numel() else 0)
    r, c, w = ops.self_loops(edge_index[0], edge_index[1], edge_attr, N, 1.0 if fill_value is None else fill_value, 0)
    return torch.stack([r, c]), w


def remove_then_add_self_loops(edge_index: Tensor, num_nodes: int) -> Tensor:
    """remove_self_loops + add_self_loops as GATConv does (gat_conv.py:342-346)."""
    r, c, _ = ops.self_loops(edge_index[0], edge_index[1], None, num_nodes, 1.0, 1)
    return torch.stack([r, c])


def gcn_norm(edge_index: Tensor, edge_weight: Optional[Tensor] = None, num_nodes: Optional[int] = None,
             improved: bool = False, add_self_loops: bool = True, flow: str = "source_to_target",
             dtype: Optional[torch.dtype] = None) -> Tuple[Tensor, Tensor]:
    """Mirror of nn/conv/gcn_conv.py:45-113 for [2,E] tensors: returns (edge_index', weights') in
    the reference's edge order.  GCNConv itself uses `gcn_norm_graph`, which keeps everything in
    CSR order and never materialises this pair."""
    g, ei = gcn_norm_graph(edge_index, edge_weight, num_nodes, improved, add_self_loops, flow, return_edge_index=True)
    return ei, g.from_csr_order(g.val)


def gcn_norm_graph(edge_index: Tensor, edge_weight: Optional[Tensor] = None, num_nodes: Optional[int] = None,
                   improved: bool = False, add_self_loops: bool = True, flow: str = "source_to_target",
                   return_edge_index: bool = False, chunk: Optional[int] = None):
    """gcn_norm + CSR build in one go: self-loop insertion (reference order), stable sort by
    destination, in-order weighted degree, D^-1/2 A D^-1/2 weights stored in CSR order."""
    assert flow in ("source_to_target", "target_to_source")
    if edge_weight is not None and edge_weight.requires_grad:
        raise NotImplementedError("gcn_norm with edge_weight.requires_grad is not supported by the fused path")
    N = num_nodes if num_nodes is not None else ((ops.index_stats(edge_index.reshape(-1))[1] + 1)
                                                  if edge_index.numel() else 0)
    row, col, w = edge_index[0], edge_index[1], edge_weight
    if add_self_loops:
        row, col, w = ops.self_loops(row, col, w, N, 2.0 if improved else 1.0, 0)
    src, dst = (row, col) if flow == "source_to_target" else (col, row)
    kw = {} if chunk is None else {"chunk": chunk}
    g = CSRGraph(src, dst, N, N, None, **kw)
    g.one_self_loop_per_row = add_self_loops      # self_loops drops the graph's own loops and adds one per node
    # deg is summed over `col` for source_to_target, `row` otherwise == the aggregation target
    w_csr = None if w is None else g.to_csr_order(w.float())
    _, w_norm = ops.gcn_norm_csr(g.rowptr, g.col, w_csr)
    g.val = w_norm
    if return_edge_index:
        return g, torch.stack([row, col])
    return g


def spmm(src: Union[CSRGraph, Tensor], other: Tensor, reduce: str = "sum") -> Tensor:
    """Mirror of torch_geometric.utils.spmm (utils/_spmm.py:12-136): `src` is a CSRGraph
    (the engine's adjacency handle) or a torch.sparse CSR tensor whose rows are destinations."""
    reduce = "sum" if reduce == "add" else reduce
    if reduce not in ("sum", "mean", "min", "max"):
        raise ValueError(f"`reduce` argument '{reduce}' not supported")
    if isinstance(src, CSRGraph):
        return Fn.aggregate(src, other, reduce)
    if isinstance(src, Tensor) and src.layout == torch.sparse_csr:
        rowptr, col, val = src.crow_indices(), src.col_indices(), src.values()
        n_rows = src.size(0)
        if other.requires_grad or val.requires_grad:
            raise NotImplementedError("pass a CSRGraph for a differentiable spmm")
        return ops.spmm_csr(rowptr, col, val.float(), other, n_rows, reduce)
    raise ValueError("`src` must be a CSRGraph or a torch.sparse_csr tensor")
