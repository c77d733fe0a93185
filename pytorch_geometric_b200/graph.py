"""CSRGraph -- the engine's cached graph structure for one edge set.

Plays the role of the reference's `EdgeIndex` caches (`_indptr`, `_T_perm`, `_T_index`,
`_T_indptr`, `_value`; torch_geometric/edge_index.py:237-246, get_csr/get_csc :626-696) and of a
`torch_sparse.SparseTensor` `adj_t` (rowptr/col/value + csr2csc): a destination-sorted CSR used
by the forward gather-reduce and, built lazily, the source-sorted CSR used by the backward.

HBM layout (DESIGN.md section 3): int32 `rowptr`/`col` whenever #nodes and #edges < 2^31 (the
reference keeps int64), fp32 edge values in CSR order, an int32 `perm` (CSR slot -> original edge
id) so per-edge tensors given in the caller's order can be permuted once.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from . import ops

DEFAULT_CHUNK = 512  # edges per long-row chunk (rows above this are split, see csr_reduce.cuh)
_INT32_MAX = 2**31 - 1


class CSRGraph:
    # Every destination row i holds exactly one edge i -> i (so does every row of the transposed CSR).  Set only by
    # utils.gcn_norm_graph with self-loops added; a graph built, adopted or narrowed any other way leaves it False.
    one_self_loop_per_row = False

    def __init__(self, src: Tensor, dst: Tensor, num_src: int, num_dst: int,
                 edge_weight: Optional[Tensor] = None, chunk: int = DEFAULT_CHUNK,
                 idx_dtype: Optional[torch.dtype] = None):
        if not src.is_cuda:
            raise RuntimeError("CSRGraph lives on a CUDA device (no CPU fallback)")
        E = src.numel()
        if idx_dtype is None:
            idx_dtype = torch.int32 if max(num_src, num_dst, E) < _INT32_MAX else torch.int64
        self.idx_dtype = idx_dtype
        self.num_src, self.num_dst, self.num_edges = int(num_src), int(num_dst), int(E)
        self.chunk = int(chunk)
        self.device = src.device
        self._src = ops.convert_index(src.contiguous(), idx_dtype)   # original edge order
        self._dst = ops.convert_index(dst.contiguous(), idx_dtype)
        # forward structure: stable sort by destination
        _, self.perm, self.rowptr = ops.sort_by_key(self._dst, self.num_dst, want_sorted=False)
        self.col = ops.permute(self._src, self.perm)
        self.val = None if edge_weight is None else ops.permute(edge_weight.detach().float().contiguous(), self.perm)
        self.plan = ops.LongRowPlan(self.rowptr, self.chunk)
        # backward structure (lazy)
        self._t_built = False
        self.perm_t = self.rowptr_t = self.col_t = self.val_t = self.plan_t = None
        self._mean_val_t = None
        self._inv_perm = None
        self._inv_perm_t = None
        self._dst_csr = None
        self._t2csr = None

    # ------------------------------------------------------------------ constructors
    @classmethod
    def from_edge_index(cls, edge_index: Tensor, num_nodes: Optional[int] = None,
                        edge_weight: Optional[Tensor] = None, num_src: Optional[int] = None,
                        num_dst: Optional[int] = None, **kw) -> "CSRGraph":
        """edge_index[0] = source (j), edge_index[1] = destination (i): flow source_to_target
        (message_passing.py:31 / collect.jinja:67-68)."""
        if edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError("edge_index must have shape [2, E]")
        if num_nodes is None and (num_src is None or num_dst is None):
            _, mx, _ = ops.index_stats(edge_index.reshape(-1)) if edge_index.numel() else (0, -1, True)
            num_nodes = mx + 1   # maybe_num_nodes (utils/num_nodes.py:12-40): a D2H sync, as in the reference
        return cls(edge_index[0], edge_index[1], num_src if num_src is not None else num_nodes,
                   num_dst if num_dst is not None else num_nodes, edge_weight, **kw)

    @classmethod
    def from_csr(cls, rowptr: Tensor, col: Tensor, num_src: int, edge_weight: Optional[Tensor] = None,
                 transposed: Optional[tuple] = None, chunk: int = DEFAULT_CHUNK,
                 idx_dtype: Optional[torch.dtype] = None, bounded_degree: bool = False) -> "CSRGraph":
        """Adopts an EXISTING destination-sorted CSR -- an `EdgeIndex`'s cached `(indptr, other index)`
        (edge_index.py:626-696), a `torch.sparse_csr` tensor's `(crow_indices, col_indices)`, a loader's `ptr` --
        without sorting anything: the caller's edge order IS the CSR order (`perm` = identity, stored as None).
        `transposed` = (rowptr_t, col_t, perm_t) adopts the cached transposed structure as well (the reference's
        `_T_indptr`, `_T_index`, `_T_perm`), otherwise it is built on first use by one stable sort.
        Indices are converted to int32 once when everything fits (a streaming pass, not a sort)."""
        if not rowptr.is_cuda:
            raise RuntimeError("CSRGraph lives on a CUDA device (no CPU fallback)")
        g = object.__new__(cls)
        E, n_dst = col.numel(), rowptr.numel() - 1
        if idx_dtype is None:
            idx_dtype = torch.int32 if max(num_src, n_dst, E) < _INT32_MAX else torch.int64
        g.idx_dtype = idx_dtype
        g.num_src, g.num_dst, g.num_edges = int(num_src), int(n_dst), int(E)
        g.chunk, g.device = int(chunk), rowptr.device
        g.rowptr = ops.convert_index(rowptr.contiguous(), idx_dtype)
        g.col = ops.convert_index(col.contiguous(), idx_dtype)
        g.perm = None
        g._src, g._dst = g.col, None                          # _dst = ptr2index(rowptr), materialised on demand
        g.val = None if edge_weight is None else edge_weight.detach().float().contiguous()
        # bounded_degree: the caller guarantees short rows (sampled mini-batches): no long-row count, no host sync
        g._bounded = bool(bounded_degree)
        g.plan = ops.LongRowPlan.empty(g.chunk) if bounded_degree else ops.LongRowPlan(g.rowptr, g.chunk)
        g._t_built = False
        g.perm_t = g.rowptr_t = g.col_t = g.val_t = g.plan_t = None
        g._mean_val_t = g._inv_perm = g._inv_perm_t = g._dst_csr = g._t2csr = None
        if transposed is not None:
            rowptr_t, col_t, perm_t = transposed
            g.rowptr_t = ops.convert_index(rowptr_t.contiguous(), idx_dtype)
            g.col_t = ops.convert_index(col_t.contiguous(), idx_dtype)
            g.perm_t = ops.convert_index(perm_t.contiguous(), idx_dtype)
            g.plan_t = ops.LongRowPlan(g.rowptr_t, g.chunk)
            g._t_built = True
            if g.val is not None:
                g.val_t = ops.permute(g.val, g.perm_t)
        return g

    # ------------------------------------------------------------------ transposed structure
    def build_transpose(self) -> None:
        if self._t_built:
            return
        if self._dst is None:
            self._dst = self.dst_csr
        _, self.perm_t, self.rowptr_t = ops.sort_by_key(self._src, self.num_src, want_sorted=False)
        self.col_t = ops.permute(self._dst, self.perm_t)
        self.plan_t = ops.LongRowPlan(self.rowptr_t, self.chunk)          # (source hubs exist even in sampled batches)
        self._t_built = True
        if self.val is not None:
            self.val_t = self.to_csc_order(self.from_csr_order(self.val))

    def trim(self, num_dst: int, num_src: int, num_edges: int) -> "CSRGraph":
        """The sub-graph of the first `num_dst` destination rows, `num_src` sources and `num_edges` CSR slots, as
        VIEWS of this graph's arrays -- `trim_to_layer` (utils/_trim_to_layer.py:20-217) for a destination-sorted
        sampled subgraph: NeighborLoader emits the hops in BFS order, so the nodes and edges a deeper layer no
        longer needs are exactly the tails of the node / CSR arrays.  No sort, no edge copy, no host sync.
        Requires an adopted CSR (caller's edge order == CSR order)."""
        if self.perm is not None:
            raise ValueError("trim() needs a graph adopted with from_csr (edge order == CSR order)")
        if not (0 <= num_dst <= self.num_dst and 0 <= num_src <= self.num_src and 0 <= num_edges <= self.num_edges):
            raise ValueError("trim(): sizes must not exceed the graph's")
        g = object.__new__(CSRGraph)
        g.idx_dtype, g.chunk, g.device = self.idx_dtype, self.chunk, self.device
        g.num_src, g.num_dst, g.num_edges = int(num_src), int(num_dst), int(num_edges)
        # rows whose in-edges all lie in the dropped tail (the previous hop's frontier: sources only from now on) must
        # end at num_edges: one clamp over the [num_dst + 1] row pointers (the edge arrays stay views)
        g.rowptr = self.rowptr[:num_dst + 1].clamp(max=num_edges)
        g.col = self.col[:num_edges]
        g.perm = None
        g._src, g._dst = g.col, None
        g.val = None if self.val is None else self.val[:num_edges]
        g._bounded = getattr(self, "_bounded", False)
        g.plan = ops.LongRowPlan.empty(g.chunk) if g._bounded else ops.LongRowPlan(g.rowptr, g.chunk)
        g._t_built = False
        g.perm_t = g.rowptr_t = g.col_t = g.val_t = g.plan_t = None
        g._mean_val_t = g._inv_perm = g._inv_perm_t = g._dst_csr = g._t2csr = None
        return g

    # per-edge tensor permutations (1-D fp32 / int tensors)
    def to_csr_order(self, per_edge: Tensor) -> Tensor:
        if self.perm is None:                                   # adopted CSR: the caller's order is the CSR order
            return per_edge.contiguous()
        return ops.permute(per_edge.contiguous(), self.perm)

    def to_csc_order(self, per_edge: Tensor) -> Tensor:
        self.build_transpose()
        return ops.permute(per_edge.contiguous(), self.perm_t)

    def _inverse(self, perm: Tensor) -> Tensor:
        inv = torch.empty_like(perm)
        inv[perm.long()] = torch.arange(perm.numel(), device=perm.device, dtype=perm.dtype)
        return inv

    def from_csr_order(self, per_edge_csr: Tensor) -> Tensor:
        if self.perm is None:
            return per_edge_csr.contiguous()
        if self._inv_perm is None:
            self._inv_perm = self._inverse(self.perm)
        return ops.permute(per_edge_csr.contiguous(), self._inv_perm)

    def from_csc_order(self, per_edge_csc: Tensor) -> Tensor:
        self.build_transpose()
        if self._inv_perm_t is None:
            self._inv_perm_t = self._inverse(self.perm_t)
        return ops.permute(per_edge_csc.contiguous(), self._inv_perm_t)

    def to_csr_order_rows(self, per_edge: Tensor) -> Tensor:
        """[E, k] per-edge rows (caller's edge order) -> CSR order."""
        if self.perm is None:
            return per_edge.contiguous()
        return ops.gather_rows(per_edge.contiguous(), self.perm)

    def from_csr_order_rows(self, per_edge_csr: Tensor) -> Tensor:
        if self.perm is None:
            return per_edge_csr.contiguous()
        if self._inv_perm is None:
            self._inv_perm = self._inverse(self.perm)
        return ops.gather_rows(per_edge_csr.contiguous(), self._inv_perm)

    @property
    def t2csr(self) -> Tensor:
        """CSR slot of every transposed-CSR slot (the reference's csr2csc / _T_perm role)."""
        if getattr(self, "_t2csr", None) is None:
            self.build_transpose()
            if self.perm is None:                                # CSR slot == caller's edge id
                self._t2csr = self.perm_t
            else:
                if self._inv_perm is None:
                    self._inv_perm = self._inverse(self.perm)
                self._t2csr = ops.permute(self._inv_perm, self.perm_t)
        return self._t2csr

    @property
    def dst_csr(self) -> Tensor:
        """destination of every CSR slot (ptr2index of rowptr)."""
        if self._dst_csr is None:
            self._dst_csr = ops.ptr2index(self.rowptr, self.num_edges)
        return self._dst_csr

    def in_degree(self) -> Tensor:
        return self.rowptr[1:] - self.rowptr[:-1]

    def mean_val_t(self) -> Tensor:
        """1 / max(in_degree(dst), 1) per transposed-CSR slot: backward weights of 'mean'."""
        if self._mean_val_t is None:
            self.build_transpose()
            inv = 1.0 / self.in_degree().clamp(min=1).to(torch.float32)
            self._mean_val_t = ops.gather_rows(inv.view(-1, 1), self.col_t).view(-1)
        return self._mean_val_t

    def with_values(self, val_csr: Optional[Tensor]) -> "CSRGraph":
        """Shallow copy sharing the structure but carrying different (static) CSR-ordered values."""
        g = object.__new__(CSRGraph)
        g.__dict__.update(self.__dict__)
        g.val = val_csr
        g.val_t = None
        if val_csr is not None and self._t_built:
            g.val_t = g.to_csc_order(g.from_csr_order(val_csr))
        return g

    def nbytes(self) -> int:
        n = 0
        for t in (self.rowptr, self.col, self.perm, self.val, self.rowptr_t, self.col_t, self.perm_t, self.val_t,
                  self._src, self._dst):
            if t is not None:
                n += t.numel() * t.element_size()
        return n

    def __repr__(self) -> str:
        return (f"CSRGraph(num_src={self.num_src}, num_dst={self.num_dst}, num_edges={self.num_edges}, "
                f"idx={self.idx_dtype}, long_rows={self.plan.n_long}, chunks={self.plan.n_chunks})")


# ---------------------------------------------------------------------------------------------- graphs cached by tensor identity
_GRAPH_CACHE: "dict" = {}
_GRAPH_CACHE_EDGES = 600_000_000        # evict oldest entries above this many cached edges


def _cache_put(key, holders, graph) -> None:
    _GRAPH_CACHE[key] = (holders, graph)
    total = sum(g.num_edges for _, g in _GRAPH_CACHE.values())
    while total > _GRAPH_CACHE_EDGES and len(_GRAPH_CACHE) > 1:
        k0 = next(iter(_GRAPH_CACHE))
        total -= _GRAPH_CACHE.pop(k0)[1].num_edges


def cached_graph(edge_index: Tensor, num_src: int, num_dst: int, flow: str = "source_to_target", loops: Optional[str] = None,
                 loop_nodes: Optional[int] = None, edge_type: Optional[Tensor] = None,
                 num_relations: Optional[int] = None) -> CSRGraph:
    """The CSRGraph of a `[2, E]` edge_index, built once per tensor (storage pointer + length + version counter; the
    cache entry keeps the tensor alive so the pointer cannot be reused) -- what `cached=True` does for GCNConv in the
    reference (gcn_conv.py:150-158), for every layer.  loops='gat': remove_self_loops + add_self_loops for the first
    `loop_nodes` nodes (gat_conv.py:334-346).  edge_type / num_relations: the relational graph of RGCNConv, keyed by
    the virtual destination dst * R + type."""
    if edge_index.dim() != 2 or edge_index.size(0) != 2:
        raise ValueError("edge_index must have shape [2, E]")
    key = (edge_index.data_ptr(), edge_index.numel(), edge_index._version, int(num_src), int(num_dst), flow, loops, loop_nodes,
           None if edge_type is None else (edge_type.data_ptr(), edge_type._version), num_relations)
    hit = _GRAPH_CACHE.get(key)
    if hit is not None:
        return hit[1]
    ei = edge_index
    if loops == "gat":
        from . import utils as U
        ei = U.remove_then_add_self_loops(edge_index, int(loop_nodes if loop_nodes is not None else min(num_src, num_dst)))
    src, dst = (ei[0], ei[1]) if flow == "source_to_target" else (ei[1], ei[0])
    if edge_type is not None:
        dst = dst.to(torch.int64) * int(num_relations) + edge_type.to(torch.int64)
    g = CSRGraph(src, dst, num_src, num_dst)
    _cache_put(key, (edge_index, edge_type), g)
    return g


def clear_graph_cache() -> None:
    _GRAPH_CACHE.clear()
