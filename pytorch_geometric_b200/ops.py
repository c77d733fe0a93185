"""Tensor-level wrappers over the C ABI (include/b200mp.h).  No autograd here (see functional.py).

PyTorch is used for device memory (the caching allocator owns every buffer) and the current
stream; all arithmetic happens in libb200mp.so.  Every function refuses non-CUDA tensors: there is
no CPU fallback.
"""
from __future__ import annotations

import ctypes
import math
from collections import OrderedDict
from typing import Optional, Tuple

import torch
from torch import Tensor

from ._lib import check, lib

F32, BF16, F64 = 0, 1, 2
I32, I64 = 0, 1
REDUCE = {"sum": 0, "add": 0, "mean": 1, "min": 2, "amin": 2, "max": 3, "amax": 3, "mul": 4}


class _Launches:
    """Number of engine kernels launched so far (bench.py reports the delta as gpu_launches)."""
    count = 0


LAUNCHES = _Launches()


class _Profile:
    """Optional per-op CUDA-event timing on the launching stream (bench.py's roofline numbers).
    Disabled by default: zero overhead on the product path."""

    def __init__(self):
        self.enabled = False
        self.events = {}

    def reset(self, enabled: bool = False):
        self.enabled = enabled
        self.events = {}

    def begin(self, name: str):
        if not self.enabled:
            return None
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        self.events.setdefault(name, []).append((e0, e1))
        return e1

    def summary(self) -> dict:
        torch.cuda.synchronize()
        out = {}
        for k, v in self.events.items():
            each = [a.elapsed_time(b) for a, b in v]
            out[k] = {"ms_total": sum(each), "calls": len(each), "ms_each": each}
        return out


PROFILE = _Profile()


def _timed(name: str, n_kernels: int, fn, *args):
    LAUNCHES.count += n_kernels
    end = PROFILE.begin(name)
    rc = fn(*args)
    if end is not None:
        end.record()
    check(rc, name)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


def _cuda(*ts: Optional[Tensor]) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("pytorch_geometric_b200 ops run on CUDA tensors only (no CPU fallback); "
                               f"got a tensor on {t.device}")


def _idt(t: Tensor) -> int:
    if t.dtype == torch.int32:
        return I32
    if t.dtype == torch.int64:
        return I64
    raise TypeError(f"index tensors must be int32 or int64, got {t.dtype}")


def _vdt(t: Tensor) -> int:
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"feature tensors must be float32 or bfloat16, got {t.dtype}")


def _same_idx(*ts: Optional[Tensor]) -> int:
    ds = {t.dtype for t in ts if t is not None}
    if len(ds) != 1:
        raise TypeError(f"index tensors of one call must share a dtype, got {ds}")
    return _idt(next(t for t in ts if t is not None))


def _ws(nbytes: int, device) -> Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


# ------------------------------------------------------------------ structure
def degree(index: Tensor, num_nodes: int) -> Tensor:
    _cuda(index)
    index = index.contiguous()
    deg = torch.empty(num_nodes, dtype=index.dtype, device=index.device)
    check(lib().b200mp_degree(_p(index), index.numel(), num_nodes, _p(deg), _idt(index), _stream()), "degree")
    return deg


def index2ptr(index: Tensor, size: int) -> Tensor:
    _cuda(index)
    index = index.contiguous()
    ptr = torch.empty(size + 1, dtype=index.dtype, device=index.device)
    check(lib().b200mp_index2ptr(_p(index), index.numel(), size, _p(ptr), _idt(index), _stream()), "index2ptr")
    return ptr


def ptr2index(ptr: Tensor, output_size: Optional[int] = None) -> Tensor:
    _cuda(ptr)
    ptr = ptr.contiguous()
    n = int(ptr[-1]) if output_size is None else int(output_size)
    index = torch.empty(n, dtype=ptr.dtype, device=ptr.device)
    check(lib().b200mp_ptr2index(_p(ptr), ptr.numel() - 1, n, _p(index), _idt(ptr), _stream()), "ptr2index")
    return index


def index_stats(index: Tensor) -> Tuple[int, int, bool]:
    """(min, max, is_sorted) of an index tensor -- one kernel + one D2H read."""
    _cuda(index)
    index = index.contiguous()
    st = torch.empty(3, dtype=torch.int64, device=index.device)
    check(lib().b200mp_index_stats(_p(index), index.numel(), _p(st), _idt(index), _stream()), "index_stats")
    mn, mx, srt = st.tolist()
    return mn, mx, bool(srt)


def sort_by_key(keys: Tensor, num_nodes: int, want_sorted: bool = True,
                want_ptr: bool = True) -> Tuple[Optional[Tensor], Tensor, Optional[Tensor]]:
    """Stable sort of keys in [0, num_nodes): (keys_sorted, perm, ptr)."""
    _cuda(keys)
    keys = keys.contiguous()
    n = keys.numel()
    it = _idt(keys)
    ws = _ws(lib().b200mp_sort_workspace_bytes(n, num_nodes, it), keys.device)
    ks = torch.empty_like(keys) if want_sorted else None
    perm = torch.empty_like(keys)
    ptr = torch.empty(num_nodes + 1, dtype=keys.dtype, device=keys.device) if want_ptr else None
    check(lib().b200mp_sort_by_key(_p(keys), n, num_nodes, _p(ks), _p(perm), _p(ptr), _p(ws), ws.numel(), it,
                                   _stream()), "sort_by_key")
    return ks, perm, ptr


def permute(src: Tensor, perm: Tensor) -> Tensor:
    """out[i] = src[perm[i]] for 1-D tensors of 4- or 8-byte elements."""
    _cuda(src, perm)
    src, perm = src.contiguous(), perm.contiguous()
    out = torch.empty(perm.numel(), dtype=src.dtype, device=src.device)
    check(lib().b200mp_permute(_p(src), _p(perm), _p(out), perm.numel(), src.element_size(), _idt(perm),
                               _stream()), "permute")
    return out


def convert_index(index: Tensor, dtype: torch.dtype) -> Tensor:
    _cuda(index)
    if index.dtype == dtype:
        return index
    index = index.contiguous()
    out = torch.empty(index.shape, dtype=dtype, device=index.device)
    check(lib().b200mp_convert_index(_p(index), _idt(index), _p(out), _idt(out), index.numel(), _stream()),
          "convert_index")
    return out


def self_loops(row: Tensor, col: Tensor, weight: Optional[Tensor], num_nodes: int, fill_value: float = 1.0,
               mode: int = 0) -> Tuple[Tensor, Tensor, Optional[Tensor]]:
    """mode 0: add_remaining_self_loops; mode 1: remove_self_loops + add_self_loops."""
    _cuda(row, col, weight)
    row, col = row.contiguous(), col.contiguous()
    it = _same_idx(row, col)
    E = row.numel()
    if weight is not None:
        weight = weight.contiguous().float()
    ws = _ws(lib().b200mp_self_loops_workspace_bytes(E, num_nodes, it), row.device)
    r2 = torch.empty(E + num_nodes, dtype=row.dtype, device=row.device)
    c2 = torch.empty_like(r2)
    w2 = torch.empty(E + num_nodes, dtype=torch.float32, device=row.device) if weight is not None else None
    n_out = torch.empty(1, dtype=torch.int64, device=row.device)
    check(lib().b200mp_self_loops(_p(row), _p(col), _p(weight), E, num_nodes, float(fill_value), mode, _p(r2),
                                  _p(c2), _p(w2), _p(n_out), _p(ws), ws.numel(), it, _stream()), "self_loops")
    n = int(n_out.item())  # one D2H sync, as the reference's boolean-mask indexing has
    return r2[:n], c2[:n], (w2[:n] if w2 is not None else None)


def gcn_norm_csr(rowptr: Tensor, src: Tensor, weight: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """(deg_inv_sqrt [N], normalised weights [E]) on a destination-sorted CSR."""
    _cuda(rowptr, src, weight)
    it = _same_idx(rowptr, src)
    N, E = rowptr.numel() - 1, src.numel()
    dinv = torch.empty(N, dtype=torch.float32, device=rowptr.device)
    w_out = torch.empty(E, dtype=torch.float32, device=rowptr.device)
    check(lib().b200mp_gcn_norm_csr(_p(rowptr), _p(src), _p(weight), N, E, _p(dinv), _p(w_out), it, _stream()),
          "gcn_norm_csr")
    return dinv, w_out


class LongRowPlan:
    """Rows with more than `chunk` edges, cut into chunks (b200mp_csr_plan_*)."""

    __slots__ = ("long_rows", "chunk_ptr", "n_long", "n_chunks", "chunk", "_partials")

    def __init__(self, rowptr: Tensor, chunk: int):
        _cuda(rowptr)
        it = _idt(rowptr)
        n_rows = rowptr.numel() - 1
        counts = torch.empty(2, dtype=torch.int64, device=rowptr.device)
        check(lib().b200mp_csr_plan_count(_p(rowptr), n_rows, chunk, _p(counts), it, _stream()), "csr_plan_count")
        self.n_long, self.n_chunks = (int(v) for v in counts.tolist())
        self.chunk = int(chunk)
        self.long_rows = self.chunk_ptr = None
        self._partials = None
        if self.n_long:
            self.long_rows = torch.empty(self.n_long, dtype=torch.int64, device=rowptr.device)
            self.chunk_ptr = torch.empty(self.n_long + 1, dtype=torch.int64, device=rowptr.device)
            ws = _ws(lib().b200mp_csr_plan_workspace_bytes(n_rows, self.n_long, it), rowptr.device)
            check(lib().b200mp_csr_plan_fill(_p(rowptr), n_rows, chunk, self.n_long, _p(self.long_rows),
                                             _p(self.chunk_ptr), _p(ws), ws.numel(), it, _stream()),
                  "csr_plan_fill")

    @classmethod
    def empty(cls, chunk: int = 512) -> "LongRowPlan":
        """A plan without long rows, built WITHOUT the device->host count: always correct (a row above `chunk` edges
        is then simply walked by one lane group), meant for graphs whose degrees are bounded by construction
        (neighbour-sampled mini-batches: degree <= fan-out)."""
        p = object.__new__(cls)
        p.n_long = p.n_chunks = 0
        p.chunk = int(chunk)
        p.long_rows = p.chunk_ptr = p._partials = None
        return p

    def partials(self, feat: int, device) -> Optional[Tensor]:
        if not self.n_long:
            return None
        need = self.n_chunks * feat
        if self._partials is None or self._partials.numel() < need:
            self._partials = torch.empty(need, dtype=torch.float32, device=device)
        return self._partials


# ------------------------------------------------------------------ the hot path
def spmm_csr(rowptr: Tensor, col: Tensor, val: Optional[Tensor], x: Tensor, n_rows: int, reduce: str = "sum",
             plan: Optional[LongRowPlan] = None, out: Optional[Tensor] = None,
             bias: Optional[Tensor] = None, x_halo: Optional[Tensor] = None, accumulate: bool = False,
             peer_ptrs: Optional[int] = None, peer_rows: int = 0, relu_mask: Optional[Tensor] = None) -> Tensor:
    """out[i,:] = REDUCE_{e in row i} val[e] * x[col[e],:] (+ bias)  (x: [n_cols, F] contiguous)."""
    _cuda(rowptr, col, val, x)
    if x.dim() != 2:
        raise ValueError("spmm_csr expects a 2-D feature matrix")
    x = x.contiguous()
    it = _same_idx(rowptr, col)
    if val is not None and (val.dtype != torch.float32 or not val.is_contiguous()):
        val = val.contiguous().float()
    F = x.size(1)
    if out is None:
        out = torch.empty(n_rows, F, dtype=x.dtype, device=x.device)
    if plan is not None and plan.n_long:
        part = plan.partials(F, x.device)
        args = (_p(plan.long_rows), _p(plan.chunk_ptr), plan.n_long, plan.n_chunks, plan.chunk, _p(part))
    else:
        args = (None, None, 0, 0, 0, None)
    if bias is not None:
        _cuda(bias)
        if bias.dtype != torch.float32 or not bias.is_contiguous():
            bias = bias.detach().float().contiguous()
        if bias.numel() != F:
            raise ValueError("bias must have one entry per feature")
    if relu_mask is not None:
        _cuda(relu_mask)
        if not accumulate or relu_mask.dtype != x.dtype or tuple(relu_mask.shape) != (n_rows, F) or not relu_mask.is_contiguous():
            raise ValueError("relu_mask needs accumulate=True and a contiguous [n_rows, F] tensor of x's dtype")
    n_cols, n_local = x.size(0), 0
    if x_halo is not None:
        _cuda(x_halo)
        if x_halo.dtype != x.dtype or x_halo.dim() != 2 or x_halo.size(1) != F or not x_halo.is_contiguous():
            raise ValueError("x_halo must be a contiguous [n_halo, F] tensor of x's dtype")
        n_local, n_cols = x.size(0), x.size(0) + x_halo.size(0)
    _timed("spmm_csr", 2 if args[2] else 1, lib().b200mp_spmm_csr, _p(rowptr), _p(col), _p(val), _p(x), _p(out),
           n_rows, n_cols, F, REDUCE[reduce], *args, _p(bias), _p(x_halo), n_local, int(bool(accumulate)),
           peer_ptrs, int(peer_rows), _p(relu_mask), it, _vdt(x), _stream())
    return out


def spmm_csr_self_colsum(rowptr: Tensor, col: Tensor, val: Tensor, x: Tensor,
                         plan: Optional[LongRowPlan] = None) -> Tuple[Tensor, Tensor]:
    """(spmm_csr(rowptr, col, val, x, N, "sum", plan), x.sum(0) in fp32) for a square graph whose every row i holds
    exactly one edge i -> i (CSRGraph.one_self_loop_per_row): the column sum is taken from the self-loop rows the
    sweep already loads, not from a second pass over x (b200mp_spmm_csr_self_colsum)."""
    _cuda(rowptr, col, val, x)
    if x.dim() != 2 or x.size(0) != rowptr.numel() - 1:
        raise ValueError("spmm_csr_self_colsum expects a square graph and an [N, F] feature matrix")
    x = x.contiguous()
    it = _same_idx(rowptr, col)
    val = val.contiguous().float()
    n, F = x.shape
    out = torch.empty(n, F, dtype=x.dtype, device=x.device)
    colsum = torch.empty(F, dtype=torch.float32, device=x.device)
    # one fp32 partial row per CTA: 16 resident 128-thread CTAs per SM at most
    parts = 16 * torch.cuda.get_device_properties(x.device).multi_processor_count
    ws = torch.empty(parts * max(F, 1), dtype=torch.float32, device=x.device)
    if plan is not None and plan.n_long:
        args = (_p(plan.long_rows), _p(plan.chunk_ptr), plan.n_long, plan.n_chunks, plan.chunk, _p(plan.partials(F, x.device)))
    else:
        args = (None, None, 0, 0, 0, None)
    _timed("spmm_csr", 3 if args[2] else 2, lib().b200mp_spmm_csr_self_colsum, _p(rowptr), _p(col), _p(val), _p(x),
           _p(out), _p(colsum), n, F, *args, _p(ws), parts, it, _vdt(x), _stream())
    return out, colsum


SEGMENT_PLAN_MIN_ROWS = 1 << 16   # below this many source rows a hub segment cannot matter: skip the plan (and its sync)
SEGMENT_CHUNK = 512               # rows per chunk of a long segment (same as graph.DEFAULT_CHUNK)


_PLAN_CACHE: "dict" = {}            # id(ptr) -> (weakref(ptr), version, plan or None)
_PLAN_CACHE_MAX = 32


def segment_plan(ptr: Tensor, n_src: int) -> Optional["LongRowPlan"]:
    """Long-segment plan for segment_csr / multi_aggr_csr (None when the input is too small to need one).
    Counting the long segments needs one device->host read, so the plan is cached per `ptr` tensor OBJECT
    (weak reference + version counter): a layer that hands over the same ptr every step -- an EdgeIndex's
    cached indptr, a loader's batch ptr -- pays that read once and enqueues asynchronously afterwards."""
    if n_src < SEGMENT_PLAN_MIN_ROWS:
        return None
    import weakref
    key = id(ptr)
    hit = _PLAN_CACHE.get(key)
    if hit is not None and hit[0]() is ptr and hit[1] == ptr._version:
        return hit[2]
    plan = LongRowPlan(ptr, SEGMENT_CHUNK)
    plan = plan if plan.n_long else None
    if len(_PLAN_CACHE) >= _PLAN_CACHE_MAX:
        for k in [k for k, v in _PLAN_CACHE.items() if v[0]() is None] or list(_PLAN_CACHE)[:1]:
            _PLAN_CACHE.pop(k, None)
    try:
        _PLAN_CACHE[key] = (weakref.ref(ptr), ptr._version, plan)
    except TypeError:
        pass
    return plan


def segment_csr(src: Tensor, ptr: Tensor, reduce: str = "sum", plan: Optional["LongRowPlan"] = None) -> Tensor:
    _cuda(src, ptr)
    src = src.contiguous()
    n_rows = ptr.numel() - 1
    flat = src.view(src.size(0), -1)
    out = torch.empty((n_rows, flat.size(1)), dtype=src.dtype, device=src.device)
    pargs, _ = _plan_args(plan, flat.size(1), src.device)
    _timed("segment_csr", 2 if pargs[2] else 1, lib().b200mp_segment_csr, _p(ptr), _p(flat), _p(out), n_rows,
           flat.size(0), flat.size(1), REDUCE[reduce], *pargs, _idt(ptr), _vdt(src), _stream())
    return out.view((n_rows, ) + tuple(src.shape[1:]))


def minmax_ties(rowptr: Tensor, col: Tensor, val: Optional[Tensor], x: Tensor, out: Tensor,
                count_self_zero: bool = True) -> Tensor:
    _cuda(rowptr, col, val, x, out)
    it = _same_idx(rowptr, col)
    ties = torch.empty(out.shape, dtype=torch.float32, device=out.device)
    check(lib().b200mp_minmax_ties(_p(rowptr), _p(col), _p(val), _p(x), _p(out), _p(ties), out.size(0),
                                   out.size(1), int(count_self_zero), it, _vdt(x), _stream()), "minmax_ties")
    return ties


def minmax_backward(rowptr_t: Tensor, col_t: Tensor, val_t: Optional[Tensor], x: Tensor, out: Tensor,
                    grad_out: Tensor, ties: Tensor) -> Tensor:
    _cuda(rowptr_t, col_t, val_t, x, out, grad_out, ties)
    it = _same_idx(rowptr_t, col_t)
    gx = torch.empty_like(x)
    check(lib().b200mp_minmax_backward(_p(rowptr_t), _p(col_t), _p(val_t), _p(x), _p(out), _p(grad_out),
                                       _p(ties), _p(gx), x.size(0), x.size(1), it, _vdt(x), _stream()),
          "minmax_backward")
    return gx


def sddmm_csr(rowptr: Tensor, col: Tensor, a: Tensor, b: Tensor) -> Tensor:
    """dot[e] = <a[row(e),:], b[col[e],:]> in CSR edge order."""
    _cuda(rowptr, col, a, b)
    it = _same_idx(rowptr, col)
    a, b = a.contiguous(), b.contiguous()
    dot = torch.empty(col.numel(), dtype=torch.float32, device=a.device)
    check(lib().b200mp_sddmm_csr(_p(rowptr), _p(col), _p(a), _p(b), _p(dot), rowptr.numel() - 1, a.size(1), it,
                                 _vdt(a), _stream()), "sddmm_csr")
    return dot


def edge_relu_csr(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], x: Tensor, edge_rows: Tensor, n_rows: int,
                  reduce: str = "sum", plan: Optional[LongRowPlan] = None,
                  want_mask: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """out[i,:] = REDUCE_{e in row i} relu(x[col[e],:] + edge_rows[perm[e],:]) for sum / mean, and (want_mask) the
    ReLU mask, [E, ceil(F / 8)] uint8 bits in CSR order.  edge_rows: [E, F] in the caller's edge order."""
    _cuda(rowptr, col, perm, x, edge_rows)
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"edge_relu_csr reduces by sum or mean, not '{reduce}'")
    x, edge_rows = x.contiguous(), edge_rows.contiguous()
    E, F = col.numel(), x.size(1)
    if edge_rows.dtype != x.dtype or tuple(edge_rows.shape) != (E, F):
        raise ValueError(f"edge_rows must be a [{E}, {F}] tensor of x's dtype, got {tuple(edge_rows.shape)} {edge_rows.dtype}")
    it = _same_idx(rowptr, col, perm)
    out = torch.empty(n_rows, F, dtype=x.dtype, device=x.device)
    mask = torch.empty(E, (F + 7) // 8, dtype=torch.uint8, device=x.device) if want_mask else None
    pargs, _ = _plan_args(plan, F, x.device)
    _timed("edge_relu_csr", 2 if pargs[2] else 1, lib().b200mp_edge_relu_csr, _p(rowptr), _p(col), _p(perm), _p(x),
           _p(edge_rows), _p(out), _p(mask), n_rows, x.size(0), E, F, REDUCE[reduce], *pargs, it, _vdt(x), _stream())
    return out, mask


def edge_relu_backward_x(rowptr_t: Tensor, col_t: Tensor, t2csr: Tensor, val_t: Optional[Tensor], grad_out: Tensor,
                         mask: Tensor, n_src: int, plan_t: Optional[LongRowPlan] = None) -> Tensor:
    """grad_x[j,:] = sum_{t in rowT(j)} mask(t2csr[t]) ? val_t[t] * grad_out[col_t[t],:] : 0 (transposed CSR)."""
    _cuda(rowptr_t, col_t, t2csr, val_t, grad_out, mask)
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr_t, col_t, t2csr)
    F = grad_out.size(1)
    grad_x = torch.empty(n_src, F, dtype=grad_out.dtype, device=grad_out.device)
    pargs, _ = _plan_args(plan_t, F, grad_out.device)
    _timed("edge_relu_backward_x", 2 if pargs[2] else 1, lib().b200mp_edge_relu_backward_x, _p(rowptr_t), _p(col_t),
           _p(t2csr), _p(val_t), _p(grad_out), _p(mask), _p(grad_x), n_src, F, *pargs, it, _vdt(grad_out), _stream())
    return grad_x


def edge_relu_backward_edge(rowptr: Tensor, perm: Optional[Tensor], grad_out: Tensor, mask: Tensor, n_edges: int,
                            reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> Tensor:
    """grad_edge_rows[perm[e],:] = mask(e) ? grad_out[row(e),:] (/ max(deg, 1) for mean) : 0, caller's edge order."""
    _cuda(rowptr, perm, grad_out, mask)
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr, perm)
    F = grad_out.size(1)
    grad = torch.empty(n_edges, F, dtype=grad_out.dtype, device=grad_out.device)
    if n_edges == 0:
        return grad
    pargs = _plan_rows(plan)
    _timed("edge_relu_backward_edge", 1, lib().b200mp_edge_relu_backward_edge, _p(rowptr), _p(perm), _p(grad_out),
           _p(mask), _p(grad), rowptr.numel() - 1, F, REDUCE[reduce], *pargs, it, _vdt(grad_out), _stream())
    return grad


def _gated_rows(k: Tensor, q: Tensor, v: Tensor) -> int:
    """Check the operands of the gated sweeps; returns the row stride `ld` that q and v (and their gradients) share."""
    F = k.size(1)
    if k.dim() != 2 or not k.is_contiguous():
        raise ValueError("k must be a contiguous 2-D tensor")
    for name, t in (("q", q), ("v", v)):
        if t.dim() != 2 or t.size(1) != F or t.dtype != k.dtype or (t.size(0) > 0 and t.stride(1) != 1):
            raise ValueError(f"{name} must be a [N, {F}] tensor of k's dtype with unit feature stride, "
                             f"got {tuple(t.shape)} {t.dtype}")
    if q.size(0) != v.size(0) or q.stride(0) != v.stride(0) or q.stride(0) < F:
        raise ValueError(f"q and v must have the same rows and one row stride >= {F}, got strides "
                         f"{q.stride()} and {v.stride()}")
    return q.stride(0)


def gated_csr(rowptr: Tensor, col: Tensor, k: Tensor, q: Tensor, v: Tensor, n_rows: int, reduce: str = "sum",
              plan: Optional[LongRowPlan] = None) -> Tensor:
    """out[i,:] = REDUCE_{e in row i} sigmoid(k[i,:] + q[col[e],:]) * v[col[e],:] for sum / mean.  k: [n_rows, F]
    contiguous; q, v: [n_src, F] rows sharing one row stride (two tensors, or the halves of one [n_src, 2F])."""
    _cuda(rowptr, col, k, q, v)
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"gated_csr reduces by sum or mean, not '{reduce}'")
    ld = _gated_rows(k, q, v)
    it = _same_idx(rowptr, col)
    F = k.size(1)
    out = torch.empty(n_rows, F, dtype=k.dtype, device=k.device)
    pargs, _ = _plan_args(plan, F, k.device)
    _timed("gated_csr", 2 if pargs[2] else 1, lib().b200mp_gated_csr, _p(rowptr), _p(col), _p(k), _p(q), _p(v),
           _p(out), n_rows, q.size(0), col.numel(), F, ld, REDUCE[reduce], *pargs, it, _vdt(k), _stream())
    return out


def gated_backward_dst(rowptr: Tensor, col: Tensor, k: Tensor, q: Tensor, v: Tensor, grad_out: Tensor,
                       reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> Tensor:
    """grad_k[i,:] = g_i * sum_{e in row i} v[col[e],:] * sigmoid'(k[i,:] + q[col[e],:]), g_i = grad_out[i,:]
    (/ max(deg_i, 1) for mean)."""
    _cuda(rowptr, col, k, q, v, grad_out)
    ld = _gated_rows(k, q, v)
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr, col)
    F = k.size(1)
    grad_k = torch.empty_like(k)
    pargs, _ = _plan_args(plan, F, k.device)
    _timed("gated_backward_dst", 2 if pargs[2] else 1, lib().b200mp_gated_backward_dst, _p(rowptr), _p(col), _p(k),
           _p(q), _p(v), _p(grad_out), _p(grad_k), k.size(0), q.size(0), col.numel(), F, ld, REDUCE[reduce], *pargs,
           it, _vdt(k), _stream())
    return grad_k


def gated_backward_src(rowptr_t: Tensor, col_t: Tensor, val_t: Optional[Tensor], k: Tensor, q: Tensor, v: Tensor,
                       grad_out: Tensor, grad_q: Tensor, grad_v: Tensor,
                       plan_t: Optional[LongRowPlan] = None) -> Tuple[Tensor, Tensor]:
    """One transposed-CSR sweep writing grad_v[j,:] = sum_t sigmoid(s_t) * w_t g_t and grad_q[j,:] = v[j,:] *
    sum_t sigmoid'(s_t) * w_t g_t (w_t = val_t[t] or 1) into grad_q / grad_v, which share q's and v's row stride."""
    _cuda(rowptr_t, col_t, val_t, k, q, v, grad_out, grad_q, grad_v)
    ld = _gated_rows(k, q, v)
    if _gated_rows(k, grad_q, grad_v) != ld or grad_q.size(0) != q.size(0):
        raise ValueError("grad_q and grad_v must have the shape and row stride of q and v")
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr_t, col_t)
    F = k.size(1)
    pargs, _ = _plan_args(plan_t, 2 * F, k.device)
    _timed("gated_backward_src", 2 if pargs[2] else 1, lib().b200mp_gated_backward_src, _p(rowptr_t), _p(col_t),
           _p(val_t), _p(k), _p(q), _p(v), _p(grad_out), _p(grad_q), _p(grad_v), q.size(0), k.size(0), col_t.numel(),
           F, ld, *pargs, it, _vdt(k), _stream())
    return grad_q, grad_v


def _cg_rows(u: Tensor, v: Tensor, c: Optional[Tensor], n_edges: int) -> int:
    """Check the operands of the crystal-graph sweeps; returns F.  u: [n_dst, 2F], v: [n_src, 2F], each with unit
    feature stride and its own row stride >= 2F; c: None or a contiguous [n_edges, 2F] tensor; one dtype."""
    if u.dim() != 2 or u.size(1) % 2:
        raise ValueError(f"u must be a [N, 2F] tensor, got {tuple(u.shape)}")
    F = u.size(1) // 2
    for name, t in (("u", u), ("v", v)):
        if t.dim() != 2 or t.size(1) != 2 * F or t.dtype != u.dtype or (t.size(0) > 0 and t.stride(1) != 1) \
                or (t.size(0) > 1 and t.stride(0) < 2 * F):
            raise ValueError(f"{name} must be a [N, {2 * F}] tensor of u's dtype with unit feature stride, "
                             f"got {tuple(t.shape)} {t.dtype} strides {t.stride()}")
    if c is not None and (tuple(c.shape) != (n_edges, 2 * F) or c.dtype != u.dtype or not c.is_contiguous()):
        raise ValueError(f"c must be a contiguous [{n_edges}, {2 * F}] tensor of u's dtype, got {tuple(c.shape)} {c.dtype}")
    return F


def _ld(t: Tensor) -> int:
    return t.stride(0) if t.size(0) > 1 else t.size(1)


def cg_csr(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], u: Tensor, v: Tensor, c: Optional[Tensor],
           n_rows: int, reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> Tensor:
    """out[i,:] = REDUCE_{e in row i} sigmoid(f_e) * softplus(s_e) for sum / mean, [f_e | s_e] = u[i] + v[col[e]]
    (+ c[perm[e]]).  u: [n_rows, 2F], v: [n_src, 2F] (each with its own row stride); c: [E, 2F] in the caller's edge
    order or None; perm: CSR slot -> caller's edge id, None for an adopted CSR."""
    _cuda(rowptr, col, perm, u, v, c)
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"cg_csr reduces by sum or mean, not '{reduce}'")
    F = _cg_rows(u, v, c, col.numel())
    it = _same_idx(rowptr, col, perm)
    out = torch.empty(n_rows, F, dtype=u.dtype, device=u.device)
    pargs, _ = _plan_args(plan, F, u.device)
    _timed("cg_csr", 2 if pargs[2] else 1, lib().b200mp_cg_csr, _p(rowptr), _p(col), _p(perm), _p(u), _p(v), _p(c),
           _p(out), n_rows, v.size(0), col.numel(), F, _ld(u), _ld(v), REDUCE[reduce], *pargs, it, _vdt(u), _stream())
    return out


def cg_backward_dst(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], u: Tensor, v: Tensor, c: Optional[Tensor],
                    grad_out: Tensor, grad_u: Tensor, want_grad_c: bool, reduce: str = "sum",
                    plan: Optional[LongRowPlan] = None) -> Optional[Tensor]:
    """Destination sweep of the crystal-graph backward: writes grad_u[i] = sum_e [df_e | ds_e] into `grad_u` (u's shape
    and row stride) and, with want_grad_c, returns grad_c [E, 2F] = [df_e | ds_e] in the caller's edge order."""
    _cuda(rowptr, col, perm, u, v, c, grad_out, grad_u)
    F = _cg_rows(u, v, c, col.numel())
    if _cg_rows(grad_u, v, None, 0) != F or grad_u.size(0) != u.size(0) or _ld(grad_u) != _ld(u):
        raise ValueError("grad_u must have the shape and row stride of u")
    if want_grad_c and c is None:
        raise ValueError("grad_c is the gradient of c: want_grad_c needs c")
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr, col, perm)
    E = col.numel()
    grad_c = torch.empty(E, 2 * F, dtype=u.dtype, device=u.device) if want_grad_c else None
    pargs, _ = _plan_args(plan, 2 * F, u.device)
    _timed("cg_backward_dst", 2 if pargs[2] else 1, lib().b200mp_cg_backward_dst, _p(rowptr), _p(col), _p(perm), _p(u),
           _p(v), _p(c), _p(grad_out), _p(grad_u), _p(grad_c), u.size(0), v.size(0), E, F, _ld(u), _ld(v),
           REDUCE[reduce], *pargs, it, _vdt(u), _stream())
    return grad_c


def cg_backward_src(rowptr_t: Tensor, col_t: Tensor, perm_t: Tensor, val_t: Optional[Tensor], u: Tensor, v: Tensor,
                    c: Optional[Tensor], grad_out: Tensor, grad_v: Tensor,
                    plan_t: Optional[LongRowPlan] = None) -> Tensor:
    """Transposed-CSR sweep of the crystal-graph backward: grad_v[j] = sum_t [df_t | ds_t] with g = val_t[t] *
    grad_out[col_t[t]] (val_t None: 1), written into `grad_v` (v's shape and row stride)."""
    _cuda(rowptr_t, col_t, perm_t, val_t, u, v, c, grad_out, grad_v)
    E = col_t.numel()
    F = _cg_rows(u, v, c, E)
    if _cg_rows(u, grad_v, None, 0) != F or grad_v.size(0) != v.size(0) or _ld(grad_v) != _ld(v):
        raise ValueError("grad_v must have the shape and row stride of v")
    grad_out = grad_out.contiguous()
    it = _same_idx(rowptr_t, col_t, perm_t)
    pargs, _ = _plan_args(plan_t, 2 * F, u.device)
    _timed("cg_backward_src", 2 if pargs[2] else 1, lib().b200mp_cg_backward_src, _p(rowptr_t), _p(col_t), _p(perm_t),
           _p(val_t), _p(u), _p(v), _p(c), _p(grad_out), _p(grad_v), v.size(0), u.size(0), E, F, _ld(u), _ld(v),
           *pargs, it, _vdt(u), _stream())
    return grad_v


def nn_conv_supported(k: int, f_in: int, dtype: torch.dtype) -> bool:
    """Whether the NNConv sweeps take K hidden edge features and F_in source channels in this dtype."""
    if dtype not in (torch.float32, torch.bfloat16):
        return False
    return bool(lib().b200mp_nn_conv_supported(int(k), int(f_in), F32 if dtype == torch.float32 else BF16))


def _nn_conv_operands(col: Tensor, x: Tensor, h: Tensor):
    if x.dim() != 2 or h.dim() != 2 or h.size(0) != col.numel() or h.dtype != x.dtype:
        raise ValueError(f"x must be [n_src, F_in] and h [{col.numel()}, K] of x's dtype, got {tuple(x.shape)} "
                         f"{x.dtype} and {tuple(h.shape)} {h.dtype}")
    return x.contiguous(), h.contiguous(), h.size(1), x.size(1)


def nn_conv_csr(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], x: Tensor, h: Tensor, row_begin: int, row_end: int,
                reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> Tensor:
    """P [row_end - row_begin, (K+1) F_in] fp32 with P[i, k F_in + a] = REDUCE_{e in row i} [h[perm[e]], 1][k] x[col[e], a]
    for sum / mean: NNConv's message with the edge network's last Linear split off (out = P W').  h: [E, K] in the
    caller's edge order; perm: CSR slot -> caller's edge id, None for an adopted CSR."""
    _cuda(rowptr, col, perm, x, h)
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"nn_conv_csr reduces by sum or mean, not '{reduce}'")
    x, h, K, Fi = _nn_conv_operands(col, x, h)
    it = _same_idx(rowptr, col, perm)
    width = (K + 1) * Fi
    p = torch.empty(row_end - row_begin, width, dtype=torch.float32, device=x.device)
    # the hub chunks' partials, n_chunks * (K+1) F_in fp32, live for this call only: a [n_chunks, 16384] buffer cached on
    # the plan would stay with the graph
    part = None if plan is None or not plan.n_long else \
        torch.empty(plan.n_chunks * width, dtype=torch.float32, device=x.device)
    pargs = (*_plan_rows(plan), _p(part))
    _timed("nn_conv_csr", 2 if pargs[2] else 1, lib().b200mp_nn_conv_csr, _p(rowptr), _p(col), _p(perm), _p(x), _p(h),
           _p(p), rowptr.numel() - 1, x.size(0), col.numel(), K, Fi, int(row_begin), int(row_end), REDUCE[reduce], *pargs,
           it, _vdt(x), _stream())
    return p


def nn_conv_backward_dst(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], x: Tensor, h: Tensor, grad_p: Tensor,
                         row_begin: int, row_end: int, grad_h: Optional[Tensor], q: Optional[Tensor], reduce: str = "sum",
                         plan: Optional[LongRowPlan] = None) -> None:
    """Destination sweep of NNConv's backward for rows [row_begin, row_end): writes, per edge in the caller's order,
    grad_h[e, k] = x_j . grad_p[i, k, :] into `grad_h` ([E, K]) and q[e, :] = h~_e . grad_p[i] into `q` ([E, F_in]),
    either of them None to skip it.  grad_p: fp32 [row_end - row_begin, (K+1) F_in]."""
    _cuda(rowptr, col, perm, x, h, grad_p, grad_h, q)
    x, h, K, Fi = _nn_conv_operands(col, x, h)
    E = col.numel()
    if tuple(grad_p.shape) != (row_end - row_begin, (K + 1) * Fi) or grad_p.dtype != torch.float32 \
            or not grad_p.is_contiguous():
        raise ValueError(f"grad_p must be a contiguous fp32 [{row_end - row_begin}, {(K + 1) * Fi}] tensor")
    for name, t, w in (("grad_h", grad_h, K), ("q", q, Fi)):
        if t is not None and (tuple(t.shape) != (E, w) or t.dtype != x.dtype or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous [{E}, {w}] tensor of x's dtype")
    it = _same_idx(rowptr, col, perm)
    _timed("nn_conv_backward_dst", 1, lib().b200mp_nn_conv_backward_dst, _p(rowptr), _p(col), _p(perm), _p(x), _p(h),
           _p(grad_p), _p(grad_h), _p(q), rowptr.numel() - 1, x.size(0), E, K, Fi, int(row_begin), int(row_end),
           REDUCE[reduce], *_plan_rows(plan), it, _vdt(x), _stream())


def spline_supported(k: int, f_in: int, s: int, dtype: torch.dtype) -> bool:
    """Whether the SplineConv sweeps take K kernel weights, F_in source channels and S basis slots in this dtype."""
    if dtype not in (torch.float32, torch.bfloat16):
        return False
    return bool(lib().b200mp_spline_supported(int(k), int(f_in), int(s), F32 if dtype == torch.float32 else BF16))


def _spline_values(*ts: Optional[Tensor]) -> None:
    for t in ts:
        if t is not None and (not t.is_cuda or t.dtype not in (torch.float32, torch.bfloat16)):
            raise RuntimeError("pytorch_geometric_b200 computes the spline ops on CUDA float32 / bfloat16 tensors only "
                               f"(it has no CPU, float16 or float64 path); got a {t.dtype} tensor on {t.device}")


def spline_slots(dim: int, degree: int) -> int:
    """S = (degree + 1)^dim basis slots per edge; ValueError outside degree 1..3 and the slots the kernels take."""
    if degree not in (1, 2, 3) or dim < 1:
        raise ValueError(f"the spline ops take degree 1, 2 or 3 and dim >= 1, got degree {degree}, dim {dim}")
    s = (degree + 1) ** dim
    if not lib().b200mp_spline_supported(1, 1, min(s, 1 << 20), F32):
        raise ValueError(f"(degree + 1)^dim = {s} basis slots per edge is more than the spline kernels take")
    return s


def _spline_knots(pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor) -> Tuple[Tensor, Tensor]:
    if pseudo.dim() != 2 or kernel_size.numel() != pseudo.size(1) or is_open_spline.numel() != pseudo.size(1):
        raise ValueError(f"pseudo must be [E, D] with D kernel sizes and open flags, got {tuple(pseudo.shape)}, "
                         f"{kernel_size.numel()} and {is_open_spline.numel()}")
    return (kernel_size.to(device=pseudo.device, dtype=torch.int64).contiguous(),
            is_open_spline.to(device=pseudo.device, dtype=torch.uint8).contiguous())


def spline_basis(pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor, degree: int,
                 wi_dtype: torch.dtype = torch.int64) -> Tuple[Tensor, Tensor]:
    """(basis [E, S] of pseudo's dtype, weight_index [E, S] of wi_dtype) of the B-spline tensor-product basis, S =
    (degree + 1)^D (pyg_lib.ops.spline_basis; csrc/spline.cu states the convention)."""
    _spline_values(pseudo)
    ks, op = _spline_knots(pseudo, kernel_size, is_open_spline)
    E, D = pseudo.shape
    S = spline_slots(D, degree)
    pseudo = pseudo.contiguous()
    basis = torch.empty(E, S, dtype=pseudo.dtype, device=pseudo.device)
    wi = torch.empty(E, S, dtype=wi_dtype, device=pseudo.device)
    _timed("spline_basis", 1, lib().b200mp_spline_basis, _p(pseudo), _p(ks), _p(op), _p(basis), _p(wi), E, D, int(degree),
           _vdt(pseudo), _idt(wi), _stream())
    return basis, wi


def spline_basis_backward(grad_basis: Tensor, pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor,
                          degree: int) -> Tensor:
    """grad_pseudo [E, D] = sum_s grad_basis[e, s] d basis[e, s] / d pseudo[e, d]."""
    _spline_values(pseudo, grad_basis)
    ks, op = _spline_knots(pseudo, kernel_size, is_open_spline)
    E, D = pseudo.shape
    S = spline_slots(D, degree)
    if tuple(grad_basis.shape) != (E, S):
        raise ValueError(f"grad_basis must be [{E}, {S}], got {tuple(grad_basis.shape)}")
    pseudo = pseudo.contiguous()
    gb = grad_basis.to(pseudo.dtype).contiguous()
    gp = torch.empty_like(pseudo)
    _timed("spline_basis_backward", 1, lib().b200mp_spline_basis_backward, _p(gb), _p(pseudo), _p(ks), _p(op), _p(gp),
           E, D, int(degree), _vdt(pseudo), _stream())
    return gp


def _spline_weighting_operands(x: Tensor, weight: Tensor, basis: Tensor, wi: Tensor):
    _spline_values(x, weight, basis)
    _cuda(wi)
    if x.dim() != 2 or weight.dim() != 3 or weight.size(1) != x.size(1) or basis.dim() != 2 \
            or basis.size(0) != x.size(0) or tuple(wi.shape) != tuple(basis.shape):
        raise ValueError(f"spline_weighting takes x [E, F_in], weight [K, F_in, F_out], basis and weight_index [E, S]; "
                         f"got {tuple(x.shape)}, {tuple(weight.shape)}, {tuple(basis.shape)}, {tuple(wi.shape)}")
    if len({x.dtype, weight.dtype, basis.dtype}) != 1:
        raise TypeError(f"x, weight and basis must share a dtype, got {x.dtype}, {weight.dtype}, {basis.dtype}")
    if not lib().b200mp_spline_supported(1, 1, basis.size(1), F32):
        raise ValueError(f"{basis.size(1)} basis slots per edge is more than the spline kernels take")
    return x.contiguous(), weight.contiguous(), basis.contiguous(), wi.contiguous()


def spline_weighting(x: Tensor, weight: Tensor, basis: Tensor, wi: Tensor) -> Tensor:
    """out[e] = sum_s basis[e, s] x[e] @ weight[wi[e, s]] (pyg_lib.ops.spline_weighting), unfused: one thread per output
    element, S F_in F_out FMAs per edge."""
    x, weight, basis, wi = _spline_weighting_operands(x, weight, basis, wi)
    (E, Fi), (K, _, Fo), S = x.shape, weight.shape, basis.size(1)
    out = torch.empty(E, Fo, dtype=x.dtype, device=x.device)
    _timed("spline_weighting", 1, lib().b200mp_spline_weighting, _p(x), _p(weight), _p(basis), _p(wi), _p(out), E, Fi, Fo,
           K, S, _idt(wi), _vdt(x), _stream())
    return out


def spline_weighting_backward(grad_out: Tensor, x: Tensor, weight: Tensor, basis: Tensor, wi: Tensor, need_x: bool,
                              need_basis: bool, need_weight: bool):
    """(grad_x, grad_basis, grad_weight) of spline_weighting, each None unless asked for; grad_weight is fp32 and sums
    each kernel's slots in the order of a stable sort of weight_index (one kernel per weight index, no atomics)."""
    x, weight, basis, wi = _spline_weighting_operands(x, weight, basis, wi)
    (E, Fi), (K, _, Fo), S = x.shape, weight.shape, basis.size(1)
    _spline_values(grad_out)
    g = grad_out.to(x.dtype).contiguous()
    gx = torch.empty_like(x) if need_x else None
    gb = torch.empty_like(basis) if need_basis else None
    gw = torch.empty(K, Fi, Fo, dtype=torch.float32, device=x.device) if need_weight else None
    order = ptr = None
    if need_weight and E > 0:
        mn, mx, _ = index_stats(wi.reshape(-1))
        if mn < 0 or mx >= K:
            raise IndexError(f"weight_index holds {mn}..{mx}, outside the weight's {K} kernels")
        _, order, ptr = sort_by_key(wi.reshape(-1), K, want_sorted=False)
    _timed("spline_weighting_backward", int(need_x) + int(need_basis) + int(need_weight),
           lib().b200mp_spline_weighting_backward, _p(g), _p(x), _p(weight), _p(basis), _p(wi), _p(order), _p(ptr),
           _p(gx), _p(gb), _p(gw), E, Fi, Fo, K, S, _idt(wi), _vdt(x), _stream())
    return gx, gb, gw


def _spline_sweep_operands(col: Tensor, x: Tensor, basis: Tensor, wi: Tensor):
    if x.dim() != 2 or basis.dim() != 2 or basis.size(0) != col.numel() or basis.dtype != x.dtype \
            or tuple(wi.shape) != tuple(basis.shape) or wi.dtype != torch.int32:
        raise ValueError(f"x must be [n_src, F_in], basis [{col.numel()}, S] of x's dtype and weight_index int32 of "
                         f"basis's shape, got {tuple(x.shape)} {x.dtype}, {tuple(basis.shape)} {basis.dtype}, "
                         f"{tuple(wi.shape)} {wi.dtype}")
    return x.contiguous(), basis.contiguous(), wi.contiguous(), x.size(1), basis.size(1)


def spline_csr(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], x: Tensor, basis: Tensor, wi: Tensor, k: int,
               row_begin: int, row_end: int, reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> Tensor:
    """P [row_end - row_begin, K F_in] fp32 with P[i, k F_in + a] = REDUCE_{e in row i} sum_{s: wi[e', s] = k}
    basis[e', s] x[col[e], a], e' = perm[e], for sum / mean: SplineConv's message before its weight (out = P W.view(K F_in,
    F_out)).  basis [E, S] and wi [E, S] int32 in the caller's edge order; perm: CSR slot -> caller's edge id, None for
    an adopted CSR."""
    _cuda(rowptr, col, perm, x, basis, wi)
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"spline_csr reduces by sum or mean, not '{reduce}'")
    x, basis, wi, Fi, S = _spline_sweep_operands(col, x, basis, wi)
    it = _same_idx(rowptr, col, perm)
    width = int(k) * Fi
    p = torch.empty(row_end - row_begin, width, dtype=torch.float32, device=x.device)
    # the hub chunks' partials, n_chunks * K F_in fp32, live for this call only (as nn_conv_csr's)
    part = None if plan is None or not plan.n_long else \
        torch.empty(plan.n_chunks * width, dtype=torch.float32, device=x.device)
    pargs = (*_plan_rows(plan), _p(part))
    _timed("spline_csr", 2 if pargs[2] else 1, lib().b200mp_spline_csr, _p(rowptr), _p(col), _p(perm), _p(x), _p(basis),
           _p(wi), _p(p), rowptr.numel() - 1, x.size(0), col.numel(), int(k), Fi, S, int(row_begin), int(row_end),
           REDUCE[reduce], *pargs, it, _vdt(x), _stream())
    return p


def spline_backward_dst(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], x: Tensor, basis: Tensor, wi: Tensor,
                        k: int, grad_p: Tensor, row_begin: int, row_end: int, grad_basis: Optional[Tensor],
                        q: Optional[Tensor], reduce: str = "sum", plan: Optional[LongRowPlan] = None) -> None:
    """Destination sweep of the fused SplineConv's backward for rows [row_begin, row_end): writes, per edge in the
    caller's order, grad_basis[e, s] = <grad_p[i, wi[e, s], :], x_j> into `grad_basis` ([E, S]) and q[e, :] =
    sum_s basis[e, s] grad_p[i, wi[e, s], :] into `q` ([E, F_in]), either None to skip it.  grad_p: fp32
    [row_end - row_begin, K F_in]."""
    _cuda(rowptr, col, perm, x, basis, wi, grad_p, grad_basis, q)
    x, basis, wi, Fi, S = _spline_sweep_operands(col, x, basis, wi)
    E = col.numel()
    if tuple(grad_p.shape) != (row_end - row_begin, int(k) * Fi) or grad_p.dtype != torch.float32 \
            or not grad_p.is_contiguous():
        raise ValueError(f"grad_p must be a contiguous fp32 [{row_end - row_begin}, {int(k) * Fi}] tensor")
    for name, t, w in (("grad_basis", grad_basis, S), ("q", q, Fi)):
        if t is not None and (tuple(t.shape) != (E, w) or t.dtype != x.dtype or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous [{E}, {w}] tensor of x's dtype")
    it = _same_idx(rowptr, col, perm)
    _timed("spline_backward_dst", 1, lib().b200mp_spline_backward_dst, _p(rowptr), _p(col), _p(perm), _p(x), _p(basis),
           _p(wi), _p(grad_p), _p(grad_basis), _p(q), rowptr.numel() - 1, x.size(0), E, int(k), Fi, S, int(row_begin),
           int(row_end), REDUCE[reduce], *_plan_rows(plan), it, _vdt(x), _stream())


SOFTMAX_MESSAGES = {"identity": 0, "relu_eps": 1}


# ------------------------------------------------------------------ point clouds (csrc/point.cu)
KNN_MAX_K = 128


def _point_values(*ts: Optional[Tensor]) -> None:
    for t in ts:
        if t is not None and (not t.is_cuda or t.dtype not in (torch.float32, torch.bfloat16)):
            raise RuntimeError("pytorch_geometric_b200 computes the point-cloud ops on CUDA float32 / bfloat16 tensors "
                               f"only (it has no CPU, float16 or float64 path); got a {t.dtype} tensor on {t.device}")


def _point_rows(t: Tensor) -> Tensor:
    """[N, F] contiguous view of a point matrix (a 1-D tensor is N points of one feature)."""
    t = t.detach()
    t = t.view(-1, 1) if t.dim() == 1 else t.reshape(t.size(0), -1)
    return t.contiguous()


def _point_ptrs(n_x: int, n_y: int, ptr_x: Optional[Tensor], ptr_y: Optional[Tensor], device):
    ptrs = [p for p in (ptr_x, ptr_y) if p is not None]
    _cuda(*ptrs)
    for p in ptrs:
        if p.device != device:
            raise RuntimeError(f"ptr must be on the points' device {device}, got {p.device}")
    pdt = _same_idx(*ptrs) if ptrs else I64
    ptr_x = None if ptr_x is None else ptr_x.contiguous()
    ptr_y = None if ptr_y is None else ptr_y.contiguous()
    from . import _debug
    if _debug.enabled():
        for p, n, name in ((ptr_x, n_x, "ptr_x"), (ptr_y, n_y, "ptr_y")):
            if p is not None and p.numel() > 0:
                h = p.cpu()
                if int(h[0]) < 0 or int(h[-1]) > n or bool((h[1:] < h[:-1]).any()):
                    raise ValueError(f"{name} must be non-decreasing within [0, {n}]")
    return ptr_x, ptr_y, pdt


def _np(p: Optional[Tensor]) -> int:
    return 0 if p is None else p.numel()


def knn(x: Tensor, y: Tensor, k: int, ptr_x: Optional[Tensor] = None, ptr_y: Optional[Tensor] = None,
        cosine: bool = False) -> Tensor:
    """[2, nnz] int64 (y index, x index): for each y point the k nearest x points of its example, distance ascending,
    ties by ascending x index (pyg_lib.ops.knn; csrc/point.cu states the distance contract)."""
    _point_values(x, y)
    k = int(k)
    if not 1 <= k <= KNN_MAX_K:
        raise ValueError(f"knn takes 1 <= k <= {KNN_MAX_K} neighbours, got k = {k}")
    if x.dtype != y.dtype:
        raise TypeError(f"x and y must share a dtype, got {x.dtype} and {y.dtype}")
    x, y = _point_rows(x), _point_rows(y)
    if x.size(1) != y.size(1):
        raise ValueError(f"x and y must have the same number of features, got {x.size(1)} and {y.size(1)}")
    ptr_x, ptr_y, pdt = _point_ptrs(x.size(0), y.size(0), ptr_x, ptr_y, x.device)
    M = y.size(0)
    slab = torch.empty(2, M * k, dtype=torch.int64, device=x.device)
    offsets = torch.empty(M + 1, dtype=torch.int64, device=x.device)
    _timed("knn", 2, lib().b200mp_knn, _p(x), _p(y), _p(ptr_x), _p(ptr_y), x.size(0), M, x.size(1), _np(ptr_x),
           _np(ptr_y), k, int(bool(cosine)), _p(slab), _p(offsets), _vdt(x), pdt, _stream())
    nnz = int(offsets[M])
    if nnz == M * k:
        return slab
    out = torch.empty(2, nnz, dtype=torch.int64, device=x.device)
    _timed("knn_compact", 1, lib().b200mp_knn_compact, _p(slab), _p(offsets), M, k, _p(out), nnz, _stream())
    return out


def radius(x: Tensor, y: Tensor, r: float, ptr_x: Optional[Tensor] = None, ptr_y: Optional[Tensor] = None,
           max_num_neighbors: int = 32, ignore_same_index: bool = False) -> Tensor:
    """[2, nnz] int64 (y index, x index): for each y point the first max_num_neighbors x points of its example, in
    ascending index order, with squared distance < r^2 (r^2 formed in fp64, rounded once to fp32)."""
    _point_values(x, y)
    if x.dtype != y.dtype:
        raise TypeError(f"x and y must share a dtype, got {x.dtype} and {y.dtype}")
    x, y = _point_rows(x), _point_rows(y)
    if x.size(1) != y.size(1):
        raise ValueError(f"x and y must have the same number of features, got {x.size(1)} and {y.size(1)}")
    ptr_x, ptr_y, pdt = _point_ptrs(x.size(0), y.size(0), ptr_x, ptr_y, x.device)
    M = y.size(0)
    r2 = float(r) * float(r)                                      # fp64; ctypes rounds it once to fp32
    args = (_p(x), _p(y), _p(ptr_x), _p(ptr_y), x.size(0), M, x.size(1), _np(ptr_x), _np(ptr_y), r2,
            int(max_num_neighbors), int(bool(ignore_same_index)))
    offsets = torch.empty(M + 1, dtype=torch.int64, device=x.device)
    _timed("radius_count", 2, lib().b200mp_radius_count, *args, _p(offsets), _vdt(x), pdt, _stream())
    nnz = int(offsets[M])
    out = torch.empty(2, nnz, dtype=torch.int64, device=x.device)
    _timed("radius_fill", 1, lib().b200mp_radius_fill, *args, _p(offsets), _p(out), nnz, _vdt(x), pdt, _stream())
    return out


def nearest(x: Tensor, y: Tensor, ptr_x: Optional[Tensor] = None, ptr_y: Optional[Tensor] = None) -> Tensor:
    """[N] int64: for each x point, the index of the nearest y point of its example (torch-cluster's cluster vector).
    ValueError when an x point finds none (its example has no y points, or only NaN / infinite distances)."""
    _point_values(x, y)
    if x.dtype != y.dtype:
        raise TypeError(f"x and y must share a dtype, got {x.dtype} and {y.dtype}")
    x, y = _point_rows(x), _point_rows(y)
    if x.size(1) != y.size(1):
        raise ValueError(f"x and y must have the same number of features, got {x.size(1)} and {y.size(1)}")
    ptr_x, ptr_y, pdt = _point_ptrs(x.size(0), y.size(0), ptr_x, ptr_y, x.device)
    N = x.size(0)
    slab = torch.empty(2, N, dtype=torch.int64, device=x.device)
    offsets = torch.empty(N + 1, dtype=torch.int64, device=x.device)
    _timed("nearest", 2, lib().b200mp_nearest, _p(x), _p(y), _p(ptr_x), _p(ptr_y), N, y.size(0), x.size(1),
           _np(ptr_x), _np(ptr_y), _p(slab), _p(offsets), _vdt(x), pdt, _stream())
    if int(offsets[N]) != N:
        raise ValueError("nearest: some x point has no y point in its example (or only NaN / infinite distances)")
    return slab[1]


def fps(src: Tensor, ptr: Optional[Tensor] = None, ratio: float = 0.5, random_start: bool = True) -> Tensor:
    """[S] int64 global indices of the farthest-point samples of each example, in selection order, examples
    concatenated; ceil(n_b ratio) samples of example b (fp64), 0 < ratio <= 1.  random_start draws the start of each
    example on the device from torch's CUDA generator; otherwise each example starts at its first point."""
    _point_values(src)
    ratio = float(ratio)
    if not 0.0 < ratio <= 1.0:
        raise ValueError(f"fps takes a sampling ratio in (0, 1], got {ratio}")
    src = _point_rows(src)
    N = src.size(0)
    ptr, _, pdt = _point_ptrs(N, N, ptr, None, src.device)
    B = 1 if ptr is None else max(ptr.numel() - 1, 0)
    offsets = torch.empty(B + 1, dtype=torch.int64, device=src.device)
    _timed("fps_count", 2, lib().b200mp_fps_count, _p(ptr), _np(ptr), N, ratio, _p(offsets), pdt, _stream())
    total = int(offsets[B])
    out = torch.empty(total, dtype=torch.int64, device=src.device)
    if total == 0:
        return out
    rnd = torch.rand(B, device=src.device) if random_start else None
    dist = torch.empty(N, dtype=torch.float32, device=src.device)
    _timed("fps", 1, lib().b200mp_fps, _p(src), _p(ptr), N, src.size(1), _np(ptr), _p(rnd), _p(offsets), _p(dist),
           _p(out), _vdt(src), pdt, _stream())
    return out


# ------------------------------------------------------------------ clustering for pooling (csrc/cluster.cu)
GRACLUS_MAX_ROUNDS = 256
_GRACLUS_WEIGHTS = {torch.float32: F32, torch.bfloat16: BF16, torch.float64: F64}


def graclus(rowptr: Tensor, col: Tensor, weight: Optional[Tensor] = None, seed: Optional[int] = None,
            return_rounds: bool = False):
    """[N] int64 cluster vector of a greedy matching of the CSR graph (rowptr [N + 1], col): min(u, v) for each
    matched pair, u for each singleton (pyg_lib.ops.graclus_cluster; csrc/cluster.cu states the rules).  weight (one
    float32 / bfloat16 / float64 value per CSR entry) makes each node pick its heaviest eligible neighbour.  The result
    is a pure function of (graph, weight, seed); seed defaults to a draw from torch's CPU generator, so it is
    reproducible under torch.manual_seed and costs no device synchronisation.  return_rounds also returns the number
    of matching rounds as a 0-dim int32 CUDA tensor (at most GRACLUS_MAX_ROUNDS)."""
    _cuda(rowptr, col, weight)
    idt = _same_idx(rowptr, col)
    if rowptr.dim() != 1 or rowptr.numel() < 1 or col.dim() != 1:
        raise ValueError(f"rowptr must be [N + 1] and col [E], got {tuple(rowptr.shape)} and {tuple(col.shape)}")
    n = rowptr.numel() - 1
    if n >= 2**31 - 1:
        raise ValueError(f"graclus takes fewer than 2^31 - 1 nodes, got {n}")
    wdt = F32
    if weight is not None:
        if weight.dtype not in _GRACLUS_WEIGHTS:
            raise TypeError(f"graclus weights must be float32, bfloat16 or float64, got {weight.dtype}")
        if weight.numel() != col.numel() or weight.device != col.device:
            raise ValueError(f"weight must hold one value per edge on {col.device}, got {weight.numel()} for "
                             f"{col.numel()} edges on {weight.device}")
        wdt = _GRACLUS_WEIGHTS[weight.dtype]
        weight = weight.detach().reshape(-1).contiguous()
    if rowptr.device != col.device:
        raise RuntimeError(f"rowptr and col must share a device, got {rowptr.device} and {col.device}")
    rowptr, col = rowptr.contiguous(), col.contiguous()
    from . import _debug
    if _debug.enabled() and n > 0:
        rp, c = rowptr.cpu(), col.cpu()
        if int(rp[0]) != 0 or int(rp[-1]) != c.numel() or bool((rp[1:] < rp[:-1]).any()):
            raise ValueError(f"rowptr must be non-decreasing from 0 to the number of edges {c.numel()}")
        if c.numel() > 0 and (int(c.min()) < 0 or int(c.max()) >= n):
            raise IndexError(f"col must hold node indices in [0, {n})")
    if seed is None:
        seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    seed = int(seed) & (2**64 - 1)
    cluster = torch.empty(n, dtype=torch.int64, device=rowptr.device)
    ws = torch.empty(2 * n + 3, dtype=torch.int32, device=rowptr.device)
    _timed("graclus", 1 if n > 0 else 0, lib().b200mp_graclus, _p(rowptr), _p(col), _p(weight), n, seed, _p(cluster),
           _p(ws), idt, wdt, _stream())
    return (cluster, ws[2 * n + 2]) if return_rounds else cluster


def grid_cluster(pos: Tensor, size: Tensor, start: Optional[Tensor] = None, end: Optional[Tensor] = None) -> Tensor:
    """[N] int64 voxel index of each point (pyg_lib.ops.grid_cluster): sum_d trunc((pos[i, d] - start[d]) / size[d])
    * prod_{d' < d} (trunc((end[d'] - start[d']) / size[d']) + 1) in pos's dtype (float32 or float64).  A missing
    start / end is the column min / max of pos (NaN propagating), computed on the device.  size, start and end hold D
    values and are cast to pos's dtype."""
    _cuda(pos, size, start, end)
    if pos.dtype in (torch.float16, torch.bfloat16):
        raise TypeError(f"grid_cluster takes float32 or float64 positions, got {pos.dtype}: voxel_grid appends the "
                        "batch index as a coordinate, which stops being exact above 2048 (float16) or 256 (bfloat16)")
    if pos.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"grid_cluster takes float32 or float64 positions, got {pos.dtype}")
    pos = pos.detach()
    pos = (pos.view(-1, 1) if pos.dim() == 1 else pos.flatten(1)).contiguous()
    n, d = pos.shape
    if not 1 <= d <= 65535:
        raise ValueError(f"grid_cluster takes 1 to 65535 coordinates per point, got {d}")

    def vec(t: Optional[Tensor], name: str) -> Optional[Tensor]:
        if t is None:
            return None
        if t.device != pos.device:
            raise RuntimeError(f"{name} must be on the points' device {pos.device}, got {t.device}")
        t = t.detach().to(pos.dtype).reshape(-1).contiguous()
        if t.numel() != d:
            raise ValueError(f"{name} must hold one value per coordinate ({d}), got {t.numel()}")
        return t

    size, start, end = vec(size, "size"), vec(start, "start"), vec(end, "end")
    out = torch.empty(n, dtype=torch.int64, device=pos.device)
    ws = torch.empty(514 * d, dtype=pos.dtype, device=pos.device) if start is None or end is None else None
    n_kernels = 0 if n == 0 else (1 if ws is None else 3)
    _timed("grid_cluster", n_kernels, lib().b200mp_grid_cluster, _p(pos), _p(size), _p(start), _p(end), n, d, _p(out),
           _p(ws), F64 if pos.dtype == torch.float64 else F32, _stream())
    return out


# ------------------------------------------------------------------ random walks (csrc/random_walk.cu)
# Trials per node2vec step before the exact draw, which scans the current row (twice, with a neighbour test per entry).
# A walk's stationary distribution favours hubs, so with 64 trials (a rejection chance of up to (15/16)^64 = 1.6 %
# at p = 1/4, q = 4) the exact draw often lands on rows of millions of entries; 1024 makes it negligible for moderate
# p and q and still bounds the work for extreme ones (README: the row_order lines).
RANDOM_WALK_MAX_TRIALS = 1024
_ROWS_UNSORTED = OrderedDict()       # (rowptr, col) identity -> (rowptr, col, versions, rows_unsorted flag [1] int32)
_ROWS_UNSORTED_ENTRIES = 8


def _rows_unsorted_flag(rowptr: Tensor, col: Tensor) -> Tuple[Tensor, bool]:
    """The device flag of the neighbour test (1 when some row of col decreases) and whether it must be computed: cached
    by the identity and version of both tensors, the strong references living in the cache entry (as plugin/graphs.py
    caches pair graphs), so repeated batches over one graph check it once."""
    key = (rowptr.data_ptr(), col.data_ptr(), rowptr.numel(), col.numel(), rowptr.dtype, rowptr.device)
    hit = _ROWS_UNSORTED.get(key)
    if hit is not None and hit[2] == (rowptr._version, col._version):
        _ROWS_UNSORTED.move_to_end(key)
        return hit[3], False
    flag = torch.empty(1, dtype=torch.int32, device=rowptr.device)
    _ROWS_UNSORTED[key] = (rowptr, col, (rowptr._version, col._version), flag)
    while len(_ROWS_UNSORTED) > _ROWS_UNSORTED_ENTRIES:
        _ROWS_UNSORTED.popitem(last=False)
    return flag, True


def random_walk(rowptr: Tensor, col: Tensor, start: Tensor, walk_length: int, p: float = 1.0, q: float = 1.0,
                seed: Optional[int] = None, max_trials: int = RANDOM_WALK_MAX_TRIALS) -> Tensor:
    """[S, walk_length + 1] random walks over the CSR graph (rowptr [N + 1], col [E]) from each node of start [S], in
    the index dtype (pyg_lib.ops.random_walk; csrc/random_walk.cu states the rules).  p = q = 1 gives uniform walks;
    other values give node2vec's second-order walks (return parameter p, in-out parameter q) by rejection sampling,
    with an exact draw after max_trials rejected trials of a step.  A node without out-edges keeps the walk where it
    is.  A start outside [0, N) gives a row of -1, and a column value outside [0, N) ends its walk with -1s (debug mode
    raises instead).  The walks are a pure function of (graph, start, walk_length, p, q, max_trials, seed); seed
    defaults to a draw from torch's CPU generator, so torch.manual_seed reproduces them and nothing synchronises."""
    _cuda(rowptr, col, start)
    idt = _same_idx(rowptr, col, start)
    if rowptr.dim() != 1 or rowptr.numel() < 1 or col.dim() != 1 or start.dim() != 1:
        raise ValueError(f"rowptr must be [N + 1], col [E] and start [S], got {tuple(rowptr.shape)}, "
                         f"{tuple(col.shape)} and {tuple(start.shape)}")
    if not (rowptr.device == col.device == start.device):
        raise RuntimeError(f"rowptr, col and start must share a device, got {rowptr.device}, {col.device} and "
                           f"{start.device}")
    walk_length, p, q, max_trials = int(walk_length), float(p), float(q), int(max_trials)
    if walk_length < 0:
        raise ValueError(f"random_walk takes walk_length >= 0, got {walk_length}")
    for name, v in (("p", p), ("q", q)):
        if not (math.isfinite(v) and v > 0.0):
            raise ValueError(f"random_walk takes a finite {name} > 0, got {v}")
    if max_trials < 0:
        raise ValueError(f"random_walk takes max_trials >= 0, got {max_trials}")
    n = rowptr.numel() - 1
    if n >= 2**31 - 1:
        raise ValueError(f"random_walk takes fewer than 2^31 - 1 nodes, got {n}")
    rowptr, col, start = rowptr.contiguous(), col.contiguous(), start.contiguous()
    from . import _debug
    if _debug.enabled():
        rp, c, s = rowptr.cpu(), col.cpu(), start.cpu()
        if int(rp[0]) != 0 or int(rp[-1]) != c.numel() or bool((rp[1:] < rp[:-1]).any()):
            raise ValueError(f"rowptr must be non-decreasing from 0 to the number of edges {c.numel()}")
        if c.numel() > 0 and (int(c.min()) < 0 or int(c.max()) >= n):
            raise IndexError(f"col must hold node indices in [0, {n})")
        if s.numel() > 0 and (int(s.min()) < 0 or int(s.max()) >= n):
            raise IndexError(f"start must hold node indices in [0, {n})")
    S = start.numel()
    out = torch.empty(S, walk_length + 1, dtype=rowptr.dtype, device=rowptr.device)
    if S == 0:
        return out
    if seed is None:
        seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    seed = int(seed) & (2**64 - 1)
    flag, refresh = None, False
    if p != 1.0 or q != 1.0:
        flag, refresh = _rows_unsorted_flag(rowptr, col)
    n_kernels = 1 + int(refresh and n > 0 and col.numel() > 1)
    _timed("random_walk", n_kernels, lib().b200mp_random_walk, _p(rowptr), _p(col), _p(start), n, col.numel(), S,
           walk_length, p, q, max_trials, seed, _p(flag), int(refresh), _p(out), idt, _stream())
    return out


def _softmax_aggr_args(x: Optional[Tensor], a: Optional[Tensor], w: Optional[Tensor], message: str, n_edges: int,
                       clamp: Optional[tuple] = None):
    """Check the operands of the softmax- and power-mean-aggregation sweeps; returns (F, message code, mode of w), and
    with power mean's clamp = (clamp_min, clamp_max) also (lo, hi).  x: [n_src, F] or None; a: [n_edges, F] in the
    caller's edge order or None, contiguous, one dtype; w (t or p): None or fp32 [1] / [F]; with p, clamp_min > 0 and
    clamp_max None (no upper bound) or >= clamp_min."""
    if message not in SOFTMAX_MESSAGES:
        raise ValueError(f"message must be one of {sorted(SOFTMAX_MESSAGES)}, got '{message}'")
    if message == "relu_eps" and x is None:
        raise ValueError("the relu_eps message needs x")
    if message == "identity" and (x is None) == (a is None):
        raise ValueError("the identity message takes exactly one of x and the edge rows")
    ref = x if x is not None else a
    F = ref.size(1)
    for name, v in (("x", x), ("edge rows", a)):
        if v is not None and (v.dim() != 2 or v.size(1) != F or v.dtype != ref.dtype or not v.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous [N, {F}] tensor of dtype {ref.dtype}, got {tuple(v.shape)}")
    if a is not None and a.size(0) != n_edges:
        raise ValueError(f"edge rows must have {n_edges} rows, got {a.size(0)}")
    mode = 0
    if w is not None:
        if w.dtype != torch.float32 or not w.is_contiguous() or w.numel() not in (1, F):
            raise ValueError(f"t must be a contiguous float32 tensor of 1 or {F} elements, got {tuple(w.shape)} {w.dtype}")
        mode = 1 if w.numel() == 1 else 2
    if clamp is None:
        return F, SOFTMAX_MESSAGES[message], mode
    lo = 0.0 if clamp[0] is None else float(clamp[0])
    hi = float("inf") if clamp[1] is None else float(clamp[1])
    if w is not None and not (lo > 0.0 and hi >= lo):
        raise ValueError(f"the power-mean sweep needs 0 < clamp_min <= clamp_max, got {clamp[0]} and {clamp[1]}")
    return F, SOFTMAX_MESSAGES[message], mode, lo, hi


def softmax_aggr_csr(rowptr: Tensor, col: Optional[Tensor], perm: Optional[Tensor], x: Optional[Tensor],
                     a: Optional[Tensor], t: Optional[Tensor], n_rows: int, n_edges: int, message: str = "identity",
                     eps: float = 0.0, plan: Optional[LongRowPlan] = None,
                     want_lse: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """out[i] = sum_e softmax_e(t * m_e) m_e over row i (b200mp_softmax_aggr_csr), m_e = x[col[e]] / a[perm[e]] /
    relu(x[col[e]] (+ a[perm[e]])) + eps; with want_lse also the fp32 lse plane the backward reads."""
    _cuda(rowptr, col, perm, x, a, t)
    F, msg, t_mode = _softmax_aggr_args(x, a, t, message, n_edges)
    it = _same_idx(rowptr, col, perm)
    ref = x if x is not None else a
    out = torch.empty(n_rows, F, dtype=ref.dtype, device=ref.device)
    lse = torch.empty(n_rows, F, dtype=torch.float32, device=ref.device) if want_lse else None
    pargs, _ = _plan_args(plan, 3 * F, ref.device)
    _timed("softmax_aggr_csr", 2 if pargs[2] else 1, lib().b200mp_softmax_aggr_csr, _p(rowptr), _p(col), _p(perm),
           _p(x), _p(a), _p(t), _p(out), _p(lse), n_rows, 0 if x is None else x.size(0), n_edges, F, msg, float(eps),
           t_mode, *pargs, it, _vdt(ref), _stream())
    return out, lse


def softmax_aggr_backward_dst(rowptr: Tensor, col: Optional[Tensor], perm: Optional[Tensor], x: Optional[Tensor],
                              a: Optional[Tensor], t: Optional[Tensor], out: Tensor, lse: Tensor, grad_out: Tensor,
                              n_edges: int, message: str, eps: float, semi_grad: bool, want_grad_a: bool,
                              want_grad_t: bool, plan: Optional[LongRowPlan] = None):
    """Destination sweep of the softmax-aggregation backward: (grad_a [E, F] in the caller's edge order or None,
    grad_t [F] fp32 per-channel sums or None)."""
    _cuda(rowptr, col, perm, x, a, t, out, lse, grad_out)
    F, msg, t_mode = _softmax_aggr_args(x, a, t, message, n_edges)
    if want_grad_t and t is None:
        raise ValueError("grad_t needs t")
    it = _same_idx(rowptr, col, perm)
    grad_out = grad_out.contiguous()
    n_rows = rowptr.numel() - 1
    grad_a = torch.empty(n_edges, F, dtype=out.dtype, device=out.device) if want_grad_a else None
    grad_t = ws = None
    pargs = _plan_rows(plan)
    if want_grad_t:
        grad_t = torch.empty(F, dtype=torch.float32, device=out.device)
        ws = torch.empty(max(int(lib().b200mp_softmax_aggr_workspace(n_rows, pargs[3], F)), 1), dtype=torch.float32,
                         device=out.device)
    _timed("softmax_aggr_backward_dst", 3 if want_grad_t else 1, lib().b200mp_softmax_aggr_backward_dst, _p(rowptr),
           _p(col), _p(perm), _p(x), _p(a), _p(t), _p(out), _p(lse), _p(grad_out), _p(grad_a), _p(grad_t), _p(ws),
           n_rows, 0 if x is None else x.size(0), n_edges, F, msg, float(eps), t_mode, int(bool(semi_grad)),
           *pargs, it, _vdt(out), _stream())
    return grad_a, grad_t


def softmax_aggr_backward_src(rowptr_t: Tensor, col_t: Tensor, perm_t: Tensor, x: Tensor, a: Optional[Tensor],
                              t: Optional[Tensor], out: Tensor, lse: Tensor, grad_out: Tensor, message: str,
                              eps: float, semi_grad: bool, plan_t: Optional[LongRowPlan] = None) -> Tensor:
    """Transposed-CSR sweep of the softmax-aggregation backward: grad_x [n_src, F] (a frozen)."""
    _cuda(rowptr_t, col_t, perm_t, x, a, t, out, lse, grad_out)
    E = col_t.numel()
    F, msg, t_mode = _softmax_aggr_args(x, a, t, message, E)
    it = _same_idx(rowptr_t, col_t, perm_t)
    grad_out = grad_out.contiguous()
    grad_x = torch.empty_like(x)
    pargs, _ = _plan_args(plan_t, F, x.device)
    _timed("softmax_aggr_backward_src", 2 if pargs[2] else 1, lib().b200mp_softmax_aggr_backward_src, _p(rowptr_t),
           _p(col_t), _p(perm_t), _p(x), _p(a), _p(t), _p(out), _p(lse), _p(grad_out), _p(grad_x), x.size(0),
           out.size(0), E, F, msg, float(eps), t_mode, int(bool(semi_grad)), *pargs, it, _vdt(x), _stream())
    return grad_x


def power_mean_csr(rowptr: Tensor, col: Optional[Tensor], perm: Optional[Tensor], x: Optional[Tensor],
                   a: Optional[Tensor], p: Optional[Tensor], n_rows: int, n_edges: int, message: str = "identity",
                   eps: float = 0.0, clamp_min: float = 1e-4, clamp_max: Optional[float] = 100.0,
                   plan: Optional[LongRowPlan] = None, want_mean: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """out[i] = clamp(mean_e clamp(m_e)^p)^(1/p) over row i (b200mp_power_mean_csr), m_e as in softmax_aggr_csr; p None
    is a plain mean.  With want_mean also the fp32 plane of the means M the backward reads."""
    _cuda(rowptr, col, perm, x, a, p)
    F, msg, p_mode, lo, hi = _softmax_aggr_args(x, a, p, message, n_edges, (clamp_min, clamp_max))
    it = _same_idx(rowptr, col, perm)
    ref = x if x is not None else a
    out = torch.empty(n_rows, F, dtype=ref.dtype, device=ref.device)
    mean = torch.empty(n_rows, F, dtype=torch.float32, device=ref.device) if want_mean else None
    pargs, _ = _plan_args(plan, F, ref.device)
    _timed("power_mean_csr", 2 if pargs[2] else 1, lib().b200mp_power_mean_csr, _p(rowptr), _p(col), _p(perm), _p(x),
           _p(a), _p(p), _p(out), _p(mean), n_rows, 0 if x is None else x.size(0), n_edges, F, msg, float(eps), p_mode,
           lo, hi, *pargs, it, _vdt(ref), _stream())
    return out, mean


def power_mean_backward_dst(rowptr: Tensor, col: Optional[Tensor], perm: Optional[Tensor], x: Optional[Tensor],
                            a: Optional[Tensor], p: Optional[Tensor], out: Tensor, mean: Optional[Tensor],
                            grad_out: Tensor, n_edges: int, message: str, eps: float, clamp_min: float,
                            clamp_max: Optional[float], want_grad_a: bool, want_grad_p: bool,
                            plan: Optional[LongRowPlan] = None):
    """Destination sweep of the power-mean backward: (grad_a [E, F] in the caller's edge order or None, grad_p [F]
    fp32 per-channel sums or None)."""
    _cuda(rowptr, col, perm, x, a, p, out, mean, grad_out)
    F, msg, p_mode, lo, hi = _softmax_aggr_args(x, a, p, message, n_edges, (clamp_min, clamp_max))
    if want_grad_p and p is None:
        raise ValueError("grad_p needs p")
    it = _same_idx(rowptr, col, perm)
    grad_out = grad_out.contiguous()
    n_rows = rowptr.numel() - 1
    grad_a = torch.empty(n_edges, F, dtype=out.dtype, device=out.device) if want_grad_a else None
    grad_p = ws = None
    pargs = _plan_rows(plan)
    if want_grad_p:
        grad_p = torch.empty(F, dtype=torch.float32, device=out.device)
        ws = torch.empty(max(int(lib().b200mp_power_mean_workspace(0, n_rows, pargs[3], F)), 1), dtype=torch.float32,
                         device=out.device)
    _timed("power_mean_backward_dst", 3 if want_grad_p else 1, lib().b200mp_power_mean_backward_dst, _p(rowptr),
           _p(col), _p(perm), _p(x), _p(a), _p(p), _p(out), _p(mean), _p(grad_out), _p(grad_a), _p(grad_p), _p(ws),
           n_rows, 0 if x is None else x.size(0), n_edges, F, msg, float(eps), p_mode, lo, hi, *pargs, it,
           _vdt(out), _stream())
    return grad_a, grad_p


def power_mean_backward_src(rowptr: Tensor, rowptr_t: Tensor, col_t: Tensor, perm_t: Tensor, x: Tensor,
                            a: Optional[Tensor], p: Optional[Tensor], out: Tensor, mean: Optional[Tensor],
                            grad_out: Tensor, message: str, eps: float, clamp_min: float, clamp_max: Optional[float],
                            want_grad_p: bool, plan_t: Optional[LongRowPlan] = None):
    """Node kernel and transposed-CSR sweep of the power-mean backward: (grad_x [n_src, F] (a frozen), grad_p [F] fp32
    per-channel sums or None).  rowptr: the destination CSR's, for the degrees."""
    _cuda(rowptr, rowptr_t, col_t, perm_t, x, a, p, out, mean, grad_out)
    E = col_t.numel()
    F, msg, p_mode, lo, hi = _softmax_aggr_args(x, a, p, message, E, (clamp_min, clamp_max))
    if want_grad_p and p is None:
        raise ValueError("grad_p needs p")
    it = _same_idx(rowptr, rowptr_t, col_t, perm_t)
    grad_out = grad_out.contiguous()
    grad_x = torch.empty_like(x)
    n_dst = out.size(0)
    grad_p = torch.empty(F, dtype=torch.float32, device=x.device) if want_grad_p else None
    pargs, _ = _plan_args(plan_t, F, x.device)
    ws = torch.empty(max(int(lib().b200mp_power_mean_workspace(n_dst, x.size(0), pargs[3], F)), 1),
                     dtype=torch.float32, device=x.device)
    _timed("power_mean_backward_src", (2 if pargs[2] else 1) + (3 if want_grad_p else 1),
           lib().b200mp_power_mean_backward_src, _p(rowptr), _p(rowptr_t), _p(col_t), _p(perm_t), _p(x), _p(a), _p(p),
           _p(out), _p(mean), _p(grad_out), _p(grad_x), _p(grad_p), _p(ws), x.size(0), n_dst, E, F, msg, float(eps),
           p_mode, lo, hi, *pargs, it, _vdt(x), _stream())
    return grad_x, grad_p


QUANTILE_INTERPOLATIONS = {"linear": 0, "lower": 1, "higher": 2, "nearest": 3, "midpoint": 4}


def _quantile_args(ref: Tensor, q: Tensor, interpolation: str) -> Tuple[int, int, int]:
    """(F, interpolation code, Q) of a quantile call: q a contiguous fp32 device tensor of Q >= 1 values."""
    if interpolation not in QUANTILE_INTERPOLATIONS:
        raise ValueError(f"interpolation must be one of {sorted(QUANTILE_INTERPOLATIONS)}, got '{interpolation}'")
    if q.dtype != torch.float32 or not q.is_contiguous() or q.numel() < 1:
        raise ValueError(f"q must be a contiguous float32 tensor of at least one value, got {tuple(q.shape)} {q.dtype}")
    _vdt(ref)
    if ref.dim() != 2 or not ref.is_contiguous():
        raise ValueError(f"the messages must be a contiguous two-dimensional tensor, got {tuple(ref.shape)}")
    return ref.size(1), QUANTILE_INTERPOLATIONS[interpolation], q.numel()


def quantile_out_dtype(dtype: torch.dtype, interpolation: str) -> torch.dtype:
    """The reference's result dtype: bf16 'linear' promotes to float32 through the fp32 frac."""
    return torch.float32 if dtype == torch.bfloat16 and interpolation == "linear" else dtype


def quantile_bits(n_edges: int, n_q: int, interpolation: str, feat: int, device) -> Tensor:
    """The pick bits of one forward: [n_edges, R * n_q, ceil(feat / 32)] int32 words (b200mp_quantile_bits_words)."""
    words = int(lib().b200mp_quantile_bits_words(n_edges, n_q, QUANTILE_INTERPOLATIONS[interpolation], feat))
    return torch.empty(max(words, 1), dtype=torch.int32, device=device)


def quantile_csr(rowptr: Tensor, col: Optional[Tensor], perm: Optional[Tensor], x: Optional[Tensor],
                 a: Optional[Tensor], q: Tensor, interpolation: str, fill_value: float, n_rows: int, n_edges: int,
                 plan: Optional[LongRowPlan] = None, want_bits: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """out[i, k F + f] = the q[k]-quantile of row i's messages in channel f (b200mp_quantile_csr): x[col[e]] or
    a[perm[e]] (perm None: a[e]).  With want_bits also the pick bits the backward reads."""
    _cuda(rowptr, col, perm, x, a, q)
    if (x is None) == (a is None):
        raise ValueError("the quantile sweep takes exactly one of x and the edge rows")
    ref = x if x is not None else a
    F, interp, Q = _quantile_args(ref, q, interpolation)
    if a is not None and a.size(0) != n_edges:
        raise ValueError(f"edge rows must have {n_edges} rows, got {a.size(0)}")
    it = _same_idx(rowptr, col, perm)
    out = torch.empty(n_rows, Q * F, dtype=quantile_out_dtype(ref.dtype, interpolation), device=ref.device)
    bits = quantile_bits(n_edges, Q, interpolation, F, ref.device) if want_bits else None
    pargs = _plan_rows(plan)
    _timed("quantile_csr", (2 if pargs[2] else 1) + int(want_bits), lib().b200mp_quantile_csr, _p(rowptr), _p(col),
           _p(perm), _p(x), _p(a), _p(q), Q, interp, float(fill_value), _p(out), _p(bits), n_rows,
           0 if x is None else x.size(0), n_edges, F, *pargs, it, _vdt(ref), _stream())
    return out, bits


def quantile_backward_dst(rowptr: Tensor, perm: Optional[Tensor], q: Tensor, interpolation: str, bits: Tensor,
                          grad_out: Tensor, n_edges: int, feat: int, dtype: torch.dtype,
                          plan: Optional[LongRowPlan] = None) -> Tensor:
    """The gradient of the edge rows [n_edges, feat] of `dtype`, in the caller's order (b200mp_quantile_backward_dst)."""
    _cuda(rowptr, perm, q, bits, grad_out)
    grad_a = torch.empty(n_edges, feat, dtype=dtype, device=grad_out.device)
    _, interp, Q = _quantile_args(grad_a, q, interpolation)
    grad_out = grad_out.to(quantile_out_dtype(dtype, interpolation)).contiguous()
    it = _same_idx(rowptr, perm)
    _timed("quantile_backward_dst", 1, lib().b200mp_quantile_backward_dst, _p(rowptr), _p(perm), _p(q), Q, interp,
           _p(bits), _p(grad_out), _p(grad_a), rowptr.numel() - 1, n_edges, feat, *_plan_rows(plan), it,
           _vdt(grad_a), _stream())
    return grad_a


def quantile_backward_src(rowptr: Tensor, rowptr_t: Tensor, col_t: Tensor, perm_t: Tensor, q: Tensor,
                          interpolation: str, bits: Tensor, grad_out: Tensor, x: Tensor,
                          plan_t: Optional[LongRowPlan] = None) -> Tensor:
    """grad_x [n_src, F] of the gathered form by one transposed sweep (b200mp_quantile_backward_src)."""
    _cuda(rowptr, rowptr_t, col_t, perm_t, q, bits, grad_out, x)
    F, interp, Q = _quantile_args(x, q, interpolation)
    grad_out = grad_out.to(quantile_out_dtype(x.dtype, interpolation)).contiguous()
    it = _same_idx(rowptr, rowptr_t, col_t, perm_t)
    grad_x = torch.empty_like(x)
    pargs, _ = _plan_args(plan_t, F, x.device)
    _timed("quantile_backward_src", 2 if pargs[2] else 1, lib().b200mp_quantile_backward_src, _p(rowptr),
           _p(rowptr_t), _p(col_t), _p(perm_t), _p(q), Q, interp, _p(bits), _p(grad_out), _p(grad_x), x.size(0),
           rowptr.numel() - 1, col_t.numel(), F, *pargs, it, _vdt(x), _stream())
    return grad_x


def scatter_coo(src: Tensor, index: Tensor, n_rows: int, reduce: str = "sum") -> Tensor:
    """Atomic COO fallback for an unsorted index; fp32, src: [E, F]."""
    _cuda(src, index)
    if src.dtype != torch.float32:
        raise TypeError("scatter_coo is fp32 only (use the CSR path for bf16)")
    src, index = src.contiguous(), index.contiguous()
    flat = src.view(src.size(0), -1)
    out = torch.empty((n_rows, flat.size(1)), dtype=torch.float32, device=src.device)
    count = torch.empty(n_rows, dtype=torch.float32, device=src.device) if REDUCE[reduce] in (1, 2, 3) else None
    check(lib().b200mp_scatter_coo(_p(flat), _p(index), _p(out), _p(count), flat.size(0), n_rows, flat.size(1),
                                   REDUCE[reduce], _idt(index), _stream()), "scatter_coo")
    return out.view((n_rows, ) + tuple(src.shape[1:]))


def scatter_arg(src: Tensor, index: Tensor, out: Tensor) -> Tensor:
    """arg[i,f] = smallest e with index[e] == i and src[e,f] == out[i,f] (src.size(0) for empty groups): the second
    output of torch_scatter.scatter_max / scatter_min for an `out` computed by scatter_coo(min / max)."""
    _cuda(src, index, out)
    if src.dtype != torch.float32 or out.dtype != torch.float32:
        raise TypeError("scatter_arg is fp32 only")
    src, index, out = src.contiguous(), index.contiguous(), out.contiguous()
    flat, oflat = src.view(src.size(0), -1), out.view(out.size(0), -1)
    arg = torch.empty(oflat.shape, dtype=torch.int64, device=src.device)
    _timed("scatter_arg", 2, lib().b200mp_scatter_arg, _p(flat), _p(index), _p(oflat), _p(arg), flat.size(0), oflat.size(0),
           flat.size(1), _idt(index), _stream())
    return arg.view(out.shape)


def spmm_csr_arg(rowptr: Tensor, col: Tensor, val: Optional[Tensor], x: Tensor, out: Tensor) -> Tensor:
    """arg[i,f] = first CSR slot of row i whose (weighted) value equals out[i,f] (nnz for empty rows): the second
    output of torch.ops.torch_sparse.spmm_min / spmm_max."""
    _cuda(rowptr, col, val, x, out)
    if x.dtype != torch.float32 or out.dtype != torch.float32:
        raise TypeError("spmm_csr_arg is fp32 only")
    it = _same_idx(rowptr, col)
    x, out = x.contiguous(), out.contiguous()
    if val is not None:
        val = val.contiguous().float()
    arg = torch.empty(out.shape, dtype=torch.int64, device=x.device)
    _timed("spmm_csr_arg", 1, lib().b200mp_spmm_csr_arg, _p(rowptr), _p(col), _p(val), _p(x), _p(out), _p(arg), out.size(0),
           out.size(1), col.numel(), it, _stream())
    return arg


def index_add_rows(out: Tensor, index: Tensor, src: Tensor) -> Tensor:
    """out[index[e], :] += src[e, :] in place (fp32, atomics)."""
    _cuda(out, index, src)
    if out.dtype != torch.float32 or src.dtype != torch.float32 or not out.is_contiguous():
        raise TypeError("index_add_rows works on contiguous fp32 tensors")
    src, index = src.contiguous(), index.contiguous()
    check(lib().b200mp_index_add_rows(_p(src), _p(index), _p(out), index.numel(), out.size(1), _idt(index),
                                      _stream()), "index_add_rows")
    return out


def gather_rows(x: Tensor, index: Tensor, scale: Optional[Tensor] = None) -> Tensor:
    _cuda(x, index, scale)
    x, index = x.contiguous(), index.contiguous()
    flat = x.view(x.size(0), -1)
    out = torch.empty((index.numel(), flat.size(1)), dtype=x.dtype, device=x.device)
    check(lib().b200mp_gather_rows(_p(flat), _p(index), _p(scale), _p(out), index.numel(), flat.size(1),
                                   _idt(index), _vdt(x), _stream()), "gather_rows")
    return out.view((index.numel(), ) + tuple(x.shape[1:]))


def _softmax_edge_op(op: int, a: Tensor, b: Optional[Tensor], row: Optional[Tensor], dst: Optional[Tensor]) -> Tensor:
    out = torch.empty_like(a)
    _timed("softmax_edge_op", 1, lib().b200mp_softmax_edge_op, op, _p(a), _p(b), _p(row), _p(dst), _p(out), a.size(0),
           a.size(1), _idt(dst) if dst is not None else I64, _stream())
    return out


def softmax_csr(src: Tensor, ptr: Tensor, plan: Optional["LongRowPlan"] = None,
                index: Optional[Tensor] = None) -> Tensor:
    """Per-group softmax over ptr ranges.  With a long-row plan (hub groups) the reference's own sequence
    -- segment max, exp(x - max), segment sum, divide (_softmax.py:82-88) -- runs on the chunked segmented
    reduce and edge-parallel kernels; otherwise one fused three-pass kernel per group."""
    _cuda(src, ptr)
    src = src.contiguous().float()
    flat = src.view(src.size(0), -1)
    if plan is not None and plan.n_long:
        if index is None:
            index = ptr2index(ptr, flat.size(0))
        mx = segment_csr(flat, ptr, "max", plan)
        ex = _softmax_edge_op(0, flat, None, mx, index)
        den = segment_csr(ex, ptr, "sum", plan)
        return _softmax_edge_op(1, ex, None, den, index).view(src.shape)
    out = torch.empty_like(flat)
    _timed("softmax_csr", 1, lib().b200mp_softmax_csr, _p(ptr), _p(flat), _p(out), ptr.numel() - 1, flat.size(0),
           flat.size(1), _idt(ptr), _stream())
    return out.view(src.shape)


def softmax_csr_backward(out: Tensor, grad_out: Tensor, ptr: Tensor, plan: Optional["LongRowPlan"] = None,
                         index: Optional[Tensor] = None) -> Tensor:
    _cuda(out, grad_out, ptr)
    out, grad_out = out.contiguous(), grad_out.contiguous().float()
    flat = out.view(out.size(0), -1)
    gflat = grad_out.view(flat.shape)
    if plan is not None and plan.n_long:
        if index is None:
            index = ptr2index(ptr, flat.size(0))
        dot = segment_csr(_softmax_edge_op(2, flat, gflat, None, None), ptr, "sum", plan)
        return _softmax_edge_op(3, flat, gflat, dot, index).view(out.shape)
    g = torch.empty_like(flat)
    _timed("softmax_csr_backward", 1, lib().b200mp_softmax_csr_backward, _p(ptr), _p(flat), _p(gflat), _p(g),
           ptr.numel() - 1, flat.size(0), flat.size(1), _idt(ptr), _stream())
    return g.view(out.shape)


def _plan_rows(plan) -> tuple:
    """(long_rows, chunk_ptr, n_long, n_chunks, chunk) for the C ABI: the plan of a sweep that splits long rows but has
    nothing to combine, so takes no partials."""
    if plan is None or not plan.n_long:
        return (None, None, 0, 0, 0)
    return (_p(plan.long_rows), _p(plan.chunk_ptr), plan.n_long, plan.n_chunks, plan.chunk)


def _plan_args(plan, feat: int, device):
    """(long_rows, chunk_ptr, n_long, n_chunks, chunk, partials[n_chunks*feat]) for the C ABI."""
    if plan is None or not plan.n_long:
        return (None, None, 0, 0, 0, None), None
    part = plan.partials(feat, device)
    return (*_plan_rows(plan), _p(part)), part


def gat_fused_csr(rowptr: Tensor, col: Tensor, xh: Tensor, a_src: Tensor, a_dst: Tensor, heads: int, chan: int,
                  slope: float, want_alpha: bool = False, plan: Optional["LongRowPlan"] = None,
                  dst_of_edge: Optional[Tensor] = None):
    """Fused GAT forward: returns (out [n_rows, H*C], row_max, row_den, alpha or None)."""
    _cuda(rowptr, col, xh, a_src, a_dst)
    it = _same_idx(rowptr, col)
    xh = xh.contiguous()
    a_src, a_dst = a_src.contiguous().float(), a_dst.contiguous().float()
    n_rows = rowptr.numel() - 1
    out = torch.empty((n_rows, heads * chan), dtype=xh.dtype, device=xh.device)
    row_max = torch.empty((n_rows, heads), dtype=torch.float32, device=xh.device)
    row_den = torch.empty_like(row_max)
    alpha = torch.empty((col.numel(), heads), dtype=torch.float32, device=xh.device) if want_alpha else None
    if want_alpha and dst_of_edge is None:
        dst_of_edge = ptr2index(rowptr, col.numel())
    pargs, _part = _plan_args(plan, heads * chan, xh.device)
    part_ms = torch.empty(plan.n_chunks * heads * 2, dtype=torch.float32, device=xh.device) if pargs[2] else None
    _timed("gat_fused_csr", 2 if pargs[2] else 1, lib().b200mp_gat_fused_csr, _p(rowptr), _p(col), _p(dst_of_edge), _p(xh),
           _p(a_src), _p(a_dst), _p(out), _p(row_max), _p(row_den), _p(alpha), n_rows, col.numel(), heads, chan,
           float(slope), *pargs, _p(part_ms), it, _vdt(xh), _stream())
    return out, row_max, row_den, alpha


def gat_fused_csr_backward(rowptr, col, dst_of_edge, rowptr_t, col_t, t2csr, xh, a_src, a_dst, row_max, row_den, out,
                           grad_out, heads: int, chan: int, slope: float, plan: Optional["LongRowPlan"] = None):
    """Returns (grad_xh [n_src, H*C], grad_a_src [n_src, H], grad_a_dst [n_rows, H])."""
    _cuda(rowptr, col, dst_of_edge, rowptr_t, col_t, t2csr, xh, grad_out)
    it = _same_idx(rowptr, col, dst_of_edge, rowptr_t, col_t, t2csr)
    grad_out = grad_out.contiguous()
    n_rows, n_src = rowptr.numel() - 1, rowptr_t.numel() - 1
    grad_pre = torch.empty((col.numel(), heads), dtype=torch.float32, device=xh.device)
    rowdot = torch.empty((n_rows, heads), dtype=torch.float32, device=xh.device)
    gxh = torch.empty_like(xh)
    gas = torch.empty((n_src, heads), dtype=torch.float32, device=xh.device)
    gad = torch.empty((n_rows, heads), dtype=torch.float32, device=xh.device)
    pargs, _part = _plan_args(plan, heads, xh.device)
    _timed("gat_fused_csr_backward", 5, lib().b200mp_gat_fused_csr_backward, _p(rowptr), _p(col), _p(dst_of_edge),
           _p(rowptr_t), _p(col_t), _p(t2csr), _p(xh), _p(a_src), _p(a_dst), _p(row_max), _p(row_den), _p(out),
           _p(grad_out), _p(grad_pre), _p(rowdot), _p(gxh), _p(gas), _p(gad), n_rows, n_src, col.numel(), heads, chan,
           float(slope), *pargs, it, _vdt(xh), _stream())
    return gxh, gas, gad


ATTN_MODES = {"gat": 0, "gatv2": 1, "dot": 2}


def attn_supported(heads: int, chan: int, dtype: torch.dtype) -> bool:
    """True when [*, heads*chan] rows of `dtype` are on the vector path of csrc/attention.cu."""
    if dtype not in (torch.float32, torch.bfloat16):
        return False
    return bool(lib().b200mp_attn_supported(heads, chan, BF16 if dtype == torch.bfloat16 else F32))


def _row_stride(t: Optional[Tensor], hc: int) -> int:
    """Row stride in elements of a [n, heads*chan] operand that may be a column slice of a wider matrix."""
    if t is None:
        return 0
    if t.dim() != 2 or t.size(1) != hc or t.stride(1) != 1:
        raise ValueError("attention operands must be [n, heads*chan] with unit inner stride")
    return t.stride(0)


def attn_forward(mode: str, rowptr: Tensor, col: Tensor, v: Tensor, heads: int, chan: int, *, k: Optional[Tensor] = None,
                 q: Optional[Tensor] = None, s_src: Optional[Tensor] = None, s_dst: Optional[Tensor] = None,
                 att: Optional[Tensor] = None, s_edge: Optional[Tensor] = None, slope: float = 0.2, scale: float = 1.0,
                 want_alpha: bool = False, plan: Optional["LongRowPlan"] = None, dropout_p: float = 0.0, dropout_seed: int = 0,
                 edge_feat: Optional[Tensor] = None):
    """Fused edge-softmax attention + aggregation (b200mp_attn_csr_forward).  v / k: [n_src, H*C] (column slices of
    a wider matrix are fine), q: [n_rows, H*C].  Returns (out, row_max, row_den, alpha or None).
    dropout_p / dropout_seed: attention dropout fused into the sweep (pass the same pair to attn_backward).
    edge_feat: [E, H*C] per-edge feature rows in CSR order (gatv2 / dot modes, `edge_dim` layers)."""
    _cuda(rowptr, col, v, k, q, s_src, s_dst, att, s_edge, edge_feat)
    if edge_feat is not None:
        if mode == "gat" or edge_feat.shape != (col.numel(), heads * chan) or edge_feat.dtype != v.dtype:
            raise ValueError("edge_feat must be [E, heads*chan] of the value dtype (gatv2 / dot modes)")
        edge_feat = edge_feat.contiguous()
    it = _same_idx(rowptr, col)
    hc = heads * chan
    n_rows = rowptr.numel() - 1
    out = torch.empty((n_rows, hc), dtype=v.dtype, device=v.device)
    row_max = torch.empty((n_rows, heads), dtype=torch.float32, device=v.device)
    row_den = torch.empty_like(row_max)
    alpha = torch.empty((col.numel(), heads), dtype=torch.float32, device=v.device) if want_alpha else None
    pargs, _part = _plan_args(plan, hc, v.device)
    part_ms = torch.empty(plan.n_chunks * heads * 2, dtype=torch.float32, device=v.device) if pargs[2] else None
    launches = 1 + (1 if pargs[2] else 0) + (1 if want_alpha else 0)
    _timed("attn_forward", launches, lib().b200mp_attn_csr_forward, ATTN_MODES[mode], _p(rowptr), _p(col), _p(v), _p(k), _p(q),
           _p(s_src), _p(s_dst), _p(att), _p(s_edge), _row_stride(v, hc), _row_stride(k, hc), _row_stride(q, hc), _p(out),
           _p(row_max), _p(row_den), _p(alpha), n_rows, col.numel(), heads, chan, float(slope), float(scale), *pargs,
           _p(part_ms), float(dropout_p), int(dropout_seed) & 0xFFFFFFFFFFFFFFFF, _p(edge_feat), it, _vdt(v), _stream())
    return out, row_max, row_den, alpha


def attn_backward(mode: str, rowptr, col, rowptr_t, col_t, t2csr, v: Tensor, heads: int, chan: int, row_max, row_den, out,
                  grad_out, *, k=None, q=None, s_src=None, s_dst=None, att=None, s_edge=None, slope: float = 0.2,
                  scale: float = 1.0, plan=None, plan_t=None, grad_v: Optional[Tensor] = None,
                  grad_k: Optional[Tensor] = None, dropout_p: float = 0.0, dropout_seed: int = 0,
                  edge_feat: Optional[Tensor] = None):
    """Backward of attn_forward.  Returns a dict with grad_v, and per mode grad_k / grad_q / grad_s_src /
    grad_s_dst / grad_att / grad_s_edge.  grad_v / grad_k may be preallocated (column slices of one matrix)."""
    _cuda(rowptr, col, rowptr_t, col_t, t2csr, v, grad_out, edge_feat)
    it = _same_idx(rowptr, col, rowptr_t, col_t, t2csr)
    grad_ef = None
    if edge_feat is not None:
        edge_feat = edge_feat.contiguous()
        grad_ef = torch.empty_like(edge_feat)
    m = ATTN_MODES[mode]
    hc = heads * chan
    dev = v.device
    n_rows, n_src, n_edges = rowptr.numel() - 1, rowptr_t.numel() - 1, col.numel()
    grad_out = grad_out.contiguous()
    out = out.contiguous()
    pair = torch.empty((n_edges, heads, 2), dtype=torch.float32, device=dev)
    if grad_v is None:
        grad_v = torch.empty((n_src, hc), dtype=v.dtype, device=dev)
    if m == 2 and grad_k is None:
        grad_k = torch.empty((n_src, hc), dtype=v.dtype, device=dev)
    if _row_stride(grad_v, hc) != _row_stride(v, hc) or (m == 2 and _row_stride(grad_k, hc) != _row_stride(k, hc)):
        raise ValueError("grad_v / grad_k must have the row stride of v / k")
    grad_q = torch.empty((n_rows, hc), dtype=v.dtype, device=dev) if m != 0 else None
    if q is not None and _row_stride(q, hc) != hc:
        q = q.contiguous()
    gss = torch.empty((n_src, heads), dtype=torch.float32, device=dev) if m == 0 else None
    gsd = torch.empty((n_rows, heads), dtype=torch.float32, device=dev) if m == 0 else None
    gatt = gatt_part = None
    if m == 1:
        gatt = torch.empty(hc, dtype=torch.float32, device=dev)
        gatt_part = torch.empty(int(lib().b200mp_attn_gatt_rows()) * hc, dtype=torch.float32, device=dev)
    w = int(lib().b200mp_attn_backward_partial_width(m, heads, chan, 0))
    wt = int(lib().b200mp_attn_backward_partial_width(m, heads, chan, 1))
    if plan is not None and plan_t is plan:   # one plan object cannot describe both the CSR and its transpose
        raise ValueError("pass distinct plans for the CSR and the transposed CSR")
    pa, _keep = _plan_args(plan, w, dev)
    pt, _keep_t = _plan_args(plan_t, wt, dev)
    _timed("attn_backward", 2 + (1 if pa[2] else 0) + (1 if pt[2] else 0) + (1 if m == 1 else 0), lib().b200mp_attn_csr_backward, m,
           _p(rowptr), _p(col), _p(rowptr_t), _p(col_t), _p(t2csr), _p(v), _p(k), _p(q), _p(s_src), _p(s_dst), _p(att),
           _p(s_edge), _row_stride(v, hc), _row_stride(k, hc), _row_stride(q, hc), _p(row_max), _p(row_den), _p(out),
           _p(grad_out), _p(pair), _p(grad_v), _p(grad_k), _p(grad_q), _p(gss), _p(gsd), _p(gatt), _p(gatt_part), n_rows,
           n_src, n_edges, heads, chan, float(slope), float(scale), pa[0], pa[1], pa[2], pa[3], pa[4], pa[5], pt[0],
           pt[1], pt[2], pt[3], pt[5], float(dropout_p), int(dropout_seed) & 0xFFFFFFFFFFFFFFFF, _p(edge_feat), _p(grad_ef), it,
           _vdt(v), _stream())
    res = {"grad_v": grad_v, "grad_k": grad_k, "grad_q": grad_q, "grad_s_src": gss, "grad_s_dst": gsd, "grad_att": gatt,
           "grad_edge_feat": grad_ef}
    if s_edge is not None:
        res["grad_s_edge"] = pair[:, :, 1]
    return res


def column_sum(x: Tensor) -> Tensor:
    """sum over rows of a [n, F] matrix in fp32 (the bias gradient); deterministic, two launches."""
    _cuda(x)
    if x.dim() != 2:
        raise ValueError("column_sum expects a 2-D matrix")
    x = x.contiguous()
    n, F = x.shape
    out = torch.empty(F, dtype=torch.float32, device=x.device)
    parts = int(lib().b200mp_column_sum_parts(n))
    ws = torch.empty(parts * max(F, 1), dtype=torch.float32, device=x.device)
    _timed("column_sum", 2, lib().b200mp_column_sum, _p(x), _p(out), _p(ws), parts, n, F, _vdt(x), _stream())
    return out


def head_dot_supported(x: Tensor, heads: int, chan: int) -> bool:
    return (x.is_cuda and x.dtype in (torch.float32, torch.bfloat16) and x.dim() == 2 and x.size(1) == heads * chan
            and bool(lib().b200mp_head_dot_supported(heads, chan, _vdt(x))))


def head_dot(x: Tensor, att_a: Tensor, att_b: Optional[Tensor], heads: int, chan: int):
    """(s_a, s_b) with s_*[n, h] = sum_c x[n, h, c] * att_*[h, c] in fp32, one read of x (b200mp_head_dot)."""
    _cuda(x, att_a, att_b)
    x = x.contiguous()
    att_a = att_a.reshape(-1).float().contiguous()
    att_b = None if att_b is None else att_b.reshape(-1).float().contiguous()
    n = x.size(0)
    s_a = torch.empty(n, heads, dtype=torch.float32, device=x.device)
    s_b = None if att_b is None else torch.empty(n, heads, dtype=torch.float32, device=x.device)
    _timed("head_dot", 1, lib().b200mp_head_dot, _p(x), _p(att_a), _p(att_b), _p(s_a), _p(s_b), n, heads, chan, _vdt(x),
           _stream())
    return s_a, s_b


def head_dot_backward(x: Tensor, att_a: Tensor, att_b: Optional[Tensor], g_a: Tensor, g_b: Optional[Tensor],
                      add: Optional[Tensor], heads: int, chan: int, want_grad_x: bool = True):
    """(grad_x, grad_att_a, grad_att_b): grad_x = g_a (x) att_a + g_b (x) att_b (+ add), grad_att_* fp32 [heads*chan]."""
    _cuda(x, att_a, att_b, g_a, g_b, add)
    x = x.contiguous()
    att_a = att_a.reshape(-1).float().contiguous()
    att_b = None if att_b is None else att_b.reshape(-1).float().contiguous()
    g_a = g_a.float().contiguous()
    g_b = None if g_b is None else g_b.float().contiguous()
    if add is not None:
        add = add.to(x.dtype).contiguous()
    n, F = x.shape
    gx = torch.empty_like(x) if want_grad_x else None
    parts = int(lib().b200mp_head_dot_parts(n, heads, chan, _vdt(x)))
    if parts == 0:
        z = torch.zeros(F, dtype=torch.float32, device=x.device)
        return gx, z, (None if att_b is None else z.clone())
    pa = torch.empty(parts, F, dtype=torch.float32, device=x.device)
    pb = None if att_b is None else torch.empty(parts, F, dtype=torch.float32, device=x.device)
    _timed("head_dot_backward", 1, lib().b200mp_head_dot_backward, _p(x), _p(att_a), _p(att_b), _p(g_a), _p(g_b), _p(add),
           _p(gx), _p(pa), _p(pb), parts, n, heads, chan, _vdt(x), _stream())
    return gx, column_sum(pa), (None if pb is None else column_sum(pb))


MULTI_AGGRS = ("sum", "mean", "min", "max", "var", "std")
MULTI_HIT_MASK = True       # emit the forward's hit bits for the backward (A/B switch for benchmarks)


def multi_aggr_csr(rowptr: Tensor, col: Optional[Tensor], x: Tensor, n_rows: int, want, plan=None,
                   with_ties: bool = False, count_self_zero: bool = True) -> dict:
    """Every aggregation named in `want` (subset of MULTI_AGGRS) from one sweep over the CSR rows.
    col=None: segment mode (x is the destination-sorted [E, F] message matrix).  Returns a dict
    name -> [n_rows, F]; with_ties adds fp32 'ties_min' / 'ties_max' when min / max are wanted."""
    _cuda(rowptr, col, x)
    if x.dim() != 2:
        raise ValueError("multi_aggr_csr expects a 2-D feature matrix")
    x = x.contiguous()
    it = _same_idx(rowptr, col) if col is not None else _idt(rowptr)
    F = x.size(1)
    res = {}
    for name in want:
        if name not in MULTI_AGGRS:
            raise ValueError(f"cannot fuse aggregation '{name}' (supported: {MULTI_AGGRS})")
        res[name] = torch.empty(n_rows, F, dtype=x.dtype, device=x.device)
    if with_ties:
        for name in ("min", "max"):
            if name in res:
                res["ties_" + name] = torch.empty(n_rows, F, dtype=torch.float32, device=x.device)
    # hit bits for the backward (one byte per edge and 16-byte vector): only where its masked kernel exists
    if (MULTI_HIT_MASK and with_ties and col is not None and ("ties_min" in res or "ties_max" in res)
            and lib().b200mp_multi_aggr_mask_supported(F, _vdt(x), 0)):
        res["hit_mask"] = torch.empty(col.numel() * (F // 4), dtype=torch.uint8, device=x.device)
    pargs, _ = _plan_args(plan, 6 * F, x.device)
    _timed("multi_aggr_csr", (3 if "hit_mask" in res else 2) if pargs[2] else 1, lib().b200mp_multi_aggr_csr, _p(rowptr),
           _p(col), _p(x), *[_p(res.get(n)) for n in MULTI_AGGRS], _p(res.get("ties_min")), _p(res.get("ties_max")),
           _p(res.get("hit_mask")), n_rows, x.size(0), F, int(bool(count_self_zero)), *pargs, it, _vdt(x), _stream())
    return res


def multi_aggr_prepare_backward(rowptr: Tensor, grads: dict, mean: Optional[Tensor], std: Optional[Tensor],
                                ties_min: Optional[Tensor], ties_max: Optional[Tensor], semi_grad: bool):
    """(term_a, term_b, g_min / ties_min, g_max / ties_max) for multi_aggr_backward from the output
    gradients `grads` (name -> [n_rows, F] or None), in one elementwise kernel."""
    ref = next(g for g in grads.values() if g is not None)
    n_rows, F = ref.shape
    g = {k: (None if v is None else v.contiguous()) for k, v in grads.items()}
    _cuda(rowptr, *g.values(), mean, std, ties_min, ties_max)

    def new():
        return torch.empty(n_rows, F, dtype=torch.float32, device=ref.device)

    need_a = any(g.get(k) is not None for k in ("sum", "mean", "var", "std"))
    need_b = any(g.get(k) is not None for k in ("var", "std"))
    term_a = new() if need_a else None
    term_b = new() if need_b else None
    gmin = new() if g.get("min") is not None else None
    gmax = new() if g.get("max") is not None else None
    _timed("multi_aggr_prepare_backward", 1, lib().b200mp_multi_aggr_prepare_backward, _p(rowptr), _p(g.get("sum")),
           _p(g.get("mean")), _p(g.get("var")), _p(g.get("std")), _p(g.get("min")), _p(g.get("max")), _p(mean),
           _p(std), _p(ties_min), _p(ties_max), _p(term_a), _p(term_b), _p(gmin), _p(gmax), n_rows, F,
           int(bool(semi_grad)), _idt(rowptr), _vdt(ref), _stream())
    return term_a, (None if semi_grad else term_b), gmin, gmax


def multi_aggr_backward(ptr: Optional[Tensor], idx: Tensor, x: Tensor, term_a: Optional[Tensor],
                        term_b: Optional[Tensor], out_min: Optional[Tensor], g_min: Optional[Tensor],
                        out_max: Optional[Tensor], g_max: Optional[Tensor], segment_mode: bool,
                        hit_mask: Optional[Tensor] = None, t2csr: Optional[Tensor] = None) -> Tensor:
    """grad wrt the message values (see b200mp_multi_aggr_backward).  segment_mode: idx = destination of
    every message; otherwise (ptr, idx) is the transposed CSR and x the [n_src, F] source matrix.
    hit_mask / t2csr: the forward's hit bits (multi_aggr_csr's 'hit_mask') and the CSR slot of every transposed slot."""
    _cuda(ptr, idx, x, term_a, term_b, out_min, g_min, out_max, g_max, hit_mask, t2csr)
    if hit_mask is not None:
        if t2csr is None or segment_mode or t2csr.dtype != idx.dtype:
            raise ValueError("hit_mask needs gather mode and t2csr of the index dtype")
        t2csr = t2csr.contiguous()
    x = x.contiguous()

    def f32(t):
        return None if t is None else t.contiguous().float()

    term_a, term_b, g_min, g_max = f32(term_a), f32(term_b), f32(g_min), f32(g_max)
    out_min = None if out_min is None else out_min.contiguous()
    out_max = None if out_max is None else out_max.contiguous()
    gx = torch.empty_like(x)
    it = _idt(idx) if segment_mode else _same_idx(ptr, idx)
    _timed("multi_aggr_backward", 1, lib().b200mp_multi_aggr_backward, _p(ptr), _p(idx), _p(x), _p(term_a),
           _p(term_b), _p(out_min), _p(g_min), _p(out_max), _p(g_max), _p(hit_mask), _p(t2csr), _p(gx), x.size(0), x.size(1),
           int(bool(segment_mode)), it, _vdt(x), _stream())
    return gx


PNA_AGGRS = ("sum", "mean", "min", "max", "var", "std")
PNA_SCALERS = ("identity", "amplification", "attenuation", "linear", "inverse_linear")


def _host_codes(names, table):
    """int32 host array of the codes of `names` in `table` (the C ABI reads it during the call)."""
    return (ctypes.c_int32 * len(names))(*[table.index(n) for n in names])


def _pna_stats_args(stats: dict):
    return [_p(stats.get(k)) for k in ("sum", "min", "max", "var")]


def _pna_stats_dtype(stats: dict, ref: Tensor) -> int:
    ts = [t for k, t in stats.items() if k in ("sum", "min", "max", "var") and t is not None]
    return _vdt(ts[0]) if ts else _vdt(ref)


def pna_epilogue(rowptr: Tensor, x: Tensor, u: Tensor, stats: dict, aggrs, scalers, avg_deg_lin: Tensor,
                 avg_deg_log: Tensor, towers: int) -> Tensor:
    """[N, towers, (1 + A S) F] = cat([x_t, scaler_1(aggr_1 .. aggr_A), ...]) per tower from the statistics of w
    (`stats`: 'sum' / 'min' / 'max' / 'var' planes [N, W]) shifted by u ([N, W], row stride u.stride(0)); x: [N, W]."""
    _cuda(rowptr, x, u, avg_deg_lin, avg_deg_log, *stats.values())
    N, W = x.shape
    F = W // towers
    if u.stride(1) != 1:
        u = u.contiguous()
    out = torch.empty(N, towers, (1 + len(aggrs) * len(scalers)) * F, dtype=x.dtype, device=x.device)
    ac, sc = _host_codes(aggrs, PNA_AGGRS), _host_codes(scalers, PNA_SCALERS)
    _timed("pna_epilogue", 1, lib().b200mp_pna_epilogue, _p(rowptr), _p(x.contiguous()), _p(u), u.stride(0),
           *_pna_stats_args(stats), ctypes.addressof(ac), len(aggrs), ctypes.addressof(sc),
           len(scalers), _p(avg_deg_lin), _p(avg_deg_log), _p(out), N, towers, F, _pna_stats_dtype(stats, x),
           _idt(rowptr), _vdt(x), _stream())
    return out


def pna_prologue(rowptr: Tensor, grad_out: Tensor, u: Tensor, stats: dict, aggrs, scalers, avg_deg_lin: Tensor,
                 avg_deg_log: Tensor, towers: int, want_u: bool, want_x: bool, want_avg: bool, grad_u: Optional[Tensor] = None):
    """Backward prologue of pna_epilogue: dict with the fp32 [N, W] rows the sweep backward reads ('term_a', 'term_b',
    'gmin', 'gmax', each present only when an aggregator needs it), 'grad_u' (written into `grad_u` when given, e.g.
    the left half of an [N, 2W] gradient), 'grad_x' [N, W] and 'avg' = (d L / d avg_deg_lin, d L / d avg_deg_log)."""
    _cuda(rowptr, grad_out, u, avg_deg_lin, avg_deg_log, *stats.values())
    grad_out = grad_out.contiguous()
    N = grad_out.size(0)
    W = u.size(1)
    F = W // towers
    dev = grad_out.device
    new = lambda: torch.empty(N, W, dtype=torch.float32, device=dev)       # noqa: E731
    res = {
        "term_a": new() if any(a in aggrs for a in ("sum", "mean", "var", "std")) else None,
        "term_b": new() if any(a in aggrs for a in ("var", "std")) else None,
        "gmin": new() if "min" in aggrs else None,
        "gmax": new() if "max" in aggrs else None,
    }
    if want_u and grad_u is None:
        grad_u = torch.empty(N, W, dtype=grad_out.dtype, device=dev)
    res["grad_u"] = grad_u if want_u else None
    res["grad_x"] = torch.empty(N, W, dtype=grad_out.dtype, device=dev) if want_x else None
    part = torch.empty(N, 2, dtype=torch.float32, device=dev) if want_avg else None
    if u.stride(1) != 1:
        u = u.contiguous()
    gu = res["grad_u"]
    ac, sc = _host_codes(aggrs, PNA_AGGRS), _host_codes(scalers, PNA_SCALERS)
    _timed("pna_prologue", 1, lib().b200mp_pna_prologue, _p(rowptr), _p(grad_out), _p(u), u.stride(0),
           *_pna_stats_args(stats), _p(stats.get("ties_min")), _p(stats.get("ties_max")),
           ctypes.addressof(ac), len(aggrs), ctypes.addressof(sc), len(scalers),
           _p(avg_deg_lin), _p(avg_deg_log), _p(res["term_a"]), _p(res["term_b"]), _p(res["gmin"]), _p(res["gmax"]),
           _p(gu), gu.stride(0) if gu is not None else W, _p(res["grad_x"]), _p(part), N, towers, F,
           _pna_stats_dtype(stats, grad_out), _idt(rowptr), _vdt(grad_out), _stream())
    res["avg"] = None if part is None else column_sum(part)
    return res


def pna_edge_stats(rowptr: Tensor, col: Tensor, perm: Optional[Tensor], v: Tensor, c: Tensor, n_rows: int, aggrs,
                   plan: Optional[LongRowPlan] = None, with_ties: bool = False) -> dict:
    """fp32 statistics of w_e = v[col[e]] + c[perm[e]] per destination row ('sum', 'min', 'max', 'var', and with_ties
    'ties_min' / 'ties_max'), only those the aggregators need.  v: [n_cols, W] (row stride v.stride(0)); c: [E, W]
    in the caller's edge order."""
    _cuda(rowptr, col, perm, v, c)
    W = v.size(1)
    if v.stride(1) != 1:
        v = v.contiguous()
    c = c.contiguous()
    need = _pna_need(aggrs)
    st = {k: torch.empty(n_rows, W, dtype=torch.float32, device=v.device) for k in need}
    if with_ties:
        for k in ("min", "max"):
            if k in st:
                st["ties_" + k] = torch.empty(n_rows, W, dtype=torch.float32, device=v.device)
    pargs, _ = _plan_args(plan, 6 * W, v.device)
    _timed("pna_edge_stats", 2 if pargs[2] else 1, lib().b200mp_pna_edge_stats, _p(rowptr), _p(col), _p(perm), _p(v),
           v.stride(0), _p(c), _p(st.get("sum")), _p(st.get("min")), _p(st.get("max")), _p(st.get("var")),
           _p(st.get("ties_min")), _p(st.get("ties_max")), n_rows, v.size(0), col.numel(), W, *pargs,
           _same_idx(rowptr, col, perm), _vdt(v), _stream())
    return st


def _pna_need(aggrs) -> tuple:
    """The statistics of w an aggregator list reads."""
    need = []
    if any(a in aggrs for a in ("sum", "mean", "var", "std")):
        need.append("sum")
    need += [a for a in ("min", "max") if a in aggrs]
    if any(a in aggrs for a in ("var", "std")):
        need.append("var")
    return tuple(need)


def pna_edge_backward(rowptr_t: Tensor, col_t: Tensor, perm_t: Tensor, v: Tensor, c: Tensor, terms: dict, stats: dict,
                      n_dst: int, grad_v: Optional[Tensor], want_c: bool) -> Optional[Tensor]:
    """One transposed-CSR sweep: d L / d w_e into grad_c [E, W] (caller's order, returned when want_c) and its sum over
    every source's out-edges into grad_v (written in place, row stride grad_v.stride(0); may be None)."""
    _cuda(rowptr_t, col_t, perm_t, v, c, grad_v)
    W = v.size(1)
    if v.stride(1) != 1:
        v = v.contiguous()
    c = c.contiguous()
    E = c.size(0)
    grad_c = torch.empty(E, W, dtype=c.dtype, device=c.device) if want_c else None
    _timed("pna_edge_backward", 1, lib().b200mp_pna_edge_backward, _p(rowptr_t), _p(col_t), _p(perm_t), _p(v),
           v.stride(0), _p(c), _p(terms.get("term_a")), _p(terms.get("term_b")), _p(stats.get("min")),
           _p(terms.get("gmin")), _p(stats.get("max")), _p(terms.get("gmax")), _p(grad_v),
           grad_v.stride(0) if grad_v is not None else W, _p(grad_c), v.size(0), n_dst, E, W,
           _same_idx(rowptr_t, col_t, perm_t), _vdt(v), _stream())
    return grad_c


def device_info() -> dict:
    import ctypes
    sm, ma, mi, l2 = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int64()
    check(lib().b200mp_device_info(ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi), ctypes.byref(l2)))
    return {"sm_count": sm.value, "cc": (ma.value, mi.value), "l2_bytes": l2.value}


def set_option(name: str, value: int) -> None:
    """Runtime switches of the library (b200mp_set_option), e.g. set_option("spmm_impl", 1)."""
    check(lib().b200mp_set_option(name.encode(), int(value)), "set_option")
