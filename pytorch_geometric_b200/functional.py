"""Differentiable front ends of the hot path (custom autograd over the C-ABI kernels).

`aggregate(graph, x, reduce, edge_weight)` is the fused replacement for the reference's
collect -> message -> aggregate sequence (nn/conv/message_passing.py:421-563) and for
`EdgeIndex.matmul` / `spmm` (edge_index.py:1925-1970, utils/_spmm.py:12-136).
Backward follows `_TorchSPMM.backward` (edge_index.py:1860-1900): the same kernel on the
transposed CSR; min/max use the ATen tie rule (oracle_scatter_backward in oracle/mp_oracle.c).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from . import dense, ops
from .graph import CSRGraph


class _Aggregate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, edge_weight: Optional[Tensor], graph: CSRGraph, reduce: str):
        val = graph.val
        if edge_weight is not None:
            val = graph.to_csr_order(edge_weight.detach().float().contiguous().view(-1))
        out = ops.spmm_csr(graph.rowptr, graph.col, val, x, graph.num_dst, reduce, graph.plan)
        ctx.graph, ctx.reduce = graph, reduce
        ctx.has_ew = edge_weight is not None
        need_x = reduce in ("min", "max") or (ctx.has_ew and edge_weight.requires_grad)
        ctx.save_for_backward(x if need_x else None, out if reduce in ("min", "max") else None, val)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        graph, reduce = ctx.graph, ctx.reduce
        x, out, val = ctx.saved_tensors
        grad_out = grad_out.contiguous()
        graph.build_transpose()
        gx = gw = None
        val_t = None
        if val is not None:
            val_t = graph.val_t if (not ctx.has_ew and graph.val_t is not None) else \
                graph.to_csc_order(graph.from_csr_order(val))
        if ctx.needs_input_grad[0]:
            if reduce in ("sum", "add"):
                gx = ops.spmm_csr(graph.rowptr_t, graph.col_t, val_t, grad_out, graph.num_src, "sum", graph.plan_t)
            elif reduce == "mean":
                mv = graph.mean_val_t()
                if val_t is not None:
                    mv = mv * val_t
                gx = ops.spmm_csr(graph.rowptr_t, graph.col_t, mv, grad_out, graph.num_src, "sum", graph.plan_t)
            else:  # min / max
                ties = ops.minmax_ties(graph.rowptr, graph.col, val, x, out, count_self_zero=True)
                gx = ops.minmax_backward(graph.rowptr_t, graph.col_t, val_t, x, out, grad_out, ties)
        if ctx.has_ew and ctx.needs_input_grad[1]:
            if reduce not in ("sum", "add", "mean"):
                raise NotImplementedError("gradient wrt edge_weight is implemented for sum/mean only")
            g = grad_out
            dot = ops.sddmm_csr(graph.rowptr, graph.col, g, x)          # CSR order
            if reduce == "mean":
                inv = 1.0 / graph.in_degree().clamp(min=1).to(torch.float32)
                dot = dot * ops.gather_rows(inv.view(-1, 1), graph.dst_csr).view(-1)
            gw = graph.from_csr_order(dot)
        return gx, gw, None, None


def aggregate(graph: CSRGraph, x: Tensor, reduce: str = "sum", edge_weight: Optional[Tensor] = None) -> Tensor:
    """out[i] = REDUCE_{(j -> i)} w_ji * x[j]; x: [num_src, F] -> [num_dst, F].

    `edge_weight` (original edge order, may require grad) overrides the static values cached in
    the graph (e.g. gcn_norm weights).  Empty destinations give 0 for every reduce.
    """
    if reduce not in ("sum", "add", "mean", "min", "max"):
        raise ValueError(f"Encountered invalid `reduce` argument '{reduce}'")
    if x.dim() == 1:
        return aggregate(graph, x.view(-1, 1), reduce, edge_weight).view(-1)
    if x.dim() > 2:
        shape = x.shape[1:]
        return aggregate(graph, x.reshape(x.size(0), -1), reduce, edge_weight).view((graph.num_dst, ) + shape)
    if x.size(0) != graph.num_src:
        raise ValueError(f"x has {x.size(0)} rows but the graph has {graph.num_src} source nodes")
    return _Aggregate.apply(x, edge_weight, graph, reduce)


class _AggregateEdgeReLU(torch.autograd.Function):
    """relu(x_j + e_ji) reduced by sum / mean (csrc/edge_relu.cu).  The forward keeps one ReLU bit per (edge, feature)
    when a gradient is needed; backward = a transposed-CSR sweep for x and, when asked for, a destination sweep that
    writes the edge-row gradient in the caller's order."""

    @staticmethod
    def forward(ctx, x: Tensor, edge_rows: Tensor, graph: CSRGraph, reduce: str):
        want_mask = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        out, mask = ops.edge_relu_csr(graph.rowptr, graph.col, graph.perm, x, edge_rows, graph.num_dst, reduce,
                                      graph.plan, want_mask=want_mask)
        ctx.graph, ctx.reduce = graph, reduce
        ctx.save_for_backward(mask)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        mask, = ctx.saved_tensors
        graph, reduce = ctx.graph, ctx.reduce
        gx = ga = None
        if ctx.needs_input_grad[0]:
            graph.build_transpose()
            val_t = graph.mean_val_t() if reduce == "mean" else None
            gx = ops.edge_relu_backward_x(graph.rowptr_t, graph.col_t, graph.t2csr, val_t, grad_out, mask, graph.num_src,
                                          graph.plan_t)
        if ctx.needs_input_grad[1]:
            ga = ops.edge_relu_backward_edge(graph.rowptr, graph.perm, grad_out, mask, graph.num_edges, reduce, graph.plan)
        return gx, ga, None, None


def aggregate_edge_relu(graph: CSRGraph, x: Tensor, edge_rows: Tensor, reduce: str = "sum") -> Tensor:
    """out[i] = REDUCE_{e = (j -> i)} relu(x[j] + edge_rows[e]) for reduce in {sum, mean}: GINEConv's message and
    aggregation (gin_conv.py:195-204) without any [E, F] intermediate.  x: [num_src, *], edge_rows: [E, *] with the
    same trailing shape and dtype, in the caller's edge order; both may require grad.  Empty destinations give 0."""
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"aggregate_edge_relu reduces by sum or mean, got '{reduce}'")
    if edge_rows.dtype != x.dtype:
        raise TypeError(f"edge_rows ({edge_rows.dtype}) and x ({x.dtype}) must share a dtype")
    if tuple(edge_rows.shape) != (graph.num_edges, ) + tuple(x.shape[1:]):
        raise ValueError(f"edge_rows must have shape {(graph.num_edges, ) + tuple(x.shape[1:])}, "
                         f"got {tuple(edge_rows.shape)}")
    if x.dim() == 1:
        return aggregate_edge_relu(graph, x.view(-1, 1), edge_rows.view(-1, 1), reduce).view(-1)
    if x.size(0) != graph.num_src:
        raise ValueError(f"x has {x.size(0)} rows but the graph has {graph.num_src} source nodes")
    shape = x.shape[1:]
    x2 = x.reshape(x.size(0), -1)
    out = _AggregateEdgeReLU.apply(x2, edge_rows.reshape(graph.num_edges, x2.size(1)), graph,
                                   "mean" if reduce == "mean" else "sum")
    return out.view((graph.num_dst, ) + tuple(shape))


class _AggregateGated(torch.autograd.Function):
    """sigmoid(k_i + q_j) * v_j reduced by sum / mean (csrc/gated.cu).  Nothing per edge is saved: the backward
    recomputes the gate from k and q.  grad_k is a destination sweep, grad_q and grad_v one transposed-CSR sweep; each
    runs only when one of its inputs needs a gradient.  `v` None means `q` is one [N, 2F] tensor holding q | v."""

    @staticmethod
    def forward(ctx, k: Tensor, q: Tensor, v: Optional[Tensor], graph: CSRGraph, reduce: str):
        F = k.size(1)
        qq, vv = (q, v) if v is not None else (q[:, :F], q[:, F:])
        out = ops.gated_csr(graph.rowptr, graph.col, k, qq, vv, graph.num_dst, reduce, graph.plan)
        ctx.graph, ctx.reduce, ctx.split = graph, reduce, v is None
        ctx.save_for_backward(k, q, v)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        k, q, v = ctx.saved_tensors
        graph, reduce = ctx.graph, ctx.reduce
        F = k.size(1)
        qq, vv = (q[:, :F], q[:, F:]) if ctx.split else (q, v)
        gk = gq = gv = None
        if ctx.needs_input_grad[0]:
            gk = ops.gated_backward_dst(graph.rowptr, graph.col, k, qq, vv, grad_out, reduce, graph.plan)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            graph.build_transpose()
            val_t = graph.mean_val_t() if reduce == "mean" else None
            gq = torch.empty_like(q)
            gv = None if ctx.split else torch.empty_like(v)
            ops.gated_backward_src(graph.rowptr_t, graph.col_t, val_t, k, qq, vv, grad_out,
                                   gq[:, :F] if ctx.split else gq, gq[:, F:] if ctx.split else gv, graph.plan_t)
        return gk, gq, gv, None, None


def _gated_check(graph: CSRGraph, k: Tensor, q: Tensor, reduce: str, name: str) -> None:
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"{name} reduces by sum or mean, got '{reduce}'")
    if q.dtype != k.dtype:
        raise TypeError(f"q ({q.dtype}) and k ({k.dtype}) must share a dtype")
    if k.size(0) != graph.num_dst:
        raise ValueError(f"k has {k.size(0)} rows but the graph has {graph.num_dst} destination nodes")
    if q.size(0) != graph.num_src:
        raise ValueError(f"q has {q.size(0)} rows but the graph has {graph.num_src} source nodes")


def aggregate_gated(graph: CSRGraph, k: Tensor, q: Tensor, v: Tensor, reduce: str = "sum") -> Tensor:
    """out[i] = REDUCE_{e = (j -> i)} sigmoid(k[i] + q[j]) * v[j] for reduce in {sum, mean}: ResGatedGraphConv's
    message and aggregation (res_gated_graph_conv.py:138-148) without any [E, F] intermediate.  k: [num_dst, *];
    q, v: [num_src, *] with k's trailing shape and dtype; all three may require grad.  Empty destinations give 0."""
    _gated_check(graph, k, q, reduce, "aggregate_gated")
    if v.dtype != k.dtype:
        raise TypeError(f"v ({v.dtype}) and k ({k.dtype}) must share a dtype")
    if q.shape[1:] != k.shape[1:] or v.shape != q.shape:
        raise ValueError(f"q and v must have shape {(graph.num_src, ) + tuple(k.shape[1:])}, "
                         f"got {tuple(q.shape)} and {tuple(v.shape)}")
    if k.dim() == 1:
        return aggregate_gated(graph, k.view(-1, 1), q.view(-1, 1), v.view(-1, 1), reduce).view(-1)
    shape = k.shape[1:]
    k2 = k.reshape(k.size(0), -1).contiguous()
    q2 = q.reshape(q.size(0), -1).contiguous()
    v2 = v.reshape(v.size(0), -1).contiguous()
    out = _AggregateGated.apply(k2, q2, v2, graph, "mean" if reduce == "mean" else "sum")
    return out.view((graph.num_dst, ) + tuple(shape))


def aggregate_gated_qv(graph: CSRGraph, k: Tensor, qv: Tensor, reduce: str = "sum") -> Tensor:
    """aggregate_gated with q and v as the two halves of one [num_src, 2F] tensor (one product with the concatenated
    query / value weights), read in place; its gradient is one [num_src, 2F] tensor as well.  k: [num_dst, F]."""
    _gated_check(graph, k, qv, reduce, "aggregate_gated_qv")
    if k.dim() != 2 or qv.dim() != 2 or qv.size(1) != 2 * k.size(1):
        raise ValueError(f"k must be [num_dst, F] and qv [num_src, 2F], got {tuple(k.shape)} and {tuple(qv.shape)}")
    return _AggregateGated.apply(k.contiguous(), qv.contiguous(), None, graph, "mean" if reduce == "mean" else "sum")


class _AggregateCG(torch.autograd.Function):
    """sigmoid(f) * softplus(s) reduced by sum / mean, [f | s] = u_i + v_j (+ c_e) (csrc/cg.cu).  Nothing per edge is
    saved: the backward recomputes f and s.  The destination sweep gives grad_u and, when c needs a gradient, grad_c;
    grad_v is then the segment sum of grad_c's rows over the transposed CSR, and otherwise one transposed sweep.  Each
    sweep runs only when one of its outputs is needed.  `v` None means `u` is one [N, 4F] tensor holding u | v."""

    @staticmethod
    def forward(ctx, u: Tensor, v: Optional[Tensor], c: Optional[Tensor], graph: CSRGraph, reduce: str):
        W = u.size(1) // (2 if v is None else 1)
        uu, vv = (u, v) if v is not None else (u[:, :W], u[:, W:])
        out = ops.cg_csr(graph.rowptr, graph.col, graph.perm, uu, vv, c, graph.num_dst, reduce, graph.plan)
        ctx.graph, ctx.reduce, ctx.packed = graph, reduce, v is None
        ctx.save_for_backward(u, v, c)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        u, v, c = ctx.saved_tensors
        graph, reduce, packed = ctx.graph, ctx.reduce, ctx.packed
        W = u.size(1) // (2 if packed else 1)
        uu, vv = (u[:, :W], u[:, W:]) if packed else (u, v)
        need_u, need_c = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        need_v = need_u if packed else ctx.needs_input_grad[1]
        grad_out = grad_out.contiguous()
        gu = gv = gc = None
        gu_dst = gv_dst = None                         # where the sweeps write: u's and v's shape and row stride
        if packed:
            if need_u or need_c:
                full = torch.empty_like(u)
                gu_dst, gv_dst = full[:, :W], full[:, W:]
                gu = full if need_u else None
        else:
            if need_u or need_c:
                gu_dst = torch.empty_like(u)
                gu = gu_dst if need_u else None
        if need_u or need_c:
            gc = ops.cg_backward_dst(graph.rowptr, graph.col, graph.perm, uu, vv, c, grad_out, gu_dst, need_c, reduce,
                                     graph.plan)
        if need_v:
            graph.build_transpose()
            if gc is not None:
                # grad_v[j] = the sum of grad_c over j's out-edges: perm_t is the caller's edge id of each transposed slot
                sums = ops.spmm_csr(graph.rowptr_t, graph.perm_t, None, gc, graph.num_src, "sum", graph.plan_t)
                if packed:
                    gv_dst.copy_(sums)
                else:
                    gv = sums
            else:
                if not packed:
                    gv = gv_dst = torch.empty_like(v)
                val_t = graph.mean_val_t() if reduce == "mean" else None
                ops.cg_backward_src(graph.rowptr_t, graph.col_t, graph.perm_t, val_t, uu, vv, c, grad_out, gv_dst,
                                    graph.plan_t)
        return gu, gv, gc, None, None


def _cg_check(graph: CSRGraph, u: Tensor, c: Optional[Tensor], reduce: str, width: int, name: str) -> None:
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"{name} reduces by sum or mean, got '{reduce}'")
    if u.dim() != 2 or u.size(1) % width:
        raise ValueError(f"{name}: u must be a [num_dst, {width}F] tensor, got {tuple(u.shape)}")
    if u.size(0) != graph.num_dst:
        raise ValueError(f"u has {u.size(0)} rows but the graph has {graph.num_dst} destination nodes")
    F = u.size(1) // width
    if c is not None and (tuple(c.shape) != (graph.num_edges, 2 * F) or c.dtype != u.dtype):
        raise ValueError(f"c must be a [{graph.num_edges}, {2 * F}] tensor of u's dtype, got {tuple(c.shape)} {c.dtype}")


def aggregate_cg(graph: CSRGraph, u: Tensor, v: Tensor, c: Optional[Tensor] = None, reduce: str = "sum") -> Tensor:
    """out[i] = REDUCE_{e = (j -> i)} sigmoid(f_e) * softplus(s_e) for reduce in {sum, mean}, with [f_e | s_e] =
    u[i] + v[j] (+ c[e]): CGConv's message and aggregation (cg_conv.py:93-98) with its two Linears split by weight
    column blocks (`nn.conv.cg_uvc`).  u: [num_dst, 2F] (f half, then s half); v: [num_src, 2F]; c: [E, 2F] in the
    caller's edge order or None; one dtype; all three may require grad.  Returns [num_dst, F]; empty rows give 0."""
    _cg_check(graph, u, c, reduce, 2, "aggregate_cg")
    if v.dtype != u.dtype or v.shape != (graph.num_src, u.size(1)):
        raise ValueError(f"v must be a [{graph.num_src}, {u.size(1)}] tensor of u's dtype, got {tuple(v.shape)} {v.dtype}")
    return _AggregateCG.apply(u.contiguous(), v.contiguous(), None if c is None else c.contiguous(), graph,
                              "mean" if reduce == "mean" else "sum")


def aggregate_cg_uv(graph: CSRGraph, uv: Tensor, c: Optional[Tensor] = None, reduce: str = "sum") -> Tensor:
    """aggregate_cg with u and v as the two halves of one [N, 4F] tensor (one product of a non-bipartite layer), read
    in place; its gradient is one [N, 4F] tensor as well.  The graph must have N sources and N destinations."""
    _cg_check(graph, uv, c, reduce, 4, "aggregate_cg_uv")
    if graph.num_src != graph.num_dst:
        raise ValueError(f"aggregate_cg_uv needs as many sources as destinations, got {graph.num_src} and {graph.num_dst}")
    return _AggregateCG.apply(uv.contiguous(), None, None if c is None else c.contiguous(), graph,
                              "mean" if reduce == "mean" else "sum")


NN_CONV_BLOCK_BYTES = 1 << 29     # fp32 bytes of P = [rows, (K+1) F_in] held at once by nn_conv_aggregate


def _nn_conv_blocks(n_dst: int, width: int):
    """Destination row ranges [r0, r1) whose P fits NN_CONV_BLOCK_BYTES (at least one row each)."""
    rows = max(1, NN_CONV_BLOCK_BYTES // (4 * width))
    return [(r0, min(r0 + rows, n_dst)) for r0 in range(0, n_dst, rows)]


class _NNConvAggregate(torch.autograd.Function):
    """out = P W' by destination-row blocks, P_i = REDUCE_e [h_e, 1] (x) x_j (csrc/nn_conv.cu).  Nothing of size
    N (K+1) F_in is saved: the backward recomputes each block's P for dW' = sum_b P_b^T G_b, forms dP_b = G_b W'^T for
    the destination sweep (grad_h and q per edge), and grad_x is one segment sum of q over the transposed CSR.  Each
    step runs only when one of its outputs is needed.  P, W' and the GEMMs are fp32; the output has x's dtype."""

    @staticmethod
    def forward(ctx, x: Tensor, h: Tensor, w_prime: Tensor, graph: CSRGraph, reduce: str):
        width = w_prime.size(0)
        w = w_prime.detach().float().contiguous()
        out = torch.zeros(graph.num_dst, w.size(1), dtype=torch.float32, device=x.device)
        for r0, r1 in _nn_conv_blocks(graph.num_dst, width):
            p = ops.nn_conv_csr(graph.rowptr, graph.col, graph.perm, x, h, r0, r1, reduce, graph.plan)
            out[r0:r1] = dense._mm(p, w)
        ctx.graph, ctx.reduce = graph, reduce
        ctx.save_for_backward(x, h, w_prime)
        return out.to(x.dtype)

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, h, w_prime = ctx.saved_tensors
        graph, reduce = ctx.graph, ctx.reduce
        need_x, need_h, need_w = ctx.needs_input_grad[:3]
        w = w_prime.detach().float().contiguous()
        g = grad_out.float().contiguous()
        E, K, Fi = graph.num_edges, h.size(1), x.size(1)
        gh = torch.empty(E, K, dtype=x.dtype, device=x.device) if need_h else None
        q = torch.empty(E, Fi, dtype=x.dtype, device=x.device) if need_x else None
        gw = None
        for r0, r1 in _nn_conv_blocks(graph.num_dst, w.size(0)):
            g_b = g[r0:r1]
            if need_w:
                p = ops.nn_conv_csr(graph.rowptr, graph.col, graph.perm, x, h, r0, r1, reduce, graph.plan)
                part = dense._mm_tn(p, g_b)
                gw = part if gw is None else gw + part
                del p
            if need_x or need_h:
                dp = dense._mm_nt(g_b, w).contiguous()
                ops.nn_conv_backward_dst(graph.rowptr, graph.col, graph.perm, x, h, dp, r0, r1, gh, q, reduce, graph.plan)
        if need_w and gw is None:
            gw = torch.zeros_like(w)
        gx = None
        if need_x:
            graph.build_transpose()
            # grad_x[j] = the sum of q over j's out-edges: perm_t is the caller's edge id of each transposed slot
            gx = ops.spmm_csr(graph.rowptr_t, graph.perm_t, None, q, graph.num_src, "sum", graph.plan_t)
        return gx, gh, (gw.to(w_prime.dtype) if need_w else None), None, None


def nn_conv_aggregate(graph: CSRGraph, x_src: Tensor, h: Tensor, w_prime: Tensor, reduce: str = "sum") -> Tensor:
    """out[i] = REDUCE_{e = (j -> i)} x[j] @ reshape(h_e W2^T + b2, [F_in, F_out]) for reduce in {sum, mean}: NNConv's
    message and aggregation (nn_conv.py:96-122) without its [E, F_in F_out] edge weights.  h: [E, K], the edge network's
    output before its last Linear, in the caller's edge order; w_prime: [(K+1) F_in, F_out] from that Linear
    (`nn.conv.nn_conv_weight`).  x_src: [num_src, F_in] of h's dtype; all three may require grad.  Destination rows are
    processed in blocks whose fp32 P stays under NN_CONV_BLOCK_BYTES; a block never splits a row."""
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"nn_conv_aggregate reduces by sum or mean, got '{reduce}'")
    if x_src.dim() != 2 or x_src.size(0) != graph.num_src:
        raise ValueError(f"x_src must be a [{graph.num_src}, F_in] tensor, got {tuple(x_src.shape)}")
    if h.dim() != 2 or h.size(0) != graph.num_edges or h.dtype != x_src.dtype:
        raise ValueError(f"h must be a [{graph.num_edges}, K] tensor of x's dtype, got {tuple(h.shape)} {h.dtype}")
    K, Fi = h.size(1), x_src.size(1)
    if w_prime.dim() != 2 or w_prime.size(0) != (K + 1) * Fi:
        raise ValueError(f"w_prime must be a [{(K + 1) * Fi}, F_out] tensor, got {tuple(w_prime.shape)}")
    if not ops.nn_conv_supported(K, Fi, x_src.dtype):
        raise ValueError(f"nn_conv_aggregate does not take K = {K}, F_in = {Fi} in {x_src.dtype}")
    return _NNConvAggregate.apply(x_src.contiguous(), h.contiguous(), w_prime, graph,
                                  "mean" if reduce == "mean" else "sum")


class _SplineBasis(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor, degree: int, wi_dtype: torch.dtype):
        basis, wi = ops.spline_basis(pseudo, kernel_size, is_open_spline, degree, wi_dtype)
        ctx.degree = degree
        ctx.save_for_backward(pseudo, kernel_size, is_open_spline)
        ctx.mark_non_differentiable(wi)
        return basis, wi

    @staticmethod
    def backward(ctx, grad_basis: Tensor, _grad_wi):
        pseudo, kernel_size, is_open_spline = ctx.saved_tensors
        gp = None
        if ctx.needs_input_grad[0]:
            gp = ops.spline_basis_backward(grad_basis, pseudo, kernel_size, is_open_spline, ctx.degree)
        return gp, None, None, None, None


def spline_basis(pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor, degree: int = 1,
                 wi_dtype: torch.dtype = torch.int64):
    """(basis [E, S], weight_index [E, S]) of pyg_lib.ops.spline_basis on CUDA float32 / bfloat16 pseudo-coordinates
    [E, D], differentiable with respect to pseudo.  S = (degree + 1)^D, degree 1..3; csrc/spline.cu states the convention.
    Pseudo-coordinates outside [0, 1] give indices reduced into [0, kernel_size) by a non-negative modulo."""
    return _SplineBasis.apply(pseudo, kernel_size, is_open_spline, int(degree), wi_dtype)


class _SplineWeighting(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, basis: Tensor, wi: Tensor):
        ctx.save_for_backward(x, weight, basis, wi)
        return ops.spline_weighting(x, weight, basis, wi)

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, weight, basis, wi = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        gx, gb, gw = ops.spline_weighting_backward(grad_out, x, weight, basis, wi, need_x, need_b, need_w)
        return gx, (gw.to(weight.dtype) if need_w else None), gb, None


def spline_weighting(x: Tensor, weight: Tensor, basis: Tensor, weight_index: Tensor) -> Tensor:
    """out[e] = sum_s basis[e, s] x[e] @ weight[weight_index[e, s]]: pyg_lib.ops.spline_weighting on CUDA float32 /
    bfloat16, differentiable with respect to x, weight and basis.  This is the unfused path (what SplineConv's
    `message` calls); `spline_conv_aggregate` fuses it with the aggregation."""
    return _SplineWeighting.apply(x, weight, basis, weight_index)


SPLINE_BLOCK_BYTES = 1 << 29      # fp32 bytes of P = [rows, K F_in] held at once by spline_conv_aggregate


class _SplineConvAggregate(torch.autograd.Function):
    """out = P W.view(K F_in, F_out) by destination-row blocks, P_i = REDUCE_e sum_s b_es x_j at kernel wi_es
    (csrc/spline.cu).  Saves x, weight, basis and wi only: the backward recomputes each block's P for dW = sum_b P_b^T G_b,
    forms dP_b = G_b W^T for the destination sweep (grad_basis and q per edge), and grad_x is one segment sum of q over
    the transposed CSR.  Each step runs only when one of its outputs is needed.  P and the GEMMs are fp32; the output
    has x's dtype."""

    @staticmethod
    def forward(ctx, x: Tensor, basis: Tensor, weight: Tensor, wi: Tensor, graph: CSRGraph, reduce: str):
        K, Fi, Fo = weight.shape
        w = weight.detach().float().reshape(K * Fi, Fo).contiguous()
        out = torch.zeros(graph.num_dst, Fo, dtype=torch.float32, device=x.device)
        for r0, r1 in _spline_blocks(graph.num_dst, K * Fi):
            p = ops.spline_csr(graph.rowptr, graph.col, graph.perm, x, basis, wi, K, r0, r1, reduce, graph.plan)
            out[r0:r1] = dense._mm(p, w)
        ctx.graph, ctx.reduce = graph, reduce
        ctx.save_for_backward(x, basis, weight, wi)
        return out.to(x.dtype)

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, basis, weight, wi = ctx.saved_tensors
        graph, reduce = ctx.graph, ctx.reduce
        need_x, need_b, need_w = ctx.needs_input_grad[:3]
        K, Fi, Fo = weight.shape
        w = weight.detach().float().reshape(K * Fi, Fo).contiguous()
        g = grad_out.float().contiguous()
        E, S = basis.shape
        gb = torch.empty(E, S, dtype=x.dtype, device=x.device) if need_b else None
        q = torch.empty(E, Fi, dtype=x.dtype, device=x.device) if need_x else None
        gw = None
        for r0, r1 in _spline_blocks(graph.num_dst, K * Fi):
            g_b = g[r0:r1]
            if need_w:
                p = ops.spline_csr(graph.rowptr, graph.col, graph.perm, x, basis, wi, K, r0, r1, reduce, graph.plan)
                part = dense._mm_tn(p, g_b)
                gw = part if gw is None else gw + part
                del p
            if need_x or need_b:
                dp = dense._mm_nt(g_b, w).contiguous()
                ops.spline_backward_dst(graph.rowptr, graph.col, graph.perm, x, basis, wi, K, dp, r0, r1, gb, q, reduce,
                                        graph.plan)
        if need_w and gw is None:
            gw = torch.zeros_like(w)
        gx = None
        if need_x:
            graph.build_transpose()
            # grad_x[j] = the sum of q over j's out-edges: perm_t is the caller's edge id of each transposed slot
            gx = ops.spmm_csr(graph.rowptr_t, graph.perm_t, None, q, graph.num_src, "sum", graph.plan_t)
        gw = gw.reshape(K, Fi, Fo).to(weight.dtype) if need_w else None
        return gx, gb, gw, None, None, None


def _spline_blocks(n_dst: int, width: int):
    """Destination row ranges [r0, r1) whose P fits SPLINE_BLOCK_BYTES (at least one row each)."""
    rows = max(1, SPLINE_BLOCK_BYTES // (4 * width))
    return [(r0, min(r0 + rows, n_dst)) for r0 in range(0, n_dst, rows)]


def spline_conv_aggregate(graph: CSRGraph, x_src: Tensor, basis: Tensor, wi: Tensor, weight: Tensor,
                          reduce: str = "sum") -> Tensor:
    """out[i] = REDUCE_{e = (j -> i)} sum_s basis[e, s] x[j] @ weight[wi[e, s]] for reduce in {sum, mean}: SplineConv's
    message and aggregation (spline_conv.py:150-153) as one CSR sweep into P [N, K F_in] and one GEMM with
    weight.view(K F_in, F_out), without the [E, F_out] messages.  basis [E, S] of x's dtype and wi [E, S] (int32, or
    int64 converted once) in the caller's edge order, as `spline_basis` returns them; weight [K, F_in, F_out].  x_src,
    basis and weight may require grad.  Destination rows are processed in blocks whose fp32 P stays under
    SPLINE_BLOCK_BYTES; a block never splits a row."""
    if reduce not in ("sum", "add", "mean"):
        raise ValueError(f"spline_conv_aggregate reduces by sum or mean, got '{reduce}'")
    if x_src.dim() != 2 or x_src.size(0) != graph.num_src:
        raise ValueError(f"x_src must be a [{graph.num_src}, F_in] tensor, got {tuple(x_src.shape)}")
    if basis.dim() != 2 or basis.size(0) != graph.num_edges or basis.dtype != x_src.dtype \
            or tuple(wi.shape) != tuple(basis.shape):
        raise ValueError(f"basis and wi must be [{graph.num_edges}, S] tensors, basis of x's dtype, got "
                         f"{tuple(basis.shape)} {basis.dtype} and {tuple(wi.shape)}")
    if weight.dim() != 3 or weight.size(1) != x_src.size(1) or weight.dtype != x_src.dtype:
        raise ValueError(f"weight must be a [K, {x_src.size(1)}, F_out] tensor of x's dtype, got {tuple(weight.shape)} "
                         f"{weight.dtype}")
    K, Fi = weight.size(0), weight.size(1)
    if not ops.spline_supported(K, Fi, basis.size(1), x_src.dtype):
        raise ValueError(f"spline_conv_aggregate does not take K = {K}, F_in = {Fi}, S = {basis.size(1)} in "
                         f"{x_src.dtype}")
    return _SplineConvAggregate.apply(x_src.contiguous(), basis.contiguous(), weight,
                                      wi.to(torch.int32).contiguous(), graph, "mean" if reduce == "mean" else "sum")


def _param_aggr_operands(graph, x: Optional[Tensor], a: Optional[Tensor], w, name: str, what: str):
    """The operands of softmax_aggregate and power_mean_aggregate: (x, a, w, where, want_saved).  `where` holds the
    sweep's (rowptr, col, perm, plan, n_edges, graph); w (t or p) becomes None for a Python 1 (the reference then
    skips the multiply, basic.py:207, or both clamps and pows, basic.py:285,290), ATen's fp32 scalar for another
    number, or a contiguous fp32 tensor of 1 or F elements; want_saved: a backward will need the saved plane."""
    if isinstance(graph, CSRGraph):
        where = (graph.rowptr, graph.col, graph.perm, graph.plan, graph.num_edges, graph)
        if x is not None and x.size(0) != graph.num_src:
            raise ValueError(f"x has {x.size(0)} rows but the graph has {graph.num_src} source nodes")
    else:
        if x is not None:
            raise ValueError("a (ptr, plan) message layout takes the messages as `a`, not x")
        ptr, plan = graph
        where = (ptr, None, None, plan, a.size(0), None)
    ref = x if x is not None else a
    if ref is None or ref.dim() != 2:
        raise ValueError(f"{what} takes two-dimensional x or a")
    if isinstance(w, Tensor):
        ww = w.reshape(-1).float().contiguous()
        if ww.numel() not in (1, ref.size(1)):
            raise ValueError(f"{name} must have 1 or {ref.size(1)} elements, got {w.numel()}")
    elif float(w) == 1.0:
        ww = None
    else:
        ww = torch.full((1, ), float(w), dtype=torch.float32, device=ref.device)
    x = None if x is None else x.contiguous()
    a = None if a is None else a.contiguous()
    want_saved = torch.is_grad_enabled() and any(v is not None and v.requires_grad for v in (x, a, ww))
    return x, a, ww, where, want_saved


def _sum_over_out_edges(graph: CSRGraph, grad_a: Tensor) -> Tensor:
    """grad_x[j] = the sum of grad_a over j's out-edges, by the segment sum over the transposed CSR (perm_t is the
    caller's edge id of each transposed slot)."""
    return ops.spmm_csr(graph.rowptr_t, graph.perm_t, None, grad_a, graph.num_src, "sum", graph.plan_t)


class _SoftmaxAggregate(torch.autograd.Function):
    """sum_e softmax_e(t * m_e) * m_e per destination and feature (csrc/softmax_aggr.cu).  The only saved state is
    the fp32 lse plane; the backward recomputes m, z and p.  The destination sweep gives grad_a and grad_t; grad_x is
    then the segment sum of grad_a's rows over the transposed CSR, and otherwise one transposed sweep.  Each sweep runs
    only when one of its outputs is needed."""

    @staticmethod
    def forward(ctx, x, a, t, where, eps: float, message: str, semi_grad: bool, want_lse: bool):
        rowptr, col, perm, plan, n_edges, _ = where
        out, lse = ops.softmax_aggr_csr(rowptr, col, perm, x, a, t, rowptr.numel() - 1, n_edges, message, eps, plan,
                                        want_lse)
        ctx.where, ctx.eps, ctx.message, ctx.semi = where, eps, message, semi_grad
        ctx.save_for_backward(x, a, t, out, lse)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, a, t, out, lse = ctx.saved_tensors
        rowptr, col, perm, plan, n_edges, graph = ctx.where
        need_x, need_a, need_t = ctx.needs_input_grad[:3]
        need_t = need_t and not ctx.semi
        gx = ga = gt = None
        if need_a or need_t:
            ga, gt = ops.softmax_aggr_backward_dst(rowptr, col, perm, x, a, t, out, lse, grad_out, n_edges, ctx.message,
                                                   ctx.eps, ctx.semi, need_a, need_t, plan)
            if gt is not None:
                gt = gt.sum().view(1) if t.numel() == 1 else gt
        if need_x:
            graph.build_transpose()
            if ga is not None:
                gx = _sum_over_out_edges(graph, ga)
            else:
                gx = ops.softmax_aggr_backward_src(graph.rowptr_t, graph.col_t, graph.perm_t, x, a, t, out, lse,
                                                   grad_out, ctx.message, ctx.eps, ctx.semi, graph.plan_t)
        return gx, ga, gt, None, None, None, None, None


def softmax_aggregate(graph, x: Optional[Tensor], a: Optional[Tensor] = None, t=1.0, eps: float = 0.0,
                      message: str = "identity", semi_grad: bool = False) -> Tensor:
    """SoftmaxAggregation (nn/aggr/basic.py:196-215, utils/_softmax.py:60-92), optionally behind GENConv's message
    relu(x_j + e_ji) + eps (gen_conv.py:231-239), in one online-softmax sweep with nothing stored per edge:

        m_e = x[j] | a[e] | relu(x[j] (+ a[e])) + eps,   out[i] = sum_{e = (j -> i)} softmax_e(t * m_e) * m_e

    graph: a CSRGraph (x: [num_src, F] gathered per edge; a: [E, F] in the caller's edge order), or (ptr, plan) for a
    destination-sorted [E, F] message matrix `a` (x None).  message: "identity" (exactly one of x, a) or "relu_eps"
    (x, a optional).  t: a Python number (1 skips the multiply, as the reference does) or a tensor of 1 or F elements
    whose values the kernel reads on the device in fp32, so a learnable t adds no host sync; t * m is formed in fp32
    and rounded to the messages' dtype, and t's gradient has t's shape and dtype.  semi_grad: the softmax
    weights carry no gradient (t gets none).  Empty rows give 0."""
    x, a, tt, where, want_lse = _param_aggr_operands(graph, x, a, t, "t", "softmax_aggregate")
    return _SoftmaxAggregate.apply(x, a, tt, where, float(eps), message, bool(semi_grad), want_lse)


class _PowerMeanAggregate(torch.autograd.Function):
    """clamp(mean_e clamp(m_e)^p)^(1/p) per destination and feature (csrc/power_mean.cu).  The only saved state is
    the fp32 plane of the means; the backward recomputes m, c and y.  The destination sweep gives grad_a and grad_p;
    grad_x is then the segment sum of grad_a's rows over the transposed CSR, and otherwise one transposed sweep (which
    then gives grad_p).  Each sweep runs only when one of its outputs is needed."""

    @staticmethod
    def forward(ctx, x, a, p, where, eps: float, message: str, lo: float, hi, want_mean: bool):
        rowptr, col, perm, plan, n_edges, _ = where
        out, mean = ops.power_mean_csr(rowptr, col, perm, x, a, p, rowptr.numel() - 1, n_edges, message, eps, lo, hi,
                                       plan, want_mean and p is not None)
        ctx.where, ctx.eps, ctx.message, ctx.lo, ctx.hi = where, eps, message, lo, hi
        ctx.save_for_backward(x, a, p, out, mean)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, a, p, out, mean = ctx.saved_tensors
        rowptr, col, perm, plan, n_edges, graph = ctx.where
        need_x, need_a, need_p = ctx.needs_input_grad[:3]
        gx = ga = gp = None
        if need_a or (need_p and not need_x):
            ga, gp = ops.power_mean_backward_dst(rowptr, col, perm, x, a, p, out, mean, grad_out, n_edges, ctx.message,
                                                 ctx.eps, ctx.lo, ctx.hi, need_a, need_p, plan)
        if need_x:
            graph.build_transpose()
            if ga is not None:
                gx = _sum_over_out_edges(graph, ga)
            else:
                gx, gp = ops.power_mean_backward_src(rowptr, graph.rowptr_t, graph.col_t, graph.perm_t, x, a, p, out,
                                                     mean, grad_out, ctx.message, ctx.eps, ctx.lo, ctx.hi, need_p,
                                                     graph.plan_t)
        if gp is not None:
            gp = gp.sum().view(1) if p.numel() == 1 else gp
        return gx, ga, gp, None, None, None, None, None, None


def power_mean_aggregate(graph, x: Optional[Tensor], a: Optional[Tensor] = None, p=1.0, eps: float = 0.0,
                         message: str = "identity", clamp_min: float = 1e-4,
                         clamp_max: Optional[float] = 100.0) -> Tensor:
    """PowerMeanAggregation (nn/aggr/basic.py:275-293), optionally behind GENConv's message relu(x_j + e_ji) + eps
    (gen_conv.py:231-239), in one sweep with nothing stored per edge:

        m_e = x[j] | a[e] | relu(x[j] (+ a[e])) + eps,
        out[i] = clamp(mean_{e = (j -> i)} clamp(m_e, clamp_min, clamp_max) ^ p, clamp_min, clamp_max) ^ (1 / p)

    graph, x, a and message as in softmax_aggregate.  p: a Python number (1 skips both clamps and both pows, as the
    reference does: a plain mean) or a tensor of 1 or F elements whose values the kernel reads on the device in fp32,
    so a learnable p adds no host sync; p's gradient has p's shape and dtype.  With p, clamp_min must be positive and
    clamp_max may be None (no upper bound).  An empty row gives clamp_min ^ (1 / p), or 0 without p."""
    x, a, pp, where, want_mean = _param_aggr_operands(graph, x, a, p, "p", "power_mean_aggregate")
    return _PowerMeanAggregate.apply(x, a, pp, where, float(eps), message, clamp_min, clamp_max, want_mean)


class _QuantileAggregate(torch.autograd.Function):
    """The q-quantiles of each destination's messages per channel (csrc/quantile.cu).  The only saved state is the
    pick bits, one per (message, rank, channel).  grad_a comes from the destination sweep, grad_x of gathered messages
    from one transposed sweep; each runs only when its output is needed."""

    @staticmethod
    def forward(ctx, x, a, q, where, interpolation: str, fill_value: float, want_bits: bool):
        rowptr, col, perm, plan, n_edges, _ = where
        out, bits = ops.quantile_csr(rowptr, col, perm, x, a, q, interpolation, fill_value, rowptr.numel() - 1,
                                     n_edges, plan, want_bits)
        ctx.where, ctx.interpolation = where, interpolation
        ctx.dtype, ctx.feat = (x if x is not None else a).dtype, (x if x is not None else a).size(1)
        ctx.save_for_backward(x, q, bits)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        x, q, bits = ctx.saved_tensors
        rowptr, col, perm, plan, n_edges, graph = ctx.where
        need_x, need_a = ctx.needs_input_grad[:2]
        gx = ga = None
        if need_a:
            ga = ops.quantile_backward_dst(rowptr, perm, q, ctx.interpolation, bits, grad_out, n_edges, ctx.feat,
                                           ctx.dtype, plan)
        if need_x:
            graph.build_transpose()
            gx = ops.quantile_backward_src(rowptr, graph.rowptr_t, graph.col_t, graph.perm_t, q, ctx.interpolation,
                                           bits, grad_out, x, graph.plan_t)
        return gx, ga, None, None, None, None, None


def quantile_aggregate(graph, x: Optional[Tensor], a: Optional[Tensor], q, interpolation: str = "linear",
                       fill_value: float = 0.0) -> Tensor:
    """QuantileAggregation / MedianAggregation (nn/aggr/quantile.py:71-130) as one selection sweep: no sort, and
    nothing float stored per message.

        out[i, k F + f] = the q[k]-quantile of {m_e[f] : e = (j -> i)},   m_e = x[j] | a[e]

    graph: a CSRGraph (x: [num_src, F] gathered per edge, or a: [E, F] in the caller's edge order), or (ptr, plan) for a
    destination-sorted [E, F] message matrix `a` (x None).  q: a float32 tensor of Q values in [0, 1] on the messages'
    device (the kernel reads it there, so a loaded state_dict takes effect with no host read), or a Python number or
    list.  interpolation: linear, lower, higher, nearest or midpoint.  Ranks, order, ties and roundings are
    csrc/quantile.cu's contract; bf16 'linear' returns float32.  Empty rows give fill_value.  Returns [N, Q * F]."""
    if (x is None) == (a is None):
        raise ValueError("quantile_aggregate takes exactly one of x and a")
    if isinstance(graph, CSRGraph):
        where = (graph.rowptr, graph.col if x is not None else None, graph.perm, graph.plan, graph.num_edges, graph)
        if x is not None and x.size(0) != graph.num_src:
            raise ValueError(f"x has {x.size(0)} rows but the graph has {graph.num_src} source nodes")
    else:
        if x is not None:
            raise ValueError("a (ptr, plan) message layout takes the messages as `a`, not x")
        ptr, plan = graph
        where = (ptr, None, None, plan, a.size(0), None)
    ref = x if x is not None else a
    if ref.dim() != 2:
        raise ValueError("quantile_aggregate takes two-dimensional x or a")
    if not isinstance(q, Tensor):
        q = torch.tensor(q if isinstance(q, (list, tuple)) else [q], dtype=torch.float32, device=ref.device)
    qq = q.reshape(-1).contiguous()
    x = None if x is None else x.contiguous()
    a = None if a is None else a.contiguous()
    want_bits = torch.is_grad_enabled() and ref.requires_grad
    return _QuantileAggregate.apply(x, a, qq, where, interpolation, float(fill_value), want_bits)


class _PNAAggregate(torch.autograd.Function):
    """PNAConv's aggregation of m_e = u_i + w_e, w_e = v_j (+ c_e) (csrc/pna.cu).  The sweep collects the statistics
    of w (b200mp_multi_aggr_csr on v, or b200mp_pna_edge_stats with c); the epilogue shifts them by u, applies the
    scalers and writes the post-network input.  Backward: the prologue gives grad_u in closed form and the per-edge
    terms, then one transposed-CSR sweep gives grad_v (and grad_c); each sweep runs only when its inputs need it."""

    @staticmethod
    def forward(ctx, x: Tensor, uv: Tensor, c: Optional[Tensor], avg_lin: Tensor, avg_log: Tensor, graph: CSRGraph,
                aggrs: tuple, scalers: tuple):
        N, T, F = x.shape
        W = T * F
        u, v = uv[:, :W], uv[:, W:]
        lin32 = avg_lin.detach().reshape(1).float().contiguous()
        log32 = avg_log.detach().reshape(1).float().contiguous()
        need_grad = any(ctx.needs_input_grad[:5])
        vv = None
        if c is None:
            vv = v.contiguous()
            res = ops.multi_aggr_csr(graph.rowptr, graph.col, vv, graph.num_dst, ops._pna_need(aggrs), graph.plan,
                                     with_ties=need_grad, count_self_zero=False)
        else:
            res = ops.pna_edge_stats(graph.rowptr, graph.col, graph.perm, v, c, graph.num_dst, aggrs, graph.plan,
                                     with_ties=need_grad)
        out = ops.pna_epilogue(graph.rowptr, x.reshape(N, W), u, res, aggrs, scalers, lin32, log32, T)
        ctx.graph, ctx.aggrs, ctx.scalers, ctx.shape = graph, aggrs, scalers, (N, T, F)
        ctx.keys, ctx.avg_dtypes = tuple(res), (avg_lin.dtype, avg_log.dtype)
        ctx.save_for_backward(uv, vv, c, lin32, log32, *res.values())
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        uv, vv, c, lin32, log32, *saved = ctx.saved_tensors
        stats = dict(zip(ctx.keys, saved))
        graph = ctx.graph
        N, T, F = ctx.shape
        W = T * F
        nx, nuv, nc, nlin, nlog = ctx.needs_input_grad[:5]
        grad_uv = torch.empty(N, 2 * W, dtype=uv.dtype, device=uv.device) if nuv else None
        r = ops.pna_prologue(graph.rowptr, grad_out.to(uv.dtype), uv[:, :W], stats, ctx.aggrs, ctx.scalers, lin32, log32,
                             T, want_u=nuv, want_x=nx, want_avg=nlin or nlog,
                             grad_u=None if grad_uv is None else grad_uv[:, :W])
        grad_c = None
        if nuv or nc:
            graph.build_transpose()
            if c is None:
                hit = stats.get("hit_mask")
                gv = ops.multi_aggr_backward(graph.rowptr_t, graph.col_t, vv, r["term_a"], r["term_b"], stats.get("min"),
                                             r["gmin"], stats.get("max"), r["gmax"], False, hit,
                                             None if hit is None else graph.t2csr)
                grad_uv[:, W:] = gv
            else:
                grad_c = ops.pna_edge_backward(graph.rowptr_t, graph.col_t, graph.perm_t, uv[:, W:], c, r, stats,
                                               graph.num_dst, None if grad_uv is None else grad_uv[:, W:], nc)
        gx = None if r["grad_x"] is None else r["grad_x"].view(N, T, F)
        avg = r["avg"]
        g_lin = avg[0:1].to(ctx.avg_dtypes[0]) if nlin else None
        g_log = avg[1:2].to(ctx.avg_dtypes[1]) if nlog else None
        return gx, grad_uv, grad_c, g_lin, g_log, None, None, None


def pna_aggregate(graph: CSRGraph, x: Tensor, uv: Tensor, c: Optional[Tensor], aggregators, scalers,
                  avg_deg_lin: Tensor, avg_deg_log: Tensor) -> Tensor:
    """PNAConv's propagate + cat([x, out]) (pna_conv.py:158-188, aggr/scaler.py:75-109) for one pre-layer per tower:
    the message of edge e = (j -> i) is u[i] + v[j] (+ c[e]) with uv = [u | v] one [N, 2W] tensor (W = towers * F)
    and c [E, W] in the caller's edge order (None without edge features).  x: [N, towers, F] (each tower's input).
    Returns [N, towers, (1 + A S) F] = cat([x_t, s_1(a_1 .. a_A), ..., s_S(a_1 .. a_A)]) per tower.  Gradients flow to
    x, uv, c and the two avg_deg tensors ([1] each, as DegreeScalerAggregation holds them)."""
    aggrs = tuple({"add": "sum"}.get(a, a) for a in aggregators)
    scalers = tuple(scalers)
    for a in aggrs:
        if a not in ops.PNA_AGGRS:
            raise ValueError(f"cannot fuse aggregator '{a}' (supported: {ops.PNA_AGGRS})")
    for s in scalers:
        if s not in ops.PNA_SCALERS:
            raise ValueError(f"Unknown scaler '{s}'")
    if len(set(aggrs)) != len(aggrs) or len(set(scalers)) != len(scalers):
        raise ValueError("each aggregator and each scaler may appear once")
    if x.dim() != 3:
        raise ValueError(f"x must be [N, towers, F], got {tuple(x.shape)}")
    N, T, F = x.shape
    if uv.shape != (N, 2 * T * F) or uv.dtype != x.dtype:
        raise ValueError(f"uv must be a [{N}, {2 * T * F}] tensor of x's dtype, got {tuple(uv.shape)} {uv.dtype}")
    if N != graph.num_dst or N != graph.num_src:
        raise ValueError(f"x has {N} rows but the graph has {graph.num_src} sources and {graph.num_dst} destinations")
    if c is not None and (c.shape != (graph.num_edges, T * F) or c.dtype != x.dtype):
        raise ValueError(f"c must be a [{graph.num_edges}, {T * F}] tensor of x's dtype, got {tuple(c.shape)} {c.dtype}")
    return _PNAAggregate.apply(x.contiguous(), uv.contiguous(), c, avg_deg_lin, avg_deg_log, graph, aggrs, scalers)


class _Segment(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src: Tensor, ptr: Tensor, reduce: str):
        ctx.plan = ops.segment_plan(ptr, src.size(0))      # hub segments are cut into chunks (csr_reduce.cuh)
        out = ops.segment_csr(src, ptr, reduce, ctx.plan)
        ctx.reduce, ctx.n_src = reduce, src.size(0)
        ctx.save_for_backward(ptr, src if reduce in ("min", "max") else None, out if reduce in ("min", "max") else None)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        ptr, src, out = ctx.saved_tensors
        reduce = ctx.reduce
        n_src = ctx.n_src                                   # == ptr[-1], known on the host: no D2H read
        index = ops.ptr2index(ptr, n_src)
        g2 = grad_out.contiguous().view(grad_out.size(0), -1)
        if reduce in ("sum", "add"):
            g = ops.gather_rows(g2, index)
        elif reduce == "mean":
            inv = 1.0 / (ptr[1:] - ptr[:-1]).clamp(min=1).to(torch.float32)
            g = ops.gather_rows(g2, index, ops.gather_rows(inv.view(-1, 1), index).view(-1))
        else:
            # _segment_reduce backward: even split among ties (no zero-initialised self here)
            s2, o2 = src.view(src.size(0), -1), out.view(out.size(0), -1)
            eq = (s2 == ops.gather_rows(o2, index)).to(s2.dtype)
            ties = ops.segment_csr(eq, ptr, "sum", ctx.plan)
            g = eq * ops.gather_rows(g2 / ties.clamp(min=1), index)
        return g.view((n_src, ) + tuple(grad_out.shape[1:])), None, None


def segment(src: Tensor, ptr: Tensor, reduce: str = "sum") -> Tensor:
    return _Segment.apply(src, ptr, reduce)


class _ScatterCOO(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src: Tensor, index: Tensor, dim_size: int, reduce: str):
        out = ops.scatter_coo(src, index, dim_size, reduce)
        ctx.reduce, ctx.dim_size = reduce, dim_size
        keep = reduce in ("min", "max", "mul")
        ctx.save_for_backward(index, src if keep else None, out if keep else None)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        index, src, out = ctx.saved_tensors
        reduce = ctx.reduce
        g2 = grad_out.contiguous().view(grad_out.size(0), -1)
        if reduce in ("sum", "add"):
            g = ops.gather_rows(g2, index)                       # scatter_add_ backward == gather
        elif reduce == "mean":
            cnt = ops.degree(index, ctx.dim_size).clamp(min=1).to(torch.float32)
            g = ops.gather_rows(g2, index, ops.gather_rows((1.0 / cnt).view(-1, 1), index).view(-1))
        elif reduce in ("min", "max"):
            s2, o2 = src.view(src.size(0), -1), out.view(out.size(0), -1)
            eq = (s2 == ops.gather_rows(o2, index)).to(torch.float32)
            # ATen scatter_reduce rule incl. the zero-initialised `self` tie (oracle_scatter_backward)
            ties = ops.scatter_coo(eq, index, ctx.dim_size, "sum") + (o2 == 0).to(torch.float32)
            g = eq * ops.gather_rows(g2 / ties, index)
        else:
            # ATen's scatter_reduce_('prod') rule (FunctionsManual.cpp, scatter_reduce_backward; `self` is all ones here):
            # a value that is the ONLY zero of its group gets grad * (product of the others), every other value gets
            # grad * result / value (0 when its group holds a zero elsewhere, 0 for every member of a group with >= 2 zeros)
            s2, o2 = src.view(src.size(0), -1).float(), out.view(out.size(0), -1).float()
            zero = s2 == 0
            n_zero = ops.gather_rows(ops.scatter_coo(zero.to(torch.float32), index, ctx.dim_size, "sum"), index)
            single = zero & (n_zero == 1)
            others = ops.scatter_coo(torch.where(single, torch.ones_like(s2), s2), index, ctx.dim_size, "mul")
            g = torch.where(single, ops.gather_rows(g2 * others, index), ops.gather_rows(g2 * o2, index) / torch.where(zero, torch.ones_like(s2), s2))
        return g.view((index.numel(), ) + tuple(grad_out.shape[1:])), None, None, None


def scatter_coo(src: Tensor, index: Tensor, dim_size: int, reduce: str = "sum") -> Tensor:
    return _ScatterCOO.apply(src, index, dim_size, reduce)


class _ScatterAny(torch.autograd.Function):
    """scatter(reduce='any') (utils/_scatter.py:75-77: `src.new_zeros(size).scatter_(dim, index, src)`): one member of
    every group.  Which one is unspecified on CUDA; here it is the LAST one in index order -- what the reference's CPU
    kernel produces -- found by an integer amax over the positions, then one row gather.  Backward = scatter_'s:
    every member receives its group's gradient."""

    @staticmethod
    def forward(ctx, src: Tensor, index: Tensor, dim_size: int):
        pos = torch.arange(index.numel(), device=index.device, dtype=torch.int64)
        last = torch.full((dim_size, ), -1, dtype=torch.int64, device=index.device).scatter_reduce_(
            0, index.long(), pos, "amax", include_self=True)
        s2 = src.contiguous().view(src.size(0), -1)
        if s2.size(0) == 0:
            out = s2.new_zeros((dim_size, s2.size(1)))
        else:
            out = ops.gather_rows(s2, ops.convert_index(last.clamp(min=0), index.dtype))
            out = out * (last >= 0).to(out.dtype).view(-1, 1)                    # empty groups stay 0
        ctx.save_for_backward(index)
        return out.view((dim_size, ) + tuple(src.shape[1:]))

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        index, = ctx.saved_tensors
        g = ops.gather_rows(grad_out.contiguous().view(grad_out.size(0), -1), index)
        return g.view((index.numel(), ) + tuple(grad_out.shape[1:])), None, None


def scatter_any(src: Tensor, index: Tensor, dim_size: int) -> Tensor:
    return _ScatterAny.apply(src, index, dim_size)


class _SoftmaxCSR(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src: Tensor, ptr: Tensor, index: Optional[Tensor]):
        ctx.plan = ops.segment_plan(ptr, src.size(0))        # hub groups: chunked path (ops.softmax_csr)
        if ctx.plan is not None and index is None:
            index = ops.ptr2index(ptr, src.size(0))
        out = ops.softmax_csr(src, ptr, ctx.plan, index)
        ctx.save_for_backward(out, ptr, index)
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        out, ptr, index = ctx.saved_tensors
        return ops.softmax_csr_backward(out, grad_out, ptr, ctx.plan, index), None, None


def softmax_csr(src: Tensor, ptr: Tensor, index: Optional[Tensor] = None) -> Tensor:
    return _SoftmaxCSR.apply(src, ptr, index)


class _GATFused(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xh: Tensor, a_src: Tensor, a_dst: Tensor, graph: CSRGraph, heads: int, chan: int, slope: float,
                want_alpha: bool):
        out, row_max, row_den, alpha = ops.gat_fused_csr(graph.rowptr, graph.col, xh, a_src, a_dst, heads, chan,
                                                         slope, want_alpha, plan=graph.plan,
                                                         dst_of_edge=graph.dst_csr if want_alpha else None)
        ctx.graph, ctx.dims = graph, (heads, chan, slope)
        ctx.save_for_backward(xh, a_src, a_dst, row_max, row_den, out)
        if alpha is None:
            alpha = xh.new_empty(0)
        ctx.mark_non_differentiable(alpha)
        return out, alpha

    @staticmethod
    def backward(ctx, grad_out: Tensor, _grad_alpha):
        xh, a_src, a_dst, row_max, row_den, out = ctx.saved_tensors
        graph = ctx.graph
        heads, chan, slope = ctx.dims
        graph.build_transpose()
        gxh, gas, gad = ops.gat_fused_csr_backward(graph.rowptr, graph.col, graph.dst_csr, graph.rowptr_t, graph.col_t,
                                                   graph.t2csr, xh, a_src.float().contiguous(),
                                                   a_dst.float().contiguous(), row_max, row_den, out, grad_out,
                                                   heads, chan, slope, plan=graph.plan)
        return gxh, gas.to(a_src.dtype), gad.to(a_dst.dtype), None, None, None, None, None


def gat_attention(graph: CSRGraph, xh: Tensor, a_src: Tensor, a_dst: Tensor, heads: int, chan: int,
                  negative_slope: float = 0.2, return_alpha: bool = False):
    """out[i,h,:] = sum_e softmax_i(leaky_relu(a_src[j,h] + a_dst[i,h]))_e * xh[j,h,:]
    (GATConv.edge_update + message + aggregate, gat_conv.py:387-409) in one fused sweep.
    xh: [num_src, H*C]; returns out [num_dst, H*C] (and alpha [E, H] in CSR order)."""
    if ops.attn_supported(heads, chan, xh.dtype) and xh.data_ptr() % 16 == 0:
        return attention("gat", graph, heads, chan, v=xh, s_src=a_src, s_dst=a_dst, negative_slope=negative_slope,
                         return_alpha=return_alpha)
    # head widths off the vector path: the scalar kernels of csrc/gat.cu (no padding copy needed for GAT)
    out, alpha = _GATFused.apply(xh, a_src, a_dst, graph, heads, chan, float(negative_slope), return_alpha)
    return (out, alpha) if return_alpha else out


class _AttnFused(torch.autograd.Function):
    """Fused attention family (csrc/attention.cu): GAT / GATv2 / dot-product scores, edge softmax and the weighted
    aggregation in one sweep; backward = destination sweep + source sweep with the attention recomputed."""

    @staticmethod
    def forward(ctx, mode: str, graph: CSRGraph, heads: int, chan: int, slope: float, scale: float, want_alpha: bool,
                v: Tensor, k: Optional[Tensor], q: Optional[Tensor], s_src: Optional[Tensor], s_dst: Optional[Tensor],
                att: Optional[Tensor], s_edge: Optional[Tensor], kv: Optional[Tensor], dropout: tuple = (0.0, 0),
                e_feat: Optional[Tensor] = None):
        hc = heads * chan
        if kv is not None:                                   # keys | values as the two halves of one [N, 2HC] product
            k, v = kv[:, :hc], kv[:, hc:]
        f32 = lambda t: None if t is None else t.detach().float().contiguous()   # noqa: E731
        s_src32, s_dst32, att32 = f32(s_src), f32(s_dst), (None if att is None else f32(att).view(-1))
        s_edge_csr = None if s_edge is None else graph.to_csr_order_rows(f32(s_edge))
        if q is not None and q.stride(1) != 1:
            q = q.contiguous()
        ref = kv if kv is not None else v
        e_csr = None if e_feat is None else graph.to_csr_order_rows(e_feat.detach().to(ref.dtype).contiguous())
        out, row_max, row_den, alpha = ops.attn_forward(mode, graph.rowptr, graph.col, v, heads, chan, k=k, q=q, s_src=s_src32,
                                                        s_dst=s_dst32, att=att32, s_edge=s_edge_csr, slope=slope, scale=scale,
                                                        want_alpha=want_alpha, plan=graph.plan, dropout_p=dropout[0],
                                                        dropout_seed=dropout[1], edge_feat=e_csr)
        ctx.mode, ctx.graph, ctx.dims, ctx.fused_kv = mode, graph, (heads, chan, slope, scale), kv is not None
        ctx.dropout = dropout
        ctx.dt = tuple(None if t is None else t.dtype for t in (s_src, s_dst, att, s_edge, e_feat))
        ctx.save_for_backward(kv if kv is not None else v, None if kv is not None else k, q, s_src32, s_dst32, att32, s_edge_csr,
                              row_max, row_den, out, e_csr)
        if alpha is None:
            alpha = out.new_empty(0)
        ctx.mark_non_differentiable(alpha)
        return out, alpha

    @staticmethod
    def backward(ctx, grad_out: Tensor, _grad_alpha):
        v, k, q, s_src, s_dst, att, s_edge, row_max, row_den, out, e_csr = ctx.saved_tensors
        graph = ctx.graph
        heads, chan, slope, scale = ctx.dims
        hc = heads * chan
        graph.build_transpose()
        grad_kv = grad_v = grad_k = None
        if ctx.fused_kv:
            kv = v
            k, v = kv[:, :hc], kv[:, hc:]
            grad_kv = torch.empty_like(kv)
            grad_k, grad_v = grad_kv[:, :hc], grad_kv[:, hc:]
        r = ops.attn_backward(ctx.mode, graph.rowptr, graph.col, graph.rowptr_t, graph.col_t, graph.t2csr, v, heads, chan,
                              row_max, row_den, out, grad_out, k=k, q=q, s_src=s_src, s_dst=s_dst, att=att, s_edge=s_edge,
                              slope=slope, scale=scale, plan=graph.plan, plan_t=graph.plan_t, grad_v=grad_v, grad_k=grad_k,
                              dropout_p=ctx.dropout[0], dropout_seed=ctx.dropout[1], edge_feat=e_csr)
        cast = lambda t, d: None if (t is None or d is None) else t.to(d)       # noqa: E731
        g_edge = None
        if s_edge is not None:
            g_edge = cast(graph.from_csr_order_rows(r["grad_s_edge"].contiguous()), ctx.dt[3])
        g_att = None if r["grad_att"] is None else cast(r["grad_att"], ctx.dt[2])
        g_ef = None
        if e_csr is not None and ctx.needs_input_grad[16]:
            g_ef = cast(graph.from_csr_order_rows(r["grad_edge_feat"]), ctx.dt[4])
        return (None, None, None, None, None, None, None,
                None if ctx.fused_kv else r["grad_v"], None if ctx.fused_kv else r["grad_k"], r["grad_q"],
                cast(r["grad_s_src"], ctx.dt[0]), cast(r["grad_s_dst"], ctx.dt[1]), g_att, g_edge, grad_kv, None, g_ef)


def _vector_shape(heads: int, chan: int, dtype: torch.dtype):
    """(chan_padded, heads_per_group) that put [*, heads*chan] rows on the vector path of csrc/attention.cu:
    a head is a power-of-two number of 16-byte vectors and a row group is at most 1 KB."""
    epv = 8 if dtype == torch.bfloat16 else 4
    vec = -(-chan // epv)
    lph = 1
    while lph < vec:
        lph *= 2
    if lph > 32:
        raise NotImplementedError(f"attention heads wider than 512 bytes (C = {chan}) are not on the fused path")
    chan_p = lph * epv
    per_group = max(1, 64 // lph)
    return chan_p, min(heads, per_group)


def attention(mode: str, graph: CSRGraph, heads: int, chan: int, *, v: Optional[Tensor] = None, k: Optional[Tensor] = None,
              q: Optional[Tensor] = None, kv: Optional[Tensor] = None, s_src: Optional[Tensor] = None,
              s_dst: Optional[Tensor] = None, att: Optional[Tensor] = None, s_edge: Optional[Tensor] = None,
              negative_slope: float = 0.2, scale: float = 1.0, return_alpha: bool = False, dropout_p: float = 0.0,
              dropout_seed: Optional[int] = None, e_feat: Optional[Tensor] = None):
    """out[i,h,:] = sum_e softmax_i(score_e,h) v[j,h,:] for mode in {"gat", "gatv2", "dot"} (see csrc/attention.cu).
    dropout_p > 0: attention dropout (F.dropout on the normalised coefficients, gat_conv.py:404) inside the sweep; the
    seed is drawn from torch's CPU generator (reproducible under torch.manual_seed, no device sync) unless given.
    e_feat [E, H*C] (caller's edge order; "gatv2" and "dot"): lin_edge(edge_attr) of `edge_dim` layers -- added inside
    GATv2's leaky_relu (gatv2_conv.py:358-360) / to the key and the value of the dot mode (transformer_conv.py:258-272).
    All feature operands are [n, H*C]; `kv` = [n_src, 2*H*C] (keys | values from one fused product) instead of k, v;
    s_edge [E, H] in the caller's edge order.  Returns out (and alpha [E, H] in CSR order).

    Head widths off the kernel's vector path (C not a power-of-two number of 16-byte vectors, rows above 1 KB) are
    mapped onto it: channels are zero-padded per head (zeros change neither a score nor a sum) and heads -- which are
    independent -- are processed in groups; the kernels are the same."""
    ref = kv if kv is not None else v
    dtype = ref.dtype
    if dtype not in (torch.float32, torch.bfloat16):
        raise TypeError(f"attention operands must be float32 or bfloat16, got {dtype}")
    chan_p, hpg = _vector_shape(heads, chan, dtype)
    if not 0.0 <= dropout_p < 1.0:
        raise ValueError(f"dropout probability has to be in [0, 1), got {dropout_p}")
    if dropout_p > 0.0 and dropout_seed is None:
        dropout_seed = int(torch.randint(0, 2 ** 62, (1, ), device="cpu"))
    drop = (float(dropout_p), int(dropout_seed or 0))
    if chan_p == chan and hpg == heads and ops.attn_supported(heads, chan, dtype):
        out, alpha = _AttnFused.apply(mode, graph, heads, chan, float(negative_slope), float(scale), return_alpha, v, k, q,
                                      s_src, s_dst, att if att is None else att.reshape(-1), s_edge, kv, drop, e_feat)
        return (out, alpha) if return_alpha else out
    if kv is not None:
        k, v = kv[:, :heads * chan], kv[:, heads * chan:]

    def group(t, h0, h1, feat: bool):
        if t is None:
            return None
        if not feat:                                        # [n, H] scalars per head
            return t[:, h0:h1]
        t3 = t.reshape(t.size(0), heads, chan)[:, h0:h1]
        if chan_p != chan:
            t3 = torch.nn.functional.pad(t3, (0, chan_p - chan))
        return t3.reshape(t.size(0), (h1 - h0) * chan_p).contiguous()

    outs, alphas = [], []
    for h0 in range(0, heads, hpg):
        h1 = min(h0 + hpg, heads)
        a_g = None if att is None else group(att.reshape(1, heads * chan), h0, h1, True).view(-1)
        o, al = _AttnFused.apply(mode, graph, h1 - h0, chan_p, float(negative_slope), float(scale), return_alpha,
                                 group(v, h0, h1, True), group(k, h0, h1, True), group(q, h0, h1, True),
                                 group(s_src, h0, h1, False), group(s_dst, h0, h1, False), a_g, group(s_edge, h0, h1, False),
                                 None, (drop[0], drop[1] + 0x51ED27 * h0),          # a different stream per head group
                                 group(e_feat, h0, h1, True))
        outs.append(o.view(o.size(0), h1 - h0, chan_p)[:, :, :chan])
        alphas.append(al)
    out = torch.cat(outs, dim=1).reshape(outs[0].size(0), heads * chan)
    if return_alpha:
        return out, torch.cat(alphas, dim=1)
    return out


class _MultiAggregate(torch.autograd.Function):
    """k aggregations of one neighbourhood in one sweep (FusedAggregation, nn/aggr/fused.py:191-336).
    `where` is a CSRGraph (gather mode: x is [num_src, F]) or a (ptr, index) pair (segment mode: x is the
    destination-sorted [E, F] message matrix)."""

    @staticmethod
    def forward(ctx, x: Tensor, where, names: tuple, semi_grad: bool, count_self_zero: bool):
        gather = isinstance(where, CSRGraph)
        if gather:
            rowptr, col, n_rows, plan = where.rowptr, where.col, where.num_dst, where.plan
        else:
            rowptr, col, n_rows, plan = where[0], None, where[0].numel() - 1, where[2]
        need_grad = x.requires_grad
        # the var / std gradients need the group mean even when it is not an output
        extra = ("mean", ) if need_grad and "mean" not in names and ("var" in names or "std" in names) else ()
        res = ops.multi_aggr_csr(rowptr, col, x, n_rows, tuple(names) + extra, plan, with_ties=need_grad,
                                 count_self_zero=count_self_zero)
        ctx.where, ctx.names, ctx.gather, ctx.semi_grad = where, tuple(names), gather, semi_grad
        ctx.save_for_backward(x, res.get("min"), res.get("max"), res.get("ties_min"), res.get("ties_max"),
                              res.get("mean"), res.get("std"), res.get("hit_mask"))
        return tuple(res[n] for n in names)

    @staticmethod
    def backward(ctx, *grads):
        x, omin, omax, tmin, tmax, mean, std, hit_mask = ctx.saved_tensors
        where = ctx.where
        g = {n: (None if gr is None else gr.to(x.dtype)) for n, gr in zip(ctx.names, grads)}
        if all(v is None for v in g.values()):
            return None, None, None, None, None
        rowptr = where.rowptr if ctx.gather else where[0]
        term_a, term_b, gmin, gmax = ops.multi_aggr_prepare_backward(rowptr, g, mean, std, tmin, tmax, ctx.semi_grad)
        omin = omin if gmin is not None else None
        omax = omax if gmax is not None else None
        if ctx.gather:
            where.build_transpose()
            gx = ops.multi_aggr_backward(where.rowptr_t, where.col_t, x, term_a, term_b, omin, gmin, omax, gmax, False,
                                         hit_mask, None if hit_mask is None else where.t2csr)
        else:
            gx = ops.multi_aggr_backward(None, where[1], x, term_a, term_b, omin, gmin, omax, gmax, True)
        return gx, None, None, None, None


def multi_aggregate(where, x: Tensor, aggrs, semi_grad: bool = False, count_self_zero: bool = True):
    """[aggr(x) for aggr in aggrs] with aggrs from {sum, mean, min, max, var, std}, one sweep over the edges.
    where: CSRGraph (x: [num_src, F]) or (ptr, index[, plan]) for a destination-sorted [E, F] message matrix."""
    names = tuple({"add": "sum"}.get(a, a) for a in aggrs)
    if len(set(names)) != len(names):
        raise ValueError("duplicate aggregation in the fused list")
    for n in names:
        if n not in ops.MULTI_AGGRS:
            raise ValueError(f"cannot fuse aggregation '{n}' (supported: {ops.MULTI_AGGRS})")
    if not isinstance(where, CSRGraph):
        where = tuple(where) + (None, ) * (3 - len(where))
    return list(_MultiAggregate.apply(x, where, names, semi_grad, count_self_zero))
