"""Node-range sharding with the halo exchange FUSED into the gather kernel over NVLink peer memory.

`dist.py` moves halo rows with NCCL (pack -> all_to_all -> second sweep): on an HBM-bound step the
pack / receive / accumulate passes cost as much HBM traffic as they save in waiting.  Here the
feature matrix of every rank lives in a *symmetric* allocation (torch symmetric memory: every rank's
buffer is mapped into every other rank's address space over NVLink/NVSwitch) and the gather kernel
itself resolves a GLOBAL column id to `peer_base[c / n_local] + (c % n_local) * row_bytes`
(`b200mp_spmm_csr(..., peer_ptrs, peer_rows)`): local rows come from HBM, remote rows straight over
NVLink, in the same warp, overlapped tile by tile by construction -- no send lists, no staging
buffers, no second pass, no atomics.

The backward uses the mirror-image structure (SURVEY.md section 8(e), option 1): every rank also
owns the OUT-edges of its sources (one edge redistribution at build time), so `A^T g` for the owned
rows is again a pure gather -- of the peers' `grad_out` rows.

Ordering between ranks is by stream-ordered barriers of the symmetric-memory handle: a rank may read
its peers' rows only after every rank has finished producing them, and may overwrite its own rows
only after every rank has finished reading them.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
from torch import Tensor

from . import dense, ops
from .graph import CSRGraph


def symmetric_empty(shape, dtype, device, group=None):
    """Allocates a tensor every rank can address (peer-mapped) and returns (tensor, handle)."""
    import torch.distributed._symmetric_memory as symm_mem
    group = group if group is not None else dist.group.WORLD
    t = symm_mem.empty(*shape, dtype=dtype, device=device)
    hdl = symm_mem.rendezvous(t, group)
    return t, hdl


class PeerShardedGraph:
    """One rank's slice of a weighted aggregation  out[r] = sum_e w_e x[src_e]  over destination ROWS owned by this rank
    (one row per node, or R virtual rows per node for a relational graph), with GLOBAL source ids:
      g_fwd: rows = owned destination rows, cols = global source ids            (forward gather of the x rows)
      g_bwd: rows = owned sources,          cols = global destination row ids   (backward gather of grad rows)
    plus the symmetric buffers the two gathers read: `x` [n_local, feat] and `gout` [n_rows_local, feat]."""

    def __init__(self, g_fwd: CSRGraph, g_bwd: CSRGraph, lo: int, n_local: int, n_total: int, n_rows_local: int, feat: int, group):
        self.g_fwd, self.g_bwd = g_fwd, g_bwd
        self.graph = g_fwd
        self.lo, self.n_local, self.n_total, self.n_rows_local, self.group = lo, n_local, n_total, n_rows_local, group
        self.world = dist.get_world_size(group)
        self.num_edges = g_fwd.num_edges
        dev = g_fwd.device
        self.xw, self.h_xw = symmetric_empty((n_local, feat), torch.float32, dev, group)
        self.gout, self.h_gout = symmetric_empty((n_rows_local, feat), torch.float32, dev, group)

    def barrier(self) -> None:
        """Stream-ordered barrier across the ranks (on the current stream)."""
        self.h_xw.barrier(channel=0)

    @classmethod
    def build_weighted(cls, src_global: Tensor, row_local: Tensor, w: Tensor, lo: int, n_local: int, n_total: int,
                       n_rows_local: int, feat: int, group=None):
        """src_global [E]: global source ids of this rank's in-edges; row_local [E]: destination row in
        [0, n_rows_local); w [E]: the edge weights (computed by the destination's owner: gcn_norm, 1 / in-degree, ...)."""
        group = group if group is not None else dist.group.WORLD
        world = dist.get_world_size(group)
        rank = dist.get_rank(group)
        dev = src_global.device
        g_fwd = CSRGraph(src_global, row_local, n_total, n_rows_local, w)
        # mirror structure: send every edge (source, GLOBAL destination row, weight) to the owner of its SOURCE
        owner = torch.div(src_global, n_local, rounding_mode="floor")
        order = torch.sort(owner, stable=True)[1]
        counts = torch.bincount(owner, minlength=world)
        send_counts = counts.tolist()
        rc = torch.empty_like(counts)
        if world > 1:
            dist.all_to_all_single(rc, counts, group=group)
        else:
            rc.copy_(counts)
        recv_counts = rc.tolist()
        n_recv = int(sum(recv_counts))

        def exchange(t: Tensor) -> Tensor:
            out = torch.empty(n_recv, dtype=t.dtype, device=dev)
            inp = t[order].contiguous()
            if world > 1:
                dist.all_to_all_single(out, inp, output_split_sizes=recv_counts, input_split_sizes=send_counts, group=group)
            else:
                out.copy_(inp)
            return out

        row_global = row_local.to(torch.int64) + rank * n_rows_local
        src_b, row_b, w_b = exchange(src_global), exchange(row_global), exchange(w)
        assert n_recv == 0 or (int(src_b.min()) >= lo and int(src_b.max()) < lo + n_local)
        g_bwd = CSRGraph(row_b, src_b - lo, world * n_rows_local, n_local, w_b)   # rows = owned sources, cols = global dst rows
        return cls(g_fwd, g_bwd, lo, n_local, n_total, n_rows_local, feat, group)


class PeerShardedGCNGraph(PeerShardedGraph):
    """The gcn_norm'ed graph (D^-1/2 (A + I) D^-1/2) sharded by node range."""

    @classmethod
    def build(cls, edge_index_global: Tensor, lo: int, n_local: int, n_total: int, feat: int, group=None,
              add_self_loops: bool = True):
        from .dist import shard_self_loops
        group = group if group is not None else dist.group.WORLD
        world = dist.get_world_size(group)
        dev = edge_index_global.device
        src, dst = edge_index_global[0], edge_index_global[1]          # dst in [lo, lo + n_local)
        if add_self_loops:
            src, dst = shard_self_loops(src, dst, lo, n_local)
        dst_l = dst - lo
        # gcn_norm: in-degrees are local; dinv of every node by one all_gather (4 B per node)
        deg = ops.degree(dst_l, n_local).to(torch.float32)
        dinv = deg.pow(-0.5)
        dinv.masked_fill_(dinv == float("inf"), 0.0)
        dinv_all = torch.empty(n_total, dtype=torch.float32, device=dev)
        if world > 1:
            dist.all_gather_into_tensor(dinv_all, dinv, group=group)
        else:
            dinv_all.copy_(dinv)
        w = ops.gather_rows(dinv_all.view(-1, 1), src).view(-1) * ops.gather_rows(dinv.view(-1, 1), dst_l).view(-1)
        return cls.build_weighted(src, dst_l, w, lo, n_local, n_total, n_local, feat, group)


class PeerShardedRelGraph(PeerShardedGraph):
    """The relational graph of RGCNConv (virtual destination row dst * R + type, per-relation mean = weight
    1 / in-degree of the virtual row), sharded by node range: every rank owns R rows per owned node."""

    @classmethod
    def build(cls, edge_index_global: Tensor, edge_type: Tensor, num_relations: int, lo: int, n_local: int, n_total: int,
              feat: int, group=None, aggr: str = "mean"):
        src, dst = edge_index_global[0], edge_index_global[1]
        row = (dst - lo).to(torch.int64) * num_relations + edge_type.to(torch.int64)
        n_rows = n_local * num_relations
        if aggr == "mean":
            cnt = ops.degree(row, n_rows).clamp(min=1).to(torch.float32)
            w = ops.gather_rows((1.0 / cnt).view(-1, 1), row).view(-1)
        elif aggr in ("sum", "add"):
            w = torch.ones(row.numel(), dtype=torch.float32, device=src.device)
        else:
            raise NotImplementedError("sharded RGCN: aggr must be mean or sum")
        shard = cls.build_weighted(src, row, w, lo, n_local, n_total, n_rows, feat, group)
        shard.num_relations = num_relations
        return shard


class _LinearInto(torch.autograd.Function):
    """x W^T written straight into the symmetric buffer the peers gather from."""

    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, out: Tensor):
        x = x.contiguous()
        if dense.get_backend() == "tf32x3" and dense.supported(x, weight):
            w_hi, w_lo = dense.prepare_weight(weight)
            ctx.save_for_backward(x, weight, w_hi, w_lo)
            ctx.fast = True
            dense.linear_forward(x, w_hi, w_lo, out=out)
        else:
            ctx.save_for_backward(x, weight)
            ctx.fast = False
            torch.mm(x, weight.t(), out=out)
        ctx.mark_dirty(out)
        return out

    @staticmethod
    def backward(ctx, g: Tensor):
        g = g.contiguous()
        if ctx.fast:
            x, weight, w_hi, w_lo = ctx.saved_tensors
            gx = dense.linear_grad_input_w(g, weight, w_hi, w_lo) if ctx.needs_input_grad[0] else None
            gw = dense.linear_grad_weight(g, x) if ctx.needs_input_grad[1] else None
        else:
            x, weight = ctx.saved_tensors
            gx = g @ weight if ctx.needs_input_grad[0] else None
            gw = g.t() @ x if ctx.needs_input_grad[1] else None
        return gx, gw, None


class _PeerAggregate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xw: Tensor, bias: Optional[Tensor], shard: PeerShardedGCNGraph):
        g = shard.g_fwd
        assert xw.data_ptr() == shard.xw.data_ptr(), "the transformed features must live in the symmetric buffer"
        ctx.shard, ctx.has_bias = shard, bias is not None
        shard.barrier()                          # every rank's x W^T is complete before anyone gathers it
        out = ops.spmm_csr(g.rowptr, g.col, g.val, xw, g.num_dst, "sum", g.plan, bias=bias,
                           peer_ptrs=shard.h_xw.buffer_ptrs_dev, peer_rows=shard.n_local)
        # every rank has finished reading my x W^T rows before anything may overwrite them: without this a
        # forward-only loop, or two stacked layers sharing one shard, would let the next _LinearInto write
        # shard.xw while slower peers are still gathering the previous contents over NVLink
        shard.barrier()
        return out

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        shard = ctx.shard
        g = shard.g_bwd
        gx = gb = None
        if grad_out.data_ptr() != shard.gout.data_ptr():
            shard.gout.copy_(grad_out.reshape(shard.gout.shape))   # upstream did not produce the gradient in the symmetric buffer
        grad_sym = shard.gout
        shard.barrier()                          # every rank's gradient rows are in place before anyone gathers them
        if ctx.needs_input_grad[0]:
            gx = ops.spmm_csr(g.rowptr, g.col, g.val, grad_sym, g.num_dst, "sum", g.plan,
                              peer_ptrs=shard.h_gout.buffer_ptrs_dev, peer_rows=shard.n_rows_local)
        if ctx.has_bias and ctx.needs_input_grad[1]:
            gb = grad_sym.sum(0, dtype=torch.float32)
        shard.barrier()                          # peers are done reading my gradient rows
        return gx, gb, None


def peer_aggregate(x_local: Tensor, shard: PeerShardedGraph, bias: Optional[Tensor] = None) -> Tensor:
    """out[r] = sum_e w_e x[src_e] (+ bias) for this rank's destination rows, sources anywhere: x_local is copied into
    the symmetric buffer unless it already lives there."""
    if x_local.data_ptr() != shard.xw.data_ptr():
        x_local = _CopyInto.apply(x_local, shard.xw.detach())
    return _PeerAggregate.apply(x_local, bias, shard)


class _CopyInto(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, out: Tensor):
        out.copy_(x)
        ctx.mark_dirty(out)
        return out

    @staticmethod
    def backward(ctx, g: Tensor):
        return g, None


def peer_sharded_rgcn_conv(weight: Tensor, root: Optional[Tensor], bias: Optional[Tensor], x_local: Tensor,
                           shard: "PeerShardedRelGraph") -> Tensor:
    """RGCNConv.forward on one shard (rgcn_conv.py:257-280): the per-relation aggregation gathers remote source rows
    over NVLink inside the kernel; the K = R*F (+ root) product is local."""
    R, Fi, Fo = weight.shape
    h = peer_aggregate(x_local, shard).view(shard.n_local, R * Fi)
    w = weight.reshape(R * Fi, Fo)
    if root is not None:
        return dense.matmul_pair(h, w, x_local, root, bias)
    out = dense.matmul(h, w)
    return out if bias is None else out + bias


def peer_sharded_gcn_conv(conv, x_local: Tensor, shard: PeerShardedGCNGraph) -> Tensor:
    """GCNConv.forward on one shard with the exchange fused into the gather kernel."""
    # a fresh alias every step: autograd rebases the history of the tensor OBJECT it is handed
    xw = _LinearInto.apply(x_local, conv.lin.weight, shard.xw.detach())
    return _PeerAggregate.apply(xw, conv.bias, shard)
