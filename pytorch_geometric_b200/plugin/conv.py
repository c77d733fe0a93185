"""Subclasses of the reference's OWN layer classes with the fused path inside (`class B200GCNConv(torch_geometric.nn.GCNConv)`).

Everything a user of the reference relies on is inherited unchanged -- constructor, parameters, `reset_parameters`,
`state_dict`, hooks, `explain`, `decomposed_layers`, jittable / TorchScript plumbing, CPU execution -- because the
object IS the reference layer.  Only `forward` is overridden: when the inputs are CUDA float32 / bfloat16 tensors and
the layer is in a mode the fused kernels implement, it runs the engine's functional core (`nn/conv.py`); otherwise it
calls `super().forward(...)`, i.e. the reference code (which, with `plugin.install()`, still lands in the engine
through the routed `scatter` / `softmax` / lazy gather).  `message_and_aggregate` is overridden too, with
`SUPPORTS_FUSED_EDGE_INDEX = True` (nn/conv/message_passing.py:108,475-497), so that `propagate` on a destination-sorted
`EdgeIndex` takes the fused branch with the EdgeIndex's cached CSR.

A fall-through happens for: CPU / other dtypes, `explain=True`, `decomposed_layers > 1`, any registered
propagate / message / aggregate hook (message_passing.py:776-922), `SparseTensor` / `torch.sparse` adjacencies,
and layer options the kernels do not cover.  Attention dropout (training mode) runs inside the fused sweep.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch_geometric.nn as tgnn
from torch import Tensor
from torch_geometric import EdgeIndex
from torch_geometric.typing import (Adj, NoneType, OptPairTensor, OptTensor, PairTensor, Size,  # noqa: F401
                                    SparseTensor)  # (names the inherited `# propagate_type:` annotations are evaluated with)

from .. import dense
from .. import functional as Fn
from .. import ops
from .. import utils as U
from ..graph import CSRGraph, cached_graph
from ..nn import conv as C
from . import graphs, routing
from ._util import plain

# reference class name -> subclass defined below.  The subclasses carry a `B200` prefix on purpose: the reference's
# Inspector caches class sources by `cls.__name__` (torch_geometric/inspector.py:323-334), so a subclass that reused
# its parent's name would hide the parent's `# propagate_type:` annotation and get a `propagate` without arguments.
LAYERS = {n: "B200" + n for n in ("GCNConv", "SAGEConv", "GraphConv", "GINConv", "GATConv", "GATv2Conv", "TransformerConv",
                                  "RGCNConv", "FastRGCNConv", "PNAConv", "CGConv", "GENConv", "NNConv",
                                  "SplineConv")}
LAYERS["ECConv"] = "B200NNConv"                 # the reference's alias of NNConv (nn/conv/__init__.py)


def _has_hooks(self) -> bool:
    for name in ("_propagate_forward_pre_hooks", "_propagate_forward_hooks", "_message_forward_pre_hooks",
                 "_message_forward_hooks", "_aggregate_forward_pre_hooks", "_aggregate_forward_hooks",
                 "_message_and_aggregate_forward_pre_hooks", "_message_and_aggregate_forward_hooks",
                 "_edge_update_forward_pre_hooks", "_edge_update_forward_hooks"):
        if len(getattr(self, name, ())) > 0:
            return True
    return False


def _fast(self, *tensors) -> bool:
    if self.explain or self.decomposed_layers > 1 or _has_hooks(self) or routing._compiling() or torch.jit.is_scripting():
        return False
    return all(t is None or routing.engine_ok(t) for t in tensors)


_plain = plain


def _graph(edge_index, num_src: int, num_dst: int, flow: str, **kw) -> Optional[CSRGraph]:
    """CSRGraph for a [2, E] tensor (cached by identity), an EdgeIndex (its own cached CSR when sorted the right way)
    or a CSRGraph; None for SparseTensor / torch.sparse inputs (those stay with the reference)."""
    if isinstance(edge_index, CSRGraph):
        return edge_index
    if not isinstance(edge_index, Tensor) or edge_index.layout != torch.strided or edge_index.dim() != 2:
        return None
    if isinstance(edge_index, EdgeIndex) and not kw:
        if flow == "source_to_target" and edge_index.is_sorted_by_col:
            return graphs.graph_from_edge_index(edge_index, transpose=True)
        if flow == "target_to_source" and edge_index.is_sorted_by_row:
            return graphs.graph_from_edge_index(edge_index, transpose=False)
    return cached_graph(_plain(edge_index), num_src, num_dst, flow=flow, **kw)


def _pair(x):
    return (x, x) if isinstance(x, Tensor) else (x[0], x[1])


def _ndst(x, size):
    if x[1] is not None:
        return x[1].size(0)
    return size[1] if size is not None and size[1] is not None else x[0].size(0)


class _FusedEdgeIndexMixin:
    """`propagate(EdgeIndex sorted by destination, x=...)` -> `message_and_aggregate` -> the CSR kernel with the
    EdgeIndex's own cached structure (graph_conv.py:104-110 is the only reference layer that does this correctly)."""
    SUPPORTS_FUSED_EDGE_INDEX = True


class B200GCNConv(tgnn.GCNConv):
    def forward(self, x, edge_index, edge_weight: Optional[Tensor] = None) -> Tensor:
        if (isinstance(x, Tensor) and x.dim() == 2 and _fast(self, x) and (edge_weight is None or not edge_weight.requires_grad)):
            g = self._b200_graph(edge_index, edge_weight, x.size(0))
            if g is not None:
                return C.gcn_conv(x, g, self.lin.weight, self.bias)
        return super().forward(x, edge_index, edge_weight)

    def _b200_graph(self, edge_index, edge_weight, num_nodes: int) -> Optional[CSRGraph]:
        if isinstance(edge_index, CSRGraph):
            return edge_index
        if not isinstance(edge_index, Tensor) or edge_index.layout != torch.strided:
            return None
        cache = self.__dict__.get("_b200_cached_graph")
        if self.cached and cache is not None:
            return cache
        ei = _plain(edge_index)
        if self.normalize:
            g = U.gcn_norm_graph(ei, edge_weight, num_nodes, self.improved, self.add_self_loops, self.flow)
        else:
            g = cached_graph(ei, num_nodes, num_nodes, flow=self.flow)
            if edge_weight is not None:
                g = g.with_values(g.to_csr_order(edge_weight.detach().float()))
        if self.cached:
            self.__dict__["_b200_cached_graph"] = g
        return g

    def reset_parameters(self):
        super().reset_parameters()
        self.__dict__.pop("_b200_cached_graph", None)


class B200SAGEConv(_FusedEdgeIndexMixin, tgnn.SAGEConv):
    def forward(self, x, edge_index, size=None) -> Tensor:
        xs = _pair(x)
        if (isinstance(self.aggr, str) and self.aggr in ("mean", "sum", "add", "max", "min") and xs[0].dim() == 2
                and _fast(self, xs[0], xs[1])):
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                if self.project and hasattr(self, "lin"):
                    xs = (dense.linear(xs[0], self.lin.weight, self.lin.bias, relu=True), xs[1])
                return C.sage_conv(xs[0], xs[1], g, self.aggr, self.lin_l.weight, self.lin_l.bias,
                                   self.lin_r.weight if self.root_weight else None, self.normalize)
        return super().forward(x, edge_index, size)

    def message_and_aggregate(self, adj_t, x) -> Tensor:
        if isinstance(adj_t, EdgeIndex):
            return adj_t.matmul(other=x[0], reduce=self.aggr, transpose=True)
        return super().message_and_aggregate(adj_t, x)


class B200GraphConv(tgnn.GraphConv):
    def forward(self, x, edge_index, edge_weight: Optional[Tensor] = None, size=None) -> Tensor:
        xs = _pair(x)
        if (isinstance(self.aggr, str) and self.aggr in ("mean", "sum", "add", "max", "min") and xs[0].dim() == 2
                and _fast(self, xs[0], xs[1])):
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                return C.graph_conv(xs[0], xs[1], g, self.aggr, self.lin_rel.weight, self.lin_rel.bias, self.lin_root.weight,
                                    edge_weight)
        return super().forward(x, edge_index, edge_weight, size)


class B200GINConv(_FusedEdgeIndexMixin, tgnn.GINConv):
    def forward(self, x, edge_index, size=None) -> Tensor:
        xs = _pair(x)
        if xs[0].dim() == 2 and _fast(self, xs[0], xs[1]):
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                return self.nn(C.gin_aggregate(xs[0], xs[1], g, self.eps))
        return super().forward(x, edge_index, size)

    def message_and_aggregate(self, adj_t, x) -> Tensor:
        if isinstance(adj_t, EdgeIndex):
            return adj_t.matmul(other=x[0], reduce=self.aggr, transpose=True)
        return super().message_and_aggregate(adj_t, x)


def _attn_fast(self, *tensors) -> bool:
    return _fast(self, *tensors)


def _drop(self) -> float:
    """Attention dropout runs inside the fused sweep (same distribution as F.dropout, its own random stream)."""
    return float(self.dropout) if self.training else 0.0


class B200GATConv(tgnn.GATConv):
    def forward(self, x, edge_index, edge_attr=None, size=None, return_attention_weights=None):
        xs = _pair(x)
        if (xs[0].dim() == 2 and _attn_fast(self, xs[0], xs[1], edge_attr) and return_attention_weights is None
                and isinstance(edge_index, Tensor) and edge_index.layout == torch.strided and size is None):
            H, Cc = self.heads, self.out_channels
            lin_s, lin_d = (self.lin, self.lin) if self.lin is not None else (self.lin_src, self.lin_dst)
            same = isinstance(x, Tensor)
            res = None
            if self.res is not None and xs[1] is not None:
                res = dense.linear(xs[1], self.res.weight)
            xh_src = dense.linear(xs[0], lin_s.weight)
            xh_dst = None if (same and self.lin is not None) else (None if xs[1] is None else dense.linear(xs[1], lin_d.weight))
            n_src, n_dst = xs[0].size(0), (xs[1].size(0) if xs[1] is not None else xs[0].size(0))
            ei = _plain(edge_index)
            g = cached_graph(ei, n_src, n_dst, flow=self.flow, loops="gat" if self.add_self_loops else None,
                             loop_nodes=min(n_src, n_dst))
            s_edge = None
            if edge_attr is not None and self.lin_edge is not None:
                ea = edge_attr if not self.add_self_loops else C.edge_attr_with_loops(ei, edge_attr, min(n_src, n_dst),
                                                                                      self.fill_value, self.flow)
                if ea.dim() == 1:
                    ea = ea.view(-1, 1)
                s_edge = C._head_dot(dense.linear(ea, self.lin_edge.weight), self.att_edge, H, Cc)
            att_dst = self.att_dst if (xs[1] is not None) else None
            return C.gat_conv(xh_src, xh_dst, g, self.att_src, att_dst, H, Cc, self.negative_slope, self.concat, res,
                              self.bias, s_edge, False, _drop(self))
        return super().forward(x, edge_index, edge_attr, size, return_attention_weights)


class B200GATv2Conv(tgnn.GATv2Conv):
    def forward(self, x, edge_index, edge_attr=None, return_attention_weights=None):
        xs = _pair(x)
        if (xs[0].dim() == 2 and xs[1] is not None and _attn_fast(self, xs[0], xs[1], edge_attr)
                and (edge_attr is None) == (self.lin_edge is None)
                and return_attention_weights is None and isinstance(edge_index, Tensor) and edge_index.layout == torch.strided):
            H, Cc = self.heads, self.out_channels
            res = dense.linear(xs[1], self.res.weight) if self.res is not None else None
            x_l = dense.linear(xs[0], self.lin_l.weight, self.lin_l.bias)
            if self.share_weights and isinstance(x, Tensor):
                x_r = x_l
            else:
                x_r = dense.linear(xs[1], self.lin_r.weight, self.lin_r.bias)
            ei = _plain(edge_index)
            g = cached_graph(ei, x_l.size(0), x_r.size(0), flow=self.flow,
                             loops="gat" if self.add_self_loops else None, loop_nodes=min(x_l.size(0), x_r.size(0)))
            e_feat = None
            if edge_attr is not None:                                           # gatv2_conv.py:318-325, 358-360
                ea = edge_attr if not self.add_self_loops else C.edge_attr_with_loops(
                    ei, edge_attr, min(x_l.size(0), x_r.size(0)), self.fill_value, self.flow)
                e_feat = dense.linear(ea.view(-1, 1) if ea.dim() == 1 else ea, self.lin_edge.weight)
            return C.gatv2_conv(x_l, x_r, g, self.att, H, Cc, self.negative_slope, self.concat, res, self.bias, False,
                                _drop(self), e_feat)
        return super().forward(x, edge_index, edge_attr, return_attention_weights)


class B200TransformerConv(tgnn.TransformerConv):
    def forward(self, x, edge_index, edge_attr=None, return_attention_weights=None):
        xs = _pair(x)
        if (xs[0].dim() == 2 and xs[1] is not None and _attn_fast(self, xs[0], xs[1], edge_attr)
                and (edge_attr is None) == (self.lin_edge is None) and return_attention_weights is None
                and isinstance(edge_index, Tensor) and edge_index.layout == torch.strided):
            H, Cc = self.heads, self.out_channels
            query = dense.linear(xs[1], self.lin_query.weight, self.lin_query.bias)
            w_kv = torch.cat([self.lin_key.weight, self.lin_value.weight], dim=0)
            b_kv = None if self.lin_key.bias is None else torch.cat([self.lin_key.bias, self.lin_value.bias], dim=0)
            kv = dense.linear(xs[0], w_kv, b_kv)
            g = _graph(edge_index, xs[0].size(0), xs[1].size(0), self.flow)
            x_skip = dense.linear(xs[1], self.lin_skip.weight, self.lin_skip.bias) if self.root_weight else None
            w_beta = self.lin_beta.weight if self.lin_beta is not None else None
            e_feat = None
            if edge_attr is not None:                                           # transformer_conv.py:258-261
                e_feat = dense.linear(edge_attr.view(-1, 1) if edge_attr.dim() == 1 else edge_attr, self.lin_edge.weight)
            return C.transformer_conv(query, kv, g, H, Cc, self.concat, x_skip, w_beta, False, _drop(self), e_feat)
        return super().forward(x, edge_index, edge_attr, return_attention_weights)


class _RGCNMixin:
    def forward(self, x, edge_index, edge_type=None) -> Tensor:
        if (isinstance(x, Tensor) and x.dim() == 2 and x.is_floating_point() and _fast(self, x) and edge_type is not None
                and isinstance(edge_index, Tensor) and edge_index.layout == torch.strided
                and isinstance(self.aggr, str) and self.aggr in ("mean", "sum", "add", "max", "min")):
            g = cached_graph(_plain(edge_index), x.size(0), x.size(0) * self.num_relations, flow=self.flow,
                             edge_type=edge_type, num_relations=self.num_relations)
            w = C.rgcn_weight(self.weight, getattr(self, "comp", None) if self.num_bases is not None else None,
                              self.num_relations, self.in_channels_l, self.out_channels, self.num_blocks)
            return C.rgcn_conv(x, g, w, self.root, self.bias, self.aggr)
        return super().forward(x, edge_index, edge_type)


class B200RGCNConv(_RGCNMixin, tgnn.RGCNConv):
    pass


class B200FastRGCNConv(_RGCNMixin, tgnn.FastRGCNConv):
    pass


def _pna_fusable(self, x, edge_index, edge_attr) -> bool:
    """The fused PNA path covers one Linear per pre-network, aggregators in {sum, mean, min, max, var, std} once each,
    the five scalers once each, a [2, E] / EdgeIndex adjacency and CUDA float32 / bfloat16 inputs."""
    if not (isinstance(x, Tensor) and x.dim() == 2 and _fast(self, x, edge_attr)):
        return False
    if not (isinstance(edge_index, Tensor) and edge_index.layout == torch.strided and edge_index.dim() == 2
            and edge_index.size(0) == 2 and not edge_index.is_floating_point()):
        return False
    if any(len(nn) != 1 or not isinstance(nn[0], tgnn.Linear) for nn in self.pre_nns):
        return False
    if (edge_attr is None) != (self.edge_dim is None) or (edge_attr is not None and edge_attr.dim() != 2):
        return False
    aggr = self.aggr_module
    if not isinstance(aggr, tgnn.aggr.DegreeScalerAggregation):
        return False
    inner = aggr.aggr.aggrs if isinstance(aggr.aggr, tgnn.aggr.MultiAggregation) else [aggr.aggr]
    names = [_PNA_AGGRS.get(type(a)) for a in inner]
    if None in names or len(set(names)) != len(names) or any(getattr(a, "semi_grad", False) for a in inner):
        return False
    if any(getattr(a, "var_aggr", None) is not None and a.var_aggr.semi_grad for a in inner):
        return False
    sc = list(aggr.scaler)
    return all(s in ("identity", "amplification", "attenuation", "linear", "inverse_linear") for s in sc) and len(set(sc)) == len(sc)


_PNA_AGGRS = {tgnn.aggr.SumAggregation: "sum", tgnn.aggr.MeanAggregation: "mean", tgnn.aggr.MinAggregation: "min",
              tgnn.aggr.MaxAggregation: "max", tgnn.aggr.VarAggregation: "var", tgnn.aggr.StdAggregation: "std"}


class B200PNAConv(tgnn.PNAConv):
    def forward(self, x, edge_index, edge_attr=None) -> Tensor:
        if _pna_fusable(self, x, edge_index, edge_attr):
            g = _graph(edge_index, x.size(0), x.size(0), self.flow)
            if g is not None:
                aggr = self.aggr_module
                inner = aggr.aggr.aggrs if isinstance(aggr.aggr, tgnn.aggr.MultiAggregation) else [aggr.aggr]
                enc = getattr(self, "edge_encoder", None)
                block = C.pna_block(x, g, edge_attr, [nn[0].weight for nn in self.pre_nns], [nn[0].bias for nn in self.pre_nns],
                                    None if enc is None else enc.weight, None if enc is None else enc.bias,
                                    [_PNA_AGGRS[type(a)] for a in inner], list(aggr.scaler), aggr.avg_deg_lin,
                                    aggr.avg_deg_log, self.towers, self.F_in, self.divide_input)
                # unbind: one [N, T, (1 + A S) F] gradient for all towers, where block[:, t] would allocate one per tower
                out = torch.cat([nn(b) for nn, b in zip(self.post_nns, block.unbind(1))], dim=1)   # pna_conv.py:170-173
                return self.lin(out)
        return super().forward(x, edge_index, edge_attr)


def _cg_fusable(self, xs, edge_attr) -> bool:
    """The fused CGConv path covers sum / mean aggregation, CUDA float32 / bfloat16 inputs with a destination tensor,
    and edge_attr given exactly when dim > 0 with dim columns (otherwise the reference raises its own error)."""
    if type(self.aggr_module) not in (tgnn.aggr.SumAggregation, tgnn.aggr.MeanAggregation):
        return False
    if xs[1] is None or xs[0].dim() != 2 or xs[1].dim() != 2:
        return False
    if (edge_attr is None) != (self.dim == 0):
        return False
    if edge_attr is not None and (edge_attr.dim() != 2 or edge_attr.size(1) != self.dim):
        return False
    return _fast(self, xs[0], xs[1], edge_attr) and len({t.dtype for t in (xs[0], xs[1], edge_attr) if t is not None}) == 1


class B200CGConv(tgnn.CGConv):
    def forward(self, x, edge_index, edge_attr=None) -> Tensor:
        xs = _pair(x)
        if _cg_fusable(self, xs, edge_attr):
            g = _graph(edge_index, xs[0].size(0), xs[1].size(0), self.flow)
            if g is not None:
                reduce = "mean" if type(self.aggr_module) is tgnn.aggr.MeanAggregation else "sum"
                u, v, c = C.cg_uvc(x if isinstance(x, Tensor) else xs, edge_attr, self.lin_f.weight, self.lin_f.bias,
                                   self.lin_s.weight, self.lin_s.bias)
                out = Fn.aggregate_cg_uv(g, u, c, reduce) if v is None else Fn.aggregate_cg(g, u, v, c, reduce)
                out = out if self.bn is None else self.bn(out)                       # cg_conv.py:86-88
                return out + xs[1]
        return super().forward(x, edge_index, edge_attr)


def _gen_fusable(self, xs, edge_index, edge_attr) -> bool:
    """The fused GENConv path covers the reference's SoftmaxAggregation (t, learn_t, softmax_sg, channels) and
    PowerMeanAggregation (p, learn_p, channels, clamp bounds the sweep takes) without lin_aggr_out, a [2, E] tensor or
    EdgeIndex adjacency, and CUDA float32 / bfloat16 inputs of one dtype whose t or p is a number or of that dtype (a
    learnable fp32 t or p with bf16 inputs promotes in the reference: it stays there)."""
    aggr = self.aggr_module
    if type(aggr) is tgnn.aggr.SoftmaxAggregation:
        w = aggr.t
    elif type(aggr) is tgnn.aggr.PowerMeanAggregation:
        w = aggr.p
    else:
        return False
    if hasattr(self, "lin_aggr_out") or xs[0] is None or xs[0].dim() != 2:
        return False
    if not (isinstance(edge_index, Tensor) and edge_index.layout == torch.strided and edge_index.dim() == 2
            and edge_index.size(0) == 2 and not edge_index.is_floating_point()):
        return False
    if edge_attr is not None and edge_attr.dim() != 2:
        return False
    ts = [t for t in (xs[0], xs[1], edge_attr) if t is not None]
    if not _fast(self, *ts) or len({t.dtype for t in ts}) != 1:
        return False
    if isinstance(w, Tensor) and (w.dtype != xs[0].dtype or w.numel() not in (1, self.out_channels)):
        return False
    if type(aggr) is tgnn.aggr.PowerMeanAggregation:
        from ..nn.aggr import power_mean_fusable
        return power_mean_fusable(xs[0], w, aggr.min_value, aggr.max_value)
    return True


class B200GENConv(tgnn.GENConv):
    def forward(self, x, edge_index, edge_attr=None, size=None) -> Tensor:
        xs = _pair(x)
        if _gen_fusable(self, xs, edge_index, edge_attr):
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                x_src = self.lin_src(xs[0]) if hasattr(self, "lin_src") else xs[0]            # gen_conv.py:209-210
                ea = edge_attr
                if ea is not None and hasattr(self, "lin_edge"):                              # gen_conv.py:232-233
                    ea = self.lin_edge(ea)
                aggr = self.aggr_module
                if type(aggr) is tgnn.aggr.SoftmaxAggregation:
                    out = Fn.softmax_aggregate(g, x_src, ea, aggr.t, self.eps, "relu_eps",
                                               aggr.semi_grad and not aggr.learn)
                else:
                    out = Fn.power_mean_aggregate(g, x_src, ea, aggr.p, self.eps, "relu_eps", aggr.min_value,
                                                  aggr.max_value)
                if hasattr(self, "msg_norm"):                                                 # gen_conv.py:218-221
                    out = self.msg_norm(xs[1] if xs[1] is not None else x_src, out)
                x_dst = xs[1]
                if x_dst is not None:
                    if hasattr(self, "lin_dst"):
                        x_dst = self.lin_dst(x_dst)
                    out = out + x_dst
                return self.mlp(out)
        return super().forward(x, edge_index, edge_attr, size)


def _nn_conv_split(self, xs, edge_index, edge_attr):
    """The split edge network (`C.nn_conv_split`) when the fused NNConv path covers the call, else None: sum / mean
    aggregation, a splittable edge network, a 2-D edge_attr, a [2, E] tensor or EdgeIndex adjacency, CUDA float32 /
    bfloat16 tensors and parameters of one dtype outside torch.autocast (which would run the edge network, and so h,
    in another dtype than x), and a shape the sweeps take."""
    if type(self.aggr_module) not in (tgnn.aggr.SumAggregation, tgnn.aggr.MeanAggregation):
        return None
    if xs[0] is not None and torch.is_autocast_enabled(xs[0].device.type):
        return None
    if xs[0] is None or xs[0].dim() != 2 or xs[0].size(1) != self.in_channels_l or edge_attr is None or edge_attr.dim() != 2:
        return None
    if not (isinstance(edge_index, Tensor) and edge_index.layout == torch.strided and edge_index.dim() == 2
            and edge_index.size(0) == 2 and not edge_index.is_floating_point()):
        return None
    split = C.nn_conv_split(self.nn, self.in_channels_l, self.out_channels)
    if split is None:
        return None
    ts = [t for t in (xs[0], xs[1], edge_attr) if t is not None]
    if not _fast(self, *ts) or len({t.dtype for t in ts} | {p.dtype for p in self.parameters()}) != 1:
        return None
    return split if ops.nn_conv_supported(split[1].weight.size(1), self.in_channels_l, xs[0].dtype) else None


class B200NNConv(tgnn.NNConv):
    def forward(self, x, edge_index, edge_attr=None, size=None) -> Tensor:
        xs = _pair(x)
        split = _nn_conv_split(self, xs, edge_index, edge_attr)
        if split is not None:
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                pre, last = split
                h = C.nn_conv_edge_hidden(pre, edge_attr)
                w_prime = C.nn_conv_weight(last.weight, last.bias, self.in_channels_l, self.out_channels)
                reduce = "mean" if type(self.aggr_module) is tgnn.aggr.MeanAggregation else "sum"
                out = Fn.nn_conv_aggregate(g, xs[0], h, w_prime, reduce)
                if xs[1] is not None and self.root_weight:                             # nn_conv.py:110-115
                    out = out + self.lin(xs[1])
                if self.bias is not None:
                    out = out + self.bias
                return out
        return super().forward(x, edge_index, edge_attr, size)


def _spline_fusable(self, xs, edge_index, edge_attr) -> bool:
    """Whether the fused SplineConv path covers the call: sum / mean aggregation, a 2-D edge_attr with `dim` columns, a
    [2, E] tensor or EdgeIndex adjacency, CUDA float32 / bfloat16 tensors and parameters of one dtype outside
    torch.autocast, no hooks, explain, decomposed layers or compiling, and a shape the sweeps take."""
    if type(self.aggr_module) not in (tgnn.aggr.SumAggregation, tgnn.aggr.MeanAggregation):
        return False
    if xs[0] is None or xs[0].dim() != 2 or torch.is_autocast_enabled(xs[0].device.type):
        return False
    if not isinstance(edge_attr, Tensor) or edge_attr.dim() != 2 or edge_attr.size(1) != self.dim:
        return False
    if not (isinstance(edge_index, Tensor) and edge_index.layout == torch.strided and edge_index.dim() == 2
            and edge_index.size(0) == 2 and not edge_index.is_floating_point()):
        return False
    if isinstance(self.weight, torch.nn.parameter.UninitializedParameter) or self.weight.size(1) != xs[0].size(1):
        return False
    ts = [t for t in (xs[0], xs[1], edge_attr) if t is not None]
    if not _fast(self, *ts) or len({t.dtype for t in ts} | {p.dtype for p in self.parameters()}) != 1:
        return False
    if self.degree not in (1, 2, 3):
        return False
    s = (self.degree + 1) ** self.dim
    return ops.spline_supported(self.weight.size(0), self.weight.size(1), s, xs[0].dtype)


class B200SplineConv(tgnn.SplineConv):
    def forward(self, x, edge_index, edge_attr=None, size=None) -> Tensor:
        xs = _pair(x)
        if _spline_fusable(self, xs, edge_index, edge_attr):
            g = _graph(edge_index, xs[0].size(0), _ndst(xs, size), self.flow)
            if g is not None:
                reduce = "mean" if type(self.aggr_module) is tgnn.aggr.MeanAggregation else "sum"
                out = C.spline_conv_forward(xs[0], g, edge_attr, self.kernel_size, self.is_open_spline, self.degree,
                                            self.weight, reduce)
                if xs[1] is not None and self.root_weight:                             # spline_conv.py:140-145
                    out = out + self.lin(xs[1])
                if self.bias is not None:
                    out = out + self.bias
                return out
        return super().forward(x, edge_index, edge_attr, size)
