"""GNN layers on the fused aggregation path.

Two layers of code:
  * functional cores (`gcn_conv`, `sage_conv`, `graph_conv`, `gin_aggregate`, `gat_conv`, `gatv2_conv`,
    `transformer_conv`, `rgcn_conv`): the layer arithmetic on explicit parameters -- shared by the standalone modules
    below and by the subclasses of the reference's own layer classes in `pytorch_geometric_b200.plugin.conv`;
  * standalone `torch.nn.Module`s whose constructor arguments, parameter names and `state_dict` layout follow the
    reference layers so checkpoints are interchangeable:

      GCNConv         nn/conv/gcn_conv.py:116-274        lin.weight [out,in], bias [out]
      SAGEConv        nn/conv/sage_conv.py:19-156        lin_l.weight/bias, lin_r.weight
      GraphConv       nn/conv/graph_conv.py:13-115       lin_rel.weight/bias, lin_root.weight
      GINConv         nn/conv/gin_conv.py:18-105         nn.*, eps [1]
      GINEConv        nn/conv/gin_conv.py:104-207        nn.*, eps [1], lin.weight/bias (edge_dim)
      ResGatedGraphConv nn/conv/res_gated_graph_conv.py:13-148  lin_key/lin_query/lin_value.weight/bias, lin_skip.weight, bias
      CGConv          nn/conv/cg_conv.py:12-101          lin_f.weight/bias, lin_s.weight/bias, bn.* (batch_norm)
      NNConv          nn/conv/nn_conv.py:13-126          nn.*, lin.weight (root_weight), bias
      SplineConv      nn/conv/spline_conv.py:21-172      weight [K,in,out], bias, kernel_size/is_open_spline (buffers), lin.weight
      GENConv         nn/conv/gen_conv.py:45-243         aggr_module.t/p, lin_src/lin_edge/lin_dst.weight, mlp.*, msg_norm.scale
      PNAConv         nn/conv/pna_conv.py:20-209         aggr_module.avg_deg_lin/log, edge_encoder.*, pre_nns.t.0.*, post_nns.*, lin.*
      RGCNConv        nn/conv/rgcn_conv.py:40-300        weight [R,in,out] (or bases/blocks + comp), root, bias
      FastRGCNConv    nn/conv/rgcn_conv.py:302-374       same parameters
      GATConv         nn/conv/gat_conv.py:27-413         lin (or lin_src/lin_dst), att_src/att_dst, lin_edge/att_edge, res, bias
      GATv2Conv       nn/conv/gatv2_conv.py:24-385       lin_l, lin_r, att [1,H,C], res, bias
      TransformerConv nn/conv/transformer_conv.py:17-285 lin_key/lin_query/lin_value/lin_skip(/lin_beta)

`forward(x, edge_index, ...)` accepts a `[2, E]` tensor or a prebuilt `CSRGraph` -- the counterpart of handing the
reference a `SparseTensor adj_t`.  Graph structures built from a `[2, E]` tensor are cached by the identity of that
tensor (`graph.cached_graph`), so a training loop that passes the same edge_index every step sorts once.
Dense transforms: hand-written wgmma 3xTF32 GEMMs where the shape allows (dense.py), a library GEMM otherwise.
"""
from __future__ import annotations

import math
from typing import Optional, Union

import torch
import torch.nn.functional as F
from torch import Tensor

from .. import dense
from .. import functional as Fn
from .. import ops
from .. import utils as U
from ..graph import CSRGraph, cached_graph

Adj = Union[Tensor, CSRGraph]


def glorot_(w: Tensor) -> Tensor:
    a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
    with torch.no_grad():
        return w.uniform_(-a, a)


class _Lin(torch.nn.Module):
    """torch_geometric.nn.dense.linear.Linear (nn/dense/linear.py:121-127): x W^T + b."""

    def __init__(self, in_channels: int, out_channels: int, bias: bool = True):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(out_channels, in_channels))
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None
        glorot_(self.weight)

    def forward(self, x: Tensor) -> Tensor:
        return dense.linear(x, self.weight, self.bias)


def _w(mod):
    return None if mod is None else mod.weight


class _BiasAggregate(torch.autograd.Function):
    """aggregate(graph, x, 'sum') + bias with the bias add fused into the kernel epilogue."""

    @staticmethod
    def forward(ctx, x: Tensor, bias: Tensor, graph: CSRGraph):
        ctx.graph = graph
        return ops.spmm_csr(graph.rowptr, graph.col, graph.val, x, graph.num_dst, "sum", graph.plan, bias=bias)

    @staticmethod
    def backward(ctx, grad_out: Tensor):
        graph = ctx.graph
        grad_out = grad_out.contiguous()
        gx = gb = None
        if ctx.needs_input_grad[0]:
            graph.build_transpose()
            if ctx.needs_input_grad[1] and graph.one_self_loop_per_row and graph.val_t is not None:
                # row i of A^T gathers grad_out[i] once, through its self-loop: the bias gradient rides the sweep
                gx, gb = ops.spmm_csr_self_colsum(graph.rowptr_t, graph.col_t, graph.val_t, grad_out, graph.plan_t)
            else:
                gx = ops.spmm_csr(graph.rowptr_t, graph.col_t, graph.val_t, grad_out, graph.num_src, "sum", graph.plan_t)
        if ctx.needs_input_grad[1] and gb is None:
            gb = ops.column_sum(grad_out)
        return gx, gb, None


# ================================================================================================ functional cores
def gcn_conv(x: Tensor, graph: CSRGraph, weight: Tensor, bias: Optional[Tensor]) -> Tensor:
    """GCNConv.forward after gcn_norm (gcn_conv.py:241-268): aggregate(x W^T) + b, bias fused into the sweep."""
    xw = dense.linear(x, weight)
    if bias is not None:
        return _BiasAggregate.apply(xw, bias, graph)
    return Fn.aggregate(graph, xw, "sum")


class _SageFused(torch.autograd.Function):
    """One SAGEConv layer on a non-bipartite graph as ONE autograd node (sage_conv.py:120-152):
        agg = aggr_j x_j;  y = act(agg W_l^T + x W_r^T + b)
    forward  = gather-reduce sweep + one pair GEMM (two A streams into one accumulator, bias / ReLU in the epilogue);
    backward = one pair GEMM for both input gradients (one read of g), the two split-K weight gradients, the bias column
               sum, and the transposed sweep ACCUMULATING into the root gradient (out += A^T g_agg in the kernel epilogue)
    -- no elementwise pass of size N x F exists in either direction except the ReLU mask."""

    @staticmethod
    def forward(ctx, x: Tensor, w_l: Tensor, b_l: Optional[Tensor], w_r: Tensor, graph: CSRGraph, aggr: str, relu: bool,
                input_is_relu: bool, grad_masked_by_consumer: bool):
        x = x.contiguous()
        agg = ops.spmm_csr(graph.rowptr, graph.col, graph.val, x, graph.num_dst, aggr, graph.plan)
        w_hi, w_lo = dense.split_tf32(torch.cat([w_l.detach(), w_r.detach()], dim=1))
        y, _ = dense.gemm_pair(agg, x, w_hi, w_lo, 0, w_l.size(0), bias=None if b_l is None else b_l.detach(), relu=relu)
        ctx.graph, ctx.aggr, ctx.relu, ctx.has_bias = graph, aggr, relu, b_l is not None
        ctx.input_is_relu, ctx.premasked = input_is_relu, grad_masked_by_consumer
        ctx.save_for_backward(x, agg, w_hi, w_lo, y if (relu and not grad_masked_by_consumer) else None)
        return y

    @staticmethod
    def backward(ctx, g: Tensor):
        x, agg, w_hi, w_lo, y = ctx.saved_tensors
        graph = ctx.graph
        g = g.contiguous()
        if ctx.relu and not ctx.premasked:
            g = g * (y > 0)
        k = x.size(1)
        gx = gwl = gwr = gb = None
        if ctx.needs_input_grad[0]:
            ga, gx = dense.gemm_pair(g, None, w_hi, w_lo, 1, k, k)                   # g . [W_l | W_r]
            graph.build_transpose()
            val_t = graph.mean_val_t() if ctx.aggr == "mean" else graph.val_t
            # gx += A^T ga in the sweep's epilogue; when this layer's input is a ReLU output (x = relu(pre)), the same
            # epilogue applies that ReLU's backward mask (x > 0), so the producing layer needs no elementwise pass
            ops.spmm_csr(graph.rowptr_t, graph.col_t, val_t, ga, graph.num_src, "sum", graph.plan_t, out=gx, accumulate=True,
                         relu_mask=x if ctx.input_is_relu else None)
        if ctx.needs_input_grad[1]:
            gwl = dense._mm_tn(g, agg)
        if ctx.needs_input_grad[3]:
            gwr = dense._mm_tn(g, x)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = ops.column_sum(g)
        return gx, gwl, gb, gwr, None, None, None, None, None


def _sage_fusable(x_src: Tensor, x_dst: Optional[Tensor], graph: CSRGraph, aggr: str, w_l: Tensor, w_r: Optional[Tensor]) -> bool:
    k, n = x_src.size(1), w_l.size(0)
    return (x_dst is x_src and w_r is not None and aggr in ("mean", "sum", "add") and graph.val is None
            and graph.num_src == graph.num_dst and x_src.is_cuda and x_src.dtype == torch.float32 and w_l.dtype == torch.float32
            and dense.get_backend() == "tf32x3" and k % 128 == 0 and n % 128 == 0 and w_l.size(1) == k and w_r.size(1) == k
            and x_src.size(0) > 0)


def sage_conv(x_src: Tensor, x_dst: Optional[Tensor], graph: CSRGraph, aggr: str, w_l: Tensor, b_l: Optional[Tensor],
              w_r: Optional[Tensor], normalize: bool = False, relu: bool = False, input_is_relu: bool = False,
              grad_masked_by_consumer: bool = False) -> Tensor:
    """SAGEConv.forward (sage_conv.py:120-152): act(lin_l(aggr_j x_j) + lin_r(x_i)).  Non-bipartite fp32 layers with
    widths on the GEMM kernel's grid run as ONE autograd node (`_SageFused`); otherwise the two products still
    accumulate into one output (dense.linear_pair).

    Stacking hints (both default False and are only honoured by the fused node; results are identical either way):
    `input_is_relu` -- x is the output of a ReLU: the gradient this layer returns is masked by (x > 0) in the sweep's
    epilogue; `grad_masked_by_consumer` -- this layer's `relu=True` output feeds ONLY a layer called with
    `input_is_relu=True`, so its own backward skips the (idempotent) mask pass."""
    if _sage_fusable(x_src, x_dst, graph, aggr, w_l, w_r):
        out = _SageFused.apply(x_src, w_l, b_l, w_r, graph, "sum" if aggr == "add" else aggr, relu, input_is_relu,
                               grad_masked_by_consumer and relu)
    else:
        agg = Fn.aggregate(graph, x_src, aggr)
        if w_r is not None and x_dst is not None:
            out = dense.linear_pair(agg, w_l, x_dst, w_r, b_l, relu=relu)
        else:
            out = dense.linear(agg, w_l, b_l, relu=relu)
    if normalize:
        out = F.normalize(out, p=2.0, dim=-1)
    return out


def graph_conv(x_src: Tensor, x_dst: Optional[Tensor], graph: CSRGraph, aggr: str, w_rel: Tensor, b_rel: Optional[Tensor],
               w_root: Tensor, edge_weight: Optional[Tensor] = None) -> Tensor:
    """GraphConv.forward (graph_conv.py:78-112): lin_rel(aggr_j e_ji x_j) + lin_root(x_i)."""
    agg = Fn.aggregate(graph, x_src, aggr, edge_weight)
    if x_dst is not None:
        return dense.linear_pair(agg, w_rel, x_dst, w_root, b_rel)
    return dense.linear(agg, w_rel, b_rel)


def gin_aggregate(x_src: Tensor, x_dst: Optional[Tensor], graph: CSRGraph, eps) -> Tensor:
    """GINConv before its MLP (gin_conv.py:86-92): sum_j x_j + (1 + eps) x_i."""
    out = Fn.aggregate(graph, x_src, "sum")
    if x_dst is not None:
        out = out + (1 + eps) * x_dst
    return out


class _HeadDot(torch.autograd.Function):
    """(s_a, s_b) = ((xh * att_a).sum(-1), (xh * att_b).sum(-1)) from ONE read of xh, and a one-pass backward
    (csrc/head_dot.cu) instead of the ten broadcast-multiply / reduce launches autograd makes of gat_conv.py:330-331."""

    @staticmethod
    def forward(ctx, xh, att_a, att_b, H, C):
        s_a, s_b = ops.head_dot(xh, att_a, att_b, H, C)
        ctx.save_for_backward(xh, att_a, att_b)
        ctx.hc = (H, C)
        return s_a, s_b                                                   # s_b is None without att_b

    @staticmethod
    def backward(ctx, g_a, g_b):
        xh, att_a, att_b = ctx.saved_tensors
        H, C = ctx.hc
        if g_a is None:
            g_a = torch.zeros(xh.size(0), H, dtype=torch.float32, device=xh.device)
        if att_b is not None and g_b is None:
            g_b = torch.zeros(xh.size(0), H, dtype=torch.float32, device=xh.device)
        gx, ga, gb = ops.head_dot_backward(xh, att_a, att_b, g_a, g_b if att_b is not None else None, None, H, C,
                                           ctx.needs_input_grad[0])
        ga = ga.view_as(att_a).to(att_a.dtype) if ctx.needs_input_grad[1] else None
        gb = gb.view_as(att_b).to(att_b.dtype) if att_b is not None and ctx.needs_input_grad[2] else None
        return gx, ga, gb, None, None


def _head_dot(xh: Tensor, att: Tensor, H: int, C: int, att2: Optional[Tensor] = None):
    """(xh.view(-1,H,C) * att).sum(-1) in fp32: the node-level attention terms (gat_conv.py:330-331).  With att2 the
    pair of terms for two attention vectors over the same features."""
    if ops.head_dot_supported(xh, H, C):
        s_a, s_b = _HeadDot.apply(xh, att, att2, H, C)
        return s_a if att2 is None else (s_a, s_b)
    x3 = xh.view(-1, H, C).float()
    s_a = (x3 * att.view(1, H, C).float()).sum(dim=-1)
    return s_a if att2 is None else (s_a, (x3 * att2.view(1, H, C).float()).sum(dim=-1))


def _finish_heads(out: Tensor, H: int, C: int, concat: bool, res: Optional[Tensor], bias: Optional[Tensor]) -> Tensor:
    if not concat:
        out = out.view(-1, H, C).mean(dim=1)
    if res is not None:
        out = out + res
    if bias is not None:
        out = out + bias.to(out.dtype)
    return out


def gat_conv(xh_src: Tensor, xh_dst: Optional[Tensor], graph: CSRGraph, att_src: Tensor, att_dst: Optional[Tensor], H: int,
             C: int, negative_slope: float = 0.2, concat: bool = True, res: Optional[Tensor] = None,
             bias: Optional[Tensor] = None, s_edge: Optional[Tensor] = None, return_alpha: bool = False,
             dropout_p: float = 0.0):
    """GATConv after its linear maps (gat_conv.py:330-385): xh_* = lin(x) [n, H*C]; xh_dst None = the sources are the
    destinations; att_dst None = no destination term (x = (x_src, None)).  s_edge [E, H] =
    (lin_edge(edge_attr) * att_edge).sum(-1) aligned with the edges the graph was built from (edge_dim)."""
    if att_dst is None:
        a_src = _head_dot(xh_src, att_src, H, C)
        a_dst = a_src.new_zeros(graph.num_dst, H)
    elif xh_dst is None:
        a_src, a_dst = _head_dot(xh_src, att_src, H, C, att_dst)         # both terms from one read of the features
    else:
        a_src = _head_dot(xh_src, att_src, H, C)
        a_dst = _head_dot(xh_dst, att_dst, H, C)
    r = Fn.attention("gat", graph, H, C, v=xh_src, s_src=a_src, s_dst=a_dst, s_edge=s_edge, negative_slope=negative_slope,
                     return_alpha=return_alpha, dropout_p=dropout_p)
    out, alpha = r if return_alpha else (r, None)
    out = _finish_heads(out, H, C, concat, res, bias)
    return (out, alpha) if return_alpha else out


def gatv2_conv(x_l: Tensor, x_r: Tensor, graph: CSRGraph, att: Tensor, H: int, C: int, negative_slope: float = 0.2,
               concat: bool = True, res: Optional[Tensor] = None, bias: Optional[Tensor] = None, return_alpha: bool = False,
               dropout_p: float = 0.0, e_feat: Optional[Tensor] = None):
    """GATv2Conv after lin_l / lin_r (gatv2_conv.py:300-331, 356-378): x_l [n_src, H*C], x_r [n_dst, H*C];
    e_feat [E, H*C] = lin_edge(edge_attr) aligned with the edges the graph was built from (edge_dim)."""
    r = Fn.attention("gatv2", graph, H, C, v=x_l, q=x_r, att=att.reshape(-1), negative_slope=negative_slope,
                     return_alpha=return_alpha, dropout_p=dropout_p, e_feat=e_feat)
    out, alpha = r if return_alpha else (r, None)
    out = _finish_heads(out, H, C, concat, res, bias)
    return (out, alpha) if return_alpha else out


def transformer_conv(query: Tensor, kv: Tensor, graph: CSRGraph, H: int, C: int, concat: bool = True,
                     x_skip: Optional[Tensor] = None, w_beta: Optional[Tensor] = None, return_alpha: bool = False,
                     dropout_p: float = 0.0, e_feat: Optional[Tensor] = None):
    """TransformerConv after its linear maps (transformer_conv.py:222-275): query [n_dst, H*C], kv [n_src, 2*H*C]
    (keys | values from ONE product with the concatenated lin_key / lin_value weights); x_skip = lin_skip(x_dst)."""
    r = Fn.attention("dot", graph, H, C, q=query, kv=kv, scale=1.0 / math.sqrt(C), return_alpha=return_alpha,
                     dropout_p=dropout_p, e_feat=e_feat)            # e_feat = lin_edge(edge_attr): added to key_j and value_j
    out, alpha = r if return_alpha else (r, None)
    if not concat:
        out = out.view(-1, H, C).mean(dim=1)
    if x_skip is not None:
        if w_beta is not None:
            beta = F.linear(torch.cat([out, x_skip, out - x_skip], dim=-1), w_beta).sigmoid()
            out = beta * x_skip + (1 - beta) * out
        else:
            out = out + x_skip
    return (out, alpha) if return_alpha else out


def rgcn_weight(weight: Tensor, comp: Optional[Tensor], num_relations: int, in_channels: int, out_channels: int,
                num_blocks: Optional[int]) -> Tensor:
    """The [R, F_in, F_out] relation weights from the basis / block-diagonal parametrisations (rgcn_conv.py:204-222)."""
    if comp is not None:                                               # basis decomposition
        return (comp @ weight.view(weight.size(0), -1)).view(num_relations, in_channels, out_channels)
    if num_blocks is not None:                                         # block-diagonal: weight [R, B, in/B, out/B]
        R, B, ci, co = weight.shape
        return torch.stack([torch.block_diag(*weight[r]) for r in range(R)])
    return weight


def rgcn_conv(x: Tensor, graph: CSRGraph, weight: Tensor, root: Optional[Tensor], bias: Optional[Tensor], aggr: str = "mean"):
    """RGCNConv with the per-relation semantics of the reference's loop path (rgcn_conv.py:257-280):
    out_i = sum_r aggr_{j in N_r(i)} x_j W_r + x_i root + bias.

    Engine mapping: edges are keyed by the virtual destination `dst * R + r`, so ONE gather-reduce sweep produces
    H [N, R*F_in] (per-relation mean/sum for every node) and the R small GEMMs of the reference collapse into ONE
    product with K = R * F_in against [W_1; ...; W_R] (+ the root product accumulated into the same output) -- a true
    GEMM, on the wgmma 3xTF32 kernel (no cuBLAS on this path when the widths are supported)."""
    N = x.size(0)
    R, Fi, Fo = weight.shape
    h = Fn.aggregate(graph, x, aggr).view(N, R * Fi)                   # [N*R, F_in] -> [N, R*F_in]
    w = weight.reshape(R * Fi, Fo)
    if root is not None:
        return dense.matmul_pair(h, w, x, root, bias)
    out = dense.matmul(h, w)
    return out if bias is None else out + bias.to(out.dtype)


# ================================================================================================ standalone modules
def _src_dst(edge_index: Tensor, flow: str):
    return (edge_index[0], edge_index[1]) if flow == "source_to_target" else (edge_index[1], edge_index[0])


def _plain_graph(edge_index: Adj, num_src: int, num_dst: int, flow: str = "source_to_target") -> CSRGraph:
    if isinstance(edge_index, CSRGraph):
        return edge_index
    return cached_graph(edge_index, num_src, num_dst, flow=flow)


class GCNConv(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int, improved: bool = False, cached: bool = False,
                 add_self_loops: Optional[bool] = None, normalize: bool = True, bias: bool = True, **kwargs):
        super().__init__()
        if add_self_loops is None:
            add_self_loops = normalize
        if add_self_loops and not normalize:
            raise ValueError(f"'{self.__class__.__name__}' does not support adding self-loops to the graph when no "
                             f"on-the-fly normalization is applied")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.improved, self.cached = improved, cached
        self.add_self_loops, self.normalize = add_self_loops, normalize
        self.flow = kwargs.get("flow", "source_to_target")
        self.lin = _Lin(in_channels, out_channels, bias=False)
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None
        self._cached_graph: Optional[CSRGraph] = None

    def reset_parameters(self):
        glorot_(self.lin.weight)
        if self.bias is not None:
            torch.nn.init.zeros_(self.bias)
        self._cached_graph = None

    def graph_for(self, edge_index: Adj, edge_weight: Optional[Tensor], num_nodes: int) -> CSRGraph:
        if isinstance(edge_index, CSRGraph):
            return edge_index
        if self._cached_graph is not None:
            return self._cached_graph
        if self.normalize:
            g = U.gcn_norm_graph(edge_index, edge_weight, num_nodes, self.improved, self.add_self_loops, self.flow)
        else:
            src, dst = _src_dst(edge_index, self.flow)
            g = CSRGraph(src, dst, num_nodes, num_nodes, edge_weight)
        if self.cached:
            self._cached_graph = g
        return g

    def forward(self, x: Tensor, edge_index: Adj, edge_weight: Optional[Tensor] = None) -> Tensor:
        if isinstance(x, (tuple, list)):
            raise ValueError(f"'{self.__class__.__name__}' received a tuple of node features as input while "
                             "this layer does not support bipartite message passing. Please try other layers "
                             "such as 'SAGEConv' or 'GraphConv' instead")
        return gcn_conv(x, self.graph_for(edge_index, edge_weight, x.size(0)), self.lin.weight, self.bias)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels})"


def _pair(x):
    return (x, x) if isinstance(x, Tensor) else (x[0], x[1])


def _num_dst(x, size):
    if x[1] is not None:
        return x[1].size(0)
    return size[1] if size is not None and size[1] is not None else x[0].size(0)


class SAGEConv(torch.nn.Module):
    def __init__(self, in_channels, out_channels: int, aggr: str = "mean", normalize: bool = False,
                 root_weight: bool = True, project: bool = False, bias: bool = True, **kwargs):
        super().__init__()
        if isinstance(in_channels, int):
            in_channels = (in_channels, in_channels)
        if aggr not in ("mean", "sum", "add", "max", "min"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.aggr, self.normalize, self.root_weight, self.project = aggr, normalize, root_weight, project
        self.flow = kwargs.get("flow", "source_to_target")
        if project:
            self.lin = _Lin(in_channels[0], in_channels[0], bias=True)
        self.lin_l = _Lin(in_channels[0], out_channels, bias=bias)
        if root_weight:
            self.lin_r = _Lin(in_channels[1], out_channels, bias=False)

    def forward(self, x, edge_index: Adj, size=None) -> Tensor:
        x = _pair(x)
        if self.project and hasattr(self, "lin"):
            x = (self.lin(x[0]).relu(), x[1])
        graph = _plain_graph(edge_index, x[0].size(0), _num_dst(x, size), self.flow)
        return sage_conv(x[0], x[1], graph, self.aggr, self.lin_l.weight, self.lin_l.bias,
                         self.lin_r.weight if self.root_weight else None, self.normalize)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, aggr={self.aggr})"


class GraphConv(torch.nn.Module):
    def __init__(self, in_channels, out_channels: int, aggr: str = "add", bias: bool = True, **kwargs):
        super().__init__()
        if isinstance(in_channels, int):
            in_channels = (in_channels, in_channels)
        if aggr not in ("mean", "sum", "add", "max", "min"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path")
        self.in_channels, self.out_channels, self.aggr = in_channels, out_channels, aggr
        self.flow = kwargs.get("flow", "source_to_target")
        self.lin_rel = _Lin(in_channels[0], out_channels, bias=bias)
        self.lin_root = _Lin(in_channels[1], out_channels, bias=False)

    def forward(self, x, edge_index: Adj, edge_weight: Optional[Tensor] = None, size=None) -> Tensor:
        x = _pair(x)
        graph = _plain_graph(edge_index, x[0].size(0), _num_dst(x, size), self.flow)
        return graph_conv(x[0], x[1], graph, self.aggr, self.lin_rel.weight, self.lin_rel.bias, self.lin_root.weight,
                          edge_weight)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels[0]}, {self.out_channels})"


class GINConv(torch.nn.Module):
    def __init__(self, nn: torch.nn.Module, eps: float = 0.0, train_eps: bool = False, **kwargs):
        super().__init__()
        self.nn = nn
        self.initial_eps = eps
        self.flow = kwargs.get("flow", "source_to_target")
        if train_eps:
            self.eps = torch.nn.Parameter(torch.full((1, ), float(eps)))     # shape [1] as gin_conv.py:63-65
        else:
            self.register_buffer("eps", torch.full((1, ), float(eps)))

    def forward(self, x, edge_index: Adj, size=None) -> Tensor:
        x = _pair(x)
        graph = _plain_graph(edge_index, x[0].size(0), _num_dst(x, size), self.flow)
        return self.nn(gin_aggregate(x[0], x[1], graph, self.eps))

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(nn={self.nn})"


class GINEConv(torch.nn.Module):
    """nn((1 + eps) x_i + AGGR_j relu(x_j + e_ji)) (gin_conv.py:104-207) with AGGR = sum (default) or mean; e_ji =
    lin(edge_attr) when `edge_dim` is set.  The message and the aggregation run as one edge-feature sweep
    (`Fn.aggregate_edge_relu`)."""

    def __init__(self, nn: torch.nn.Module, eps: float = 0.0, train_eps: bool = False, edge_dim: Optional[int] = None,
                 **kwargs):
        super().__init__()
        aggr = kwargs.get("aggr", "add")
        if aggr not in ("add", "sum", "mean"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path (sum or mean)")
        self.aggr = "mean" if aggr == "mean" else "sum"
        self.flow = kwargs.get("flow", "source_to_target")
        self.nn = nn
        self.initial_eps = eps
        if train_eps:
            self.eps = torch.nn.Parameter(torch.full((1, ), float(eps)))     # shape [1] as gin_conv.py:146-149
        else:
            self.register_buffer("eps", torch.full((1, ), float(eps)))
        if edge_dim is not None:                                             # gin_conv.py:150-160
            first = self.nn[0] if isinstance(self.nn, torch.nn.Sequential) else self.nn
            if hasattr(first, "in_features"):
                in_channels = first.in_features
            elif hasattr(first, "in_channels"):
                in_channels = first.in_channels
            else:
                raise ValueError("Could not infer input channels from `nn`.")
            self.lin = _Lin(edge_dim, in_channels)
        else:
            self.lin = None

    def forward(self, x, edge_index: Adj, edge_attr: Optional[Tensor] = None, size=None) -> Tensor:
        x = _pair(x)
        if self.lin is None and x[0].size(-1) != edge_attr.size(-1):        # gin_conv.py:197-200
            raise ValueError("Node and edge feature dimensionalities do not match. Consider setting the 'edge_dim' "
                             "attribute of 'GINEConv'")
        graph = _plain_graph(edge_index, x[0].size(0), _num_dst(x, size), self.flow)
        e = edge_attr if self.lin is None else self.lin(edge_attr)
        out = Fn.aggregate_edge_relu(graph, x[0], e, self.aggr)
        if x[1] is not None:
            out = out + (1 + self.eps) * x[1]
        return self.nn(out)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(nn={self.nn})"


class ResGatedGraphConv(torch.nn.Module):
    """W_1 x_i + AGGR_j sigmoid(W_3 x_i + W_4 x_j) * W_2 x_j (+ bias) (res_gated_graph_conv.py:13-148) with AGGR = sum
    (default) or mean.  q | v come from one product with the concatenated query / value weights, and the gated
    message runs with its aggregation as one sweep (`Fn.aggregate_gated_qv`).  `edge_dim` and gates other than the
    sigmoid are not on the fused path and raise ValueError."""

    def __init__(self, in_channels, out_channels: int, act=torch.nn.Sigmoid(), edge_dim: Optional[int] = None,
                 root_weight: bool = True, bias: bool = True, **kwargs):
        super().__init__()
        aggr = kwargs.get("aggr", "add")
        if aggr not in ("add", "sum", "mean"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path (sum or mean)")
        if edge_dim is not None:
            raise ValueError("edge_dim is not on the fused path (the gate would need per-edge Linear inputs)")
        if not (isinstance(act, torch.nn.Sigmoid) or act in (torch.sigmoid, F.sigmoid)):
            raise ValueError(f"act={act!r} is not on the fused path (only the sigmoid gate is)")
        self.aggr = "mean" if aggr == "mean" else "sum"
        self.flow = kwargs.get("flow", "source_to_target")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.act, self.edge_dim, self.root_weight = act, edge_dim, root_weight
        ic = (in_channels, in_channels) if isinstance(in_channels, int) else tuple(in_channels)
        self.lin_key = _Lin(ic[1], out_channels)                            # res_gated_graph_conv.py:80-93
        self.lin_query = _Lin(ic[0], out_channels)
        self.lin_value = _Lin(ic[0], out_channels)
        self.lin_skip = _Lin(ic[1], out_channels, bias=False) if root_weight else None
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None

    def forward(self, x, edge_index: Adj, edge_attr: Optional[Tensor] = None) -> Tensor:
        assert edge_attr is None                                             # res_gated_graph_conv.py:141
        x = _pair(x)
        k = self.lin_key(x[1])
        w_qv = torch.cat([self.lin_query.weight, self.lin_value.weight], dim=0)
        b_qv = torch.cat([self.lin_query.bias, self.lin_value.bias], dim=0)
        qv = dense.linear(x[0], w_qv, b_qv)
        graph = _plain_graph(edge_index, x[0].size(0), x[1].size(0), self.flow)
        out = Fn.aggregate_gated_qv(graph, k, qv, self.aggr)
        if self.lin_skip is not None:
            out = out + self.lin_skip(x[1])
        if self.bias is not None:
            out = out + self.bias
        return out

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels})"


def cg_uvc(x, edge_attr: Optional[Tensor], w_f: Tensor, b_f: Optional[Tensor], w_s: Tensor, b_s: Optional[Tensor]):
    """(u, v, c) of CGConv's message (cg_conv.py:93-98) with lin_f and lin_s split by the column blocks of
    z = [x_i, x_j, edge_attr]: u = x_dst [W_f,a; W_s,a]^T + [b_f; b_s], v = x_src [W_f,b; W_s,b]^T and
    c = edge_attr [W_f,c; W_s,c]^T ([E, 2F], None without edge_attr).  For one node tensor x, u | v come from one
    [N, 4F] product and are returned as (uv, None, c); for a pair (x_src, x_dst), one product per side.  Slicing and
    concatenating the module's own parameters keeps every parameter gradient with autograd."""
    x_src, x_dst = (x, x) if isinstance(x, Tensor) else (x[0], x[1])
    fd, fs = x_dst.size(-1), x_src.size(-1)
    w = torch.cat([w_f, w_s], dim=0)                                              # [2F, F_dst + F_src + dim]
    b = None if b_f is None else torch.cat([b_f, b_s])
    w_a, w_b = w[:, :fd], w[:, fd:fd + fs]
    c = None if edge_attr is None else dense.linear(edge_attr, w[:, fd + fs:].contiguous())
    if isinstance(x, Tensor):
        b_uv = None if b is None else torch.cat([b, torch.zeros_like(b)])
        return dense.linear(x, torch.cat([w_a, w_b], dim=0), b_uv), None, c
    return dense.linear(x_dst, w_a.contiguous(), b), dense.linear(x_src, w_b.contiguous()), c


class CGConv(torch.nn.Module):
    """x_i + AGGR_j sigmoid(z_ij W_f + b_f) * softplus(z_ij W_s + b_s), z_ij = [x_i, x_j, e_ji] (cg_conv.py:12-101),
    with AGGR = sum (default) or mean and an optional BatchNorm1d before the residual.  The two Linears are split into
    per-node products and the per-edge c (`cg_uvc`), and the message runs with its aggregation as one sweep
    (`Fn.aggregate_cg`).  Other aggregations raise ValueError."""

    def __init__(self, channels, dim: int = 0, aggr: str = "add", batch_norm: bool = False, bias: bool = True,
                 **kwargs):
        super().__init__()
        if aggr not in ("add", "sum", "mean"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path (sum or mean)")
        self.aggr = "mean" if aggr == "mean" else "sum"
        self.flow = kwargs.get("flow", "source_to_target")
        self.channels, self.dim, self.batch_norm = channels, dim, batch_norm
        ch = (channels, channels) if isinstance(channels, int) else tuple(channels)
        self.lin_f = _Lin(sum(ch) + dim, ch[1], bias=bias)                        # cg_conv.py:62-67
        self.lin_s = _Lin(sum(ch) + dim, ch[1], bias=bias)
        self.bn = torch.nn.BatchNorm1d(ch[1]) if batch_norm else None

    def forward(self, x, edge_index: Adj, edge_attr: Optional[Tensor] = None) -> Tensor:
        if (edge_attr is not None) != (self.dim > 0):
            raise ValueError(f"edge_attr must be given exactly when dim > 0 (dim={self.dim})")
        pair = _pair(x)
        graph = _plain_graph(edge_index, pair[0].size(0), pair[1].size(0), self.flow)
        u, v, c = cg_uvc(x if isinstance(x, Tensor) else pair, edge_attr, self.lin_f.weight, self.lin_f.bias,
                         self.lin_s.weight, self.lin_s.bias)
        out = Fn.aggregate_cg_uv(graph, u, c, self.aggr) if v is None else Fn.aggregate_cg(graph, u, v, c, self.aggr)
        if self.bn is not None:
            out = self.bn(out)
        return out + pair[1]

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.channels}, dim={self.dim})"


def _plain_linear(m) -> bool:
    t = type(m)
    return t is torch.nn.Linear or (t.__name__ == "Linear" and t.__module__ == "torch_geometric.nn.dense.linear")


def _module_hooks(m) -> bool:
    return bool(m._forward_hooks or m._forward_pre_hooks or m._backward_hooks or m._backward_pre_hooks)


def _global_module_hooks() -> bool:
    from torch.nn.modules import module as M
    return bool(M._global_forward_hooks or M._global_forward_pre_hooks or M._global_backward_hooks
                or M._global_backward_pre_hooks)


def nn_conv_split(net, f_in: int, f_out: int):
    """(modules before the last Linear, the last Linear) of NNConv's edge network, or None where it cannot be split:
    the network must be a `torch.nn.Linear` / `torch_geometric.nn.Linear`, or a `torch.nn.Sequential` ending in one,
    whose weight is initialised (not lazy) with F_in F_out rows.  The fused path never calls the network itself nor its
    last Linear, so any forward or backward hook on either, and any global module hook, makes it unsplittable: the
    reference would fire them."""
    mods = list(net) if type(net) is torch.nn.Sequential else [net]
    if not mods or not _plain_linear(mods[-1]):
        return None
    last = mods[-1]
    w = last.weight
    if isinstance(w, torch.nn.parameter.UninitializedParameter) or w.dim() != 2 or w.size(0) != f_in * f_out:
        return None
    if _module_hooks(net) or _module_hooks(last) or _global_module_hooks():
        return None
    return mods[:-1], last


def nn_conv_weight(w2: Tensor, b2: Optional[Tensor], f_in: int, f_out: int) -> Tensor:
    """W' [(K+1) F_in, F_out] of NNConv's last edge-network Linear (weight w2 [F_in F_out, K], bias b2): row k F_in + a
    holds W2.view(F_in, F_out, K)[a, :, k] and the last F_in rows b2.view(F_in, F_out), so that
    out_i = vec(P_i) W' with P_i = sum_e [h_e, 1] (x) x_j (nn_conv.py:119-122).  Views and a cat of the parameters, so
    autograd maps dW' back to w2 and b2."""
    K = w2.size(1)
    wp = w2.view(f_in, f_out, K).permute(2, 0, 1)
    bp = b2.view(1, f_in, f_out) if b2 is not None else w2.new_zeros(1, f_in, f_out)
    return torch.cat([wp, bp], dim=0).reshape((K + 1) * f_in, f_out)


def nn_conv_edge_hidden(pre, edge_attr: Tensor) -> Tensor:
    """The edge network's output before its last Linear: the user's own modules, run as torch runs them."""
    h = edge_attr
    for m in pre:
        h = m(h)
    return h


class NNConv(torch.nn.Module):
    """x_i Theta + AGGR_j x_j h(e_ji) + bias (nn_conv.py:13-126) with AGGR = sum (default) or mean.  The edge network
    h must end in a Linear (`nn_conv_split`); everything before it runs as torch modules, and the message runs with its
    aggregation as one sweep into P plus one GEMM (`Fn.nn_conv_aggregate`), without the [E, F_in F_out] weights.  Other
    aggregations and edge networks raise ValueError."""

    def __init__(self, in_channels, out_channels: int, nn, aggr: str = "add", root_weight: bool = True,
                 bias: bool = True, **kwargs):
        super().__init__()
        if aggr not in ("add", "sum", "mean"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path (add, sum or mean)")
        ch = (in_channels, in_channels) if isinstance(in_channels, int) else tuple(in_channels)
        if nn_conv_split(nn, ch[0], out_channels) is None:
            raise ValueError("the edge network must be a Linear, or a torch.nn.Sequential ending in one, with "
                             f"{ch[0]} * {out_channels} = {ch[0] * out_channels} initialised output features")
        self.in_channels, self.out_channels, self.aggr = in_channels, out_channels, aggr
        self.nn = nn
        self.root_weight = root_weight
        self.in_channels_l = ch[0]
        self.flow = kwargs.get("flow", "source_to_target")
        if root_weight:
            self.lin = _Lin(ch[1], out_channels, bias=False)                          # nn_conv.py:79-81
            bound = 1.0 / math.sqrt(ch[1])
            with torch.no_grad():
                self.lin.weight.uniform_(-bound, bound)
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None

    def forward(self, x, edge_index: Adj, edge_attr: Tensor, size=None) -> Tensor:
        pair = _pair(x)
        split = nn_conv_split(self.nn, self.in_channels_l, self.out_channels)
        if split is None:
            raise ValueError("the edge network can no longer be split at its last Linear (a hook on it or on that "
                             "Linear, a global module hook, or a changed Linear); NNConv has no unfused path")
        if torch.is_autocast_enabled(pair[0].device.type):
            raise ValueError("NNConv runs in the dtype of its inputs; it does not run under torch.autocast")
        graph = _plain_graph(edge_index, pair[0].size(0), _num_dst(pair, size), self.flow)
        pre, last = split
        w_prime = nn_conv_weight(last.weight, last.bias, self.in_channels_l, self.out_channels)
        out = Fn.nn_conv_aggregate(graph, pair[0], nn_conv_edge_hidden(pre, edge_attr), w_prime,
                                   "mean" if self.aggr == "mean" else "sum")
        if pair[1] is not None and self.root_weight:                                   # nn_conv.py:110-115
            out = out + self.lin(pair[1])
        if self.bias is not None:
            out = out + self.bias
        return out

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, aggr={self.aggr}, nn={self.nn})"


def _repeat(v, n: int) -> list:
    """torch_geometric.utils.repeat: a scalar n times, a shorter list padded with its last element."""
    if not isinstance(v, (list, tuple)):
        return [v] * n
    v = list(v)
    return v + [v[-1]] * (n - len(v)) if len(v) < n else v[:n]


def spline_conv_forward(x_src: Tensor, graph: CSRGraph, pseudo: Tensor, kernel_size: Tensor, is_open_spline: Tensor,
                        degree: int, weight: Tensor, reduce: str) -> Tensor:
    """SplineConv's message and aggregation (spline_conv.py:128-153): the CUDA basis of the pseudo-coordinates in int32
    weight indices, then one CSR sweep into P and one GEMM (`Fn.spline_conv_aggregate`)."""
    basis, wi = Fn.spline_basis(pseudo, kernel_size, is_open_spline, degree, torch.int32)
    return Fn.spline_conv_aggregate(graph, x_src, basis, wi, weight, reduce)


class SplineConv(torch.nn.Module):
    """x_i Theta + AGGR_j x_j h_Theta(e_ij) + bias (spline_conv.py:21-172) with AGGR = mean (default) or sum and h the
    B-spline kernel over the pseudo-coordinates `edge_attr` [E, dim].  The basis runs on CUDA and the message runs with
    its aggregation as one sweep into P plus one GEMM (`Fn.spline_conv_aggregate`).  Other aggregations, lazy input
    sizes and shapes the sweeps do not take raise ValueError."""

    def __init__(self, in_channels, out_channels: int, dim: int, kernel_size, is_open_spline=True, degree: int = 1,
                 aggr: str = "mean", root_weight: bool = True, bias: bool = True, **kwargs):
        super().__init__()
        if aggr not in ("add", "sum", "mean"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path (add, sum or mean)")
        ch = (in_channels, in_channels) if isinstance(in_channels, int) else tuple(in_channels)
        if ch[0] <= 0 or ch[1] <= 0:
            raise ValueError("SplineConv needs its input sizes at construction (no lazy -1)")
        self.in_channels, self.out_channels, self.dim = in_channels, out_channels, dim
        self.degree, self.root_weight, self.aggr = degree, root_weight, aggr
        self.flow = kwargs.get("flow", "source_to_target")
        self.register_buffer("kernel_size", torch.tensor(_repeat(kernel_size, dim), dtype=torch.long))
        self.register_buffer("is_open_spline", torch.tensor(_repeat(is_open_spline, dim), dtype=torch.uint8))
        self.K = int(self.kernel_size.prod().item())
        S = ops.spline_slots(dim, degree)
        if not ops.spline_supported(self.K, ch[0], S, torch.float32):
            raise ValueError(f"K = {self.K} kernels x F_in = {ch[0]} channels with {S} basis slots is outside what the "
                             "fused SplineConv takes")
        self.weight = torch.nn.Parameter(torch.empty(self.K, ch[0], out_channels))
        if root_weight:
            self.lin = _Lin(ch[1], out_channels, bias=False)      # draws as the reference's Linear(.., 'uniform') does
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None
        with torch.no_grad():                                     # spline_conv.py:118-125, in the reference's order
            bound = 1.0 / math.sqrt(self.K * ch[0])
            self.weight.uniform_(-bound, bound)
            if root_weight:
                bound = 1.0 / math.sqrt(ch[1])
                self.lin.weight.uniform_(-bound, bound)

    def forward(self, x, edge_index: Adj, edge_attr: Tensor, size=None) -> Tensor:
        pair = _pair(x)
        if torch.is_autocast_enabled(pair[0].device.type):
            raise ValueError("SplineConv runs in the dtype of its inputs; it does not run under torch.autocast")
        graph = _plain_graph(edge_index, pair[0].size(0), _num_dst(pair, size), self.flow)
        out = spline_conv_forward(pair[0], graph, edge_attr, self.kernel_size, self.is_open_spline, self.degree,
                                  self.weight, "mean" if self.aggr == "mean" else "sum")
        if pair[1] is not None and self.root_weight:                                  # spline_conv.py:140-145
            out = out + self.lin(pair[1])
        if self.bias is not None:
            out = out + self.bias
        return out

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, dim={self.dim})"


def pna_uv_c(x: Tensor, edge_attr: Optional[Tensor], pre_weights, pre_biases, enc_w: Optional[Tensor],
             enc_b: Optional[Tensor], towers: int, f_in: int, divide_input: bool):
    """u | v ([N, 2W], W = towers * f_in) and c ([E, W] or None) from the towers' one-layer pre-transforms
    Linear(cat(x_i, x_j[, edge_encoder(edge_attr)])) (pna_conv.py:167-188), split by weight column blocks:
    u = x_t Wa_t^T + b_t, v = x_t Wb_t^T, c = edge_encoder(edge_attr) Wc_t^T.  Slicing and concatenating the module's
    own parameters keeps every parameter gradient with autograd."""
    wa = [w[:, :f_in] for w in pre_weights]
    wb = [w[:, f_in:2 * f_in] for w in pre_weights]
    if divide_input:                                        # tower t reads x[:, t F : (t + 1) F]: block-diagonal weights
        w_uv = torch.cat([torch.block_diag(*wa), torch.block_diag(*wb)], dim=0)
    else:
        w_uv = torch.cat(wa + wb, dim=0)
    b_uv = torch.cat(list(pre_biases) + [torch.zeros_like(b) for b in pre_biases])
    uv = dense.linear(x, w_uv, b_uv)
    c = None
    if edge_attr is not None:
        wc = torch.cat([w[:, 2 * f_in:] for w in pre_weights], dim=0)           # [W, f_in]
        c = dense.linear(dense.linear(edge_attr, enc_w, enc_b), wc)
    return uv, c


def pna_block(x: Tensor, graph: CSRGraph, edge_attr: Optional[Tensor], pre_weights, pre_biases, enc_w, enc_b,
              aggregators, scalers, avg_deg_lin: Tensor, avg_deg_log: Tensor, towers: int, f_in: int,
              divide_input: bool) -> Tensor:
    """PNAConv's post-network input cat([x_t, scaled aggregations]) [N, towers, (1 + A S) f_in] (pna_conv.py:158-169)."""
    uv, c = pna_uv_c(x, edge_attr, pre_weights, pre_biases, enc_w, enc_b, towers, f_in, divide_input)
    x3 = x.view(-1, towers, f_in) if divide_input else x.view(-1, 1, f_in).expand(-1, towers, f_in)
    return Fn.pna_aggregate(graph, x3, uv, c, aggregators, scalers, avg_deg_lin, avg_deg_log)


_ACTS = {"relu": torch.nn.ReLU, "elu": torch.nn.ELU, "leaky_relu": torch.nn.LeakyReLU, "gelu": torch.nn.GELU,
         "tanh": torch.nn.Tanh, "sigmoid": torch.nn.Sigmoid, "silu": torch.nn.SiLU, "swish": torch.nn.SiLU}


def _activation(act, act_kwargs):
    if isinstance(act, str):
        key = act.lower().replace("_", "")
        for name, cls in _ACTS.items():
            if name.replace("_", "") == key:
                return cls(**(act_kwargs or {}))
        raise ValueError(f"Could not resolve '{act}' among choices {sorted(_ACTS)}")
    if isinstance(act, type):
        return act(**(act_kwargs or {}))
    return act


class _DegreeScalerState(torch.nn.Module):
    """avg_deg_lin / avg_deg_log of DegreeScalerAggregation (nn/aggr/scaler.py:60-75): buffers, or parameters with
    train_norm, initialised from the in-degree histogram."""

    def __init__(self, deg: Tensor, train_norm: bool):
        super().__init__()
        deg = deg.to(torch.float)
        n = float(deg.sum())
        bins = torch.arange(deg.numel(), device=deg.device, dtype=torch.float)
        self.init_avg_deg_lin = float((bins * deg).sum()) / n
        self.init_avg_deg_log = float(((bins + 1).log() * deg).sum()) / n
        if train_norm:
            self.avg_deg_lin = torch.nn.Parameter(torch.empty(1))
            self.avg_deg_log = torch.nn.Parameter(torch.empty(1))
        else:
            self.register_buffer("avg_deg_lin", torch.empty(1))
            self.register_buffer("avg_deg_log", torch.empty(1))
        self.reset_parameters()

    def reset_parameters(self):
        self.avg_deg_lin.data.fill_(self.init_avg_deg_lin)
        self.avg_deg_log.data.fill_(self.init_avg_deg_log)


class PNAConv(torch.nn.Module):
    """Principal Neighbourhood Aggregation (pna_conv.py:20-209) with one pre-layer per tower: the towers' message
    Linear is split into per-node products and the per-edge c (with `edge_dim`), and the aggregators in {sum, mean,
    min, max, var, std} with the five degree scalers run as one CSR sweep plus node-level kernels
    (`Fn.pna_aggregate`).  `pre_layers != 1` and other aggregators or scalers raise ValueError."""

    def __init__(self, in_channels: int, out_channels: int, aggregators, scalers, deg: Tensor,
                 edge_dim: Optional[int] = None, towers: int = 1, pre_layers: int = 1, post_layers: int = 1,
                 divide_input: bool = False, act="relu", act_kwargs=None, train_norm: bool = False, **kwargs):
        super().__init__()
        if pre_layers != 1:
            raise ValueError(f"pre_layers={pre_layers} is not on the fused path (only one pre-layer per tower is)")
        aggregators = [aggregators] if isinstance(aggregators, str) else list(aggregators)
        scalers = [scalers] if isinstance(scalers, str) else list(scalers)
        for a in aggregators:
            if {"add": "sum"}.get(a, a) not in ops.PNA_AGGRS:
                raise ValueError(f"aggregator '{a}' is not on the fused path (supported: {ops.PNA_AGGRS})")
        for sc in scalers:
            if sc not in ops.PNA_SCALERS:
                raise ValueError(f"Unknown scaler '{sc}'")
        if divide_input:
            assert in_channels % towers == 0
        assert out_channels % towers == 0
        self.aggregators, self.scalers = aggregators, scalers
        self.flow = kwargs.get("flow", "source_to_target")
        self.in_channels, self.out_channels, self.edge_dim = in_channels, out_channels, edge_dim
        self.towers, self.divide_input = towers, divide_input
        self.F_in = in_channels // towers if divide_input else in_channels
        self.F_out = out_channels // towers
        self.aggr_module = _DegreeScalerState(deg, train_norm)
        if edge_dim is not None:
            self.edge_encoder = _Lin(edge_dim, self.F_in)
        self.pre_nns = torch.nn.ModuleList(
            [torch.nn.Sequential(_Lin((3 if edge_dim else 2) * self.F_in, self.F_in)) for _ in range(towers)])
        self.post_nns = torch.nn.ModuleList()
        for _ in range(towers):
            mods = [_Lin((len(aggregators) * len(scalers) + 1) * self.F_in, self.F_out)]
            for _ in range(post_layers - 1):
                mods += [_activation(act, act_kwargs), _Lin(self.F_out, self.F_out)]
            self.post_nns.append(torch.nn.Sequential(*mods))
        self.lin = _Lin(out_channels, out_channels)

    def forward(self, x: Tensor, edge_index: Adj, edge_attr: Optional[Tensor] = None) -> Tensor:
        graph = _plain_graph(edge_index, x.size(0), x.size(0), self.flow)
        enc = getattr(self, "edge_encoder", None)
        block = pna_block(x, graph, edge_attr if self.edge_dim is not None else None,
                          [nn[0].weight for nn in self.pre_nns], [nn[0].bias for nn in self.pre_nns],
                          _w(enc), None if enc is None else enc.bias, self.aggregators, self.scalers,
                          self.aggr_module.avg_deg_lin, self.aggr_module.avg_deg_log, self.towers, self.F_in,
                          self.divide_input)
        # unbind: one [N, T, (1 + A S) F] gradient for all towers, where block[:, t] would allocate one per tower
        out = torch.cat([nn(b) for nn, b in zip(self.post_nns, block.unbind(1))], dim=1)
        return self.lin(out)

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, towers={self.towers}, "
                f"edge_dim={self.edge_dim})")

    @staticmethod
    def get_degree_histogram(loader) -> Tensor:
        """Histogram of the in-degrees of every graph in `loader` (index = degree), for the `deg` argument."""
        hist = torch.zeros(1, dtype=torch.long)
        for data in loader:
            dst = data.edge_index[1]
            deg = torch.zeros(data.num_nodes, dtype=torch.long, device=dst.device).index_add_(
                0, dst, torch.ones_like(dst, dtype=torch.long))
            counts = torch.bincount(deg, minlength=hist.numel())
            hist = hist.to(counts.device)
            if counts.numel() > hist.numel():
                hist = torch.cat([hist, hist.new_zeros(counts.numel() - hist.numel())])
            hist = hist + counts
        return hist


class RGCNConv(torch.nn.Module):
    """See `rgcn_conv`.  `num_bases` / `num_blocks` (rgcn_conv.py:140-160) are parametrisations of the same
    [R, F_in, F_out] weights and are expanded before the single K = R F_in (+ root) product."""

    def __init__(self, in_channels: int, out_channels: int, num_relations: int, num_bases: Optional[int] = None,
                 num_blocks: Optional[int] = None, aggr: str = "mean", root_weight: bool = True, bias: bool = True, **kwargs):
        super().__init__()
        if num_bases is not None and num_blocks is not None:
            raise ValueError("Can not apply both basis-decomposition and block-diagonal-decomposition at the same time.")
        if aggr not in ("mean", "sum", "add", "max", "min"):
            raise ValueError(f"aggr='{aggr}' is not on the fused path")
        if isinstance(in_channels, (tuple, list)):
            in_channels = in_channels[0]
        self.in_channels, self.out_channels, self.num_relations, self.aggr = in_channels, out_channels, num_relations, aggr
        self.num_bases, self.num_blocks = num_bases, num_blocks
        if num_bases is not None:
            self.weight = torch.nn.Parameter(torch.empty(num_bases, in_channels, out_channels))
            self.comp = torch.nn.Parameter(torch.empty(num_relations, num_bases))
            glorot_(self.comp)
        elif num_blocks is not None:
            assert in_channels % num_blocks == 0 and out_channels % num_blocks == 0
            self.weight = torch.nn.Parameter(torch.empty(num_relations, num_blocks, in_channels // num_blocks,
                                                         out_channels // num_blocks))
            self.register_parameter("comp", None)
        else:
            self.weight = torch.nn.Parameter(torch.empty(num_relations, in_channels, out_channels))
            self.register_parameter("comp", None)
        self.root = torch.nn.Parameter(torch.empty(in_channels, out_channels)) if root_weight else None
        self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias else None
        glorot_(self.weight)
        if self.root is not None:
            glorot_(self.root)

    def relation_graph(self, edge_index: Tensor, edge_type: Tensor, num_nodes: int) -> CSRGraph:
        return cached_graph(edge_index, num_nodes, num_nodes * self.num_relations, edge_type=edge_type,
                            num_relations=self.num_relations)

    def forward(self, x: Tensor, edge_index: Adj, edge_type: Optional[Tensor] = None) -> Tensor:
        if isinstance(edge_index, CSRGraph):
            graph = edge_index
        else:
            assert edge_type is not None
            graph = self.relation_graph(edge_index, edge_type, x.size(0))
        w = rgcn_weight(self.weight, self.comp, self.num_relations, self.in_channels, self.out_channels, self.num_blocks)
        return rgcn_conv(x, graph, w, self.root, self.bias, self.aggr)

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, "
                f"num_relations={self.num_relations})")


class FastRGCNConv(RGCNConv):
    """rgcn_conv.py:302-374 trades memory for speed with one [E, F_in] x W[edge_type] product per edge; the fused
    path above is already one sweep + one GEMM without any [E, *] tensor, so the fast variant IS the same code."""


def _attention_graph(edge_index: Adj, num_src: int, num_dst: int, add_self_loops: bool, flow: str = "source_to_target"):
    if isinstance(edge_index, CSRGraph):
        return edge_index
    return cached_graph(edge_index, num_src, num_dst, flow=flow, loops="gat" if add_self_loops else None,
                        loop_nodes=min(num_src, num_dst))


def edge_attr_with_loops(edge_index: Tensor, edge_attr: Tensor, num_nodes: int, fill_value, flow: str = "source_to_target"):
    """remove_self_loops + add_self_loops on the edge features, in the order of the graph built with loops='gat'
    (gat_conv.py:342-346; utils/loop.py:382-492: fill_value 'mean' = scatter-mean of the incoming edge features)."""
    if edge_attr.dim() == 1:
        edge_attr = edge_attr.view(-1, 1)
    keep = edge_index[0] != edge_index[1]
    ea = edge_attr[keep]
    dst = (edge_index[1] if flow == "source_to_target" else edge_index[0])[keep]
    if isinstance(fill_value, str):
        loop = U.scatter(ea.float(), dst, 0, num_nodes, fill_value).to(ea.dtype)
    elif isinstance(fill_value, Tensor):
        loop = fill_value.to(ea.dtype).view(1, -1).expand(num_nodes, ea.size(1))
    else:
        loop = ea.new_full((num_nodes, ea.size(1)), float(fill_value))
    return torch.cat([ea, loop], dim=0)


class GATConv(torch.nn.Module):
    """Mirror of torch_geometric.nn.GATConv (nn/conv/gat_conv.py:27-413) incl. bipartite inputs and `edge_dim`;
    attention + aggregation run in the fused kernel (csrc/attention.cu), attention dropout (training-time,
    gat_conv.py:404) included: the kept (edge, head) pairs come from a counter-based hash seeded from torch's CPU generator
    -- the same distribution as F.dropout, not the same random stream."""

    def __init__(self, in_channels, out_channels: int, heads: int = 1, concat: bool = True, negative_slope: float = 0.2,
                 dropout: float = 0.0, add_self_loops: bool = True, edge_dim: Optional[int] = None, fill_value="mean",
                 bias: bool = True, residual: bool = False, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.add_self_loops, self.residual = negative_slope, dropout, add_self_loops, residual
        self.edge_dim, self.fill_value = edge_dim, fill_value
        self.flow = kwargs.get("flow", "source_to_target")
        self.lin = self.lin_src = self.lin_dst = None
        if isinstance(in_channels, int):
            self.lin = _Lin(in_channels, heads * out_channels, bias=False)
        else:
            self.lin_src = _Lin(in_channels[0], heads * out_channels, bias=False)
            self.lin_dst = _Lin(in_channels[1], heads * out_channels, bias=False)
        self.att_src = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        self.att_dst = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        glorot_(self.att_src)
        glorot_(self.att_dst)
        if edge_dim is not None:
            self.lin_edge = _Lin(edge_dim, heads * out_channels, bias=False)
            self.att_edge = torch.nn.Parameter(torch.empty(1, heads, out_channels))
            glorot_(self.att_edge)
        else:
            self.lin_edge = None
            self.register_parameter("att_edge", None)
        total = heads * out_channels if concat else out_channels
        self.res = _Lin(in_channels if isinstance(in_channels, int) else in_channels[1], total, bias=False) if residual else None
        self.bias = torch.nn.Parameter(torch.zeros(total)) if bias else None

    def graph_for(self, edge_index: Adj, num_nodes: int, num_dst: Optional[int] = None) -> CSRGraph:
        return _attention_graph(edge_index, num_nodes, num_nodes if num_dst is None else num_dst, self.add_self_loops, self.flow)

    def forward(self, x, edge_index: Adj, edge_attr: Optional[Tensor] = None, size=None,
                return_attention_weights: Optional[bool] = None):
        drop = float(self.dropout) if self.training else 0.0        # attention dropout runs inside the sweep
        H, C = self.heads, self.out_channels
        att_dst = self.att_dst
        if isinstance(x, Tensor):
            assert x.dim() == 2, "Static graphs not supported in 'GATConv'"
            res = self.res(x) if self.res is not None else None
            if self.lin is not None:
                xh_src, xh_dst = self.lin(x), None
            else:
                xh_src, xh_dst = self.lin_src(x), self.lin_dst(x)
            n_src = n_dst = x.size(0)
        else:
            xs, xd = x
            assert xs.dim() == 2, "Static graphs not supported in 'GATConv'"
            res = self.res(xd) if (xd is not None and self.res is not None) else None
            lin_s, lin_d = (self.lin, self.lin) if self.lin is not None else (self.lin_src, self.lin_dst)
            xh_src, n_src = lin_s(xs), xs.size(0)
            if xd is not None:
                xh_dst, n_dst = lin_d(xd), xd.size(0)
            else:                                                        # alpha_i is absent (gat_conv.py:331)
                xh_dst, n_dst, att_dst = None, (size[1] if size is not None else n_src), None
        graph = self.graph_for(edge_index, n_src, n_dst)
        s_edge = None
        if edge_attr is not None and self.lin_edge is not None:
            if isinstance(edge_index, CSRGraph):
                raise NotImplementedError("edge_attr needs the [2, E] edge_index it is aligned with")
            ea = edge_attr if not self.add_self_loops else edge_attr_with_loops(
                edge_index, edge_attr, min(n_src, n_dst), self.fill_value, self.flow)
            if ea.dim() == 1:
                ea = ea.view(-1, 1)
            s_edge = _head_dot(self.lin_edge(ea), self.att_edge, H, C)
        want = return_attention_weights is not None
        r = gat_conv(xh_src, xh_dst, graph, self.att_src, att_dst, H, C, self.negative_slope, self.concat, res, self.bias,
                     s_edge, want, drop)
        if want:
            out, alpha = r
            ei = torch.stack([graph.col.long(), graph.dst_csr.long()])         # alpha is in the engine's CSR order
            return out, (ei, alpha)
        return r

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, heads={self.heads})"


class GATv2Conv(torch.nn.Module):
    """Mirror of torch_geometric.nn.GATv2Conv (nn/conv/gatv2_conv.py:24-385) incl. `edge_dim`: the score
    att . leaky_relu(x_l[j] + x_r[i] (+ lin_edge(e_ij))), the edge softmax and the aggregation are ONE sweep (csrc/attention.cu)."""

    def __init__(self, in_channels, out_channels: int, heads: int = 1, concat: bool = True, negative_slope: float = 0.2,
                 dropout: float = 0.0, add_self_loops: bool = True, edge_dim: Optional[int] = None, fill_value="mean",
                 bias: bool = True, residual: bool = False, share_weights: bool = False, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.add_self_loops = negative_slope, dropout, add_self_loops
        self.edge_dim, self.fill_value = edge_dim, fill_value
        self.residual, self.share_weights = residual, share_weights
        self.flow = kwargs.get("flow", "source_to_target")
        ic = (in_channels, in_channels) if isinstance(in_channels, int) else in_channels
        self.lin_l = _Lin(ic[0], heads * out_channels, bias=bias)
        self.lin_r = self.lin_l if share_weights else _Lin(ic[1], heads * out_channels, bias=bias)
        self.att = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        glorot_(self.att)
        self.lin_edge = _Lin(edge_dim, heads * out_channels, bias=False) if edge_dim is not None else None
        total = heads * out_channels if concat else out_channels
        self.res = _Lin(ic[1], total, bias=False) if residual else None
        self.bias = torch.nn.Parameter(torch.zeros(total)) if bias else None

    def forward(self, x, edge_index: Adj, edge_attr=None, return_attention_weights: Optional[bool] = None):
        drop = float(self.dropout) if self.training else 0.0        # attention dropout runs inside the sweep
        H, C = self.heads, self.out_channels
        if isinstance(x, Tensor):
            res = self.res(x) if self.res is not None else None
            x_l = self.lin_l(x)
            x_r = x_l if self.share_weights else self.lin_r(x)
        else:
            res = self.res(x[1]) if (x[1] is not None and self.res is not None) else None
            x_l = self.lin_l(x[0])
            x_r = self.lin_r(x[1])
        graph = _attention_graph(edge_index, x_l.size(0), x_r.size(0), self.add_self_loops, self.flow)
        e_feat = None
        if edge_attr is not None and self.lin_edge is not None:         # gatv2_conv.py:318-325, 358-360
            if isinstance(edge_index, CSRGraph):
                raise ValueError("edge_attr needs the [2, E] edge_index it is aligned with")
            ea = edge_attr
            if self.add_self_loops:
                ea = edge_attr_with_loops(edge_index, edge_attr, min(x_l.size(0), x_r.size(0)), self.fill_value, self.flow)
            e_feat = self.lin_edge(ea.view(-1, 1) if ea.dim() == 1 else ea)
        want = return_attention_weights is not None
        r = gatv2_conv(x_l, x_r, graph, self.att, H, C, self.negative_slope, self.concat, res, self.bias, want, drop, e_feat)
        if want:
            out, alpha = r
            return out, (torch.stack([graph.col.long(), graph.dst_csr.long()]), alpha)
        return r

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, heads={self.heads})"


class TransformerConv(torch.nn.Module):
    """Mirror of torch_geometric.nn.TransformerConv (nn/conv/transformer_conv.py:17-285) incl. `edge_dim` (lin_edge(e_ij) added
    to the key and to the value): q.k / sqrt(C) scores, edge softmax and the value aggregation in ONE sweep; keys and values come from one GEMM
    with the concatenated lin_key / lin_value weights and are read as the two halves of one [N, 2HC] matrix."""

    def __init__(self, in_channels, out_channels: int, heads: int = 1, concat: bool = True, beta: bool = False,
                 dropout: float = 0.0, edge_dim: Optional[int] = None, bias: bool = True, root_weight: bool = True, **kwargs):
        super().__init__()
        self.edge_dim = edge_dim
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.beta, self.root_weight, self.dropout = beta and root_weight, root_weight, dropout
        self.flow = kwargs.get("flow", "source_to_target")
        ic = (in_channels, in_channels) if isinstance(in_channels, int) else in_channels
        hc = heads * out_channels
        self.lin_key = _Lin(ic[0], hc, bias=bias)
        self.lin_query = _Lin(ic[1], hc, bias=bias)
        self.lin_value = _Lin(ic[0], hc, bias=bias)
        self.lin_edge = _Lin(edge_dim, hc, bias=False) if edge_dim is not None else None
        total = hc if concat else out_channels
        self.lin_skip = _Lin(ic[1], total, bias=bias)
        self.lin_beta = _Lin(3 * total, 1, bias=False) if self.beta else None

    def forward(self, x, edge_index: Adj, edge_attr=None, return_attention_weights: Optional[bool] = None):
        drop = float(self.dropout) if self.training else 0.0        # attention dropout runs inside the sweep
        H, C = self.heads, self.out_channels
        x = _pair(x)
        e_feat = None
        if self.lin_edge is not None:                                   # transformer_conv.py:258-261
            assert edge_attr is not None
            if isinstance(edge_index, CSRGraph):
                raise ValueError("edge_attr needs the [2, E] edge_index it is aligned with")
            e_feat = self.lin_edge(edge_attr.view(-1, 1) if edge_attr.dim() == 1 else edge_attr)
        query = self.lin_query(x[1])
        w_kv = torch.cat([self.lin_key.weight, self.lin_value.weight], dim=0)
        b_kv = None if self.lin_key.bias is None else torch.cat([self.lin_key.bias, self.lin_value.bias], dim=0)
        kv = dense.linear(x[0], w_kv, b_kv)
        graph = _plain_graph(edge_index, x[0].size(0), x[1].size(0), self.flow)
        x_skip = self.lin_skip(x[1]) if self.root_weight else None
        want = isinstance(return_attention_weights, bool)
        r = transformer_conv(query, kv, graph, H, C, self.concat, x_skip, _w(self.lin_beta), want, drop, e_feat)
        if want:
            out, alpha = r
            return out, (torch.stack([graph.col.long(), graph.dst_csr.long()]), alpha)
        return r

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, heads={self.heads})"


class HeteroLinear(torch.nn.Module):
    """Mirror of torch_geometric.nn.HeteroLinear (nn/dense/linear.py:174-340): x_k W_k + b_k per type k.  The per-type
    products are ONE launch of the grouped wgmma kernel (dense.segment_matmul); unsorted type vectors are sorted
    with the engine's stable radix sort and the result is un-permuted, as the reference does."""

    def __init__(self, in_channels: int, out_channels: int, num_types: int, is_sorted: bool = False, bias: bool = True, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels, self.num_types, self.is_sorted = in_channels, out_channels, num_types, is_sorted
        self.weight = torch.nn.Parameter(torch.empty(num_types, in_channels, out_channels))
        self.bias = torch.nn.Parameter(torch.zeros(num_types, out_channels)) if bias else None
        bound = 1.0 / math.sqrt(in_channels)                          # reset_weight_ (linear.py:42-60): kaiming_uniform(a=sqrt(5))
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
            if self.bias is not None:
                self.bias.uniform_(-bound, bound)

    def forward(self, x: Tensor, type_vec: Tensor) -> Tensor:
        perm = None
        if not self.is_sorted:
            type_vec, perm = U.index_sort(type_vec, self.num_types - 1)
            x = ops.gather_rows(x, perm) if x.dtype in (torch.float32, torch.bfloat16) and not x.requires_grad else x[perm]
        ptr = ops.index2ptr(type_vec, self.num_types)
        out = dense.segment_matmul(x, ptr, self.weight)
        if self.bias is not None:
            out = out + self.bias[type_vec.long()]
        if perm is not None:
            out_unsorted = torch.empty_like(out)
            out_unsorted[perm] = out
            out = out_unsorted
        return out

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, num_types={self.num_types}, "
                f"bias={self.bias is not None})")


class _MessageNorm(torch.nn.Module):
    """torch_geometric.nn.norm.MessageNorm (nn/norm/msg_norm.py:8-50): normalize(msg) * ||x|| * scale."""

    def __init__(self, learn_scale: bool = False):
        super().__init__()
        self.scale = torch.nn.Parameter(torch.ones(1), requires_grad=learn_scale)

    def reset_parameters(self):
        self.scale.data.fill_(1.0)

    def forward(self, x: Tensor, msg: Tensor) -> Tensor:
        return F.normalize(msg, p=2.0, dim=-1) * x.norm(p=2.0, dim=-1, keepdim=True) * self.scale


def _gen_mlp(channels, norm: Optional[str], bias: bool) -> torch.nn.Sequential:
    """GENConv's MLP (gen_conv.py:21-42) for norm in {'batch', None}: Linear, [BatchNorm1d,] ReLU, Dropout(0) per hidden
    layer, so that the state_dict keys are the reference's (mlp.0.weight, mlp.1.running_mean, ...)."""
    m = []
    for i in range(1, len(channels)):
        m.append(_Lin(channels[i - 1], channels[i], bias=bias))
        if i < len(channels) - 1:
            if norm == "batch":
                m.append(torch.nn.BatchNorm1d(channels[i], affine=True))
            m.append(torch.nn.ReLU())
            m.append(torch.nn.Dropout(0.0))
    return torch.nn.Sequential(*m)


class GENConv(torch.nn.Module):
    """x_dst + MLP(AGGR_j (relu(x_j + e_ji) + eps)) (gen_conv.py:45-243) with AGGR the softmax aggregation (t, learn_t,
    'softmax_sg') or the power mean (p, learn_p): the message and its aggregation run as one sweep
    (`Fn.softmax_aggregate` / `Fn.power_mean_aggregate` with the relu_eps message), nothing stored per edge.  t and p
    are read in fp32 on the device.  Other aggregations, and norms other than 'batch' and None, raise ValueError."""

    AGGRS = ("softmax", "softmax_sg", "powermean", "power")

    def __init__(self, in_channels, out_channels: int, aggr: str = "softmax", t: float = 1.0, learn_t: bool = False,
                 p: float = 1.0, learn_p: bool = False, msg_norm: bool = False, learn_msg_scale: bool = False,
                 norm: Optional[str] = "batch", num_layers: int = 2, expansion: int = 2, eps: float = 1e-7,
                 bias: bool = False, edge_dim: Optional[int] = None, **kwargs):
        super().__init__()
        from .aggr import PowerMeanAggregation, SoftmaxAggregation
        if not isinstance(aggr, str) or aggr not in self.AGGRS:
            raise ValueError(f"aggr={aggr!r} is not on the fused path (supported: {self.AGGRS})")
        if norm not in ("batch", None):
            raise ValueError(f"norm={norm!r} is not supported (supported: 'batch', None)")
        semi_grad = aggr == "softmax_sg"
        self.aggr = "softmax" if aggr in ("softmax", "softmax_sg") else "powermean"   # gen_conv.py:141-143
        akw = kwargs.pop("aggr_kwargs", None)
        if akw is None:
            akw = dict(t=t, learn=learn_t, semi_grad=semi_grad) if self.aggr == "softmax" else dict(p=p, learn=learn_p)
        self.aggr_module = SoftmaxAggregation(**akw) if self.aggr == "softmax" else PowerMeanAggregation(**akw)
        self.flow = kwargs.pop("flow", "source_to_target")
        self.in_channels, self.out_channels, self.eps = in_channels, out_channels, eps
        ch = (in_channels, in_channels) if isinstance(in_channels, int) else tuple(in_channels)
        if ch[0] != out_channels:
            self.lin_src = _Lin(ch[0], out_channels, bias=bias)
        if edge_dim is not None and edge_dim != out_channels:
            self.lin_edge = _Lin(edge_dim, out_channels, bias=bias)
        if ch[1] != out_channels:
            self.lin_dst = _Lin(ch[1], out_channels, bias=bias)
        self.mlp = _gen_mlp([out_channels] + [out_channels * expansion] * (num_layers - 1) + [out_channels], norm, bias)
        if msg_norm:
            self.msg_norm = _MessageNorm(learn_msg_scale)

    def forward(self, x, edge_index: Adj, edge_attr: Optional[Tensor] = None, size=None) -> Tensor:
        from .aggr import SoftmaxAggregation
        pair = _pair(x)
        x_src = self.lin_src(pair[0]) if hasattr(self, "lin_src") else pair[0]
        n_dst = pair[1].size(0) if pair[1] is not None else (size[1] if size is not None else x_src.size(0))
        graph = _plain_graph(edge_index, x_src.size(0), n_dst, self.flow)
        ea = edge_attr
        if ea is not None and hasattr(self, "lin_edge"):
            ea = self.lin_edge(ea)
        if ea is not None and ea.size(-1) != x_src.size(-1):
            raise ValueError(f"edge features have {ea.size(-1)} channels, the messages {x_src.size(-1)}")
        a = self.aggr_module
        if isinstance(a, SoftmaxAggregation):
            out = Fn.softmax_aggregate(graph, x_src, ea, a.t, self.eps, "relu_eps", a.semi_grad and not a.learn)
        else:
            out = Fn.power_mean_aggregate(graph, x_src, ea, a.p, self.eps, "relu_eps", a.min_value, a.max_value)
        if hasattr(self, "msg_norm"):                                             # gen_conv.py:218-221
            out = self.msg_norm(pair[1] if pair[1] is not None else x_src, out)
        if pair[1] is not None:
            out = out + (self.lin_dst(pair[1]) if hasattr(self, "lin_dst") else pair[1])
        return self.mlp(out)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, aggr={self.aggr})"
