"""Restatement of the reference's DEFAULT CPU path for GCNConv on a plain [2,E] edge_index, as the
exact sequence of ATen calls the reference issues (SURVEY.md section 3.1) -- used as the timed CPU
arm (`bench.py --impl reference`, `cpu_baseline`) when the reference package is not installed in
oracle/_ref.  TEST / BENCH INFRASTRUCTURE ONLY: never imported by pytorch_geometric_b200/.

  gcn_norm                 nn/conv/gcn_conv.py:95-113   (add_remaining_self_loops loop.py:623-657,
                                                         scatter _scatter.py:68-70)
  lin                      nn/dense/linear.py:121-127   F.linear
  collect: x_j             nn/conv/message_passing.py:263-290  index_select
  message                  gcn_conv.py:270-271          edge_weight.view(-1,1) * x_j
  aggregate                aggr/base.py:173-185 -> _scatter.py:68-70  zeros.scatter_add_(0, index.expand, src)
  + bias                   gcn_conv.py:265-266

It is validated against the golden GCNConv fixture (tests/test_oracle_golden.py) so it is the
reference's arithmetic, not an approximation of it.  Backward is torch autograd over these ops,
exactly what the reference gets.
"""
from __future__ import annotations

import torch


def add_remaining_self_loops(edge_index, edge_weight, fill_value, num_nodes):
    mask = edge_index[0] != edge_index[1]
    loop_index = torch.arange(0, num_nodes, device=edge_index.device).view(1, -1).repeat(2, 1)
    if edge_weight is not None:
        loop_attr = edge_weight.new_full((num_nodes, ), fill_value)
        inv_mask = ~mask
        loop_attr[edge_index[0][inv_mask]] = edge_weight[inv_mask]
        edge_weight = torch.cat([edge_weight[mask], loop_attr], dim=0)
    edge_index = torch.cat([edge_index[:, mask], loop_index], dim=1)
    return edge_index, edge_weight


def gcn_norm(edge_index, edge_weight, num_nodes, improved=False, add_self_loops=True, dtype=torch.float32):
    fill_value = 2.0 if improved else 1.0
    if add_self_loops:
        edge_index, edge_weight = add_remaining_self_loops(edge_index, edge_weight, fill_value, num_nodes)
    if edge_weight is None:
        edge_weight = torch.ones((edge_index.size(1), ), dtype=dtype, device=edge_index.device)
    row, col = edge_index[0], edge_index[1]
    deg = edge_weight.new_zeros(num_nodes).scatter_add_(0, col, edge_weight)
    deg_inv_sqrt = deg.pow_(-0.5)
    deg_inv_sqrt.masked_fill_(deg_inv_sqrt == float("inf"), 0)
    edge_weight = deg_inv_sqrt[row] * edge_weight * deg_inv_sqrt[col]
    return edge_index, edge_weight


def gcn_conv_forward(x, edge_index, edge_weight, weight, bias):
    """edge_index / edge_weight are the gcn_norm outputs (GCNConv(cached=True) after the first call)."""
    xw = torch.nn.functional.linear(x, weight)
    x_j = xw.index_select(0, edge_index[0])
    msg = edge_weight.view(-1, 1) * x_j
    index = edge_index[1].view(-1, 1).expand_as(msg)
    out = msg.new_zeros((x.size(0), msg.size(1))).scatter_add_(0, index, msg)
    if bias is not None:
        out = out + bias
    return out
