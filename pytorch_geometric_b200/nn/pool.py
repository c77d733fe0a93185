"""Graph construction on point clouds and cluster vectors for pooling: mirrors of torch_geometric.nn.{fps, knn,
knn_graph, radius, radius_graph, nearest} (nn/pool/__init__.py:41-375) on the sm_90a kernels of csrc/point.cu, and of
graclus and voxel_grid (nn/pool/graclus.py, nn/pool/voxel_grid.py) on those of csrc/cluster.cu.

Signatures, defaults, `flow` and `loop` handling and `batch_size` are the reference's; `num_workers` is accepted and
ignored, as the reference documents for inputs on the GPU.  Inputs are CUDA float32 / bfloat16 tensors (CPU, float16
and float64 inputs raise RuntimeError: the engine has no CPU path).  Inputs may require grad; the outputs are integer
and never do.
"""
from __future__ import annotations

import warnings
from typing import Optional

import torch
from torch import Tensor

from .. import ops


def _batch_to_ptr(batch: Optional[Tensor], batch_size: Optional[int] = None) -> Optional[Tensor]:
    if batch is None:
        return None
    if batch_size is None:
        batch_size = int(batch.max()) + 1 if batch.numel() > 0 else 0
    return ops.index2ptr(batch, batch_size)


def fps(x: Tensor, batch: Optional[Tensor] = None, ratio: float = 0.5, random_start: bool = True,
        batch_size: Optional[int] = None) -> Tensor:
    ptr = _batch_to_ptr(batch, batch_size)
    src = x.view(x.size(0), -1) if x.dim() > 2 else x
    return ops.fps(src, ptr, ratio, random_start)


def knn(x: Tensor, y: Tensor, k: int, batch_x: Optional[Tensor] = None, batch_y: Optional[Tensor] = None,
        cosine: bool = False, num_workers: int = 1, batch_size: Optional[int] = None) -> Tensor:
    return ops.knn(x, y, k, _batch_to_ptr(batch_x, batch_size), _batch_to_ptr(batch_y, batch_size), cosine)


def knn_graph(x: Tensor, k: int, batch: Optional[Tensor] = None, loop: bool = False, flow: str = 'source_to_target',
              cosine: bool = False, num_workers: int = 1, batch_size: Optional[int] = None) -> Tensor:
    if batch is not None and x.device != batch.device:
        warnings.warn("Input tensor 'x' and 'batch' are on different devices in 'knn_graph'. Performing blocking "
                      "device transfer", stacklevel=2)
        batch = batch.to(x.device)
    assert flow in ['source_to_target', 'target_to_source']
    ptr = _batch_to_ptr(batch, batch_size)
    # the reference's composition: k + 1 neighbours, then drop each point itself
    edge_index = ops.knn(x, x, k if loop else k + 1, ptr, ptr, cosine)
    if not loop:
        edge_index = edge_index[:, edge_index[0] != edge_index[1]]
    return edge_index.flip([0]) if flow == 'source_to_target' else edge_index


def radius(x: Tensor, y: Tensor, r: float, batch_x: Optional[Tensor] = None, batch_y: Optional[Tensor] = None,
           max_num_neighbors: int = 32, num_workers: int = 1, batch_size: Optional[int] = None) -> Tensor:
    return ops.radius(x, y, r, _batch_to_ptr(batch_x, batch_size), _batch_to_ptr(batch_y, batch_size),
                      max_num_neighbors, False)


def radius_graph(x: Tensor, r: float, batch: Optional[Tensor] = None, loop: bool = False, max_num_neighbors: int = 32,
                 flow: str = 'source_to_target', num_workers: int = 1, batch_size: Optional[int] = None) -> Tensor:
    if batch is not None and x.device != batch.device:
        warnings.warn("Input tensor 'x' and 'batch' are on different devices in 'radius_graph'. Performing blocking "
                      "device transfer", stacklevel=2)
        batch = batch.to(x.device)
    assert flow in ['source_to_target', 'target_to_source']
    ptr = _batch_to_ptr(batch, batch_size)
    edge_index = ops.radius(x, x, r, ptr, ptr, max_num_neighbors, not loop)
    return edge_index.flip([0]) if flow == 'source_to_target' else edge_index


def nearest(x: Tensor, y: Tensor, batch_x: Optional[Tensor] = None, batch_y: Optional[Tensor] = None) -> Tensor:
    """For each element of x, the index of the nearest element of y in the same example (torch-cluster's cluster
    vector of size x.size(0)).  ValueError when an example of x has no y points."""
    return ops.nearest(x, y, _batch_to_ptr(batch_x), _batch_to_ptr(batch_y))


def graclus(edge_index: Tensor, weight: Optional[Tensor] = None, num_nodes: Optional[int] = None) -> Tensor:
    """Greedy matching of the graph (nn/pool/graclus.py:12-39): the edges sorted by source, then ops.graclus on the
    CSR adjacency.  Returns the cluster vector: min(u, v) for each matched pair, u for each singleton.  The colouring
    seed is drawn from torch's CPU generator."""
    if num_nodes is None:
        num_nodes = int(edge_index.max()) + 1 if edge_index.numel() > 0 else 0
    row, col = edge_index[0], edge_index[1]
    # sort_edge_index's order: by row, then by column (a stable sort of the key row * N + col)
    perm = torch.sort(row.long() * num_nodes + col.long(), stable=True)[1]
    row, col = row[perm], col[perm]
    weight = None if weight is None else weight[perm]
    return ops.graclus(ops.index2ptr(row, num_nodes), col, weight)


def _coords(v, dim: int, like: Tensor) -> Tensor:
    """The reference's `repeat(v, dim)` of a number, list or tensor, as a tensor of like's dtype and device."""
    if not isinstance(v, Tensor):
        v = torch.tensor(v, dtype=like.dtype, device=like.device)
    v = v.reshape(-1)
    if v.numel() == 1:
        return v.repeat(dim)
    if v.numel() >= dim:
        return v[:dim]
    return torch.cat([v, v[-1:].repeat(dim - v.numel())])


def voxel_grid(pos: Tensor, size, batch: Optional[Tensor] = None, start=None, end=None) -> Tensor:
    """Voxel grid pooling's cluster vector (nn/pool/voxel_grid.py:9-66): the batch index is appended to pos as one more
    coordinate of voxel size 1 (start 0, end batch.max()), then ops.grid_cluster.  pos is CUDA float32 / float64."""
    pos = pos.unsqueeze(-1) if pos.dim() == 1 else pos
    dim = pos.size(1)
    if batch is None:
        batch = pos.new_zeros(pos.size(0), dtype=torch.long)
    pos = torch.cat([pos, batch.view(-1, 1).to(pos.dtype)], dim=-1)
    size = torch.cat([_coords(size, dim, pos), pos.new_ones(1)])
    if start is not None:
        start = torch.cat([_coords(start, dim, pos), pos.new_zeros(1)])
    if end is not None:
        end = torch.cat([_coords(end, dim, pos), batch.max().unsqueeze(0).to(pos.dtype)])
    return ops.grid_cluster(pos, size, start, end)


__all__ = ['fps', 'knn', 'knn_graph', 'radius', 'radius_graph', 'nearest', 'graclus', 'voxel_grid']
