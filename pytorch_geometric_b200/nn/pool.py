"""Graph construction on point clouds: mirrors of torch_geometric.nn.{fps, knn, knn_graph, radius, radius_graph,
nearest} (nn/pool/__init__.py:41-375) on the sm_90a kernels of csrc/point.cu.

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


__all__ = ['fps', 'knn', 'knn_graph', 'radius', 'radius_graph', 'nearest']
