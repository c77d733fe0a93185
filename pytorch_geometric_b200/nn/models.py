"""Node2Vec (nn/models/node2vec.py): skip-gram node embeddings trained on random walks, with the walks drawn by
ops.random_walk (csrc/random_walk.cu).

Same constructor arguments, methods and state_dict keys ({'embedding.weight'}) as the reference.  The CSR graph the
walks run on is held in non-persistent buffers, so `.to(device)` moves it with the embedding; the walks need it on a
CUDA device (the engine has no CPU path).  `loader()` samples in the main process on a CUDA model: the walks are CUDA
kernels, and forked DataLoader workers cannot launch them.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import torch
from torch import Tensor
from torch.nn import Embedding
from torch.utils.data import DataLoader

from .. import ops
from .. import utils as U

_WORKER_ONLY = ("num_workers", "persistent_workers", "prefetch_factor", "worker_init_fn", "multiprocessing_context",
                "pin_memory", "pin_memory_device", "timeout")


class Node2Vec(torch.nn.Module):
    """Node2Vec(edge_index, embedding_dim, walk_length, context_size, walks_per_node=1, p=1, q=1,
    num_negative_samples=1, num_nodes=None, sparse=False).  Each walk of walk_length nodes (walk_length - 1 steps,
    return parameter p, in-out parameter q) gives walk_length + 1 - context_size windows of context_size nodes."""

    EPS = 1e-15

    def __init__(self, edge_index: Tensor, embedding_dim: int, walk_length: int, context_size: int,
                 walks_per_node: int = 1, p: float = 1.0, q: float = 1.0, num_negative_samples: int = 1,
                 num_nodes: Optional[int] = None, sparse: bool = False):
        super().__init__()
        if walk_length < context_size:
            raise ValueError(f"walk_length ({walk_length}) must be at least context_size ({context_size})")
        if num_nodes is None:
            num_nodes = int(edge_index.max()) + 1 if edge_index.numel() > 0 else 0
        self.num_nodes = num_nodes
        dev = edge_index.device
        row, col, _ = U.sort_edge_index_by_row_col(edge_index.cuda(), num_nodes)
        self.register_buffer("rowptr", ops.index2ptr(row, num_nodes).to(dev), persistent=False)
        self.register_buffer("col", col.to(dev), persistent=False)
        self.embedding_dim = embedding_dim
        self.walk_length = walk_length - 1
        self.context_size = context_size
        self.walks_per_node = walks_per_node
        self.p, self.q = p, q
        self.num_negative_samples = num_negative_samples
        self.embedding = Embedding(num_nodes, embedding_dim, sparse=sparse)
        self.reset_parameters()

    def reset_parameters(self):
        self.embedding.reset_parameters()

    def forward(self, batch: Optional[Tensor] = None) -> Tensor:
        return self.embedding.weight if batch is None else self.embedding.weight[batch]

    def loader(self, **kwargs) -> DataLoader:
        if self.rowptr.is_cuda:
            kwargs = {k: v for k, v in kwargs.items() if k not in _WORKER_ONLY}
        return DataLoader(range(self.num_nodes), collate_fn=self.sample, **kwargs)

    def _windows(self, rw: Tensor) -> Tensor:
        """The context windows of every walk: rows rw[:, j:j + context_size], j = 0 .. walk_length + 1 - context."""
        return torch.cat([rw[:, j:j + self.context_size] for j in range(self.walk_length + 2 - self.context_size)])

    def pos_sample(self, batch: Tensor) -> Tensor:
        start = batch.repeat(self.walks_per_node)
        return self._windows(ops.random_walk(self.rowptr, self.col, start, self.walk_length, self.p, self.q))

    def neg_sample(self, batch: Tensor) -> Tensor:
        start = batch.repeat(self.walks_per_node * self.num_negative_samples)
        rest = torch.randint(self.num_nodes, (start.size(0), self.walk_length), dtype=start.dtype, device=start.device)
        return self._windows(torch.cat([start.view(-1, 1), rest], dim=-1))

    def sample(self, batch: Union[List[int], Tensor]) -> Tuple[Tensor, Tensor]:
        if not isinstance(batch, Tensor):
            batch = torch.tensor(batch)
        batch = batch.to(self.rowptr.device, self.rowptr.dtype)
        return self.pos_sample(batch), self.neg_sample(batch)

    def _scores(self, rw: Tensor) -> Tensor:
        first = self.embedding(rw[:, 0]).unsqueeze(1)
        rest = self.embedding(rw[:, 1:].reshape(-1)).view(rw.size(0), -1, self.embedding_dim)
        return (first * rest).sum(dim=-1).view(-1)

    def loss(self, pos_rw: Tensor, neg_rw: Tensor) -> Tensor:
        """Negative-sampling skip-gram loss: -log sigmoid(s) over the positive pairs, -log(1 - sigmoid(s)) over the
        negative ones, each averaged."""
        pos = -torch.log(torch.sigmoid(self._scores(pos_rw)) + self.EPS).mean()
        neg = -torch.log(1 - torch.sigmoid(self._scores(neg_rw)) + self.EPS).mean()
        return pos + neg

    def test(self, train_z: Tensor, train_y: Tensor, test_z: Tensor, test_y: Tensor, solver: str = "lbfgs", *args,
             **kwargs) -> float:
        """Accuracy of a logistic regression fitted on (train_z, train_y), scored on (test_z, test_y)."""
        from sklearn.linear_model import LogisticRegression
        clf = LogisticRegression(*args, solver=solver, **kwargs).fit(train_z.detach().cpu().numpy(),
                                                                     train_y.detach().cpu().numpy())
        return clf.score(test_z.detach().cpu().numpy(), test_y.detach().cpu().numpy())

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.embedding.weight.size(0)}, {self.embedding.weight.size(1)})"
