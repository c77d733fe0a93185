"""Subclasses of the reference's models that keep their data where the engine can use it.

`B200Node2Vec(Node2Vec)`: the reference keeps the CSR graph its walks run on as plain CPU attributes
(nn/models/node2vec.py:68-69) and samples in DataLoader workers on the CPU, where it needs pyg-lib.  Here rowptr and
col are non-persistent buffers, so `.to(device)` moves them with the embedding and `state_dict()` stays
`{'embedding.weight'}`; `sample()` moves each batch to their device, so the walks of a CUDA model run in
csrc/random_walk.cu through torch.ops.pyg.random_walk.  Everything else (loss, negative sampling, test) is the
reference's own code.
"""
from __future__ import annotations

from typing import List, Tuple, Union

import torch
import torch_geometric.nn.models.node2vec as tg_node2vec
from torch import Tensor
from torch.utils.data import DataLoader

from . import shims

# DataLoader arguments that only mean something with worker processes
_WORKER_ONLY = ("num_workers", "persistent_workers", "prefetch_factor", "worker_init_fn", "multiprocessing_context",
                "pin_memory", "pin_memory_device", "timeout")


class B200Node2Vec(tg_node2vec.Node2Vec):
    def __init__(self, *args, **kwargs):
        shims.register_walk_ops()
        # the reference's constructor checks its module's binding of WITH_PYG_LIB; the walks it needs are served here
        had = tg_node2vec.WITH_PYG_LIB
        tg_node2vec.WITH_PYG_LIB = True
        try:
            super().__init__(*args, **kwargs)
        finally:
            tg_node2vec.WITH_PYG_LIB = had
        rowptr, col = self.rowptr, self.col
        del self.rowptr, self.col
        self.register_buffer("rowptr", rowptr, persistent=False)
        self.register_buffer("col", col, persistent=False)

    def loader(self, **kwargs) -> DataLoader:
        """The reference's loader.  On a CUDA model the batches are sampled in the main process (num_workers = 0, and
        the worker-only arguments dropped): the walks are CUDA kernels, and forked DataLoader workers cannot launch
        them.  examples/node2vec.py asks for 4 workers, which on the CPU hide the sampling; on the GPU a batch's walks
        take a kernel launch."""
        if self.rowptr.is_cuda:
            kwargs = {k: v for k, v in kwargs.items() if k not in _WORKER_ONLY}
        return super().loader(**kwargs)

    def sample(self, batch: Union[List[int], Tensor]) -> Tuple[Tensor, Tensor]:
        if not isinstance(batch, Tensor):
            batch = torch.tensor(batch)
        return super().sample(batch.to(self.rowptr.device))
