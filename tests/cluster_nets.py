"""The two MNIST-superpixel networks of the reference's examples (examples/mnist_graclus.py and
examples/mnist_voxel_grid.py), restated layer for layer on the reference's public API for the golden data, the GPU
tests and benchmarks/cluster.py, with a synthetic superpixel batch in place of the MNISTSuperpixels download.  The
only addition is that each network records the cluster vectors it computes in `self.clusters`.

Each function imports torch_geometric when called, so the caller decides which copy is importable and whether the
plug-in is installed (SplineConv is looked up at construction time).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

NUM_FEATURES, NUM_CLASSES = 1, 10
GRAD_FULL = 16384       # parameter gradients up to this many entries are kept whole in the golden data
GRAD_SAMPLE = 4096      # entries kept of a larger one


def seed_parameters(model, seed):
    """Sets every parameter from a seeded CPU generator, U(-b, b) with b = 1 / sqrt(entries per leading index), in
    named_parameters order.  The values do not depend on how the layer classes initialise themselves, so the golden
    data need not store them."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, p in model.named_parameters():
            b = 1.0 / math.sqrt(p[0].numel() if p.dim() > 1 else p.numel())
            p.copy_((torch.rand(p.shape, generator=g) * 2.0 - 1.0) * b)
    return model


def grad_entries(numel):
    """Flat indices of the gradient entries the golden data keeps: all of them up to GRAD_FULL entries, else
    GRAD_SAMPLE spread over the whole tensor (one per stride, at a varying offset within it)."""
    if numel <= GRAD_FULL:
        return np.arange(numel)
    i = np.arange(GRAD_SAMPLE, dtype=np.int64)
    stride = numel // GRAD_SAMPLE
    return i * stride + (i * 2654435761) % stride


def graclus_net():
    import torch_geometric.nn as tgnn
    import torch_geometric.transforms as T
    from torch_geometric.utils import normalized_cut

    transform = T.Cartesian(cat=False)

    def cut_weights(edge_index, pos):
        row, col = edge_index
        return normalized_cut(edge_index, torch.norm(pos[row] - pos[col], p=2, dim=1), num_nodes=pos.size(0))

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = tgnn.SplineConv(NUM_FEATURES, 32, dim=2, kernel_size=5)
            self.conv2 = tgnn.SplineConv(32, 64, dim=2, kernel_size=5)
            self.fc1 = torch.nn.Linear(64, 128)
            self.fc2 = torch.nn.Linear(128, NUM_CLASSES)
            self.clusters = []

        def forward(self, data):
            self.clusters = []
            data.x = F.elu(self.conv1(data.x, data.edge_index, data.edge_attr))
            cluster = tgnn.graclus(data.edge_index, cut_weights(data.edge_index, data.pos), data.x.size(0))
            self.clusters.append(cluster)
            data.edge_attr = None
            data = tgnn.max_pool(cluster, data, transform=transform)
            data.x = F.elu(self.conv2(data.x, data.edge_index, data.edge_attr))
            cluster = tgnn.graclus(data.edge_index, cut_weights(data.edge_index, data.pos), data.x.size(0))
            self.clusters.append(cluster)
            x, batch = tgnn.max_pool_x(cluster, data.x, data.batch)
            x = tgnn.global_mean_pool(x, batch)
            x = F.dropout(F.elu(self.fc1(x)), training=self.training)
            return F.log_softmax(self.fc2(x), dim=1)

    return Net()


def voxel_grid_net():
    import torch_geometric.nn as tgnn
    import torch_geometric.transforms as T

    transform = T.Cartesian(cat=False)

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv1 = tgnn.SplineConv(NUM_FEATURES, 32, dim=2, kernel_size=5)
            self.conv2 = tgnn.SplineConv(32, 64, dim=2, kernel_size=5)
            self.conv3 = tgnn.SplineConv(64, 64, dim=2, kernel_size=5)
            self.fc1 = torch.nn.Linear(4 * 64, 128)
            self.fc2 = torch.nn.Linear(128, NUM_CLASSES)
            self.clusters = []

        def forward(self, data):
            self.clusters = []
            for conv, size, end in ((self.conv1, 5, 28), (self.conv2, 7, 28)):
                data.x = F.elu(conv(data.x, data.edge_index, data.edge_attr))
                cluster = tgnn.voxel_grid(data.pos, batch=data.batch, size=size, start=0, end=end)
                self.clusters.append(cluster)
                data.edge_attr = None
                data = tgnn.max_pool(cluster, data, transform=transform)
            data.x = F.elu(self.conv3(data.x, data.edge_index, data.edge_attr))
            cluster = tgnn.voxel_grid(data.pos, batch=data.batch, size=14, start=0, end=27.99)
            self.clusters.append(cluster)
            x, _ = tgnn.max_pool_x(cluster, data.x, data.batch, size=4)
            x = F.dropout(F.elu(self.fc1(x.view(-1, self.fc1.weight.size(1)))), training=self.training)
            return F.log_softmax(self.fc2(x), dim=1)

    return Net()


def superpixel_arrays(n_graphs, n_nodes=75, k=6, seed=0):
    """A synthetic MNIST-superpixel batch as numpy arrays: positions in [0, 28)^2 (float32, rounded to 1/64 so that
    every coordinate is exact), one intensity feature, and each node joined to its k nearest neighbours, made
    symmetric.  Returns (x [N, 1], pos [N, 2], edge_index [2, E] sorted by (row, col), batch [N], y [B])."""
    rng = np.random.default_rng(seed)
    xs, ps, es, bs = [], [], [], []
    for g in range(n_graphs):
        pos = np.round(rng.random((n_nodes, 2)) * 28.0 * 64) / 64
        pos = np.minimum(pos, 28.0 - 1 / 64).astype(np.float32)
        d = ((pos[:, None, :].astype(np.float64) - pos[None, :, :]) ** 2).sum(-1)
        np.fill_diagonal(d, np.inf)
        nb = np.argsort(d, axis=1, kind="stable")[:, :k]
        row = np.repeat(np.arange(n_nodes), k)
        col = nb.reshape(-1)
        key = np.unique(np.concatenate([row * n_nodes + col, col * n_nodes + row]))
        es.append(np.stack([key // n_nodes, key % n_nodes]) + g * n_nodes)
        xs.append(rng.random((n_nodes, 1)).astype(np.float32))
        ps.append(pos)
        bs.append(np.full(n_nodes, g))
    y = rng.integers(0, NUM_CLASSES, n_graphs)
    return np.concatenate(xs), np.concatenate(ps), np.concatenate(es, axis=1), np.concatenate(bs), y


def superpixel_batch(arrays, device="cpu"):
    """The reference's Batch of superpixel_arrays(), with edge_attr from T.Cartesian(cat=False) as the examples'
    dataset transform computes it."""
    import torch_geometric.transforms as T
    from torch_geometric.data import Batch
    x, pos, ei, batch, y = (torch.from_numpy(np.asarray(a)) for a in arrays)
    data = Batch(x=x, pos=pos, edge_index=ei.long(), batch=batch.long(), y=y.long(),
                 ptr=torch.from_numpy(np.concatenate([[0], np.cumsum(np.bincount(arrays[3]))])).long())
    data = data.to(device)
    return T.Cartesian(cat=False)(data)
