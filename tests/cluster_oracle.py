"""numpy restatement of the clustering ops of csrc/cluster.cu (pyg_lib.ops graclus_cluster / grid_cluster), the
contract the GPU kernels are tested against bit for bit.

graclus: the same splitmix64 colouring, the same three phases per round (propose, respond, settle), the same choice
rules (first in CSR order, or the largest weight with ties to the earlier CSR position), the same cap of 256 rounds.
Each phase is vectorised over nodes, which is exact because a phase reads only what earlier phases wrote.

grid_cluster: one float32 / float64 subtract and one divide per term, one operation at a time, converted toward zero
(saturating; NaN -> INT64_MIN) and summed with int64 wrap-around.
"""
import numpy as np
import torch

MAX_ROUNDS = 256
SINGLETON = -2


def blue(seed, rnd, n, nodes):
    """Colour of `nodes` in round `rnd`: the top bit of splitmix64's finaliser on seed + (rnd n + u) * golden ratio."""
    with np.errstate(over="ignore"):
        key = np.uint64(rnd) * np.uint64(n) + np.asarray(nodes, dtype=np.uint64)
        z = np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF) + key * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return (z >> np.uint64(63)) == 1


def _pick(src, pos, w, n):
    """For each node, the chosen entry among the edges (src, pos, w): the largest w, ties to the lowest position;
    -1 where a node has none."""
    out = np.full(n, -1, dtype=np.int64)
    if src.size == 0:
        return out
    order = np.lexsort((pos, -w, src))
    s = src[order]
    first = np.ones(s.size, dtype=bool)
    first[1:] = s[1:] != s[:-1]
    out[s[first]] = pos[order][first]
    return out


def _node(col, pick):
    """The node at each picked CSR position, -1 where nothing was picked."""
    return np.where(pick >= 0, col[np.maximum(pick, 0)], -1) if col.size else np.full(pick.size, -1, np.int64)


def graclus(rowptr, col, weight=None, seed=0):
    """(cluster [N] int64, rounds).  weight: one value per CSR entry (compared in float64)."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    col = np.asarray(col, dtype=np.int64)
    n = rowptr.size - 1
    cluster = np.full(n, -1, dtype=np.int64)
    if n == 0:
        return cluster, 0
    src = np.repeat(np.arange(n, dtype=np.int64), np.diff(rowptr))
    pos = np.arange(col.size, dtype=np.int64)
    w = np.zeros(col.size) if weight is None else np.asarray(weight, dtype=np.float64)
    keep = (col != src) & ~np.isnan(w)                   # self-loops and NaN weights are never candidates
    src, dst, pos, w = src[keep], col[keep], pos[keep], w[keep]
    nodes = np.arange(n, dtype=np.int64)
    proposal = np.full(n, -1, dtype=np.int64)
    accept = np.full(n, -1, dtype=np.int64)
    rnd = 0
    while rnd < MAX_ROUNDS:
        b = blue(seed, rnd, n, nodes)
        free = cluster == -1
        cand = free[src] & free[dst]
        s, d, p, ww = src[cand], dst[cand], pos[cand], w[cand]
        has = np.bincount(s, minlength=n) > 0
        # propose: unmatched blue nodes to a red candidate
        m = b[s] & ~b[d]
        pick = _pick(s[m], p[m], ww[m], n)
        prop_node = _node(col, pick)
        bf = free & b
        proposal[bf] = np.where(has[bf], prop_node[bf], SINGLETON)
        # respond: unmatched red nodes accept a blue candidate that proposed to them
        m = ~b[s] & b[d] & (proposal[d] == s)
        pick = _pick(s[m], p[m], ww[m], n)
        acc_node = _node(col, pick)
        rf = free & ~b
        accept[rf] = np.where(has[rf], acc_node[rf], SINGLETON)
        # settle
        new = cluster.copy()
        u = nodes[bf]
        pu = proposal[u]
        single = pu == SINGLETON
        new[u[single]] = u[single]
        ok = (pu >= 0) & (accept[np.maximum(pu, 0)] == u)
        new[u[ok]] = np.minimum(u[ok], pu[ok])
        u = nodes[rf]
        au = accept[u]
        single = au == SINGLETON
        new[u[single]] = u[single]
        ok = au >= 0
        new[u[ok]] = np.minimum(u[ok], au[ok])
        cluster = new
        rnd += 1
        if not (cluster == -1).any():
            break
    left = cluster == -1
    cluster[left] = nodes[left]
    return cluster, rnd


def _trunc(v):
    """Toward zero, saturating to int64, NaN -> INT64_MIN (the kernel's conversion)."""
    v = np.asarray(v, dtype=np.float64)
    out = np.full(v.shape, np.iinfo(np.int64).min, dtype=np.int64)
    ok = ~np.isnan(v)
    big = ok & (v >= 2.0**63)
    mid = ok & ~big & (v > -(2.0**63))
    out[big] = np.iinfo(np.int64).max
    out[mid] = np.trunc(v[mid]).astype(np.int64)
    return out


def grid_cluster(pos, size, start=None, end=None):
    """[N] int64 voxel index of each point, in pos's dtype (float32 or float64)."""
    pos = np.asarray(pos)
    pos = pos.reshape(pos.shape[0], -1)
    dt = pos.dtype.type
    size = np.asarray(size, dtype=dt).reshape(-1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        start = (np.min(pos, axis=0) if pos.shape[0] else np.zeros(pos.shape[1], dt)) if start is None \
            else np.asarray(start, dtype=dt).reshape(-1)
        end = (np.max(pos, axis=0) if pos.shape[0] else np.zeros(pos.shape[1], dt)) if end is None \
            else np.asarray(end, dtype=dt).reshape(-1)
        c = np.zeros(pos.shape[0], dtype=np.int64)
        stride = np.int64(1)
        for k in range(pos.shape[1]):
            t = (pos[:, k] - start[k]).astype(dt)
            t = (t / size[k]).astype(dt)
            c = c + _trunc(t) * stride
            stride = stride * (_trunc(dt(dt(end[k] - start[k]) / size[k])) + 1)[()]
    return c


def torch_ops():
    """CPU implementations of torch.ops.pyg.{graclus_cluster, grid_cluster} on this oracle, for the golden generator.
    graclus draws its seed from torch's CPU generator exactly as pytorch_geometric_b200.ops.graclus does."""
    def graclus_cluster(rowptr, col, weight=None):
        seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
        w = None if weight is None else weight.detach().double().numpy()
        return torch.from_numpy(graclus(rowptr.numpy(), col.numpy(), w, seed)[0])

    def grid(pos, size, start=None, end=None):
        p = pos.detach().numpy()
        cast = (lambda t: None if t is None else t.detach().to(pos.dtype).numpy())
        return torch.from_numpy(grid_cluster(p, cast(size), cast(start), cast(end)))

    return {"graclus_cluster": graclus_cluster, "grid_cluster": grid}
