"""float32 numpy restatement of the point-cloud ops of csrc/point.cu (pyg_lib.ops knn / radius / fps / nearest), one
operation at a time, so that it reproduces the kernels' distances bit for bit:

  squared distance  d = sum_f (x_f - y_f)^2, accumulated in feature order, each subtraction, product and sum rounded
  cosine distance   1 - dot / (sqrt(|x|^2) sqrt(|y|^2)), each of the three sums as above
  selection         strict <, so NaN and infinite distances are never selected; k-NN ties by ascending x index

Examples are ptr ranges; a None ptr is one example of every point, and examples missing at the end of the shorter ptr
are empty.  The order, the tie rule, the strict < of radius and the ceil of fps are restated from torch-cluster's CUDA
kernels, which pyg-lib's were ported from; they have not been checked against pyg-lib itself.

`torch_ops()` wraps the functions with torch.ops.pyg's argument lists for CPU tensors (golden-data generation).
"""
import math

import numpy as np

F32 = np.float32


def _ranges(ptr, n):
    if ptr is None:
        return [(0, n)]
    p = [int(v) for v in np.asarray(ptr)]
    return [(p[b], max(p[b], p[b + 1])) for b in range(len(p) - 1)]


def _pair_ranges(ptr_x, ptr_y, n_x, n_y):
    """[(x range, y range)] per example, empty where one ptr has no such example."""
    rx, ry = _ranges(ptr_x, n_x), _ranges(ptr_y, n_y)
    nb = max(len(rx), len(ry))
    rx += [(0, 0)] * (nb - len(rx))
    ry += [(0, 0)] * (nb - len(ry))
    return list(zip(rx, ry))


def distances(x, y, cosine=False):
    """[len(y), len(x)] float32 distances, in the kernels' operation order."""
    x = np.asarray(x, dtype=F32).reshape(len(x), -1)
    y = np.asarray(y, dtype=F32).reshape(len(y), -1)
    F = x.shape[1]
    with np.errstate(all="ignore"):
        if not cosine:
            d = np.zeros((len(y), len(x)), dtype=F32)
            for f in range(F):
                t = (x[None, :, f] - y[:, None, f]).astype(F32)
                d = (d + (t * t).astype(F32)).astype(F32)
            return d
        dot = np.zeros((len(y), len(x)), dtype=F32)
        nx = np.zeros(len(x), dtype=F32)
        ny = np.zeros(len(y), dtype=F32)
        for f in range(F):
            dot = (dot + (x[None, :, f] * y[:, None, f]).astype(F32)).astype(F32)
            nx = (nx + (x[:, f] * x[:, f]).astype(F32)).astype(F32)
            ny = (ny + (y[:, f] * y[:, f]).astype(F32)).astype(F32)
        den = (np.sqrt(nx)[None, :] * np.sqrt(ny)[:, None]).astype(F32)
        return (F32(1) - (dot / den).astype(F32)).astype(F32)


def knn(x, y, k, ptr_x=None, ptr_y=None, cosine=False):
    """[2, nnz] int64 (y index, x index): the k nearest x points of each y point's example."""
    rows, cols = [], []
    for (xs, xe), (ys, ye) in _pair_ranges(ptr_x, ptr_y, len(x), len(y)):
        if ye <= ys or xe <= xs:
            continue
        d = distances(np.asarray(x)[xs:xe], np.asarray(y)[ys:ye], cosine)
        for qi in range(ye - ys):
            row = d[qi]
            order = np.argsort(row, kind="stable")
            order = [j for j in order if np.isfinite(row[j])][:k]
            rows += [ys + qi] * len(order)
            cols += [xs + j for j in order]
    return np.array([rows, cols], dtype=np.int64).reshape(2, -1)


def radius(x, y, r, ptr_x=None, ptr_y=None, max_num_neighbors=32, ignore_same_index=False):
    """[2, nnz] int64: the first max_num_neighbors x points (ascending index) of each y point's example with d < r^2."""
    r2 = F32(float(r) * float(r))
    rows, cols = [], []
    for (xs, xe), (ys, ye) in _pair_ranges(ptr_x, ptr_y, len(x), len(y)):
        if ye <= ys or xe <= xs:
            continue
        d = distances(np.asarray(x)[xs:xe], np.asarray(y)[ys:ye])
        for qi in range(ye - ys):
            sel = [xs + j for j in range(xe - xs) if d[qi, j] < r2 and not (ignore_same_index and xs + j == ys + qi)]
            sel = sel[:max(int(max_num_neighbors), 0)]
            rows += [ys + qi] * len(sel)
            cols += sel
    return np.array([rows, cols], dtype=np.int64).reshape(2, -1)


def fps_counts(ptr, n, ratio):
    return [int(math.ceil(float(e - s) * float(ratio))) for s, e in _ranges(ptr, n)]


def fps(src, ptr=None, ratio=0.5, starts=None):
    """Global indices of the farthest-point samples, examples concatenated; starts[b] (local) or each example's first
    point.  Each step takes the argmax of the running min squared distance, ties to the lowest index."""
    src = np.asarray(src, dtype=F32).reshape(len(src), -1)
    out = []
    for b, ((s, e), m) in enumerate(zip(_ranges(ptr, len(src)), fps_counts(ptr, len(src), ratio))):
        if m == 0:
            continue
        pts = src[s:e]
        mind = np.full(e - s, np.inf, dtype=F32)
        last = 0 if starts is None else int(starts[b])
        out.append(s + last)
        for _ in range(m - 1):
            d = distances(pts, pts[last:last + 1])[0]
            upd = d < mind
            mind = np.where(upd, d, mind).astype(F32)
            last = int(np.argmax(mind))
            out.append(s + last)
    return np.array(out, dtype=np.int64)


def nearest(x, y, ptr_x=None, ptr_y=None):
    """[len(x)] int64: for each x point the nearest y point of its example; ValueError when there is none."""
    e = knn(y, x, 1, ptr_y, ptr_x)
    if e.shape[1] != len(x):
        raise ValueError("nearest: some x point has no y point in its example")
    out = np.empty(len(x), dtype=np.int64)
    out[e[0]] = e[1]
    return out


def torch_ops():
    """{name: CPU implementation with torch.ops.pyg's argument list}."""
    import torch

    def n(t):
        return None if t is None else t.detach().cpu().numpy()

    def t64(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64))

    return {
        "knn": lambda x, y, ptr_x, ptr_y, k, cosine, num_workers: t64(knn(n(x.float()), n(y.float()), k, n(ptr_x),
                                                                          n(ptr_y), cosine)),
        "radius": lambda x, y, ptr_x, ptr_y, r, max_num_neighbors, num_workers, ignore_same_index: t64(
            radius(n(x.float()), n(y.float()), r, n(ptr_x), n(ptr_y), max_num_neighbors, ignore_same_index)),
        "fps": lambda src, ptr, ratio, random_start: t64(fps(n(src.float()), n(ptr), ratio)),
        "nearest": lambda x, y, ptr_x, ptr_y: t64(nearest(n(x.float()), n(y.float()), n(ptr_x), n(ptr_y))),
    }
