"""A numpy restatement of the quantile-aggregation contract (csrc/quantile.cu's header, DESIGN.md section 4.2): ranks
from the reference's fp32 arithmetic (quantile.py:88), exact integer offsets past 2^24 and ranks clamped into the
group, order-preserving keys with
ties in slot order, ATen's per-op roundings, and the backward's per-element sums.  bf16 roundings go through torch
CPU bf16 tensors.  Values travel as float32 arrays (bf16 values are exact in them)."""
import numpy as np
import torch

INTERP = ("linear", "lower", "higher", "nearest", "midpoint")


def rnd(v, bf16: bool):
    """v rounded to the storage dtype (a no-op for fp32)."""
    v = np.asarray(v, dtype=np.float32)
    if not bf16:
        return v
    return torch.from_numpy(np.ascontiguousarray(v)).to(torch.bfloat16).float().numpy()


def keys(v, bf16: bool):
    """Order-preserving unsigned keys: -0.0 == +0.0, every NaN above +inf."""
    v = np.ascontiguousarray(v, dtype=np.float32)
    kb = 16 if bf16 else 32
    u = (v.view(np.uint32) >> np.uint32(32 - kb)).astype(np.uint64)
    sign = np.uint64(1 << (kb - 1))
    allb = np.uint64((1 << kb) - 1)
    u = np.where(u == sign, np.uint64(0), u)
    k = np.where(u & sign, ~u & allb, u | sign)
    return np.where(np.isnan(v), allb, k)


def ranks(q: float, ptr: int, count: int, interp: str):
    """(floor or single rank, ceil or single rank, frac) of one q in a group of `count` at offset `ptr`."""
    h = np.float32(q) * np.float32(count - 1)
    if ptr + count - 1 < (1 << 24):
        P = np.float32(h + np.float32(ptr))
        frac = np.float32(P - np.floor(P))
        fl, ce, ne = int(np.floor(P)) - ptr, int(np.ceil(P)) - ptr, int(np.rint(P)) - ptr
    else:
        hf = np.floor(h)
        frac = np.float32(h - hf)
        fl = int(hf)
        ce = fl + 1 if frac > 0 else fl
        ne = fl if frac < 0.5 else (fl + 1 if frac > 0.5 else fl + ((fl + ptr) & 1))
    lo = {"higher": ce, "nearest": ne}.get(interp, fl)
    hi = {"lower": fl, "nearest": ne}.get(interp, ce)
    # clamped into the group: past 2^24 fl32(count - 1) may round up (count = 2^24 + 4, q = 1 gives h = count)
    return min(max(lo, 0), count - 1), min(max(hi, 0), count - 1), np.float32(frac)


def out_is_f32(bf16: bool, interp: str) -> bool:
    return bf16 and interp == "linear"


def forward(rowptr, V, q, interp: str, fill: float, bf16: bool, offsets=None):
    """V: [E, F] message values in CSR slot order; offsets: each row's CSR offset in the whole graph when the rows
    are a sample of it (default: rowptr).  Returns (out [N, Q F] float32, picks) where picks[(j, k)] is an
    [N, F] array of the picked slot (-1: empty row) for floor (j = 0) / ceil (j = 1) picks of q[k]."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    V = np.asarray(V, dtype=np.float32)
    N, F, Q = rowptr.size - 1, V.shape[1], len(q)
    R = 2 if interp in ("linear", "midpoint") else 1
    out = np.empty((N, Q * F), dtype=np.float32)
    picks = {(j, k): np.full((N, F), -1, dtype=np.int64) for j in range(R) for k in range(Q)}
    fill_v = np.float32(fill) if (out_is_f32(bf16, interp) or not bf16) else rnd(np.float32(fill), True)
    cols = np.arange(F)
    for i in range(N):
        p0, c = int(rowptr[i]), int(rowptr[i + 1] - rowptr[i])
        if c == 0:
            out[i] = fill_v
            continue
        vals = V[p0:p0 + c]
        order = np.argsort(keys(vals, bf16), axis=0, kind="stable")         # ties in slot order
        for k, qv in enumerate(q):
            lo, hi, frac = ranks(float(qv), p0 if offsets is None else int(offsets[i]), c, interp)
            sl, sh = order[lo], order[hi]
            l, r = vals[sl, cols], vals[sh, cols]
            if interp == "linear":
                with np.errstate(invalid="ignore"):                       # inf - inf and NaN, as ATen gives them
                    v = (l + rnd(r - l, bf16) * frac).astype(np.float32)
            elif interp == "midpoint":
                v = rnd(rnd(np.float32(0.5) * l, bf16) + rnd(np.float32(0.5) * r, bf16), bf16)
            else:
                v = l
            out[i, k * F:(k + 1) * F] = v
            picks[(0, k)][i] = p0 + sl
            if R == 2:
                picks[(1, k)][i] = p0 + sh
    return out, picks


def backward(rowptr, picks, q, interp: str, g, n_edges: int, bf16: bool):
    """The gradient of every message [E, F] in CSR slot order, from g [N, Q F] (float32 values of the output dtype)."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    g = np.asarray(g, dtype=np.float32)
    N = rowptr.size - 1
    Q = len(q)
    F = g.shape[1] // Q
    R = 2 if interp in ("linear", "midpoint") else 1
    cols = np.arange(F)
    s = [np.zeros((n_edges, F), dtype=np.float32) for _ in range(R)]
    counts = np.diff(rowptr)
    for j in range(R):
        for k in range(Q):
            slots = picks[(j, k)]
            for i in np.nonzero(counts > 0)[0]:
                gi = g[i, k * F:(k + 1) * F]
                if interp == "midpoint":
                    c = rnd(np.float32(0.5) * gi, bf16)
                elif interp == "linear":
                    frac = ranks(float(q[k]), int(rowptr[i]), int(counts[i]), interp)[2]
                    gf = rnd(gi * frac, bf16)
                    c = gf if j == 1 else rnd(rnd(gi, bf16) - gf, bf16)
                else:
                    c = gi
                sl = slots[i]
                s[j][sl, cols] = rnd(s[j][sl, cols] + c, bf16)
    return rnd(s[0] + s[1], bf16) if R == 2 else s[0]


def csr_of_index(index, n_rows: int):
    """(rowptr, perm): a stable CSR of an unsorted destination index; perm[slot] = the message's position."""
    index = np.asarray(index, dtype=np.int64)
    perm = np.argsort(index, kind="stable")
    rowptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(index, minlength=n_rows), out=rowptr[1:])
    return rowptr, perm


def aggregate(x2, index, n_rows: int, q, interp: str, fill: float, bf16: bool, g=None):
    """The contract over a [E, W] message matrix grouped by `index` (caller order): (out [N, Q W], grad [E, W] in the
    caller's order or None)."""
    rowptr, perm = csr_of_index(index, n_rows)
    out, picks = forward(rowptr, np.asarray(x2)[perm], q, interp, fill, bf16)
    if g is None:
        return out, None
    gs = backward(rowptr, picks, q, interp, g, len(perm), bf16)
    grad = np.empty_like(gs)
    grad[perm] = gs
    return out, grad


def sum_out_edges(grad_e, src, n_src: int, bf16: bool, chunk=None):
    """grad_x[j] = the fp32 sum of grad_e over j's out-edges in caller order, rounded once.  With `chunk` (the
    transposed CSR's long-row plan), a source of more than `chunk` out-edges is summed per chunk of `chunk` out-edges
    and the chunk sums are then folded in chunk order, as the transposed sweep splits hub sources."""
    src = np.asarray(src, dtype=np.int64)
    grad_e = np.asarray(grad_e, dtype=np.float32)
    order = np.argsort(src, kind="stable")
    counts = np.bincount(src, minlength=n_src)
    acc = np.zeros((n_src, grad_e.shape[1]), dtype=np.float32)
    start = 0
    for j in range(n_src):
        rows = grad_e[order[start:start + counts[j]]]
        start += counts[j]
        step = chunk if chunk is not None and len(rows) > chunk else max(len(rows), 1)
        for k in range(0, len(rows), step):
            part = np.zeros(grad_e.shape[1], dtype=np.float32)
            for r in rows[k:k + step]:
                part = part + r
            acc[j] = acc[j] + part
    return rnd(acc, bf16)


def tie_class_sums(x2, grad, index, bf16: bool):
    """Per (group, column, tied value) class: (class ids sorted, fp64 sum of grad, fp64 sum of |grad|)."""
    x2 = np.asarray(x2, dtype=np.float32)
    E, W = x2.shape
    k = keys(x2, bf16)
    grp = np.repeat(np.asarray(index, dtype=np.int64), W).reshape(E, W)
    col = np.broadcast_to(np.arange(W), (E, W))
    ids = np.stack([grp.ravel(), col.ravel(), k.ravel().astype(np.int64)], axis=1)
    uniq, inv = np.unique(ids, axis=0, return_inverse=True)
    inv = inv.ravel()
    gs = np.asarray(grad, dtype=np.float64).ravel()
    return uniq, np.bincount(inv, weights=gs, minlength=len(uniq)), np.bincount(inv, weights=np.abs(gs),
                                                                                 minlength=len(uniq))


# ---------------------------------------------------------------- the reference's layout and the golden cases
def fold(x, d: int):
    """x with dimension d first and every other one folded into the width: [E, W]."""
    xm = np.moveaxis(np.asarray(x), d, 0)
    return xm.reshape(xm.shape[0], -1)


def unfold(x2, shape, d: int):
    rest = tuple(shape[:d]) + tuple(shape[d + 1:])
    return np.moveaxis(np.asarray(x2).reshape(x2.shape[0], *rest), 0, d)


def layout(out, n_q: int, shape, d: int):
    """A [N, Q W] result in the reference's layout (quantile.py:125-129) for x of `shape` aggregated along d."""
    rest = list(shape[:d]) + list(shape[d + 1:])
    n = out.shape[0]
    o = np.moveaxis(np.asarray(out).reshape(n, n_q, *rest), (0, 1), (d, d + 1))
    if n_q == 1:
        return o.reshape(*shape[:d], n, *shape[d + 1:])
    if d + 1 < len(shape):
        return o.reshape(*shape[:d], n, n_q * shape[d + 1], *shape[d + 2:])
    return o.reshape(*shape[:d], n, n_q)


def unlayout(y, n_q: int, shape, d: int, n: int, width: int):
    pos = layout(np.arange(n * n_q * width).reshape(n, n_q * width), n_q, shape, d)
    flat = np.empty(n * n_q * width, dtype=np.asarray(y).dtype)
    flat[pos.ravel()] = np.asarray(y).ravel()
    return flat.reshape(n, n_q * width)


def golden_cases(z):
    """{case name: {field: array}} of quantile.npz."""
    out = {}
    for k, v in z.items():
        name, field = k.split("/", 1)
        out.setdefault(name, {})[field] = v
    return out


def case_args(c):
    """(x, d, index, N, q fp32, interpolation, fill, bf16, g in the kernel's [N, Q W] layout)."""
    x = c["x"]
    d = int(c["dim"]) + x.ndim if int(c["dim"]) < 0 else int(c["dim"])
    idx = c["index"].astype(np.int64)
    n = int(c["dim_size"]) if int(c["dim_size"]) >= 0 else int(idx.max()) + 1
    q = c["q"].astype(np.float32)
    interp, bf16 = str(c["interpolation"]), bool(c["bf16"])
    g = c["w"] if str(c["out_dtype"]) == "torch.float32" else rnd(c["w"], bf16)
    width = fold(x, d).shape[1]
    return x, d, idx, n, q, interp, float(c["fill"]), bf16, unlayout(g, len(q), x.shape, d, n, width)


def check_golden(c, out, grad):
    """out (reference layout) bit for bit with +-0 equal and NaN positions equal; grad by tie-class sums."""
    x, d, idx, _, _, _, _, bf16, _ = case_args(c)
    exp = c["out"]
    out = np.asarray(out, dtype=np.float32)
    assert out.shape == exp.shape, (out.shape, exp.shape)
    nan = np.isnan(exp)
    assert (np.isnan(out) == nan).all(), "NaN positions differ"
    bad = out[~nan] != exp[~nan]
    assert not bad.any(), f"{bad.sum()} values differ"
    tol = 1.6e-2 if bf16 else 1e-6
    u1, s1, a1 = tie_class_sums(fold(x, d), fold(c["grad"], d), idx, bf16)
    u2, s2, _ = tie_class_sums(fold(x, d), fold(grad, d), idx, bf16)
    assert (u1 == u2).all()
    err = np.abs(s1 - s2)
    assert (err <= tol * np.maximum(1.0, a1)).all(), f"grad class sums differ by up to {err.max():.3e}"
