"""numpy restatement of the random-walk contract of csrc/random_walk.cu: the splitmix64 stream of each walk, the uniform
step, the dead-end rule, node2vec's rejection trials, the exact fallback after max_trials rejections and both neighbour
tests (binary search on non-decreasing rows, linear scan otherwise).

`random_walk` is vectorised over the walks, with the neighbour test as a lookup of row * N + col keys (which gives
the same answer as either search); `random_walk_scalar` is the rule book one walk at a time with the two searches
themselves, for small cases.  Both return int64 [S, L + 1] with -1 where a walk has no node.
"""
import numpy as np

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
MAX_TRIALS = 1024                 # ops.RANDOM_WALK_MAX_TRIALS
_M1, _M2 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def splitmix64(seed, key):
    """mix(seed + key * 0x9E3779B97F4A7C15 mod 2^64), elementwise on uint64."""
    with np.errstate(over="ignore"):
        z = np.asarray(seed, np.uint64) + np.asarray(key, np.uint64) * GOLDEN
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
    return z ^ (z >> np.uint64(31))


def umulhi(r, d):
    """High 64 bits of the 128-bit product r * d (d < 2^32), elementwise."""
    r, d = np.asarray(r, np.uint64), np.asarray(d, np.uint64)
    lo, hi = r & np.uint64(0xFFFFFFFF), r >> np.uint64(32)
    with np.errstate(over="ignore"):
        return (hi * d + ((lo * d) >> np.uint64(32))) >> np.uint64(32)


def uniform(r):
    return (np.asarray(r, np.uint64) >> np.uint64(11)).astype(np.float64) * 2.0**-53


def probabilities(p, q):
    """(1/p, 1/q, a_t, a_1, a_q) in fp64, formed as the host code forms them."""
    w_t, w_q = 1.0 / p, 1.0 / q
    m = max(max(w_t, 1.0), w_q)
    return w_t, w_q, w_t / m, 1.0 / m, w_q / m


def rows_sorted(rowptr, col):
    rowptr, col = np.asarray(rowptr, np.int64), np.asarray(col, np.int64)
    if col.size < 2:
        return True
    dec = col[1:] < col[:-1]
    starts = np.zeros(col.size, bool)
    inner = rowptr[1:-1]
    starts[inner[(inner > 0) & (inner < col.size)]] = True    # a decrease across a row boundary does not count
    return not (dec & ~starts[1:]).any()


def _row_ok(rowptr, E, v):
    s, e = rowptr[v], rowptr[v + 1]
    return (s >= 0) & (s <= e) & (e <= E), s, e


# ---------------------------------------------------------------------------------------------- scalar rule book
def _has_edge(col, s, e, x, sorted_rows):
    if sorted_rows:
        lo, hi = s, e
        while lo < hi:
            mid = lo + ((hi - lo) >> 1)
            if col[mid] < x:
                lo = mid + 1
            else:
                hi = mid
        return lo < e and col[lo] == x
    return any(col[i] == x for i in range(s, e))


def random_walk_scalar(rowptr, col, start, walk_length, p=1.0, q=1.0, seed=0, max_trials=MAX_TRIALS):
    rowptr, col = [int(v) for v in np.asarray(rowptr, np.int64)], [int(v) for v in np.asarray(col, np.int64)]
    n, E = len(rowptr) - 1, len(col)
    biased = p != 1.0 or q != 1.0
    w_t, w_q, a_t, a_1, a_q = probabilities(p, q)
    srt = rows_sorted(rowptr, col)
    out = np.full((len(start), walk_length + 1), -1, np.int64)
    for w, v in enumerate(np.asarray(start, np.int64).tolist()):
        key = int(splitmix64(np.uint64(seed & (2**64 - 1)), np.uint64(w)))
        draws = [0]

        def draw():
            draws[0] += 1
            return int(splitmix64(np.uint64(key), np.uint64(draws[0])))

        if not 0 <= v < n:
            continue
        out[w, 0] = v
        t, ts, te = -1, 0, 0

        def cls(x):
            return 0 if x == t else (1 if _has_edge(col, ts, te, x, srt) else 2)

        for k in range(1, walk_length + 1):
            s, e = rowptr[v], rowptr[v + 1]
            if not (0 <= s <= e <= E):
                break
            if s == e:
                x = v
            elif not biased or k == 1:
                x = col[s + int(umulhi(draw(), e - s))]
            else:
                done = stray = False
                for _ in range(max_trials):
                    x = col[s + int(umulhi(draw(), e - s))]
                    if not 0 <= x < n:
                        stray = True
                        break
                    u = float(uniform(draw()))
                    done = u < (a_t, a_1, a_q)[cls(x)]
                    if done:
                        break
                if not done and not stray:
                    u = float(uniform(draw()))
                    ws = [(w_t, 1.0, w_q)[cls(col[i])] for i in range(s, e)]
                    total = 0.0
                    for wi in ws:
                        total += wi
                    target, run, pick = u * total, 0.0, e - 1
                    for i, wi in zip(range(s, e), ws):
                        run += wi
                        if run > target:
                            pick = i
                            break
                    x = col[pick]
            if not 0 <= x < n:
                break
            t, ts, te, v = v, s, e, x
            out[w, k] = v
    return out


# ---------------------------------------------------------------------------------------------- vectorised
def random_walk(rowptr, col, start, walk_length, p=1.0, q=1.0, seed=0, max_trials=MAX_TRIALS):
    rowptr, col = np.asarray(rowptr, np.int64), np.asarray(col, np.int64)
    start = np.asarray(start, np.int64)
    n, E, S = rowptr.size - 1, col.size, start.size
    biased = p != 1.0 or q != 1.0
    w_t, w_q, a_t, a_1, a_q = probabilities(p, q)
    acc = np.array([a_t, a_1, a_q])
    wts = np.array([w_t, 1.0, w_q])
    out = np.full((S, walk_length + 1), -1, np.int64)
    key = splitmix64(np.uint64(int(seed) & (2**64 - 1)), np.arange(S, dtype=np.uint64))
    draws = np.zeros(S, np.uint64)
    alive = (start >= 0) & (start < n)
    v = np.where(alive, start, 0)
    t, ts, te = np.full(S, -1, np.int64), np.zeros(S, np.int64), np.zeros(S, np.int64)
    out[alive, 0] = v[alive]
    # the neighbour test: membership of the pair (t, x) among the CSR's (row, col) pairs
    src = np.repeat(np.arange(n, dtype=np.int64), np.clip(np.diff(rowptr), 0, None)) if biased else None
    keys, lo, span = None, 0, 1
    if biased and rowptr[0] == 0 and rowptr[-1] == E and (np.diff(rowptr) >= 0).all():
        if E:      # the values of col as they are, out-of-range ones included, as the searches compare them
            lo, span = min(int(col.min()), 0), int(col.max()) - min(int(col.min()), 0) + 1
        keys = np.unique(src * span + (col - lo))

    def cls(tt, x):
        nb = np.zeros(x.shape, bool)
        if keys is not None and keys.size:
            inside = (x >= lo) & (x < lo + span)
            k = tt * span + np.where(inside, x - lo, 0)
            nb = (keys[np.minimum(np.searchsorted(keys, k), keys.size - 1)] == k) & inside
        return np.where(x == tt, 0, np.where(nb, 1, 2))

    def draw(idx):
        draws[idx] += np.uint64(1)
        return splitmix64(key[idx], draws[idx])

    for k in range(1, walk_length + 1):
        idx = np.nonzero(alive)[0]
        ok, s, e = _row_ok(rowptr, E, v[idx])
        alive[idx[~ok]] = False
        idx, s, e = idx[ok], s[ok], e[ok]
        x = np.full(idx.size, -1, np.int64)
        dead = s == e
        x[dead] = v[idx[dead]]
        mv = ~dead
        if not biased or k == 1:
            ii = idx[mv]
            x[mv] = col[s[mv] + umulhi(draw(ii), (e - s)[mv]).astype(np.int64)]
        else:
            if keys is None and mv.any():
                raise NotImplementedError("the vectorised oracle needs a well-formed CSR for biased walks")
            pending = np.nonzero(mv)[0]            # positions into idx still drawing
            stray = np.zeros(idx.size, bool)
            for _ in range(max_trials):
                if pending.size == 0:
                    break
                ii = idx[pending]
                cand = col[s[pending] + umulhi(draw(ii), (e - s)[pending]).astype(np.int64)]
                bad = (cand < 0) | (cand >= n)
                x[pending] = cand
                stray[pending[bad]] = True
                pending, cand, ii = pending[~bad], cand[~bad], ii[~bad]
                u = uniform(draw(ii))
                take = u < acc[cls(t[ii], cand)]
                pending = pending[~take]
            for j in pending.tolist():                 # the exact draw
                i = idx[j]
                u = float(uniform(draw(np.array([i]))[0]))
                row = col[s[j]:e[j]]
                wv = wts[cls(np.full(row.size, t[i]), row)]
                cs = np.cumsum(wv)
                over = np.nonzero(cs > u * cs[-1])[0]
                x[j] = row[over[0]] if over.size else row[-1]
        bad = (x < 0) | (x >= n)
        alive[idx[bad]] = False
        good = ~bad
        gi = idx[good]
        t[gi], ts[gi], te[gi], v[gi] = v[gi], s[good], e[good], x[good]
        out[gi, k] = x[good]
    return out


def torch_op(max_trials=MAX_TRIALS):
    """A CPU stand-in of torch.ops.pyg.random_walk on this oracle: the seed drawn from torch's CPU generator as
    ops.random_walk draws it."""
    import torch

    def op(rowptr, col, start, walk_length, p=1.0, q=1.0):
        seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
        w = random_walk(rowptr.numpy(), col.numpy(), start.numpy(), walk_length, p, q, seed, max_trials)
        return torch.from_numpy(w).to(rowptr.dtype)
    return op
