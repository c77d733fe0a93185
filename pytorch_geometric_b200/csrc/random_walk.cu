// random_walk.cu -- uniform and node2vec random walks over a CSR graph (pyg_lib.ops.random_walk, reached as
// torch.ops.pyg.random_walk in nn/models/node2vec.py:64,103, utils/dropout.py:285 and
// transforms/rooted_subgraph.py:171).
//
// The output is a pure function of (graph, start, L, p, q, max_trials, seed), independent of the launch
// configuration.  Walk w (row w of out, out[w, 0] = start[w]) takes L steps under these rules:
//   RNG.          Draw c = 0, 1, 2, ... of walk w is r = splitmix64(k_w, c + 1) with k_w = splitmix64(seed, w), where
//                 splitmix64(s, k) = mix(s + k * 0x9E3779B97F4A7C15 mod 2^64) and mix is splitmix64's finaliser
//                 (z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9; z = (z ^ z >> 27) * 0x94D049BB133111EB; z ^ z >> 31),
//                 the generator of graclus's colours (common.cuh): a splitmix64 stream seeded by k_w.  A uniform
//                 real is u = (r >> 11) * 2^-53.
//   Uniform step  (the first step of every walk, and every step when p = q = 1): from v with row [s, e),
//                 x = col[s + umulhi64(r, e - s)] for one draw r.
//   Dead end.     deg(v) = 0: the walk stays at v and consumes no draw; the previous node becomes v.
//   node2vec step (p != 1 or q != 1, from v with previous node t): rejection sampling as in torch-cluster's GPU kernel.
//                 With max_prob = max(1/p, 1, 1/q), the acceptance probabilities a_t = (1/p) / max_prob,
//                 a_1 = 1 / max_prob and a_q = (1/q) / max_prob are formed once on the host in fp64.  A trial takes
//                 two draws: a candidate x picked as in the uniform step, then u; x is accepted when u < a_t (x = t),
//                 u < a_1 (x is a neighbour of t) or u < a_q (otherwise).  After max_trials rejected trials, one more
//                 draw gives u and the step is drawn exactly from the same distribution: v's row is scanned in order,
//                 summing each entry's weight (1/p, 1 or 1/q, by the same classes) in fp64, and the first entry whose
//                 running sum exceeds u * W (W the row's total) is taken, or the row's last entry when rounding leaves
//                 none.  The cap bounds every step's work whatever p and q are, and leaves the distribution unchanged.
//   Membership.   "x is a neighbour of t" is a binary search of t's row when every row of col is non-decreasing, a
//                 linear scan otherwise.  The choice is a one-element device flag computed by walk_rows_unsorted_kernel
//                 (O(E), only for biased walks, and only when the caller asks for it: the Python side caches it per
//                 graph); the walk kernel reads it, so nothing is read back to the host.
//   Guards.       A start outside [0, N) gives a row of -1.  A picked node outside [0, N), or a row whose bounds are
//                 not 0 <= rowptr[v] <= rowptr[v + 1] <= E, ends the walk: that step and the rest of the row are -1.
//                 Nothing outside rowptr [N + 1] and col [E] is ever read.
// Layout: one thread per walk, kWalkThreads walks per CTA.  Each pass stages kWalkChunk steps of every walk of the CTA
// in shared memory as int32 (N < 2^31 - 1, the graclus limit) and the CTA then writes them out as contiguous row
// segments, so consecutive threads store consecutive addresses.
//
// -Xptxas -v for sm_90a (CUDA 12.9): every instantiation has no stack frame and no spills.
#include <cmath>

#include "common.cuh"

namespace b200mp {

constexpr int kWalkThreads = 128;
constexpr int kWalkChunk = 32;               // steps staged per pass
constexpr int kWalkPad = kWalkChunk + 1;     // row stride of the staging tile: no bank conflicts
constexpr int kWalkCheckThreads = 256;

struct WalkArgs {
    const void* rowptr;
    const void* col;
    const void* start;
    void* out;
    const int32_t* rows_unsorted;   // [1]: some row of col decreases (biased walks only)
    int64_t n, n_edges, n_walks, walk_length;
    unsigned long long seed;
    double acc_t, acc_1, acc_q, acc_lo;   // acceptance probabilities, acc_lo their minimum
    double w_t, w_q;                      // fallback weights 1/p and 1/q
    int max_trials;
};

__device__ __forceinline__ double walk_uniform(unsigned long long r) {
    return static_cast<double>(r >> 11) * 0x1.0p-53;
}

// Row bounds of v; false when they are not 0 <= s <= e <= E.
template <typename I>
__device__ __forceinline__ bool walk_row(const I* rowptr, int64_t n_edges, int64_t v, int64_t& s, int64_t& e) {
    s = static_cast<int64_t>(__ldg(rowptr + v));
    e = static_cast<int64_t>(__ldg(rowptr + v + 1));
    return 0 <= s && s <= e && e <= n_edges;
}

template <typename I>
__device__ __forceinline__ bool walk_has_edge(const I* col, int64_t s, int64_t e, int64_t x, bool sorted) {
    if (sorted) {
        int64_t lo = s, hi = e;
        while (lo < hi) {
            const int64_t mid = lo + ((hi - lo) >> 1);
            if (static_cast<int64_t>(__ldg(col + mid)) < x) lo = mid + 1;
            else hi = mid;
        }
        return lo < e && static_cast<int64_t>(__ldg(col + lo)) == x;
    }
    for (int64_t i = s; i < e; ++i)
        if (static_cast<int64_t>(__ldg(col + i)) == x) return true;
    return false;
}

// Weight class of candidate x given the previous node t and its row [ts, te): 0 = t, 1 = neighbour of t, 2 = other.
template <typename I>
__device__ __forceinline__ int walk_class(const I* col, int64_t t, int64_t ts, int64_t te, int64_t x, bool sorted) {
    if (x == t) return 0;
    return walk_has_edge(col, ts, te, x, sorted) ? 1 : 2;
}

template <typename I, bool BIASED>
__global__ void __launch_bounds__(kWalkThreads) walk_kernel(WalkArgs a) {
    __shared__ int32_t tile[kWalkThreads * kWalkPad];
    const I* rowptr = static_cast<const I*>(a.rowptr);
    const I* col = static_cast<const I*>(a.col);
    I* out = static_cast<I*>(a.out);
    const int64_t w0 = static_cast<int64_t>(blockIdx.x) * kWalkThreads;
    const int64_t w = w0 + threadIdx.x;
    const int64_t n_rows = min(static_cast<int64_t>(kWalkThreads), a.n_walks - w0);
    const int64_t width = a.walk_length + 1;
    bool sorted = false;
    if constexpr (BIASED) sorted = __ldg(a.rows_unsorted) == 0;

    int64_t v = -1, t = -1, ts = 0, te = 0;   // current node, previous node and the previous node's row
    bool alive = false;
    unsigned long long key = 0ull, draws = 0ull;
    if (w < a.n_walks) {
        v = static_cast<int64_t>(__ldg(static_cast<const I*>(a.start) + w));
        alive = 0 <= v && v < a.n;
        key = splitmix64(a.seed, static_cast<unsigned long long>(w));
    }

    for (int64_t c0 = 0; c0 < width; c0 += kWalkChunk) {
        const int cw = static_cast<int>(min(static_cast<int64_t>(kWalkChunk), width - c0));
        if (w < a.n_walks) {
            for (int j = 0; j < cw; ++j) {
                const int64_t k = c0 + j;
                if (k > 0 && alive) {
                    int64_t s, e;
                    int64_t x = -1;
                    if (!walk_row(rowptr, a.n_edges, v, s, e)) {
                        alive = false;
                    } else if (s == e) {
                        x = v;   // dead end: stay, no draw
                    } else if (!BIASED || k == 1) {
                        const unsigned long long r = splitmix64(key, ++draws);
                        x = static_cast<int64_t>(__ldg(col + s + static_cast<int64_t>(
                                                                  __umul64hi(r, static_cast<unsigned long long>(e - s)))));
                    } else {
                        const unsigned long long deg = static_cast<unsigned long long>(e - s);
                        bool done = false, stray = false;
                        for (int trial = 0; trial < a.max_trials && !done && !stray; ++trial) {
                            x = static_cast<int64_t>(__ldg(col + s + static_cast<int64_t>(
                                                                      __umul64hi(splitmix64(key, ++draws), deg))));
                            stray = x < 0 || x >= a.n;   // ends the walk below
                            if (stray) break;
                            const double u = walk_uniform(splitmix64(key, ++draws));
                            if (u < a.acc_lo) {
                                done = true;   // below every class's probability: no membership test needed
                            } else {
                                const int cls = walk_class(col, t, ts, te, x, sorted);
                                done = u < (cls == 0 ? a.acc_t : (cls == 1 ? a.acc_1 : a.acc_q));
                            }
                        }
                        if (!done && !stray) {
                            // the exact draw after max_trials rejections (or with max_trials = 0)
                            const double u = walk_uniform(splitmix64(key, ++draws));
                            double total = 0.0;
                            for (int64_t i = s; i < e; ++i) {
                                const int cls = walk_class(col, t, ts, te, static_cast<int64_t>(__ldg(col + i)), sorted);
                                total += cls == 0 ? a.w_t : (cls == 1 ? 1.0 : a.w_q);
                            }
                            const double target = u * total;
                            double run = 0.0;
                            int64_t pick = e - 1;
                            for (int64_t i = s; i < e; ++i) {
                                const int64_t y = static_cast<int64_t>(__ldg(col + i));
                                const int cls = walk_class(col, t, ts, te, y, sorted);
                                run += cls == 0 ? a.w_t : (cls == 1 ? 1.0 : a.w_q);
                                if (run > target) {
                                    pick = i;
                                    break;
                                }
                            }
                            x = static_cast<int64_t>(__ldg(col + pick));
                        }
                    }
                    if (alive && (x < 0 || x >= a.n)) alive = false;
                    if (alive) {
                        t = v;
                        ts = s;
                        te = e;
                        v = x;
                    }
                }
                tile[threadIdx.x * kWalkPad + j] = alive ? static_cast<int32_t>(v) : -1;
            }
        }
        __syncthreads();
        // the CTA's walks cover rows [w0, w0 + n_rows): each row's columns [c0, c0 + cw) are one contiguous segment
        const int64_t total = n_rows * cw;
        for (int64_t f = threadIdx.x; f < total; f += kWalkThreads) {
            const int64_t r = f / cw, j = f - r * cw;
            out[(w0 + r) * width + c0 + j] = static_cast<I>(tile[r * kWalkPad + j]);
        }
        __syncthreads();
    }
}

// flag[0] = 1 when some row of col decreases (flag zeroed by the caller).  One warp per row.
template <typename I>
__global__ void __launch_bounds__(kWalkCheckThreads) walk_rows_unsorted_kernel(const I* __restrict__ rowptr,
                                                                               const I* __restrict__ col, int64_t n,
                                                                               int64_t n_edges, int32_t* flag) {
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    bool bad = false;
    for (int64_t u = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; u < n; u += n_warps) {
        const int64_t s = max(static_cast<int64_t>(__ldg(rowptr + u)), int64_t{0});
        const int64_t e = min(static_cast<int64_t>(__ldg(rowptr + u + 1)), n_edges);
        for (int64_t i = s + lane; i + 1 < e; i += 32) bad |= __ldg(col + i) > __ldg(col + i + 1);
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) *flag = 1;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_random_walk(const void* rowptr, const void* col, const void* start, int64_t n, int64_t n_edges,
                                  int64_t n_walks, int64_t walk_length, double p, double q, int64_t max_trials,
                                  uint64_t seed, int32_t* rows_unsorted, int refresh_rows_unsorted, void* out,
                                  int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n >= 0 && n < INT32_MAX && n_edges >= 0 && n_walks >= 0);
    B200MP_CHECK_ARG(walk_length >= 0 && walk_length < INT32_MAX);
    B200MP_CHECK_ARG(std::isfinite(p) && p > 0.0 && std::isfinite(q) && q > 0.0);
    B200MP_CHECK_ARG(max_trials >= 0 && max_trials <= INT32_MAX);
    B200MP_CHECK_ARG(idx_dtype == B200MP_I32 || idx_dtype == B200MP_I64);
    const bool biased = p != 1.0 || q != 1.0;
    B200MP_CHECK_ARG(!biased || rows_unsorted);
    if (n_walks == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && start && out && (col || n_edges == 0));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);

    WalkArgs a{};
    a.rowptr = rowptr;
    a.col = col;
    a.start = start;
    a.out = out;
    a.rows_unsorted = rows_unsorted;
    a.n = n;
    a.n_edges = n_edges;
    a.n_walks = n_walks;
    a.walk_length = walk_length;
    a.seed = seed;
    a.max_trials = static_cast<int>(max_trials);
    a.w_t = 1.0 / p;
    a.w_q = 1.0 / q;
    const double max_prob = std::fmax(std::fmax(a.w_t, 1.0), a.w_q);
    a.acc_t = a.w_t / max_prob;
    a.acc_1 = 1.0 / max_prob;
    a.acc_q = a.w_q / max_prob;
    a.acc_lo = std::fmin(std::fmin(a.acc_t, a.acc_1), a.acc_q);

    auto run = [&](auto ti) -> int {
        using I = decltype(ti);
        if (biased && refresh_rows_unsorted) {
            B200MP_CUDA(cudaMemsetAsync(rows_unsorted, 0, sizeof(int32_t), st));
            if (n > 0 && n_edges > 1) {
                const int64_t blocks = std::min(ceil_div(n, kWalkCheckThreads / 32), static_cast<int64_t>(num_sms()) * 16);
                walk_rows_unsorted_kernel<I><<<static_cast<unsigned>(blocks), kWalkCheckThreads, 0, st>>>(
                    static_cast<const I*>(rowptr), static_cast<const I*>(col), n, n_edges, rows_unsorted);
                B200MP_LAUNCH_CHECK();
            }
        }
        const int64_t blocks = ceil_div(n_walks, kWalkThreads);
        B200MP_CHECK_ARG(blocks <= INT32_MAX);
        if (biased) walk_kernel<I, true><<<static_cast<unsigned>(blocks), kWalkThreads, 0, st>>>(a);
        else walk_kernel<I, false><<<static_cast<unsigned>(blocks), kWalkThreads, 0, st>>>(a);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    };
    return idx_dtype == B200MP_I64 ? run(int64_t{}) : run(int32_t{});
}
