// cluster.cu -- cluster vectors for pooling: greedy graph matching (graclus) and regular-grid clustering (voxel grid)
// (pyg_lib.ops graclus_cluster / grid_cluster, reached through torch.ops.pyg.* in nn/pool/graclus.py:39 and
// nn/pool/voxel_grid.py:66).
//
// Graclus.  torch-cluster's GPU greedy matching (after Auer and Bisseling), restated so that the result is a pure
// function of (graph, weights, seed) and stays race-free on directed inputs.  Nodes start unmatched (cluster = -1).
// In round r, node u is blue when the top bit of splitmix64(seed, r N + u) is set and red otherwise; colours are
// recomputed wherever they are needed.  A candidate of u is an adjacency entry v != u with a non-NaN weight and v still
// unmatched.  Each round has three phases; a phase reads only what earlier phases wrote and writes only its own node's
// slot:
//   propose:  an unmatched blue u with no candidate records "singleton"; otherwise it proposes to one red candidate,
//             the first in CSR order (unweighted) or the one of largest weight, ties to the earlier CSR position.
//   respond:  an unmatched red u with no candidate records "singleton"; otherwise it accepts one blue candidate that
//             proposed to it, chosen the same way.
//   settle:   a matched pair (blue u proposed to v and v accepted u) gets min(u, v) -- torch-cluster's GPU convention
//             -- and a singleton gets u.  A per-round flag (two slots alternating by round parity) records whether any
//             node is still unmatched.
// Every round runs inside ONE cooperative persistent launch: a grid sized by the occupancy API, one warp per node
// (lanes stride the adjacency, a warp argmax sends ties to the lowest position), a grid sync after each phase, and no
// host read at any graph size.  Every thread takes the same branch at every sync: the done flag is read by all threads
// after a sync, and no thread leaves the round loop early.  The loop stops after kGraclusMaxRounds rounds at the latest
// (on a directed 3-cycle no red node ever sees its proposer, so the matching alone never ends); then every node still
// unmatched becomes a singleton.  The number of rounds used is written to the workspace.  Weights are fp32, bf16 or
// fp64 and are only compared, after an exact widening to fp64.  A hub row costs deg / 32 steps per phase in its warp.
//
// Grid.  For point i, c_i = sum_d trunc((pos[i, d] - start[d]) / size[d]) * stride_d, with
// stride_d = prod_{d' < d} (trunc((end[d'] - start[d']) / size[d']) + 1), in the input dtype (fp32 or fp64) with one
// IEEE subtract and one IEEE divide per term, converted toward zero (saturating; NaN gives INT64_MIN) and summed in
// wrapping 64-bit integer arithmetic.  A missing start / end is the column min / max of pos, NaN propagating as
// torch.min / torch.max do, computed by a two-kernel reduction on the device.
//
// -Xptxas -v for sm_90a (CUDA 12.9): every instantiation has no stack frame and no spills.
#include <cooperative_groups.h>

#include <climits>

#include "common.cuh"

namespace b200mp {

namespace cg = cooperative_groups;

constexpr int kGraclusMaxRounds = 256;   // GRACLUS_MAX_ROUNDS
constexpr int kGraclusThreads = 256;
constexpr int32_t kGcSingleton = -2;     // proposal / acceptance record of a node with no candidate
constexpr int kGcBatch = 4;              // adjacency entries per lane loaded together
constexpr int kGridThreads = 256;
constexpr int64_t kGridParts = 256;      // partial min / max per column, at most
constexpr int64_t kGridRowsPerPart = 4096;

inline int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }

struct GcNoWeight {};

struct GcArgs {
    const void* rowptr;
    const void* col;
    const void* weight;
    int64_t n;
    unsigned long long seed;
    int64_t* cluster;
    int32_t* proposal;   // [n]: the red node u proposed to, -1, or kGcSingleton (blue nodes, this round)
    int32_t* accept;     // [n]: the blue node u accepted, -1, or kGcSingleton (red nodes, this round)
    int32_t* flags;      // [2]: some node is still unmatched after round r, slot r & 1
    int32_t* rounds;     // [1]: rounds used
};

// splitmix64's finaliser on seed + key * golden ratio (common.cuh), as attention dropout (attention.cu) hashes its slots.
__device__ __forceinline__ bool gc_blue(unsigned long long seed, int round, int64_t n, int64_t u) {
    const unsigned long long key =
        static_cast<unsigned long long>(round) * static_cast<unsigned long long>(n) + static_cast<unsigned long long>(u);
    return (splitmix64(seed, key) >> 63) != 0ull;
}

__device__ __forceinline__ double gc_weight(const float* w, int64_t e) { return static_cast<double>(__ldg(w + e)); }
__device__ __forceinline__ double gc_weight(const __nv_bfloat16* w, int64_t e) {
    return static_cast<double>(__bfloat162float(w[e]));
}
__device__ __forceinline__ double gc_weight(const double* w, int64_t e) { return __ldg(w + e); }

// One warp scans u's adjacency.  Returns, in every lane, kGcSingleton when u has no candidate, else the chosen node
// (the largest weight, ties to the lowest CSR position; unweighted: the lowest position) or -1 when none qualifies.
// Propose (RESPOND = false) chooses among red candidates; respond among blue candidates whose proposal is u.
template <bool RESPOND, typename I, typename WT>
__device__ __forceinline__ int32_t gc_scan(const GcArgs& a, int round, int64_t u, int lane) {
    const I* rowptr = static_cast<const I*>(a.rowptr);
    const I* col = static_cast<const I*>(a.col);
    const int64_t s = static_cast<int64_t>(__ldg(rowptr + u)), e = static_cast<int64_t>(__ldg(rowptr + u + 1));
    bool any = false;
    double bw = -__longlong_as_double(0x7ff0000000000000ll);   // -inf
    int64_t bpos = LLONG_MAX;
    // kGcBatch entries per lane are loaded before any is examined, so a hub row keeps several gathers in flight
    for (int64_t p0 = s + lane; p0 < e; p0 += 32 * kGcBatch) {
        int64_t v[kGcBatch], c[kGcBatch];
#pragma unroll
        for (int j = 0; j < kGcBatch; ++j) v[j] = p0 + 32 * j < e ? static_cast<int64_t>(__ldg(col + p0 + 32 * j)) : u;
#pragma unroll
        for (int j = 0; j < kGcBatch; ++j) c[j] = v[j] != u ? __ldcg(a.cluster + v[j]) : 0;
#pragma unroll
        for (int j = 0; j < kGcBatch; ++j) {
            const int64_t p = p0 + 32 * j;
            if (v[j] == u || c[j] != -1) continue;
            double w = 0.0;
            if constexpr (!std::is_same<WT, GcNoWeight>::value) {
                w = gc_weight(static_cast<const WT*>(a.weight), p);
                if (w != w) continue;
            }
            any = true;
            bool ok;
            if constexpr (RESPOND)
                ok = gc_blue(a.seed, round, a.n, v[j]) && __ldcg(a.proposal + v[j]) == static_cast<int32_t>(u);
            else ok = !gc_blue(a.seed, round, a.n, v[j]);
            // positions rise within a lane, so a strict > keeps the lane's earliest of equal weights
            if (ok && (w > bw || bpos == LLONG_MAX)) {
                bw = w;
                bpos = p;
            }
        }
    }
    if (!__any_sync(0xffffffffu, any)) return kGcSingleton;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double ow = __shfl_xor_sync(0xffffffffu, bw, off);
        const long long op = __shfl_xor_sync(0xffffffffu, static_cast<long long>(bpos), off);
        if (op != LLONG_MAX && (bpos == LLONG_MAX || ow > bw || (ow == bw && op < bpos))) {
            bw = ow;
            bpos = op;
        }
    }
    return bpos == LLONG_MAX ? -1 : static_cast<int32_t>(__ldg(col + bpos));
}

template <typename I, typename WT>
__global__ void __launch_bounds__(kGraclusThreads, 4) cluster_graclus_kernel(GcArgs a) {
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t n_threads = static_cast<int64_t>(gridDim.x) * blockDim.x;
    int round = 0;
    bool done = false;
    for (; round < kGraclusMaxRounds && !done; ++round) {
        // propose: unmatched blue nodes
        for (int64_t u = warp; u < a.n; u += n_warps) {
            if (__ldcg(a.cluster + u) != -1 || !gc_blue(a.seed, round, a.n, u)) continue;
            const int32_t pick = gc_scan<false, I, WT>(a, round, u, lane);
            if (lane == 0) a.proposal[u] = pick;
        }
        grid.sync();
        // respond: unmatched red nodes.  The flag slot of the next round was last read before this round's first
        // sync, so it can be cleared here.
        if (tid == 0) a.flags[(round + 1) & 1] = 0;
        for (int64_t u = warp; u < a.n; u += n_warps) {
            if (__ldcg(a.cluster + u) != -1 || gc_blue(a.seed, round, a.n, u)) continue;
            const int32_t pick = gc_scan<true, I, WT>(a, round, u, lane);
            if (lane == 0) a.accept[u] = pick;
        }
        grid.sync();
        // settle: one thread per node
        bool pending = false;
        for (int64_t u = tid; u < a.n; u += n_threads) {
            if (__ldcg(a.cluster + u) != -1) continue;
            int64_t c = -1;
            if (gc_blue(a.seed, round, a.n, u)) {
                const int32_t p = __ldcg(a.proposal + u);
                if (p == kGcSingleton) c = u;
                else if (p >= 0 && __ldcg(a.accept + p) == static_cast<int32_t>(u)) c = p < u ? p : u;
            } else {
                const int32_t q = __ldcg(a.accept + u);
                if (q == kGcSingleton) c = u;
                else if (q >= 0) c = q < u ? q : u;
            }
            if (c >= 0) a.cluster[u] = c;
            else pending = true;
        }
        if (__syncthreads_or(pending) && threadIdx.x == 0) a.flags[round & 1] = 1;
        grid.sync();
        done = __ldcg(a.flags + (round & 1)) == 0;
    }
    if (!done) {
        // the round cap: every node still unmatched becomes a singleton
        for (int64_t u = tid; u < a.n; u += n_threads)
            if (__ldcg(a.cluster + u) == -1) a.cluster[u] = u;
    }
    if (tid == 0) *a.rounds = round;
}

// ---------------------------------------------------------------- grid
__device__ __forceinline__ float grid_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double grid_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float grid_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double grid_div(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ unsigned long long grid_trunc(float v) {
    return static_cast<unsigned long long>(v != v ? LLONG_MIN : __float2ll_rz(v));
}
__device__ __forceinline__ unsigned long long grid_trunc(double v) {
    return static_cast<unsigned long long>(v != v ? LLONG_MIN : __double2ll_rz(v));
}

template <typename T>
__device__ __forceinline__ T grid_min(T m, T v) { return (v < m || v != v) ? v : m; }
template <typename T>
__device__ __forceinline__ T grid_max(T m, T v) { return (v > m || v != v) ? v : m; }

// Block reduction of (lo, hi); the result is valid in thread 0.
template <typename T>
__device__ __forceinline__ void grid_block_minmax(T& lo, T& hi) {
    __shared__ T s_lo[kGridThreads / 32], s_hi[kGridThreads / 32];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        lo = grid_min(lo, __shfl_xor_sync(0xffffffffu, lo, off));
        hi = grid_max(hi, __shfl_xor_sync(0xffffffffu, hi, off));
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        s_lo[w] = lo;
        s_hi[w] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < kGridThreads / 32; ++i) {
            lo = grid_min(lo, s_lo[i]);
            hi = grid_max(hi, s_hi[i]);
        }
    }
}

// Partial column min / max: block (b, c) covers rows b, b + gridDim.x, ... of its chunk loop over column c.
template <typename T>
__global__ void __launch_bounds__(kGridThreads) cluster_minmax_kernel(const T* __restrict__ pos, int64_t n, int64_t d,
                                                                     T* __restrict__ part) {
    const int64_t c = blockIdx.y;
    T lo = pos[c], hi = pos[c];
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const T v = __ldg(pos + i * d + c);
        lo = grid_min(lo, v);
        hi = grid_max(hi, v);
    }
    grid_block_minmax(lo, hi);
    if (threadIdx.x == 0) {
        part[(c * gridDim.x + blockIdx.x) * 2] = lo;
        part[(c * gridDim.x + blockIdx.x) * 2 + 1] = hi;
    }
}

// Folds the parts of column blockIdx.x into lo[c] / hi[c].
template <typename T>
__global__ void __launch_bounds__(kGridThreads) cluster_minmax_fold_kernel(const T* __restrict__ part, int64_t n_parts,
                                                                          T* __restrict__ lo_out, T* __restrict__ hi_out) {
    const int64_t c = blockIdx.x;
    const T* p = part + c * n_parts * 2;
    T lo = p[0], hi = p[1];
    for (int64_t i = threadIdx.x; i < n_parts; i += blockDim.x) {
        lo = grid_min(lo, p[2 * i]);
        hi = grid_max(hi, p[2 * i + 1]);
    }
    grid_block_minmax(lo, hi);
    if (threadIdx.x == 0) {
        lo_out[c] = lo;
        hi_out[c] = hi;
    }
}

template <typename T>
__global__ void __launch_bounds__(kGridThreads) cluster_grid_kernel(const T* __restrict__ pos, const T* __restrict__ size,
                                                                   const T* __restrict__ start, const T* __restrict__ end,
                                                                   int64_t n, int64_t d, int64_t* __restrict__ out) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        unsigned long long c = 0ull, stride = 1ull;
        for (int64_t k = 0; k < d; ++k) {
            const T s = __ldg(start + k), sz = __ldg(size + k);
            c += grid_trunc(grid_div(grid_sub(__ldg(pos + i * d + k), s), sz)) * stride;
            stride *= grid_trunc(grid_div(grid_sub(__ldg(end + k), s), sz)) + 1ull;
        }
        out[i] = static_cast<int64_t>(c);
    }
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_graclus(const void* rowptr, const void* col, const void* weight, int64_t n, uint64_t seed,
                              int64_t* cluster, int32_t* ws, int idx_dtype, int weight_dtype, void* stream) {
    B200MP_CHECK_ARG(n >= 0 && n < INT32_MAX);
    B200MP_CHECK_ARG(idx_dtype == B200MP_I32 || idx_dtype == B200MP_I64);
    B200MP_CHECK_ARG(ws);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n == 0) {
        B200MP_CUDA(cudaMemsetAsync(ws, 0, 3 * sizeof(int32_t), st));
        return B200MP_OK;
    }
    B200MP_CHECK_ARG(rowptr && cluster);   // col may be NULL: a graph without edges
    int dev = 0, coop = 0;
    B200MP_CUDA(cudaGetDevice(&dev));
    B200MP_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) {
        set_error("graclus: device %d does not support cooperative launches", dev);
        return B200MP_ERR_UNSUPPORTED;
    }
    GcArgs a{};
    a.rowptr = rowptr;
    a.col = col;
    a.weight = weight;
    a.n = n;
    a.seed = seed;
    a.cluster = cluster;
    a.proposal = ws;
    a.accept = ws + n;
    a.flags = ws + 2 * n;
    a.rounds = ws + 2 * n + 2;
    auto launch = [&](auto ti, auto tw) -> int {
        using I = decltype(ti);
        using WT = decltype(tw);
        void (*kern)(GcArgs) = cluster_graclus_kernel<I, WT>;
        int per_sm = 0;
        B200MP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kGraclusThreads, 0));
        if (per_sm < 1) {
            set_error("graclus: the kernel cannot be resident on an SM");
            return B200MP_ERR_UNSUPPORTED;
        }
        const int64_t blocks = min64(static_cast<int64_t>(per_sm) * num_sms(), ceil_div(n, kGraclusThreads / 32));
        B200MP_CUDA(cudaMemsetAsync(cluster, 0xff, static_cast<size_t>(n) * sizeof(int64_t), st));
        B200MP_CUDA(cudaMemsetAsync(a.flags, 0, 2 * sizeof(int32_t), st));
        void* args[] = {&a};
        B200MP_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kern), dim3(static_cast<unsigned>(blocks)),
                                                dim3(kGraclusThreads), args, 0, st));
        return B200MP_OK;
    };
    auto by_weight = [&](auto ti) -> int {
        if (weight == nullptr) return launch(ti, GcNoWeight{});
        if (weight_dtype == B200MP_F32) return launch(ti, float{});
        if (weight_dtype == B200MP_BF16) return launch(ti, __nv_bfloat16{});
        if (weight_dtype == B200MP_F64) return launch(ti, double{});
        set_error("graclus: unsupported weight dtype %d", weight_dtype);
        return B200MP_ERR_UNSUPPORTED;
    };
    return idx_dtype == B200MP_I64 ? by_weight(int64_t{}) : by_weight(int32_t{});
}

extern "C" int b200mp_grid_cluster(const void* pos, const void* size, const void* start, const void* end, int64_t n,
                                   int64_t d, int64_t* out, void* ws, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n >= 0 && d >= 1 && d <= 65535);
    if (val_dtype != B200MP_F32 && val_dtype != B200MP_F64) {
        set_error("grid_cluster: unsupported value dtype %d (float32 or float64 only)", val_dtype);
        return B200MP_ERR_UNSUPPORTED;
    }
    if (n == 0) return B200MP_OK;
    B200MP_CHECK_ARG(pos && size && out && ((start && end) || ws));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto run = [&](auto tv) -> int {
        using T = decltype(tv);
        const T* lo = static_cast<const T*>(start);
        const T* hi = static_cast<const T*>(end);
        if (!lo || !hi) {
            T* w = static_cast<T*>(ws);
            const int64_t parts = min64(ceil_div(n, kGridRowsPerPart), kGridParts);
            T* part = w + 2 * d;
            cluster_minmax_kernel<T><<<dim3(static_cast<unsigned>(parts), static_cast<unsigned>(d)), kGridThreads, 0,
                                       st>>>(static_cast<const T*>(pos), n, d, part);
            B200MP_LAUNCH_CHECK();
            cluster_minmax_fold_kernel<T><<<static_cast<unsigned>(d), kGridThreads, 0, st>>>(part, parts, w, w + d);
            B200MP_LAUNCH_CHECK();
            if (!lo) lo = w;
            if (!hi) hi = w + d;
        }
        const int64_t blocks = min64(ceil_div(n, kGridThreads), static_cast<int64_t>(num_sms()) * 16);
        cluster_grid_kernel<T><<<static_cast<unsigned>(blocks), kGridThreads, 0, st>>>(
            static_cast<const T*>(pos), static_cast<const T*>(size), lo, hi, n, d, out);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    };
    return val_dtype == B200MP_F64 ? run(double{}) : run(float{});
}
