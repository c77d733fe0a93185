// structure.cu -- graph-structure (integer) work: degree, index<->ptr, stable sort by key,
// self-loop insertion, gcn_norm weights, long-row plan.  Results are bit-exact with the
// reference (oracle/mp_oracle.c section "integer work").  Sorting and stream compaction use CUB
// (library calls, as cuBLAS would be for a GEMM); everything else is hand-written.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"

namespace b200mp {

constexpr int kThreads = 256;
inline unsigned grid_for(int64_t n, int per_block = kThreads) {
    int64_t b = ceil_div(n, per_block);
    return static_cast<unsigned>(b < 1 ? 1 : b);
}

template <typename I>
__global__ void degree_kernel(const I* __restrict__ index, int64_t n, I* __restrict__ deg) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= n) return;
    if (sizeof(I) == 8)
        atomicAdd(reinterpret_cast<unsigned long long*>(deg + index[e]), 1ull);
    else
        atomicAdd(reinterpret_cast<unsigned int*>(deg + index[e]), 1u);
}

// ptr[i] = #(index < i) for sorted index: thread e in [0, E] fills ptr[(prev, cur]] = e.
template <typename I>
__global__ void index2ptr_kernel(const I* __restrict__ index, int64_t n, int64_t n_nodes, I* __restrict__ ptr) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e > n) return;
    const int64_t prev = e == 0 ? -1 : static_cast<int64_t>(index[e - 1]);
    const int64_t cur = e == n ? n_nodes : static_cast<int64_t>(index[e]);
    for (int64_t i = prev + 1; i <= cur; ++i) ptr[i] = static_cast<I>(e);
}

template <typename I>
__device__ __forceinline__ int64_t row_of_edge(const I* __restrict__ ptr, int64_t n_nodes, int64_t e) {
    // largest i with ptr[i] <= e  (rows may be empty: upper bound - 1)
    int64_t lo = 0, hi = n_nodes;  // answer in [lo, hi)
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (static_cast<int64_t>(__ldg(ptr + mid)) <= e) lo = mid; else hi = mid;
    }
    return lo;
}

template <typename I>
__global__ void ptr2index_kernel(const I* __restrict__ ptr, int64_t n_nodes, int64_t n, I* __restrict__ index) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= n) return;
    index[e] = static_cast<I>(row_of_edge(ptr, n_nodes, e));
}

template <typename I>
__global__ void index_stats_kernel(const I* __restrict__ index, int64_t n, long long* __restrict__ stats) {
    long long mn = LLONG_MAX, mx = LLONG_MIN;
    int unsorted = 0;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
         e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const long long v = index[e];
        mn = v < mn ? v : mn;
        mx = v > mx ? v : mx;
        if (e > 0 && static_cast<long long>(index[e - 1]) > v) unsorted = 1;
    }
    typedef cub::BlockReduce<long long, kThreads> BR;
    __shared__ typename BR::TempStorage tmp;
    mn = BR(tmp).Reduce(mn, cub::Min());
    __syncthreads();
    mx = BR(tmp).Reduce(mx, cub::Max());
    __syncthreads();
    const long long us = BR(tmp).Reduce(static_cast<long long>(unsorted), cub::Max());
    if (threadIdx.x == 0) {
        atomicMin(stats + 0, mn);
        atomicMax(stats + 1, mx);
        if (us) atomicMin(stats + 2, 0ll);
    }
}
__global__ void index_stats_init(long long* stats, int64_t n) {
    stats[0] = n ? LLONG_MAX : 0;
    stats[1] = n ? LLONG_MIN : -1;
    stats[2] = 1;
}

template <typename I>
__global__ void iota_kernel(I* __restrict__ out, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = static_cast<I>(i);
}

template <typename E, typename I>
__global__ void permute_kernel(const E* __restrict__ in, const I* __restrict__ perm, E* __restrict__ out, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[perm[i]];
}

template <typename A, typename B>
__global__ void convert_kernel(const A* __restrict__ in, B* __restrict__ out, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) out[i] = static_cast<B>(in[i]);
}

inline int bits_for(int64_t n_nodes) {
    int b = 1;
    while (b < 63 && (int64_t(1) << b) < n_nodes) ++b;
    return b;
}
inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

template <typename I>
size_t sort_temp_bytes(int64_t n, int64_t n_nodes) {
    size_t t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, static_cast<const I*>(nullptr), static_cast<I*>(nullptr),
                                    static_cast<const I*>(nullptr), static_cast<I*>(nullptr), n, 0,
                                    bits_for(n_nodes));
    return t;
}

template <typename I>
int sort_typed(const void* keys, int64_t n, int64_t n_nodes, void* keys_sorted, void* perm, void* ptr,
               void* workspace, int64_t ws_bytes, cudaStream_t stream) {
    const size_t arr = align_up(sizeof(I) * static_cast<size_t>(n));
    size_t temp = sort_temp_bytes<I>(n, n_nodes);
    const size_t need = arr * 2 + align_up(temp);
    if (static_cast<size_t>(ws_bytes) < need) {
        set_error("sort_by_key: workspace %lld < %zu", static_cast<long long>(ws_bytes), need);
        return B200MP_ERR_WORKSPACE;
    }
    char* ws = static_cast<char*>(workspace);
    I* iota = reinterpret_cast<I*>(ws);
    I* kout = keys_sorted ? static_cast<I*>(keys_sorted) : reinterpret_cast<I*>(ws + arr);
    void* tmp = ws + 2 * arr;
    if (n > 0) {
        iota_kernel<I><<<grid_for(n), kThreads, 0, stream>>>(iota, n);
        B200MP_LAUNCH_CHECK();
        // LSD radix sort is stable: equal keys keep input order (== torch.sort(stable=True)).
        B200MP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, temp, static_cast<const I*>(keys), kout, iota,
                                                    static_cast<I*>(perm), n, 0, bits_for(n_nodes), stream));
    }
    if (ptr) {
        index2ptr_kernel<I><<<grid_for(n + 1), kThreads, 0, stream>>>(kout, n, n_nodes, static_cast<I*>(ptr));
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

// ---------------------------------------------------------------- self loops
template <typename I>
struct NotLoop {
    const I* row;
    const I* col;
    __device__ __forceinline__ bool operator()(const int64_t& e) const { return row[e] != col[e]; }
};

template <typename I>
__global__ void self_loops_write_kernel(const I* __restrict__ row, const I* __restrict__ col,
                                        const float* __restrict__ w_in, const int64_t* __restrict__ kept,
                                        const int64_t* __restrict__ n_kept_dev, int64_t n_nodes,
                                        float fill, I* __restrict__ row_out, I* __restrict__ col_out,
                                        float* __restrict__ w_out, int64_t* __restrict__ n_out_dev) {
    const int64_t n_kept = *n_kept_dev;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i == 0) *n_out_dev = n_kept + n_nodes;
    if (i < n_kept) {
        const int64_t e = kept[i];
        row_out[i] = row[e];
        col_out[i] = col[e];
        if (w_in) w_out[i] = w_in[e];
    } else if (i < n_kept + n_nodes) {
        const int64_t v = i - n_kept;
        row_out[i] = static_cast<I>(v);
        col_out[i] = static_cast<I>(v);
        if (w_in) w_out[i] = fill;
    }
}
// existing self-loop weights override fill; duplicates: the LAST edge in input order wins
template <typename I>
__global__ void loop_last_edge_kernel(const I* __restrict__ row, const I* __restrict__ col, int64_t n_edges,
                                      long long* __restrict__ last) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e < n_edges && row[e] == col[e]) atomicMax(last + row[e], static_cast<long long>(e));
}
__global__ void fill_ll_kernel(long long* p, int64_t n, long long v) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void loop_weight_kernel(const float* __restrict__ w_in, const long long* __restrict__ last,
                                   const int64_t* __restrict__ n_kept_dev, int64_t n_nodes,
                                   float* __restrict__ w_out) {
    const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (v < n_nodes && last[v] >= 0) w_out[*n_kept_dev + v] = w_in[last[v]];
}

template <typename I>
size_t select_temp_bytes(int64_t n) {
    size_t t = 0;
    thrust::counting_iterator<int64_t> it(0);
    NotLoop<I> pred{nullptr, nullptr};
    cub::DeviceSelect::If(nullptr, t, it, static_cast<int64_t*>(nullptr), static_cast<int64_t*>(nullptr), n, pred);
    return t;
}

template <typename I>
int self_loops_typed(const void* row_, const void* col_, const float* w_in, int64_t n_edges, int64_t n_nodes,
                     float fill, int mode, void* row_out, void* col_out, float* w_out, int64_t* n_out_dev,
                     void* workspace, int64_t ws_bytes, cudaStream_t stream) {
    const I* row = static_cast<const I*>(row_);
    const I* col = static_cast<const I*>(col_);
    size_t temp = select_temp_bytes<I>(n_edges);
    const size_t kept_b = align_up(sizeof(int64_t) * static_cast<size_t>(n_edges));
    const size_t last_b = align_up(sizeof(long long) * static_cast<size_t>(n_nodes));
    const size_t need = kept_b + last_b + 256 + align_up(temp);
    if (static_cast<size_t>(ws_bytes) < need) {
        set_error("self_loops: workspace %lld < %zu", static_cast<long long>(ws_bytes), need);
        return B200MP_ERR_WORKSPACE;
    }
    char* ws = static_cast<char*>(workspace);
    int64_t* kept = reinterpret_cast<int64_t*>(ws);
    long long* last = reinterpret_cast<long long*>(ws + kept_b);
    int64_t* n_kept = reinterpret_cast<int64_t*>(ws + kept_b + last_b);
    void* tmp = ws + kept_b + last_b + 256;
    thrust::counting_iterator<int64_t> it(0);
    NotLoop<I> pred{row, col};
    B200MP_CUDA(cub::DeviceSelect::If(tmp, temp, it, kept, n_kept, n_edges, pred, stream));
    self_loops_write_kernel<I><<<grid_for(n_edges + n_nodes), kThreads, 0, stream>>>(
        row, col, w_in, kept, n_kept, n_nodes, fill, static_cast<I*>(row_out), static_cast<I*>(col_out), w_out,
        n_out_dev);
    B200MP_LAUNCH_CHECK();
    if (w_in && mode == 0 && n_nodes > 0) {
        fill_ll_kernel<<<grid_for(n_nodes), kThreads, 0, stream>>>(last, n_nodes, -1ll);
        if (n_edges > 0) loop_last_edge_kernel<I><<<grid_for(n_edges), kThreads, 0, stream>>>(row, col, n_edges, last);
        loop_weight_kernel<<<grid_for(n_nodes), kThreads, 0, stream>>>(w_in, last, n_kept, n_nodes, w_out);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

// ---------------------------------------------------------------- gcn_norm on the dst-sorted CSR
// deg[i] = in-order sum of w over row i (bit-identical to the reference's serial scatter_add_).
template <typename I>
__global__ void gcn_deg_kernel(const I* __restrict__ rowptr, const float* __restrict__ w, int64_t n_nodes,
                               float* __restrict__ dinv) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const int64_t b = rowptr[i], e = rowptr[i + 1];
    float deg;
    if (w) {
        deg = 0.0f;
        for (int64_t k = b; k < e; ++k) deg = __fadd_rn(deg, __ldg(w + k));
    } else {
        deg = static_cast<float>(e - b);  // sum of ones, exact below 2^24 and correctly rounded above
    }
    float d = powf(deg, -0.5f);  // gcn_conv.py:109 deg.pow_(-0.5)
    if (isinf(d)) d = 0.0f;      // :110 masked_fill_(== inf, 0)
    dinv[i] = d;
}
template <typename I>
__global__ void gcn_weight_kernel(const I* __restrict__ rowptr, const I* __restrict__ src,
                                  const float* __restrict__ w, const float* __restrict__ dinv, int64_t n_nodes,
                                  int64_t n_edges, float* __restrict__ w_out) {
    const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int64_t dst = row_of_edge(rowptr, n_nodes, e);
    const float we = w ? w[e] : 1.0f;
    // gcn_conv.py:111: deg_inv_sqrt[row] * edge_weight * deg_inv_sqrt[col], left to right
    w_out[e] = __fmul_rn(__fmul_rn(dinv[src[e]], we), dinv[dst]);
}

// ---------------------------------------------------------------- long-row plan
template <typename I>
__global__ void plan_count_kernel(const I* __restrict__ rowptr, int64_t n_rows, int64_t chunk,
                                  unsigned long long* __restrict__ counts) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_rows) return;
    const int64_t deg = static_cast<int64_t>(rowptr[i + 1]) - static_cast<int64_t>(rowptr[i]);
    if (deg > chunk) {
        atomicAdd(counts + 0, 1ull);
        atomicAdd(counts + 1, static_cast<unsigned long long>((deg + chunk - 1) / chunk));
    }
}
template <typename I>
struct IsLong {
    const I* rowptr;
    int64_t chunk;
    __device__ __forceinline__ bool operator()(const int64_t& i) const {
        return static_cast<int64_t>(rowptr[i + 1]) - static_cast<int64_t>(rowptr[i]) > chunk;
    }
};
template <typename I>
__global__ void plan_chunks_kernel(const I* __restrict__ rowptr, const int64_t* __restrict__ long_rows,
                                   int64_t n_long, int64_t chunk, int64_t* __restrict__ nchunks) {
    const int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j > n_long) return;
    if (j == n_long) { nchunks[j] = 0; return; }
    const int64_t r = long_rows[j];
    const int64_t deg = static_cast<int64_t>(rowptr[r + 1]) - static_cast<int64_t>(rowptr[r]);
    nchunks[j] = (deg + chunk - 1) / chunk;
}

}  // namespace b200mp

using namespace b200mp;

#define IDX_DISPATCH(EXPR32, EXPR64)                                        \
    do {                                                                    \
        if (idx_dtype == B200MP_I32) { EXPR32; }                            \
        else if (idx_dtype == B200MP_I64) { EXPR64; }                       \
        else { set_error("bad idx_dtype %d", idx_dtype); return B200MP_ERR_UNSUPPORTED; } \
    } while (0)

extern "C" int b200mp_degree(const void* index, int64_t n_index, int64_t n_nodes, void* deg, int idx_dtype,
                             void* stream) {
    B200MP_CHECK_ARG(n_index >= 0 && n_nodes >= 0);
    B200MP_CHECK_ARG(deg || n_nodes == 0);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t isz = idx_dtype == B200MP_I64 ? 8 : 4;
    if (n_nodes) B200MP_CUDA(cudaMemsetAsync(deg, 0, isz * n_nodes, s));
    if (n_index == 0) return B200MP_OK;
    B200MP_CHECK_ARG(index);
    IDX_DISPATCH((degree_kernel<int32_t><<<grid_for(n_index), kThreads, 0, s>>>(static_cast<const int32_t*>(index), n_index, static_cast<int32_t*>(deg))),
                 (degree_kernel<int64_t><<<grid_for(n_index), kThreads, 0, s>>>(static_cast<const int64_t*>(index), n_index, static_cast<int64_t*>(deg))));
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_index2ptr(const void* index_sorted, int64_t n_index, int64_t n_nodes, void* ptr,
                                int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_index >= 0 && n_nodes >= 0 && ptr);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    IDX_DISPATCH((index2ptr_kernel<int32_t><<<grid_for(n_index + 1), kThreads, 0, s>>>(static_cast<const int32_t*>(index_sorted), n_index, n_nodes, static_cast<int32_t*>(ptr))),
                 (index2ptr_kernel<int64_t><<<grid_for(n_index + 1), kThreads, 0, s>>>(static_cast<const int64_t*>(index_sorted), n_index, n_nodes, static_cast<int64_t*>(ptr))));
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_ptr2index(const void* ptr, int64_t n_nodes, int64_t n_index, void* index, int idx_dtype,
                                void* stream) {
    B200MP_CHECK_ARG(n_index >= 0 && n_nodes >= 0 && ptr);
    if (n_index == 0) return B200MP_OK;
    B200MP_CHECK_ARG(index);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    IDX_DISPATCH((ptr2index_kernel<int32_t><<<grid_for(n_index), kThreads, 0, s>>>(static_cast<const int32_t*>(ptr), n_nodes, n_index, static_cast<int32_t*>(index))),
                 (ptr2index_kernel<int64_t><<<grid_for(n_index), kThreads, 0, s>>>(static_cast<const int64_t*>(ptr), n_nodes, n_index, static_cast<int64_t*>(index))));
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_index_stats(const void* index, int64_t n_index, int64_t* stats, int idx_dtype,
                                  void* stream) {
    B200MP_CHECK_ARG(n_index >= 0 && stats);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    long long* st = reinterpret_cast<long long*>(stats);
    index_stats_init<<<1, 1, 0, s>>>(st, n_index);
    if (n_index > 0) {
        B200MP_CHECK_ARG(index);
        int64_t blocks = ceil_div(n_index, kThreads);
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        IDX_DISPATCH((index_stats_kernel<int32_t><<<static_cast<unsigned>(blocks), kThreads, 0, s>>>(static_cast<const int32_t*>(index), n_index, st)),
                     (index_stats_kernel<int64_t><<<static_cast<unsigned>(blocks), kThreads, 0, s>>>(static_cast<const int64_t*>(index), n_index, st)));
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int64_t b200mp_sort_workspace_bytes(int64_t n_index, int64_t n_nodes, int idx_dtype) {
    if (n_index < 0 || n_nodes < 0) return B200MP_ERR_INVALID_ARG;
    const size_t isz = idx_dtype == B200MP_I64 ? 8 : 4;
    const size_t arr = align_up(isz * static_cast<size_t>(n_index));
    const size_t temp = idx_dtype == B200MP_I64 ? sort_temp_bytes<int64_t>(n_index, n_nodes)
                                                : sort_temp_bytes<int32_t>(n_index, n_nodes);
    return static_cast<int64_t>(arr * 2 + align_up(temp) + 256);
}

extern "C" int b200mp_sort_by_key(const void* keys, int64_t n_index, int64_t n_nodes, void* keys_sorted,
                                  void* perm, void* ptr, void* workspace, int64_t workspace_bytes,
                                  int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_index >= 0 && n_nodes >= 0);
    B200MP_CHECK_ARG(n_index == 0 || (keys && perm && workspace));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (idx_dtype == B200MP_I32)
        return sort_typed<int32_t>(keys, n_index, n_nodes, keys_sorted, perm, ptr, workspace, workspace_bytes, s);
    if (idx_dtype == B200MP_I64)
        return sort_typed<int64_t>(keys, n_index, n_nodes, keys_sorted, perm, ptr, workspace, workspace_bytes, s);
    set_error("bad idx_dtype %d", idx_dtype);
    return B200MP_ERR_UNSUPPORTED;
}

extern "C" int b200mp_permute(const void* in, const void* perm, void* out, int64_t n, int elem_bytes,
                              int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n >= 0);
    if (n == 0) return B200MP_OK;
    B200MP_CHECK_ARG(in && perm && out);
    B200MP_CHECK_ARG(elem_bytes == 4 || elem_bytes == 8);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (elem_bytes == 4) {
        IDX_DISPATCH((permute_kernel<uint32_t, int32_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const uint32_t*>(in), static_cast<const int32_t*>(perm), static_cast<uint32_t*>(out), n)),
                     (permute_kernel<uint32_t, int64_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const uint32_t*>(in), static_cast<const int64_t*>(perm), static_cast<uint32_t*>(out), n)));
    } else {
        IDX_DISPATCH((permute_kernel<uint64_t, int32_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const uint64_t*>(in), static_cast<const int32_t*>(perm), static_cast<uint64_t*>(out), n)),
                     (permute_kernel<uint64_t, int64_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const uint64_t*>(in), static_cast<const int64_t*>(perm), static_cast<uint64_t*>(out), n)));
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_convert_index(const void* in, int in_dtype, void* out, int out_dtype, int64_t n,
                                    void* stream) {
    B200MP_CHECK_ARG(n >= 0);
    if (n == 0) return B200MP_OK;
    B200MP_CHECK_ARG(in && out);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (in_dtype == B200MP_I64 && out_dtype == B200MP_I32)
        convert_kernel<int64_t, int32_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const int64_t*>(in), static_cast<int32_t*>(out), n);
    else if (in_dtype == B200MP_I32 && out_dtype == B200MP_I64)
        convert_kernel<int32_t, int64_t><<<grid_for(n), kThreads, 0, s>>>(static_cast<const int32_t*>(in), static_cast<int64_t*>(out), n);
    else if (in_dtype == out_dtype && (in_dtype == B200MP_I32 || in_dtype == B200MP_I64))
        B200MP_CUDA(cudaMemcpyAsync(out, in, (in_dtype == B200MP_I64 ? 8 : 4) * static_cast<size_t>(n), cudaMemcpyDeviceToDevice, s));
    else {
        set_error("convert_index: bad dtypes %d -> %d", in_dtype, out_dtype);
        return B200MP_ERR_UNSUPPORTED;
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int64_t b200mp_self_loops_workspace_bytes(int64_t n_edges, int64_t n_nodes, int idx_dtype) {
    if (n_edges < 0 || n_nodes < 0) return B200MP_ERR_INVALID_ARG;
    const size_t temp = idx_dtype == B200MP_I64 ? select_temp_bytes<int64_t>(n_edges) : select_temp_bytes<int32_t>(n_edges);
    return static_cast<int64_t>(align_up(8 * static_cast<size_t>(n_edges)) + align_up(8 * static_cast<size_t>(n_nodes)) + 256 + align_up(temp) + 256);
}

extern "C" int b200mp_self_loops(const void* row, const void* col, const float* w_in, int64_t n_edges,
                                 int64_t n_nodes, float fill_value, int mode, void* row_out, void* col_out,
                                 float* w_out, int64_t* n_out_dev, void* workspace, int64_t workspace_bytes,
                                 int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_edges >= 0 && n_nodes >= 0 && n_out_dev && workspace);
    B200MP_CHECK_ARG(n_edges == 0 || (row && col));
    B200MP_CHECK_ARG(n_edges + n_nodes == 0 || (row_out && col_out));
    B200MP_CHECK_ARG(!w_in || w_out);
    B200MP_CHECK_ARG(mode == 0 || mode == 1);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (idx_dtype == B200MP_I32)
        return self_loops_typed<int32_t>(row, col, w_in, n_edges, n_nodes, fill_value, mode, row_out, col_out, w_out, n_out_dev, workspace, workspace_bytes, s);
    if (idx_dtype == B200MP_I64)
        return self_loops_typed<int64_t>(row, col, w_in, n_edges, n_nodes, fill_value, mode, row_out, col_out, w_out, n_out_dev, workspace, workspace_bytes, s);
    set_error("bad idx_dtype %d", idx_dtype);
    return B200MP_ERR_UNSUPPORTED;
}

extern "C" int b200mp_gcn_norm_csr(const void* rowptr, const void* src, const float* w, int64_t n_nodes,
                                   int64_t n_edges, float* deg_inv_sqrt, float* w_out, int idx_dtype,
                                   void* stream) {
    B200MP_CHECK_ARG(n_nodes >= 0 && n_edges >= 0);
    if (n_nodes == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && deg_inv_sqrt);
    B200MP_CHECK_ARG(n_edges == 0 || (src && w_out));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    IDX_DISPATCH(({
                     gcn_deg_kernel<int32_t><<<grid_for(n_nodes), kThreads, 0, s>>>(static_cast<const int32_t*>(rowptr), w, n_nodes, deg_inv_sqrt);
                     if (n_edges) gcn_weight_kernel<int32_t><<<grid_for(n_edges), kThreads, 0, s>>>(static_cast<const int32_t*>(rowptr), static_cast<const int32_t*>(src), w, deg_inv_sqrt, n_nodes, n_edges, w_out);
                 }),
                 ({
                     gcn_deg_kernel<int64_t><<<grid_for(n_nodes), kThreads, 0, s>>>(static_cast<const int64_t*>(rowptr), w, n_nodes, deg_inv_sqrt);
                     if (n_edges) gcn_weight_kernel<int64_t><<<grid_for(n_edges), kThreads, 0, s>>>(static_cast<const int64_t*>(rowptr), static_cast<const int64_t*>(src), w, deg_inv_sqrt, n_nodes, n_edges, w_out);
                 }));
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_csr_plan_count(const void* rowptr, int64_t n_rows, int64_t chunk, int64_t* counts_dev,
                                     int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && chunk > 0 && counts_dev);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    B200MP_CUDA(cudaMemsetAsync(counts_dev, 0, 16, s));
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr);
    unsigned long long* c = reinterpret_cast<unsigned long long*>(counts_dev);
    IDX_DISPATCH((plan_count_kernel<int32_t><<<grid_for(n_rows), kThreads, 0, s>>>(static_cast<const int32_t*>(rowptr), n_rows, chunk, c)),
                 (plan_count_kernel<int64_t><<<grid_for(n_rows), kThreads, 0, s>>>(static_cast<const int64_t*>(rowptr), n_rows, chunk, c)));
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

namespace b200mp {
template <typename I>
size_t plan_temp_bytes(int64_t n_rows, int64_t n_long) {
    size_t t1 = 0, t2 = 0;
    thrust::counting_iterator<int64_t> it(0);
    IsLong<I> pred{nullptr, 1};
    cub::DeviceSelect::If(nullptr, t1, it, static_cast<int64_t*>(nullptr), static_cast<int64_t*>(nullptr), n_rows, pred);
    cub::DeviceScan::ExclusiveSum(nullptr, t2, static_cast<int64_t*>(nullptr), static_cast<int64_t*>(nullptr), n_long + 1);
    return t1 > t2 ? t1 : t2;
}
template <typename I>
int plan_fill_typed(const void* rowptr_, int64_t n_rows, int64_t chunk, int64_t n_long, int64_t* long_rows,
                    int64_t* chunk_ptr, void* workspace, int64_t ws_bytes, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    size_t temp = plan_temp_bytes<I>(n_rows, n_long);
    const size_t nch_b = align_up(8 * static_cast<size_t>(n_long + 1));
    if (static_cast<size_t>(ws_bytes) < nch_b + 256 + align_up(temp)) {
        set_error("csr_plan_fill: workspace too small");
        return B200MP_ERR_WORKSPACE;
    }
    char* ws = static_cast<char*>(workspace);
    int64_t* nchunks = reinterpret_cast<int64_t*>(ws);
    int64_t* n_sel = reinterpret_cast<int64_t*>(ws + nch_b);
    void* tmp = ws + nch_b + 256;
    thrust::counting_iterator<int64_t> it(0);
    IsLong<I> pred{rowptr, chunk};
    size_t t = temp;
    B200MP_CUDA(cub::DeviceSelect::If(tmp, t, it, long_rows, n_sel, n_rows, pred, s));
    plan_chunks_kernel<I><<<grid_for(n_long + 1), kThreads, 0, s>>>(rowptr, long_rows, n_long, chunk, nchunks);
    B200MP_LAUNCH_CHECK();
    t = temp;
    B200MP_CUDA(cub::DeviceScan::ExclusiveSum(tmp, t, nchunks, chunk_ptr, n_long + 1, s));
    return B200MP_OK;
}
}  // namespace b200mp

extern "C" int64_t b200mp_csr_plan_workspace_bytes(int64_t n_rows, int64_t n_long_rows, int idx_dtype) {
    if (n_rows < 0 || n_long_rows < 0) return B200MP_ERR_INVALID_ARG;
    const size_t temp = idx_dtype == B200MP_I64 ? plan_temp_bytes<int64_t>(n_rows, n_long_rows)
                                                : plan_temp_bytes<int32_t>(n_rows, n_long_rows);
    return static_cast<int64_t>(align_up(8 * static_cast<size_t>(n_long_rows + 1)) + 256 + align_up(temp) + 256);
}

extern "C" int b200mp_csr_plan_fill(const void* rowptr, int64_t n_rows, int64_t chunk, int64_t n_long_rows,
                                    int64_t* long_rows, int64_t* chunk_ptr, void* workspace,
                                    int64_t workspace_bytes, int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && chunk > 0 && n_long_rows >= 0);
    if (n_long_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && long_rows && chunk_ptr && workspace);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (idx_dtype == B200MP_I32)
        return plan_fill_typed<int32_t>(rowptr, n_rows, chunk, n_long_rows, long_rows, chunk_ptr, workspace, workspace_bytes, s);
    if (idx_dtype == B200MP_I64)
        return plan_fill_typed<int64_t>(rowptr, n_rows, chunk, n_long_rows, long_rows, chunk_ptr, workspace, workspace_bytes, s);
    set_error("bad idx_dtype %d", idx_dtype);
    return B200MP_ERR_UNSUPPORTED;
}
