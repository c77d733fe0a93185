// nn_conv.cu -- NNConv's edge-conditioned message (nn_conv.py:96-122) as one CSR sweep into P plus one GEMM.
//
// The edge network's last Linear, h~_e = [h_e, 1] -> W2 h_e + b2, is linear, so the per-edge [F_in, F_out] weights
// never need to exist.  With W' = [W2.view(F_in, F_out, K).permute(2, 0, 1); b2.view(1, F_in, F_out)] reshaped to
// [(K+1) F_in, F_out] (nn/conv.py nn_conv_weight):
//   out_i = sum_{e = (j -> i)} x_j^T reshape(W2 h_e + b2) = vec(P_i) W',   P_i[k, a] = sum_e h~_e[k] x_j[a]
// and for mean P_i is divided by max(deg_i, 1).  This file computes P for a contiguous range of destination rows
// [row_begin, row_end) in fp32, and the destination half of the backward: with dP_i = dL/dP_i (from dL/dout by the
// caller's GEMM, dP = G W'^T),
//   grad_h[eid(e), k] = sum_a x_j[a] dP_i[k, a]  (k < K)        q[eid(e), a] = sum_k h~_e[k] dP_i[k, a]
// both scaled by 1 / max(deg_i, 1) for mean.  grad_x is the segment sum of q over each source's out-edges (the caller's
// b200mp_spmm_csr over the transposed CSR).  eid(e) = perm[e] (CSR slot -> the caller's edge id), or e for an adopted
// CSR (perm == NULL).  Every sum runs in fp32 in CSR order; nothing uses float atomics.
//
// Forward mapping.  One CTA per work item (a row, or one chunk of a hub row from the long-row plan), times grid.y
// slabs of P.  The CTA stages a batch of edges' h~ and x rows in shared memory as fp32, each row zero-padded to a
// multiple of 4 (Kp = roundup(K + 1, 4), Fp = roundup(F_in, 4)); each thread owns a 4 x 4 register tile of P_i and
// per edge does one float4 read of h~, one of x and 16 FMAs -- P_i = H~_i^T X_i as a small GEMM whose reduction
// dimension is the row's degree.  Chunk partials go to the plan's fp32 buffer and nn_conv_combine_kernel folds them
// in chunk order.  Rows without edges give P_i = 0.
//
// Backward mapping.  One CTA per work item reads dP_i (scaled for mean) into shared memory once, stages batches of
// edges like the forward, and gives each (edge, output) pair to one thread: an F_in-long dot product for grad_h and a
// (K+1)-long one for q.  grad_h's loop starts at a = k mod F_in and wraps, so the lanes of a warp (consecutive k) hit
// distinct banks of dP.  Each edge's outputs depend on no other edge, so chunks of a hub row need no combine step.
//
// Supported range: (K + 1) F_in <= 16384 (kNnMaxWidth), i.e. dP_i of at most 64 KiB in shared memory, with K >= 0
// and F_in >= 1; anything else is B200MP_ERR_UNSUPPORTED (b200mp_nn_conv_supported).  Shared memory per CTA: forward
// eb (Kp + Fp) 4 bytes with eb = clamp(32 KiB / ((Kp + Fp) 4), 1, 32) edges per batch; backward 4 (K + 1) F_in plus
// the same staging with a 16 KiB target -- at most about 130 KiB, under the H100's 227 KiB per-CTA limit.
//
// -Xptxas -v for sm_90a (CUDA 12.9): every instantiation has no stack frame and no spills.
//   nn_conv_fwd_kernel      fp32 / bf16 x int32 / int64: 49 (int64) and 53 (int32) registers
//   nn_conv_bwd_kernel      fp32 / bf16 x int32 / int64: 31 (int64) and 32 (int32) registers
//   nn_conv_combine_kernel  int32 / int64: 32 registers
#include "csr_reduce.cuh"

namespace b200mp {

constexpr int64_t kNnMaxWidth = 16384;        // (K + 1) F_in
constexpr int kNnFwdThreads = 512;            // most threads of a forward CTA (one 4 x 4 tile each)
constexpr int kNnBwdThreads = 256;
constexpr int kNnMaxBatch = 32;               // edges staged per batch

struct NnArgs {
    const void* x;      // [n_cols, fin]
    const void* h;      // [n_edges, K] in the caller's edge order (null when K == 0)
    const void* perm;   // index dtype: caller's edge id of each CSR slot, or null (= the slot)
    float* p;           // fwd: P [row_end - row_begin, (K+1) fin]
    const float* dp;    // bwd: dP, same layout
    void* grad_h;       // bwd: [n_edges, K] or null
    void* q;            // bwd: [n_edges, fin] or null
    int64_t k;
    int64_t fin;
    int64_t row_begin;
    int64_t row_end;
    int kp, fp;         // padded staging widths
    int eb;             // edges per staged batch
    bool is_mean;
};

template <typename I>
__device__ __forceinline__ int64_t nn_eid(const NnArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// The work item of this CTA: items [0, n_chunks) are plan chunks (skipped when their row is outside the range), the
// rest are the range's rows in order.  CTA-uniform.
template <typename I>
__device__ __forceinline__ bool nn_item(const I* rowptr, const NnArgs& a, const LongRowPlan& plan, int64_t& row,
                                        int64_t& begin, int64_t& end, bool& is_chunk) {
    const int64_t item = blockIdx.x;
    const int64_t it = item < plan.n_chunks ? item : item + a.row_begin;
    if (!decode_item(it, rowptr, a.row_end, plan, row, begin, end, is_chunk)) return false;
    return row >= a.row_begin && row < a.row_end;
}

// Stage edges [e0, e0 + nb) of the row: hs[b][k] = h~ (zero past K), xs[b][a] = x_j (zero past fin).
template <typename T, typename I>
__device__ __forceinline__ void nn_stage(const I* __restrict__ col, const NnArgs& a, int64_t e0, int nb, float* hs,
                                         float* xs) {
    const T* h = static_cast<const T*>(a.h);
    const T* x = static_cast<const T*>(a.x);
    for (int idx = threadIdx.x; idx < nb * a.kp; idx += blockDim.x) {
        const int b = idx / a.kp, k = idx - b * a.kp;
        float v = k == a.k ? 1.0f : 0.0f;
        if (k < a.k) v = ElemTraits<T>::to_float(h[nn_eid<I>(a, e0 + b) * a.k + k]);
        hs[idx] = v;
    }
    for (int idx = threadIdx.x; idx < nb * a.fp; idx += blockDim.x) {
        const int b = idx / a.fp, f = idx - b * a.fp;
        float v = 0.0f;
        if (f < a.fin) v = ElemTraits<T>::to_float(x[static_cast<int64_t>(ldg_idx(col + e0 + b)) * a.fin + f]);
        xs[idx] = v;
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(kNnFwdThreads)
nn_conv_fwd_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, NnArgs a, LongRowPlan plan) {
    extern __shared__ float4 nn_smem[];
    int64_t row, begin, end;
    bool is_chunk;
    if (!nn_item(rowptr, a, plan, row, begin, end, is_chunk)) return;
    float* hs = reinterpret_cast<float*>(nn_smem);
    float* xs = hs + a.eb * a.kp;
    const int a_tiles = a.fp / 4;
    const int tile = blockIdx.y * blockDim.x + threadIdx.x;
    const bool active = tile < a_tiles * (a.kp / 4);
    const int k0 = (tile / a_tiles) * 4, a0 = (tile % a_tiles) * 4;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (int64_t e0 = begin; e0 < end; e0 += a.eb) {
        const int nb = static_cast<int>(end - e0 < a.eb ? end - e0 : a.eb);
        __syncthreads();
        nn_stage<T, I>(col, a, e0, nb, hs, xs);
        __syncthreads();
        if (!active) continue;
        for (int b = 0; b < nb; ++b) {
            const float4 hv = *reinterpret_cast<const float4*>(hs + b * a.kp + k0);
            const float4 xv = *reinterpret_cast<const float4*>(xs + b * a.fp + a0);
            const float hk[4] = {hv.x, hv.y, hv.z, hv.w}, xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(hk[i], xa[j], acc[i][j]);
        }
    }
    if (!active) return;
    const int64_t width = (a.k + 1) * a.fin;
    float* dst = is_chunk ? plan.partials + static_cast<int64_t>(blockIdx.x) * width : a.p + (row - a.row_begin) * width;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (k0 + i > a.k) break;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (a0 + j >= a.fin) break;
            const float v = is_chunk ? acc[i][j] : finalize<B200MP_SUM>(acc[i][j], end - begin, a.is_mean, false);
            dst[(k0 + i) * a.fin + a0 + j] = v;
        }
    }
}

// Fold the fp32 partials of every long row of the range in chunk order and write its P row.
template <typename I>
__global__ void __launch_bounds__(256)
nn_conv_combine_kernel(const I* __restrict__ rowptr, NnArgs a, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    if (row < a.row_begin || row >= a.row_end) return;
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const int64_t width = (a.k + 1) * a.fin;
    float* dst = a.p + (row - a.row_begin) * width;
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x) {
        float acc = 0.0f;
        for (int64_t c = c0; c < c1; ++c) acc = __fadd_rn(acc, plan.partials[c * width + m]);
        dst[m] = finalize<B200MP_SUM>(acc, deg, a.is_mean, false);
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(kNnBwdThreads)
nn_conv_bwd_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, NnArgs a, LongRowPlan plan) {
    extern __shared__ float4 nn_smem[];
    int64_t row, begin, end;
    bool is_chunk;
    if (!nn_item(rowptr, a, plan, row, begin, end, is_chunk)) return;
    if (begin == end) return;
    const int64_t K = a.k, fin = a.fin, width = (K + 1) * fin;
    float* dps = reinterpret_cast<float*>(nn_smem);
    float* hs = dps + ((width + 3) & ~static_cast<int64_t>(3));
    float* xs = hs + a.eb * a.kp;
    const int64_t deg = static_cast<int64_t>(__ldg(rowptr + row + 1)) - static_cast<int64_t>(__ldg(rowptr + row));
    const float* src = a.dp + (row - a.row_begin) * width;
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x) dps[m] = finalize<B200MP_SUM>(src[m], deg, a.is_mean, false);
    T* gh = static_cast<T*>(a.grad_h);
    T* q = static_cast<T*>(a.q);
    const int k_out = gh ? static_cast<int>(K) : 0;
    const int w_out = k_out + (q ? static_cast<int>(fin) : 0);
    for (int64_t e0 = begin; e0 < end; e0 += a.eb) {
        const int nb = static_cast<int>(end - e0 < a.eb ? end - e0 : a.eb);
        __syncthreads();
        nn_stage<T, I>(col, a, e0, nb, hs, xs);
        __syncthreads();
        for (int o = threadIdx.x; o < nb * w_out; o += blockDim.x) {
            const int b = o / w_out, r = o - b * w_out;
            const int64_t eid = nn_eid<I>(a, e0 + b);
            float acc = 0.0f;
            if (r < k_out) {
                const float* xr = xs + b * a.fp;
                const float* dr = dps + static_cast<int64_t>(r) * fin;
                int f = static_cast<int>(r % fin);
                for (int t = 0; t < fin; ++t) {
                    acc = fmaf(xr[f], dr[f], acc);
                    f = f + 1 == fin ? 0 : f + 1;
                }
                gh[eid * K + r] = ElemTraits<T>::from_float(acc);
            } else {
                const int f = r - k_out;
                const float* hr = hs + b * a.kp;
                for (int64_t k = 0; k <= K; ++k) acc = fmaf(hr[k], dps[k * fin + f], acc);
                q[eid * fin + f] = ElemTraits<T>::from_float(acc);
            }
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
inline bool nn_supported(int64_t k, int64_t fin) { return k >= 0 && fin >= 1 && (k + 1) * fin <= kNnMaxWidth; }

inline NnArgs nn_args(const void* x, const void* h, const void* perm, int64_t k, int64_t fin, int64_t row_begin,
                      int64_t row_end, bool is_mean, int64_t stage_bytes) {
    NnArgs a{};
    a.x = x; a.h = h; a.perm = perm; a.k = k; a.fin = fin; a.row_begin = row_begin; a.row_end = row_end;
    a.is_mean = is_mean;
    a.kp = static_cast<int>((k + 1 + 3) / 4 * 4);
    a.fp = static_cast<int>((fin + 3) / 4 * 4);
    const int64_t row_bytes = static_cast<int64_t>(a.kp + a.fp) * 4;
    const int64_t eb = stage_bytes / row_bytes;
    a.eb = static_cast<int>(eb < 1 ? 1 : (eb > kNnMaxBatch ? kNnMaxBatch : eb));
    return a;
}

template <typename Kern>
int nn_smem_opt_in(Kern kernel, size_t smem) {
    if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    return B200MP_OK;
}

template <typename T, typename I>
int nn_fwd_typed(const void* rowptr_, const void* col_, NnArgs a, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + (a.row_end - a.row_begin);
    const int64_t tiles = static_cast<int64_t>(a.kp / 4) * (a.fp / 4);
    const int64_t slabs = ceil_div(tiles, kNnFwdThreads);
    const int threads = static_cast<int>(ceil_div(ceil_div(tiles, slabs), 32) * 32);
    const size_t smem = static_cast<size_t>(a.eb) * (a.kp + a.fp) * sizeof(float);
    if (int rc = nn_smem_opt_in(nn_conv_fwd_kernel<T, I>, smem)) return rc;
    nn_conv_fwd_kernel<T, I><<<dim3(static_cast<unsigned>(items), static_cast<unsigned>(slabs)), threads, smem, stream>>>(
        rowptr, col, a, plan);
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        nn_conv_combine_kernel<I><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, a, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int nn_bwd_typed(const void* rowptr_, const void* col_, NnArgs a, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + (a.row_end - a.row_begin);
    const int64_t width = (a.k + 1) * a.fin;
    const size_t smem = (static_cast<size_t>((width + 3) & ~static_cast<int64_t>(3)) +
                         static_cast<size_t>(a.eb) * (a.kp + a.fp)) * sizeof(float);
    if (int rc = nn_smem_opt_in(nn_conv_bwd_kernel<T, I>, smem)) return rc;
    nn_conv_bwd_kernel<T, I><<<static_cast<unsigned>(items), kNnBwdThreads, smem, stream>>>(rowptr, col, a, plan);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_nn_conv_supported(int64_t k, int64_t fin, int val_dtype) {
    return (val_dtype == B200MP_F32 || val_dtype == B200MP_BF16) && nn_supported(k, fin);
}

extern "C" int b200mp_nn_conv_csr(const void* rowptr, const void* col, const void* perm, const void* x, const void* h,
                                  float* p, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t k, int64_t fin,
                                  int64_t row_begin, int64_t row_end, int reduce, const int64_t* plan_rows,
                                  const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks,
                                  int64_t plan_chunk, float* plan_partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0);
    B200MP_CHECK_ARG(0 <= row_begin && row_begin <= row_end && row_end <= n_rows);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (!nn_supported(k, fin)) {
        set_error("nn_conv_csr: K = %lld, F_in = %lld is outside (K + 1) F_in <= %lld", static_cast<long long>(k),
                  static_cast<long long>(fin), static_cast<long long>(kNnMaxWidth));
        return B200MP_ERR_UNSUPPORTED;
    }
    LongRowPlan plan;
    if (int rc = make_plan(plan, plan_rows, plan_chunk_ptr, plan_n_long, plan_n_chunks, plan_chunk, plan_partials, true))
        return rc;
    if (row_begin == row_end) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && p);
    B200MP_CHECK_ARG(n_edges == 0 || (col && x && (h || k == 0)));
    NnArgs a = nn_args(x, h, perm, k, fin, row_begin, row_end, reduce == B200MP_MEAN, 32 * 1024);
    a.p = p;
    return dispatch_val_idx(val_dtype, idx_dtype, "nn_conv_csr", [&](auto tv, auto ti) {
        return nn_fwd_typed<decltype(tv), decltype(ti)>(rowptr, col, a, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_nn_conv_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                           const void* h, const float* grad_p, void* grad_h, void* q, int64_t n_rows,
                                           int64_t n_cols, int64_t n_edges, int64_t k, int64_t fin, int64_t row_begin,
                                           int64_t row_end, int reduce, const int64_t* plan_rows,
                                           const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks,
                                           int64_t plan_chunk, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0);
    B200MP_CHECK_ARG(0 <= row_begin && row_begin <= row_end && row_end <= n_rows);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (!nn_supported(k, fin)) {
        set_error("nn_conv_backward_dst: K = %lld, F_in = %lld is outside (K + 1) F_in <= %lld",
                  static_cast<long long>(k), static_cast<long long>(fin), static_cast<long long>(kNnMaxWidth));
        return B200MP_ERR_UNSUPPORTED;
    }
    LongRowPlan plan;
    if (int rc = make_plan(plan, plan_rows, plan_chunk_ptr, plan_n_long, plan_n_chunks, plan_chunk, nullptr, false))
        return rc;
    if (row_begin == row_end || n_edges == 0 || (grad_h == nullptr && q == nullptr)) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && col && x && grad_p && (h || k == 0));
    NnArgs a = nn_args(x, h, perm, k, fin, row_begin, row_end, reduce == B200MP_MEAN, 16 * 1024);
    a.dp = grad_p;
    a.grad_h = k > 0 ? grad_h : nullptr;
    a.q = q;
    return dispatch_val_idx(val_dtype, idx_dtype, "nn_conv_backward_dst", [&](auto tv, auto ti) {
        return nn_bwd_typed<decltype(tv), decltype(ti)>(rowptr, col, a, plan, static_cast<cudaStream_t>(stream));
    });
}
