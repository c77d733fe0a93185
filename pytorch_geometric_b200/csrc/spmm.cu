// spmm.cu -- C ABI for the gather + segmented-reduce path (b200mp_spmm_csr) and its backward
// helpers (min/max tie counting, SDDMM for the edge-weight gradient).
#include "csr_dispatch.cuh"

namespace b200mp {

// ---------------------------------------------------------------- min/max backward
// ties[i,f] = [count_self_zero && out[i,f] == 0] + #{e in row i : val[e]*x[col[e],f] == out[i,f]}
template <typename T, typename I>
__global__ void __launch_bounds__(256)
minmax_ties_kernel(const I* __restrict__ rowptr, const I* __restrict__ col,
                   const float* __restrict__ val, const T* __restrict__ x, const T* __restrict__ out,
                   float* __restrict__ ties, int64_t n_rows, int64_t feat, int g, bool count_self_zero) {
    const int lig = threadIdx.x & (g - 1);
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / g;
    if (row >= n_rows) return;
    const int64_t begin = rowptr[row], end = rowptr[row + 1];
    for (int64_t f = lig; f < feat; f += g) {
        const float o = ElemTraits<T>::to_float(out[row * feat + f]);
        float cnt = (count_self_zero && o == 0.0f) ? 1.0f : 0.0f;
        for (int64_t e = begin; e < end; e += 4) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                v[u] = 0.f;
                if (e + u < end) {
                    const int64_t c = col[e + u];
                    const float xv = ElemTraits<T>::to_float(x[c * feat + f]);
                    // the forward rounds the product to T before comparing (out is stored as T)
                    v[u] = ElemTraits<T>::to_float(ElemTraits<T>::from_float(val ? __fmul_rn(__ldg(val + e + u), xv) : xv));
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (e + u < end && v[u] == o) cnt += 1.0f;
        }
        ties[row * feat + f] = cnt;
    }
}

// grad_x[j,f] = sum_{e in rowT(j)} [valT*x[j,f] == out[d,f]] * valT * g[d,f] / ties[d,f],  d = colT[e]
template <typename T, typename I>
__global__ void __launch_bounds__(256)
minmax_backward_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t,
                       const float* __restrict__ val_t, const T* __restrict__ x,
                       const T* __restrict__ out, const T* __restrict__ grad_out,
                       const float* __restrict__ ties, T* __restrict__ grad_x, int64_t n_src,
                       int64_t feat, int g) {
    const int lig = threadIdx.x & (g - 1);
    const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / g;
    if (j >= n_src) return;
    const int64_t begin = rowptr_t[j], end = rowptr_t[j + 1];
    for (int64_t f = lig; f < feat; f += g) {
        const float xv = ElemTraits<T>::to_float(x[j * feat + f]);
        float acc = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t d = col_t[e];
            const float w = val_t ? __ldg(val_t + e) : 1.0f;
            const float m = ElemTraits<T>::to_float(ElemTraits<T>::from_float(val_t ? __fmul_rn(w, xv) : xv));
            const float o = ElemTraits<T>::to_float(out[d * feat + f]);
            if (m == o) {
                const float gd = __fdiv_rn(ElemTraits<T>::to_float(grad_out[d * feat + f]), ties[d * feat + f]);
                acc = __fadd_rn(acc, val_t ? __fmul_rn(w, gd) : gd);
            }
        }
        grad_x[j * feat + f] = ElemTraits<T>::from_float(acc);
    }
}

// ---------------------------------------------------------------- SDDMM
// dot[e] = <a[row,:], b[col[e],:]>, one warp per CSR row, a[row] held in registers (up to 8
// values per lane, re-read from L1 beyond that), 5-step xor-shuffle reduction per edge.
template <typename T, typename I>
__global__ void __launch_bounds__(256)
sddmm_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const T* __restrict__ a,
             const T* __restrict__ b, float* __restrict__ dot, int64_t n_rows, int64_t feat) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_rows) return;
    const int64_t begin = rowptr[row], end = rowptr[row + 1];
    const T* ar = a + row * feat;
    for (int64_t e = begin; e < end; e += 2) {
        const bool has1 = e + 1 < end;
        const T* b0 = b + static_cast<int64_t>(col[e]) * feat;
        const T* b1 = has1 ? b + static_cast<int64_t>(col[e + 1]) * feat : b0;
        float s0 = 0.f, s1 = 0.f;
        for (int64_t f = lane; f < feat; f += 32) {
            const float av = ElemTraits<T>::to_float(ar[f]);
            s0 = fmaf(av, ElemTraits<T>::to_float(b0[f]), s0);
            s1 = fmaf(av, ElemTraits<T>::to_float(b1[f]), s1);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        }
        if (lane == 0) {
            dot[e] = s0;
            if (has1) dot[e + 1] = s1;
        }
    }
}

inline int group_width(int64_t feat) {
    int g = 1;
    while (g < 32 && g < feat) g <<= 1;
    return g;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_spmm_csr(const void* rowptr, const void* col, const float* val, const void* x,
                               void* out, int64_t n_rows, int64_t n_cols, int64_t feat, int reduce,
                               const int64_t* long_rows, const int64_t* chunk_ptr,
                               int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                               const float* bias, const void* x_halo, int64_t n_local_cols, int flags,
                               const void* peer_ptrs, int64_t peer_rows, const void* relu_mask, int idx_dtype,
                               int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && feat >= 0);
    B200MP_CHECK_ARG((flags & ~1) == 0 && (!(flags & 1) || (reduce == B200MP_SUM && !bias)));
    B200MP_CHECK_ARG(!relu_mask || (flags & 1));
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(x || n_cols == 0 || peer_ptrs);
    B200MP_CHECK_ARG(!peer_ptrs || (peer_rows > 0 && !x_halo && (feat * (val_dtype == B200MP_BF16 ? 2 : 4)) % 16 == 0));
    // the scalar fallback, taken when a matrix is not 16-byte aligned, has no peer-table addressing
    B200MP_CHECK_ARG(!peer_ptrs || (aligned16(x) && aligned16(out) && aligned16(relu_mask) &&
                                    (n_long_rows == 0 || aligned16(partials))));
    B200MP_CHECK_ARG(!x_halo || (n_local_cols >= 0 && n_local_cols <= n_cols));
    plan.x2 = x_halo;
    plan.split = x_halo ? n_local_cols : 0;
    plan.accumulate = flags & 1;
    plan.peers = static_cast<const unsigned long long*>(peer_ptrs);
    plan.peer_rows = peer_ptrs ? peer_rows : 0;
    plan.relu_mask = relu_mask;
    return dispatch_val_idx(val_dtype, idx_dtype, "spmm_csr", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        return csr_reduce_auto<T, I, true>(static_cast<const I*>(rowptr), static_cast<const I*>(col), val,
                                            static_cast<const T*>(x), static_cast<T*>(out), n_rows, feat, reduce,
                                            false, plan, bias, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_spmm_csr_self_colsum(const void* rowptr_t, const void* col_t, const float* val_t, const void* x,
                                           void* out, float* colsum_out, int64_t n_rows, int64_t feat,
                                           const int64_t* long_rows_t, const int64_t* chunk_ptr_t, int64_t n_long_rows_t,
                                           int64_t n_chunks_t, int64_t chunk, float* partials_t, float* colsum_parts,
                                           int64_t n_parts, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && feat >= 0 && n_parts >= 1);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows_t, chunk_ptr_t, n_long_rows_t, n_chunks_t, chunk, partials_t, true)) return rc;
    if (feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(colsum_out && colsum_parts);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n_rows == 0) return b200mp_column_sum(nullptr, colsum_out, colsum_parts, 1, 0, feat, val_dtype, stream);
    B200MP_CHECK_ARG(rowptr_t && col_t && val_t && x && out);
    return dispatch_val_idx(val_dtype, idx_dtype, "spmm_csr_self_colsum", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        int64_t parts = 0;
        if (int rc = csr_sum_self_colsum<T, I>(static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t), val_t,
                                               static_cast<const T*>(x), static_cast<T*>(out), n_rows, feat, plan,
                                               colsum_parts, n_parts - ceil_div(n_parts, 64), parts, s))
            return rc;
        // the per-CTA partials are a [parts, feat] fp32 matrix: fold them by the column sum, its second level behind them
        if (parts > 0)
            return b200mp_column_sum(colsum_parts, colsum_out, colsum_parts + parts * feat, b200mp_column_sum_parts(parts),
                                     parts, feat, B200MP_F32, stream);
        // no vector kernel for this row shape: the plain sweep, then a column sum of x (one row per self-loop)
        if (int rc = csr_reduce_dispatch<T, I, B200MP_SUM, true>(static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t),
                                                                 val_t, static_cast<const T*>(x), static_cast<T*>(out),
                                                                 n_rows, feat, false, false, plan, nullptr, s))
            return rc;
        return b200mp_column_sum(x, colsum_out, colsum_parts, std::min(n_parts, b200mp_column_sum_parts(n_rows)), n_rows,
                                 feat, val_dtype, stream);
    });
}

extern "C" int b200mp_minmax_ties(const void* rowptr, const void* col, const float* val, const void* x,
                                  const void* out, float* ties, int64_t n_rows, int64_t feat,
                                  int count_self_zero, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && feat >= 0);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out && ties);
    return dispatch_val_idx(val_dtype, idx_dtype, "minmax_ties", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        const int g = group_width(feat);
        minmax_ties_kernel<T, I><<<static_cast<unsigned>(ceil_div(n_rows, 256 / g)), 256, 0,
                                   static_cast<cudaStream_t>(stream)>>>(
            static_cast<const I*>(rowptr), static_cast<const I*>(col), val, static_cast<const T*>(x),
            static_cast<const T*>(out), ties, n_rows, feat, g, count_self_zero != 0);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_minmax_backward(const void* rowptr_t, const void* col_t, const float* val_t,
                                      const void* x, const void* out, const void* grad_out,
                                      const float* ties, void* grad_x, int64_t n_src, int64_t feat,
                                      int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_src >= 0 && feat >= 0);
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && x && grad_x);
    return dispatch_val_idx(val_dtype, idx_dtype, "minmax_backward", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        const int g = group_width(feat);
        minmax_backward_kernel<T, I><<<static_cast<unsigned>(ceil_div(n_src, 256 / g)), 256, 0,
                                       static_cast<cudaStream_t>(stream)>>>(
            static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t), val_t, static_cast<const T*>(x),
            static_cast<const T*>(out), static_cast<const T*>(grad_out), ties, static_cast<T*>(grad_x), n_src,
            feat, g);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_sddmm_csr(const void* rowptr, const void* col, const void* a, const void* b,
                                float* dot, int64_t n_rows, int64_t feat, int idx_dtype, int val_dtype,
                                void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && feat >= 0);
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && dot);
    return dispatch_val_idx(val_dtype, idx_dtype, "sddmm_csr", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        sddmm_kernel<T, I><<<static_cast<unsigned>(ceil_div(n_rows, 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            static_cast<const I*>(rowptr), static_cast<const I*>(col), static_cast<const T*>(a),
            static_cast<const T*>(b), dot, n_rows, feat);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}
