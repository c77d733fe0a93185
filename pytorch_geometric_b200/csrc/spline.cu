// spline.cu -- SplineConv's B-spline basis and weighting (spline_conv.py:150-153, pyg_lib.ops.spline_basis /
// spline_weighting), and its message fused with the aggregation as one CSR sweep into P plus one GEMM.
//
// Basis.  For edge e, slot s in [0, S), S = (degree + 1)^D, dimension 0 varying fastest in s and in the index:
//   v_d = pseudo[e, d] * (kernel_size[d] - degree * is_open_spline[d])      (one fp32 multiply, so floor(v) is exact)
//   k_d = (s / (degree + 1)^d) mod (degree + 1)
//   wi[e, s] = sum_d ((floor(v_d) + k_d) mod kernel_size[d]) * prod_{d' < d} kernel_size[d']
//   basis[e, s] = prod_d B_degree(v_d - floor(v_d), k_d)
// The modulo is non-negative and a kernel size below 1 counts as 1, so pseudo outside [0, 1] (which the reference does
// not define) never yields an index outside [0, K): a deliberate difference from the reference, which may read out of
// bounds there.  grad_pseudo[e, d] = sum_s grad_basis[e, s] B'(t_d, k_d) prod_{d' != d} B(t_d', k_d') * scale_d.
//
// Weighting.  out[e] = sum_s basis[e, s] x[e] @ weight[wi[e, s]], weight [K, F_in, F_out].  The standalone kernels give
// one thread per output element and spend S F_in F_out FMAs per edge; grad_weight reduces each kernel's slots, sorted
// by wi once by the caller, in that order.  Slots whose wi lies outside [0, K) contribute nothing.
//
// Fused message.  out_i = REDUCE_{e = (j -> i)} sum_s b_es x_j W[wi_es] = vec(P_i) W.view(K F_in, F_out) with
//   P_i[k F_in + a] = sum_{e, s : wi_es = k} b_es x_j[a]           (mean: / max(deg_i, 1))
// b200mp_spline_csr writes P in fp32 for destination rows [row_begin, row_end); the GEMM is the caller's.  One CTA per
// work item (a row, or one chunk of a hub row from the long-row plan) holds P_i in shared memory; each thread owns
// feature columns a, so the S scaled adds per edge never conflict.  Batches of edges stage their source index, basis
// and wi (pre-multiplied by F_in) in shared memory.  Per edge a thread does one read of x_j[a] and S FMAs: S F_in FMAs
// per edge, not K F_in.  Chunk partials go to the plan's fp32 buffer and spline_combine_kernel folds them in chunk
// order.  The destination half of the backward holds dP_i (scaled for mean) in shared memory and gives each (edge,
// output) pair to one thread: grad_basis[e, s] = <dP_i[wi_es], x_j> (an F_in-long dot product whose start rotates with
// the slot, to spread shared-memory banks) and q[e, a] = sum_s b_es dP_i[wi_es, a].  grad_x is the caller's segment sum
// of q over the transposed CSR.  Every sum runs in fp32 in a fixed order; nothing uses float atomics.
//
// Supported range (b200mp_spline_supported): degree 1..3 for the basis; 1 <= S <= 64 (kSplMaxS: degree 3 up to D = 3,
// degree 1 up to D = 6) for every kernel; for the sweeps also K >= 1, F_in >= 1 and K F_in <= 16384 (P_i or dP_i of at
// most 64 KiB in shared memory), else B200MP_ERR_UNSUPPORTED.  Shared memory per CTA: 4 K F_in plus a batch of
// eb <= 32 edges' staging, at most about 100 KiB.
//
// -Xptxas -v for sm_90a (CUDA 12.9): every instantiation has no stack frame and no spills.
//   spline_basis_kernel                  fp32 / bf16 x int32 / int64 wi: 32 registers
//   spline_basis_bwd_kernel              fp32 / bf16: 32 registers
//   spline_weighting_fwd_kernel          fp32 / bf16 x int32 / int64 wi: 32 registers
//   spline_weighting_bwd_x_kernel        fp32 / bf16 x int32 / int64 wi: 32 registers
//   spline_weighting_bwd_basis_kernel    fp32 / bf16 x int32 / int64 wi: 32 registers
//   spline_weighting_bwd_weight_kernel   fp32 / bf16 x int32 / int64 wi: 31 (fp32) and 32 (bf16) registers
//   spline_fwd_kernel                    fp32 / bf16 x int32 / int64: 28 (fp32) and 32 (bf16) registers
//   spline_bwd_kernel                    fp32 / bf16 x int32 / int64: 32 registers
//   spline_combine_kernel                int32 / int64: 32 registers
#include "csr_reduce.cuh"

namespace b200mp {

constexpr int kSplMaxS = 64;                  // (degree + 1)^D
constexpr int64_t kSplMaxWidth = 16384;       // K F_in
constexpr int kSplMaxBatch = 32;              // edges staged per batch
constexpr int kSplThreads = 512;

// ---------------------------------------------------------------- basis
__device__ __forceinline__ float spline_piece(int degree, float t, int k) {
    if (degree == 1) return 1.0f - t - static_cast<float>(k) + 2.0f * t * static_cast<float>(k);
    if (degree == 2) {
        if (k == 0) return 0.5f * t * t - t + 0.5f;
        if (k == 1) return -t * t + t + 0.5f;
        return 0.5f * t * t;
    }
    if (k == 0) {
        const float u = 1.0f - t;
        return u * u * u / 6.0f;
    }
    if (k == 1) return (3.0f * t * t * t - 6.0f * t * t + 4.0f) / 6.0f;
    if (k == 2) return (-3.0f * t * t * t + 3.0f * t * t + 3.0f * t + 1.0f) / 6.0f;
    return t * t * t / 6.0f;
}

__device__ __forceinline__ float spline_piece_grad(int degree, float t, int k) {
    if (degree == 1) return 2.0f * static_cast<float>(k) - 1.0f;
    if (degree == 2) {
        if (k == 0) return t - 1.0f;
        if (k == 1) return -2.0f * t + 1.0f;
        return t;
    }
    if (k == 0) {
        const float u = 1.0f - t;
        return -0.5f * u * u;
    }
    if (k == 1) return 1.5f * t * t - 2.0f * t;
    if (k == 2) return -1.5f * t * t + t + 0.5f;
    return 0.5f * t * t;
}

// v_d of edge e's pseudo-coordinate d, its kernel size (at least 1) and scale (kernel_size - degree * is_open)
template <typename T>
__device__ __forceinline__ float spline_v(const T* pseudo, const int64_t* ks, const uint8_t* open, int64_t e, int dim,
                                          int d, int degree, int64_t& ksd, float& scale) {
    const int64_t k = __ldg(ks + d);
    ksd = k < 1 ? 1 : k;
    scale = static_cast<float>(ksd - (__ldg(open + d) ? degree : 0));
    return ElemTraits<T>::to_float(pseudo[e * dim + d]) * scale;
}

template <typename T, typename W>
__global__ void __launch_bounds__(256)
spline_basis_kernel(const T* __restrict__ pseudo, const int64_t* __restrict__ ks, const uint8_t* __restrict__ open,
                    T* __restrict__ basis, W* __restrict__ wi, int64_t n, int dim, int degree, int S) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= n * S) return;
    const int64_t e = idx / S;
    int k = static_cast<int>(idx - e * S);
    int64_t w = 0, off = 1;
    float b = 1.0f;
    for (int d = 0; d < dim; ++d) {
        const int km = k % (degree + 1);
        k /= degree + 1;
        int64_t ksd;
        float scale;
        const float v = spline_v(pseudo, ks, open, e, dim, d, degree, ksd, scale);
        const float fl = floorf(v);
        const int64_t fi = fabsf(fl) < 4.0e18f ? static_cast<int64_t>(fl) : 0;    // inf / NaN: any in-range index
        int64_t i = (fi + km) % ksd;
        if (i < 0) i += ksd;
        w += i * off;
        off *= ksd;
        b *= spline_piece(degree, v - fl, km);
    }
    basis[idx] = ElemTraits<T>::from_float(b);
    wi[idx] = static_cast<W>(w);
}

template <typename T>
__global__ void __launch_bounds__(256)
spline_basis_bwd_kernel(const T* __restrict__ grad_basis, const T* __restrict__ pseudo, const int64_t* __restrict__ ks,
                        const uint8_t* __restrict__ open, T* __restrict__ grad_pseudo, int64_t n, int dim, int degree,
                        int S) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= n * dim) return;
    const int64_t e = idx / dim;
    const int dg = static_cast<int>(idx - e * dim);
    float acc = 0.0f;
    for (int s = 0; s < S; ++s) {
        int k = s;
        float prod = 1.0f;
        for (int d = 0; d < dim; ++d) {
            const int km = k % (degree + 1);
            k /= degree + 1;
            int64_t ksd;
            float scale;
            const float v = spline_v(pseudo, ks, open, e, dim, d, degree, ksd, scale);
            const float t = v - floorf(v);
            prod *= d == dg ? spline_piece_grad(degree, t, km) * scale : spline_piece(degree, t, km);
        }
        acc = fmaf(ElemTraits<T>::to_float(grad_basis[e * S + s]), prod, acc);
    }
    grad_pseudo[idx] = ElemTraits<T>::from_float(acc);
}

// ---------------------------------------------------------------- standalone weighting (one thread per output)
struct SwArgs {
    const void* x;        // [E, fin]
    const void* weight;   // [K, fin, fout]
    const void* basis;    // [E, S]
    const void* wi;       // [E, S], index dtype
    const void* grad_out; // [E, fout]
    int64_t n, fin, fout, k;
    int s;
};

template <typename I>
__device__ __forceinline__ int64_t sw_index(const SwArgs& a, int64_t slot) {
    const int64_t w = static_cast<int64_t>(static_cast<const I*>(a.wi)[slot]);
    return w >= 0 && w < a.k ? w : -1;
}

template <typename T, typename I>
__global__ void __launch_bounds__(256) spline_weighting_fwd_kernel(SwArgs a, T* __restrict__ out) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= a.n * a.fout) return;
    const int64_t e = idx / a.fout, o = idx - e * a.fout;
    const T* x = static_cast<const T*>(a.x) + e * a.fin;
    const T* W = static_cast<const T*>(a.weight);
    const T* B = static_cast<const T*>(a.basis);
    float acc = 0.0f;
    for (int s = 0; s < a.s; ++s) {
        const int64_t w = sw_index<I>(a, e * a.s + s);
        if (w < 0) continue;
        const T* wk = W + w * a.fin * a.fout + o;
        float t = 0.0f;
        for (int64_t f = 0; f < a.fin; ++f) t = fmaf(ElemTraits<T>::to_float(x[f]), ElemTraits<T>::to_float(wk[f * a.fout]), t);
        acc = fmaf(ElemTraits<T>::to_float(B[e * a.s + s]), t, acc);
    }
    out[idx] = ElemTraits<T>::from_float(acc);
}

template <typename T, typename I>
__global__ void __launch_bounds__(256) spline_weighting_bwd_x_kernel(SwArgs a, T* __restrict__ grad_x) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= a.n * a.fin) return;
    const int64_t e = idx / a.fin, f = idx - e * a.fin;
    const T* g = static_cast<const T*>(a.grad_out) + e * a.fout;
    const T* W = static_cast<const T*>(a.weight);
    const T* B = static_cast<const T*>(a.basis);
    float acc = 0.0f;
    for (int s = 0; s < a.s; ++s) {
        const int64_t w = sw_index<I>(a, e * a.s + s);
        if (w < 0) continue;
        const T* wk = W + (w * a.fin + f) * a.fout;
        float t = 0.0f;
        for (int64_t o = 0; o < a.fout; ++o) t = fmaf(ElemTraits<T>::to_float(g[o]), ElemTraits<T>::to_float(wk[o]), t);
        acc = fmaf(ElemTraits<T>::to_float(B[e * a.s + s]), t, acc);
    }
    grad_x[idx] = ElemTraits<T>::from_float(acc);
}

template <typename T, typename I>
__global__ void __launch_bounds__(256) spline_weighting_bwd_basis_kernel(SwArgs a, T* __restrict__ grad_basis) {
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= a.n * a.s) return;
    const int64_t e = idx / a.s;
    const int64_t w = sw_index<I>(a, idx);
    float acc = 0.0f;
    if (w >= 0) {
        const T* x = static_cast<const T*>(a.x) + e * a.fin;
        const T* g = static_cast<const T*>(a.grad_out) + e * a.fout;
        const T* wk = static_cast<const T*>(a.weight) + w * a.fin * a.fout;
        for (int64_t f = 0; f < a.fin; ++f) {
            float t = 0.0f;
            for (int64_t o = 0; o < a.fout; ++o)
                t = fmaf(ElemTraits<T>::to_float(wk[f * a.fout + o]), ElemTraits<T>::to_float(g[o]), t);
            acc = fmaf(ElemTraits<T>::to_float(x[f]), t, acc);
        }
    }
    grad_basis[idx] = ElemTraits<T>::from_float(acc);
}

// grad_weight[k, f, o] = sum over the slots of kernel k, in the caller's sorted order, of basis x[e, f] g[e, o].
// Grid: (K, tiles of 256 (f, o) pairs).
template <typename T, typename I>
__global__ void __launch_bounds__(256)
spline_weighting_bwd_weight_kernel(SwArgs a, const I* __restrict__ order, const I* __restrict__ kptr,
                                   float* __restrict__ grad_weight) {
    const int64_t k = blockIdx.x;
    const int64_t m = static_cast<int64_t>(blockIdx.y) * blockDim.x + threadIdx.x;
    if (m >= a.fin * a.fout) return;
    const int64_t f = m / a.fout, o = m - f * a.fout;
    const T* x = static_cast<const T*>(a.x);
    const T* g = static_cast<const T*>(a.grad_out);
    const T* B = static_cast<const T*>(a.basis);
    float acc = 0.0f;
    const int64_t j1 = static_cast<int64_t>(ldg_idx(kptr + k + 1));
    for (int64_t j = static_cast<int64_t>(ldg_idx(kptr + k)); j < j1; ++j) {
        const int64_t slot = static_cast<int64_t>(ldg_idx(order + j));
        const int64_t e = slot / a.s;
        const float bx = ElemTraits<T>::to_float(B[slot]) * ElemTraits<T>::to_float(x[e * a.fin + f]);
        acc = fmaf(bx, ElemTraits<T>::to_float(g[e * a.fout + o]), acc);
    }
    grad_weight[k * a.fin * a.fout + m] = acc;
}

// ---------------------------------------------------------------- fused CSR sweeps
struct SplArgs {
    const void* x;        // [n_cols, fin]
    const void* basis;    // [n_edges, S] in the caller's edge order
    const int32_t* wi;    // [n_edges, S] in the caller's edge order
    const void* perm;     // index dtype: caller's edge id of each CSR slot, or null (= the slot)
    float* p;             // fwd: P [row_end - row_begin, K fin]
    const float* dp;      // bwd: dP, same layout
    void* grad_basis;     // bwd: [n_edges, S] or null
    void* q;              // bwd: [n_edges, fin] or null
    int64_t k;
    int64_t fin;
    int64_t row_begin;
    int64_t row_end;
    int s;
    int fp;               // fin padded to a multiple of 4 (backward staging)
    int eb;               // edges per staged batch
    bool is_mean;
};

template <typename I>
__device__ __forceinline__ int64_t spl_eid(const SplArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// The work item of this CTA: items [0, n_chunks) are plan chunks (skipped when their row is outside the range), the
// rest are the range's rows in order.  CTA-uniform.
template <typename I>
__device__ __forceinline__ bool spl_item(const I* rowptr, const SplArgs& a, const LongRowPlan& plan, int64_t& row,
                                         int64_t& begin, int64_t& end, bool& is_chunk) {
    const int64_t item = blockIdx.x;
    const int64_t it = item < plan.n_chunks ? item : item + a.row_begin;
    if (!decode_item(it, rowptr, a.row_end, plan, row, begin, end, is_chunk)) return false;
    return row >= a.row_begin && row < a.row_end;
}

// Stage edges [e0, e0 + nb): cs[b] = source row, bs[b][s] = basis, ws[b][s] = wi * fin (a slot whose wi lies outside
// [0, K) gets basis 0 and offset 0, so it adds nothing and reads nothing out of bounds).
template <typename T, typename I>
__device__ __forceinline__ void spl_stage(const I* __restrict__ col, const SplArgs& a, int64_t e0, int nb,
                                          int64_t* cs, float* bs, int* ws) {
    const T* basis = static_cast<const T*>(a.basis);
    for (int b = threadIdx.x; b < nb; b += blockDim.x) cs[b] = static_cast<int64_t>(ldg_idx(col + e0 + b));
    for (int idx = threadIdx.x; idx < nb * a.s; idx += blockDim.x) {
        const int b = idx / a.s, s = idx - b * a.s;
        const int64_t slot = spl_eid<I>(a, e0 + b) * a.s + s;
        const int32_t w = __ldg(a.wi + slot);
        const bool ok = w >= 0 && w < a.k;
        bs[idx] = ok ? ElemTraits<T>::to_float(basis[slot]) : 0.0f;
        ws[idx] = ok ? w * static_cast<int>(a.fin) : 0;
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(kSplThreads)
spline_fwd_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, SplArgs a, LongRowPlan plan) {
    extern __shared__ float4 spl_smem[];
    int64_t row, begin, end;
    bool is_chunk;
    if (!spl_item(rowptr, a, plan, row, begin, end, is_chunk)) return;
    const int64_t width = a.k * a.fin;
    const int64_t wpad = (width + 3) & ~static_cast<int64_t>(3);
    float* ps = reinterpret_cast<float*>(spl_smem);
    int64_t* cs = reinterpret_cast<int64_t*>(ps + wpad);
    float* bs = reinterpret_cast<float*>(cs + a.eb);
    int* ws = reinterpret_cast<int*>(bs + a.eb * a.s);
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x) ps[m] = 0.0f;
    const T* x = static_cast<const T*>(a.x);
    for (int64_t e0 = begin; e0 < end; e0 += a.eb) {
        const int nb = static_cast<int>(end - e0 < a.eb ? end - e0 : a.eb);
        __syncthreads();
        spl_stage<T, I>(col, a, e0, nb, cs, bs, ws);
        __syncthreads();
        for (int64_t f = threadIdx.x; f < a.fin; f += blockDim.x) {
            for (int b = 0; b < nb; ++b) {
                const float xv = ElemTraits<T>::to_float(x[cs[b] * a.fin + f]);
                const float* bb = bs + b * a.s;
                const int* wb = ws + b * a.s;
                for (int s = 0; s < a.s; ++s) ps[wb[s] + f] = fmaf(bb[s], xv, ps[wb[s] + f]);
            }
        }
    }
    __syncthreads();
    float* dst = is_chunk ? plan.partials + static_cast<int64_t>(blockIdx.x) * width : a.p + (row - a.row_begin) * width;
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x)
        dst[m] = is_chunk ? ps[m] : finalize<B200MP_SUM>(ps[m], end - begin, a.is_mean, false);
}

// Fold the fp32 partials of every long row of the range in chunk order and write its P row.
template <typename I>
__global__ void __launch_bounds__(256)
spline_combine_kernel(const I* __restrict__ rowptr, SplArgs a, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    if (row < a.row_begin || row >= a.row_end) return;
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const int64_t width = a.k * a.fin;
    float* dst = a.p + (row - a.row_begin) * width;
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x) {
        float acc = 0.0f;
        for (int64_t c = c0; c < c1; ++c) acc = __fadd_rn(acc, plan.partials[c * width + m]);
        dst[m] = finalize<B200MP_SUM>(acc, deg, a.is_mean, false);
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(256)
spline_bwd_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, SplArgs a, LongRowPlan plan) {
    extern __shared__ float4 spl_smem[];
    int64_t row, begin, end;
    bool is_chunk;
    if (!spl_item(rowptr, a, plan, row, begin, end, is_chunk)) return;
    if (begin == end) return;
    const int64_t fin = a.fin, width = a.k * fin;
    const int64_t wpad = (width + 3) & ~static_cast<int64_t>(3);
    float* dps = reinterpret_cast<float*>(spl_smem);
    int64_t* cs = reinterpret_cast<int64_t*>(dps + wpad);
    float* xs = reinterpret_cast<float*>(cs + a.eb);
    float* bs = xs + a.eb * a.fp;
    int* ws = reinterpret_cast<int*>(bs + a.eb * a.s);
    const int64_t deg = static_cast<int64_t>(__ldg(rowptr + row + 1)) - static_cast<int64_t>(__ldg(rowptr + row));
    const float* src = a.dp + (row - a.row_begin) * width;
    for (int64_t m = threadIdx.x; m < width; m += blockDim.x) dps[m] = finalize<B200MP_SUM>(src[m], deg, a.is_mean, false);
    const T* x = static_cast<const T*>(a.x);
    T* gb = static_cast<T*>(a.grad_basis);
    T* q = static_cast<T*>(a.q);
    const int s_out = gb ? a.s : 0;
    const int w_out = s_out + (q ? static_cast<int>(fin) : 0);
    for (int64_t e0 = begin; e0 < end; e0 += a.eb) {
        const int nb = static_cast<int>(end - e0 < a.eb ? end - e0 : a.eb);
        __syncthreads();
        spl_stage<T, I>(col, a, e0, nb, cs, bs, ws);
        __syncthreads();
        for (int idx = threadIdx.x; idx < nb * a.fp; idx += blockDim.x) {
            const int b = idx / a.fp, f = idx - b * a.fp;
            xs[idx] = f < fin ? ElemTraits<T>::to_float(x[cs[b] * fin + f]) : 0.0f;
        }
        __syncthreads();
        for (int o = threadIdx.x; o < nb * w_out; o += blockDim.x) {
            const int b = o / w_out, r = o - b * w_out;
            const int64_t eid = spl_eid<I>(a, e0 + b);
            float acc = 0.0f;
            if (r < s_out) {
                const int32_t w = __ldg(a.wi + eid * a.s + r);
                if (w >= 0 && w < a.k) {                       // a slot outside [0, K) gets gradient 0
                    const float* xr = xs + b * a.fp;
                    const float* dr = dps + ws[b * a.s + r];
                    int f = static_cast<int>(r % fin);
                    for (int t = 0; t < fin; ++t) {
                        acc = fmaf(xr[f], dr[f], acc);
                        f = f + 1 == fin ? 0 : f + 1;
                    }
                }
                gb[eid * a.s + r] = ElemTraits<T>::from_float(acc);
            } else {
                const int f = r - s_out;
                const float* bb = bs + b * a.s;
                const int* wb = ws + b * a.s;
                for (int s = 0; s < a.s; ++s) acc = fmaf(bb[s], dps[wb[s] + f], acc);
                q[eid * fin + f] = ElemTraits<T>::from_float(acc);
            }
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
inline bool spl_s_ok(int64_t s) { return s >= 1 && s <= kSplMaxS; }
inline bool spl_sweep_ok(int64_t k, int64_t fin, int64_t s) {
    return k >= 1 && fin >= 1 && spl_s_ok(s) && k * fin <= kSplMaxWidth;
}

inline int spl_unsupported(const char* what, int64_t k, int64_t fin, int64_t s) {
    set_error("%s: K = %lld, F_in = %lld, S = %lld is outside K >= 1, F_in >= 1, 1 <= S <= %d, K F_in <= %lld", what,
              static_cast<long long>(k), static_cast<long long>(fin), static_cast<long long>(s), kSplMaxS,
              static_cast<long long>(kSplMaxWidth));
    return B200MP_ERR_UNSUPPORTED;
}

inline int spl_basis_shape(int64_t dim, int degree, int64_t& S) {
    if (degree < 1 || degree > 3 || dim < 1) {
        set_error("spline_basis: degree %d, dim %lld is outside degree 1..3, dim >= 1", degree, static_cast<long long>(dim));
        return B200MP_ERR_UNSUPPORTED;
    }
    S = 1;
    for (int64_t d = 0; d < dim && S <= kSplMaxS; ++d) S *= degree + 1;
    if (!spl_s_ok(S)) {
        set_error("spline_basis: (degree + 1)^dim = (%d + 1)^%lld exceeds %d basis slots", degree,
                  static_cast<long long>(dim), kSplMaxS);
        return B200MP_ERR_UNSUPPORTED;
    }
    return B200MP_OK;
}

inline SplArgs spl_args(const void* x, const void* basis, const int32_t* wi, const void* perm, int64_t k, int64_t fin,
                        int64_t s, int64_t row_begin, int64_t row_end, bool is_mean, bool stage_x) {
    SplArgs a{};
    a.x = x; a.basis = basis; a.wi = wi; a.perm = perm; a.k = k; a.fin = fin; a.s = static_cast<int>(s);
    a.row_begin = row_begin; a.row_end = row_end; a.is_mean = is_mean;
    a.fp = static_cast<int>((fin + 3) / 4 * 4);
    // the staging of one edge: its source row, S basis values and S offsets, and (backward) its x row
    const int64_t row_bytes = 8 + 8 * s + (stage_x ? 4 * a.fp : 0);
    const int64_t eb = 16 * 1024 / row_bytes;
    a.eb = static_cast<int>(eb < 1 ? 1 : (eb > kSplMaxBatch ? kSplMaxBatch : eb));
    return a;
}

inline size_t spl_smem_bytes(const SplArgs& a, bool stage_x) {
    const int64_t wpad = (a.k * a.fin + 3) & ~static_cast<int64_t>(3);
    return static_cast<size_t>(wpad) * 4 + static_cast<size_t>(a.eb) * (8 + 8 * a.s + (stage_x ? 4 * a.fp : 0));
}

template <typename Kern>
int spl_smem_opt_in(Kern kernel, size_t smem) {
    if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    return B200MP_OK;
}

inline unsigned spl_blocks(int64_t n, int threads) { return static_cast<unsigned>(ceil_div(n, threads)); }

template <typename T, typename I>
int spl_fwd_typed(const void* rowptr_, const void* col_, SplArgs a, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + (a.row_end - a.row_begin);
    const int64_t t = ceil_div(a.fin, 32) * 32;
    const int threads = static_cast<int>(t < 64 ? 64 : (t > kSplThreads ? kSplThreads : t));
    const size_t smem = spl_smem_bytes(a, false);
    if (int rc = spl_smem_opt_in(spline_fwd_kernel<T, I>, smem)) return rc;
    spline_fwd_kernel<T, I><<<static_cast<unsigned>(items), threads, smem, stream>>>(rowptr, col, a, plan);
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        spline_combine_kernel<I><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, a, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int spl_bwd_typed(const void* rowptr_, const void* col_, SplArgs a, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + (a.row_end - a.row_begin);
    const size_t smem = spl_smem_bytes(a, true);
    if (int rc = spl_smem_opt_in(spline_bwd_kernel<T, I>, smem)) return rc;
    spline_bwd_kernel<T, I><<<static_cast<unsigned>(items), 256, smem, stream>>>(rowptr, col, a, plan);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_spline_supported(int64_t k, int64_t fin, int64_t s, int val_dtype) {
    return (val_dtype == B200MP_F32 || val_dtype == B200MP_BF16) && spl_sweep_ok(k, fin, s);
}

extern "C" int b200mp_spline_basis(const void* pseudo, const int64_t* kernel_size, const uint8_t* is_open_spline,
                                   void* basis, void* weight_index, int64_t n_edges, int64_t dim, int degree,
                                   int val_dtype, int wi_dtype, void* stream) {
    B200MP_CHECK_ARG(n_edges >= 0);
    int64_t S;
    if (int rc = spl_basis_shape(dim, degree, S)) return rc;
    if (n_edges == 0) return B200MP_OK;
    B200MP_CHECK_ARG(pseudo && kernel_size && is_open_spline && basis && weight_index);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned blocks = spl_blocks(n_edges * S, 256);
    return dispatch_val_idx(val_dtype, wi_dtype, "spline_basis", [&](auto tv, auto ti) -> int {
        using T = decltype(tv);
        using W = decltype(ti);
        spline_basis_kernel<T, W><<<blocks, 256, 0, st>>>(static_cast<const T*>(pseudo), kernel_size, is_open_spline,
                                                          static_cast<T*>(basis), static_cast<W*>(weight_index), n_edges,
                                                          static_cast<int>(dim), degree, static_cast<int>(S));
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_spline_basis_backward(const void* grad_basis, const void* pseudo, const int64_t* kernel_size,
                                            const uint8_t* is_open_spline, void* grad_pseudo, int64_t n_edges,
                                            int64_t dim, int degree, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_edges >= 0);
    int64_t S;
    if (int rc = spl_basis_shape(dim, degree, S)) return rc;
    if (n_edges == 0) return B200MP_OK;
    B200MP_CHECK_ARG(grad_basis && pseudo && kernel_size && is_open_spline && grad_pseudo);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned blocks = spl_blocks(n_edges * dim, 256);
    return dispatch_val_idx(val_dtype, B200MP_I64, "spline_basis_backward", [&](auto tv, auto) -> int {
        using T = decltype(tv);
        spline_basis_bwd_kernel<T><<<blocks, 256, 0, st>>>(static_cast<const T*>(grad_basis), static_cast<const T*>(pseudo),
                                                           kernel_size, is_open_spline, static_cast<T*>(grad_pseudo),
                                                           n_edges, static_cast<int>(dim), degree, static_cast<int>(S));
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_spline_weighting(const void* x, const void* weight, const void* basis, const void* weight_index,
                                       void* out, int64_t n_edges, int64_t fin, int64_t fout, int64_t k, int64_t s,
                                       int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_edges >= 0 && fin >= 1 && fout >= 1 && k >= 1);
    if (!spl_s_ok(s)) return spl_unsupported("spline_weighting", k, fin, s);
    if (n_edges == 0) return B200MP_OK;
    B200MP_CHECK_ARG(x && weight && basis && weight_index && out);
    const SwArgs a{x, weight, basis, weight_index, nullptr, n_edges, fin, fout, k, static_cast<int>(s)};
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return dispatch_val_idx(val_dtype, idx_dtype, "spline_weighting", [&](auto tv, auto ti) -> int {
        using T = decltype(tv);
        spline_weighting_fwd_kernel<T, decltype(ti)><<<spl_blocks(n_edges * fout, 256), 256, 0, st>>>(a, static_cast<T*>(out));
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_spline_weighting_backward(const void* grad_out, const void* x, const void* weight,
                                                const void* basis, const void* weight_index, const void* slot_order,
                                                const void* slot_ptr, void* grad_x, void* grad_basis,
                                                float* grad_weight, int64_t n_edges, int64_t fin, int64_t fout,
                                                int64_t k, int64_t s, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_edges >= 0 && fin >= 1 && fout >= 1 && k >= 1);
    if (!spl_s_ok(s)) return spl_unsupported("spline_weighting_backward", k, fin, s);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (grad_weight && n_edges == 0) {
        B200MP_CUDA(cudaMemsetAsync(grad_weight, 0, static_cast<size_t>(k * fin * fout) * sizeof(float), st));
        return B200MP_OK;
    }
    if (n_edges == 0) return B200MP_OK;
    B200MP_CHECK_ARG(grad_out && x && weight && basis && weight_index);
    B200MP_CHECK_ARG(!grad_weight || (slot_order && slot_ptr));
    const SwArgs a{x, weight, basis, weight_index, grad_out, n_edges, fin, fout, k, static_cast<int>(s)};
    return dispatch_val_idx(val_dtype, idx_dtype, "spline_weighting_backward", [&](auto tv, auto ti) -> int {
        using T = decltype(tv);
        using I = decltype(ti);
        if (grad_x) {
            spline_weighting_bwd_x_kernel<T, I><<<spl_blocks(n_edges * fin, 256), 256, 0, st>>>(a, static_cast<T*>(grad_x));
            B200MP_LAUNCH_CHECK();
        }
        if (grad_basis) {
            spline_weighting_bwd_basis_kernel<T, I><<<spl_blocks(n_edges * s, 256), 256, 0, st>>>(
                a, static_cast<T*>(grad_basis));
            B200MP_LAUNCH_CHECK();
        }
        if (grad_weight) {
            const dim3 grid(static_cast<unsigned>(k), spl_blocks(fin * fout, 256));
            spline_weighting_bwd_weight_kernel<T, I><<<grid, 256, 0, st>>>(a, static_cast<const I*>(slot_order),
                                                                             static_cast<const I*>(slot_ptr), grad_weight);
            B200MP_LAUNCH_CHECK();
        }
        return B200MP_OK;
    });
}

extern "C" int b200mp_spline_csr(const void* rowptr, const void* col, const void* perm, const void* x, const void* basis,
                                 const int32_t* weight_index, float* p, int64_t n_rows, int64_t n_cols, int64_t n_edges,
                                 int64_t k, int64_t fin, int64_t s, int64_t row_begin, int64_t row_end, int reduce,
                                 const int64_t* plan_rows, const int64_t* plan_chunk_ptr, int64_t plan_n_long,
                                 int64_t plan_n_chunks, int64_t plan_chunk, float* plan_partials, int idx_dtype,
                                 int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0);
    B200MP_CHECK_ARG(0 <= row_begin && row_begin <= row_end && row_end <= n_rows);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (!spl_sweep_ok(k, fin, s)) return spl_unsupported("spline_csr", k, fin, s);
    LongRowPlan plan;
    if (int rc = make_plan(plan, plan_rows, plan_chunk_ptr, plan_n_long, plan_n_chunks, plan_chunk, plan_partials, true))
        return rc;
    if (row_begin == row_end) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && p);
    B200MP_CHECK_ARG(n_edges == 0 || (col && x && basis && weight_index));
    SplArgs a = spl_args(x, basis, weight_index, perm, k, fin, s, row_begin, row_end, reduce == B200MP_MEAN, false);
    a.p = p;
    return dispatch_val_idx(val_dtype, idx_dtype, "spline_csr", [&](auto tv, auto ti) {
        return spl_fwd_typed<decltype(tv), decltype(ti)>(rowptr, col, a, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_spline_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                          const void* basis, const int32_t* weight_index, const float* grad_p,
                                          void* grad_basis, void* q, int64_t n_rows, int64_t n_cols, int64_t n_edges,
                                          int64_t k, int64_t fin, int64_t s, int64_t row_begin, int64_t row_end,
                                          int reduce, const int64_t* plan_rows, const int64_t* plan_chunk_ptr,
                                          int64_t plan_n_long, int64_t plan_n_chunks, int64_t plan_chunk,
                                          int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0);
    B200MP_CHECK_ARG(0 <= row_begin && row_begin <= row_end && row_end <= n_rows);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (!spl_sweep_ok(k, fin, s)) return spl_unsupported("spline_backward_dst", k, fin, s);
    LongRowPlan plan;
    if (int rc = make_plan(plan, plan_rows, plan_chunk_ptr, plan_n_long, plan_n_chunks, plan_chunk, nullptr, false))
        return rc;
    if (row_begin == row_end || n_edges == 0 || (grad_basis == nullptr && q == nullptr)) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && col && x && basis && weight_index && grad_p);
    SplArgs a = spl_args(x, basis, weight_index, perm, k, fin, s, row_begin, row_end, reduce == B200MP_MEAN, true);
    a.dp = grad_p;
    a.grad_basis = grad_basis;
    a.q = q;
    return dispatch_val_idx(val_dtype, idx_dtype, "spline_backward_dst", [&](auto tv, auto ti) {
        return spl_bwd_typed<decltype(tv), decltype(ti)>(rowptr, col, a, plan, static_cast<cudaStream_t>(stream));
    });
}
