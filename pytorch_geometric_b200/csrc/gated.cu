// gated.cu -- ResGatedGraphConv's gated message sigmoid(k_i + q_j) * v_j fused into the CSR gather-reduce, and its
// backward.
//
//   out[i,:] = REDUCE_{e in [rowptr[i], rowptr[i+1])} sigma(s_e) * v[col[e],:]        REDUCE = sum | mean
//   s_e      = k[i,:] + q[col[e],:], rounded to the storage dtype (the reference adds in that dtype)
//
// The forward rounds sigma and then the product to the storage dtype, as the reference's sigmoid and mul do, and
// accumulates in fp32 in CSR order.  Nothing per edge is stored: the backward recomputes s from k and q.
//   grad_k[i,:] = g_i * sum_{e in row i} v[col[e],:] * sigma'(s_e)                          (destination CSR)
//   grad_v[j,:] = sum_{t in rowT(j)} sigma(s_t) * g_t,  grad_q[j,:] = v[j,:] * sum_t sigma'(s_t) * g_t  (transposed CSR)
// with g_i = grad_out[i,:] / (mean ? max(deg_i, 1) : 1) (val_t carries the 1 / deg on the transposed sweep).
//
// Sigmoid numerics: t = exp(-|s|) by __expf (ex2.approx), r = 1 / (1 + t) by __fdividef (rcp.approx): two MUFU
// operations per element.  sigma = s >= 0 ? r : t * r and sigma' = t * r * r -- never sigma * (1 - sigma), which
// cancels at large |s| and loses sigma' there.  s = +inf gives sigma = 1, sigma' = 0; s = -inf gives 0, 0; NaN stays
// NaN (s >= 0 is false, t = NaN); 0 * inf products give NaN as in the reference.
//
// q and v (and grad_q, grad_v) share one row stride `ld` in elements, so they can be two [N, F] tensors or the two
// halves of one [N, 2F] product; k, grad_out, out and grad_k are [N, F] with stride F.
//
// Mapping as in csr_reduce.cuh / edge_relu.cu: a lane group of G lanes per row, VPL 16-byte vectors per lane, rows
// longer than the plan's chunk split into chunks whose fp32 partials gated_combine_kernel folds in chunk order (the
// row-wise factor g_i or v[j] is applied after the fold).  Rows that are not a whole number of aligned 16-byte vectors
// take a one-warp scalar kernel.
#include "csr_reduce.cuh"
#include "gate_math.cuh"

namespace b200mp {

enum GatedMode { kGatedFwd = 0, kGatedDst = 1, kGatedSrc = 2 };

struct GatedArgs {
    const void* k;       // [n_dst, feat]
    const void* q;       // [n_src, ld]
    const void* v;       // [n_src, ld]
    const void* g;       // grad_out [n_dst, feat] (backward)
    const float* val_t;  // per transposed slot, 1 / max(deg_dst, 1) for mean (source sweep), or null
    void* out0;          // fwd: out [n_dst, feat]; dst: grad_k [n_dst, feat]; src: grad_v [n_src, ld]
    void* out1;          // src: grad_q [n_src, ld]
    int64_t feat;
    int64_t ld;
    bool is_mean;
};

// One (edge, feature) term.  fwd / dst: a = q[j], b = v[j], rowop = k[i]; src: a = k[i], b = g[i] (times w), rowop = q[j].
template <typename T, int MODE>
__device__ __forceinline__ void gated_term(float rowop, float a, float b, float w, bool weighted, float& acc0,
                                           float& acc1) {
    const float s = round_to<T>(__fadd_rn(rowop, a));
    float sig, dsig;
    sigmoid_pair(s, sig, dsig);
    if (MODE == kGatedFwd) {
        acc0 = __fadd_rn(acc0, round_to<T>(__fmul_rn(round_to<T>(sig), b)));
    } else if (MODE == kGatedDst) {
        acc0 = __fadd_rn(acc0, __fmul_rn(b, dsig));
    } else {
        const float gw = weighted ? __fmul_rn(w, b) : b;
        acc0 = __fadd_rn(acc0, __fmul_rn(sig, gw));
        acc1 = __fadd_rn(acc1, __fmul_rn(dsig, gw));
    }
}

// The finished value of output o (0 / 1) at (row, f) from the fp32 sums; `mul` is the row-wise factor: g[row, f]
// (dst) or v[row, f] (src, output 1).  A row without edges gets 0 even where the factor is inf or NaN: the reference
// adds no term there.
template <int MODE>
__device__ __forceinline__ float gated_finish(int o, float acc, float mul, int64_t deg, bool is_mean) {
    if (MODE == kGatedFwd) return finalize<B200MP_SUM>(acc, deg, is_mean, false);
    if (deg == 0) return 0.0f;
    if (MODE == kGatedDst) return __fmul_rn(finalize<B200MP_SUM>(mul, deg, is_mean, false), acc);
    return o == 0 ? acc : __fmul_rn(mul, acc);
}

// Element pointers of the four operands by role: the row operand, the two gathered operands, the row-wise factor.
template <typename T, int MODE>
struct GatedRoles {
    const T *row, *ga, *gb, *mul;
    int64_t row_ld, g_ld, mul_ld, out_ld;
    __device__ __forceinline__ explicit GatedRoles(const GatedArgs& a) {
        const T* k = static_cast<const T*>(a.k);
        const T* q = static_cast<const T*>(a.q);
        const T* v = static_cast<const T*>(a.v);
        const T* g = static_cast<const T*>(a.g);
        if (MODE == kGatedSrc) {
            row = q; row_ld = a.ld; ga = k; gb = g; g_ld = a.feat; mul = v; mul_ld = a.ld; out_ld = a.ld;
        } else {
            row = k; row_ld = a.feat; ga = q; gb = v; g_ld = a.ld; mul = g; mul_ld = a.feat; out_ld = a.feat;
        }
    }
};

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int G, int VPL, int UNR>
__global__ void __launch_bounds__(128)
gated_reduce_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, GatedArgs args, int64_t n_rows,
                    int n_vec, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int NACC = MODE == kGatedSrc ? 2 : 1;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // uniform per group
    const GatedRoles<T, MODE> R(args);
    const size_t g_bytes = static_cast<size_t>(R.g_ld) * sizeof(T);
    const char* gab = reinterpret_cast<const char*>(R.ga);
    const char* gbb = reinterpret_cast<const char*>(R.gb);
    const bool weighted = MODE == kGatedSrc && args.val_t != nullptr;

    for (int vbase = 0; vbase < n_vec; vbase += G * VPL) {
        float acc[NACC][VPL][EPV], rop[VPL][EPV];
        bool vvalid[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int v = vbase + lig + k * G;
            vvalid[k] = v < n_vec;
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                rop[k][i] = 0.0f;
#pragma unroll
                for (int o = 0; o < NACC; ++o) acc[o][k][i] = 0.0f;
            }
            if (vvalid[k])
                ElemTraits<T>::unpack(ldg_stream16(R.row + row * R.row_ld + static_cast<int64_t>(v) * EPV), rop[k]);
        }
        const size_t voff = static_cast<size_t>(vbase + lig) * 16;
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 av[UNR][VPL], bv[UNR][VPL];
            float w[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                w[u] = 1.0f;
                if (e + u < end) {
                    const int64_t c = static_cast<int64_t>(ldg_idx(col + e + u));
                    if (weighted) w[u] = __ldg(args.val_t + e + u);
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (vvalid[k]) {
                            av[u][k] = ldg_row16(gab + c * g_bytes + voff + static_cast<size_t>(k) * G * 16);
                            bv[u][k] = ldg_row16(gbb + c * g_bytes + voff + static_cast<size_t>(k) * G * 16);
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (vvalid[k]) {
                            float fa[EPV], fb[EPV];
                            ElemTraits<T>::unpack(av[u][k], fa);
                            ElemTraits<T>::unpack(bv[u][k], fb);
#pragma unroll
                            for (int i = 0; i < EPV; ++i)
                                gated_term<T, MODE>(rop[k][i], fa[i], fb[i], w[u], weighted, acc[0][k][i],
                                                    acc[NACC - 1][k][i]);
                        }
                    }
                }
            }
        }
        const int64_t deg = end - begin;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (!vvalid[k]) continue;
            const int v = vbase + lig + k * G;
            if (is_chunk) {
#pragma unroll
                for (int o = 0; o < NACC; ++o)
                    store_partial<EPV>(plan.partials + (static_cast<size_t>(item * NACC + o) * n_vec + v) * EPV, acc[o][k]);
                continue;
            }
            float mul[EPV];
            if (MODE != kGatedFwd)
                ElemTraits<T>::unpack(ldg_stream16(R.mul + row * R.mul_ld + static_cast<int64_t>(v) * EPV), mul);
#pragma unroll
            for (int o = 0; o < NACC; ++o) {
                float f[EPV];
#pragma unroll
                for (int i = 0; i < EPV; ++i) f[i] = gated_finish<MODE>(o, acc[o][k][i], MODE == kGatedFwd ? 0.0f : mul[i], deg, args.is_mean);
                T* out = static_cast<T*>(o == 0 ? args.out0 : args.out1);
                stg_stream16(out + row * R.out_ld + static_cast<int64_t>(v) * EPV, ElemTraits<T>::pack(f));
            }
        }
    }
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE>
__global__ void __launch_bounds__(256)
gated_reduce_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, GatedArgs args, int64_t n_rows,
                           LongRowPlan plan) {
    constexpr int NACC = MODE == kGatedSrc ? 2 : 1;
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // warp-uniform
    const GatedRoles<T, MODE> R(args);
    const int64_t feat = args.feat;
    const bool weighted = MODE == kGatedSrc && args.val_t != nullptr;
    for (int64_t f = lane; f < feat; f += 32) {
        const float rop = ElemTraits<T>::to_float(R.row[row * R.row_ld + f]);
        float acc0 = 0.0f, acc1 = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            gated_term<T, MODE>(rop, ElemTraits<T>::to_float(R.ga[c * R.g_ld + f]),
                                ElemTraits<T>::to_float(R.gb[c * R.g_ld + f]), weighted ? __ldg(args.val_t + e) : 1.0f,
                                weighted, acc0, acc1);
        }
        if (is_chunk) {
            plan.partials[(item * NACC) * feat + f] = acc0;
            if (NACC == 2) plan.partials[(item * NACC + 1) * feat + f] = acc1;
            continue;
        }
        const float mul = MODE == kGatedFwd ? 0.0f : ElemTraits<T>::to_float(R.mul[row * R.mul_ld + f]);
        static_cast<T*>(args.out0)[row * R.out_ld + f] =
            ElemTraits<T>::from_float(gated_finish<MODE>(0, acc0, mul, end - begin, args.is_mean));
        if (NACC == 2)
            static_cast<T*>(args.out1)[row * R.out_ld + f] =
                ElemTraits<T>::from_float(gated_finish<MODE>(1, acc1, mul, end - begin, args.is_mean));
    }
}

// Fold the fp32 partials of every long row in chunk order, then apply the row-wise factor and write the row.
template <typename T, typename I, int MODE>
__global__ void __launch_bounds__(256)
gated_combine_kernel(const I* __restrict__ rowptr, GatedArgs args, LongRowPlan plan) {
    constexpr int NACC = MODE == kGatedSrc ? 2 : 1;
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const GatedRoles<T, MODE> R(args);
    const int64_t feat = args.feat;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        const float mul = MODE == kGatedFwd ? 0.0f : ElemTraits<T>::to_float(R.mul[row * R.mul_ld + f]);
#pragma unroll
        for (int o = 0; o < NACC; ++o) {
            float acc = 0.0f;
            for (int64_t c = c0; c < c1; ++c) acc = __fadd_rn(acc, plan.partials[(c * NACC + o) * feat + f]);
            static_cast<T*>(o == 0 ? args.out0 : args.out1)[row * R.out_ld + f] =
                ElemTraits<T>::from_float(gated_finish<MODE>(o, acc, mul, deg, args.is_mean));
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
template <typename T, int MODE>
bool gated_vec_ok(const GatedArgs& a, const LongRowPlan& plan) {
    return (a.feat * sizeof(T)) % 16 == 0 && (a.ld * sizeof(T)) % 16 == 0 && aligned16(a.k) && aligned16(a.q) &&
           aligned16(a.v) && aligned16(a.out0) && (MODE == kGatedFwd || aligned16(a.g)) &&
           (MODE != kGatedSrc || aligned16(a.out1)) && (plan.n_chunks == 0 || aligned16(plan.partials));
}

template <typename T, typename I, int MODE>
int gated_typed(const void* rowptr_, const void* col_, GatedArgs args, int64_t n_rows, LongRowPlan plan,
                cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + n_rows;
    if (gated_vec_ok<T, MODE>(args, plan)) {
        const int n_vec = static_cast<int>(args.feat * sizeof(T) / 16);
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            gated_reduce_kernel<T, I, MODE, G(), VPL(), unroll_for_vpl<VPL()>()>
                <<<static_cast<unsigned>(ceil_div(items, 128 / G())), 128, 0, stream>>>(rowptr, col, args, n_rows, n_vec,
                                                                                       plan);
        });
    } else {
        gated_reduce_scalar_kernel<T, I, MODE><<<static_cast<unsigned>(ceil_div(items, 8)), 256, 0, stream>>>(
            rowptr, col, args, n_rows, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        gated_combine_kernel<T, I, MODE><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, args, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_gated_csr(const void* rowptr, const void* col, const void* k, const void* q, const void* v,
                                void* out, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld,
                                int reduce, const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0 && ld >= feat);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && k && out);
    B200MP_CHECK_ARG(n_edges == 0 || (col && q && v));
    const GatedArgs a{k, q, v, nullptr, nullptr, out, nullptr, feat, ld, reduce == B200MP_MEAN};
    return dispatch_val_idx(val_dtype, idx_dtype, "gated_csr", [&](auto tv, auto ti) {
        return gated_typed<decltype(tv), decltype(ti), kGatedFwd>(rowptr, col, a, n_rows, plan,
                                                                static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_gated_backward_dst(const void* rowptr, const void* col, const void* k, const void* q,
                                         const void* v, const void* grad_out, void* grad_k, int64_t n_rows,
                                         int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld, int reduce,
                                         const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                         int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype,
                                         int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0 && ld >= feat);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && k && grad_out && grad_k);
    B200MP_CHECK_ARG(n_edges == 0 || (col && q && v));
    const GatedArgs a{k, q, v, grad_out, nullptr, grad_k, nullptr, feat, ld, reduce == B200MP_MEAN};
    return dispatch_val_idx(val_dtype, idx_dtype, "gated_backward_dst", [&](auto tv, auto ti) {
        return gated_typed<decltype(tv), decltype(ti), kGatedDst>(rowptr, col, a, n_rows, plan,
                                                                static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_gated_backward_src(const void* rowptr_t, const void* col_t, const float* val_t, const void* k,
                                         const void* q, const void* v, const void* grad_out, void* grad_q,
                                         void* grad_v, int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t feat,
                                         int64_t ld, const int64_t* long_rows, const int64_t* chunk_ptr,
                                         int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                         int idx_dtype, int val_dtype, void* stream) {
    const int64_t n_rows = n_src, n_cols = n_dst;
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0 && ld >= feat);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && q && v && grad_q && grad_v);
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && k && grad_out));
    const GatedArgs a{k, q, v, grad_out, val_t, grad_v, grad_q, feat, ld, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "gated_backward_src", [&](auto tv, auto ti) {
        return gated_typed<decltype(tv), decltype(ti), kGatedSrc>(rowptr_t, col_t, a, n_src, plan,
                                                                static_cast<cudaStream_t>(stream));
    });
}
