// softmax_aggr.cu -- SoftmaxAggregation (and GENConv's message relu(x_j + e_ji) + eps in front of it) as one
// online-softmax sweep over the destination CSR, and its backward.
//
// Per destination i, feature f and in-edge e = (j -> i), eid(e) = perm[e] (CSR slot -> the caller's edge id) or e:
//   s_e = round(x[j] + a[eid(e)])  |  x[j]  |  a[eid(e)]            (which of x / a are present: template FORM)
//   m_e = round(relu(s_e) + eps)  or  s_e                            (relu keeps NaN)
//   z_e = round(t_f * m_e)  or  m_e                   (t fp32: none, t[0] or t[f]: template TMODE; a Python-number t
//                                                      is multiplied at fp32, as ATen does, and only z is rounded)
//   out_i = sum_e p_e m_e,  p_e = exp(z_e - M) / (sum_e exp(z_e - M) + 1e-16),  M = max_e z_e;  empty row -> 0
// The sweep keeps a running (M, S, A) per element and spends ONE exponential per (edge, feature): with d = z - M and
// q = exp(-|d|), a new maximum rescales the state by q and adds 1 (S) / m (A), anything else adds q / q m, with
// compensated (Kahan) sums so that long rows keep lse to a few ulp.  The only
// saved state is lse = M + log(S + 1e-16), one fp32 [n_rows, F] plane.  As in the reference, a row whose maximum is
// +inf gives NaN (z - M = inf - inf), as does a non-empty row whose z are all -inf; a z of -inf next to a finite
// maximum adds exp(-inf) = 0 wherever it sits in the row, and 0 * inf products give NaN.
//
// Backward, with g = grad_out[i], o = out[i], p_e = exp(z_e - lse_i) (the 1e-16 is below fp32 resolution there):
//   grad_m = g p (1 + t (m - o))   (g p with semi_grad: the softmax was computed without a gradient)
//   grad_t = sum_i sum_e g p m (m - o)          per-CTA fp32 partials folded by b200mp_column_sum
//   grad_s = grad_m [s > 0 or NaN]  (relu form; threshold_backward's rule)
// The destination sweep writes grad_s into grad_a in the caller's edge order and the grad_t partials; the transposed
// sweep sums grad_s over a source's out-edges into grad_x when no grad_a was written.
//
// Mapping as in cg.cu: a lane group of G lanes per row (runtime power of two), one 16-byte vector per lane and trip,
// rows longer than the plan's chunk split into chunks whose fp32 partials a combine kernel folds in chunk order.
// Rows that are not a whole number of aligned 16-byte vectors take a one-warp scalar kernel.
#include "gate_math.cuh"
#include "param_aggr.cuh"

namespace b200mp {

template <typename T, int TMODE>
__device__ __forceinline__ float sm_logit(float m, float tv) {
    return TMODE == kParamNone ? m : round_to<T>(__fmul_rn(tv, m));
}

// Compensated (Kahan) add: the running sum is s - c.  A hub row adds hundreds of terms of one sign in sequence, whose
// plain fp32 sum drifts by about n * 2^-26 relative -- enough to move lse, and with it every p of the backward.
__device__ __forceinline__ void sm_kahan(float& s, float& c, float v) {
    const float y = __fsub_rn(v, c);
    const float t = __fadd_rn(s, y);
    c = __fsub_rn(__fsub_rn(t, s), y);
    s = t;
}

// One online-softmax step: one exponential.  z = -inf adds q = 0 even while M is still -inf (d = NaN there).
__device__ __forceinline__ void sm_push(float z, float m, float& M, float& S, float& A, float& cS, float& cA) {
    const float d = z - M;
    const float q = z == -INFINITY ? 0.0f : __expf(-fabsf(d));
    if (d > 0.0f) {
        S = fmaf(__fsub_rn(S, cS), q, 1.0f);
        A = fmaf(__fsub_rn(A, cA), q, m);
        cS = cA = 0.0f;
        M = z;
    } else {
        sm_kahan(S, cS, q);
        sm_kahan(A, cA, __fmul_rn(q, m));
    }
}

// Merge state (M2, S2, A2) into (M, S, A), also with one exponential; a part whose z were all -inf adds nothing.
__device__ __forceinline__ void sm_merge(float M2, float S2, float A2, float& M, float& S, float& A) {
    const float d = M2 - M;
    const float q = M2 == -INFINITY ? 0.0f : __expf(-fabsf(d));
    if (d > 0.0f) {
        S = fmaf(S, q, S2);
        A = fmaf(A, q, A2);
        M = M2;
    } else {
        S = fmaf(S2, q, S);
        A = fmaf(A2, q, A);
    }
}

// `any`: the row has edges (an empty row gives 0; a non-empty one whose maximum is -inf or +inf gives NaN).
__device__ __forceinline__ void sm_final(float M, float S, float A, bool any, float& out, float& lse) {
    const float den = __fadd_rn(S, 1e-16f);
    const bool bad = M == INFINITY || (any && M == -INFINITY);
    out = bad ? __int_as_float(0x7fffffff) : __fdiv_rn(A, den);
    lse = bad ? __int_as_float(0x7fffffff) : __fadd_rn(M, logf(den));
}

// Backward term of one (edge, feature): returns grad_s, adds the grad_t term to gt.
template <int FORM, int TMODE, bool WANT_T>
__device__ __forceinline__ float sm_grad(float z, float m, bool on, float tv, float g, float o, float lse, bool semi,
                                         float& gt) {
    const float p = __expf(z - lse);
    const float gp = __fmul_rn(g, p);
    const float dm = __fsub_rn(m, o);
    if (WANT_T) gt = fmaf(__fmul_rn(gp, m), dm, gt);
    float gm = gp;
    if (!semi) gm = __fmul_rn(gp, fmaf(TMODE == kParamNone ? 1.0f : tv, dm, 1.0f));
    return (SmForms<FORM>::kRelu && !on) ? 0.0f : gm;
}

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
__global__ void __launch_bounds__(128)
softmax_aggr_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AggrArgs args, int64_t n_rows, int n_vec,
                    int lg, LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    constexpr int EPV = ElemTraits<T>::kPerVec;
    // bf16 backward: fewer edges in flight, so that the per-row operands stay in registers
    constexpr int UNR = (MODE == kSweepFwd || sizeof(T) == 4) ? 4 : ((WANT_T || TMODE == kParamChannel) ? 1 : 2);
    extern __shared__ float sm_sh[];
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = aggr_item<WANT_T>(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // uniform per group
    if (!active && !WANT_T) return;
    const int64_t F = args.feat;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = static_cast<const char*>(args.x);
    const char* ab = static_cast<const char*>(args.a);
    const char* gb = static_cast<const char*>(args.g);
    const char* ob = static_cast<const char*>(args.o);
    float ts = 1.0f;
    if (TMODE == kParamScalar) ts = __ldg(args.param);

    for (int vi = lig; vi < n_vec; vi += G) {
        const size_t voff = static_cast<size_t>(vi) * 16;
        const int64_t f0 = static_cast<int64_t>(vi) * EPV;
        float tv[EPV], rx[EPV], rg[EPV], ro[EPV], rl[EPV];
        float acc0[EPV], acc1[EPV], acc2[EPV], c1[EPV], c2[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            tv[i] = ts;
            rx[i] = rg[i] = ro[i] = rl[i] = 0.0f;
            acc0[i] = MODE == kSweepFwd ? -INFINITY : 0.0f;
            acc1[i] = acc2[i] = c1[i] = c2[i] = 0.0f;
        }
        if (TMODE == kParamChannel) ldg_f32(args.param + f0, tv);
        {
            if (MODE == kSweepDst) {
                ElemTraits<T>::unpack(ldg_stream16(gb + row * row_bytes + voff), rg);
                ElemTraits<T>::unpack(ldg_stream16(ob + row * row_bytes + voff), ro);
                ldg_f32(args.saved + row * F + f0, rl);
            }
            if (MODE == kSweepSrc) ElemTraits<T>::unpack(ldg_stream16(xb + row * row_bytes + voff), rx);
        }
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 xv[UNR], av[UNR], gv[UNR], ov[UNR];
            float4 lv[UNR][EPV / 4];
            int64_t id[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                id[u] = 0;
                if (e + u < end) {
                    const int64_t c = static_cast<int64_t>(ldg_idx(col + e + u));
                    if (Fm::kA || (MODE == kSweepDst && args.out)) id[u] = aggr_eid<I>(args, e + u);
                    if (MODE != kSweepSrc && Fm::kX) xv[u] = ldg_row16(xb + c * row_bytes + voff);
                    if (Fm::kA) av[u] = ldg_stream16(ab + id[u] * row_bytes + voff);
                    if (MODE == kSweepSrc) {
                        gv[u] = ldg_row16(gb + c * row_bytes + voff);
                        ov[u] = ldg_row16(ob + c * row_bytes + voff);
                        const float4* lp = reinterpret_cast<const float4*>(args.saved + c * F + f0);
#pragma unroll
                        for (int q = 0; q < EPV / 4; ++q) lv[u][q] = __ldg(lp + q);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float fx[EPV], fa[EPV], fg[EPV], fo[EPV], fl[EPV], gs[EPV];
                    if (MODE == kSweepSrc) {
#pragma unroll
                        for (int i = 0; i < EPV; ++i) fx[i] = rx[i];
                        ElemTraits<T>::unpack(gv[u], fg);
                        ElemTraits<T>::unpack(ov[u], fo);
#pragma unroll
                        for (int q = 0; q < EPV / 4; ++q) {
                            fl[4 * q] = lv[u][q].x; fl[4 * q + 1] = lv[u][q].y;
                            fl[4 * q + 2] = lv[u][q].z; fl[4 * q + 3] = lv[u][q].w;
                        }
                    } else if (Fm::kX) {
                        ElemTraits<T>::unpack(xv[u], fx);
                    }
                    if (Fm::kA) ElemTraits<T>::unpack(av[u], fa);
#pragma unroll
                    for (int i = 0; i < EPV; ++i) {
                        bool on;
                        const float m = sm_message<T, FORM>(fx[i], Fm::kA ? fa[i] : 0.0f, args.eps, on);
                        const float z = sm_logit<T, TMODE>(m, tv[i]);
                        if (MODE == kSweepFwd) {
                            sm_push(z, m, acc0[i], acc1[i], acc2[i], c1[i], c2[i]);
                        } else if (MODE == kSweepDst) {
                            gs[i] = sm_grad<FORM, TMODE, WANT_T>(z, m, on, tv[i], rg[i], ro[i], rl[i], args.semi, acc0[i]);
                        } else {
                            float unused = 0.0f;
                            acc0[i] = __fadd_rn(acc0[i], sm_grad<FORM, TMODE, false>(z, m, on, tv[i], fg[i], fo[i], fl[i],
                                                                                    args.semi, unused));
                        }
                    }
                    if (MODE == kSweepDst && args.out)
                        stg_stream16(static_cast<char*>(args.out) + id[u] * row_bytes + voff, ElemTraits<T>::pack(gs));
                }
            }
        }
        if (MODE == kSweepFwd) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                acc1[i] = __fsub_rn(acc1[i], c1[i]);
                acc2[i] = __fsub_rn(acc2[i], c2[i]);
            }
        }
        if (MODE == kSweepDst) {
            if (WANT_T) {
                float* sh = sm_sh + static_cast<int64_t>(threadIdx.x >> lg) * F + f0;
#pragma unroll
                for (int i = 0; i < EPV; ++i) sh[i] = acc0[i];
            }
            continue;
        }
        if (is_chunk) {
            constexpr int NACC = MODE == kSweepFwd ? 3 : 1;
            store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC) * F + f0, acc0);
            if (MODE == kSweepFwd) {
                store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC + 1) * F + f0, acc1);
                store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC + 2) * F + f0, acc2);
            }
            continue;
        }
        char* dst = static_cast<char*>(args.out) + row * row_bytes + voff;
        if (MODE == kSweepFwd) {
            float f[EPV], l[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i) sm_final(acc0[i], acc1[i], acc2[i], end > begin, f[i], l[i]);
            stg_stream16(dst, ElemTraits<T>::pack(f));
            if (args.saved) store_partial<EPV>(args.saved + row * F + f0, l);
        } else {
            stg_stream16(dst, ElemTraits<T>::pack(acc0));
        }
    }
    if (MODE == kSweepDst && WANT_T) store_param_part(sm_sh, blockDim.x >> lg, F, args.param_part);
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
__global__ void __launch_bounds__(256)
softmax_aggr_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AggrArgs args, int64_t n_rows,
                           LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    extern __shared__ float sm_sh[];
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = aggr_item<WANT_T>(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // warp-uniform
    if (!active && !WANT_T) return;
    const int64_t F = args.feat;
    const T* x = static_cast<const T*>(args.x);
    const T* a = static_cast<const T*>(args.a);
    const T* g = static_cast<const T*>(args.g);
    const T* o = static_cast<const T*>(args.o);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = lane; f < F; f += 32) {
        const float tv = TMODE == kParamNone ? 1.0f : __ldg(args.param + (TMODE == kParamChannel ? f : 0));
        float acc0 = MODE == kSweepFwd ? -INFINITY : 0.0f, acc1 = 0.0f, acc2 = 0.0f, c1 = 0.0f, c2 = 0.0f;
        float rx = 0.0f, rg = 0.0f, ro = 0.0f, rl = 0.0f;
        if (MODE == kSweepDst) {
            rg = ElemTraits<T>::to_float(g[row * F + f]);
            ro = ElemTraits<T>::to_float(o[row * F + f]);
            rl = args.saved[row * F + f];
        }
        if (MODE == kSweepSrc) rx = ElemTraits<T>::to_float(x[row * F + f]);
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t id = (Fm::kA || (MODE == kSweepDst && out)) ? aggr_eid<I>(args, e) : 0;
            const float xv = MODE == kSweepSrc ? rx : (Fm::kX ? ElemTraits<T>::to_float(x[c * F + f]) : 0.0f);
            const float av = Fm::kA ? ElemTraits<T>::to_float(a[id * F + f]) : 0.0f;
            bool on;
            const float m = sm_message<T, FORM>(xv, av, args.eps, on);
            const float z = sm_logit<T, TMODE>(m, tv);
            if (MODE == kSweepFwd) {
                sm_push(z, m, acc0, acc1, acc2, c1, c2);
            } else if (MODE == kSweepDst) {
                const float gs = sm_grad<FORM, TMODE, WANT_T>(z, m, on, tv, rg, ro, rl, args.semi, acc0);
                if (out) out[id * F + f] = ElemTraits<T>::from_float(gs);
            } else {
                float unused = 0.0f;
                acc0 = __fadd_rn(acc0, sm_grad<FORM, TMODE, false>(z, m, on, tv, ElemTraits<T>::to_float(g[c * F + f]),
                                                                  ElemTraits<T>::to_float(o[c * F + f]),
                                                                  args.saved[c * F + f], args.semi, unused));
            }
        }
        if (MODE == kSweepFwd) {
            acc1 = __fsub_rn(acc1, c1);
            acc2 = __fsub_rn(acc2, c2);
        }
        if (MODE == kSweepDst) {
            if (WANT_T) sm_sh[(threadIdx.x >> 5) * F + f] = acc0;
            continue;
        }
        if (is_chunk) {
            if (MODE == kSweepFwd) {
                plan.partials[(item * 3) * F + f] = acc0;
                plan.partials[(item * 3 + 1) * F + f] = acc1;
                plan.partials[(item * 3 + 2) * F + f] = acc2;
            } else {
                plan.partials[item * F + f] = acc0;
            }
            continue;
        }
        if (MODE == kSweepFwd) {
            float ov, l;
            sm_final(acc0, acc1, acc2, end > begin, ov, l);
            out[row * F + f] = ElemTraits<T>::from_float(ov);
            if (args.saved) args.saved[row * F + f] = l;
        } else {
            out[row * F + f] = ElemTraits<T>::from_float(acc0);
        }
    }
    if (MODE == kSweepDst && WANT_T) store_param_part(sm_sh, blockDim.x >> 5, F, args.param_part);
}

// Merge the (M, S, A) partials of every long row in chunk order and write out and lse.
template <typename T>
__global__ void __launch_bounds__(256)
softmax_aggr_combine_kernel(AggrArgs args, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t F = args.feat;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    T* out = static_cast<T*>(args.out);
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
        float M = -INFINITY, S = 0.0f, A = 0.0f;
        for (int64_t c = c0; c < c1; ++c) {
            const float* p = plan.partials + c * 3 * F + f;
            if (c == c0) {
                M = p[0]; S = p[F]; A = p[2 * F];
            } else {
                sm_merge(p[0], p[F], p[2 * F], M, S, A);
            }
        }
        float ov, l;
        sm_final(M, S, A, true, ov, l);
        out[row * F + f] = ElemTraits<T>::from_float(ov);
        if (args.saved) args.saved[row * F + f] = l;
    }
}

struct SoftmaxAggrOp {
    static constexpr const char* kName = "softmax_aggr";
    static constexpr const char* kParam = "t";
    static constexpr bool collects(int mode) { return mode == kSweepDst; }
    template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
    static auto vec() { return softmax_aggr_kernel<T, I, MODE, FORM, TMODE, WANT_T>; }
    template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
    static auto scalar() { return softmax_aggr_scalar_kernel<T, I, MODE, FORM, TMODE, WANT_T>; }
    template <typename T, typename I, int TMODE>
    static void combine(const I*, const AggrArgs& args, const LongRowPlan& plan, cudaStream_t s) {
        softmax_aggr_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), 256, 0, s>>>(args, plan);
    }
};

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_softmax_aggr_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                       const void* edge_rows, const float* t, void* out, float* lse, int64_t n_rows,
                                       int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps,
                                       int t_mode, const int64_t* long_rows, const int64_t* chunk_ptr,
                                       int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                       int idx_dtype, int val_dtype, void* stream) {
    if (int rc = check_aggr_args(n_rows, n_cols, n_edges, feat, message, x, edge_rows, t_mode, t, false, 0, 0)) return rc;
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const AggrArgs a{x, edge_rows, t, perm, nullptr, nullptr, lse, nullptr, out, nullptr, feat, eps, 0, 0, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_csr", [&](auto tv, auto ti) {
        return aggr_sweep<SoftmaxAggrOp, decltype(tv), decltype(ti), kSweepFwd>(
            rowptr, col, a, sm_form(x, edge_rows, message), t_mode, n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int64_t b200mp_softmax_aggr_workspace(int64_t n_rows, int64_t n_chunks, int64_t feat) {
    return b200mp_power_mean_workspace(0, n_rows, n_chunks, feat);
}

extern "C" int b200mp_softmax_aggr_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                                const void* edge_rows, const float* t, const void* out,
                                                const float* lse, const void* grad_out, void* grad_edge_rows,
                                                float* grad_t, float* workspace, int64_t n_rows, int64_t n_cols,
                                                int64_t n_edges, int64_t feat, int message, float eps, int t_mode,
                                                int semi_grad, const int64_t* long_rows, const int64_t* chunk_ptr,
                                                int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype,
                                                int val_dtype, void* stream) {
    if (int rc = check_aggr_args(n_rows, n_cols, n_edges, feat, message, x, edge_rows, t_mode, t, false, 0, 0)) return rc;
    B200MP_CHECK_ARG(grad_t == nullptr || (t_mode != 0 && workspace));
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, nullptr, false)) return rc;
    if (feat == 0) return B200MP_OK;
    if (n_rows == 0) {
        if (grad_t) return cudaMemsetAsync(grad_t, 0, feat * sizeof(float), static_cast<cudaStream_t>(stream)) == cudaSuccess
                               ? B200MP_OK : B200MP_ERR_CUDA;
        return B200MP_OK;
    }
    B200MP_CHECK_ARG(rowptr && out && lse && grad_out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const AggrArgs a{x, edge_rows, t, perm, grad_out, out, const_cast<float*>(lse), nullptr, grad_edge_rows, nullptr,
                     feat, eps, 0, 0, semi_grad != 0};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_backward_dst", [&](auto tv, auto ti) {
        return aggr_dst<SoftmaxAggrOp, decltype(tv), decltype(ti)>(rowptr, col, a, sm_form(x, edge_rows, message),
                                                                   t_mode, grad_t, workspace, n_rows, plan,
                                                                   static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_softmax_aggr_backward_src(const void* rowptr_t, const void* col_t, const void* perm_t,
                                                const void* x, const void* edge_rows, const float* t, const void* out,
                                                const float* lse, const void* grad_out, void* grad_x, int64_t n_src,
                                                int64_t n_dst, int64_t n_edges, int64_t feat, int message, float eps,
                                                int t_mode, int semi_grad, const int64_t* long_rows,
                                                const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                                int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                                void* stream) {
    if (int rc = check_aggr_args(n_src, n_dst, n_edges, feat, message, x, edge_rows, t_mode, t, false, 0, 0)) return rc;
    B200MP_CHECK_ARG(x != nullptr);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && grad_x);
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && out && lse && grad_out && (edge_rows == nullptr || perm_t)));
    const AggrArgs a{x, edge_rows, t, perm_t, grad_out, out, const_cast<float*>(lse), nullptr, grad_x, nullptr, feat,
                     eps, 0, 0, semi_grad != 0};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_backward_src", [&](auto tv, auto ti) {
        return aggr_sweep<SoftmaxAggrOp, decltype(tv), decltype(ti), kSweepSrc>(
            rowptr_t, col_t, a, sm_form(x, edge_rows, message), t_mode, n_src, plan, static_cast<cudaStream_t>(stream));
    });
}
