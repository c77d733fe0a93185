// power_mean.cu -- PowerMeanAggregation (and GENConv's message relu(x_j + e_ji) + eps in front of it) as one sweep
// over the destination CSR, and its backward.  The op sequence is the reference's (nn/aggr/basic.py:275-293):
//
// Per destination i, feature f and in-edge e = (j -> i), eid(e) = perm[e] (CSR slot -> the caller's edge id) or e:
//   m_e = x[j] | a[eid(e)] | round(relu(round(x[j] + a[eid(e)])) + eps)      (template FORM, as in softmax_aggr.cu)
//   c_e = clamp(m_e, lo, hi)             y_e = round(c_e ^ p_f)
//   M_i = round(sum_e y_e / max(deg_i, 1))          (fp32 compensated sum)
//   C_i = clamp(M_i, lo, hi)             out_i = round(C_i ^ (1 / p_f))
// p is fp32 in device memory: none (a Python-number p of 1: no clamp and no pow, a plain mean), p[0] or p[f] (template
// PMODE), so a learnable p costs no host read.  1 / p is formed once in fp32, as the reference's `1. / p`.  lo > 0, so
// every base is positive, +inf (hi = +inf) or NaN; the clamp keeps NaN as ATen's does.  An empty row gives lo ^ (1/p)
// in the pow modes (the reference clamps the zero mean) and 0 without p.  The only saved state is M, one fp32
// [n_rows, F] plane, written only when a gradient is needed.
//
// c ^ p is ex2.approx(p * lg2.approx(c)).  lg2.approx has an absolute error of at most 2^-22.6 and ex2.approx a relative
// error of at most 2^-22.5 (PTX ISA); the fp32 product adds 2^-24 |p lg2 c|.  The relative error of c ^ p is therefore
// below ln2 (|p| 2^-22.6 + 2^-24 |p lg2 c|) + 2^-22.5, which for |p| <= 4 and c <= 100 (lg2 c < 6.7) is 1.4e-6: inside
// the 1e-5 bar.  The final pow divides M's relative error by p, hence the bar's max(1, 1/|p|).  powf / log2f / exp2f
// would cost about 40 FP32 instructions per element, more than the SMs issue at HBM rate for 4 bytes per element.
//
// Backward, with g = grad_out[i], o = out[i], deg = max(deg_i, 1):
//   G_i = g (1/p) C_i ^ (1/p - 1) / deg [lo <= M_i <= hi]   (g / deg without p; the mask is ATen's clamp backward)
//   grad_m_e = G_i p c_e ^ (p - 1) [lo <= m_e <= hi]    grad_s = grad_m [s > 0 or NaN]   (relu form)
//   grad_p = sum_i sum_e G_i y_e ln c_e - sum_i g o ln C_i / p^2      (the second sum includes empty rows)
// grad_p is collected as per-CTA fp32 partials folded by b200mp_column_sum in a fixed order.  The destination sweep
// writes grad_s into grad_a in the caller's edge order; the transposed sweep sums grad_s over a source's out-edges into
// grad_x when no grad_a was written, reading one fp32 row of the node plane G per out-edge, which a node kernel writes
// first (with the per-row grad_p terms).
//
// Mapping as in softmax_aggr.cu: a lane group of G lanes per row, one 16-byte vector per lane and trip, rows longer
// than the plan's chunk split into chunks whose fp32 partials a combine kernel folds in chunk order.  Rows that are not
// a whole number of aligned 16-byte vectors take a one-warp scalar kernel.
#include "param_aggr.cuh"

namespace b200mp {

constexpr int kPmNodeRows = 32;   // destination rows per CTA of the node kernel

// clamp(v, lo, hi) keeping NaN (fminf / fmaxf would drop it).
__device__ __forceinline__ float pm_clamp(float v, float lo, float hi) {
    return v != v ? v : fminf(fmaxf(v, lo), hi);
}

__device__ __forceinline__ float pm_lg2(float v) {
    float r;
    asm("lg2.approx.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}

__device__ __forceinline__ float pm_ex2(float v) {
    float r;
    asm("ex2.approx.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}

// c ^ p for c > 0, +inf or NaN; p = 0 gives 1 for every c, as powf does.
__device__ __forceinline__ float pm_pow(float c, float p) {
    return p == 0.0f ? 1.0f : pm_ex2(__fmul_rn(p, pm_lg2(c)));
}

// y = round(clamp(m) ^ p), or m without p.
template <typename T, int PMODE>
__device__ __forceinline__ float pm_term(float m, float p, float lo, float hi) {
    return PMODE == kParamNone ? m : round_to<T>(pm_pow(pm_clamp(m, lo, hi), p));
}

// out from the fp32 sum of a row's terms; M is the saved (rounded) mean.
template <typename T, int PMODE>
__device__ __forceinline__ float pm_final(float S, float d, float p, float lo, float hi, float& M) {
    M = round_to<T>(__fdiv_rn(S, d));
    return PMODE == kParamNone ? M : round_to<T>(pm_pow(pm_clamp(M, lo, hi), __frcp_rn(p)));
}

// G_i of a destination element: g (1/p) C ^ (1/p - 1) / deg under the clamp mask, as ATen's pow backward forms it (so
// that C = +inf gives 0, not inf / inf); subtracts the row's grad_p term g o ln C / p^2 from gp when WANT_P.  The
// backward divides with __fdividef (2 ulp): an IEEE division's slow-path call would cost the sweeps a stack frame.
template <int PMODE, bool WANT_P>
__device__ __forceinline__ float pm_node(float g, float o, float M, float d, float p, float lo, float hi, float& gp) {
    if (PMODE == kParamNone) return __fdividef(g, d);
    const float C = pm_clamp(M, lo, hi);
    const float lC = pm_lg2(C);
    const float rp = __frcp_rn(p);
    if (WANT_P) gp = fmaf(-__fdividef(__fmul_rn(g, o), __fmul_rn(p, p)), __fmul_rn(lC, 0.69314718055994531f), gp);
    const float dC = __fmul_rn(__fmul_rn(g, rp), pm_ex2(__fmul_rn(__fsub_rn(rp, 1.0f), lC)));
    return (M >= lo && M <= hi) ? __fdividef(dC, d) : 0.0f;
}

// grad_m of one (edge, feature) from G: G p c ^ (p - 1), as ATen's pow backward forms it; adds G y ln c to gp when
// WANT_P.
template <int PMODE, bool WANT_P>
__device__ __forceinline__ float pm_grad(float m, float G, float p, float lo, float hi, float& gp) {
    if (PMODE == kParamNone) return G;
    const float c = pm_clamp(m, lo, hi);
    const float l = pm_lg2(c);
    if (WANT_P) gp = fmaf(__fmul_rn(G, pm_ex2(__fmul_rn(p, l))), __fmul_rn(l, 0.69314718055994531f), gp);
    return (m >= lo && m <= hi) ? __fmul_rn(__fmul_rn(G, p), pm_ex2(__fmul_rn(__fsub_rn(p, 1.0f), l))) : 0.0f;
}

// Compensated (Kahan) add: every term is positive and hub rows are long, and a drift of M is scaled by 1 / p in out.
// Once the sum is infinite or NaN the compensation (inf - inf) is dropped, so that the sum keeps the reference's
// inf or NaN.
__device__ __forceinline__ void pm_kahan(float& s, float& c, float v) {
    const float y = __fsub_rn(v, c);
    const float t = __fadd_rn(s, y);
    c = fabsf(t) < INFINITY ? __fsub_rn(__fsub_rn(t, s), y) : 0.0f;
    s = t;
}

// max(deg, 1) of a row as fp32: the divisor of the mean.
template <typename I>
__device__ __forceinline__ float pm_deg(const I* rowptr, int64_t row) {
    const int64_t d = static_cast<int64_t>(ldg_idx(rowptr + row + 1)) - static_cast<int64_t>(ldg_idx(rowptr + row));
    return static_cast<float>(d < 1 ? 1 : d);
}

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(128, 1)
power_mean_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AggrArgs args, int64_t n_rows, int n_vec,
                  int lg, LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int UNR = (MODE == kSweepFwd || sizeof(T) == 4) ? 4 : 2;
    extern __shared__ float pm_sh[];
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = aggr_item<WANT_P>(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // uniform per group
    if (!active && !WANT_P) return;
    // the destination sweep adds a row's grad_p term once: in its whole-row item or its first chunk
    const bool row_term = active && (!is_chunk || begin == static_cast<int64_t>(ldg_idx(rowptr + row)));
    const float deg = active ? pm_deg(rowptr, row) : 1.0f;
    const int64_t F = args.feat;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const size_t row_off = static_cast<size_t>(row) * row_bytes;     // this row's byte offset in g, o, x (src) and out
    const float* Mrow = args.saved + static_cast<size_t>(row) * F;
    const char* xb = static_cast<const char*>(args.x);
    const char* ab = static_cast<const char*>(args.a);
    float ps = 1.0f;
    if (PMODE == kParamScalar) ps = __ldg(args.param);

#pragma unroll 1
    for (int vi = lig; vi < n_vec; vi += G) {
        const size_t voff = static_cast<size_t>(vi) * 16;
        const int64_t f0 = static_cast<int64_t>(vi) * EPV;
        float pv[EPV], rx[EPV], rG[EPV], acc[EPV], cc[EPV], gp[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) pv[i] = ps, rx[i] = rG[i] = acc[i] = cc[i] = gp[i] = 0.0f;
        if (PMODE == kParamChannel) ldg_f32(args.param + f0, pv);
        if (MODE == kSweepDst && active) {
            float rg[EPV], ro[EPV];
            ElemTraits<T>::unpack(ldg_stream16(static_cast<const char*>(args.g) + row_off + voff), rg);
            ElemTraits<T>::unpack(ldg_stream16(static_cast<const char*>(args.o) + row_off + voff), ro);
            const float* mp = Mrow + f0;
#pragma unroll
            for (int i = 0; i < EPV; i += 4) {
                const float4 m4 = __ldg(reinterpret_cast<const float4*>(mp + i));
                float t[4] = {0.0f, 0.0f, 0.0f, 0.0f};
                rG[i] = pm_node<PMODE, WANT_P>(rg[i], ro[i], m4.x, deg, pv[i], args.lo, args.hi, t[0]);
                rG[i + 1] = pm_node<PMODE, WANT_P>(rg[i + 1], ro[i + 1], m4.y, deg, pv[i + 1], args.lo, args.hi, t[1]);
                rG[i + 2] = pm_node<PMODE, WANT_P>(rg[i + 2], ro[i + 2], m4.z, deg, pv[i + 2], args.lo, args.hi, t[2]);
                rG[i + 3] = pm_node<PMODE, WANT_P>(rg[i + 3], ro[i + 3], m4.w, deg, pv[i + 3], args.lo, args.hi, t[3]);
#pragma unroll
                for (int q = 0; q < 4; ++q) gp[i + q] = row_term ? t[q] : 0.0f;
            }
        }
        if (MODE == kSweepSrc) ElemTraits<T>::unpack(ldg_stream16(xb + row_off + voff), rx);
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 xv[UNR], av[UNR];
            float4 gv[UNR][EPV / 4];
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
                        const float4* gp4 = reinterpret_cast<const float4*>(args.G + c * F + f0);
#pragma unroll
                        for (int q = 0; q < EPV / 4; ++q) gv[u][q] = __ldg(gp4 + q);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float fx[EPV], fa[EPV], fG[EPV], gs[EPV];
                    if (MODE == kSweepSrc) {
#pragma unroll
                        for (int i = 0; i < EPV; ++i) fx[i] = rx[i];
#pragma unroll
                        for (int q = 0; q < EPV / 4; ++q) {
                            fG[4 * q] = gv[u][q].x; fG[4 * q + 1] = gv[u][q].y;
                            fG[4 * q + 2] = gv[u][q].z; fG[4 * q + 3] = gv[u][q].w;
                        }
                    } else if (Fm::kX) {
                        ElemTraits<T>::unpack(xv[u], fx);
                    }
                    if (Fm::kA) ElemTraits<T>::unpack(av[u], fa);
#pragma unroll
                    for (int i = 0; i < EPV; ++i) {
                        bool on;
                        const float m = sm_message<T, FORM>(fx[i], Fm::kA ? fa[i] : 0.0f, args.eps, on);
                        if (MODE == kSweepFwd) {
                            pm_kahan(acc[i], cc[i], pm_term<T, PMODE>(m, pv[i], args.lo, args.hi));
                        } else {
                            float gm = pm_grad<PMODE, WANT_P>(m, MODE == kSweepSrc ? fG[i] : rG[i], pv[i], args.lo,
                                                              args.hi, gp[i]);
                            if (Fm::kRelu && !on) gm = 0.0f;
                            if (MODE == kSweepDst) gs[i] = gm;
                            else acc[i] = __fadd_rn(acc[i], gm);
                        }
                    }
                    if (MODE == kSweepDst && args.out)
                        stg_stream16(static_cast<char*>(args.out) + id[u] * row_bytes + voff, ElemTraits<T>::pack(gs));
                }
            }
        }
        if (WANT_P) {
            float* sh = pm_sh + static_cast<int64_t>(threadIdx.x >> lg) * F + f0;
#pragma unroll
            for (int i = 0; i < EPV; ++i) sh[i] = gp[i];
        }
        if (MODE == kSweepDst || !active) continue;
        if (MODE == kSweepFwd) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) acc[i] = __fsub_rn(acc[i], cc[i]);
        }
        if (is_chunk) {
            store_partial<EPV>(plan.partials + static_cast<size_t>(item) * F + f0, acc);
            continue;
        }
        char* dst = static_cast<char*>(args.out) + row_off + voff;
        if (MODE == kSweepFwd) {
            float f[EPV], Mv[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i) f[i] = pm_final<T, PMODE>(acc[i], deg, pv[i], args.lo, args.hi, Mv[i]);
            stg_stream16(dst, ElemTraits<T>::pack(f));
            if (args.saved) store_partial<EPV>(args.saved + static_cast<size_t>(row) * F + f0, Mv);
        } else {
            stg_stream16(dst, ElemTraits<T>::pack(acc));
        }
    }
    if (WANT_P) store_param_part(pm_sh, blockDim.x >> lg, F, args.param_part);
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(256, 1)
power_mean_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AggrArgs args, int64_t n_rows,
                         LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    extern __shared__ float pm_sh[];
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = aggr_item<WANT_P>(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // warp-uniform
    if (!active && !WANT_P) return;
    const bool row_term = active && (!is_chunk || begin == static_cast<int64_t>(ldg_idx(rowptr + row)));
    const float deg = active ? pm_deg(rowptr, row) : 1.0f;
    const int64_t F = args.feat;
    const T* x = static_cast<const T*>(args.x);
    const T* a = static_cast<const T*>(args.a);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = lane; f < F; f += 32) {
        const float pv = PMODE == kParamNone ? 1.0f : __ldg(args.param + (PMODE == kParamChannel ? f : 0));
        float acc = 0.0f, cc = 0.0f, gp = 0.0f, rx = 0.0f, rG = 0.0f;
        if (MODE == kSweepDst && active) {
            float t = 0.0f;
            rG = pm_node<PMODE, WANT_P>(ElemTraits<T>::to_float(static_cast<const T*>(args.g)[row * F + f]),
                                        ElemTraits<T>::to_float(static_cast<const T*>(args.o)[row * F + f]),
                                        args.saved[row * F + f], deg, pv, args.lo, args.hi, t);
            if (row_term) gp = t;
        }
        if (MODE == kSweepSrc) rx = ElemTraits<T>::to_float(x[row * F + f]);
#pragma unroll 2
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t id = (Fm::kA || (MODE == kSweepDst && out)) ? aggr_eid<I>(args, e) : 0;
            const float xv = MODE == kSweepSrc ? rx : (Fm::kX ? ElemTraits<T>::to_float(x[c * F + f]) : 0.0f);
            const float av = Fm::kA ? ElemTraits<T>::to_float(a[id * F + f]) : 0.0f;
            bool on;
            const float m = sm_message<T, FORM>(xv, av, args.eps, on);
            if (MODE == kSweepFwd) {
                pm_kahan(acc, cc, pm_term<T, PMODE>(m, pv, args.lo, args.hi));
            } else {
                float gm = pm_grad<PMODE, WANT_P>(m, MODE == kSweepSrc ? args.G[c * F + f] : rG, pv, args.lo, args.hi, gp);
                if (Fm::kRelu && !on) gm = 0.0f;
                if (MODE == kSweepSrc) acc = __fadd_rn(acc, gm);
                else if (out) out[id * F + f] = ElemTraits<T>::from_float(gm);
            }
        }
        if (WANT_P) pm_sh[(threadIdx.x >> 5) * F + f] = gp;
        if (MODE == kSweepDst || !active) continue;
        if (MODE == kSweepFwd) acc = __fsub_rn(acc, cc);
        if (is_chunk) {
            plan.partials[item * F + f] = acc;
            continue;
        }
        if (MODE == kSweepFwd) {
            float Mv;
            out[row * F + f] = ElemTraits<T>::from_float(pm_final<T, PMODE>(acc, deg, pv, args.lo, args.hi, Mv));
            if (args.saved) args.saved[row * F + f] = Mv;
        } else {
            out[row * F + f] = ElemTraits<T>::from_float(acc);
        }
    }
    if (WANT_P) store_param_part(pm_sh, blockDim.x >> 5, F, args.param_part);
}

// Sum the partials of every long row in chunk order and write out and M.
template <typename T, typename I, int PMODE>
__global__ void __launch_bounds__(256)
power_mean_combine_kernel(const I* __restrict__ rowptr, AggrArgs args, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t F = args.feat;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const float deg = pm_deg(rowptr, row);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
        const float pv = PMODE == kParamNone ? 1.0f : __ldg(args.param + (PMODE == kParamChannel ? f : 0));
        float S = 0.0f;
        for (int64_t c = c0; c < c1; ++c) S = __fadd_rn(S, plan.partials[c * F + f]);
        float Mv;
        out[row * F + f] = ElemTraits<T>::from_float(pm_final<T, PMODE>(S, deg, pv, args.lo, args.hi, Mv));
        if (args.saved) args.saved[row * F + f] = Mv;
    }
}

// The node plane of the transposed sweep: G for kPmNodeRows destination rows per CTA, and the rows' grad_p terms as
// one fp32 partial row per CTA.
template <typename T, typename I, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(256)
power_mean_node_kernel(const I* __restrict__ rowptr, AggrArgs args, int64_t n_dst) {
    const int64_t F = args.feat;
    const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kPmNodeRows;
    const int64_t r1 = r0 + kPmNodeRows < n_dst ? r0 + kPmNodeRows : n_dst;
    const T* g = static_cast<const T*>(args.g);
    const T* o = static_cast<const T*>(args.o);
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
        const float pv = PMODE == kParamNone ? 1.0f : __ldg(args.param + (PMODE == kParamChannel ? f : 0));
        float gp = 0.0f;
        for (int64_t r = r0; r < r1; ++r)
            args.G[r * F + f] = pm_node<PMODE, WANT_P>(ElemTraits<T>::to_float(g[r * F + f]),
                                                       ElemTraits<T>::to_float(o[r * F + f]),
                                                       PMODE == kParamNone ? 0.0f : args.saved[r * F + f], pm_deg(rowptr, r),
                                                       pv, args.lo, args.hi, gp);
        if (WANT_P) args.param_part[static_cast<int64_t>(blockIdx.x) * F + f] = gp;
    }
}

struct PowerMeanOp {
    static constexpr const char* kName = "power_mean";
    static constexpr const char* kParam = "p";
    static constexpr bool collects(int mode) { return mode != kSweepFwd; }
    template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
    static auto vec() { return power_mean_kernel<T, I, MODE, FORM, PMODE, WANT_P>; }
    template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
    static auto scalar() { return power_mean_scalar_kernel<T, I, MODE, FORM, PMODE, WANT_P>; }
    template <typename T, typename I, int PMODE>
    static void combine(const I* rowptr, const AggrArgs& args, const LongRowPlan& plan, cudaStream_t s) {
        power_mean_combine_kernel<T, I, PMODE><<<static_cast<unsigned>(plan.n_long), 256, 0, s>>>(rowptr, args, plan);
    }
};

// The node kernel's CTAs over n_node destination rows.
inline int64_t pm_node_ctas(int64_t n_node) { return ceil_div(n_node, kPmNodeRows); }

// The node kernel, then the transposed sweep; grad_p from the node kernel's partial rows followed by the sweep's.
template <typename T, typename I>
int pm_src(const void* rowptr, const void* rowptr_t, const void* col_t, AggrArgs a, int form, int p_mode, float* grad_p,
           float* ws, int64_t n_src, int64_t n_dst, const LongRowPlan& plan, cudaStream_t s) {
    const int64_t F = a.feat;
    a.G = ws;
    SweepShape sh;
    if (int rc = sweep_shape<PowerMeanOp, T>(a, plan, n_src, grad_p != nullptr, sh)) return rc;
    float* parts = ws + n_dst * F;
    const int64_t node_ctas = pm_node_ctas(n_dst);
    a.param_part = parts;
    if (node_ctas > 0) {
        const unsigned grid = static_cast<unsigned>(node_ctas);
        auto node = [&](auto k) { k<<<grid, 256, 0, s>>>(static_cast<const I*>(rowptr), a, n_dst); };
        if (grad_p == nullptr && p_mode == kParamScalar) node(power_mean_node_kernel<T, I, kParamScalar, false>);
        else if (grad_p == nullptr && p_mode == kParamChannel) node(power_mean_node_kernel<T, I, kParamChannel, false>);
        else if (grad_p == nullptr) node(power_mean_node_kernel<T, I, kParamNone, false>);
        else if (p_mode == kParamScalar) node(power_mean_node_kernel<T, I, kParamScalar, true>);
        else node(power_mean_node_kernel<T, I, kParamChannel, true>);
        B200MP_LAUNCH_CHECK();
    }
    a.param_part = parts + node_ctas * F;
    if (int rc = aggr_typed<PowerMeanOp, T, I, kSweepSrc>(rowptr_t, col_t, a, form, p_mode, grad_p != nullptr, n_src,
                                                          plan, sh, s))
        return rc;
    return grad_p == nullptr ? B200MP_OK : fold_param_parts(parts, node_ctas + sh.grid, grad_p, F, s);
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_power_mean_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                     const void* edge_rows, const float* p, void* out, float* mean, int64_t n_rows,
                                     int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps, int p_mode,
                                     float clamp_min, float clamp_max, const int64_t* long_rows,
                                     const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                     float* partials, int idx_dtype, int val_dtype, void* stream) {
    if (int rc = check_aggr_args(n_rows, n_cols, n_edges, feat, message, x, edge_rows, p_mode, p, true, clamp_min,
                                 clamp_max))
        return rc;
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const AggrArgs a{x, edge_rows, p, perm, nullptr, nullptr, mean, nullptr, out, nullptr, feat, eps, clamp_min,
                     clamp_max, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_csr", [&](auto tv, auto ti) {
        return aggr_sweep<PowerMeanOp, decltype(tv), decltype(ti), kSweepFwd>(
            rowptr, col, a, sm_form(x, edge_rows, message), p_mode, n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

// The grad_p partial rows are an upper bound over both sweep kernels (a vector CTA holds at least 4 work items, a
// scalar CTA 8), after the node kernel's.
extern "C" int64_t b200mp_power_mean_workspace(int64_t n_node, int64_t n_rows, int64_t n_chunks, int64_t feat) {
    const int64_t parts = pm_node_ctas(n_node) + ceil_div(n_rows + n_chunks, 4);
    return (n_node + parts + b200mp_column_sum_parts(parts)) * feat;
}

extern "C" int b200mp_power_mean_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                              const void* edge_rows, const float* p, const void* out, const float* mean,
                                              const void* grad_out, void* grad_edge_rows, float* grad_p,
                                              float* workspace, int64_t n_rows, int64_t n_cols, int64_t n_edges,
                                              int64_t feat, int message, float eps, int p_mode, float clamp_min,
                                              float clamp_max, const int64_t* long_rows, const int64_t* chunk_ptr,
                                              int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype,
                                              int val_dtype, void* stream) {
    if (int rc = check_aggr_args(n_rows, n_cols, n_edges, feat, message, x, edge_rows, p_mode, p, true, clamp_min,
                                 clamp_max))
        return rc;
    B200MP_CHECK_ARG(grad_p == nullptr || (p_mode != 0 && workspace));
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, nullptr, false)) return rc;
    if (feat == 0) return B200MP_OK;
    if (n_rows == 0) {
        if (grad_p) return cudaMemsetAsync(grad_p, 0, feat * sizeof(float), static_cast<cudaStream_t>(stream)) == cudaSuccess
                               ? B200MP_OK : B200MP_ERR_CUDA;
        return B200MP_OK;
    }
    B200MP_CHECK_ARG(rowptr && out && grad_out && (p_mode == 0 || mean));
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const AggrArgs a{x, edge_rows, p, perm, grad_out, out, const_cast<float*>(mean), nullptr, grad_edge_rows, nullptr,
                     feat, eps, clamp_min, clamp_max, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_backward_dst", [&](auto tv, auto ti) {
        return aggr_dst<PowerMeanOp, decltype(tv), decltype(ti)>(rowptr, col, a, sm_form(x, edge_rows, message), p_mode,
                                                                 grad_p, workspace, n_rows, plan,
                                                                 static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_power_mean_backward_src(const void* rowptr, const void* rowptr_t, const void* col_t,
                                              const void* perm_t, const void* x, const void* edge_rows, const float* p,
                                              const void* out, const float* mean, const void* grad_out, void* grad_x,
                                              float* grad_p, float* workspace, int64_t n_src, int64_t n_dst,
                                              int64_t n_edges, int64_t feat, int message, float eps, int p_mode,
                                              float clamp_min, float clamp_max, const int64_t* long_rows,
                                              const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                              int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                              void* stream) {
    if (int rc = check_aggr_args(n_src, n_dst, n_edges, feat, message, x, edge_rows, p_mode, p, true, clamp_min,
                                 clamp_max))
        return rc;
    B200MP_CHECK_ARG(x != nullptr);
    B200MP_CHECK_ARG(grad_p == nullptr || p_mode != 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (feat == 0) return B200MP_OK;
    if (n_src == 0 && grad_p == nullptr) return B200MP_OK;
    B200MP_CHECK_ARG(workspace && rowptr && rowptr_t && (n_src == 0 || grad_x));
    B200MP_CHECK_ARG(n_dst == 0 || (out && grad_out && (p_mode == 0 || mean)));
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && (edge_rows == nullptr || perm_t)));
    const AggrArgs a{x, edge_rows, p, perm_t, grad_out, out, const_cast<float*>(mean), nullptr, grad_x, nullptr, feat,
                     eps, clamp_min, clamp_max, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_backward_src", [&](auto tv, auto ti) {
        return pm_src<decltype(tv), decltype(ti)>(rowptr, rowptr_t, col_t, a, sm_form(x, edge_rows, message), p_mode,
                                                  grad_p, workspace, n_src, n_dst, plan,
                                                  static_cast<cudaStream_t>(stream));
    });
}
