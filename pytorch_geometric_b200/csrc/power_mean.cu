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
#include "aggr_message.cuh"
#include "csr_reduce.cuh"

extern "C" int b200mp_column_sum(const void* x, float* out, float* partials, int64_t n_parts, int64_t n_rows,
                                 int64_t feat, int val_dtype, void* stream);
extern "C" int64_t b200mp_column_sum_parts(int64_t n_rows);

namespace b200mp {

enum PmMode { kPmFwd = 0, kPmDst = 1, kPmSrc = 2 };
enum PmP { kPmPNone = 0, kPmPScalar = 1, kPmPChannel = 2 };

constexpr int kPmNodeRows = 32;   // destination rows per CTA of the node kernel
// The grad_p sweeps keep one fp32 row of F per lane group in shared memory: H100's opt-in limit per CTA.
constexpr size_t kPmMaxSmem = 227 * 1024;

struct PmArgs {
    const void* x;       // [n_src, feat] gathered through col (fwd / dst) or the row operand (src)
    const void* a;       // [n_edges, feat] in the caller's edge order
    const float* p;      // [1] or [feat] fp32
    const void* perm;    // caller's edge id of each CSR (fwd / dst) or transposed (src) slot; null = slot
    const void* g;       // grad_out [n_dst, feat]
    const void* o;       // out [n_dst, feat]
    float* M;            // [n_dst, feat]: written by fwd (nullable), read by the backward
    float* G;            // src: the node plane [n_dst, feat] the transposed sweep gathers
    void* out;           // fwd: out; dst: grad_a (nullable); src: grad_x
    float* gp_part;      // [gridDim.x, feat] grad_p partials, or null
    int64_t feat;
    float eps, lo, hi;
};

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
    return PMODE == kPmPNone ? m : round_to<T>(pm_pow(pm_clamp(m, lo, hi), p));
}

// out from the fp32 sum of a row's terms; M is the saved (rounded) mean.
template <typename T, int PMODE>
__device__ __forceinline__ float pm_final(float S, float d, float p, float lo, float hi, float& M) {
    M = round_to<T>(__fdiv_rn(S, d));
    return PMODE == kPmPNone ? M : round_to<T>(pm_pow(pm_clamp(M, lo, hi), __frcp_rn(p)));
}

// G_i of a destination element: g (1/p) C ^ (1/p - 1) / deg under the clamp mask, as ATen's pow backward forms it (so
// that C = +inf gives 0, not inf / inf); subtracts the row's grad_p term g o ln C / p^2 from gp when WANT_P.  The
// backward divides with __fdividef (2 ulp): an IEEE division's slow-path call would cost the sweeps a stack frame.
template <int PMODE, bool WANT_P>
__device__ __forceinline__ float pm_node(float g, float o, float M, float d, float p, float lo, float hi, float& gp) {
    if (PMODE == kPmPNone) return __fdividef(g, d);
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
    if (PMODE == kPmPNone) return G;
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

template <typename I>
__device__ __forceinline__ int64_t pm_eid(const PmArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// max(deg, 1) of a row as fp32: the divisor of the mean.
template <typename I>
__device__ __forceinline__ float pm_deg(const I* rowptr, int64_t row) {
    const int64_t d = static_cast<int64_t>(ldg_idx(rowptr + row + 1)) - static_cast<int64_t>(ldg_idx(rowptr + row));
    return static_cast<float>(d < 1 ? 1 : d);
}

// Per-CTA grad_p partial: every group has written its row of `sh` (zeros when idle); fold the groups in order.
__device__ __forceinline__ void pm_store_gp(const float* sh, int groups, int64_t feat, float* gp_part) {
    __syncthreads();
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        float s = 0.0f;
        for (int k = 0; k < groups; ++k) s = __fadd_rn(s, sh[k * feat + f]);
        gp_part[static_cast<int64_t>(blockIdx.x) * feat + f] = s;
    }
}

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(128, 1)
power_mean_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, PmArgs args, int64_t n_rows, int n_vec,
                  int lg, LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int UNR = (MODE == kPmFwd || sizeof(T) == 4) ? 4 : 2;
    extern __shared__ float pm_sh[];
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // uniform per group
    if (!active && !WANT_P) return;
    if (!active) row = begin = end = 0;                  // an idle group still writes its (zero) grad_p row
    // the destination sweep adds a row's grad_p term once: in its whole-row item or its first chunk
    const bool row_term = active && (!is_chunk || begin == static_cast<int64_t>(ldg_idx(rowptr + row)));
    const float deg = active ? pm_deg(rowptr, row) : 1.0f;
    const int64_t F = args.feat;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const size_t row_off = static_cast<size_t>(row) * row_bytes;     // this row's byte offset in g, o, x (src) and out
    const float* Mrow = args.M + static_cast<size_t>(row) * F;
    const char* xb = static_cast<const char*>(args.x);
    const char* ab = static_cast<const char*>(args.a);
    float ps = 1.0f;
    if (PMODE == kPmPScalar) ps = __ldg(args.p);

#pragma unroll 1
    for (int vi = lig; vi < n_vec; vi += G) {
        const size_t voff = static_cast<size_t>(vi) * 16;
        const int64_t f0 = static_cast<int64_t>(vi) * EPV;
        float pv[EPV], rx[EPV], rG[EPV], acc[EPV], cc[EPV], gp[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) pv[i] = ps, rx[i] = rG[i] = acc[i] = cc[i] = gp[i] = 0.0f;
        if (PMODE == kPmPChannel) {
#pragma unroll
            for (int i = 0; i < EPV; i += 4) {
                const float4 p4 = __ldg(reinterpret_cast<const float4*>(args.p + f0 + i));
                pv[i] = p4.x; pv[i + 1] = p4.y; pv[i + 2] = p4.z; pv[i + 3] = p4.w;
            }
        }
        if (MODE == kPmDst && active) {
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
        if (MODE == kPmSrc) ElemTraits<T>::unpack(ldg_stream16(xb + row_off + voff), rx);
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 xv[UNR], av[UNR];
            float4 gv[UNR][EPV / 4];
            int64_t id[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                id[u] = 0;
                if (e + u < end) {
                    const int64_t c = static_cast<int64_t>(ldg_idx(col + e + u));
                    if (Fm::kA || (MODE == kPmDst && args.out)) id[u] = pm_eid<I>(args, e + u);
                    if (MODE != kPmSrc && Fm::kX) xv[u] = ldg_row16(xb + c * row_bytes + voff);
                    if (Fm::kA) av[u] = ldg_stream16(ab + id[u] * row_bytes + voff);
                    if (MODE == kPmSrc) {
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
                    if (MODE == kPmSrc) {
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
                        if (MODE == kPmFwd) {
                            pm_kahan(acc[i], cc[i], pm_term<T, PMODE>(m, pv[i], args.lo, args.hi));
                        } else {
                            float gm = pm_grad<PMODE, WANT_P>(m, MODE == kPmSrc ? fG[i] : rG[i], pv[i], args.lo,
                                                              args.hi, gp[i]);
                            if (Fm::kRelu && !on) gm = 0.0f;
                            if (MODE == kPmDst) gs[i] = gm;
                            else acc[i] = __fadd_rn(acc[i], gm);
                        }
                    }
                    if (MODE == kPmDst && args.out)
                        stg_stream16(static_cast<char*>(args.out) + id[u] * row_bytes + voff, ElemTraits<T>::pack(gs));
                }
            }
        }
        if (WANT_P) {
            float* sh = pm_sh + static_cast<int64_t>(threadIdx.x >> lg) * F + f0;
#pragma unroll
            for (int i = 0; i < EPV; ++i) sh[i] = gp[i];
        }
        if (MODE == kPmDst || !active) continue;
        if (MODE == kPmFwd) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) acc[i] = __fsub_rn(acc[i], cc[i]);
        }
        if (is_chunk) {
            store_partial<EPV>(plan.partials + static_cast<size_t>(item) * F + f0, acc);
            continue;
        }
        char* dst = static_cast<char*>(args.out) + row_off + voff;
        if (MODE == kPmFwd) {
            float f[EPV], Mv[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i) f[i] = pm_final<T, PMODE>(acc[i], deg, pv[i], args.lo, args.hi, Mv[i]);
            stg_stream16(dst, ElemTraits<T>::pack(f));
            if (args.M) store_partial<EPV>(args.M + static_cast<size_t>(row) * F + f0, Mv);
        } else {
            stg_stream16(dst, ElemTraits<T>::pack(acc));
        }
    }
    if (WANT_P) pm_store_gp(pm_sh, blockDim.x >> lg, F, args.gp_part);
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(256, 1)
power_mean_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, PmArgs args, int64_t n_rows,
                         LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    extern __shared__ float pm_sh[];
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // warp-uniform
    if (!active && !WANT_P) return;
    if (!active) row = begin = end = 0;                  // an idle group still writes its (zero) grad_p row
    const bool row_term = active && (!is_chunk || begin == static_cast<int64_t>(ldg_idx(rowptr + row)));
    const float deg = active ? pm_deg(rowptr, row) : 1.0f;
    const int64_t F = args.feat;
    const T* x = static_cast<const T*>(args.x);
    const T* a = static_cast<const T*>(args.a);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = lane; f < F; f += 32) {
        const float pv = PMODE == kPmPNone ? 1.0f : __ldg(args.p + (PMODE == kPmPChannel ? f : 0));
        float acc = 0.0f, cc = 0.0f, gp = 0.0f, rx = 0.0f, rG = 0.0f;
        if (MODE == kPmDst && active) {
            float t = 0.0f;
            rG = pm_node<PMODE, WANT_P>(ElemTraits<T>::to_float(static_cast<const T*>(args.g)[row * F + f]),
                                        ElemTraits<T>::to_float(static_cast<const T*>(args.o)[row * F + f]),
                                        args.M[row * F + f], deg, pv, args.lo, args.hi, t);
            if (row_term) gp = t;
        }
        if (MODE == kPmSrc) rx = ElemTraits<T>::to_float(x[row * F + f]);
#pragma unroll 2
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t id = (Fm::kA || (MODE == kPmDst && out)) ? pm_eid<I>(args, e) : 0;
            const float xv = MODE == kPmSrc ? rx : (Fm::kX ? ElemTraits<T>::to_float(x[c * F + f]) : 0.0f);
            const float av = Fm::kA ? ElemTraits<T>::to_float(a[id * F + f]) : 0.0f;
            bool on;
            const float m = sm_message<T, FORM>(xv, av, args.eps, on);
            if (MODE == kPmFwd) {
                pm_kahan(acc, cc, pm_term<T, PMODE>(m, pv, args.lo, args.hi));
            } else {
                float gm = pm_grad<PMODE, WANT_P>(m, MODE == kPmSrc ? args.G[c * F + f] : rG, pv, args.lo, args.hi, gp);
                if (Fm::kRelu && !on) gm = 0.0f;
                if (MODE == kPmSrc) acc = __fadd_rn(acc, gm);
                else if (out) out[id * F + f] = ElemTraits<T>::from_float(gm);
            }
        }
        if (WANT_P) pm_sh[(threadIdx.x >> 5) * F + f] = gp;
        if (MODE == kPmDst || !active) continue;
        if (MODE == kPmFwd) acc = __fsub_rn(acc, cc);
        if (is_chunk) {
            plan.partials[item * F + f] = acc;
            continue;
        }
        if (MODE == kPmFwd) {
            float Mv;
            out[row * F + f] = ElemTraits<T>::from_float(pm_final<T, PMODE>(acc, deg, pv, args.lo, args.hi, Mv));
            if (args.M) args.M[row * F + f] = Mv;
        } else {
            out[row * F + f] = ElemTraits<T>::from_float(acc);
        }
    }
    if (WANT_P) pm_store_gp(pm_sh, blockDim.x >> 5, F, args.gp_part);
}

// Sum the partials of every long row in chunk order and write out and M.
template <typename T, typename I, int PMODE>
__global__ void __launch_bounds__(256)
power_mean_combine_kernel(const I* __restrict__ rowptr, PmArgs args, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t F = args.feat;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const float deg = pm_deg(rowptr, row);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
        const float pv = PMODE == kPmPNone ? 1.0f : __ldg(args.p + (PMODE == kPmPChannel ? f : 0));
        float S = 0.0f;
        for (int64_t c = c0; c < c1; ++c) S = __fadd_rn(S, plan.partials[c * F + f]);
        float Mv;
        out[row * F + f] = ElemTraits<T>::from_float(pm_final<T, PMODE>(S, deg, pv, args.lo, args.hi, Mv));
        if (args.M) args.M[row * F + f] = Mv;
    }
}

// The node plane of the transposed sweep: G for kPmNodeRows destination rows per CTA, and the rows' grad_p terms as
// one fp32 partial row per CTA.
template <typename T, typename I, int PMODE, bool WANT_P>
__global__ void __launch_bounds__(256)
power_mean_node_kernel(const I* __restrict__ rowptr, PmArgs args, int64_t n_dst) {
    const int64_t F = args.feat;
    const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kPmNodeRows;
    const int64_t r1 = r0 + kPmNodeRows < n_dst ? r0 + kPmNodeRows : n_dst;
    const T* g = static_cast<const T*>(args.g);
    const T* o = static_cast<const T*>(args.o);
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
        const float pv = PMODE == kPmPNone ? 1.0f : __ldg(args.p + (PMODE == kPmPChannel ? f : 0));
        float gp = 0.0f;
        for (int64_t r = r0; r < r1; ++r)
            args.G[r * F + f] = pm_node<PMODE, WANT_P>(ElemTraits<T>::to_float(g[r * F + f]),
                                                       ElemTraits<T>::to_float(o[r * F + f]),
                                                       PMODE == kPmPNone ? 0.0f : args.M[r * F + f], pm_deg(rowptr, r),
                                                       pv, args.lo, args.hi, gp);
        if (WANT_P) args.gp_part[static_cast<int64_t>(blockIdx.x) * F + f] = gp;
    }
}

// ---------------------------------------------------------------- host-side dispatch
template <typename T>
bool pm_vec_ok(const PmArgs& a, const LongRowPlan& plan) {
    return (a.feat * sizeof(T)) % 16 == 0 && aligned16(a.x) && aligned16(a.a) && aligned16(a.p) && aligned16(a.g) &&
           aligned16(a.o) && aligned16(a.M) && aligned16(a.G) && aligned16(a.out) &&
           (plan.n_chunks == 0 || aligned16(plan.partials));
}

// CTAs of the sweep that pm_launch runs, so that the caller can place the grad_p partials.
template <typename T>
int64_t pm_grid(const PmArgs& a, const LongRowPlan& plan, int64_t n_rows, int& lg, bool& vec) {
    const int64_t items = plan.n_chunks + n_rows;
    vec = pm_vec_ok<T>(a, plan);
    if (vec) {
        lane_group_shape<1>(static_cast<int>(a.feat * sizeof(T) / 16), [&](auto G, auto) {
            lg = 0;
            while ((1 << lg) < decltype(G)::value) ++lg;
        });
        return ceil_div(items, 128 >> lg);
    }
    lg = 5;
    return ceil_div(items, 8);
}

template <typename T, typename I, int MODE, int FORM, int PMODE, bool WANT_P>
int pm_launch(const I* rowptr, const I* col, const PmArgs& args, int64_t n_rows, const LongRowPlan& plan,
              cudaStream_t stream) {
    int lg;
    bool vec;
    const int64_t grid = pm_grid<T>(args, plan, n_rows, lg, vec);
    if (grid == 0) return B200MP_OK;
    const size_t smem = WANT_P ? static_cast<size_t>(vec ? (128 >> lg) : 8) * args.feat * sizeof(float) : 0;
    if (smem > kPmMaxSmem) {
        set_error("power_mean: grad_p of %lld channels needs %zu bytes of shared memory per CTA (at most %zu)",
                  static_cast<long long>(args.feat), smem, kPmMaxSmem);
        return B200MP_ERR_UNSUPPORTED;
    }
    if (vec) {
        auto k = power_mean_kernel<T, I, MODE, FORM, PMODE, WANT_P>;
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<static_cast<unsigned>(grid), 128, smem, stream>>>(rowptr, col, args, n_rows,
                                                              static_cast<int>(args.feat * sizeof(T) / 16), lg, plan);
    } else {
        auto k = power_mean_scalar_kernel<T, I, MODE, FORM, PMODE, WANT_P>;
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<static_cast<unsigned>(grid), 256, smem, stream>>>(rowptr, col, args, n_rows, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (MODE != kPmDst && plan.n_long > 0) {
        if (MODE == kPmFwd)
            power_mean_combine_kernel<T, I, PMODE><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, args,
                                                                                                          plan);
        else
            csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
                rowptr, static_cast<T*>(args.out), args.feat, false, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I, int MODE, int FORM>
int pm_dispatch_p(const I* rowptr, const I* col, const PmArgs& args, int pmode, bool want_p, int64_t n_rows,
                  const LongRowPlan& plan, cudaStream_t s) {
    if constexpr (MODE != kPmFwd) {
        if (want_p && pmode == kPmPScalar) return pm_launch<T, I, MODE, FORM, kPmPScalar, true>(rowptr, col, args, n_rows, plan, s);
        if (want_p) return pm_launch<T, I, MODE, FORM, kPmPChannel, true>(rowptr, col, args, n_rows, plan, s);
    }
    if (pmode == kPmPScalar) return pm_launch<T, I, MODE, FORM, kPmPScalar, false>(rowptr, col, args, n_rows, plan, s);
    if (pmode == kPmPChannel) return pm_launch<T, I, MODE, FORM, kPmPChannel, false>(rowptr, col, args, n_rows, plan, s);
    return pm_launch<T, I, MODE, FORM, kPmPNone, false>(rowptr, col, args, n_rows, plan, s);
}

template <typename T, typename I, int MODE>
int pm_typed(const void* rowptr_, const void* col_, PmArgs args, int form, int pmode, bool want_p, int64_t n_rows,
             LongRowPlan plan, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    switch (form) {
        case kSmX: return pm_dispatch_p<T, I, MODE, kSmX>(rowptr, col, args, pmode, want_p, n_rows, plan, s);
        case kSmXRelu: return pm_dispatch_p<T, I, MODE, kSmXRelu>(rowptr, col, args, pmode, want_p, n_rows, plan, s);
        case kSmXARelu: return pm_dispatch_p<T, I, MODE, kSmXARelu>(rowptr, col, args, pmode, want_p, n_rows, plan, s);
        default:
            if (MODE == kPmSrc) break;                    // rows-only messages have no source operand
            return pm_dispatch_p<T, I, MODE, kSmA>(rowptr, col, args, pmode, want_p, n_rows, plan, s);
    }
    set_error("power_mean: the transposed sweep needs x");
    return B200MP_ERR_INVALID_ARG;
}

// Sweep CTAs of a grad_p-collecting sweep over n_rows rows (an upper bound over both kernels: a vector CTA holds at
// least 4 work items, a scalar CTA 8), and the node kernel's CTAs.
inline int64_t pm_sweep_ctas(int64_t n_rows, int64_t n_chunks) { return ceil_div(n_rows + n_chunks, 4); }
inline int64_t pm_node_ctas(int64_t n_node) { return ceil_div(n_node, kPmNodeRows); }

// Fold `parts` fp32 partial rows at ws into grad_p (zeros when there are none).
inline int pm_fold(float* ws, int64_t parts, float* grad_p, int64_t feat, cudaStream_t s) {
    if (parts == 0) return cudaMemsetAsync(grad_p, 0, feat * sizeof(float), s) == cudaSuccess ? B200MP_OK : B200MP_ERR_CUDA;
    return b200mp_column_sum(ws, grad_p, ws + parts * feat, b200mp_column_sum_parts(parts), parts, feat, B200MP_F32, s);
}

template <typename T, typename I>
int pm_dst(const void* rowptr, const void* col, PmArgs a, int form, int p_mode, float* grad_p, float* ws,
           int64_t n_rows, LongRowPlan plan, cudaStream_t s) {
    int lg;
    bool vec;
    const int64_t ctas = pm_grid<T>(a, plan, n_rows, lg, vec);
    a.gp_part = ws;
    const int rc = pm_typed<T, I, kPmDst>(rowptr, col, a, form, p_mode, grad_p != nullptr, n_rows, plan, s);
    if (rc != B200MP_OK || grad_p == nullptr) return rc;
    return pm_fold(ws, ctas, grad_p, a.feat, s);
}

template <typename T, typename I>
int pm_src(const void* rowptr, const void* rowptr_t, const void* col_t, PmArgs a, int form, int p_mode, float* grad_p,
           float* ws, int64_t n_src, int64_t n_dst, LongRowPlan plan, cudaStream_t s) {
    const int64_t F = a.feat;
    a.G = ws;
    float* parts = ws + n_dst * F;
    const int64_t node_ctas = pm_node_ctas(n_dst);
    a.gp_part = parts;
    if (node_ctas > 0) {
        if (grad_p == nullptr) {
            if (p_mode == kPmPScalar)
                power_mean_node_kernel<T, I, kPmPScalar, false><<<static_cast<unsigned>(node_ctas), 256, 0, s>>>(
                    static_cast<const I*>(rowptr), a, n_dst);
            else if (p_mode == kPmPChannel)
                power_mean_node_kernel<T, I, kPmPChannel, false><<<static_cast<unsigned>(node_ctas), 256, 0, s>>>(
                    static_cast<const I*>(rowptr), a, n_dst);
            else
                power_mean_node_kernel<T, I, kPmPNone, false><<<static_cast<unsigned>(node_ctas), 256, 0, s>>>(
                    static_cast<const I*>(rowptr), a, n_dst);
        } else if (p_mode == kPmPScalar) {
            power_mean_node_kernel<T, I, kPmPScalar, true><<<static_cast<unsigned>(node_ctas), 256, 0, s>>>(
                static_cast<const I*>(rowptr), a, n_dst);
        } else {
            power_mean_node_kernel<T, I, kPmPChannel, true><<<static_cast<unsigned>(node_ctas), 256, 0, s>>>(
                static_cast<const I*>(rowptr), a, n_dst);
        }
        B200MP_LAUNCH_CHECK();
    }
    int lg;
    bool vec;
    const int64_t ctas = n_src > 0 ? pm_grid<T>(a, plan, n_src, lg, vec) : 0;
    a.gp_part = parts + node_ctas * F;
    if (n_src > 0) {
        const int rc = pm_typed<T, I, kPmSrc>(rowptr_t, col_t, a, form, p_mode, grad_p != nullptr, n_src, plan, s);
        if (rc != B200MP_OK) return rc;
    }
    return grad_p == nullptr ? B200MP_OK : pm_fold(parts, node_ctas + ctas, grad_p, F, s);
}

}  // namespace b200mp

using namespace b200mp;

#define B200MP_CHECK_PM()                                                                                       \
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);                                  \
    B200MP_CHECK_ARG(message == 0 || message == 1);                                                             \
    B200MP_CHECK_ARG(p_mode >= 0 && p_mode <= 2 && (p_mode == 0 || (p && clamp_min > 0.0f && clamp_max >= clamp_min))); \
    B200MP_CHECK_ARG(message == 1 ? x != nullptr : (x == nullptr) != (edge_rows == nullptr))

extern "C" int b200mp_power_mean_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                     const void* edge_rows, const float* p, void* out, float* mean, int64_t n_rows,
                                     int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps, int p_mode,
                                     float clamp_min, float clamp_max, const int64_t* long_rows,
                                     const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                     float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_PM();
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const PmArgs a{x, edge_rows, p, perm, nullptr, nullptr, mean, nullptr, out, nullptr, feat, eps, clamp_min, clamp_max};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_csr", [&](auto tv, auto ti) {
        return pm_typed<decltype(tv), decltype(ti), kPmFwd>(rowptr, col, a, sm_form(x, edge_rows, message), p_mode, false,
                                                          n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int64_t b200mp_power_mean_workspace(int64_t n_node, int64_t n_rows, int64_t n_chunks, int64_t feat) {
    const int64_t parts = pm_node_ctas(n_node) + pm_sweep_ctas(n_rows, n_chunks);
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
    B200MP_CHECK_PM();
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
    const PmArgs a{x, edge_rows, p, perm, grad_out, out, const_cast<float*>(mean), nullptr, grad_edge_rows, nullptr,
                   feat, eps, clamp_min, clamp_max};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_backward_dst", [&](auto tv, auto ti) {
        return pm_dst<decltype(tv), decltype(ti)>(rowptr, col, a, sm_form(x, edge_rows, message), p_mode, grad_p,
                                                  workspace, n_rows, plan, static_cast<cudaStream_t>(stream));
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
    const int64_t n_rows = n_src, n_cols = n_dst;
    B200MP_CHECK_PM();
    B200MP_CHECK_ARG(x != nullptr);
    B200MP_CHECK_ARG(grad_p == nullptr || p_mode != 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (feat == 0) return B200MP_OK;
    if (n_src == 0 && grad_p == nullptr) return B200MP_OK;
    B200MP_CHECK_ARG(workspace && rowptr && rowptr_t && (n_src == 0 || grad_x));
    B200MP_CHECK_ARG(n_dst == 0 || (out && grad_out && (p_mode == 0 || mean)));
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && (edge_rows == nullptr || perm_t)));
    const PmArgs a{x, edge_rows, p, perm_t, grad_out, out, const_cast<float*>(mean), nullptr, grad_x, nullptr, feat,
                   eps, clamp_min, clamp_max};
    return dispatch_val_idx(val_dtype, idx_dtype, "power_mean_backward_src", [&](auto tv, auto ti) {
        return pm_src<decltype(tv), decltype(ti)>(rowptr, rowptr_t, col_t, a, sm_form(x, edge_rows, message), p_mode,
                                                  grad_p, workspace, n_src, n_dst, plan,
                                                  static_cast<cudaStream_t>(stream));
    });
}
