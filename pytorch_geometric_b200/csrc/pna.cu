// pna.cu -- PNAConv's pre-transform, multi-aggregation and degree scalers around one CSR sweep.
//
// With one pre-layer per tower, the message of edge e = (j -> i) splits into a destination part and a per-edge part
// (the tower Linear on cat(x_i, x_j, enc(edge_attr)), pna_conv.py:167-188, split by weight column blocks):
//     m_e = u_i + w_e,    u = x_t Wa_t^T + b_t,    w_e = v_j (+ c_e),    v = x_t Wb_t^T,    c = enc(edge_attr) Wc_t^T
// with every tower side by side in one width W = T * F.  The sweep only needs the statistics of w; the shift by u is
// applied per destination:
//     sum = deg u + sum w     mean = sum / max(deg, 1)     min = u + min w     max = u + max w     (0 for an empty row)
//     var, std: shift-invariant, from the statistics of w (fused.py:319-325's clamp / sqrt / zeroing)
// Without edge features the statistics come from b200mp_multi_aggr_csr in gather mode on v; with them, from
// pna_edge_stats_kernel below (w_e = v[col[e]] + c[perm[e]] rounded to the storage dtype, c read in the caller's edge
// order).  Either way these kernels complete the layer's aggregation:
//   pna_epilogue_kernel      the aggregators, the scalers (scaler.py:92-107) and the x slot, written straight into
//                            the post-network input [N, T, (1 + A S) F] (pna_conv.py:169)
//   pna_prologue_kernel      the gradient of that block folded into what the sweep backward reads (term_a, term_b,
//                            g_min / ties, g_max / ties), the closed-form grad_u, the x-slot gradient and per-row
//                            partials of the avg_deg gradients
//   pna_edge_backward_kernel (edge features only) one transposed-CSR sweep: grad_v per source row, grad_c per edge
// Ties of min / max are counted on w; the zero-initialised self of the reference's scatter (the engine's
// count_self_zero rule) is a tie of the SHIFTED extremum, so it is added by the prologue, not the sweep.
#include "csr_reduce.cuh"

namespace b200mp {

enum { PA_SUM = 0, PA_MEAN, PA_MIN, PA_MAX, PA_VAR, PA_STD, PA_KINDS };
enum { PS_IDENTITY = 0, PS_AMPLIFICATION, PS_ATTENUATION, PS_LINEAR, PS_INVERSE_LINEAR };
constexpr int kPnaMaxAggr = 6, kPnaMaxScaler = 5;    // the supported aggregators and scalers, each at most once

struct PnaShape {
    int n_aggr, n_scaler;
    int aggr[kPnaMaxAggr];
    int scaler[kPnaMaxScaler];
    int64_t towers, feat;                 // W = towers * feat
    const float* avg_lin;                 // device scalars (the module's avg_deg_lin / avg_deg_log)
    const float* avg_log;
};

struct PnaStats {                         // statistics of w, [n_rows, W]: sum / min / max / var of dtype S, ties fp32
    const void *sum, *mn, *mx, *var;
    const float *ties_min, *ties_max;
};

// scaler factor (scaler.py:92-107) for a degree already rounded to the output dtype
__device__ __forceinline__ float pna_factor(int s, float d, float lin, float lg) {
    switch (s) {
        case PS_AMPLIFICATION: return logf(d + 1.f) / lg;
        case PS_ATTENUATION: return lg / logf(fmaxf(d, 1.f) + 1.f);
        case PS_LINEAR: return d / lin;
        case PS_INVERSE_LINEAR: return lin / fmaxf(d, 1.f);
        default: return 1.f;
    }
}
// d factor / d avg_deg_lin and d factor / d avg_deg_log
__device__ __forceinline__ void pna_factor_grad(int s, float f, float lin, float lg, float& d_lin, float& d_log) {
    d_lin = s == PS_LINEAR ? -f / lin : s == PS_INVERSE_LINEAR ? f / lin : 0.f;
    d_log = s == PS_AMPLIFICATION ? -f / lg : s == PS_ATTENUATION ? f / lg : 0.f;
}

// Every aggregator of one (row, column) from the statistics of w, rounded to the output dtype as the reference's
// separate aggregation modules produce them.
template <typename T, typename S>
__device__ __forceinline__ void pna_aggregates(const PnaStats& st, size_t di, float u, int64_t deg, float (&agg)[PA_KINDS],
                                               float& sum_w) {
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    auto ld = [&](const void* p) { return p ? ElemTraits<S>::to_float(static_cast<const S*>(p)[di]) : 0.f; };
    sum_w = ld(st.sum);
    const float s = __fadd_rn(__fmul_rn(static_cast<float>(deg), u), sum_w);
    agg[PA_SUM] = round_to<T>(s);
    agg[PA_MEAN] = round_to<T>(__fdiv_rn(s, cnt));
    agg[PA_MIN] = deg == 0 ? 0.f : round_to<T>(__fadd_rn(u, ld(st.mn)));
    agg[PA_MAX] = deg == 0 ? 0.f : round_to<T>(__fadd_rn(u, ld(st.mx)));
    const float var = ld(st.var);
    float sd = __fsqrt_rn(var < 1e-5f ? 1e-5f : var);
    if (sd <= static_cast<float>(0.0031622776601683794)) sd = 0.f;            // math.sqrt(1e-5), basic.py:136
    agg[PA_VAR] = round_to<T>(var);
    agg[PA_STD] = round_to<T>(sd);
}

// agg[kind] without a dynamically indexed (local-memory) array
__device__ __forceinline__ float pna_pick(const float (&agg)[PA_KINDS], int kind) {
    float r = agg[0];
#pragma unroll
    for (int k = 1; k < PA_KINDS; ++k) r = kind == k ? agg[k] : r;
    return r;
}

// One warp per destination row; lanes walk the W = T * F columns.
template <typename T, typename S, typename I>
__global__ void __launch_bounds__(128)
pna_epilogue_kernel(const I* __restrict__ rowptr, const T* __restrict__ x, const T* __restrict__ u, int64_t u_ld,
                    PnaStats st, PnaShape sh, T* __restrict__ out, int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_rows) return;
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const float d = round_to<T>(static_cast<float>(deg));       // degree(..., dtype=out.dtype) on the CPU, scaler.py:82
    const float lin = *sh.avg_lin, lg = *sh.avg_log;
    float fac[kPnaMaxScaler];
#pragma unroll
    for (int s = 0; s < kPnaMaxScaler; ++s) fac[s] = s < sh.n_scaler ? round_to<T>(pna_factor(sh.scaler[s], d, lin, lg)) : 0.f;
    const int64_t W = sh.towers * sh.feat, slots = 1 + static_cast<int64_t>(sh.n_aggr) * sh.n_scaler;
    T* orow = out + static_cast<size_t>(row) * W * slots;
    for (int64_t c = lane; c < W; c += 32) {
        const int64_t t = c / sh.feat, f = c - t * sh.feat;
        const size_t di = static_cast<size_t>(row) * W + c;
        float agg[PA_KINDS], sum_w;
        pna_aggregates<T, S>(st, di, ElemTraits<T>::to_float(u[static_cast<size_t>(row) * u_ld + c]), deg, agg, sum_w);
        T* o = orow + t * slots * sh.feat + f;
        o[0] = x[di];
#pragma unroll
        for (int s = 0; s < kPnaMaxScaler; ++s) {
            if (s >= sh.n_scaler) break;
#pragma unroll
            for (int a = 0; a < kPnaMaxAggr; ++a) {
                if (a >= sh.n_aggr) break;
                o[(1 + s * sh.n_aggr + a) * sh.feat] = ElemTraits<T>::from_float(__fmul_rn(pna_pick(agg, sh.aggr[a]), fac[s]));
            }
        }
    }
}

struct PnaBwd {
    const void* grad_out;                 // [N, T, (1 + A S) F], value dtype
    float *term_a, *term_b, *gmin, *gmax; // [N, W] fp32, each nullable
    void* grad_u;                         // [N, W] rows of stride gu_ld, value dtype, nullable
    int64_t gu_ld;
    void* grad_x;                         // [N, W] value dtype (the x slot), nullable
    float* avg_part;                      // [N, 2] fp32: per-row d L / d avg_deg_lin, d L / d avg_deg_log; nullable
};

template <typename T, typename S, typename I>
__global__ void __launch_bounds__(128)
pna_prologue_kernel(const I* __restrict__ rowptr, const T* __restrict__ u, int64_t u_ld, PnaStats st, PnaShape sh,
                    PnaBwd b, int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_rows) return;
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    const float d = round_to<T>(static_cast<float>(deg));
    const float lin = *sh.avg_lin, lg = *sh.avg_log;
    float fac[kPnaMaxScaler], dlin[kPnaMaxScaler], dlog[kPnaMaxScaler];
#pragma unroll
    for (int s = 0; s < kPnaMaxScaler; ++s) {
        fac[s] = s < sh.n_scaler ? round_to<T>(pna_factor(sh.scaler[s], d, lin, lg)) : 0.f;
        pna_factor_grad(s < sh.n_scaler ? sh.scaler[s] : PS_IDENTITY, fac[s], lin, lg, dlin[s], dlog[s]);
    }
    const int64_t W = sh.towers * sh.feat, slots = 1 + static_cast<int64_t>(sh.n_aggr) * sh.n_scaler;
    const T* grow = static_cast<const T*>(b.grad_out) + static_cast<size_t>(row) * W * slots;
    float p_lin = 0.f, p_log = 0.f;
    for (int64_t c = lane; c < W; c += 32) {
        const int64_t t = c / sh.feat, f = c - t * sh.feat;
        const size_t di = static_cast<size_t>(row) * W + c;
        const T* gp = grow + t * slots * sh.feat + f;
        float agg[PA_KINDS], sum_w;
        pna_aggregates<T, S>(st, di, ElemTraits<T>::to_float(u[static_cast<size_t>(row) * u_ld + c]), deg, agg, sum_w);
        float ga[PA_KINDS] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int s = 0; s < kPnaMaxScaler; ++s) {
            if (s >= sh.n_scaler) break;
            float gs = 0.f;
#pragma unroll
            for (int a = 0; a < kPnaMaxAggr; ++a) {
                if (a >= sh.n_aggr) break;
                const int kind = sh.aggr[a];
                const float g = ElemTraits<T>::to_float(gp[(1 + s * sh.n_aggr + a) * sh.feat]);
#pragma unroll
                for (int k = 0; k < PA_KINDS; ++k)
                    if (k == kind) ga[k] += g * fac[s];
                gs += g * pna_pick(agg, kind);
            }
            p_lin += gs * dlin[s];
            p_log += gs * dlog[s];
        }
        if (b.grad_x) static_cast<T*>(b.grad_x)[di] = gp[0];
        // per-edge terms of d L / d w_e = term_a + w_e term_b + [w_e == min w] gmin + [w_e == max w] gmax
        const float mean_w = __fdiv_rn(sum_w, cnt);
        float ta = ga[PA_SUM] + ga[PA_MEAN] / cnt;
        float gv = ga[PA_VAR];
        if (agg[PA_STD] > 0.f) gv += ga[PA_STD] * 0.5f / agg[PA_STD];
        ta -= 2.f * gv * mean_w / cnt;
        if (b.term_a) b.term_a[di] = ta;
        if (b.term_b) b.term_b[di] = 2.f * gv / cnt;
        // the reference's scatter counts its zero-initialised self as a tie when the (shifted) extremum is 0
        const float cmn = st.ties_min ? st.ties_min[di] : 0.f, cmx = st.ties_max ? st.ties_max[di] : 0.f;
        const float gmn = ga[PA_MIN] / fmaxf(cmn + (agg[PA_MIN] == 0.f ? 1.f : 0.f), 1.f);
        const float gmx = ga[PA_MAX] / fmaxf(cmx + (agg[PA_MAX] == 0.f ? 1.f : 0.f), 1.f);
        if (b.gmin) b.gmin[di] = gmn;
        if (b.gmax) b.gmax[di] = gmx;
        // d L / d u_i = sum over the in-edges of d L / d m_e: var and std do not depend on the shift
        if (b.grad_u) {
            const float gu = static_cast<float>(deg) * ga[PA_SUM] + (deg > 0 ? ga[PA_MEAN] : 0.f) + gmn * cmn + gmx * cmx;
            static_cast<T*>(b.grad_u)[static_cast<size_t>(row) * b.gu_ld + c] = ElemTraits<T>::from_float(gu);
        }
    }
    if (b.avg_part) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            p_lin += __shfl_xor_sync(0xffffffffu, p_lin, o);
            p_log += __shfl_xor_sync(0xffffffffu, p_log, o);
        }
        if (lane == 0) {
            b.avg_part[2 * row] = p_lin;
            b.avg_part[2 * row + 1] = p_log;
        }
    }
}

// ---------------------------------------------------------------- edge-feature sweep
struct PnaState {
    float s, q, mn, mx, cmn, cmx;
};
__device__ __forceinline__ void ps_init(PnaState& a) {
    a.s = a.q = a.cmn = a.cmx = 0.f;
    a.mn = __int_as_float(0x7f800000);
    a.mx = __int_as_float(0xff800000);
}
__device__ __forceinline__ void ps_push(PnaState& a, float v) {        // the tie rule of multi_aggr.cu's sweep
    a.s = __fadd_rn(a.s, v);
    a.q = __fadd_rn(a.q, __fmul_rn(v, v));
    if (v < a.mn || v != v) { a.mn = v; a.cmn = 1.f; } else if (v == a.mn) a.cmn += 1.f;
    if (v > a.mx || v != v) { a.mx = v; a.cmx = 1.f; } else if (v == a.mx) a.cmx += 1.f;
}
__device__ __forceinline__ void ps_merge(PnaState& a, const PnaState& b) {   // a then b, in edge order
    a.s = __fadd_rn(a.s, b.s);
    a.q = __fadd_rn(a.q, b.q);
    if (b.mn < a.mn || b.mn != b.mn) { a.mn = b.mn; a.cmn = b.cmn; } else if (b.mn == a.mn) a.cmn += b.cmn;
    if (b.mx > a.mx || b.mx != b.mx) { a.mx = b.mx; a.cmx = b.cmx; } else if (b.mx == a.mx) a.cmx += b.cmx;
}

struct PnaStatsOut {                      // fp32 [n_rows, W] planes, each nullable
    float *sum, *mn, *mx, *var, *ties_min, *ties_max;
};

__device__ __forceinline__ void ps_store(const PnaStatsOut& o, size_t di, const PnaState& a, int64_t deg) {
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    const float mean = __fdiv_rn(a.s, cnt);
    if (o.sum) o.sum[di] = a.s;
    if (o.mn) o.mn[di] = deg == 0 ? 0.f : a.mn;
    if (o.mx) o.mx[di] = deg == 0 ? 0.f : a.mx;
    if (o.var) o.var[di] = __fsub_rn(__fdiv_rn(a.q, cnt), __fmul_rn(mean, mean));
    if (o.ties_min) o.ties_min[di] = a.cmn;
    if (o.ties_max) o.ties_max[di] = a.cmx;
}

// w of CSR slot e for column cidx: v[col[e]] + c[perm[e]] rounded to the storage dtype (the message the reference's
// Linear would produce in that dtype, before the destination's shift)
template <typename T>
__device__ __forceinline__ float pna_w(const T* v, int64_t v_ld, const T* c, int64_t W, int64_t j, int64_t ce, int64_t cidx) {
    return round_to<T>(__fadd_rn(ElemTraits<T>::to_float(v[static_cast<size_t>(j) * v_ld + cidx]),
                                  ElemTraits<T>::to_float(c[static_cast<size_t>(ce) * W + cidx])));
}

// One warp per work item (a row, or a chunk of a hub row); a lane keeps K columns' running state, so the row's index
// arrays are read once per 32 K columns.
template <typename T, typename I, int K>
__global__ void __launch_bounds__(128)
pna_edge_stats_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const I* __restrict__ perm,
                      const T* __restrict__ v, int64_t v_ld, const T* __restrict__ c, PnaStatsOut so, int64_t n_rows,
                      int64_t W, LongRowPlan plan) {
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    for (int64_t c0 = 0; c0 < W; c0 += 32 * K) {
        PnaState a[K];
#pragma unroll
        for (int k = 0; k < K; ++k) ps_init(a[k]);
#pragma unroll 2
        for (int64_t e = begin; e < end; ++e) {
            const int64_t j = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t ce = perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int64_t cidx = c0 + lane + 32 * k;
                if (cidx < W) ps_push(a[k], pna_w<T>(v, v_ld, c, W, j, ce, cidx));
            }
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int64_t cidx = c0 + lane + 32 * k;
            if (cidx >= W) continue;
            if (is_chunk) {                                          // partial state: [n_chunks][6][W] fp32
                float* pb = plan.partials + static_cast<size_t>(item) * 6 * W + cidx;
                pb[0] = a[k].s;
                pb[W] = a[k].q;
                pb[2 * W] = a[k].mn;
                pb[3 * W] = a[k].mx;
                pb[4 * W] = a[k].cmn;
                pb[5 * W] = a[k].cmx;
            } else {
                ps_store(so, static_cast<size_t>(row) * W + cidx, a[k], end - begin);
            }
        }
    }
}

// Fold the chunk states of every hub row in chunk (= edge) order.
template <typename I>
__global__ void __launch_bounds__(256)
pna_edge_combine_kernel(const I* __restrict__ rowptr, PnaStatsOut so, int64_t W, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = threadIdx.x; f < W; f += blockDim.x) {
        PnaState a;
        ps_init(a);
        for (int64_t ch = c0; ch < c1; ++ch) {
            const float* pb = plan.partials + static_cast<size_t>(ch) * 6 * W + f;
            const PnaState b{pb[0], pb[W], pb[2 * W], pb[3 * W], pb[4 * W], pb[5 * W]};
            ps_merge(a, b);
        }
        ps_store(so, static_cast<size_t>(row) * W + f, a, deg);
    }
}

struct PnaEdgeGrad {
    const float *term_a, *term_b, *mn, *gmin, *mx, *gmax;     // [n_dst, W] fp32, each nullable
};

// One warp per SOURCE row of the transposed CSR: d L / d w_e of every out-edge is written to grad_c[e] (caller's edge
// order) and summed in registers into grad_v[j] -- both gradients from one sweep, no atomics.
template <typename T, typename I, int K>
__global__ void __launch_bounds__(128)
pna_edge_backward_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t, const I* __restrict__ perm_t,
                         const T* __restrict__ v, int64_t v_ld, const T* __restrict__ c, PnaEdgeGrad g,
                         T* __restrict__ grad_v, int64_t gv_ld, T* __restrict__ grad_c, int64_t n_src, int64_t W) {
    const int lane = threadIdx.x & 31;
    const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (j >= n_src) return;
    const int64_t begin = static_cast<int64_t>(rowptr_t[j]), end = static_cast<int64_t>(rowptr_t[j + 1]);
    for (int64_t c0 = 0; c0 < W; c0 += 32 * K) {
        float acc[K];
#pragma unroll
        for (int k = 0; k < K; ++k) acc[k] = 0.f;
        for (int64_t p = begin; p < end; ++p) {
            const int64_t i = static_cast<int64_t>(ldg_idx(col_t + p));
            const int64_t ce = static_cast<int64_t>(ldg_idx(perm_t + p));
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int64_t cidx = c0 + lane + 32 * k;
                if (cidx >= W) continue;
                const float w = pna_w<T>(v, v_ld, c, W, j, ce, cidx);
                const size_t di = static_cast<size_t>(i) * W + cidx;
                float t = g.term_a ? __ldg(g.term_a + di) : 0.f;
                if (g.term_b) t = fmaf(w, __ldg(g.term_b + di), t);
                if (g.gmin && w == __ldg(g.mn + di)) t += __ldg(g.gmin + di);
                if (g.gmax && w == __ldg(g.mx + di)) t += __ldg(g.gmax + di);
                if (grad_c) grad_c[static_cast<size_t>(ce) * W + cidx] = ElemTraits<T>::from_float(t);
                acc[k] = __fadd_rn(acc[k], t);
            }
        }
        if (grad_v) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const int64_t cidx = c0 + lane + 32 * k;
                if (cidx < W) grad_v[static_cast<size_t>(j) * gv_ld + cidx] = ElemTraits<T>::from_float(acc[k]);
            }
        }
    }
}

inline unsigned pna_warp_blocks(int64_t n) { return static_cast<unsigned>(ceil_div(n, 4)); }   // 4 warps per CTA

template <typename T, typename I>
int pna_epilogue_typed(const void* rowptr, const void* x, const void* u, int64_t u_ld, PnaStats st, PnaShape sh, void* out,
                       int64_t n_rows, int stats_f32, cudaStream_t stream) {
    if (stats_f32)
        pna_epilogue_kernel<T, float, I><<<pna_warp_blocks(n_rows), 128, 0, stream>>>(
            static_cast<const I*>(rowptr), static_cast<const T*>(x), static_cast<const T*>(u), u_ld, st, sh, static_cast<T*>(out), n_rows);
    else
        pna_epilogue_kernel<T, T, I><<<pna_warp_blocks(n_rows), 128, 0, stream>>>(
            static_cast<const I*>(rowptr), static_cast<const T*>(x), static_cast<const T*>(u), u_ld, st, sh, static_cast<T*>(out), n_rows);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename T, typename I>
int pna_prologue_typed(const void* rowptr, const void* u, int64_t u_ld, PnaStats st, PnaShape sh, PnaBwd b, int64_t n_rows,
                       int stats_f32, cudaStream_t stream) {
    if (stats_f32)
        pna_prologue_kernel<T, float, I><<<pna_warp_blocks(n_rows), 128, 0, stream>>>(
            static_cast<const I*>(rowptr), static_cast<const T*>(u), u_ld, st, sh, b, n_rows);
    else
        pna_prologue_kernel<T, T, I><<<pna_warp_blocks(n_rows), 128, 0, stream>>>(
            static_cast<const I*>(rowptr), static_cast<const T*>(u), u_ld, st, sh, b, n_rows);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename T, typename I>
int pna_edge_stats_typed(const void* rowptr, const void* col, const void* perm, const void* v, int64_t v_ld, const void* c,
                         PnaStatsOut so, int64_t n_rows, int64_t W, LongRowPlan plan, cudaStream_t stream) {
    const int64_t items = plan.n_chunks + n_rows;
#define B200MP_PNA_STATS(K_)                                                                                              \
    pna_edge_stats_kernel<T, I, K_><<<pna_warp_blocks(items), 128, 0, stream>>>(                                         \
        static_cast<const I*>(rowptr), static_cast<const I*>(col), static_cast<const I*>(perm), static_cast<const T*>(v), \
        v_ld, static_cast<const T*>(c), so, n_rows, W, plan)
    if (W <= 32) B200MP_PNA_STATS(1);
    else if (W <= 64) B200MP_PNA_STATS(2);
    else B200MP_PNA_STATS(4);
#undef B200MP_PNA_STATS
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        pna_edge_combine_kernel<I><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(static_cast<const I*>(rowptr), so, W, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int pna_edge_backward_typed(const void* rowptr_t, const void* col_t, const void* perm_t, const void* v, int64_t v_ld,
                            const void* c, PnaEdgeGrad g, void* grad_v, int64_t gv_ld, void* grad_c, int64_t n_src, int64_t W,
                            cudaStream_t stream) {
#define B200MP_PNA_BWD(K_)                                                                                                \
    pna_edge_backward_kernel<T, I, K_><<<pna_warp_blocks(n_src), 128, 0, stream>>>(                                      \
        static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t), static_cast<const I*>(perm_t),                    \
        static_cast<const T*>(v), v_ld, static_cast<const T*>(c), g, static_cast<T*>(grad_v), gv_ld, static_cast<T*>(grad_c), \
        n_src, W)
    if (W <= 32) B200MP_PNA_BWD(1);
    else if (W <= 64) B200MP_PNA_BWD(2);
    else B200MP_PNA_BWD(4);
#undef B200MP_PNA_BWD
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

inline int pna_shape(PnaShape& sh, const int32_t* aggr_host, int n_aggr, const int32_t* scaler_host, int n_scaler,
                     int64_t towers, int64_t feat, const float* avg_lin, const float* avg_log) {
    B200MP_CHECK_ARG(n_aggr >= 1 && n_aggr <= kPnaMaxAggr && n_scaler >= 1 && n_scaler <= kPnaMaxScaler);
    B200MP_CHECK_ARG(aggr_host && scaler_host && avg_lin && avg_log && towers >= 1 && feat >= 0);
    sh = PnaShape{};
    sh.n_aggr = n_aggr;
    sh.n_scaler = n_scaler;
    for (int a = 0; a < n_aggr; ++a) {
        B200MP_CHECK_ARG(aggr_host[a] >= PA_SUM && aggr_host[a] <= PA_STD);
        sh.aggr[a] = aggr_host[a];
    }
    for (int s = 0; s < n_scaler; ++s) {
        B200MP_CHECK_ARG(scaler_host[s] >= PS_IDENTITY && scaler_host[s] <= PS_INVERSE_LINEAR);
        sh.scaler[s] = scaler_host[s];
    }
    sh.towers = towers;
    sh.feat = feat;
    sh.avg_lin = avg_lin;
    sh.avg_log = avg_log;
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_pna_epilogue(const void* rowptr, const void* x, const void* u, int64_t u_ld, const void* stat_sum,
                                   const void* stat_min, const void* stat_max, const void* stat_var,
                                   const int32_t* aggr_host, int n_aggr, const int32_t* scaler_host, int n_scaler,
                                   const float* avg_deg_lin, const float* avg_deg_log, void* out, int64_t n_rows,
                                   int64_t towers, int64_t feat, int stats_dtype, int idx_dtype, int val_dtype,
                                   void* stream) {
    PnaShape sh;
    if (const int rc = pna_shape(sh, aggr_host, n_aggr, scaler_host, n_scaler, towers, feat, avg_deg_lin, avg_deg_log)) return rc;
    B200MP_CHECK_ARG(n_rows >= 0 && u_ld >= towers * feat);
    B200MP_CHECK_ARG(stats_dtype == B200MP_F32 || stats_dtype == val_dtype);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && x && u && out);
    const PnaStats st{stat_sum, stat_min, stat_max, stat_var, nullptr, nullptr};
    return dispatch_val_idx(val_dtype, idx_dtype, "pna_epilogue", [&](auto tv, auto ti) {
        return pna_epilogue_typed<decltype(tv), decltype(ti)>(rowptr, x, u, u_ld, st, sh, out, n_rows,
                                                              stats_dtype == B200MP_F32 && val_dtype != B200MP_F32,
                                                              static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_pna_prologue(const void* rowptr, const void* grad_out, const void* u, int64_t u_ld,
                                   const void* stat_sum, const void* stat_min, const void* stat_max, const void* stat_var,
                                   const float* ties_min, const float* ties_max, const int32_t* aggr_host, int n_aggr,
                                   const int32_t* scaler_host, int n_scaler, const float* avg_deg_lin,
                                   const float* avg_deg_log, float* term_a, float* term_b, float* gmin, float* gmax,
                                   void* grad_u, int64_t gu_ld, void* grad_x, float* avg_part, int64_t n_rows,
                                   int64_t towers, int64_t feat, int stats_dtype, int idx_dtype, int val_dtype,
                                   void* stream) {
    PnaShape sh;
    if (const int rc = pna_shape(sh, aggr_host, n_aggr, scaler_host, n_scaler, towers, feat, avg_deg_lin, avg_deg_log)) return rc;
    B200MP_CHECK_ARG(n_rows >= 0 && u_ld >= towers * feat && (!grad_u || gu_ld >= towers * feat));
    B200MP_CHECK_ARG(stats_dtype == B200MP_F32 || stats_dtype == val_dtype);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && grad_out && u);
    B200MP_CHECK_ARG(!gmin || (stat_min && ties_min));
    B200MP_CHECK_ARG(!gmax || (stat_max && ties_max));
    const PnaStats st{stat_sum, stat_min, stat_max, stat_var, ties_min, ties_max};
    const PnaBwd b{grad_out, term_a, term_b, gmin, gmax, grad_u, gu_ld, grad_x, avg_part};
    return dispatch_val_idx(val_dtype, idx_dtype, "pna_prologue", [&](auto tv, auto ti) {
        return pna_prologue_typed<decltype(tv), decltype(ti)>(rowptr, u, u_ld, st, sh, b, n_rows,
                                                              stats_dtype == B200MP_F32 && val_dtype != B200MP_F32,
                                                              static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_pna_edge_stats(const void* rowptr, const void* col, const void* perm, const void* v, int64_t v_ld,
                                     const void* c, float* stat_sum, float* stat_min, float* stat_max, float* stat_var,
                                     float* ties_min, float* ties_max, int64_t n_rows, int64_t n_cols, int64_t n_edges,
                                     int64_t width, const int64_t* long_rows, const int64_t* chunk_ptr,
                                     int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype,
                                     int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && width >= 0 && v_ld >= width);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || width == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && (n_edges == 0 || (col && v && c)));
    const PnaStatsOut so{stat_sum, stat_min, stat_max, stat_var, ties_min, ties_max};
    return dispatch_val_idx(val_dtype, idx_dtype, "pna_edge_stats", [&](auto tv, auto ti) {
        return pna_edge_stats_typed<decltype(tv), decltype(ti)>(rowptr, col, perm, v, v_ld, c, so, n_rows, width, plan,
                                                                static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_pna_edge_backward(const void* rowptr_t, const void* col_t, const void* perm_t, const void* v,
                                        int64_t v_ld, const void* c, const float* term_a, const float* term_b,
                                        const float* stat_min, const float* gmin, const float* stat_max,
                                        const float* gmax, void* grad_v, int64_t gv_ld, void* grad_c, int64_t n_src,
                                        int64_t n_dst, int64_t n_edges, int64_t width, int idx_dtype, int val_dtype,
                                        void* stream) {
    B200MP_CHECK_ARG(n_src >= 0 && n_dst >= 0 && n_edges >= 0 && width >= 0 && v_ld >= width);
    B200MP_CHECK_ARG(!grad_v || gv_ld >= width);
    if (n_src == 0 || width == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && v && (grad_v || grad_c));
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && perm_t && c));
    B200MP_CHECK_ARG((!gmin || stat_min) && (!gmax || stat_max));
    const PnaEdgeGrad g{term_a, term_b, stat_min, gmin, stat_max, gmax};
    return dispatch_val_idx(val_dtype, idx_dtype, "pna_edge_backward", [&](auto tv, auto ti) {
        return pna_edge_backward_typed<decltype(tv), decltype(ti)>(rowptr_t, col_t, perm_t, v, v_ld, c, g, grad_v, gv_ld,
                                                                   grad_c, n_src, width, static_cast<cudaStream_t>(stream));
    });
}
