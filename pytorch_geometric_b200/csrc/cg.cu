// cg.cu -- CGConv's crystal-graph message sigmoid(z W_f + b_f) * softplus(z W_s + b_s), z = [x_i, x_j, e_ji], fused
// into the CSR gather-reduce, and its backward.
//
// The layer's two Linears are split by weight column blocks into per-node and per-edge products (nn/conv.py cg_uvc):
//   u = x_dst [W_f,a; W_s,a]^T + [b_f; b_s]   [n_dst, 2F]      v = x_src [W_f,b; W_s,b]^T   [n_src, 2F]
//   c = edge_attr [W_f,c; W_s,c]^T            [E, 2F] in the caller's edge order, or absent (dim = 0)
// Each row holds the f half in [0, F) and the s half in [F, 2F).  Per edge e = (j -> i) and feature k:
//   f = u_f[i] + v_f[j] (+ c_f[eid(e)]),  s = likewise,  each summed in fp32 and rounded to the storage dtype once
//   out[i,:] = REDUCE_{e in row i} round(round(sigma(f)) * round(softplus(s)))          REDUCE = sum | mean
// eid(e) = perm[e] (CSR slot -> the caller's edge id), or e for an adopted CSR (perm == NULL).  Nothing per edge is
// stored: the backward recomputes f and s.  With g_i = grad_out[i,:] / (mean ? max(deg_i, 1) : 1),
//   df = g_i sigma'(f) softplus(s),  ds = g_i sigma(f) softplus'(s)
//   grad_u[i] = sum_{e in row i} (df, ds), and grad_c[eid(e)] = (df, ds) in the same sweep  (destination CSR)
//   grad_v[j] = sum_{t in rowT(j)} (df, ds)                                                  (transposed CSR)
// When grad_c exists, grad_v is the segment sum of its rows over the transposed CSR (b200mp_spmm_csr with perm_t as
// the column), which reads less than the transposed sweep here.
//
// Numerics: softplus follows ATen's threshold 20 -- s > 20 gives s (derivative exactly 1), otherwise
// max(s, 0) + log1p(t) with t = exp(-|s|), and softplus' = sigma(s) from the same t.  sigma and sigma' of f come from
// sigmoid_pair (gate_math.cuh).  s = -inf gives 0, s = +inf gives +inf, NaN stays NaN, and 0 * inf products give NaN
// as in the reference.
//
// Mapping as in gated.cu: a lane group of G lanes per row, one 16-byte vector of the f half (and the matching vector of
// the s half) per lane and trip, rows longer than the plan's chunk split into chunks whose fp32 partials
// cg_combine_kernel folds in chunk order.  Rows that are not a whole number of aligned 16-byte vectors take a one-warp
// scalar kernel.
#include "csr_reduce.cuh"
#include "gate_math.cuh"

namespace b200mp {

enum CgMode { kCgFwd = 0, kCgDst = 1, kCgSrc = 2 };

struct CgArgs {
    const void* u;       // [n_dst, ld_u]
    const void* v;       // [n_src, ld_v]
    const void* c;       // [n_edges, 2 feat] in the caller's edge order, or null
    const void* perm;    // index dtype: caller's edge id of each CSR (fwd / dst) or transposed (src) slot; null = slot
    const void* g;       // grad_out [n_dst, feat] (backward)
    const float* val_t;  // per transposed slot, 1 / max(deg_dst, 1) for mean (source sweep), or null
    void* out;           // fwd: out [n_dst, feat]; dst: grad_u [n_dst, ld_u]; src: grad_v [n_src, ld_v]
    void* grad_c;        // dst: [n_edges, 2 feat] or null
    int64_t feat;
    int64_t ld_u;
    int64_t ld_v;
    bool is_mean;
};

// log1p(t) for t in [0, 1] (NaN stays NaN): 2 atanh(y) with y = t / (2 + t) in [0, 1/3], i.e. 2 y (1 + z/3 + z^2/5 +
// ... + z^7/15) with z = y^2; the truncation error is below 2e-9 relative.  One MUFU operation and ten FMA-pipe
// operations without branches, where log1pf's range reduction costs about twice as many and a branch.
__device__ __forceinline__ float log1p_unit(float t) {
    const float y = __fdividef(t, 2.0f + t);
    const float z = __fmul_rn(y, y);
    float p = 1.0f / 15.0f;
    p = fmaf(p, z, 1.0f / 13.0f);
    p = fmaf(p, z, 1.0f / 11.0f);
    p = fmaf(p, z, 1.0f / 9.0f);
    p = fmaf(p, z, 1.0f / 7.0f);
    p = fmaf(p, z, 1.0f / 5.0f);
    p = fmaf(p, z, 1.0f / 3.0f);
    p = fmaf(p, z, 1.0f);
    return __fmul_rn(__fmul_rn(2.0f, y), p);
}

// softplus(s) with ATen's threshold 20, and its derivative, from one t = exp(-|s|).
__device__ __forceinline__ void softplus_pair(float s, float& sp, float& dsp) {
    const float t = __expf(-fabsf(s));
    const float r = __fdividef(1.0f, 1.0f + t);
    const bool lin = s > 20.0f;
    sp = lin ? s : __fadd_rn(fmaxf(s, 0.0f), log1p_unit(t));
    dsp = lin ? 1.0f : (s >= 0.0f ? r : __fmul_rn(t, r));
}

// One (edge, feature) term from the fp32 pre-activation sums pf, ps.  fwd: acc0 += the rounded message.  dst / src:
// df, ds with the (weighted) gradient row gw; acc0 += df, acc1 += ds.
template <typename T, int MODE>
__device__ __forceinline__ void cg_term(float pf, float ps, float gw, float& acc0, float& acc1, float& df, float& ds) {
    const float f = round_to<T>(pf), s = round_to<T>(ps);
    float sig, dsig, sp, dsp;
    sigmoid_pair(f, sig, dsig);
    softplus_pair(s, sp, dsp);
    if (MODE == kCgFwd) {
        acc0 = __fadd_rn(acc0, round_to<T>(__fmul_rn(round_to<T>(sig), round_to<T>(sp))));
    } else {
        df = __fmul_rn(__fmul_rn(gw, dsig), sp);
        ds = __fmul_rn(__fmul_rn(gw, sig), dsp);
        acc0 = __fadd_rn(acc0, df);
        acc1 = __fadd_rn(acc1, ds);
    }
}

// The row operand (read once per row or chunk) and the gathered operand by mode.
template <typename T, int MODE>
struct CgRoles {
    const T *row, *gat;
    int64_t row_ld, gat_ld, out_ld;
    __device__ __forceinline__ explicit CgRoles(const CgArgs& a) {
        const T* u = static_cast<const T*>(a.u);
        const T* v = static_cast<const T*>(a.v);
        if (MODE == kCgSrc) {
            row = v; row_ld = a.ld_v; gat = u; gat_ld = a.ld_u; out_ld = a.ld_v;
        } else {
            row = u; row_ld = a.ld_u; gat = v; gat_ld = a.ld_v; out_ld = MODE == kCgFwd ? a.feat : a.ld_u;
        }
    }
};

template <typename I>
__device__ __forceinline__ int64_t cg_eid(const CgArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int G, int UNR, bool HAS_C>
__global__ void __launch_bounds__(128)
cg_reduce_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, CgArgs args, int64_t n_rows, int n_vec,
                 LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int NACC = MODE == kCgFwd ? 1 : 2;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // uniform per group
    const CgRoles<T, MODE> R(args);
    const int64_t F = args.feat;
    const size_t half = static_cast<size_t>(F) * sizeof(T);                 // byte offset of the s half
    const size_t gat_bytes = static_cast<size_t>(R.gat_ld) * sizeof(T);
    const size_t g_bytes = half;
    const size_t c_bytes = 2 * half;
    const char* gatb = reinterpret_cast<const char*>(R.gat);
    const char* gb = static_cast<const char*>(args.g);
    const char* cb = static_cast<const char*>(args.c);
    const bool weighted = MODE == kCgSrc && args.val_t != nullptr;
    // dst: 1 / max(deg, 1) of the whole row for mean (a chunk's own length is not the degree)
    int64_t deg_row = end - begin;
    if (MODE == kCgDst && is_chunk) deg_row = static_cast<int64_t>(__ldg(rowptr + row + 1)) - static_cast<int64_t>(__ldg(rowptr + row));

    for (int vbase = 0; vbase < n_vec; vbase += G) {
        const int vi = vbase + lig;
        if (vi >= n_vec) break;
        const size_t voff = static_cast<size_t>(vi) * 16;
        float acc[NACC][EPV], ruf[EPV], rus[EPV], gr[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            gr[i] = 1.0f;
#pragma unroll
            for (int o = 0; o < NACC; ++o) acc[o][i] = 0.0f;
        }
        {
            const char* rb = reinterpret_cast<const char*>(R.row + row * R.row_ld);
            ElemTraits<T>::unpack(ldg_stream16(rb + voff), ruf);
            ElemTraits<T>::unpack(ldg_stream16(rb + half + voff), rus);
            if (MODE == kCgDst) {
                ElemTraits<T>::unpack(ldg_stream16(gb + row * g_bytes + voff), gr);
#pragma unroll
                for (int i = 0; i < EPV; ++i) gr[i] = finalize<B200MP_SUM>(gr[i], deg_row, args.is_mean, false);
            }
        }
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 af[UNR], as[UNR], cf[UNR], cs[UNR], gv[UNR];
            float w[UNR];
            int64_t id[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                w[u] = 1.0f;
                id[u] = 0;
                if (e + u < end) {
                    const int64_t c = static_cast<int64_t>(ldg_idx(col + e + u));
                    const char* p = gatb + c * gat_bytes + voff;
                    af[u] = ldg_row16(p);
                    as[u] = ldg_row16(p + half);
                    if (MODE == kCgSrc) {
                        gv[u] = ldg_row16(gb + c * g_bytes + voff);
                        if (weighted) w[u] = __ldg(args.val_t + e + u);
                    }
                    if (HAS_C) {
                        id[u] = cg_eid<I>(args, e + u);
                        cf[u] = ldg_stream16(cb + id[u] * c_bytes + voff);
                        cs[u] = ldg_stream16(cb + id[u] * c_bytes + half + voff);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float fa[EPV], fs[EPV], fcf[EPV], fcs[EPV], fg[EPV], df[EPV], ds[EPV];
                    ElemTraits<T>::unpack(af[u], fa);
                    ElemTraits<T>::unpack(as[u], fs);
                    if (HAS_C) {
                        ElemTraits<T>::unpack(cf[u], fcf);
                        ElemTraits<T>::unpack(cs[u], fcs);
                    }
                    if (MODE == kCgSrc) ElemTraits<T>::unpack(gv[u], fg);
#pragma unroll
                    for (int i = 0; i < EPV; ++i) {
                        float pf = __fadd_rn(ruf[i], fa[i]), ps = __fadd_rn(rus[i], fs[i]);
                        if (HAS_C) {
                            pf = __fadd_rn(pf, fcf[i]);
                            ps = __fadd_rn(ps, fcs[i]);
                        }
                        const float gw = MODE == kCgSrc ? (weighted ? __fmul_rn(w[u], fg[i]) : fg[i]) : gr[i];
                        cg_term<T, MODE>(pf, ps, gw, acc[0][i], acc[NACC - 1][i], df[i], ds[i]);
                    }
                    if (MODE == kCgDst && HAS_C && args.grad_c) {
                        char* gcb = static_cast<char*>(args.grad_c) + id[u] * c_bytes + voff;
                        stg_stream16(gcb, ElemTraits<T>::pack(df));
                        stg_stream16(gcb + half, ElemTraits<T>::pack(ds));
                    }
                }
            }
        }
        if (is_chunk) {
#pragma unroll
            for (int o = 0; o < NACC; ++o)
                store_partial<EPV>(plan.partials + (static_cast<size_t>(item * NACC + o) * n_vec + vi) * EPV, acc[o]);
            continue;
        }
        char* ob = static_cast<char*>(args.out) + row * R.out_ld * static_cast<int64_t>(sizeof(T));
#pragma unroll
        for (int o = 0; o < NACC; ++o) {
            float f[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i)
                f[i] = MODE == kCgFwd ? finalize<B200MP_SUM>(acc[o][i], end - begin, args.is_mean, false) : acc[o][i];
            stg_stream16(ob + o * half + voff, ElemTraits<T>::pack(f));
        }
    }
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE>
__global__ void __launch_bounds__(256)
cg_reduce_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, CgArgs args, int64_t n_rows,
                        LongRowPlan plan) {
    constexpr int NACC = MODE == kCgFwd ? 1 : 2;
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // warp-uniform
    const CgRoles<T, MODE> R(args);
    const int64_t F = args.feat;
    const T* g = static_cast<const T*>(args.g);
    const T* cp = static_cast<const T*>(args.c);
    T* gc = static_cast<T*>(args.grad_c);
    const bool weighted = MODE == kCgSrc && args.val_t != nullptr;
    int64_t deg_row = end - begin;
    if (MODE == kCgDst && is_chunk) deg_row = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = lane; f < F; f += 32) {
        const float ruf = ElemTraits<T>::to_float(R.row[row * R.row_ld + f]);
        const float rus = ElemTraits<T>::to_float(R.row[row * R.row_ld + F + f]);
        const float gr = MODE == kCgDst
                             ? finalize<B200MP_SUM>(ElemTraits<T>::to_float(g[row * F + f]), deg_row, args.is_mean, false)
                             : 1.0f;
        float acc0 = 0.0f, acc1 = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            float pf = __fadd_rn(ruf, ElemTraits<T>::to_float(R.gat[c * R.gat_ld + f]));
            float ps = __fadd_rn(rus, ElemTraits<T>::to_float(R.gat[c * R.gat_ld + F + f]));
            const int64_t id = (cp || gc) ? cg_eid<I>(args, e) : 0;
            if (cp) {
                pf = __fadd_rn(pf, ElemTraits<T>::to_float(cp[id * 2 * F + f]));
                ps = __fadd_rn(ps, ElemTraits<T>::to_float(cp[id * 2 * F + F + f]));
            }
            float gw = gr;
            if (MODE == kCgSrc) {
                gw = ElemTraits<T>::to_float(g[c * F + f]);
                if (weighted) gw = __fmul_rn(__ldg(args.val_t + e), gw);
            }
            float df, ds;
            cg_term<T, MODE>(pf, ps, gw, acc0, acc1, df, ds);
            if (MODE == kCgDst && gc) {
                gc[id * 2 * F + f] = ElemTraits<T>::from_float(df);
                gc[id * 2 * F + F + f] = ElemTraits<T>::from_float(ds);
            }
        }
        if (is_chunk) {
            plan.partials[(item * NACC) * F + f] = acc0;
            if (NACC == 2) plan.partials[(item * NACC + 1) * F + f] = acc1;
            continue;
        }
        T* out = static_cast<T*>(args.out) + row * R.out_ld;
        if (MODE == kCgFwd) {
            out[f] = ElemTraits<T>::from_float(finalize<B200MP_SUM>(acc0, end - begin, args.is_mean, false));
        } else {
            out[f] = ElemTraits<T>::from_float(acc0);
            out[F + f] = ElemTraits<T>::from_float(acc1);
        }
    }
}

// Fold the fp32 partials of every long row in chunk order and write the row.
template <typename T, typename I, int MODE>
__global__ void __launch_bounds__(256)
cg_combine_kernel(const I* __restrict__ rowptr, CgArgs args, LongRowPlan plan) {
    constexpr int NACC = MODE == kCgFwd ? 1 : 2;
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const CgRoles<T, MODE> R(args);
    const int64_t F = args.feat;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    T* out = static_cast<T*>(args.out) + row * R.out_ld;
    for (int64_t f = threadIdx.x; f < F; f += blockDim.x) {
#pragma unroll
        for (int o = 0; o < NACC; ++o) {
            float acc = 0.0f;
            for (int64_t c = c0; c < c1; ++c) acc = __fadd_rn(acc, plan.partials[(c * NACC + o) * F + f]);
            if (MODE == kCgFwd) acc = finalize<B200MP_SUM>(acc, deg, args.is_mean, false);
            out[o * F + f] = ElemTraits<T>::from_float(acc);
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
template <typename T, int MODE>
bool cg_vec_ok(const CgArgs& a, const LongRowPlan& plan) {
    return (a.feat * sizeof(T)) % 16 == 0 && (a.ld_u * sizeof(T)) % 16 == 0 && (a.ld_v * sizeof(T)) % 16 == 0 &&
           aligned16(a.u) && aligned16(a.v) && aligned16(a.c) && aligned16(a.g) && aligned16(a.out) &&
           aligned16(a.grad_c) && (plan.n_chunks == 0 || aligned16(plan.partials));
}

template <typename T, typename I, int MODE>
int cg_typed(const void* rowptr_, const void* col_, CgArgs args, int64_t n_rows, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int64_t items = plan.n_chunks + n_rows;
    if (cg_vec_ok<T, MODE>(args, plan)) {
        const int n_vec = static_cast<int>(args.feat * sizeof(T) / 16);
        lane_group_shape<1>(n_vec, [&](auto G, auto) {
            const unsigned blocks = static_cast<unsigned>(ceil_div(items, 128 / G()));
            if (args.c) cg_reduce_kernel<T, I, MODE, G(), 4, true><<<blocks, 128, 0, stream>>>(rowptr, col, args, n_rows, n_vec, plan);
            else cg_reduce_kernel<T, I, MODE, G(), 4, false><<<blocks, 128, 0, stream>>>(rowptr, col, args, n_rows, n_vec, plan);
        });
    } else {
        cg_reduce_scalar_kernel<T, I, MODE><<<static_cast<unsigned>(ceil_div(items, 8)), 256, 0, stream>>>(
            rowptr, col, args, n_rows, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        cg_combine_kernel<T, I, MODE><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, args, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_cg_csr(const void* rowptr, const void* col, const void* perm, const void* u, const void* v,
                             const void* c, void* out, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat,
                             int64_t ld_u, int64_t ld_v, int reduce, const int64_t* long_rows,
                             const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                             float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);
    B200MP_CHECK_ARG(ld_u >= 2 * feat && ld_v >= 2 * feat);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && u && out);
    B200MP_CHECK_ARG(n_edges == 0 || (col && v));
    const CgArgs a{u, v, c, perm, nullptr, nullptr, out, nullptr, feat, ld_u, ld_v, reduce == B200MP_MEAN};
    return dispatch_val_idx(val_dtype, idx_dtype, "cg_csr", [&](auto tv, auto ti) {
        return cg_typed<decltype(tv), decltype(ti), kCgFwd>(rowptr, col, a, n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_cg_backward_dst(const void* rowptr, const void* col, const void* perm, const void* u,
                                      const void* v, const void* c, const void* grad_out, void* grad_u, void* grad_c,
                                      int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld_u,
                                      int64_t ld_v, int reduce, const int64_t* long_rows, const int64_t* chunk_ptr,
                                      int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                      int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);
    B200MP_CHECK_ARG(ld_u >= 2 * feat && ld_v >= 2 * feat);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && u && grad_out && grad_u);
    B200MP_CHECK_ARG(n_edges == 0 || (col && v));
    B200MP_CHECK_ARG(grad_c == nullptr || c);
    const CgArgs a{u, v, c, perm, grad_out, nullptr, grad_u, grad_c, feat, ld_u, ld_v, reduce == B200MP_MEAN};
    return dispatch_val_idx(val_dtype, idx_dtype, "cg_backward_dst", [&](auto tv, auto ti) {
        return cg_typed<decltype(tv), decltype(ti), kCgDst>(rowptr, col, a, n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_cg_backward_src(const void* rowptr_t, const void* col_t, const void* perm_t, const float* val_t,
                                      const void* u, const void* v, const void* c, const void* grad_out, void* grad_v,
                                      int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t feat, int64_t ld_u,
                                      int64_t ld_v, const int64_t* long_rows, const int64_t* chunk_ptr,
                                      int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                      int idx_dtype, int val_dtype, void* stream) {
    const int64_t n_rows = n_src, n_cols = n_dst;
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);
    B200MP_CHECK_ARG(ld_u >= 2 * feat && ld_v >= 2 * feat);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && v && grad_v);
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && u && grad_out && (c == nullptr || perm_t)));
    const CgArgs a{u, v, c, perm_t, grad_out, val_t, grad_v, nullptr, feat, ld_u, ld_v, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "cg_backward_src", [&](auto tv, auto ti) {
        return cg_typed<decltype(tv), decltype(ti), kCgSrc>(rowptr_t, col_t, a, n_src, plan,
                                                          static_cast<cudaStream_t>(stream));
    });
}
