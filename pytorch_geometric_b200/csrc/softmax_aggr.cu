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
#include "aggr_message.cuh"
#include "csr_reduce.cuh"
#include "gate_math.cuh"

extern "C" int b200mp_column_sum(const void* x, float* out, float* partials, int64_t n_parts, int64_t n_rows,
                                 int64_t feat, int val_dtype, void* stream);
extern "C" int64_t b200mp_column_sum_parts(int64_t n_rows);

namespace b200mp {

enum SmMode { kSmFwd = 0, kSmDst = 1, kSmSrc = 2 };
enum SmT { kSmTNone = 0, kSmTScalar = 1, kSmTChannel = 2 };

struct SmArgs {
    const void* x;       // [n_src, feat] gathered through col (fwd / dst) or the row operand (src)
    const void* a;       // [n_edges, feat] in the caller's edge order
    const float* t;      // [1] or [feat] fp32
    const void* perm;    // caller's edge id of each CSR (fwd / dst) or transposed (src) slot; null = slot
    const void* g;       // grad_out [n_dst, feat]
    const void* o;       // out [n_dst, feat]
    float* lse;          // [n_dst, feat]: written by fwd (nullable), read by the backward
    void* out;           // fwd: out; dst: grad_a (nullable); src: grad_x
    float* gt_part;      // dst: [gridDim.x, feat] grad_t partials, or null
    int64_t feat;
    float eps;
    bool semi;
};

template <typename T, int TMODE>
__device__ __forceinline__ float sm_logit(float m, float tv) {
    return TMODE == kSmTNone ? m : round_to<T>(__fmul_rn(tv, m));
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
    if (!semi) gm = __fmul_rn(gp, fmaf(TMODE == kSmTNone ? 1.0f : tv, dm, 1.0f));
    return (SmForms<FORM>::kRelu && !on) ? 0.0f : gm;
}

template <typename I>
__device__ __forceinline__ int64_t sm_eid(const SmArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// Per-CTA grad_t partial: every group has written its row of `sh` (zeros when idle); fold the groups in order.
__device__ __forceinline__ void sm_store_gt(const float* sh, int groups, int64_t feat, float* gt_part) {
    __syncthreads();
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        float s = 0.0f;
        for (int k = 0; k < groups; ++k) s = __fadd_rn(s, sh[k * feat + f]);
        gt_part[static_cast<int64_t>(blockIdx.x) * feat + f] = s;
    }
}

// ---------------------------------------------------------------- the three sweeps, 16-byte vector path
template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
__global__ void __launch_bounds__(128)
softmax_aggr_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, SmArgs args, int64_t n_rows, int n_vec,
                    int lg, LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    constexpr int EPV = ElemTraits<T>::kPerVec;
    // bf16 backward: fewer edges in flight, so that the per-row operands stay in registers
    constexpr int UNR = (MODE == kSmFwd || sizeof(T) == 4) ? 4 : ((WANT_T || TMODE == kSmTChannel) ? 1 : 2);
    extern __shared__ float sm_sh[];
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // uniform per group
    if (!active && !WANT_T) return;
    if (!active) row = begin = end = 0;                  // an idle group still writes its (zero) grad_t row
    const int64_t F = args.feat;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = static_cast<const char*>(args.x);
    const char* ab = static_cast<const char*>(args.a);
    const char* gb = static_cast<const char*>(args.g);
    const char* ob = static_cast<const char*>(args.o);
    float ts = 1.0f;
    if (TMODE == kSmTScalar) ts = __ldg(args.t);

    for (int vi = lig; vi < n_vec; vi += G) {
        const size_t voff = static_cast<size_t>(vi) * 16;
        const int64_t f0 = static_cast<int64_t>(vi) * EPV;
        float tv[EPV], rx[EPV], rg[EPV], ro[EPV], rl[EPV];
        float acc0[EPV], acc1[EPV], acc2[EPV], c1[EPV], c2[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            tv[i] = ts;
            rx[i] = rg[i] = ro[i] = rl[i] = 0.0f;
            acc0[i] = MODE == kSmFwd ? -INFINITY : 0.0f;
            acc1[i] = acc2[i] = c1[i] = c2[i] = 0.0f;
        }
        if (TMODE == kSmTChannel) {
#pragma unroll
            for (int i = 0; i < EPV; i += 4) {
                const float4 t4 = __ldg(reinterpret_cast<const float4*>(args.t + f0 + i));
                tv[i] = t4.x; tv[i + 1] = t4.y; tv[i + 2] = t4.z; tv[i + 3] = t4.w;
            }
        }
        {
            if (MODE == kSmDst) {
                ElemTraits<T>::unpack(ldg_stream16(gb + row * row_bytes + voff), rg);
                ElemTraits<T>::unpack(ldg_stream16(ob + row * row_bytes + voff), ro);
                const float* lp = args.lse + row * F + f0;
#pragma unroll
                for (int i = 0; i < EPV; i += 4) {
                    const float4 l4 = __ldg(reinterpret_cast<const float4*>(lp + i));
                    rl[i] = l4.x; rl[i + 1] = l4.y; rl[i + 2] = l4.z; rl[i + 3] = l4.w;
                }
            }
            if (MODE == kSmSrc) ElemTraits<T>::unpack(ldg_stream16(xb + row * row_bytes + voff), rx);
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
                    if (Fm::kA || (MODE == kSmDst && args.out)) id[u] = sm_eid<I>(args, e + u);
                    if (MODE != kSmSrc && Fm::kX) xv[u] = ldg_row16(xb + c * row_bytes + voff);
                    if (Fm::kA) av[u] = ldg_stream16(ab + id[u] * row_bytes + voff);
                    if (MODE == kSmSrc) {
                        gv[u] = ldg_row16(gb + c * row_bytes + voff);
                        ov[u] = ldg_row16(ob + c * row_bytes + voff);
                        const float4* lp = reinterpret_cast<const float4*>(args.lse + c * F + f0);
#pragma unroll
                        for (int q = 0; q < EPV / 4; ++q) lv[u][q] = __ldg(lp + q);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float fx[EPV], fa[EPV], fg[EPV], fo[EPV], fl[EPV], gs[EPV];
                    if (MODE == kSmSrc) {
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
                        if (MODE == kSmFwd) {
                            sm_push(z, m, acc0[i], acc1[i], acc2[i], c1[i], c2[i]);
                        } else if (MODE == kSmDst) {
                            gs[i] = sm_grad<FORM, TMODE, WANT_T>(z, m, on, tv[i], rg[i], ro[i], rl[i], args.semi, acc0[i]);
                        } else {
                            float unused = 0.0f;
                            acc0[i] = __fadd_rn(acc0[i], sm_grad<FORM, TMODE, false>(z, m, on, tv[i], fg[i], fo[i], fl[i],
                                                                                    args.semi, unused));
                        }
                    }
                    if (MODE == kSmDst && args.out)
                        stg_stream16(static_cast<char*>(args.out) + id[u] * row_bytes + voff, ElemTraits<T>::pack(gs));
                }
            }
        }
        if (MODE == kSmFwd) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                acc1[i] = __fsub_rn(acc1[i], c1[i]);
                acc2[i] = __fsub_rn(acc2[i], c2[i]);
            }
        }
        if (MODE == kSmDst) {
            if (WANT_T) {
                float* sh = sm_sh + static_cast<int64_t>(threadIdx.x >> lg) * F + f0;
#pragma unroll
                for (int i = 0; i < EPV; ++i) sh[i] = acc0[i];
            }
            continue;
        }
        if (is_chunk) {
            constexpr int NACC = MODE == kSmFwd ? 3 : 1;
            store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC) * F + f0, acc0);
            if (MODE == kSmFwd) {
                store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC + 1) * F + f0, acc1);
                store_partial<EPV>(plan.partials + static_cast<size_t>(item * NACC + 2) * F + f0, acc2);
            }
            continue;
        }
        char* dst = static_cast<char*>(args.out) + row * row_bytes + voff;
        if (MODE == kSmFwd) {
            float f[EPV], l[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i) sm_final(acc0[i], acc1[i], acc2[i], end > begin, f[i], l[i]);
            stg_stream16(dst, ElemTraits<T>::pack(f));
            if (args.lse) store_partial<EPV>(args.lse + row * F + f0, l);
        } else {
            stg_stream16(dst, ElemTraits<T>::pack(acc0));
        }
    }
    if (MODE == kSmDst && WANT_T) sm_store_gt(sm_sh, blockDim.x >> lg, F, args.gt_part);
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature.
template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
__global__ void __launch_bounds__(256)
softmax_aggr_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, SmArgs args, int64_t n_rows,
                           LongRowPlan plan) {
    using Fm = SmForms<FORM>;
    extern __shared__ float sm_sh[];
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row = 0, begin = 0, end = 0;
    bool is_chunk = false;
    const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);   // warp-uniform
    if (!active && !WANT_T) return;
    if (!active) row = begin = end = 0;                  // an idle group still writes its (zero) grad_t row
    const int64_t F = args.feat;
    const T* x = static_cast<const T*>(args.x);
    const T* a = static_cast<const T*>(args.a);
    const T* g = static_cast<const T*>(args.g);
    const T* o = static_cast<const T*>(args.o);
    T* out = static_cast<T*>(args.out);
    for (int64_t f = lane; f < F; f += 32) {
        const float tv = TMODE == kSmTNone ? 1.0f : __ldg(args.t + (TMODE == kSmTChannel ? f : 0));
        float acc0 = MODE == kSmFwd ? -INFINITY : 0.0f, acc1 = 0.0f, acc2 = 0.0f, c1 = 0.0f, c2 = 0.0f;
        float rx = 0.0f, rg = 0.0f, ro = 0.0f, rl = 0.0f;
        if (MODE == kSmDst) {
            rg = ElemTraits<T>::to_float(g[row * F + f]);
            ro = ElemTraits<T>::to_float(o[row * F + f]);
            rl = args.lse[row * F + f];
        }
        if (MODE == kSmSrc) rx = ElemTraits<T>::to_float(x[row * F + f]);
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t id = (Fm::kA || (MODE == kSmDst && out)) ? sm_eid<I>(args, e) : 0;
            const float xv = MODE == kSmSrc ? rx : (Fm::kX ? ElemTraits<T>::to_float(x[c * F + f]) : 0.0f);
            const float av = Fm::kA ? ElemTraits<T>::to_float(a[id * F + f]) : 0.0f;
            bool on;
            const float m = sm_message<T, FORM>(xv, av, args.eps, on);
            const float z = sm_logit<T, TMODE>(m, tv);
            if (MODE == kSmFwd) {
                sm_push(z, m, acc0, acc1, acc2, c1, c2);
            } else if (MODE == kSmDst) {
                const float gs = sm_grad<FORM, TMODE, WANT_T>(z, m, on, tv, rg, ro, rl, args.semi, acc0);
                if (out) out[id * F + f] = ElemTraits<T>::from_float(gs);
            } else {
                float unused = 0.0f;
                acc0 = __fadd_rn(acc0, sm_grad<FORM, TMODE, false>(z, m, on, tv, ElemTraits<T>::to_float(g[c * F + f]),
                                                                  ElemTraits<T>::to_float(o[c * F + f]),
                                                                  args.lse[c * F + f], args.semi, unused));
            }
        }
        if (MODE == kSmFwd) {
            acc1 = __fsub_rn(acc1, c1);
            acc2 = __fsub_rn(acc2, c2);
        }
        if (MODE == kSmDst) {
            if (WANT_T) sm_sh[(threadIdx.x >> 5) * F + f] = acc0;
            continue;
        }
        if (is_chunk) {
            if (MODE == kSmFwd) {
                plan.partials[(item * 3) * F + f] = acc0;
                plan.partials[(item * 3 + 1) * F + f] = acc1;
                plan.partials[(item * 3 + 2) * F + f] = acc2;
            } else {
                plan.partials[item * F + f] = acc0;
            }
            continue;
        }
        if (MODE == kSmFwd) {
            float ov, l;
            sm_final(acc0, acc1, acc2, end > begin, ov, l);
            out[row * F + f] = ElemTraits<T>::from_float(ov);
            if (args.lse) args.lse[row * F + f] = l;
        } else {
            out[row * F + f] = ElemTraits<T>::from_float(acc0);
        }
    }
    if (MODE == kSmDst && WANT_T) sm_store_gt(sm_sh, blockDim.x >> 5, F, args.gt_part);
}

// Merge the (M, S, A) partials of every long row in chunk order and write out and lse.
template <typename T>
__global__ void __launch_bounds__(256)
softmax_aggr_combine_kernel(SmArgs args, LongRowPlan plan) {
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
        if (args.lse) args.lse[row * F + f] = l;
    }
}

// ---------------------------------------------------------------- host-side dispatch
template <typename T>
bool sm_vec_ok(const SmArgs& a, const LongRowPlan& plan) {
    return (a.feat * sizeof(T)) % 16 == 0 && aligned16(a.x) && aligned16(a.a) && aligned16(a.t) && aligned16(a.g) &&
           aligned16(a.o) && aligned16(a.lse) && aligned16(a.out) && (plan.n_chunks == 0 || aligned16(plan.partials));
}

// Lane-group width for a row of n_vec vectors: the smallest power of two >= n_vec, at most 32.
inline int sm_lg(int n_vec) {
    int lg = 0;
    while (lg < 5 && (1 << lg) < n_vec) ++lg;
    return lg;
}

// CTAs of the sweep that sm_typed launches, so that the destination sweep's caller can size the grad_t partials.
template <typename T>
int64_t sm_grid(const SmArgs& a, const LongRowPlan& plan, int64_t n_rows, int& lg, bool& vec) {
    const int64_t items = plan.n_chunks + n_rows;
    vec = sm_vec_ok<T>(a, plan);
    if (vec) {
        lg = sm_lg(static_cast<int>(a.feat * sizeof(T) / 16));
        return ceil_div(items, 128 >> lg);
    }
    lg = 5;
    return ceil_div(items, 8);
}

template <typename T, typename I, int MODE, int FORM, int TMODE, bool WANT_T>
int sm_launch(const I* rowptr, const I* col, const SmArgs& args, int64_t n_rows, const LongRowPlan& plan,
              cudaStream_t stream) {
    int lg;
    bool vec;
    const int64_t grid = sm_grid<T>(args, plan, n_rows, lg, vec);
    if (grid == 0) return B200MP_OK;
    const size_t smem = WANT_T ? static_cast<size_t>(vec ? (128 >> lg) : 8) * args.feat * sizeof(float) : 0;
    if (vec) {
        auto k = softmax_aggr_kernel<T, I, MODE, FORM, TMODE, WANT_T>;
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<static_cast<unsigned>(grid), 128, smem, stream>>>(rowptr, col, args, n_rows,
                                                              static_cast<int>(args.feat * sizeof(T) / 16), lg, plan);
    } else {
        auto k = softmax_aggr_scalar_kernel<T, I, MODE, FORM, TMODE, WANT_T>;
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<static_cast<unsigned>(grid), 256, smem, stream>>>(rowptr, col, args, n_rows, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (MODE != kSmDst && plan.n_long > 0) {
        if (MODE == kSmFwd)
            softmax_aggr_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(args, plan);
        else
            csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
                rowptr, static_cast<T*>(args.out), args.feat, false, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I, int MODE, int FORM>
int sm_dispatch_t(const I* rowptr, const I* col, const SmArgs& args, int tmode, bool want_t, int64_t n_rows,
                  const LongRowPlan& plan, cudaStream_t s) {
    if (MODE == kSmDst && want_t) {
        if (tmode == kSmTScalar) return sm_launch<T, I, MODE, FORM, kSmTScalar, true>(rowptr, col, args, n_rows, plan, s);
        if (tmode == kSmTChannel) return sm_launch<T, I, MODE, FORM, kSmTChannel, true>(rowptr, col, args, n_rows, plan, s);
        return sm_launch<T, I, MODE, FORM, kSmTNone, true>(rowptr, col, args, n_rows, plan, s);
    }
    if (tmode == kSmTScalar) return sm_launch<T, I, MODE, FORM, kSmTScalar, false>(rowptr, col, args, n_rows, plan, s);
    if (tmode == kSmTChannel) return sm_launch<T, I, MODE, FORM, kSmTChannel, false>(rowptr, col, args, n_rows, plan, s);
    return sm_launch<T, I, MODE, FORM, kSmTNone, false>(rowptr, col, args, n_rows, plan, s);
}

template <typename T, typename I, int MODE>
int sm_typed(const void* rowptr_, const void* col_, SmArgs args, int form, int tmode, bool want_t, int64_t n_rows,
             LongRowPlan plan, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    switch (form) {
        case kSmX: return sm_dispatch_t<T, I, MODE, kSmX>(rowptr, col, args, tmode, want_t, n_rows, plan, s);
        case kSmXRelu: return sm_dispatch_t<T, I, MODE, kSmXRelu>(rowptr, col, args, tmode, want_t, n_rows, plan, s);
        case kSmXARelu: return sm_dispatch_t<T, I, MODE, kSmXARelu>(rowptr, col, args, tmode, want_t, n_rows, plan, s);
        default:
            if (MODE == kSmSrc) break;                    // rows-only messages have no source operand
            return sm_dispatch_t<T, I, MODE, kSmA>(rowptr, col, args, tmode, want_t, n_rows, plan, s);
    }
    set_error("softmax_aggr: the transposed sweep needs x");
    return B200MP_ERR_INVALID_ARG;
}

}  // namespace b200mp

using namespace b200mp;

#define B200MP_CHECK_SM()                                                                                       \
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);                                  \
    B200MP_CHECK_ARG(message == 0 || message == 1);                                                             \
    B200MP_CHECK_ARG(t_mode >= 0 && t_mode <= 2 && (t_mode == 0 || t));                                        \
    B200MP_CHECK_ARG(message == 1 ? x != nullptr : (x == nullptr) != (edge_rows == nullptr))

extern "C" int b200mp_softmax_aggr_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                       const void* edge_rows, const float* t, void* out, float* lse, int64_t n_rows,
                                       int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps,
                                       int t_mode, const int64_t* long_rows, const int64_t* chunk_ptr,
                                       int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                       int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_SM();
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const SmArgs a{x, edge_rows, t, perm, nullptr, nullptr, lse, out, nullptr, feat, eps, false};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_csr", [&](auto tv, auto ti) {
        return sm_typed<decltype(tv), decltype(ti), kSmFwd>(rowptr, col, a, sm_form(x, edge_rows, message), t_mode, false,
                                                          n_rows, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int64_t b200mp_softmax_aggr_workspace(int64_t n_rows, int64_t n_chunks, int64_t feat) {
    // Upper bound over both kernels: a vector CTA holds at least 4 work items, a scalar CTA 8.
    const int64_t ctas = ceil_div(n_rows + n_chunks, 4);
    return (ctas + b200mp_column_sum_parts(ctas)) * feat;
}

template <typename T, typename I>
int sm_dst_with_t(const void* rowptr, const void* col, SmArgs a, int form, int t_mode, float* grad_t, float* ws,
                  int64_t n_rows, LongRowPlan plan, cudaStream_t s) {
    int lg;
    bool vec;
    const int64_t ctas = sm_grid<T>(a, plan, n_rows, lg, vec);
    a.gt_part = ws;
    const int rc = sm_typed<T, I, kSmDst>(rowptr, col, a, form, t_mode, grad_t != nullptr, n_rows, plan, s);
    if (rc != B200MP_OK || grad_t == nullptr) return rc;
    if (ctas == 0) return cudaMemsetAsync(grad_t, 0, a.feat * sizeof(float), s) == cudaSuccess ? B200MP_OK : B200MP_ERR_CUDA;
    return b200mp_column_sum(ws, grad_t, ws + ctas * a.feat, b200mp_column_sum_parts(ctas), ctas, a.feat, B200MP_F32, s);
}

extern "C" int b200mp_softmax_aggr_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                                const void* edge_rows, const float* t, const void* out,
                                                const float* lse, const void* grad_out, void* grad_edge_rows,
                                                float* grad_t, float* workspace, int64_t n_rows, int64_t n_cols,
                                                int64_t n_edges, int64_t feat, int message, float eps, int t_mode,
                                                int semi_grad, const int64_t* long_rows, const int64_t* chunk_ptr,
                                                int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype,
                                                int val_dtype, void* stream) {
    B200MP_CHECK_SM();
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
    const SmArgs a{x, edge_rows, t, perm, grad_out, out, const_cast<float*>(lse), grad_edge_rows, nullptr, feat, eps,
                   semi_grad != 0};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_backward_dst", [&](auto tv, auto ti) {
        return sm_dst_with_t<decltype(tv), decltype(ti)>(rowptr, col, a, sm_form(x, edge_rows, message), t_mode, grad_t,
                                                       workspace, n_rows, plan, static_cast<cudaStream_t>(stream));
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
    const int64_t n_rows = n_src, n_cols = n_dst;
    B200MP_CHECK_SM();
    B200MP_CHECK_ARG(x != nullptr);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && grad_x);
    B200MP_CHECK_ARG(n_edges == 0 || (col_t && out && lse && grad_out && (edge_rows == nullptr || perm_t)));
    const SmArgs a{x, edge_rows, t, perm_t, grad_out, out, const_cast<float*>(lse), grad_x, nullptr, feat, eps,
                   semi_grad != 0};
    return dispatch_val_idx(val_dtype, idx_dtype, "softmax_aggr_backward_src", [&](auto tv, auto ti) {
        return sm_typed<decltype(tv), decltype(ti), kSmSrc>(rowptr_t, col_t, a, sm_form(x, edge_rows, message), t_mode,
                                                          false, n_src, plan, static_cast<cudaStream_t>(stream));
    });
}
