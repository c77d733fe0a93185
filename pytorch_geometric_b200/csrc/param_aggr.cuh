// param_aggr.cuh -- what the softmax- and power-mean-aggregation sweeps (softmax_aggr.cu, power_mean.cu) share: the
// per-edge message (x gathered through col, an edge row in the caller's edge order, or GENConv's relu(x_j + e_ji) + eps,
// nn/conv/gen_conv.py:231-239), the operands, the device helpers around the per-element math, and the host side that
// shapes, checks and launches a sweep and folds its parameter gradient.
//
// Each op supplies its vector and scalar kernels and its combine through an Op struct:
//   kName, kParam                        names for error messages ("softmax_aggr", "t")
//   collects(mode)                       whether that sweep collects the parameter's gradient
//   vec<T, I, MODE, FORM, PMODE, WANT>() / scalar<...>()   the kernels
//   combine<T, I, PMODE>(rowptr, args, plan, stream)       launches the forward's long-row combine
#pragma once

#include "csr_reduce.cuh"

namespace b200mp {

enum SmForm { kSmX = 0, kSmA = 1, kSmXRelu = 2, kSmXARelu = 3 };   // which rows are read, and the message

template <int FORM>
struct SmForms {
    static constexpr bool kX = FORM != kSmA;
    static constexpr bool kA = FORM == kSmA || FORM == kSmXARelu;
    static constexpr bool kRelu = FORM == kSmXRelu || FORM == kSmXARelu;
};

// The message m and its pre-activation gate `on` from the fp32 loads.
template <typename T, int FORM>
__device__ __forceinline__ float sm_message(float xv, float av, float eps, bool& on) {
    using Fm = SmForms<FORM>;
    const float s = (Fm::kX && Fm::kA) ? round_to<T>(__fadd_rn(xv, av)) : (Fm::kX ? xv : av);
    on = !(s <= 0.0f);
    return Fm::kRelu ? round_to<T>(__fadd_rn(on ? s : 0.0f, eps)) : s;
}

// Message form from the operands: x and / or a, identity or relu + eps.
inline int sm_form(const void* x, const void* a, int message) {
    if (message == 1) return a ? kSmXARelu : kSmXRelu;
    return x ? kSmX : kSmA;
}

// The parameter (t or p): absent, one value or one per channel.  The values are the C ABI's t_mode and p_mode.
enum ParamMode { kParamNone = 0, kParamScalar = 1, kParamChannel = 2 };
// The forward sweep, the backward's destination sweep, and its transposed (source) sweep.
enum SweepMode { kSweepFwd = 0, kSweepDst = 1, kSweepSrc = 2 };

// The grad-parameter sweeps keep one fp32 row of F per lane group in shared memory: H100's opt-in limit per CTA.
constexpr size_t kMaxParamSmem = 227 * 1024;

struct AggrArgs {
    const void* x;       // [n_src, feat] gathered through col (fwd / dst) or the row operand (src)
    const void* a;       // [n_edges, feat] in the caller's edge order
    const float* param;  // t or p: [1] or [feat] fp32
    const void* perm;    // caller's edge id of each CSR (fwd / dst) or transposed (src) slot; null = slot
    const void* g;       // grad_out [n_dst, feat]
    const void* o;       // out [n_dst, feat]
    float* saved;        // lse or M [n_dst, feat]: written by fwd (nullable), read by the backward
    float* G;            // power mean's src: the node plane [n_dst, feat] the transposed sweep gathers
    void* out;           // fwd: out; dst: grad_a (nullable); src: grad_x
    float* param_part;   // [gridDim.x, feat] grad-parameter partials, or null
    int64_t feat;
    float eps, lo, hi;   // lo, hi: power mean's clamp
    bool semi;           // softmax's semi_grad
};

// ---------------------------------------------------------------- device helpers
template <typename I>
__device__ __forceinline__ int64_t aggr_eid(const AggrArgs& a, int64_t e) {
    return a.perm ? static_cast<int64_t>(ldg_idx(static_cast<const I*>(a.perm) + e)) : e;
}

// EPV fp32 values (one 16-byte vector's worth of channels) as EPV / 4 float4 loads.
template <int EPV>
__device__ __forceinline__ void ldg_f32(const float* p, float (&v)[EPV]) {
#pragma unroll
    for (int i = 0; i < EPV; i += 4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(p + i));
        v[i] = q.x; v[i + 1] = q.y; v[i + 2] = q.z; v[i + 3] = q.w;
    }
}

// decode_item for a sweep that may have to keep its idle groups: with KEEP_IDLE an idle group gets the empty row 0,
// so that a sweep collecting the parameter's gradient still writes its (zero) row of shared memory.
template <bool KEEP_IDLE, typename I>
__device__ __forceinline__ bool aggr_item(int64_t item, const I* __restrict__ rowptr, int64_t n_rows,
                                          const LongRowPlan& plan, int64_t& row, int64_t& begin, int64_t& end,
                                          bool& is_chunk) {
    const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);
    if (KEEP_IDLE && !active) row = begin = end = 0;
    return active;
}

// Per-CTA grad-parameter partial: every group has written its row of `sh` (zeros when idle); fold the groups in order.
__device__ __forceinline__ void store_param_part(const float* sh, int groups, int64_t feat, float* part) {
    __syncthreads();
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        float s = 0.0f;
        for (int k = 0; k < groups; ++k) s = __fadd_rn(s, sh[k * feat + f]);
        part[static_cast<int64_t>(blockIdx.x) * feat + f] = s;
    }
}

// ---------------------------------------------------------------- host side
// The argument checks every entry point shares.  `clamp`: the op has power mean's clamp, which needs
// 0 < lo <= hi whenever there is a p.
inline int check_aggr_args(int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int message, const void* x,
                           const void* a, int mode, const float* param, bool clamp, float lo, float hi) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);
    B200MP_CHECK_ARG(message == 0 || message == 1);
    B200MP_CHECK_ARG(mode >= kParamNone && mode <= kParamChannel && (mode == kParamNone || param));
    B200MP_CHECK_ARG(!clamp || mode == kParamNone || (lo > 0.0f && hi >= lo));
    B200MP_CHECK_ARG(message == 1 ? x != nullptr : (x == nullptr) != (a == nullptr));
    return B200MP_OK;
}

// A sweep's launch: 128-thread CTAs of lane groups of 1 << lg lanes (16-byte vectors), or 256-thread CTAs of one warp
// per row (scalar), and the dynamic shared memory of the grad-parameter row per group.
struct SweepShape {
    int64_t grid;
    int lg;
    bool vec;
    size_t smem;
};

// The shape of a sweep over n_rows rows, or B200MP_ERR_UNSUPPORTED when the grad-parameter rows of a CTA do not fit
// in shared memory.  Called before anything is launched, so that such a call launches nothing.
template <class Op, typename T>
int sweep_shape(const AggrArgs& a, const LongRowPlan& plan, int64_t n_rows, bool want, SweepShape& sh) {
    sh.vec = (a.feat * sizeof(T)) % 16 == 0 && aligned16(a.x) && aligned16(a.a) && aligned16(a.param) &&
             aligned16(a.g) && aligned16(a.o) && aligned16(a.saved) && aligned16(a.G) && aligned16(a.out) &&
             (plan.n_chunks == 0 || aligned16(plan.partials));
    sh.lg = sh.vec ? lane_group_log2(static_cast<int>(a.feat * sizeof(T) / 16)) : 5;
    const int groups = sh.vec ? 128 >> sh.lg : 8;
    sh.grid = ceil_div(plan.n_chunks + n_rows, groups);
    sh.smem = want ? static_cast<size_t>(groups) * a.feat * sizeof(float) : 0;
    if (sh.grid > 0 && sh.smem > kMaxParamSmem) {
        set_error("%s: grad_%s of %lld channels needs %zu bytes of shared memory per CTA (at most %zu)", Op::kName,
                  Op::kParam, static_cast<long long>(a.feat), sh.smem, kMaxParamSmem);
        return B200MP_ERR_UNSUPPORTED;
    }
    return B200MP_OK;
}

template <class Op, typename T, typename I, int MODE, int FORM, int PMODE, bool WANT>
int aggr_launch(const I* rowptr, const I* col, const AggrArgs& args, int64_t n_rows, const LongRowPlan& plan,
                const SweepShape& sh, cudaStream_t stream) {
    if (sh.grid == 0) return B200MP_OK;
    const size_t smem = WANT ? sh.smem : 0;
    const unsigned grid = static_cast<unsigned>(sh.grid);
    if (sh.vec) {
        auto k = Op::template vec<T, I, MODE, FORM, PMODE, WANT>();
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<grid, 128, smem, stream>>>(rowptr, col, args, n_rows, static_cast<int>(args.feat * sizeof(T) / 16), sh.lg,
                                       plan);
    } else {
        auto k = Op::template scalar<T, I, MODE, FORM, PMODE, WANT>();
        if (smem > 48 * 1024) B200MP_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                                    static_cast<int>(smem)));
        k<<<grid, 256, smem, stream>>>(rowptr, col, args, n_rows, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (MODE != kSweepDst && plan.n_long > 0) {
        if constexpr (MODE == kSweepFwd)
            Op::template combine<T, I, PMODE>(rowptr, args, plan, stream);
        else
            csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
                rowptr, static_cast<T*>(args.out), args.feat, false, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

// Kernels with WANT exist only for the sweeps that collect the parameter's gradient, and only with a parameter: the
// entry points refuse a gradient without one.
template <class Op, typename T, typename I, int MODE, int FORM>
int aggr_dispatch_param(const I* rowptr, const I* col, const AggrArgs& args, int mode, bool want, int64_t n_rows,
                        const LongRowPlan& plan, const SweepShape& sh, cudaStream_t s) {
    if constexpr (Op::collects(MODE)) {
        if (want && mode == kParamScalar)
            return aggr_launch<Op, T, I, MODE, FORM, kParamScalar, true>(rowptr, col, args, n_rows, plan, sh, s);
        if (want) return aggr_launch<Op, T, I, MODE, FORM, kParamChannel, true>(rowptr, col, args, n_rows, plan, sh, s);
    }
    if (mode == kParamScalar)
        return aggr_launch<Op, T, I, MODE, FORM, kParamScalar, false>(rowptr, col, args, n_rows, plan, sh, s);
    if (mode == kParamChannel)
        return aggr_launch<Op, T, I, MODE, FORM, kParamChannel, false>(rowptr, col, args, n_rows, plan, sh, s);
    return aggr_launch<Op, T, I, MODE, FORM, kParamNone, false>(rowptr, col, args, n_rows, plan, sh, s);
}

template <class Op, typename T, typename I, int MODE>
int aggr_typed(const void* rowptr_, const void* col_, const AggrArgs& args, int form, int mode, bool want,
               int64_t n_rows, const LongRowPlan& plan, const SweepShape& sh, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    switch (form) {
        case kSmX: return aggr_dispatch_param<Op, T, I, MODE, kSmX>(rowptr, col, args, mode, want, n_rows, plan, sh, s);
        case kSmXRelu:
            return aggr_dispatch_param<Op, T, I, MODE, kSmXRelu>(rowptr, col, args, mode, want, n_rows, plan, sh, s);
        case kSmXARelu:
            return aggr_dispatch_param<Op, T, I, MODE, kSmXARelu>(rowptr, col, args, mode, want, n_rows, plan, sh, s);
        default:
            if constexpr (MODE == kSweepSrc) {              // rows-only messages have no source operand
                set_error("%s: the transposed sweep needs x", Op::kName);
                return B200MP_ERR_INVALID_ARG;
            } else {
                return aggr_dispatch_param<Op, T, I, MODE, kSmA>(rowptr, col, args, mode, want, n_rows, plan, sh, s);
            }
    }
}

// One sweep that collects no parameter gradient: the forward, or softmax's transposed sweep.
template <class Op, typename T, typename I, int MODE>
int aggr_sweep(const void* rowptr, const void* col, const AggrArgs& a, int form, int mode, int64_t n_rows,
               const LongRowPlan& plan, cudaStream_t s) {
    SweepShape sh;
    if (int rc = sweep_shape<Op, T>(a, plan, n_rows, false, sh)) return rc;
    return aggr_typed<Op, T, I, MODE>(rowptr, col, a, form, mode, false, n_rows, plan, sh, s);
}

// Fold `parts` fp32 partial rows at ws into the parameter's gradient (zeros when there are none).
inline int fold_param_parts(float* ws, int64_t parts, float* grad, int64_t feat, cudaStream_t s) {
    if (parts == 0) return cudaMemsetAsync(grad, 0, feat * sizeof(float), s) == cudaSuccess ? B200MP_OK : B200MP_ERR_CUDA;
    return b200mp_column_sum(ws, grad, ws + parts * feat, b200mp_column_sum_parts(parts), parts, feat, B200MP_F32, s);
}

// The destination sweep of the backward, and with `grad` its parameter gradient from one partial row per CTA in ws.
template <class Op, typename T, typename I>
int aggr_dst(const void* rowptr, const void* col, AggrArgs a, int form, int mode, float* grad, float* ws,
             int64_t n_rows, const LongRowPlan& plan, cudaStream_t s) {
    SweepShape sh;
    if (int rc = sweep_shape<Op, T>(a, plan, n_rows, grad != nullptr, sh)) return rc;
    a.param_part = ws;
    if (int rc = aggr_typed<Op, T, I, kSweepDst>(rowptr, col, a, form, mode, grad != nullptr, n_rows, plan, sh, s))
        return rc;
    return grad ? fold_param_parts(ws, sh.grid, grad, a.feat, s) : B200MP_OK;
}

}  // namespace b200mp
