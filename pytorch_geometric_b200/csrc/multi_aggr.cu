// multi_aggr.cu -- several aggregations of the same neighbourhood in ONE sweep over the edges.
//
// The reference's FusedAggregation (nn/aggr/fused.py:191-336) shares the degree count and the
// sum between sum / mean / var / std, but still issues one scatter per base reduction (sum, x*x sum,
// min, max), i.e. up to four passes over the [E, F] messages.  Here a lane group walks the CSR row
// once and keeps six running values per feature in registers:
//     s = sum x          q = sum x*x         mn, mx = min, max       cmn, cmx = #edges attaining them
// and the epilogue derives every requested output:
//     mean = s / max(deg,1)                       (fused.py:243-256)
//     var  = q / max(deg,1) - mean*mean           (fused.py:258-283)
//     std  = sqrt(max(var, 1e-5)), -> 0 where <= sqrt(1e-5)   (fused.py:319-323)
//     min / max of an empty group = 0             (_scatter.py:98-100)
//     ties_{min,max} = cm{n,x} (+1 if the result is 0: ATen's scatter_reduce backward counts the
//                      zero-initialised `self`, see oracle_scatter_backward)
// The additions are separate __fmul_rn / __fadd_rn in CSR order, so fp32 results are bit-identical
// to the reference's CPU scatter_add_ for rows that are not chunked.
//
// Two addressing modes: GATHER (x is [n_cols, F], row e reads x[col[e]]) and segment mode
// (col == nullptr: x is the materialised [E, F] message matrix, sorted by destination).
// Hub rows use the same LongRowPlan as the SpMM; their partial state is six fp32 planes per chunk.
//
// Backward: an elementwise prologue folds the output gradients into per-destination fp32 rows
//     A  = g_sum + g_mean/cnt - 2 * g_var' * mean / cnt,   B = 2 * g_var' / cnt,
//     Gmin = g_min / ties_min,  Gmax = g_max / ties_max          (g_var' = g_var + g_std / (2 std))
// and the gradient of one message value x is  A + x * B + [x == mn] * Gmin + [x == mx] * Gmax, summed over
// the destinations the value was sent to (one in segment mode, the out-neighbours in gather mode).  Kernels:
//   multi_aggr_backward_staged_kernel   gather mode, fp32, 64 < F <= 256: warp per source row, A / B rows staged by
//                                       cp.async, the [x == mn] / [x == mx] tests read from the forward's hit bits
//   multi_aggr_backward_vec_kernel      gather mode, other vector shapes: 4 rows + 2 conditional rows per edge
//   multi_aggr_backward_segment_kernel  segment mode: runs of 8 consecutive messages per lane group
//   multi_aggr_backward_kernel          scalar fallback (odd widths, bf16)
// Training forward with hit bits: multi_aggr_masked_kernel (+ multi_aggr_mask_chunks_kernel for hub rows).
#include "csr_reduce.cuh"

namespace b200mp {

int get_option_attn_staged();   // core.cu: cp.async-staged gathers on (default) / off; also gates the hit-bit path
int get_option_multi_tune();    // core.cu: 6 (default) = one-warp CTAs for the row sweeps, 5 = the 128-thread form (A/B)

enum { MA_SUM = 0, MA_MEAN, MA_MIN, MA_MAX, MA_VAR, MA_STD, MA_TIES_MIN, MA_TIES_MAX, MA_SLOTS };

struct MultiOut {
    void* p[MA_SLOTS];      // [n_rows, feat]; slots 0..5 of the value dtype, the two tie planes fp32
    int self_zero;          // count the zero-initialised self as a tie (scatter semantics)
    uint8_t* hit_mask;      // nullable [n_edges, feat / 4] (fp32 gather mode): bit i = x == row min, bit 4 + i = x == row max
};

// What the sweep has to carry per feature (compile-time: unused running values cost registers, and
// the kernel's speed is set by how many warps fit on an SM).
enum { MA_NEED_SUM = 1, MA_NEED_SQ = 2, MA_NEED_MM = 4, MA_NEED_TIES = 8 };
constexpr int kModeSums = MA_NEED_SUM | MA_NEED_SQ;                                   // sum, mean, var, std
constexpr int kModeMM = MA_NEED_MM;                                                   // min, max (inference)
constexpr int kModeAll = MA_NEED_SUM | MA_NEED_SQ | MA_NEED_MM;                       // everything, inference
constexpr int kModeAllTies = MA_NEED_SUM | MA_NEED_SQ | MA_NEED_MM | MA_NEED_TIES;    // training with min / max

struct MultiState {
    float s, q, mn, mx, cmn, cmx;
};

__device__ __forceinline__ void ms_init(MultiState& a) {
    a.s = 0.f;
    a.q = 0.f;
    a.mn = __int_as_float(0x7f800000);
    a.mx = __int_as_float(0xff800000);
    a.cmn = 0.f;
    a.cmx = 0.f;
}
template <int MODE>
__device__ __forceinline__ void ms_push(MultiState& a, float v) {
    if (MODE & MA_NEED_SUM) a.s = __fadd_rn(a.s, v);
    if (MODE & MA_NEED_SQ) a.q = __fadd_rn(a.q, __fmul_rn(v, v));
    if (MODE & MA_NEED_TIES) {
        if (v < a.mn || v != v) { a.mn = v; a.cmn = 1.f; } else if (v == a.mn) a.cmn += 1.f;
        if (v > a.mx || v != v) { a.mx = v; a.cmx = 1.f; } else if (v == a.mx) a.cmx += 1.f;
    } else if (MODE & MA_NEED_MM) {
        // NaN-propagating min / max (= "v < mn || v != v ? v : mn", ATen's amin / amax rule) in one instruction each
        asm("min.NaN.f32 %0, %1, %2;" : "=f"(a.mn) : "f"(a.mn), "f"(v));
        asm("max.NaN.f32 %0, %1, %2;" : "=f"(a.mx) : "f"(a.mx), "f"(v));
    }
}
__device__ __forceinline__ void ms_merge(MultiState& a, const MultiState& b) {   // a then b, in edge order
    a.s = __fadd_rn(a.s, b.s);
    a.q = __fadd_rn(a.q, b.q);
    if (b.mn < a.mn || b.mn != b.mn) { a.mn = b.mn; a.cmn = b.cmn; } else if (b.mn == a.mn) a.cmn += b.cmn;
    if (b.mx > a.mx || b.mx != b.mx) { a.mx = b.mx; a.cmx = b.cmx; } else if (b.mx == a.mx) a.cmx += b.cmx;
}

// Epilogue for one (row, feature): derive the requested outputs from the running state.
template <typename T>
__device__ __forceinline__ void ms_store(const MultiOut& o, size_t idx, const MultiState& a, int64_t deg) {
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    const float mean = __fdiv_rn(a.s, cnt);
    if (o.p[MA_SUM]) static_cast<T*>(o.p[MA_SUM])[idx] = ElemTraits<T>::from_float(a.s);
    if (o.p[MA_MEAN]) static_cast<T*>(o.p[MA_MEAN])[idx] = ElemTraits<T>::from_float(mean);
    const float mn = deg == 0 ? 0.f : a.mn, mx = deg == 0 ? 0.f : a.mx;
    if (o.p[MA_MIN]) static_cast<T*>(o.p[MA_MIN])[idx] = ElemTraits<T>::from_float(mn);
    if (o.p[MA_MAX]) static_cast<T*>(o.p[MA_MAX])[idx] = ElemTraits<T>::from_float(mx);
    if (o.p[MA_TIES_MIN]) static_cast<float*>(o.p[MA_TIES_MIN])[idx] = a.cmn + ((o.self_zero && mn == 0.f) ? 1.f : 0.f);
    if (o.p[MA_TIES_MAX]) static_cast<float*>(o.p[MA_TIES_MAX])[idx] = a.cmx + ((o.self_zero && mx == 0.f) ? 1.f : 0.f);
    if (o.p[MA_VAR] || o.p[MA_STD]) {
        const float var = __fsub_rn(__fdiv_rn(a.q, cnt), __fmul_rn(mean, mean));
        if (o.p[MA_VAR]) static_cast<T*>(o.p[MA_VAR])[idx] = ElemTraits<T>::from_float(var);
        if (o.p[MA_STD]) {
            float sd = __fsqrt_rn(var < 1e-5f ? 1e-5f : var);
            if (sd <= static_cast<float>(0.0031622776601683794)) sd = 0.f;   // math.sqrt(1e-5), fused.py:321
            static_cast<T*>(o.p[MA_STD])[idx] = ElemTraits<T>::from_float(sd);
        }
    }
}

// Vector epilogue: the same, one 16-byte store per requested output.
template <typename T>
__device__ __forceinline__ void ms_store_vec(const MultiOut& o, size_t row, size_t row_bytes, size_t voff,
                                             const MultiState (&a)[ElemTraits<T>::kPerVec], int64_t deg) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    float f[EPV], mean[EPV];
#pragma unroll
    for (int i = 0; i < EPV; ++i) mean[i] = __fdiv_rn(a[i].s, cnt);
    auto put = [&](int slot) {
        stg_stream16(static_cast<char*>(o.p[slot]) + row * row_bytes + voff, ElemTraits<T>::pack(f));
    };
    if (o.p[MA_SUM]) {
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = a[i].s;
        put(MA_SUM);
    }
    if (o.p[MA_MEAN]) {
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = mean[i];
        put(MA_MEAN);
    }
    if (o.p[MA_MIN]) {
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = deg == 0 ? 0.f : a[i].mn;
        put(MA_MIN);
    }
    if (o.p[MA_MAX]) {
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = deg == 0 ? 0.f : a[i].mx;
        put(MA_MAX);
    }
    if (o.p[MA_VAR] || o.p[MA_STD]) {
        float var[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) var[i] = __fsub_rn(__fdiv_rn(a[i].q, cnt), __fmul_rn(mean[i], mean[i]));
        if (o.p[MA_VAR]) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) f[i] = var[i];
            put(MA_VAR);
        }
        if (o.p[MA_STD]) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                float sd = __fsqrt_rn(var[i] < 1e-5f ? 1e-5f : var[i]);
                f[i] = sd <= static_cast<float>(0.0031622776601683794) ? 0.f : sd;
            }
            put(MA_STD);
        }
    }
    // tie planes are fp32 whatever T is: EPV floats = EPV / 4 16-byte stores
    const size_t e0 = row * (row_bytes / sizeof(T)) + voff / sizeof(T);
    auto put_ties = [&](int slot, bool is_min) {
        float t[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            const float ext = deg == 0 ? 0.f : (is_min ? a[i].mn : a[i].mx);
            t[i] = (is_min ? a[i].cmn : a[i].cmx) + ((o.self_zero && ext == 0.f) ? 1.f : 0.f);
        }
        float* dst = static_cast<float*>(o.p[slot]) + e0;
#pragma unroll
        for (int q = 0; q < EPV / 4; ++q) {
            const float t4[4] = {t[4 * q], t[4 * q + 1], t[4 * q + 2], t[4 * q + 3]};
            stg_stream16(dst + 4 * q, ElemTraits<float>::pack(t4));
        }
    };
    if (o.p[MA_TIES_MIN]) put_ties(MA_TIES_MIN, true);
    if (o.p[MA_TIES_MAX]) put_ties(MA_TIES_MAX, false);
}

// Resident 128-thread CTAs per SM the register budget is capped for (occupancy is what hides the
// gather latency: csr_reduce.cuh's sweep found 40 registers / 48 warps per SM best for the plain sum).
constexpr int multi_minb(int mode, int epv) {
    const int state = ((mode & MA_NEED_SUM) ? 1 : 0) + ((mode & MA_NEED_SQ) ? 1 : 0) + ((mode & MA_NEED_MM) ? 2 : 0) +
                      ((mode & MA_NEED_TIES) ? 2 : 0);
    const int regs = state * epv + 16 + 28;          // running values + 4 row vectors in flight + addressing / epilogue
    return regs <= 40 ? 12 : regs <= 48 ? 10 : regs <= 64 ? 8 : regs <= 80 ? 6 : regs <= 96 ? 5 : 4;
}

// One lane group of G lanes per work item (row or hub chunk); a lane owns whole 16-byte vectors
// (v = lig, lig + G, ...) and keeps 4 independent row loads in flight.
template <typename T, typename I, int G, bool GATHER, int MODE>
__global__ void __launch_bounds__(128, multi_minb(MODE, ElemTraits<T>::kPerVec))
multi_aggr_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const T* __restrict__ x, MultiOut outs,
                  int64_t n_rows, int n_vec, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int UNR = 4;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const int64_t feat = static_cast<int64_t>(n_vec) * EPV;
    const char* xb = reinterpret_cast<const char*>(x);
    for (int v = lig; v < n_vec; v += G) {
        MultiState a[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) ms_init(a[i]);
        const size_t voff = static_cast<size_t>(v) * 16;
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 buf[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    const int64_t c = GATHER ? static_cast<int64_t>(ldg_idx(col + e + u)) : (e + u);
                    buf[u] = GATHER ? ldg_row16(xb + static_cast<size_t>(c) * row_bytes + voff)
                                    : ldg_stream16(xb + static_cast<size_t>(c) * row_bytes + voff);
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float f[EPV];
                    ElemTraits<T>::unpack(buf[u], f);
#pragma unroll
                    for (int i = 0; i < EPV; ++i) ms_push<MODE>(a[i], f[i]);
                }
            }
        }
        if (is_chunk) {
            // partial state: [n_chunks][6][feat] fp32
            float* pb = plan.partials + static_cast<size_t>(item) * 6 * feat + static_cast<size_t>(v) * EPV;
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                pb[i] = a[i].s;
                pb[feat + i] = a[i].q;
                pb[2 * feat + i] = a[i].mn;
                pb[3 * feat + i] = a[i].mx;
                pb[4 * feat + i] = a[i].cmn;
                pb[5 * feat + i] = a[i].cmx;
            }
        } else {
            ms_store_vec<T>(outs, static_cast<size_t>(row), row_bytes, voff, a, end - begin);
        }
    }
}

// Training sweep with hit bits (gather mode, fp32, 16 < n_vec <= 64): one WARP per work item.
//   pass 1  the register-form walk above with the four running values s, q, mn, mx (no tie counters: 64 instead of 80
//           registers), and every 16-byte vector it consumes is also parked in a lane-private shared-memory slot
//           (the first kKeep edges of the row: 98 % of the rows of a mean-degree-10 graph fit);
//   pass 2  the row's min / max are final: walk the parked vectors (re-gather only edges >= kKeep), emit one byte per
//           (edge, vector) -- bit i: value i attains the min, bit 4 + i: the max -- and count the bits = the tie counts.
// Hub chunks are not handled here: they go through multi_aggr_kernel<kModeAllTies> (launched over the chunk items only);
// their min / max are final after the combine and their bits are written by multi_aggr_mask_chunks_kernel.  A first version re-gathered every row in pass 2 and cost +28 ms at the 100 M-edge
// shape; parking the vectors makes pass 2 a shared-memory walk.
constexpr int kKeep = 16;
template <typename I, int MINB>
__global__ void __launch_bounds__(32, 4 * MINB)      // ONE warp per CTA: a CTA of four rows lives as long as its longest row, and
multi_aggr_masked_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const float* __restrict__ x,
                         MultiOut outs, int64_t n_rows, int n_vec, LongRowPlan plan) {
    constexpr int UNR = 4;
    constexpr int kSums = MA_NEED_SUM | MA_NEED_SQ | MA_NEED_MM;
    // on a power-law graph that left 11 of the 24 resident warps busy (ncu: 17 % achieved of 37.5 % theoretical occupancy)
    __shared__ Vec16 keep[kKeep][32];
    const int lane = threadIdx.x;
    const int64_t item = plan.n_chunks + static_cast<int64_t>(blockIdx.x);   // rows only
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = reinterpret_cast<const char*>(x);
    for (int v = lane; v < n_vec; v += 32) {
        MultiState a[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) ms_init(a[i]);
        const size_t voff = static_cast<size_t>(v) * 16;
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 buf[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (e + u < end) buf[u] = ldg_row16(xb + static_cast<size_t>(ldg_idx(col + e + u)) * row_bytes + voff);
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    float f[4];
                    ElemTraits<float>::unpack(buf[u], f);
#pragma unroll
                    for (int i = 0; i < 4; ++i) ms_push<kSums>(a[i], f[i]);
                    if (e + u - begin < kKeep) keep[e + u - begin][threadIdx.x] = buf[u];
                }
            }
        }
        uint8_t* mrow = outs.hit_mask + static_cast<size_t>(begin) * n_vec + v;
        const int deg = static_cast<int>(end - begin);
        auto emit = [&](int e, const Vec16& vec) {
            float f[4];
            ElemTraits<float>::unpack(vec, f);
            unsigned bits = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const bool hmn = f[i] == a[i].mn, hmx = f[i] == a[i].mx;
                a[i].cmn += hmn ? 1.f : 0.f;
                a[i].cmx += hmx ? 1.f : 0.f;
                bits |= (hmn ? 1u << i : 0u) | (hmx ? 16u << i : 0u);
            }
            mrow[static_cast<size_t>(e) * n_vec] = static_cast<uint8_t>(bits);
        };
        const int kept = deg < kKeep ? deg : kKeep;
        for (int e = 0; e < kept; ++e) emit(e, keep[e][threadIdx.x]);
        for (int e = kKeep; e < deg; e += UNR) {
            Vec16 buf[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (e + u < deg) buf[u] = ldg_row16(xb + static_cast<size_t>(ldg_idx(col + begin + e + u)) * row_bytes + voff);
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (e + u < deg) emit(e + u, buf[u]);
        }
        ms_store_vec<float>(outs, static_cast<size_t>(row), row_bytes, voff, a, end - begin);
    }
}

// Scalar variant for feature rows that are not whole aligned 16-byte vectors (F = 1 read-outs, odd widths).
template <typename T, typename I, bool GATHER>
__global__ void __launch_bounds__(128)
multi_aggr_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const T* __restrict__ x,
                         MultiOut outs, int64_t n_rows, int64_t feat, int g, LongRowPlan plan) {
    const int lig = threadIdx.x & (g - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / g;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    for (int64_t f = lig; f < feat; f += g) {
        MultiState a;
        ms_init(a);
        for (int64_t e = begin; e < end; e += 4) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                v[u] = 0.f;
                if (e + u < end) {
                    const int64_t c = GATHER ? static_cast<int64_t>(ldg_idx(col + e + u)) : (e + u);
                    v[u] = ElemTraits<T>::to_float(x[c * feat + f]);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (e + u < end) ms_push<kModeAllTies>(a, v[u]);
        }
        if (is_chunk) {
            float* pb = plan.partials + static_cast<size_t>(item) * 6 * feat + f;
            pb[0] = a.s;
            pb[feat] = a.q;
            pb[2 * feat] = a.mn;
            pb[3 * feat] = a.mx;
            pb[4 * feat] = a.cmn;
            pb[5 * feat] = a.cmx;
        } else {
            ms_store<T>(outs, static_cast<size_t>(row) * feat + f, a, end - begin);
        }
    }
}

// Fold the chunk states of every hub row in chunk (= edge) order.
template <typename T, typename I>
__global__ void __launch_bounds__(256)
multi_aggr_combine_kernel(const I* __restrict__ rowptr, MultiOut outs, int64_t feat, LongRowPlan plan) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        MultiState a;
        ms_init(a);
        for (int64_t c = c0; c < c1; ++c) {
            const float* pb = plan.partials + static_cast<size_t>(c) * 6 * feat + f;
            MultiState b{pb[0], pb[feat], pb[2 * feat], pb[3 * feat], pb[4 * feat], pb[5 * feat]};
            ms_merge(a, b);
        }
        ms_store<T>(outs, static_cast<size_t>(row) * feat + f, a, deg);
    }
}

// Hit bits and tie counts of the hub rows' edges (their min / max are only known after the combine): one warp per chunk,
// four gathered vectors in flight.  The combine left ties = (0 | 1 for the zero self); the chunks add their counts
// with atomics -- integers in fp32, exact in any order.
template <typename I>
__global__ void __launch_bounds__(32, 32)
multi_aggr_mask_chunks_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const float* __restrict__ x,
                              const float* __restrict__ out_min, const float* __restrict__ out_max,
                              float* __restrict__ ties_min, float* __restrict__ ties_max,
                              uint8_t* __restrict__ mask, int64_t n_rows, int n_vec, LongRowPlan plan) {
    constexpr int UNR = 4;
    const int lane = threadIdx.x;
    const int64_t item = blockIdx.x;
    if (item >= plan.n_chunks) return;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = reinterpret_cast<const char*>(x);
    for (int v = lane; v < n_vec; v += 32) {
        const size_t voff = static_cast<size_t>(v) * 16;
        float mn[4], mx[4], cmn[4] = {0.f, 0.f, 0.f, 0.f}, cmx[4] = {0.f, 0.f, 0.f, 0.f};
        Vec16 t = {};
        if (out_min) t = ldg_row16(reinterpret_cast<const char*>(out_min) + static_cast<size_t>(row) * row_bytes + voff);
        ElemTraits<float>::unpack(t, mn);
        if (out_max) t = ldg_row16(reinterpret_cast<const char*>(out_max) + static_cast<size_t>(row) * row_bytes + voff);
        ElemTraits<float>::unpack(t, mx);
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 buf[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (e + u < end) buf[u] = ldg_row16(xb + static_cast<size_t>(ldg_idx(col + e + u)) * row_bytes + voff);
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u >= end) continue;
                float f[4];
                ElemTraits<float>::unpack(buf[u], f);
                unsigned bits = 0;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const bool hmn = out_min && f[i] == mn[i], hmx = out_max && f[i] == mx[i];
                    cmn[i] += hmn ? 1.f : 0.f;
                    cmx[i] += hmx ? 1.f : 0.f;
                    bits |= (hmn ? 1u << i : 0u) | (hmx ? 16u << i : 0u);
                }
                mask[static_cast<size_t>(e + u) * n_vec + v] = static_cast<uint8_t>(bits);
            }
        }
        const size_t o = static_cast<size_t>(row) * n_vec * 4 + static_cast<size_t>(v) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (ties_min && cmn[i] != 0.f) atomicAdd(ties_min + o + i, cmn[i]);
            if (ties_max && cmx[i] != 0.f) atomicAdd(ties_max + o + i, cmx[i]);
        }
    }
}

// ---------------------------------------------------------------- backward
struct MultiGrad {
    const float* a;      // additive term              [n_dst, feat] or null
    const float* b;      // multiplier of x            [n_dst, feat] or null
    const void* mn;      // forward min (value dtype)  [n_dst, feat] or null
    const float* gmin;   // g_min / ties_min
    const void* mx;
    const float* gmax;
    const uint8_t* hit_mask;   // gather mode, fp32: the forward's per-(edge, vector) hit bits in CSR edge order ...
    const void* t2csr;         // ... and the CSR slot of every transposed slot (index dtype); replaces mn / mx
};

template <typename T>
__device__ __forceinline__ float mg_term(const MultiGrad& g, size_t di, float xv) {
    float t = g.a ? __ldg(g.a + di) : 0.f;
    if (g.b) t = fmaf(xv, __ldg(g.b + di), t);
    if (g.mn && xv == ElemTraits<T>::to_float(static_cast<const T*>(g.mn)[di])) t += __ldg(g.gmin + di);
    if (g.mx && xv == ElemTraits<T>::to_float(static_cast<const T*>(g.mx)[di])) t += __ldg(g.gmax + di);
    return t;
}

// SEGMENT: item = message e, its single destination is dst_of_edge[e].
// !SEGMENT: item = source row j; destinations are col_t[rowptr_t[j] : rowptr_t[j+1]].
template <typename T, typename I, bool SEGMENT>
__global__ void __launch_bounds__(256)
multi_aggr_backward_kernel(const I* __restrict__ ptr, const I* __restrict__ idx, const T* __restrict__ x,
                           MultiGrad g, T* __restrict__ grad_x, int64_t n_items, int64_t feat, int gw) {
    const int lig = threadIdx.x & (gw - 1);
    const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / gw;
    if (j >= n_items) return;
    if (SEGMENT) {
        const size_t d = static_cast<size_t>(idx[j]) * feat;
        for (int64_t f = lig; f < feat; f += gw) {
            const float xv = ElemTraits<T>::to_float(x[j * feat + f]);
            grad_x[j * feat + f] = ElemTraits<T>::from_float(mg_term<T>(g, d + f, xv));
        }
    } else {
        const int64_t begin = ptr[j], end = ptr[j + 1];
        for (int64_t f = lig; f < feat; f += gw) {
            const float xv = ElemTraits<T>::to_float(x[j * feat + f]);
            float acc = 0.f;
            for (int64_t e = begin; e < end; ++e)
                acc = __fadd_rn(acc, mg_term<T>(g, static_cast<size_t>(idx[e]) * feat + f, xv));
            grad_x[j * feat + f] = ElemTraits<T>::from_float(acc);
        }
    }
}

// Folds the output gradients of one multi-aggregation call into the four per-destination fp32 rows the
// backward sweep reads (one elementwise pass instead of ~15 separate tensor ops on [n_rows, feat]).
struct MultiPrep {
    const void *g_sum, *g_mean, *g_var, *g_std, *g_min, *g_max, *mean, *std;
    const float *ties_min, *ties_max;
    float *term_a, *term_b, *gmin, *gmax;
};

template <typename T, typename I>
__global__ void __launch_bounds__(256)
multi_aggr_prepare_kernel(const I* __restrict__ rowptr, MultiPrep p, int64_t n_rows, int64_t feat, bool semi_grad) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_rows * feat) return;
    const int64_t row = i / feat;
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    auto ld = [&](const void* q) { return ElemTraits<T>::to_float(static_cast<const T*>(q)[i]); };
    if (p.term_a) {
        float a = p.g_sum ? ld(p.g_sum) : 0.f;
        if (p.g_mean) a += ld(p.g_mean) / cnt;
        if (p.g_var || p.g_std) {
            float gv = p.g_var ? ld(p.g_var) : 0.f;
            if (p.g_std) {
                // out = sqrt(clamp(var, 1e-5)) masked to 0 where <= sqrt(1e-5): gradient only where it survived
                const float sd = ld(p.std);
                if (sd > 0.f) gv += ld(p.g_std) * 0.5f / sd;
            }
            // var = E[x^2] - mean^2:  d/dx = 2 x / cnt (dropped under semi_grad, basic.py:106-110) - 2 mean / cnt
            a -= 2.f * gv * ld(p.mean) / cnt;
            if (p.term_b) p.term_b[i] = semi_grad ? 0.f : 2.f * gv / cnt;
        }
        p.term_a[i] = a;
    }
    if (p.gmin) p.gmin[i] = ld(p.g_min) / fmaxf(p.ties_min[i], 1.f);
    if (p.gmax) p.gmax[i] = ld(p.g_max) / fmaxf(p.ties_max[i], 1.f);
}

// fp32 rows of whole 16-byte vectors: one vector per thread, 16-byte streaming loads / stores (the scalar form spends its
// time on a 64-bit division and 4-byte accesses per element: 38 ms for 12 planes of 10 GB, this one is bound by the bytes).
template <typename I>
__global__ void __launch_bounds__(256)
multi_aggr_prepare_vec_kernel(const I* __restrict__ rowptr, MultiPrep p, int64_t n_total, unsigned n_vec, bool semi_grad) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_total) return;
    const int64_t row = n_total < (int64_t{1} << 32) ? static_cast<int64_t>(static_cast<unsigned>(i) / n_vec) : i / n_vec;
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    const float cnt = static_cast<float>(deg < 1 ? 1 : deg);
    const size_t off = static_cast<size_t>(i) * 16;
    auto ld = [&](const void* q, float (&f)[4]) { ElemTraits<float>::unpack(ldg_stream16(static_cast<const char*>(q) + off), f); };
    auto st = [&](float* q, const float (&f)[4]) { stg_stream16(reinterpret_cast<char*>(q) + off, ElemTraits<float>::pack(f)); };
    float t[4], u[4];
    if (p.term_a) {
        float a[4] = {0.f, 0.f, 0.f, 0.f};
        if (p.g_sum) ld(p.g_sum, a);
        if (p.g_mean) {
            ld(p.g_mean, t);
#pragma unroll
            for (int k = 0; k < 4; ++k) a[k] += t[k] / cnt;
        }
        if (p.g_var || p.g_std) {
            float gv[4] = {0.f, 0.f, 0.f, 0.f};
            if (p.g_var) ld(p.g_var, gv);
            if (p.g_std) {
                ld(p.std, t);
                ld(p.g_std, u);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (t[k] > 0.f) gv[k] += u[k] * 0.5f / t[k];
            }
            ld(p.mean, t);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                a[k] -= 2.f * gv[k] * t[k] / cnt;
                u[k] = semi_grad ? 0.f : 2.f * gv[k] / cnt;
            }
            if (p.term_b) st(p.term_b, u);
        }
        st(p.term_a, a);
    }
    if (p.gmin) {
        ld(p.g_min, t);
        ld(p.ties_min, u);
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] = t[k] / fmaxf(u[k], 1.f);
        st(p.gmin, t);
    }
    if (p.gmax) {
        ld(p.g_max, t);
        ld(p.ties_max, u);
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] = t[k] / fmaxf(u[k], 1.f);
        st(p.gmax, t);
    }
}

template <typename T, typename I>
int multi_prep_typed(const void* rowptr, MultiPrep p, int64_t n_rows, int64_t feat, int semi_grad, cudaStream_t stream) {
    const int64_t n = n_rows * feat;
    if constexpr (sizeof(T) == 4) {
        bool vec_ok = feat % 4 == 0;
        for (const void* q : {p.g_sum, p.g_mean, p.g_var, p.g_std, p.g_min, p.g_max, p.mean, p.std, static_cast<const void*>(p.ties_min),
                              static_cast<const void*>(p.ties_max), static_cast<const void*>(p.term_a), static_cast<const void*>(p.term_b),
                              static_cast<const void*>(p.gmin), static_cast<const void*>(p.gmax)})
            vec_ok = vec_ok && aligned16(q);
        if (vec_ok) {
            multi_aggr_prepare_vec_kernel<I><<<static_cast<unsigned>(ceil_div(n / 4, 256)), 256, 0, stream>>>(
                static_cast<const I*>(rowptr), p, n / 4, static_cast<unsigned>(feat / 4), semi_grad != 0);
            B200MP_LAUNCH_CHECK();
            return B200MP_OK;
        }
    }
    multi_aggr_prepare_kernel<T, I><<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, stream>>>(
        static_cast<const I*>(rowptr), p, n_rows, feat, semi_grad != 0);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

// fp32 vector form of the gather-mode backward (rows the masked warp-per-row kernel does not take): a lane group per source
// row, 16-byte loads of the (four + two conditional) per-destination rows, two destinations in flight.
template <typename I, int G>
__global__ void __launch_bounds__(128, 6)
multi_aggr_backward_vec_kernel(const I* __restrict__ ptr, const I* __restrict__ idx, const float* __restrict__ x,
                               MultiGrad g, float* __restrict__ grad_x, int64_t n_items, int n_vec) {
    constexpr int UNR = 2;
    const int lig = threadIdx.x & (G - 1);
    const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    if (j >= n_items) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const int64_t begin = static_cast<int64_t>(ptr[j]);
    const int64_t end = static_cast<int64_t>(ptr[j + 1]);
    for (int v = lig; v < n_vec; v += G) {
        const size_t voff = static_cast<size_t>(v) * 16;
        float xv[4], acc[4] = {0.f, 0.f, 0.f, 0.f};
        ElemTraits<float>::unpack(ldg_stream16(reinterpret_cast<const char*>(x) + static_cast<size_t>(j) * row_bytes + voff), xv);
        for (int64_t e = begin; e < end; e += UNR) {
            // Four rows per destination are always read (additive term, multiplier of x, forward min, forward max);
            // the two tie-normalised gradient rows (g_min / ties, g_max / ties) only by the lanes whose x equals the
            // extremum -- on a hub destination that is ~1 edge in deg per feature, so the sweep moves ~4 rows per edge
            // instead of 6 (the dependent load is rare; on degree-1 rows it always happens and costs what it did).
            Vec16 b[UNR][4];
            size_t offs[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    const size_t off = static_cast<size_t>(idx[e + u]) * row_bytes + voff;
                    offs[u] = off;
                    if (g.a) b[u][0] = ldg_row16(reinterpret_cast<const char*>(g.a) + off);
                    if (g.b) b[u][1] = ldg_row16(reinterpret_cast<const char*>(g.b) + off);
                    if (g.mn) b[u][2] = ldg_row16(static_cast<const char*>(g.mn) + off);
                    if (g.mx) b[u][3] = ldg_row16(static_cast<const char*>(g.mx) + off);
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    bool hit_mn = false, hit_mx = false;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        hit_mn = hit_mn || (g.mn && xv[i] == __uint_as_float(b[u][2].w[i]));
                        hit_mx = hit_mx || (g.mx && xv[i] == __uint_as_float(b[u][3].w[i]));
                    }
                    Vec16 gmn, gmx;
                    if (hit_mn) gmn = ldg_row16(reinterpret_cast<const char*>(g.gmin) + offs[u]);
                    if (hit_mx) gmx = ldg_row16(reinterpret_cast<const char*>(g.gmax) + offs[u]);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float t = g.a ? __uint_as_float(b[u][0].w[i]) : 0.f;
                        if (g.b) t = fmaf(xv[i], __uint_as_float(b[u][1].w[i]), t);
                        if (hit_mn && xv[i] == __uint_as_float(b[u][2].w[i])) t += __uint_as_float(gmn.w[i]);
                        if (hit_mx && xv[i] == __uint_as_float(b[u][3].w[i])) t += __uint_as_float(gmx.w[i]);
                        acc[i] = __fadd_rn(acc[i], t);
                    }
                }
            }
        }
        stg_stream16(reinterpret_cast<char*>(grad_x) + static_cast<size_t>(j) * row_bytes + voff, ElemTraits<float>::pack(acc));
    }
}

// Warp-per-source-row form of the gather-mode backward for wide fp32 rows (n_vec in (16, 64]).  The per-destination rows
// are fetched with cp.async into lane-private shared-memory slots one iteration ahead (the attention kernels' scheme,
// attention.cu): the edge loop no longer alternates "index -> rows -> conditional rows" round trips, the next two
// destinations' rows are already in flight while the tie-gradient rows of the current two are fetched.  Destination
// indices are read 32 at a time (one coalesced load per lane) and broadcast with shuffles.
// The forward's hit bits (one byte per edge and vector, CSR edge order, addressed through t2csr) replace the two 16-byte
// min / max vectors of the destination: 2 rows + 1 byte per edge instead of 4 rows, plus the tie-gradient vectors of the
// lanes that hit (on a degree-d destination every edge attains the extremum of ~1/d of the features).  (A variant of this
// kernel that staged all four rows instead of using the bits was slower than the register form: 113 vs 73 ms.)
template <typename I, int VPL, int kMbT>
__global__ void __launch_bounds__(kMbT, kMbT == 32 ? 20 : 5)
multi_aggr_backward_staged_kernel(const I* __restrict__ ptr, const I* __restrict__ idx, const float* __restrict__ x,
                                  MultiGrad g, float* __restrict__ grad_x, int64_t n_items, int n_vec) {
    constexpr int D = 2, UNR = 2, NR = 2;                  // staged rows: additive term, multiplier of x
    extern __shared__ __align__(16) unsigned char mb_stage[];
    const int lane = threadIdx.x & 31;
    const int64_t j = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    if (j >= n_items) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    bool valid[VPL];
    float xv[VPL][4], acc[VPL][4];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        valid[k] = lane + k * 32 < n_vec;
#pragma unroll
        for (int i = 0; i < 4; ++i) xv[k][i] = acc[k][i] = 0.f;
        if (valid[k])
            ElemTraits<float>::unpack(ldg_stream16(reinterpret_cast<const char*>(x) + static_cast<size_t>(j) * row_bytes +
                                                   static_cast<size_t>(lane + k * 32) * 16), xv[k]);
    }
    const int64_t begin = static_cast<int64_t>(ptr[j]);
    const int deg = static_cast<int>(static_cast<int64_t>(ptr[j + 1]) - begin);
    const int n_it = (deg + UNR - 1) / UNR;
    unsigned char* base = mb_stage + static_cast<size_t>(threadIdx.x) * 16;
    auto slot = [&](int d, int u, int r, int k) {
        return base + static_cast<size_t>(((d * UNR + u) * NR + r) * VPL + k) * (kMbT * 16);
    };
    const char* rows[NR] = {reinterpret_cast<const char*>(g.a), reinterpret_cast<const char*>(g.b)};
    const I* t2csr = static_cast<const I*>(g.t2csr);
    const bool use_mn = g.gmin != nullptr, use_mx = g.gmax != nullptr;
    I i0 = 0, i1 = 0, p0 = 0, p1 = 0;
    int cb = 0;
    auto load_batch = [&](int b, I& ireg, I& preg) {
        ireg = preg = 0;
        if (b * 32 + lane < deg) {
            ireg = ldg_idx(idx + begin + b * 32 + lane);
            preg = ldg_idx(t2csr + begin + b * 32 + lane);
        }
    };
    load_batch(0, i0, p0);
    load_batch(1, i1, p1);
    size_t off_cur[UNR] = {}, off_nxt[UNR] = {};
    unsigned m_cur[UNR][VPL] = {}, m_nxt[UNR][VPL] = {};
    auto issue = [&](int t) {
        const int d = t & (D - 1);
        const bool cur = ((t * UNR) >> 5) == cb;          // UNR divides 32: one iteration never straddles two index batches
        const I ireg = cur ? i0 : i1, preg = cur ? p0 : p1;
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int e = t * UNR + u;
            const size_t off = static_cast<size_t>(__shfl_sync(0xffffffffu, ireg, e & 31)) * row_bytes;
            const size_t moff = static_cast<size_t>(__shfl_sync(0xffffffffu, preg, e & 31)) * n_vec;
            off_nxt[u] = off;
            if (e < deg) {
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    if (!valid[k]) continue;
                    const size_t o = off + static_cast<size_t>(lane + k * 32) * 16;
#pragma unroll
                    for (int r = 0; r < NR; ++r)
                        if (rows[r]) cp_async16(slot(d, u, r, k), rows[r] + o);
                    m_nxt[u][k] = __ldg(g.hit_mask + moff + lane + k * 32);
                }
            }
        }
        cp_async_commit();
    };
    if (n_it > 0) issue(0);
    for (int t = 0; t < n_it; ++t) {
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            off_cur[u] = off_nxt[u];
#pragma unroll
            for (int k = 0; k < VPL; ++k) m_cur[u][k] = m_nxt[u][k];
        }
        if (t + 1 < n_it) {
            issue(t + 1);
            if ((((t + 1) * UNR) >> 5) > cb) {
                i0 = i1;
                p0 = p1;
                ++cb;
                load_batch(cb + 1, i1, p1);
            }
        } else {
            cp_async_commit();
        }
        cp_async_wait<1>();
        const int d = t & (D - 1);
        // first the hit tests of both destinations, so that the (frequent on low-degree destinations) tie-gradient loads
        // of the two go out together
        Vec16 gmn[UNR][VPL], gmx[UNR][VPL];
        unsigned hits[UNR][VPL];                           // bits 0-3: value i attains the min, bits 4-7: the max
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                hits[u][k] = 0;
                if (t * UNR + u >= deg || !valid[k]) continue;
                hits[u][k] = m_cur[u][k] & ((use_mn ? 0x0fu : 0u) | (use_mx ? 0xf0u : 0u));
                const size_t o = off_cur[u] + static_cast<size_t>(lane + k * 32) * 16;
                if (hits[u][k] & 0x0fu) gmn[u][k] = ldg_row16(reinterpret_cast<const char*>(g.gmin) + o);
                if (hits[u][k] & 0xf0u) gmx[u][k] = ldg_row16(reinterpret_cast<const char*>(g.gmax) + o);
            }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (t * UNR + u >= deg || !valid[k]) continue;
                float tm[4] = {0.f, 0.f, 0.f, 0.f};
                if (g.a) {
                    const Vec16 r = *reinterpret_cast<const Vec16*>(slot(d, u, 0, k));
#pragma unroll
                    for (int i = 0; i < 4; ++i) tm[i] = __uint_as_float(r.w[i]);
                }
                if (g.b) {
                    const Vec16 r = *reinterpret_cast<const Vec16*>(slot(d, u, 1, k));
#pragma unroll
                    for (int i = 0; i < 4; ++i) tm[i] = fmaf(xv[k][i], __uint_as_float(r.w[i]), tm[i]);
                }
                if (hits[u][k] & 0x0fu) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (hits[u][k] & (1u << i)) tm[i] += __uint_as_float(gmn[u][k].w[i]);
                }
                if (hits[u][k] & 0xf0u) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (hits[u][k] & (16u << i)) tm[i] += __uint_as_float(gmx[u][k].w[i]);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[k][i] = __fadd_rn(acc[k][i], tm[i]);
            }
        }
    }
    cp_async_wait<0>();
#pragma unroll
    for (int k = 0; k < VPL; ++k)
        if (valid[k])
            stg_stream16(reinterpret_cast<char*>(grad_x) + static_cast<size_t>(j) * row_bytes + static_cast<size_t>(lane + k * 32) * 16,
                         ElemTraits<float>::pack(acc[k]));
}

template <typename I, int VPL, int kMbT>
int multi_bwd_staged_launch(const I* ptr, const I* idx, const float* x, const MultiGrad& g, float* grad_x, int64_t n_items,
                            int n_vec, cudaStream_t stream) {
    // 2 stages x 2 destinations x 2 rows x VPL vectors of 16 bytes per thread
    const size_t smem = static_cast<size_t>(2) * 2 * 2 * VPL * kMbT * 16;
    static bool attr_set = false;
    if (!attr_set && smem > 48 * 1024) {
        B200MP_CUDA(cudaFuncSetAttribute(multi_aggr_backward_staged_kernel<I, VPL, kMbT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem)));
        attr_set = true;
    }
    multi_aggr_backward_staged_kernel<I, VPL, kMbT><<<static_cast<unsigned>(ceil_div(n_items, kMbT / 32)), kMbT, smem, stream>>>(
        ptr, idx, x, g, grad_x, n_items, n_vec);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename T, typename I, bool GATHER, int MODE>
void multi_launch_mode(const I* rowptr, const I* col, const T* x, const MultiOut& outs, int64_t n_rows, int n_vec,
                       const LongRowPlan& plan, cudaStream_t stream) {
    const int64_t items = plan.n_chunks + n_rows;
    // one-warp CTAs (every mode holds >= 52 registers, so 32 resident CTAs per SM are never the limit): a CTA's slots are
    // free as soon as ITS rows are done instead of after the longest row of four warps (power-law degrees); multi_tune 5 =
    // the 128-thread form, kept for A/B
    const int bt = get_option_multi_tune() == 5 ? 128 : 32;
    lane_group_shape<1>(n_vec, [&](auto G, auto) {
        multi_aggr_kernel<T, I, G(), GATHER, MODE><<<static_cast<unsigned>(ceil_div(items, bt / G())), bt, 0, stream>>>(
            rowptr, col, x, outs, n_rows, n_vec, plan);
    });
}

template <typename T, typename I, bool GATHER>
int multi_launch(const I* rowptr, const I* col, const T* x, MultiOut outs, int64_t n_rows, int64_t feat,
                 LongRowPlan plan, cudaStream_t stream) {
    const size_t row_bytes = static_cast<size_t>(feat) * sizeof(T);
    const int64_t items = plan.n_chunks + n_rows;
    bool vec_ok = row_bytes % 16 == 0 && aligned16(x);
    for (int k = 0; k < MA_SLOTS; ++k) vec_ok = vec_ok && aligned16(outs.p[k]);
    if (vec_ok) {
        const int n_vec = static_cast<int>(row_bytes / 16);
        const bool ties = outs.p[MA_TIES_MIN] || outs.p[MA_TIES_MAX];
        const bool mm = ties || outs.p[MA_MIN] || outs.p[MA_MAX];
        const bool sums = outs.p[MA_SUM] || outs.p[MA_MEAN] || outs.p[MA_VAR] || outs.p[MA_STD];
        bool done = false;
        if constexpr (GATHER && sizeof(T) == 4) {
            if (outs.hit_mask) {                                        // (the C entry point checked the shape)
                multi_aggr_masked_kernel<I, 5><<<static_cast<unsigned>(n_rows), 32, 0, stream>>>(
                    rowptr, col, reinterpret_cast<const float*>(x), outs, n_rows, n_vec, plan);   // (<I, 6>: 80 registers with spills, 63.0 vs 60.5 ms)
                if (plan.n_chunks > 0)                                  // n_rows = 0: the chunk items only; no tie counters
                    multi_aggr_kernel<T, I, 32, GATHER, kModeAll><<<static_cast<unsigned>(plan.n_chunks), 32, 0, stream>>>(
                        rowptr, col, x, outs, 0, n_vec, plan);          // (multi_aggr_mask_chunks_kernel counts the hub rows' ties)
                done = true;
            }
        }
        if (done) {
        } else if (ties) multi_launch_mode<T, I, GATHER, kModeAllTies>(rowptr, col, x, outs, n_rows, n_vec, plan, stream);
        else if (mm && sums) multi_launch_mode<T, I, GATHER, kModeAll>(rowptr, col, x, outs, n_rows, n_vec, plan, stream);
        else if (mm) multi_launch_mode<T, I, GATHER, kModeMM>(rowptr, col, x, outs, n_rows, n_vec, plan, stream);
        else multi_launch_mode<T, I, GATHER, kModeSums>(rowptr, col, x, outs, n_rows, n_vec, plan, stream);
    } else {
        int g = 1;
        while (g < 32 && g < feat) g <<= 1;
        multi_aggr_scalar_kernel<T, I, GATHER><<<static_cast<unsigned>(ceil_div(items, 128 / g)), 128, 0, stream>>>(
            rowptr, col, x, outs, n_rows, feat, g, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        multi_aggr_combine_kernel<T, I><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(rowptr, outs, feat, plan);
        B200MP_LAUNCH_CHECK();
        if constexpr (GATHER && sizeof(T) == 4) {
            if (outs.hit_mask) {
                const int n_vec = static_cast<int>(row_bytes / 16);
                multi_aggr_mask_chunks_kernel<I><<<static_cast<unsigned>(plan.n_chunks), 32, 0, stream>>>(
                    rowptr, col, reinterpret_cast<const float*>(x), static_cast<const float*>(outs.p[MA_MIN]),
                    static_cast<const float*>(outs.p[MA_MAX]), static_cast<float*>(outs.p[MA_TIES_MIN]),
                    static_cast<float*>(outs.p[MA_TIES_MAX]), outs.hit_mask, n_rows, n_vec, plan);
                B200MP_LAUNCH_CHECK();
            }
        }
    }
    return B200MP_OK;
}

template <typename T, typename I>
int multi_typed(const void* rowptr, const void* col, const void* x, MultiOut outs, int64_t n_rows, int64_t feat,
                LongRowPlan plan, cudaStream_t stream) {
    if (col)
        return multi_launch<T, I, true>(static_cast<const I*>(rowptr), static_cast<const I*>(col),
                                        static_cast<const T*>(x), outs, n_rows, feat, plan, stream);
    return multi_launch<T, I, false>(static_cast<const I*>(rowptr), static_cast<const I*>(nullptr),
                                     static_cast<const T*>(x), outs, n_rows, feat, plan, stream);
}

template <typename I>
void multi_bwd_vec_launch(const I* ptr, const I* idx, const float* x, const MultiGrad& g, float* grad_x,
                          int64_t n_items, int n_vec, cudaStream_t stream) {
    lane_group_shape<1>(n_vec, [&](auto G, auto) {
        multi_aggr_backward_vec_kernel<I, G()><<<static_cast<unsigned>(ceil_div(n_items, 128 / G())), 128, 0, stream>>>(
            ptr, idx, x, g, grad_x, n_items, n_vec);
    });
}

// Segment-mode backward (one destination per message, messages sorted by destination): a lane group walks kSegRun
// CONSECUTIVE messages, two in flight.  The one-message-per-lane-group form launched E / 8 CTAs of 8 messages each
// (12.5 M CTAs at the 100 M-message shape) and had one dependent load chain per thread; consecutive messages mostly share
// their destination, so its four rows are read through L1 (ld.global.nc with allocation) instead of L2 every time.
constexpr int kSegRun = 8;
template <typename I, int G>
__global__ void __launch_bounds__(128, 6)
multi_aggr_backward_segment_kernel(const I* __restrict__ dst_of_msg, const float* __restrict__ x, MultiGrad g,
                                   float* __restrict__ grad_x, int64_t n_msgs, int n_vec) {
    constexpr int UNR = 2;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    const int64_t begin = item * kSegRun;
    if (begin >= n_msgs) return;
    const int64_t end = begin + kSegRun < n_msgs ? begin + kSegRun : n_msgs;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    auto ld_l1 = [](const void* p) { return *reinterpret_cast<const Vec16*>(__builtin_assume_aligned(p, 16)); };
    for (int v = lig; v < n_vec; v += G) {
        const size_t voff = static_cast<size_t>(v) * 16;
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 xb[UNR], b[UNR][4];
            size_t offs[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    xb[u] = ldg_stream16(reinterpret_cast<const char*>(x) + static_cast<size_t>(e + u) * row_bytes + voff);
                    const size_t off = static_cast<size_t>(dst_of_msg[e + u]) * row_bytes + voff;
                    offs[u] = off;
                    if (g.a) b[u][0] = ld_l1(reinterpret_cast<const char*>(g.a) + off);
                    if (g.b) b[u][1] = ld_l1(reinterpret_cast<const char*>(g.b) + off);
                    if (g.mn) b[u][2] = ld_l1(static_cast<const char*>(g.mn) + off);
                    if (g.mx) b[u][3] = ld_l1(static_cast<const char*>(g.mx) + off);
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u >= end) continue;
                float xv[4], t[4];
                ElemTraits<float>::unpack(xb[u], xv);
                bool hit_mn = false, hit_mx = false;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    hit_mn = hit_mn || (g.mn && xv[i] == __uint_as_float(b[u][2].w[i]));
                    hit_mx = hit_mx || (g.mx && xv[i] == __uint_as_float(b[u][3].w[i]));
                }
                Vec16 gmn = {}, gmx = {};
                if (hit_mn) gmn = ld_l1(reinterpret_cast<const char*>(g.gmin) + offs[u]);
                if (hit_mx) gmx = ld_l1(reinterpret_cast<const char*>(g.gmax) + offs[u]);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    t[i] = g.a ? __uint_as_float(b[u][0].w[i]) : 0.f;
                    if (g.b) t[i] = fmaf(xv[i], __uint_as_float(b[u][1].w[i]), t[i]);
                    if (hit_mn && xv[i] == __uint_as_float(b[u][2].w[i])) t[i] += __uint_as_float(gmn.w[i]);
                    if (hit_mx && xv[i] == __uint_as_float(b[u][3].w[i])) t[i] += __uint_as_float(gmx.w[i]);
                }
                stg_stream16(reinterpret_cast<char*>(grad_x) + static_cast<size_t>(e + u) * row_bytes + voff, ElemTraits<float>::pack(t));
            }
        }
    }
}

template <typename I>
void multi_bwd_segment_launch(const I* idx, const float* x, const MultiGrad& g, float* grad_x, int64_t n_msgs, int n_vec,
                              cudaStream_t stream) {
    const int64_t items = ceil_div(n_msgs, kSegRun);
    lane_group_shape<1>(n_vec, [&](auto G, auto) {
        multi_aggr_backward_segment_kernel<I, G()><<<static_cast<unsigned>(ceil_div(items, 128 / G())), 128, 0, stream>>>(
            idx, x, g, grad_x, n_msgs, n_vec);
    });
}

template <typename T, typename I>
int multi_bwd_typed(const void* ptr, const void* idx, const void* x, MultiGrad g, void* grad_x, int64_t n_items,
                    int64_t feat, int segment, cudaStream_t stream) {
    const bool vec_ok = sizeof(T) == 4 && feat % 4 == 0 && aligned16(x) && aligned16(grad_x) && aligned16(g.a) &&
                        aligned16(g.b) && aligned16(g.mn) && aligned16(g.gmin) && aligned16(g.mx) && aligned16(g.gmax);
    if (vec_ok) {
        const int n_vec = static_cast<int>(feat / 4);
        if (segment)
            multi_bwd_segment_launch<I>(static_cast<const I*>(idx), static_cast<const float*>(x), g, static_cast<float*>(grad_x),
                                        n_items, n_vec, stream);
        else if (g.hit_mask && n_vec > 16 && n_vec <= 64) {
            // (without the mask the staged form holds 4 rows x 2 destinations x 2 stages per thread = 64 KB per CTA; 12 warps
            //  per SM ran the sweep at 113 ms against 73 ms for the register form below at 24 -- measured, r2c_multi_*.json)
            const I* p = static_cast<const I*>(ptr);
            const I* ix = static_cast<const I*>(idx);
            const float* xf = static_cast<const float*>(x);
            float* gx = static_cast<float*>(grad_x);
            // one-warp CTAs (multi_tune 6, default): no warp waits for the longest of four rows
            if (get_option_multi_tune() == 5)
                return n_vec > 32 ? multi_bwd_staged_launch<I, 2, 128>(p, ix, xf, g, gx, n_items, n_vec, stream)
                                  : multi_bwd_staged_launch<I, 1, 128>(p, ix, xf, g, gx, n_items, n_vec, stream);
            return n_vec > 32 ? multi_bwd_staged_launch<I, 2, 32>(p, ix, xf, g, gx, n_items, n_vec, stream)
                              : multi_bwd_staged_launch<I, 1, 32>(p, ix, xf, g, gx, n_items, n_vec, stream);
        } else
            multi_bwd_vec_launch<I>(static_cast<const I*>(ptr), static_cast<const I*>(idx),
                                           static_cast<const float*>(x), g, static_cast<float*>(grad_x), n_items, n_vec, stream);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    }
    int gw = 1;
    while (gw < 32 && gw < feat) gw <<= 1;
    const unsigned blocks = static_cast<unsigned>(ceil_div(n_items, 256 / gw));
    if (segment)
        multi_aggr_backward_kernel<T, I, true><<<blocks, 256, 0, stream>>>(
            static_cast<const I*>(ptr), static_cast<const I*>(idx), static_cast<const T*>(x), g,
            static_cast<T*>(grad_x), n_items, feat, gw);
    else
        multi_aggr_backward_kernel<T, I, false><<<blocks, 256, 0, stream>>>(
            static_cast<const I*>(ptr), static_cast<const I*>(idx), static_cast<const T*>(x), g,
            static_cast<T*>(grad_x), n_items, feat, gw);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_multi_aggr_mask_supported(int64_t feat, int val_dtype, int segment_mode) {
    return val_dtype == B200MP_F32 && !segment_mode && feat % 4 == 0 && feat > 64 && feat <= 256 && get_option_attn_staged();
}

extern "C" int b200mp_multi_aggr_csr(const void* rowptr, const void* col, const void* x, void* out_sum,
                                     void* out_mean, void* out_min, void* out_max, void* out_var, void* out_std,
                                     float* ties_min, float* ties_max, void* hit_mask, int64_t n_rows, int64_t n_src,
                                     int64_t feat, int count_self_zero, const int64_t* long_rows,
                                     const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                     int64_t chunk, float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_src >= 0 && feat >= 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && (x || n_src == 0));
    // the hit mask is a by-product of the tie-counting fp32 vector sweep in gather mode
    B200MP_CHECK_ARG(!hit_mask || (col && b200mp_multi_aggr_mask_supported(feat, val_dtype, 0) && (ties_min || ties_max)));
    MultiOut outs{{out_sum, out_mean, out_min, out_max, out_var, out_std, ties_min, ties_max}, count_self_zero != 0,
                  static_cast<uint8_t*>(hit_mask)};
    return dispatch_val_idx(val_dtype, idx_dtype, "multi_aggr_csr", [&](auto tv, auto ti) {
        return multi_typed<decltype(tv), decltype(ti)>(rowptr, col, x, outs, n_rows, feat, plan,
                                                       static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_multi_aggr_backward(const void* ptr, const void* idx, const void* x, const float* term_a,
                                          const float* term_b, const void* out_min, const float* g_min,
                                          const void* out_max, const float* g_max, const void* hit_mask,
                                          const void* t2csr, void* grad_x, int64_t n_items, int64_t feat,
                                          int segment_mode, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_items >= 0 && feat >= 0);
    if (n_items == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(idx && x && grad_x && (segment_mode || ptr));
    B200MP_CHECK_ARG((!out_min || g_min) && (!out_max || g_max));
    B200MP_CHECK_ARG(!hit_mask || (t2csr && !segment_mode && val_dtype == B200MP_F32 && feat % 4 == 0));
    // the mask is only read by the staged warp-per-row kernel; every other shape compares against out_min / out_max
    const bool masked = hit_mask && b200mp_multi_aggr_mask_supported(feat, val_dtype, segment_mode) && aligned16(x) &&
                        aligned16(grad_x) && aligned16(term_a) && aligned16(term_b) && aligned16(g_min) && aligned16(g_max);
    MultiGrad g{term_a, term_b, masked ? nullptr : out_min, g_min, masked ? nullptr : out_max, g_max,
                masked ? static_cast<const uint8_t*>(hit_mask) : nullptr, masked ? t2csr : nullptr};
    B200MP_CHECK_ARG(masked || ((!g_min || out_min) && (!g_max || out_max)));
    return dispatch_val_idx(val_dtype, idx_dtype, "multi_aggr_backward", [&](auto tv, auto ti) {
        return multi_bwd_typed<decltype(tv), decltype(ti)>(ptr, idx, x, g, grad_x, n_items, feat, segment_mode,
                                                           static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_multi_aggr_prepare_backward(const void* rowptr, const void* g_sum, const void* g_mean,
                                                  const void* g_var, const void* g_std, const void* g_min,
                                                  const void* g_max, const void* mean, const void* std,
                                                  const float* ties_min, const float* ties_max, float* term_a,
                                                  float* term_b, float* gmin_out, float* gmax_out, int64_t n_rows,
                                                  int64_t feat, int semi_grad, int idx_dtype, int val_dtype,
                                                  void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && feat >= 0);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr);
    B200MP_CHECK_ARG(!(g_sum || g_mean || g_var || g_std) || term_a);
    B200MP_CHECK_ARG(!(g_var || g_std) || (mean && term_b));
    B200MP_CHECK_ARG(!g_std || std);
    B200MP_CHECK_ARG(!gmin_out || (g_min && ties_min));
    B200MP_CHECK_ARG(!gmax_out || (g_max && ties_max));
    MultiPrep p{g_sum, g_mean, g_var, g_std, g_min, g_max, mean, std, ties_min, ties_max,
                (g_sum || g_mean || g_var || g_std) ? term_a : nullptr, (g_var || g_std) ? term_b : nullptr,
                gmin_out, gmax_out};
    return dispatch_val_idx(val_dtype, idx_dtype, "multi_aggr_prepare_backward", [&](auto tv, auto ti) {
        return multi_prep_typed<decltype(tv), decltype(ti)>(rowptr, p, n_rows, feat, semi_grad,
                                                            static_cast<cudaStream_t>(stream));
    });
}
