// quantile.cu -- QuantileAggregation and MedianAggregation (nn/aggr/quantile.py:71-130) as one selection sweep over
// the destination CSR, and its backward.  No [E, F] message matrix is sorted, gathered or stored.
//
// Contract (shared with the numpy restatement in tests/quantile_oracle.py and DESIGN.md section 4.2):
//
// Groups and ranks.  Destination row i holds count_i messages from CSR offset ptr_i (the same number as the
// reference's cumsum(bincount(index))).  For each q (the module's fp32 buffer, read on the device):
//   h = fl32(q * fl32(count_i - 1)),   P = fl32(h + fl32(ptr_i))                        (quantile.py:88)
//   lower: floor(P) - ptr_i   higher: ceil(P) - ptr_i   nearest: rint(P) - ptr_i (round half to even of the global
//   P, so an odd offset rounds k + 0.5 up and an even one down)   linear / midpoint: both, frac = P - floor(P).
// When ptr_i + count_i - 1 < 2^24 that is the reference's fp32 arithmetic bit for bit.  Beyond it fl32(ptr_i) is no
// longer exact and the reference picks outside the group; here the same ranks are formed exactly from h and the
// integer offset (floor(h), ceil(h), frac = h - floor(h), and the half-even tie decided by the parity of
// floor(h) + ptr_i).  Every rank is then clamped into [0, count_i - 1]: past 2^24 fl32(count_i - 1) may round up
// (count_i = 2^24 + 4 and q = 1 give h = count_i), and the clamp keeps that pick on the group's last element, which
// is what q = 1 means; so every pick stays inside its group.  (Below 2^24 the clamp never acts for q in [0, 1].)
//
// Order.  Keys are order-preserving unsigned images of the value (32 bits for fp32, 16 for bf16): -0.0 and +0.0 get
// one key, every NaN one key above +inf (torch.sort puts NaN last), and ties are ordered by CSR slot, which is the
// caller's message order.  The value returned is the chosen element's own bits.
//
// Output, rounded as ATen rounds each op (no contraction):  midpoint = 0.5 l + 0.5 r in the storage dtype; fp32
// linear = l + (r - l) frac; bf16 linear rounds r - l to bf16, multiplies by the fp32 frac and adds l in fp32, and the
// result is fp32 (the reference's type promotion).  An empty row gives fill_value in the output dtype.  With Q
// quantiles row i of the output is [q_0 | q_1 | ... | q_{Q-1}], F channels each (quantile.py:125-129).
//
// Gradient.  g goes to the chosen element for lower / higher / nearest, 0.5 g to each of the two for midpoint, and
// g - g frac (floor) and g frac (ceil) for linear (bf16: round(round(g) - round(g frac)) and round(g frac), as
// autograd casts each into the bf16 messages).  Contributions to one element are summed: first over q in order for
// the floor picks and for the ceil picks, each add rounded to the storage dtype, then the two sums.
//
// Algorithm.  A lane group per destination row, one lane per channel (lanes stride over wider rows).  A lane selects
// each rank by radix select on its own channel's keys: 4-bit digits from the top, 16 counters per lane in lane-private
// shared memory (no atomics), accumulating the count of smaller keys; once the chosen digit holds a single key, or
// after the last digit, one tie pass walks the row in slot order for the (rank - less)-th matching key.  Every pass
// re-reads the row through L1 / L2.  Rows of the long-row plan (hubs) take one CTA per 32 channels instead: eight
// warps split the row into contiguous ranges, count per range, and warp 0 sums the eight histograms (integers: the
// order does not matter) and picks the digit; the tie pass takes an exclusive prefix of the per-range tie counts in
// range order.  A known limit: a hub row never spans more than one CTA per 32 channels, so its forward time grows
// with its length (DESIGN.md section 4.2).  The forward records each pick as one bit per (message, rank, channel) --
// the saved state, E * R * Q * ceil(F / 32) words for R = 2 (linear, midpoint) or 1 ranks per q -- set by integer
// atomicOr, as the channels of one word belong to different lanes.  The destination sweep of the backward writes the
// edge rows' gradient densely in the caller's order; the transposed sweep sums, over each source's out-edges, the
// gradient of the picked elements, reading g only where a bit is set, and splits hub sources by the transposed plan
// (fp32 chunk partials folded in chunk order).  Nothing is float-atomic, and a second run gives the same bits.
#include "csr_reduce.cuh"

namespace b200mp {

enum QuantInterp { kQLinear = 0, kQLower = 1, kQHigher = 2, kQNearest = 3, kQMidpoint = 4 };

constexpr int kQBlock = 128;      // threads per CTA of the row sweeps
constexpr int kQHubWarps = 8;     // warps (row ranges) per CTA of the hub kernel

__host__ __device__ __forceinline__ int q_ranks(int interp) {
    return (interp == kQLinear || interp == kQMidpoint) ? 2 : 1;
}

struct QArgs {
    const void* src;     // x [n_src, feat] (gathered through col) or edge rows [n_edges, feat] (read through perm)
    const float* q;      // [n_q] fp32
    int64_t n_q;
    int interp;
    float fill;
    bool out_f32;        // bf16 linear: the output (and grad_out) is fp32
    void* out;           // fwd: [n_rows, n_q * feat]; dst: grad of the edge rows [n_edges, feat]; src: grad_x
    uint32_t* bits;      // [n_edges (caller order), R * n_q, words] pick bits
    const void* g;       // grad_out [n_dst, n_q * feat]
    int64_t feat;
    int64_t words;       // ceil(feat / 32)
};

// The order-preserving key of a value loaded as fp32; bf16 values convert exactly, so their key is the top half.
template <typename T>
__device__ __forceinline__ uint32_t q_key(float v) {
    constexpr int KB = sizeof(T) * 8;
    if (v != v) return KB == 32 ? 0xffffffffu : 0xffffu;
    uint32_t u = __float_as_uint(v) >> (32 - KB);
    const uint32_t sign = 1u << (KB - 1);
    if (u == sign) u = 0;                                         // -0.0 == +0.0
    const uint32_t all = KB == 32 ? 0xffffffffu : 0xffffu;
    return (u & sign) ? (~u & all) : (u | sign);
}

template <typename T>
__device__ __forceinline__ float q_ld(const void* p, int64_t i) {
    return ElemTraits<T>::to_float(__ldg(static_cast<const T*>(p) + i));
}

// The value of CSR slot e in channel f: x[col[e]] or the edge row perm[e] (e without perm).
template <typename T, typename I, bool GATHER>
__device__ __forceinline__ float q_val(const QArgs& a, const I* __restrict__ col, const I* __restrict__ perm,
                                       int64_t e, int64_t f) {
    const int64_t r = GATHER ? static_cast<int64_t>(ldg_idx(col + e))
                             : (perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e);
    return q_ld<T>(a.src, r * a.feat + f);
}

template <typename I>
__device__ __forceinline__ int64_t q_eid(const I* __restrict__ perm, int64_t e) {
    return perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e;
}

// The floor and ceil (or the single) rank of one q in a group of `count` at offset `ptr`, and frac.
struct QRank {
    int64_t lo, hi;
    float frac;
};

// A rank clamped into the group [0, count - 1].  Past 2^24 messages fl32(count - 1) may round up, so h (and with it
// every rank) may name the slot one past the group's end; a q outside [0, 1] (a loaded state_dict) could name any.
__device__ __forceinline__ int64_t q_clamp_rank(int64_t r, int64_t count) {
    return r < 0 ? 0 : (r > count - 1 ? count - 1 : r);
}

__device__ __forceinline__ QRank q_rank(float q, int64_t ptr, int64_t count, int interp) {
    const float h = __fmul_rn(q, static_cast<float>(count - 1));
    int64_t fl, ce, ne;
    float frac;
    if (ptr + count - 1 < (int64_t{1} << 24)) {                   // the reference's fp32 arithmetic
        const float P = __fadd_rn(h, static_cast<float>(ptr));
        const float pf = floorf(P);
        frac = __fsub_rn(P, pf);
        fl = static_cast<int64_t>(pf) - ptr;
        ce = static_cast<int64_t>(ceilf(P)) - ptr;
        ne = static_cast<int64_t>(rintf(P)) - ptr;
    } else {                                                      // exact: the offset is an integer
        const float hf = floorf(h);
        frac = __fsub_rn(h, hf);
        fl = static_cast<int64_t>(hf);
        ce = frac > 0.0f ? fl + 1 : fl;
        ne = frac < 0.5f ? fl : (frac > 0.5f ? fl + 1 : fl + ((fl + ptr) & 1));
    }
    QRank r;
    r.frac = frac;
    r.lo = q_clamp_rank(interp == kQHigher ? ce : (interp == kQNearest ? ne : fl), count);
    r.hi = q_clamp_rank(interp == kQLower ? fl : (interp == kQNearest ? ne : ce), count);
    return r;
}

// The output of one q from its picked values l (floor) and r (ceil).
template <typename T>
__device__ __forceinline__ float q_value(int interp, float l, float r, float frac) {
    if (interp == kQLinear) return __fadd_rn(l, __fmul_rn(round_to<T>(__fsub_rn(r, l)), frac));
    if (interp == kQMidpoint)
        return round_to<T>(__fadd_rn(round_to<T>(__fmul_rn(0.5f, l)), round_to<T>(__fmul_rn(0.5f, r))));
    return l;
}

template <typename T>
__device__ __forceinline__ void q_store(const QArgs& a, int64_t i, float v) {
    if (a.out_f32) static_cast<float*>(a.out)[i] = v;
    else static_cast<T*>(a.out)[i] = ElemTraits<T>::from_float(v);
}

__device__ __forceinline__ void q_set_bit(const QArgs& a, int64_t eid, int64_t k, int64_t f) {
    atomicOr(a.bits + (eid * (q_ranks(a.interp) * a.n_q) + k) * a.words + (f >> 5), 1u << (f & 31));
}

// The sum over q, in order, of the weights of one pick (j = 0: floor or single, 1: ceil) whose bit is set for message
// eid (w: its words at channel f's word) of destination row `row` (count messages at offset ptr).
template <typename T>
__device__ __forceinline__ float q_pick_grad(const QArgs& a, const uint32_t* w, int j, int64_t row, int64_t ptr,
                                             int64_t count, int64_t f) {
    const int64_t Q = a.n_q;
    const uint32_t bit = 1u << (f & 31);
    float s = 0.0f;
#pragma unroll 1
    for (int64_t q = 0; q < Q; ++q) {
        if (!(__ldg(w + (j * Q + q) * a.words) & bit)) continue;
        const int64_t gi = row * Q * a.feat + q * a.feat + f;
        const float g = a.out_f32 ? __ldg(static_cast<const float*>(a.g) + gi) : q_ld<T>(a.g, gi);
        float c = g;
        if (a.interp == kQMidpoint) {
            c = round_to<T>(__fmul_rn(0.5f, g));
        } else if (a.interp == kQLinear) {
            const float gf = round_to<T>(__fmul_rn(g, q_rank(__ldg(a.q + q), ptr, count, a.interp).frac));
            c = j == 1 ? gf : round_to<T>(__fsub_rn(round_to<T>(g), gf));
        }
        s = round_to<T>(__fadd_rn(s, c));
    }
    return s;
}

// The gradient of message eid in channel f, in the storage dtype: the floor picks' sum plus the ceil picks' sum.
template <typename T>
__device__ __forceinline__ float q_edge_grad(const QArgs& a, int64_t eid, int64_t row, int64_t ptr, int64_t count,
                                             int64_t f) {
    const int R = q_ranks(a.interp);
    const uint32_t* w = a.bits + eid * (R * a.n_q) * a.words + (f >> 5);
    const float s0 = q_pick_grad<T>(a, w, 0, row, ptr, count, f);
    return R == 2 ? round_to<T>(__fadd_rn(s0, q_pick_grad<T>(a, w, 1, row, ptr, count, f))) : s0;
}

// ---------------------------------------------------------------- forward: rows walked by one lane
// Slot of rank r (0-based, in (key, slot) order) among the slots [begin, end) in channel f.  cnt: this lane's 16
// counters, kQBlock apart.
template <typename T, typename I, bool GATHER>
__device__ __forceinline__ int64_t q_select(const QArgs& a, const I* __restrict__ col, const I* __restrict__ perm,
                                            int64_t begin, int64_t end, int64_t f, int64_t r, uint32_t* cnt) {
    constexpr int KB = sizeof(T) * 8;
    uint32_t prefix = 0, mask = 0;
    int64_t less = 0;
#pragma unroll 1
    for (int shift = KB - 4; shift >= 0; shift -= 4) {
#pragma unroll
        for (int b = 0; b < 16; ++b) cnt[b * kQBlock] = 0;
#pragma unroll 4
        for (int64_t e = begin; e < end; ++e) {
            const uint32_t k = q_key<T>(q_val<T, I, GATHER>(a, col, perm, e, f));
            if ((k & mask) == prefix) ++cnt[((k >> shift) & 15u) * kQBlock];
        }
        int64_t acc = less;
        uint32_t c = 0;
        int digit = 15;
#pragma unroll 1
        for (int b = 0; b < 16; ++b) {
            c = cnt[b * kQBlock];
            if (r < acc + c) { digit = b; break; }
            acc += c;
        }
        less = acc;
        prefix |= static_cast<uint32_t>(digit) << shift;
        mask |= 15u << shift;
        if (c == 1) break;                                        // the only candidate left
    }
    int64_t t = r - less;
#pragma unroll 1
    for (int64_t e = begin; e < end; ++e) {
        if ((q_key<T>(q_val<T, I, GATHER>(a, col, perm, e, f)) & mask) == prefix) {
            if (t == 0) return e;
            --t;
        }
    }
    return begin;                                                 // not reached: rank < count
}

template <typename T, typename I, bool GATHER>
__global__ void __launch_bounds__(kQBlock)
quantile_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const I* __restrict__ perm, QArgs a,
                int64_t n_rows, int lg, LongRowPlan plan) {
    __shared__ uint32_t q_cnt[16 * kQBlock];
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t r_, begin, end;
    bool is_chunk;
    if (!decode_item(row, rowptr, n_rows, plan, r_, begin, end, is_chunk)) return;   // plan rows: the hub kernel
    const int64_t count = end - begin;
    const int64_t Q = a.n_q;
    const int R = q_ranks(a.interp);
    uint32_t* cnt = q_cnt + threadIdx.x;
#pragma unroll 1
    for (int64_t f = lig; f < a.feat; f += G) {
#pragma unroll 1
        for (int64_t q = 0; q < Q; ++q) {
            float v = a.fill;
            if (count > 0) {
                const QRank rk = q_rank(__ldg(a.q + q), begin, count, a.interp);
                const int64_t sl = q_select<T, I, GATHER>(a, col, perm, begin, end, f, rk.lo, cnt);
                const int64_t sh =
                    rk.hi == rk.lo ? sl : q_select<T, I, GATHER>(a, col, perm, begin, end, f, rk.hi, cnt);
                v = q_value<T>(a.interp, q_val<T, I, GATHER>(a, col, perm, sl, f),
                               q_val<T, I, GATHER>(a, col, perm, sh, f), rk.frac);
                if (a.bits) {
                    q_set_bit(a, q_eid(perm, sl), q, f);
                    if (R == 2) q_set_bit(a, q_eid(perm, sh), Q + q, f);
                }
            }
            q_store<T>(a, row * Q * a.feat + q * a.feat + f, v);
        }
    }
}

// ---------------------------------------------------------------- forward: hub rows, one CTA per 32 channels
struct QHubShared {
    uint32_t cnt[16][kQHubWarps * 32];
    uint32_t prefix[32], mask[32];
    int64_t less[32], slot[32];
    int32_t done[32], warp[32];
};

template <typename T, typename I, bool GATHER>
__device__ __forceinline__ int64_t q_hub_select(const QArgs& a, const I* __restrict__ col, const I* __restrict__ perm,
                                                int64_t begin, int64_t b0, int64_t b1, int64_t f, bool valid,
                                                int64_t r, QHubShared& sh) {
    constexpr int KB = sizeof(T) * 8;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (w == 0) sh.prefix[lane] = sh.mask[lane] = 0, sh.less[lane] = 0, sh.done[lane] = 0;
    __syncthreads();
#pragma unroll 1
    for (int shift = KB - 4; shift >= 0; shift -= 4) {
        const uint32_t prefix = sh.prefix[lane], mask = sh.mask[lane];
        const bool live = valid && !sh.done[lane];
        uint32_t* cnt = &sh.cnt[0][threadIdx.x];
#pragma unroll
        for (int b = 0; b < 16; ++b) cnt[b * kQHubWarps * 32] = 0;
        if (live) {
#pragma unroll 4
            for (int64_t e = b0; e < b1; ++e) {
                const uint32_t k = q_key<T>(q_val<T, I, GATHER>(a, col, perm, e, f));
                if ((k & mask) == prefix) ++cnt[((k >> shift) & 15u) * kQHubWarps * 32];
            }
        }
        __syncthreads();
        if (w == 0 && live) {
            int64_t acc = sh.less[lane];
            uint32_t c = 0;
            int digit = 15;
#pragma unroll 1
            for (int b = 0; b < 16; ++b) {
                c = 0;
#pragma unroll
                for (int k = 0; k < kQHubWarps; ++k) c += sh.cnt[b][k * 32 + lane];
                if (r < acc + c) { digit = b; break; }
                acc += c;
            }
            sh.less[lane] = acc;
            sh.prefix[lane] = prefix | (static_cast<uint32_t>(digit) << shift);
            sh.mask[lane] = mask | (15u << shift);
            sh.done[lane] = c == 1;
        }
        __syncthreads();
    }
    // tie pass: this range's matches, an exclusive prefix over the ranges in order, then the owning range finds it
    const uint32_t prefix = sh.prefix[lane], mask = sh.mask[lane];
    uint32_t m = 0;
    if (valid) {
#pragma unroll 4
        for (int64_t e = b0; e < b1; ++e)
            m += (q_key<T>(q_val<T, I, GATHER>(a, col, perm, e, f)) & mask) == prefix;
    }
    sh.cnt[0][threadIdx.x] = m;
    if (w == 0) sh.slot[lane] = begin;       // written for every lane: the owning range overwrites it (rank < count)
    __syncthreads();
    if (w == 0 && valid) {
        int64_t t = r - sh.less[lane];
        int k = 0;
        for (; k < kQHubWarps - 1; ++k) {
            const uint32_t c = sh.cnt[0][k * 32 + lane];
            if (t < c) break;
            t -= c;
        }
        sh.warp[lane] = k;
        sh.less[lane] = t;                                        // the rank among the owning range's matches
    }
    __syncthreads();
    if (valid && sh.warp[lane] == w) {
        int64_t t = sh.less[lane];
#pragma unroll 1
        for (int64_t e = b0; e < b1; ++e) {
            if ((q_key<T>(q_val<T, I, GATHER>(a, col, perm, e, f)) & mask) == prefix) {
                if (t == 0) { sh.slot[lane] = e; break; }
                --t;
            }
        }
    }
    __syncthreads();
    return sh.slot[lane];
}

// Declared with a minimum of one resident CTA per SM: without it ptxas keeps a 64-bit slot in local memory in two of
// the instantiations.
template <typename T, typename I, bool GATHER>
__global__ void __launch_bounds__(kQHubWarps * 32, 1)
quantile_hub_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const I* __restrict__ perm, QArgs a,
                    LongRowPlan plan) {
    __shared__ QHubShared sh;
    const int64_t row = plan.long_rows[blockIdx.x];
    const int64_t f = static_cast<int64_t>(blockIdx.y) * 32 + (threadIdx.x & 31);
    const bool valid = f < a.feat;
    const int w = threadIdx.x >> 5;
    const int64_t begin = static_cast<int64_t>(ldg_idx(rowptr + row));
    const int64_t count = static_cast<int64_t>(ldg_idx(rowptr + row + 1)) - begin;
    const int64_t len = (count + kQHubWarps - 1) / kQHubWarps;
    const int64_t b0 = begin + (w * len < count ? w * len : count);
    const int64_t b1 = begin + ((w + 1) * len < count ? (w + 1) * len : count);
    const int64_t Q = a.n_q;
    const int R = q_ranks(a.interp);
#pragma unroll 1
    for (int64_t q = 0; q < Q; ++q) {
        const QRank rk = q_rank(__ldg(a.q + q), begin, count, a.interp);
        const int64_t sl = q_hub_select<T, I, GATHER>(a, col, perm, begin, b0, b1, f, valid, rk.lo, sh);
        const int64_t sr =
            rk.hi == rk.lo ? sl : q_hub_select<T, I, GATHER>(a, col, perm, begin, b0, b1, f, valid, rk.hi, sh);
        if (w == 0 && valid) {
            const float v = q_value<T>(a.interp, q_val<T, I, GATHER>(a, col, perm, sl, f),
                                       q_val<T, I, GATHER>(a, col, perm, sr, f), rk.frac);
            q_store<T>(a, row * Q * a.feat + q * a.feat + f, v);
            if (a.bits) {
                q_set_bit(a, q_eid(perm, sl), q, f);
                if (R == 2) q_set_bit(a, q_eid(perm, sr), Q + q, f);
            }
        }
    }
}

// ---------------------------------------------------------------- backward
// Destination sweep: the gradient of every edge row, written densely in the caller's order; hub rows are split into
// the plan's chunks (each message's gradient is its own, so there is nothing to combine).
template <typename T, typename I>
__global__ void __launch_bounds__(kQBlock)
quantile_dst_kernel(const I* __restrict__ rowptr, const I* __restrict__ perm, QArgs a, int64_t n_rows, int lg,
                    LongRowPlan plan) {
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const int64_t ptr = static_cast<int64_t>(ldg_idx(rowptr + row));
    const int64_t count = static_cast<int64_t>(ldg_idx(rowptr + row + 1)) - ptr;
    T* out = static_cast<T*>(a.out);
#pragma unroll 1
    for (int64_t e = begin; e < end; ++e) {
        const int64_t eid = q_eid(perm, e);
        for (int64_t f = lig; f < a.feat; f += G)
            out[eid * a.feat + f] = ElemTraits<T>::from_float(q_edge_grad<T>(a, eid, row, ptr, count, f));
    }
}

// Transposed sweep: grad_x[j] = the sum over j's out-edges of the picked elements' gradient (fp32, in transposed slot
// order), hub sources split into chunks summed from zero, whose fp32 partials csr_combine_kernel folds in chunk order.
template <typename T, typename I>
__global__ void __launch_bounds__(kQBlock)
quantile_src_kernel(const I* __restrict__ rowptr, const I* __restrict__ rowptr_t, const I* __restrict__ col_t,
                    const I* __restrict__ perm_t, QArgs a, int64_t n_src, int lg, LongRowPlan plan) {
    const int G = 1 << lg;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> lg;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr_t, n_src, plan, row, begin, end, is_chunk)) return;
    const int R = q_ranks(a.interp);
    const int64_t RQ = R * a.n_q;
#pragma unroll 1
    for (int64_t f = lig; f < a.feat; f += G) {
        const uint32_t bit = 1u << (f & 31);
        float acc = 0.0f;
#pragma unroll 1
        for (int64_t t = begin; t < end; ++t) {
            const int64_t eid = static_cast<int64_t>(ldg_idx(perm_t + t));
            const uint32_t* w = a.bits + eid * RQ * a.words + (f >> 5);
            uint32_t any = 0;
            for (int64_t k = 0; k < RQ; ++k) any |= __ldg(w + k * a.words);
            if (!(any & bit)) continue;
            const int64_t i = static_cast<int64_t>(ldg_idx(col_t + t));
            const int64_t ptr = static_cast<int64_t>(ldg_idx(rowptr + i));
            const int64_t count = static_cast<int64_t>(ldg_idx(rowptr + i + 1)) - ptr;
            acc = __fadd_rn(acc, q_edge_grad<T>(a, eid, i, ptr, count, f));
        }
        if (is_chunk) plan.partials[item * a.feat + f] = acc;
        else static_cast<T*>(a.out)[row * a.feat + f] = ElemTraits<T>::from_float(acc);
    }
}

// ---------------------------------------------------------------- host side
inline int q_lg(int64_t feat) {
    int lg = 0;
    while (lg < 5 && (int64_t{1} << lg) < feat) ++lg;
    return lg;
}

inline unsigned q_grid(int64_t items, int lg) { return static_cast<unsigned>(ceil_div(items, kQBlock >> lg)); }

inline int q_check(int64_t n_q, int interp, const float* q, int64_t feat) {
    B200MP_CHECK_ARG(n_q >= 1 && q != nullptr && feat >= 0);
    B200MP_CHECK_ARG(interp >= kQLinear && interp <= kQMidpoint);
    return B200MP_OK;
}

template <typename T, typename I, bool GATHER>
int q_forward(const void* rowptr_, const void* col_, const void* perm_, QArgs a, int64_t n_rows,
              const LongRowPlan& plan, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const I* perm = static_cast<const I*>(perm_);
    LongRowPlan rows = plan;
    rows.n_chunks = 0;                                            // plan rows are the hub kernel's, not chunks
    const int lg = q_lg(a.feat);
    quantile_kernel<T, I, GATHER><<<q_grid(n_rows, lg), kQBlock, 0, s>>>(rowptr, col, perm, a, n_rows, lg, rows);
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        const dim3 grid(static_cast<unsigned>(plan.n_long), static_cast<unsigned>(ceil_div(a.feat, 32)));
        quantile_hub_kernel<T, I, GATHER><<<grid, kQHubWarps * 32, 0, s>>>(rowptr, col, perm, a, plan);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int64_t b200mp_quantile_bits_words(int64_t n_edges, int64_t n_q, int interpolation, int64_t feat) {
    if (n_edges < 0 || n_q < 1 || feat < 0 || interpolation < kQLinear || interpolation > kQMidpoint) return -1;
    return n_edges * q_ranks(interpolation) * n_q * ceil_div(feat, 32);
}

extern "C" int b200mp_quantile_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                   const void* edge_rows, const float* q, int64_t n_q, int interpolation,
                                   float fill_value, void* out, uint32_t* bits, int64_t n_rows, int64_t n_cols,
                                   int64_t n_edges, int64_t feat, const int64_t* long_rows, const int64_t* chunk_ptr,
                                   int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype, int val_dtype,
                                   void* stream) {
    if (int rc = q_check(n_q, interpolation, q, feat)) return rc;
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0);
    B200MP_CHECK_ARG((x == nullptr) != (edge_rows == nullptr));
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, nullptr, false)) return rc;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (bits && n_edges > 0 && feat > 0)
        B200MP_CUDA(cudaMemsetAsync(bits, 0, b200mp_quantile_bits_words(n_edges, n_q, interpolation, feat) * 4, s));
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || x == nullptr || col);
    const bool out_f32 = val_dtype == B200MP_BF16 && interpolation == kQLinear;
    const QArgs a{x ? x : edge_rows, q, n_q, interpolation, fill_value, out_f32, out, bits, nullptr, feat,
                  ceil_div(feat, 32)};
    return dispatch_val_idx(val_dtype, idx_dtype, "quantile_csr", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        return x ? q_forward<T, I, true>(rowptr, col, perm, a, n_rows, plan, s)
                 : q_forward<T, I, false>(rowptr, col, perm, a, n_rows, plan, s);
    });
}

extern "C" int b200mp_quantile_backward_dst(const void* rowptr, const void* perm, const float* q, int64_t n_q,
                                            int interpolation, const uint32_t* bits, const void* grad_out,
                                            void* grad_edge_rows, int64_t n_rows, int64_t n_edges, int64_t feat,
                                            const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                            int64_t n_chunks, int64_t chunk, int idx_dtype, int val_dtype,
                                            void* stream) {
    if (int rc = q_check(n_q, interpolation, q, feat)) return rc;
    B200MP_CHECK_ARG(n_rows >= 0 && n_edges >= 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, nullptr, false)) return rc;
    if (n_rows == 0 || n_edges == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && bits && grad_out && grad_edge_rows);
    const QArgs a{nullptr, q, n_q, interpolation, 0.0f, val_dtype == B200MP_BF16 && interpolation == kQLinear,
                  grad_edge_rows, const_cast<uint32_t*>(bits), grad_out, feat, ceil_div(feat, 32)};
    const int lg = q_lg(feat);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dispatch_val_idx(val_dtype, idx_dtype, "quantile_backward_dst", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        quantile_dst_kernel<T, I><<<q_grid(plan.n_chunks + n_rows, lg), kQBlock, 0, s>>>(
            static_cast<const I*>(rowptr), static_cast<const I*>(perm), a, n_rows, lg, plan);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}

extern "C" int b200mp_quantile_backward_src(const void* rowptr, const void* rowptr_t, const void* col_t,
                                            const void* perm_t, const float* q, int64_t n_q, int interpolation,
                                            const uint32_t* bits, const void* grad_out, void* grad_x, int64_t n_src,
                                            int64_t n_dst, int64_t n_edges, int64_t feat, const int64_t* long_rows,
                                            const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                            int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                            void* stream) {
    if (int rc = q_check(n_q, interpolation, q, feat)) return rc;
    B200MP_CHECK_ARG(n_src >= 0 && n_dst >= 0 && n_edges >= 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && grad_x);
    B200MP_CHECK_ARG(n_edges == 0 || (rowptr && col_t && perm_t && bits && grad_out));
    const QArgs a{nullptr, q, n_q, interpolation, 0.0f, val_dtype == B200MP_BF16 && interpolation == kQLinear,
                  grad_x, const_cast<uint32_t*>(bits), grad_out, feat, ceil_div(feat, 32)};
    const int lg = q_lg(feat);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dispatch_val_idx(val_dtype, idx_dtype, "quantile_backward_src", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        quantile_src_kernel<T, I><<<q_grid(plan.n_chunks + n_src, lg), kQBlock, 0, s>>>(
            static_cast<const I*>(rowptr), static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t),
            static_cast<const I*>(perm_t), a, n_src, lg, plan);
        B200MP_LAUNCH_CHECK();
        if (plan.n_long > 0) {
            csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, s>>>(
                static_cast<const I*>(rowptr_t), static_cast<T*>(grad_x), feat, false, false, plan, nullptr);
            B200MP_LAUNCH_CHECK();
        }
        return B200MP_OK;
    });
}
