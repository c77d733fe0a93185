// csr_reduce.cuh -- the hot kernel: gather feature rows along a CSR row range and reduce them.
//
//   out[i,:] = REDUCE_{e in [rowptr[i], rowptr[i+1])} val[e] * x[col[e], :]        (GATHER)
//   out[i,:] = REDUCE_{e in [ptr[i],    ptr[i+1])}    src[e, :]                    (!GATHER)
//
// Mapping (DESIGN.md section 4.1).  A feature row is cut into 16-byte vectors.  A *lane group* of
// G lanes (G = smallest power of two >= #vectors, capped at a full warp) owns one CSR row; each
// lane keeps VPL vectors of fp32 accumulators in registers and never exchanges data with its
// neighbours, so the reduction order is the CSR order (deterministic, and bit-identical to the
// reference's CPU scatter for fp32).  Narrow rows (G < 32) pack 32/G CSR rows into one warp.  All
// HBM traffic for features is 128-bit, fully coalesced per row (G*16 contiguous bytes), with UNR
// independent row loads in flight per lane.  Column indices and weights are loaded coalesced by
// the whole warp, 32 edges at a time, and broadcast with shuffles (G == 32).
//
// Power-law hubs: rows longer than `chunk` edges are not walked by their own group; the plan
// (b200mp_csr_plan_*) lists them and the kernel's first n_chunks work items each reduce one
// chunk into an fp32 partial; csr_combine_kernel folds the partials in chunk order
// (deterministic, no atomics).
#pragma once

#include <algorithm>

#include "common.cuh"

namespace b200mp {

int get_option_spmm_tune();  // b200mp_set_option("spmm_tune", k): see launch_vec

struct LongRowPlan {
    const int64_t* long_rows;   // [n_long]
    const int64_t* chunk_ptr;   // [n_long + 1]
    int64_t n_long;
    int64_t n_chunks;
    int64_t chunk;              // edges per chunk
    float* partials;            // [n_chunks, feat] fp32
    // optional second source segment (multi-GPU halo rows): column ids >= split are read from
    // x2[(c - split), :] instead of x[c, :], so local and received rows never need concatenating
    const void* x2;
    int64_t split;
    // accumulate != 0: out[i,:] += result for rows that have edges (rows without edges are left
    // untouched) -- used to add the halo-edge contributions after the local-edge sweep (sum only)
    int accumulate;
    // peers != nullptr: the source matrix is sharded over GPUs by contiguous row ranges of
    // peer_rows rows; peers[r] is the (NVLink peer-mapped) base address of rank r's rows.  Column c
    // is read from peers[c / peer_rows] + (c % peer_rows) * row_bytes -- remote rows are gathered
    // straight over NVLink inside the kernel, no pack / exchange / unpack pass.
    const unsigned long long* peers;
    int64_t peer_rows;
    // relu_mask != nullptr (with accumulate): after the add, out[i,f] is zeroed where relu_mask[i,f] <= 0 -- the ReLU
    // backward of the layer that PRODUCED this layer's input, applied by the last writer of its gradient (the input
    // x = relu(pre) is its own mask: x > 0 <=> pre > 0) instead of a separate 3-pass elementwise kernel.  Same dtype
    // and shape as out; rows without edges are masked too.
    const void* relu_mask;
};

// The plan of a C-ABI call from its six long-row arguments (include/b200mp.h): counts are non-negative, and long rows
// need their row list, chunk offsets and a positive chunk, plus fp32 partials when `needs_partials` (sweeps that only
// split rows write none).  Without long rows n_chunks is ignored.  The optional fields stay zero.
inline int make_plan(LongRowPlan& plan, const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                     int64_t n_chunks, int64_t chunk, float* partials, bool needs_partials) {
    B200MP_CHECK_ARG(n_long_rows >= 0 && n_chunks >= 0);
    B200MP_CHECK_ARG(n_long_rows == 0 || (long_rows && chunk_ptr && chunk > 0 && (partials || !needs_partials)));
    plan = LongRowPlan{long_rows, chunk_ptr, n_long_rows, n_long_rows ? n_chunks : 0, chunk, partials,
                       nullptr, 0, 0, nullptr, 0, nullptr};
    return B200MP_OK;
}

// Base address of source row c for the three addressing modes (plain, [local | halo], peer table).
__device__ __forceinline__ const char* row_base(const LongRowPlan& plan, const char* xb, const char* xb2, int64_t split,
                                                size_t row_bytes, int64_t c) {
    if (plan.peers) {
        const int64_t r = c / plan.peer_rows;
        return reinterpret_cast<const char*>(__ldg(plan.peers + r)) + static_cast<size_t>(c - r * plan.peer_rows) * row_bytes;
    }
    return (c < split ? xb : xb2) + static_cast<size_t>(c) * row_bytes;
}

// Decode a work item into (row, begin, end, is_chunk).  Items [0, n_chunks) are chunks of long
// rows (scheduled first: they are the long poles), items [n_chunks, n_chunks + n_rows) are rows.
template <typename I>
__device__ __forceinline__ bool decode_item(int64_t item, const I* __restrict__ rowptr, int64_t n_rows,
                                            const LongRowPlan& plan, int64_t& row, int64_t& begin,
                                            int64_t& end, bool& is_chunk) {
    if (item < plan.n_chunks) {
        // binary search: largest j with chunk_ptr[j] <= item
        int64_t lo = 0, hi = plan.n_long;
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(plan.chunk_ptr + mid) <= item) lo = mid; else hi = mid;
        }
        row = __ldg(plan.long_rows + lo);
        const int64_t k = item - __ldg(plan.chunk_ptr + lo);
        begin = static_cast<int64_t>(__ldg(rowptr + row)) + k * plan.chunk;
        const int64_t row_end = static_cast<int64_t>(__ldg(rowptr + row + 1));
        end = begin + plan.chunk < row_end ? begin + plan.chunk : row_end;
        is_chunk = true;
        return true;
    }
    row = item - plan.n_chunks;
    if (row >= n_rows) return false;
    begin = static_cast<int64_t>(__ldg(rowptr + row));
    end = static_cast<int64_t>(__ldg(rowptr + row + 1));
    is_chunk = false;
    if (plan.n_long > 0 && end - begin > plan.chunk) return false;  // handled as chunks
    return true;
}

template <int RED>
__device__ __forceinline__ float finalize(float acc, int64_t deg, bool is_mean, bool inf_to_zero) {
    if (RED == B200MP_SUM) {
        if (is_mean) acc = __fdiv_rn(acc, static_cast<float>(deg < 1 ? 1 : deg));
    } else if (RED == B200MP_MIN || RED == B200MP_MAX) {
        if (deg == 0) acc = 0.0f;                                   // _scatter.py:98-100
        if (inf_to_zero && isinf(acc)) acc = 0.0f;                  // _segment.py:48-49
    }
    return acc;
}

// Adds one unpacked 16-byte vector into a shared-memory column slot (SELF_COLSUM below).
template <int EPV>
__device__ __forceinline__ void add_to_slot(float* s, const float (&f)[EPV]) {
#pragma unroll
    for (int q = 0; q < EPV / 4; ++q) {
        float4 t = reinterpret_cast<float4*>(s)[q];
        t.x += f[4 * q];
        t.y += f[4 * q + 1];
        t.z += f[4 * q + 2];
        t.w += f[4 * q + 3];
        reinterpret_cast<float4*>(s)[q] = t;
    }
}

// UNR_OVR / BLOCK / MINB are tuning knobs (independent row loads in flight per lane, CTA size,
// minimum resident CTAs per SM => register cap); defaults below.
//
// SELF_COLSUM (weighted sum with gather; plain addressing and none of the plan's optional fields): the sweep also sums,
// unweighted, the x row of every edge whose column is its own row.  On a graph with exactly one self-loop per row that
// is the column sum of x, taken from rows the sweep loads anyway (GCNConv's bias gradient from the transposed sweep).
// Each lane group adds into its own F-float slot in dynamic shared memory, one read-modify-write per row, and a lane
// touches only its own columns: no atomics, no accumulator registers in the edge loop.  So that a CTA's slots cover
// many rows, the grid is a set of resident CTAs and lane group q takes the items q, q + Q, q + 2Q, ... (Q lane groups
// in the grid); the per-row work and the CSR order of each row's sum are those of the one-item-per-group launch.  At
// the end each CTA folds its slots in group order into colsum_parts[blockIdx.x, :].
template <typename T, typename I, int G, int VPL, int RED, bool GATHER, int UNR_OVR = 0, int BLOCK = 256,
          int MINB = 1, bool SELF_COLSUM = false>
__global__ void __launch_bounds__(BLOCK, MINB)
csr_reduce_kernel(const I* __restrict__ rowptr, const I* __restrict__ col,
                  const float* __restrict__ val, const T* __restrict__ x, T* __restrict__ out,
                  int64_t n_rows, int n_vec, bool is_mean, bool inf_to_zero, LongRowPlan plan,
                  const float* __restrict__ bias, float* __restrict__ colsum_parts) {
    static_assert(!SELF_COLSUM || (RED == B200MP_SUM && GATHER), "the self-loop column sum rides a weighted-sum gather");
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int UNR = UNR_OVR ? UNR_OVR : (VPL == 1 ? 8 : (VPL == 2 ? 4 : 2));
    constexpr int GROUPS = BLOCK / G;
    extern __shared__ float4 csr_colsum_smem[];              // SELF_COLSUM: [GROUPS][feat] fp32
    const int lig = threadIdx.x & (G - 1);                     // lane in group
    const int feat = n_vec * EPV;
    float* const slot = reinterpret_cast<float*>(csr_colsum_smem) + static_cast<size_t>(threadIdx.x / G) * feat;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = reinterpret_cast<const char*>(x);
    const char* xb2 = plan.x2 ? reinterpret_cast<const char*>(plan.x2) - static_cast<size_t>(plan.split) * row_bytes : xb;
    const int64_t split = plan.x2 ? plan.split : INT64_MAX;
    const bool weighted = SELF_COLSUM || val;
    auto src_row = [&](int64_t c) {
        return SELF_COLSUM ? xb + static_cast<size_t>(c) * row_bytes : row_base(plan, xb, xb2, split, row_bytes, c);
    };

    auto reduce_item = [&](const int64_t item) {
        int64_t row, begin, end;
        bool is_chunk;
        const bool active = decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk);
        if (G < 32 && !active) return;          // groups are independent below warp width
        if (G == 32 && !active) return;         // warp-uniform

        for (int vbase = 0; vbase < n_vec; vbase += G * VPL) {   // one trip unless feat is huge
            float acc[VPL][EPV];
#pragma unroll
            for (int k = 0; k < VPL; ++k)
#pragma unroll
                for (int i = 0; i < EPV; ++i) acc[k][i] = red_identity<RED>();
            bool vvalid[VPL];
#pragma unroll
            for (int k = 0; k < VPL; ++k) vvalid[k] = (vbase + lig + k * G) < n_vec;
            const size_t voff = static_cast<size_t>(vbase + lig) * 16;

            if (G == 32) {
                for (int64_t e0 = begin; e0 < end; e0 += 32) {
                    const int n = static_cast<int>(end - e0 < 32 ? end - e0 : 32);
                    int64_t c_l = 0;
                    float w_l = 1.0f;
                    bool self_l = false;
                    if (lig < n) {
                        c_l = GATHER ? static_cast<int64_t>(ldg_idx(col + e0 + lig)) : (e0 + lig);
                        if (weighted) w_l = __ldg(val + e0 + lig);
                        if (SELF_COLSUM) self_l = c_l == row;
                        // each lane resolves the row address of ITS edge once; the address is what is broadcast
                        c_l = static_cast<int64_t>(reinterpret_cast<uintptr_t>(src_row(c_l)));
                    }
                    const unsigned self_bits = SELF_COLSUM ? __ballot_sync(0xffffffffu, self_l) : 0u;
                    for (int j = 0; j < n; j += UNR) {
                        Vec16 buf[UNR][VPL];
                        float w[UNR];
#pragma unroll
                        for (int u = 0; u < UNR; ++u) {
                            const int64_t c = __shfl_sync(0xffffffffu, c_l, (j + u) & 31);
                            w[u] = __shfl_sync(0xffffffffu, w_l, (j + u) & 31);
                            if (j + u < n) {
                                const char* p = reinterpret_cast<const char*>(static_cast<uintptr_t>(c)) + voff;
#pragma unroll
                                for (int k = 0; k < VPL; ++k)
                                    if (vvalid[k]) buf[u][k] = ldg_row16(p + static_cast<size_t>(k) * G * 16);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < UNR; ++u) {
                            if (j + u < n) {
#pragma unroll
                                for (int k = 0; k < VPL; ++k) {
                                    if (vvalid[k]) {
                                        float f[EPV];
                                        ElemTraits<T>::unpack(buf[u][k], f);
#pragma unroll
                                        for (int i = 0; i < EPV; ++i) {
                                            const float m = weighted ? __fmul_rn(w[u], f[i]) : f[i];
                                            acc[k][i] = red_combine<RED>(acc[k][i], m);
                                        }
                                        if (SELF_COLSUM && ((self_bits >> (j + u)) & 1u))
                                            add_to_slot<EPV>(slot + static_cast<size_t>(vbase + lig + k * G) * EPV, f);
                                    }
                                }
                            }
                        }
                    }
                }
            } else {
                for (int64_t e = begin; e < end; e += UNR) {
                    Vec16 buf[UNR][VPL];
                    float w[UNR];
                    unsigned self_bits = 0;
#pragma unroll
                    for (int u = 0; u < UNR; ++u) {
                        w[u] = 1.0f;
                        if (e + u < end) {
                            const int64_t c = GATHER ? static_cast<int64_t>(ldg_idx(col + e + u)) : (e + u);
                            if (weighted) w[u] = __ldg(val + e + u);
                            if (SELF_COLSUM && c == row) self_bits |= 1u << u;
                            if (vvalid[0]) buf[u][0] = ldg_row16(src_row(c) + voff);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UNR; ++u) {
                        if (e + u < end && vvalid[0]) {
                            float f[EPV];
                            ElemTraits<T>::unpack(buf[u][0], f);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) {
                                const float m = weighted ? __fmul_rn(w[u], f[i]) : f[i];
                                acc[0][i] = red_combine<RED>(acc[0][i], m);
                            }
                            if (SELF_COLSUM && ((self_bits >> u) & 1u))
                                add_to_slot<EPV>(slot + static_cast<size_t>(vbase + lig) * EPV, f);
                        }
                    }
                }
            }

            // ---- epilogue: one 128-bit store per vector
            if (is_chunk) {
                float* pbase = plan.partials + static_cast<size_t>(item) * n_vec * EPV;
#pragma unroll
                for (int k = 0; k < VPL; ++k)
                    if (vvalid[k]) store_partial<EPV>(pbase + static_cast<size_t>(vbase + lig + k * G) * EPV, acc[k]);
            } else {
                const int64_t deg = end - begin;
                char* ob = reinterpret_cast<char*>(out) + static_cast<size_t>(row) * row_bytes;
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    if (!vvalid[k]) continue;
                    float f[EPV];
#pragma unroll
                    for (int i = 0; i < EPV; ++i) f[i] = finalize<RED>(acc[k][i], deg, !SELF_COLSUM && is_mean, inf_to_zero);
                    if (!SELF_COLSUM && bias) {
                        const float* bp = bias + static_cast<size_t>(vbase + lig + k * G) * EPV;
#pragma unroll
                        for (int i = 0; i < EPV; ++i) f[i] = __fadd_rn(f[i], __ldg(bp + i));
                    }
                    if (!SELF_COLSUM && plan.accumulate) {
                        if (deg == 0 && !plan.relu_mask) continue;
                        float o[EPV];
                        ElemTraits<T>::unpack(*reinterpret_cast<const Vec16*>(ob + static_cast<size_t>(vbase + lig + k * G) * 16), o);
#pragma unroll
                        for (int i = 0; i < EPV; ++i) f[i] = deg == 0 ? o[i] : __fadd_rn(o[i], f[i]);
                        if (plan.relu_mask) {
                            float mk[EPV];
                            ElemTraits<T>::unpack(ldg_stream16(static_cast<const char*>(plan.relu_mask) + static_cast<size_t>(row) * row_bytes +
                                                               static_cast<size_t>(vbase + lig + k * G) * 16), mk);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) f[i] = mk[i] > 0.0f ? f[i] : 0.0f;
                        }
                    }
                    stg_stream16(ob + static_cast<size_t>(vbase + lig + k * G) * 16, ElemTraits<T>::pack(f));
                }
            }
        }
    };

    const int64_t first = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    if constexpr (SELF_COLSUM) {
        for (int i = threadIdx.x; i < GROUPS * feat; i += BLOCK) reinterpret_cast<float*>(csr_colsum_smem)[i] = 0.0f;
        __syncthreads();
        const int64_t n_items = plan.n_chunks + n_rows;
        for (int64_t item = first; item < n_items; item += static_cast<int64_t>(gridDim.x) * GROUPS) reduce_item(item);
        __syncthreads();
        for (int f = threadIdx.x; f < feat; f += BLOCK) {
            float s = 0.0f;
            for (int q = 0; q < GROUPS; ++q) s += reinterpret_cast<const float*>(csr_colsum_smem)[q * feat + f];
            colsum_parts[static_cast<size_t>(blockIdx.x) * feat + f] = s;
        }
    } else {
        reduce_item(first);
    }
}

// Fold the fp32 partials of every long row, in chunk order, and write the row.
template <typename T, typename I, int RED>
__global__ void __launch_bounds__(256)
csr_combine_kernel(const I* __restrict__ rowptr, T* __restrict__ out, int64_t feat, bool is_mean,
                   bool inf_to_zero, LongRowPlan plan, const float* __restrict__ bias) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = threadIdx.x; f < feat; f += blockDim.x) {
        float acc = red_identity<RED>();
        for (int64_t c = c0; c < c1; ++c) acc = red_combine<RED>(acc, plan.partials[c * feat + f]);
        acc = finalize<RED>(acc, deg, is_mean, inf_to_zero);
        if (bias) acc = __fadd_rn(acc, bias[f]);
        if (plan.accumulate) acc = __fadd_rn(ElemTraits<T>::to_float(out[row * feat + f]), acc);
        if (plan.relu_mask && !(ElemTraits<T>::to_float(static_cast<const T*>(plan.relu_mask)[row * feat + f]) > 0.0f)) acc = 0.0f;
        out[row * feat + f] = ElemTraits<T>::from_float(acc);
    }
}

// Scalar fallback: feature rows that are not a whole number of aligned 16-byte vectors
// (feat = 1 degree-style sums, odd widths).  One lane group (runtime power-of-two width g) per
// work item, lanes stride over features, 4 edges in flight.
template <typename T, typename I, int RED, bool GATHER>
__global__ void __launch_bounds__(256)
csr_reduce_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col,
                         const float* __restrict__ val, const T* __restrict__ x, T* __restrict__ out,
                         int64_t n_rows, int64_t feat, int g, bool is_mean, bool inf_to_zero,
                         LongRowPlan plan, const float* __restrict__ bias) {
    const int lig = threadIdx.x & (g - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / g;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    for (int64_t f = lig; f < feat; f += g) {
        float acc = red_identity<RED>();
        for (int64_t e = begin; e < end; e += 4) {
            float v[4], w[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                w[u] = 1.0f;
                v[u] = 0.0f;
                if (e + u < end) {
                    const int64_t c = GATHER ? static_cast<int64_t>(ldg_idx(col + e + u)) : (e + u);
                    if (val) w[u] = __ldg(val + e + u);
                    v[u] = ElemTraits<T>::to_float((plan.x2 && c >= plan.split)
                                                       ? static_cast<const T*>(plan.x2)[(c - plan.split) * feat + f]
                                                       : x[c * feat + f]);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (e + u < end) acc = red_combine<RED>(acc, val ? __fmul_rn(w[u], v[u]) : v[u]);
        }
        if (is_chunk)
            plan.partials[item * feat + f] = acc;
        else {
            acc = finalize<RED>(acc, end - begin, is_mean, inf_to_zero);
            if (bias) acc = __fadd_rn(acc, bias[f]);
            if (plan.accumulate) {
                if (end == begin && !plan.relu_mask) continue;
                const float o = ElemTraits<T>::to_float(out[row * feat + f]);
                acc = end == begin ? o : __fadd_rn(o, acc);
                if (plan.relu_mask && !(ElemTraits<T>::to_float(static_cast<const T*>(plan.relu_mask)[row * feat + f]) > 0.0f)) acc = 0.0f;
            }
            out[row * feat + f] = ElemTraits<T>::from_float(acc);
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
// Default launch shape of the lane-group kernel: occupancy over per-lane memory parallelism -- 4 sixteen-byte row loads
// in flight per lane, 128-thread CTAs, registers capped at 40 (fp32) / 64 (bf16: twice the accumulators) => 48 / 32
// warps per SM.
constexpr int kCsrBlock = 128;
template <typename T>
constexpr int csr_min_blocks() { return sizeof(T) == 4 ? 12 : 8; }

template <typename T, typename I, int RED, bool GATHER, int G, int VPL>
inline void launch_vec(const I* rowptr, const I* col, const float* val, const T* x, T* out,
                       int64_t n_rows, int n_vec, bool is_mean, bool inf_to_zero,
                       const LongRowPlan& plan, const float* bias, cudaStream_t stream) {
    const int64_t items = plan.n_chunks + n_rows;
    if (items == 0) return;
#define B200MP_LAUNCH_TUNED(UNR_, BLOCK_, MINB_)                                                           \
    csr_reduce_kernel<T, I, G, VPL, RED, GATHER, UNR_, BLOCK_, MINB_>                                      \
        <<<static_cast<unsigned>(ceil_div(items, BLOCK_ / G)), BLOCK_, 0, stream>>>(                       \
            rowptr, col, val, x, out, n_rows, n_vec, is_mean, inf_to_zero, plan, bias, nullptr)
    if (G == 32 && VPL == 2 && RED == B200MP_SUM && GATHER) {
        // the headline shape (F = 256 fp32 / 512 bf16): tuning variants selectable at run time
        switch (get_option_spmm_tune()) {
            case 1: B200MP_LAUNCH_TUNED(4, 256, 1); return;     // unconstrained registers (86): 16 warps / SM
            case 2: B200MP_LAUNCH_TUNED(4, 256, 4); return;     // <= 64 regs, 32 warps / SM
            case 3: B200MP_LAUNCH_TUNED(1, 256, 8); return;     // <= 32 regs, 64 warps / SM, 2 loads in flight
            default: break;
        }
    }
    B200MP_LAUNCH_TUNED(unroll_for_vpl<VPL>(), kCsrBlock, csr_min_blocks<T>());
#undef B200MP_LAUNCH_TUNED
}

template <typename T, typename I, int RED, bool GATHER>
int csr_reduce_dispatch(const I* rowptr, const I* col, const float* val, const T* x, T* out,
                        int64_t n_rows, int64_t feat, bool is_mean, bool inf_to_zero,
                        LongRowPlan plan, const float* bias, cudaStream_t stream) {
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    const size_t row_bytes = static_cast<size_t>(feat) * sizeof(T);
    // every matrix the vector kernel reads or writes with 128-bit accesses: the halo segment and the ReLU mask too
    const bool vec_ok = (row_bytes % 16 == 0) && aligned16(x) && aligned16(out) && aligned16(plan.x2) &&
                        aligned16(plan.relu_mask) && (plan.n_chunks == 0 || aligned16(plan.partials));
    if (vec_ok) {
        const int n_vec = static_cast<int>(row_bytes / 16);
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            launch_vec<T, I, RED, GATHER, G(), VPL()>(rowptr, col, val, x, out, n_rows, n_vec, is_mean, inf_to_zero,
                                                      plan, bias, stream);
        });
    } else {
        int g = 1;
        while (g < 32 && g < feat) g <<= 1;
        const int64_t items = plan.n_chunks + n_rows;
        const int64_t blocks = ceil_div(items, 256 / g);
        csr_reduce_scalar_kernel<T, I, RED, GATHER><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
            rowptr, col, val, x, out, n_rows, feat, g, is_mean, inf_to_zero, plan, bias);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        csr_combine_kernel<T, I, RED><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
            rowptr, out, feat, is_mean, inf_to_zero, plan, bias);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

// Launch shape of the SELF_COLSUM sweep: 128-thread CTAs as above, but registers capped at 64 (8 resident CTAs, 32 warps
// per SM) for fp32 too.  At the plain launch's 40 the grid-stride loop's state pushes the edge loop's broadcast column
// address and weight into local memory, reloaded before every gather; on an H100 that sweep took 20.4 ms against
// 16.5 ms at 64 registers at the headline shape (48 registers, 40 warps: 17.1 ms).
constexpr int kSelfColsumMinBlocks = 8;

// Weighted sum plus the column sum of x over the self-loop edges (SELF_COLSUM):
// colsum_parts[parts, feat] receives one fp32 partial per CTA, with parts <= max_parts the grid size.  parts comes back
// 0, and nothing is launched, when the rows are not whole 16-byte vectors or the lane groups' slots would not fit in
// 48 KB of shared memory.
template <typename T, typename I>
int csr_sum_self_colsum(const I* rowptr, const I* col, const float* val, const T* x, T* out, int64_t n_rows,
                        int64_t feat, const LongRowPlan& plan, float* colsum_parts, int64_t max_parts, int64_t& parts,
                        cudaStream_t stream) {
    parts = 0;
    const size_t row_bytes = static_cast<size_t>(feat) * sizeof(T);
    if (row_bytes % 16 != 0 || !aligned16(x) || !aligned16(out) || (plan.n_chunks != 0 && !aligned16(plan.partials)))
        return B200MP_OK;
    const int n_vec = static_cast<int>(row_bytes / 16);
    const int64_t items = plan.n_chunks + n_rows;
    cudaError_t err = cudaSuccess;
    lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
        auto kernel = csr_reduce_kernel<T, I, G(), VPL(), B200MP_SUM, true, unroll_for_vpl<VPL()>(), kCsrBlock,
                                        kSelfColsumMinBlocks, true>;
        const size_t smem = static_cast<size_t>(kCsrBlock / G()) * feat * sizeof(float);
        if (smem > 48 * 1024) return;
        // items are dealt out statically, so the whole grid must be resident at once (a CTA left for a second wave
        // would walk its rows alone at the end): ask for a carveout that holds the register-bound CTA count's slots
        int dev = 0, smem_sm = 0;
        if ((err = cudaGetDevice(&dev)) != cudaSuccess ||
            (err = cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev)) != cudaSuccess)
            return;
        const int64_t need = static_cast<int64_t>(kSelfColsumMinBlocks) * (smem + 1024) * 100;   // 1 KB reserved per CTA
        const int pct = static_cast<int>(std::min<int64_t>(100, ceil_div(need, smem_sm)));
        if ((err = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct)) != cudaSuccess) return;
        int per_sm = 0;
        err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCsrBlock, smem);
        if (err != cudaSuccess) return;
        parts = std::min(std::min(static_cast<int64_t>(per_sm) * num_sms(), ceil_div(items, kCsrBlock / G())),
                         max_parts);
        if (parts == 0) return;
        kernel<<<static_cast<unsigned>(parts), kCsrBlock, smem, stream>>>(rowptr, col, val, x, out, n_rows, n_vec, false,
                                                                           false, plan, nullptr, colsum_parts);
    });
    B200MP_CUDA(err);
    B200MP_LAUNCH_CHECK();
    if (parts > 0 && plan.n_long > 0) {
        csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
            rowptr, out, feat, false, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

// Expands the runtime (reduce) code into template instantiations.
template <typename T, typename I, bool GATHER>
int csr_reduce_by_op(const I* rowptr, const I* col, const float* val, const T* x, T* out,
                     int64_t n_rows, int64_t feat, int reduce, bool inf_to_zero, LongRowPlan plan,
                     const float* bias, cudaStream_t stream) {
    switch (reduce) {
        case B200MP_SUM:
            return csr_reduce_dispatch<T, I, B200MP_SUM, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, false, plan, bias, stream);
        case B200MP_MEAN:
            return csr_reduce_dispatch<T, I, B200MP_SUM, GATHER>(rowptr, col, val, x, out, n_rows, feat, true, false, plan, bias, stream);
        case B200MP_MIN:
            return csr_reduce_dispatch<T, I, B200MP_MIN, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, inf_to_zero, plan, bias, stream);
        case B200MP_MAX:
            return csr_reduce_dispatch<T, I, B200MP_MAX, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, inf_to_zero, plan, bias, stream);
        default:
            set_error("csr_reduce: unsupported reduce %d", reduce);
            return B200MP_ERR_UNSUPPORTED;
    }
}

}  // namespace b200mp
