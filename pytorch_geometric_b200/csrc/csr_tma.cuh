// csr_tma.cuh -- persistent, TMA-fed variant of the gather + segmented-reduce kernel for wide
// feature rows (row_bytes >= 512 B, i.e. >= 32 sixteen-byte vectors).
//
// Why: with one lane group per CSR row the chain rowptr -> col -> gather
// is serialised per row (average degree 11) and the bytes in flight per SM are bounded by
// registers (8 x 16 B per lane).  Here
//   * one CTA per SM, persistent; every WARP owns a ring of 32 row slots in shared memory and
//     pulls work units (32 consecutive CSR rows, or one 512-edge chunk of a hub row) from a global
//     atomic counter -- long poles first, no tail;
//   * the gather is issued by the 1-D TMA engine: lane l holds the column index of edge l of the
//     current 32-edge batch and issues `cp.async.bulk.shared.global` of that neighbour's whole
//     feature row (row_bytes, 16 B aligned) into slot l, completion on the slot's mbarrier
//     (SASS: UBLKCP + SYNCS.ARRIVE.TRANS64).  No register staging, so a warp keeps 24..32 rows
//     (24..32 KB at F=256 fp32) in flight and the SM ~190 KB -- 4x the latency-bandwidth product;
//   * the edge stream is continuous across row boundaries: the warp walks the unit's edge range in
//     CSR order, lanes read their 16-byte column of each landed row from shared memory
//     (conflict-free LDS.128), accumulate in fp32 registers and flush a row (one coalesced 128-bit
//     store per lane) whenever the stream crosses a rowptr boundary.  Order of additions per row is
//     still the CSR order => deterministic and bit-identical to the reference's CPU scatter.
//   * slots are re-armed in quarters (8 slots) as soon as they are consumed, with the next batch's
//     column indices prefetched, so the TMA queue never drains inside a unit.
#pragma once

#include "csr_reduce.cuh"

namespace b200mp {

constexpr int kTmaSlots = 32;        // one slot per lane
constexpr int kTmaQuarter = 8;       // re-arm granularity
constexpr int kTmaUnitRows = 32;     // CSR rows per work unit (one rowptr value per lane)

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
// 1-D bulk async copy global -> shared, completion counted in bytes on an mbarrier (TMA engine).
__device__ __forceinline__ void tma_load_row(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ Vec16 lds16(uint32_t addr) {
    Vec16 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "r"(addr));
    return v;
}

template <typename T, typename I, int VPL, int RED, bool GATHER>
__global__ void __launch_bounds__(512, 1)
csr_tma_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const float* __restrict__ val,
               const T* __restrict__ x, T* __restrict__ out, int64_t n_rows, int n_vec, bool is_mean,
               bool inf_to_zero, LongRowPlan plan, const float* __restrict__ bias,
               unsigned long long* __restrict__ counter) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int n_warps = blockDim.x >> 5;
    const uint32_t row_bytes = static_cast<uint32_t>(n_vec) * 16u;
    const uint32_t ring = smem_u32(smem_raw) + static_cast<uint32_t>(warp) * kTmaSlots * row_bytes;
    const uint32_t bars = smem_u32(smem_raw) + static_cast<uint32_t>(n_warps) * kTmaSlots * row_bytes +
                          static_cast<uint32_t>(warp) * kTmaSlots * 8u;
    mbar_init(bars + lane * 8u, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    uint32_t phases = 0;                        // bit k: parity to wait for on slot k (warp-uniform)

    const char* xb = reinterpret_cast<const char*>(x);
    const char* xb2 = plan.x2 ? reinterpret_cast<const char*>(plan.x2) - static_cast<size_t>(plan.split) * row_bytes : xb;
    const int64_t split = plan.x2 ? plan.split : INT64_MAX;
    const int64_t n_blocks = (n_rows + kTmaUnitRows - 1) / kTmaUnitRows;
    const int64_t n_units = plan.n_chunks + n_blocks;
    bool vvalid[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) vvalid[k] = (lane + k * 32) < n_vec;

    float acc[VPL][EPV];
    auto reset_acc = [&]() {
#pragma unroll
        for (int k = 0; k < VPL; ++k)
#pragma unroll
            for (int i = 0; i < EPV; ++i) acc[k][i] = red_identity<RED>();
    };
    auto flush_row = [&](int64_t row, int64_t deg) {
        char* ob = reinterpret_cast<char*>(out) + static_cast<size_t>(row) * row_bytes;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (!vvalid[k]) continue;
            float f[EPV];
#pragma unroll
            for (int i = 0; i < EPV; ++i) f[i] = finalize<RED>(acc[k][i], deg, is_mean, inf_to_zero);
            if (bias) {
                const float* bp = bias + static_cast<size_t>(lane + k * 32) * EPV;
#pragma unroll
                for (int i = 0; i < EPV; ++i) f[i] = __fadd_rn(f[i], __ldg(bp + i));
            }
            stg_stream16(ob + static_cast<size_t>(lane + k * 32) * 16, ElemTraits<T>::pack(f));
        }
    };
    auto flush_partial = [&](int64_t chunk_item) {
        float* pbase = plan.partials + static_cast<size_t>(chunk_item) * n_vec * EPV;
#pragma unroll
        for (int k = 0; k < VPL; ++k)
            if (vvalid[k]) store_partial<EPV>(pbase + static_cast<size_t>(lane + k * 32) * EPV, acc[k]);
    };

    // Streams the edge range [e_begin, e_end).  Row bookkeeping: rows [row_lo, row_hi) of the unit
    // (unit-relative indices into the per-lane my_b / my_e registers); with is_chunk the whole range
    // belongs to one partial.
    auto stream = [&](int64_t e_begin, int64_t e_end, bool is_chunk, int64_t chunk_item, int64_t r0, int row_lo,
                      int row_hi, int64_t my_b, int64_t my_e) {
        int row = row_lo;
        int64_t row_end = is_chunk ? e_end : __shfl_sync(0xffffffffu, my_e, row & 31);
        reset_acc();
        // prologue: column indices / weights of the first batch, arm all of its slots
        int64_t c_next = 0;
        float w_next = 1.0f;
        if (e_begin + lane < e_end) {
            c_next = GATHER ? static_cast<int64_t>(ldg_idx(col + e_begin + lane)) : (e_begin + lane);
            if (val) w_next = __ldg(val + e_begin + lane);
            mbar_expect_tx(bars + lane * 8u, row_bytes);
            tma_load_row(ring + lane * row_bytes, (c_next < split ? xb : xb2) + static_cast<size_t>(c_next) * row_bytes, row_bytes, bars + lane * 8u);
        }
        for (int64_t e0 = e_begin; e0 < e_end; e0 += kTmaSlots) {
            const int n = static_cast<int>(e_end - e0 < kTmaSlots ? e_end - e0 : kTmaSlots);
            const float w_cur = w_next;
            // prefetch the next batch's indices while this one is in flight
            const int64_t e1 = e0 + kTmaSlots;
            const bool have_next = e1 + lane < e_end;
            if (have_next) {
                c_next = GATHER ? static_cast<int64_t>(ldg_idx(col + e1 + lane)) : (e1 + lane);
                w_next = val ? __ldg(val + e1 + lane) : 1.0f;
            }
#pragma unroll 1
            for (int q0 = 0; q0 < n; q0 += kTmaQuarter) {
                const int q1 = q0 + kTmaQuarter < n ? q0 + kTmaQuarter : n;
                for (int k = q0; k < q1; ++k) {
                    const int64_t e = e0 + k;
                    while (e >= row_end) {            // crossed a rowptr boundary: flush (also empty rows)
                        const int64_t rb = __shfl_sync(0xffffffffu, my_b, row & 31);
                        flush_row(r0 + row, row_end - rb);
                        reset_acc();
                        ++row;
                        row_end = __shfl_sync(0xffffffffu, my_e, row & 31);
                    }
                    mbar_wait(bars + k * 8u, (phases >> k) & 1u);
                    phases ^= (1u << k);
                    const float w = __shfl_sync(0xffffffffu, w_cur, k);
                    const uint32_t slot = ring + static_cast<uint32_t>(k) * row_bytes + static_cast<uint32_t>(lane) * 16u;
#pragma unroll
                    for (int v = 0; v < VPL; ++v) {
                        if (vvalid[v]) {
                            float f[EPV];
                            ElemTraits<T>::unpack(lds16(slot + static_cast<uint32_t>(v) * 512u), f);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) {
                                const float m = val ? __fmul_rn(w, f[i]) : f[i];
                                acc[v][i] = red_combine<RED>(acc[v][i], m);
                            }
                        }
                    }
                }
                // re-arm this quarter with the next batch's rows
                if (e1 < e_end) {
                    fence_proxy_async_smem();       // generic-proxy reads of the slots before the async overwrite
                    __syncwarp();
                    if (lane >= q0 && lane < q1 && have_next) {
                        mbar_expect_tx(bars + lane * 8u, row_bytes);
                        tma_load_row(ring + lane * row_bytes, (c_next < split ? xb : xb2) + static_cast<size_t>(c_next) * row_bytes, row_bytes,
                                     bars + lane * 8u);
                    }
                }
            }
        }
        if (is_chunk) {
            flush_partial(chunk_item);
        } else {
            while (row < row_hi) {                    // last non-empty row and trailing empty rows
                const int64_t rb = __shfl_sync(0xffffffffu, my_b, row & 31);
                const int64_t re = __shfl_sync(0xffffffffu, my_e, row & 31);
                flush_row(r0 + row, re - rb);
                reset_acc();
                ++row;
            }
        }
    };

    while (true) {
        unsigned long long u = 0;
        if (lane == 0) u = atomicAdd(counter, 1ull);
        const int64_t unit = static_cast<int64_t>(__shfl_sync(0xffffffffu, u, 0));
        if (unit >= n_units) break;
        if (unit < plan.n_chunks) {
            int64_t row, begin, end;
            bool is_chunk;
            decode_item(unit, rowptr, n_rows, plan, row, begin, end, is_chunk);
            stream(begin, end, true, unit, 0, 0, 0, 0, 0);
            continue;
        }
        const int64_t r0 = (unit - plan.n_chunks) * kTmaUnitRows;
        const int nrows = static_cast<int>(n_rows - r0 < kTmaUnitRows ? n_rows - r0 : kTmaUnitRows);
        int64_t my_b = 0, my_e = 0;
        if (lane < nrows) {
            my_b = static_cast<int64_t>(ldg_idx(rowptr + r0 + lane));
            my_e = static_cast<int64_t>(ldg_idx(rowptr + r0 + lane + 1));
        }
        const unsigned long_mask =
            plan.n_long > 0 ? __ballot_sync(0xffffffffu, lane < nrows && (my_e - my_b) > plan.chunk) : 0u;
        int cur = 0;
        while (cur < nrows) {
            const unsigned m = long_mask & (0xffffffffu << cur);
            const int nl = m ? (__ffs(m) - 1) : nrows;          // next hub row handled by the chunk units
            if (nl > cur) {
                const int64_t eb = __shfl_sync(0xffffffffu, my_b, cur);
                const int64_t ee = __shfl_sync(0xffffffffu, my_e, nl - 1);
                stream(eb, ee, false, 0, r0, cur, nl, my_b, my_e);
            }
            cur = nl + 1;
        }
    }
}

// device-resident work counters: one slot per launch (round robin), zeroed on the launch's stream
unsigned long long* tma_counter_slot(cudaStream_t stream);

template <typename T, typename I, int RED, bool GATHER>
int csr_tma_launch(const I* rowptr, const I* col, const float* val, const T* x, T* out, int64_t n_rows,
                   int64_t feat, bool is_mean, bool inf_to_zero, LongRowPlan plan, const float* bias,
                   cudaStream_t stream) {
    const int n_vec = static_cast<int>(static_cast<size_t>(feat) * sizeof(T) / 16);
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const size_t per_warp = kTmaSlots * row_bytes + kTmaSlots * 8;
    int warps = static_cast<int>((200 * 1024) / per_warp);
    if (warps > 16) warps = 16;
    if (warps < 1) return B200MP_ERR_UNSUPPORTED;
    const size_t smem = static_cast<size_t>(warps) * per_warp;
    unsigned long long* counter = tma_counter_slot(stream);
    if (!counter) return B200MP_ERR_CUDA;
    const int grid = num_sms();
#define B200MP_TMA(V_)                                                                                         \
    do {                                                                                                       \
        auto kfn = csr_tma_kernel<T, I, V_, RED, GATHER>;                                                      \
        B200MP_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem))); \
        kfn<<<grid, warps * 32, smem, stream>>>(rowptr, col, val, x, out, n_rows, n_vec, is_mean, inf_to_zero, plan,  \
                                                bias, counter);                                                \
    } while (0)
    if (n_vec <= 32) B200MP_TMA(1);
    else if (n_vec <= 64) B200MP_TMA(2);
    else B200MP_TMA(4);
#undef B200MP_TMA
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        csr_combine_kernel<T, I, RED><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
            rowptr, out, feat, is_mean, inf_to_zero, plan, bias);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

}  // namespace b200mp
