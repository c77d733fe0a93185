// gemm_tf32x3.cu -- fp32-accurate dense transform on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// The only GEMM-shaped work on the path is the layer's dense transform (SURVEY.md a14):
//     y  = x  W^T      [M,K] x [N,K]^T        (forward,       nn/dense/linear.py:121-127)
//     gx = g  W        [M,N] x [N,K]          (grad wrt input)
//     gW = g^T x       [N,M] x [M,K]          (grad wrt weight, reduction over the M = #nodes rows)
// The reference runs them as strict-fp32 cuBLAS SIMT kernels (allow_tf32=False).  A single-pass TF32
// GEMM would be much faster but only ~1e-3 accurate, so this kernel uses an error-compensated
// split:  a = a_hi + a_lo  (a_hi = rn_tf32(a), a_lo = a - a_hi exactly, |a_lo| <= 2^-11 |a|), and
//     a*b ~= [bf16(a_lo)*bf16(b_hi) + bf16(a_hi)*bf16(b_lo)] + a_hi*b_hi      (dropped term a_lo*b_lo ~ 2^-22 |a b|)
// accumulated in fp32 registers.  The two correction products are 2^-11 of the result, so BF16's 8 significant bits
// suffice for them (per term at most 2^-17 + 2^-22 of |a b|), and both fit in ONE wgmma k16 BF16 instruction: logical k
// becomes the bf16 pair (2k, 2k+1) holding (a_lo, a_hi) in A and (b_hi, b_lo) in B.  A k-step of 8 thus costs one BF16
// and one TF32 MMA of equal issue cost instead of three TF32 ones -- fp32-class accuracy at half the TF32 tensor rate.
// (The "tf32x3" names of the entry points date from the three-product form.)
//
// Structure (one persistent CTA per SM, 384 threads = three warpgroups, 256 x BN output tiles, BK = 32):
//   warpgroup 0, warp 0   TMA producer: one thread streams the raw fp32 A and B tiles into a ring of shared-memory
//                         stages (cp.async.bulk.tensor.2d, mbarrier complete_tx)
//   warpgroup 0, warps 1-3  B preparation, only when B is MN-major or arrives unsplit: split (and transpose) the
//                         stage's B tile into a 2-slot ring of (hi, correction) K-major 128B-swizzled buffers, one
//                         k-block ahead of the tensor cores.  The correction tile's 32-bit words are
//                         pack(bf16(b_hi), bf16(b_lo)) at the place of the fp32 element.  A pre-split K-major B
//                         (W_hi, W_lo of the forward) is packed once per call into a global correction matrix
//                         (pack_corr_kernel); TMA then writes hi and correction tiles in the wgmma layout, and the
//                         descriptors point at the stage itself.
//   warpgroups 1-2        consumers, 128 output rows each, as two m64 halves that share the stage's B tile.  Per
//                         k-block each issues 4 k-steps x 2 halves x (one wgmma.m64nBNk16.f32.bf16.bf16 correction,
//                         then one wgmma.m64nBNk8.f32.tf32.tf32 hi*hi) as one group (A from registers, B from shared
//                         memory), then wgmma.wait_group 0, releases the stage (and split slot), stores the tile if it
//                         was its last k-block, and loads and splits the next k-block's A fragments.  The two run
//                         independently on the same stages, so one's group keeps the tensor cores busy while the other
//                         drains, loads or stores.  (Keeping a group in flight across k-blocks with wait_group 1 made
//                         ptxas serialize every wgmma: C7518.)
//                         The epilogue adds the bias, applies ReLU and stores the fragments with masked rows.
// Operands may be K-major (row-major [rows, K]) or MN-major (row-major [K, rows]), so all three products
// read x, g and W exactly as they lie in HBM (no transposes in global memory).
#include <cuda.h>

#include <mutex>

#include "common.cuh"

namespace b200mp {

constexpr int kBM = 256;             // output rows per CTA tile (two warpgroups x two m64 halves)
constexpr int kBK = 32;              // fp32 elements of K per stage = one 128-byte swizzle row
constexpr int kMaxStages = 4;
constexpr int kSplitSlots = 2;       // ring of split B buffers written by the B-preparation warps
constexpr int kPrepWarps = 3;        // warps 1-3 of warpgroup 0
constexpr int kGemmThreads = 384;
constexpr int kSmemLimit = 227 * 1024;
constexpr int kMaxSegments = 120;    // grouped form: the tile -> segment table lives in static shared memory

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t s2u(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void bar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
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
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ float rn_tf32(float a) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(a));
    return __uint_as_float(r);
}
// bf16 pair (lower half, upper half) = (rn_bf16(lower), rn_bf16(upper)): positions 2k and 2k+1 of a bf16 operand
__device__ __forceinline__ uint32_t pack_bf16x2(float lower, float upper) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(upper), "f"(lower));
    return r;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Stall trace, compiled in only with -DB200MP_GEMM_TRACE (benchmarks/gemm_stalls.py builds such a library on the side):
// clock64 totals per role, summed over CTAs into g_gemm_trace by one thread per consumer warpgroup / producer thread /
// preparation warp.  The normal build keeps an empty GemmTrace and untimed calls.
enum TraceSlot {
    kTrFullWait,      // consumers: waiting on bar_full (A, and B when read from the stage) or bar_sfull (prepared B)
    kTrMmaWait,       // consumers: wgmma.wait_group
    kTrEpilogue,      // consumers: store_tile
    kTrConsumer,      // consumers: whole loop
    kTrEmptyWait,     // TMA producer: waiting on bar_empty
    kTrProducer,      // TMA producer: whole loop
    kTrPrepFullWait,  // B preparation: waiting on bar_full
    kTrPrepSlotWait,  // B preparation: waiting on bar_sempty
    kTrPrep,          // B preparation: whole loop
    kTrSlots
};
#ifdef B200MP_GEMM_TRACE
__device__ unsigned long long g_gemm_trace[kTrSlots];
struct GemmTrace {
    long long t[kTrSlots] = {};
    __device__ void flush(bool leader) const {
        if (leader)
            for (int i = 0; i < kTrSlots; ++i) atomicAdd(&g_gemm_trace[i], static_cast<unsigned long long>(t[i]));
    }
};
template <int SLOT, class F>
__device__ __forceinline__ void traced(GemmTrace& tr, F&& f) {
    const long long t0 = clock64();
    f();
    tr.t[SLOT] += clock64() - t0;
}
#else
struct GemmTrace {
    __device__ void flush(bool) const {}
};
template <int SLOT, class F>
__device__ __forceinline__ void traced(GemmTrace&, F&& f) {
    f();
}
#endif

// A fragments of one k-block, split: [k-step][register].  Register i of the m64k8 tf32 fragment holds (row r or r+8,
// k = t or t+4); register i of the m64k16 bf16 fragment holds the same row at bf16 positions 2k, 2k+1 -- so corr[j][i]
// = pack(bf16(a_lo), bf16(a_hi)) of the thread's own element i, no shuffles.  Fenced like the accumulators, so that
// their definitions stay ahead of wgmma.fence and ptxas has no reason to inject warpgroup.arrive inside the MMA window.
struct AFrag {
    uint32_t hi[4][4], corr[4][4];
};
__device__ __forceinline__ void fence_frag(AFrag& f) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(f.hi[j][i]), "+r"(f.corr[j][i])::"memory");
}

// d[64 x N] (+)= a[64 x 8] (registers, tf32) . b[8 x N] (shared memory, K-major, tf32)
__device__ __forceinline__ void wgmma_m64n64k8_tf32_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k8_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
// d[64 x N] (+)= a[64 x 16] (registers, bf16) . b[16 x N] (shared memory, K-major, bf16; trans-b = 0)
__device__ __forceinline__ void wgmma_m64n64k16_bf16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k16_bf16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d)
        : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    if constexpr (BN == 64) wgmma_m64n64k8_tf32_rs(d, a, bdesc, scale_d);
    else wgmma_m64n128k8_tf32_rs(d, a, bdesc, scale_d);
}
template <int BN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    if constexpr (BN == 64) wgmma_m64n64k16_bf16_rs(d, a, bdesc, scale_d);
    else wgmma_m64n128k16_bf16_rs(d, a, bdesc, scale_d);
}

// Shared-memory matrix descriptor of a K-major 128B-swizzled operand (rows of 128 B = 32 tf32 along K,
// 8-row atoms of 1024 B, as TMA CU_TENSOR_MAP_SWIZZLE_128B writes them): start>>4 [0,14), LBO>>4 [16,30)
// (unused for swizzled K-major), SBO>>4 [32,46) = 1024 B between 8-row groups, swizzle mode [62,64) = 1 (128B).
// The k-step j of a 32-wide block starts 32 B further along the swizzle row.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t addr) {
    return static_cast<uint64_t>((addr & 0x3ffffu) >> 4) | (1ull << 16) | (static_cast<uint64_t>(1024u >> 4) << 32) | (1ull << 62);
}
// byte offset of element (row, k) in a [rows x 32] fp32 tile stored K-major with the 128-byte swizzle
__device__ __forceinline__ uint32_t sw128_offset(int row, int k) {
    return static_cast<uint32_t>(row * 128 + ((((k >> 2) ^ (row & 7))) << 4) + ((k & 3) << 2));
}

struct GemmArgs {
    float* c;             // output [M, ldc] (or split-K partials [splits, M, ldc]); n-tiles [0, n_tiles_c1)
    float* c2;            // second output [M, ldc2]: n-tiles [n_tiles_c1, n_tiles_n) (pair form), else unused
    const float* bias;    // epilogue: + bias[n] over the concatenated output columns (nullable)
    int64_t m;            // rows of the output tile space (A's MN extent)
    int64_t ldc, ldc2;
    int n_tiles_m, n_tiles_n, n_tiles_c1;
    int k_blocks;         // total 32-wide k-blocks
    int k_blocks_per_split;
    int n_splits;
    int k_blocks_a1;      // k-blocks [0, k_blocks_a1) stream from tmap_a, the rest from tmap_a2 (A = [a1 | a2] along K):
                          // two products accumulate into ONE accumulator (SAGE: agg W_l^T + x W_r^T)
    int relu;             // epilogue: max(., 0)
    // ---- grouped (segment_matmul) form ----
    const int64_t* seg_ptr;   // [n_seg + 1] row offsets of the segments of A / C (device memory: no host read of the sizes)
    int n_seg;                // segment r multiplies with B block r
    int b_seg_rows;           // rows of the stacked B matrix per segment
};

struct Tile {
    int64_t m0;           // first output row
    int n0, seg, rows, split;
};
// w -> tile; GROUPED: tiles never straddle a segment (the last tile of a segment is partial)
template <bool GROUPED>
__device__ __forceinline__ bool decode_tile(int w, const GemmArgs& args, const int* tile_prefix, Tile& t) {
    const int tiles_per_split = (GROUPED ? tile_prefix[args.n_seg] : args.n_tiles_m) * args.n_tiles_n;
    t.split = w / tiles_per_split;
    const int r0 = w - t.split * tiles_per_split;
    const int mt = r0 / args.n_tiles_n;                  // n fastest: the column tiles of a row block are adjacent
    t.n0 = r0 % args.n_tiles_n;
    if (!GROUPED) {
        t.m0 = static_cast<int64_t>(mt) * kBM;
        t.seg = 0;
        t.rows = static_cast<int>(args.m - t.m0 < kBM ? args.m - t.m0 : kBM);
        return true;
    }
    int r = 0;
    while (r < args.n_seg && tile_prefix[r + 1] <= mt) ++r;          // few segments: a linear scan of shared memory
    if (r >= args.n_seg) return false;
    const int64_t s1 = args.seg_ptr[r + 1];
    t.m0 = args.seg_ptr[r] + static_cast<int64_t>(mt - tile_prefix[r]) * kBM;
    t.seg = r;
    t.rows = static_cast<int>(s1 - t.m0 < kBM ? s1 - t.m0 : kBM);
    return true;
}

// Shared-memory plan of one instantiation: a ring of raw stages (A tile, then B: raw, or hi and correction when
// pre-split K-major, or hi and lo when pre-split MN-major) and, when B needs preparing, kSplitSlots (hi, correction)
// buffers.  As many stages as fit, up to kMaxStages.
template <int BN, bool B_MN, bool B_PRE>
struct GemmPlan {
    static constexpr bool kDirectB = B_PRE && !B_MN;               // wgmma reads B straight from the stage
    static constexpr uint32_t kABytes = kBM * kBK * 4;             // 32 KB
    static constexpr uint32_t kBBytes = BN * kBK * 4;
    static constexpr uint32_t kStageBytes = kABytes + (B_PRE ? 2 : 1) * kBBytes;
    static constexpr uint32_t kSplitBytes = kDirectB ? 0 : kSplitSlots * 2 * kBBytes;
    static constexpr uint32_t kFixed = kSplitBytes + 8 * 2 * (kMaxStages + kSplitSlots) + 1024;
    static constexpr int kFit = static_cast<int>((kSmemLimit - kFixed) / kStageBytes);
    static constexpr int kStages = kFit < kMaxStages ? kFit : kMaxStages;
    static constexpr size_t kSmem = kStages * kStageBytes + kFixed;
    static_assert(kStages >= 2 && kSmem <= kSmemLimit, "one CTA per SM must fit the 227 KB opt-in shared memory of sm_90");
};

// A_MN / B_MN: operand is MN-major (stored row-major as [K, MN]); B_PRE: B arrives pre-split (tmap_b_hi, and tmap_b_lo
// = the packed correction when K-major, lo when MN-major), else tmap_b_hi is the raw matrix and the B-preparation warps
// split it.  An MN-major A arrives as
// up to eight [32 k][32 m] boxes (one per 32 rows of the tile) with the 128B swizzle, so the column-wise fragment loads do not collide in one bank.
template <int BN, bool A_MN, bool B_MN, bool B_PRE, bool GROUPED>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2,
                   const __grid_constant__ CUtensorMap tmap_b_hi, const __grid_constant__ CUtensorMap tmap_b_lo, GemmArgs args) {
    using Plan = GemmPlan<BN, B_MN, B_PRE>;
    constexpr bool kDirectB = Plan::kDirectB;
    constexpr int kStages = Plan::kStages;
    constexpr uint32_t kABytes = Plan::kABytes, kBBytes = Plan::kBBytes, kStageBytes = Plan::kStageBytes;
    constexpr int kAcc = BN / 2;                                // fp32 accumulators per thread (m64 x BN per warpgroup)

    extern __shared__ __align__(1024) unsigned char gemm_smem[];
    const uint32_t smem_base = (s2u(gemm_smem) + 1023u) & ~1023u;
    unsigned char* smem_gen = gemm_smem + (smem_base - s2u(gemm_smem));
    const uint32_t split_base = smem_base + kStages * kStageBytes;   // prepared B slots (K-major, 128B swizzle): hi, corr
    const uint32_t bars = split_base + Plan::kSplitBytes;
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (kStages + s); };
    auto bar_sfull = [&](int s) { return bars + 8u * (2 * kStages + s); };
    auto bar_sempty = [&](int s) { return bars + 8u * (2 * kStages + kSplitSlots + s); };

    __shared__ int tile_prefix[GROUPED ? kMaxSegments + 2 : 1];
    if (GROUPED && threadIdx.x == 32) {                          // tiles of kBM rows per segment, exclusive prefix
        int acc = 0;
        for (int r = 0; r < args.n_seg; ++r) {
            tile_prefix[r] = acc;
            acc += static_cast<int>((args.seg_ptr[r + 1] - args.seg_ptr[r] + kBM - 1) / kBM);
        }
        tile_prefix[args.n_seg] = acc;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            bar_init(bar_full(s), 1);
            bar_init(bar_empty(s), 2 + (kDirectB ? 0 : kPrepWarps));   // one arrive per consumer warpgroup, per prep warp
        }
        for (int s = 0; s < kSplitSlots; ++s) {
            bar_init(bar_sfull(s), kPrepWarps);
            bar_init(bar_sempty(s), 2);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int n_work = (GROUPED ? tile_prefix[args.n_seg] : args.n_tiles_m) * args.n_tiles_n * args.n_splits;
    const int wg = threadIdx.x >> 7;
    const int lane = threadIdx.x & 31;
    auto k_range = [&](const Tile& t, int& kb0, int& kb1) {
        kb0 = t.split * args.k_blocks_per_split;
        kb1 = min(kb0 + args.k_blocks_per_split, args.k_blocks);
    };

    // registers: the producer and B-preparation warpgroup gives up what the two MMA warpgroups need beyond the even
    // share of 168 (two m64 accumulators + one A fragment set per half); 128 x 40 + 256 x 232 <= 64 K
    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        const int warp = threadIdx.x >> 5;
        GemmTrace tr;
        if (threadIdx.x == 0) {
            // ===================== TMA producer =====================
            int stage = 0;
            uint32_t phase = 0;
            traced<kTrProducer>(tr, [&] {
            for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
                Tile t;
                decode_tile<GROUPED>(w, args, tile_prefix, t);
                const int m0 = static_cast<int>(t.m0), n0 = t.n0 * BN;
                const int b_row0 = GROUPED ? t.seg * args.b_seg_rows : 0;       // this segment's block of the stacked B
                int kb0, kb1;
                k_range(t, kb0, kb1);
                for (int kb = kb0; kb < kb1; ++kb) {
                    traced<kTrEmptyWait>(tr, [&] { bar_wait(bar_empty(stage), phase ^ 1u); });
                    const uint32_t sa = smem_base + stage * kStageBytes;
                    const uint32_t sb = sa + kABytes;
                    if (A_MN) {
                        // only the 32-row boxes that hold rows of the tile (a 128-row output fills half of one); the
                        // rows of the stage past them are never stored
                        const int boxes = (t.rows + 31) / 32;
                        bar_expect_tx(bar_full(stage), kStageBytes - (kBM / 32 - boxes) * 4096u);
                        for (int b = 0; b < boxes; ++b) tma_load_2d(sa + b * 4096u, &tmap_a, m0 + 32 * b, kb * kBK, bar_full(stage));
                    } else {
                        bar_expect_tx(bar_full(stage), kStageBytes);
                        if (kb < args.k_blocks_a1) tma_load_2d(sa, &tmap_a, kb * kBK, m0, bar_full(stage));
                        else tma_load_2d(sa, &tmap_a2, (kb - args.k_blocks_a1) * kBK, m0, bar_full(stage));
                    }
                    if (B_MN) {
                        tma_load_2d(sb, &tmap_b_hi, n0, b_row0 + kb * kBK, bar_full(stage));
                        if (B_PRE) tma_load_2d(sb + kBBytes, &tmap_b_lo, n0, b_row0 + kb * kBK, bar_full(stage));
                    } else {
                        tma_load_2d(sb, &tmap_b_hi, kb * kBK, b_row0 + n0, bar_full(stage));
                        if (B_PRE) tma_load_2d(sb + kBBytes, &tmap_b_lo, kb * kBK, b_row0 + n0, bar_full(stage));
                    }
                    if (++stage == kStages) { stage = 0; phase ^= 1u; }
                }
            }
            });
            tr.flush(true);
        } else if (!kDirectB && warp >= 1) {
            // ============ B preparation: stage -> prepared slot (hi, corr), K-major 128B swizzle ============
            // corr word of element (n, k) = pack(bf16(b_hi), bf16(b_lo)) at the byte offset of the fp32 element: a
            // K-major bf16 row of 128 B holds the 32 logical k as pairs, so hi and corr share swizzle and descriptors.
            const int pt = threadIdx.x - 32;                    // 0 .. 95
            int stage = 0, slot = 0;
            uint32_t phase = 0, sphase = 0;
            traced<kTrPrep>(tr, [&] {
            for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
                Tile t;
                decode_tile<GROUPED>(w, args, tile_prefix, t);
                int kb0, kb1;
                k_range(t, kb0, kb1);
                for (int kb = kb0; kb < kb1; ++kb) {
                    traced<kTrPrepFullWait>(tr, [&] { bar_wait(bar_full(stage), phase); });
                    traced<kTrPrepSlotWait>(tr, [&] { bar_wait(bar_sempty(slot), sphase ^ 1u); });
                    const unsigned char* sb = smem_gen + stage * kStageBytes + kABytes;
                    unsigned char* bh = smem_gen + (split_base - smem_base) + slot * 2 * kBBytes;
                    unsigned char* bc = bh + kBBytes;
                    if (!B_MN) {
                        // raw TMA tile already has the target layout: element-wise
                        for (uint32_t off = pt * 16u; off < kBBytes; off += kPrepWarps * 32 * 16u) {
                            const float4 v = *reinterpret_cast<const float4*>(sb + off);
                            const float4 h = make_float4(rn_tf32(v.x), rn_tf32(v.y), rn_tf32(v.z), rn_tf32(v.w));
                            const float4 l = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
                            *reinterpret_cast<float4*>(bh + off) = h;
                            *reinterpret_cast<uint4*>(bc + off) = make_uint4(pack_bf16x2(h.x, l.x), pack_bf16x2(h.y, l.y),
                                                                             pack_bf16x2(h.z, l.z), pack_bf16x2(h.w, l.w));
                        }
                    } else {
                        // raw tile is [32 k][BN n] (unswizzled): gather 4 consecutive k of one n, store one 16-byte chunk
                        const float* rb = reinterpret_cast<const float*>(sb);
                        for (int idx = pt; idx < BN * 8; idx += kPrepWarps * 32) {
                            const int n = idx % BN, kc = idx / BN;
                            float h[4];
                            uint32_t c[4];
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float v = rb[(4 * kc + i) * BN + n];
                                float l;
                                if (B_PRE) {
                                    h[i] = v;
                                    l = rb[BN * kBK + (4 * kc + i) * BN + n];
                                } else {
                                    h[i] = rn_tf32(v);
                                    l = v - h[i];
                                }
                                c[i] = pack_bf16x2(h[i], l);
                            }
                            const uint32_t off = sw128_offset(n, 4 * kc);
                            *reinterpret_cast<float4*>(bh + off) = make_float4(h[0], h[1], h[2], h[3]);
                            *reinterpret_cast<uint4*>(bc + off) = make_uint4(c[0], c[1], c[2], c[3]);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> wgmma (async proxy) reads
                    __syncwarp();
                    if (lane == 0) {
                        bar_arrive(bar_empty(stage));          // this warp has read the raw B of the stage
                        bar_arrive(bar_sfull(slot));
                    }
                    if (++stage == kStages) { stage = 0; phase ^= 1u; }
                    if (++slot == kSplitSlots) { slot = 0; sphase ^= 1u; }
                }
            }
            });
            tr.flush(lane == 0);
        }
        return;
    }

    // ===================== consumers: warpgroups 1 and 2 =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    // this warpgroup's 128 rows of the tile are two m64 halves; fragment rows of half hf: row_base + 64 hf, +8
    const int row_base = (wg - 1) * 128 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    const int kq = lane & 3;
    const bool signal = (threadIdx.x & 127) == 0;               // releases stages / slots for its warpgroup
    int w = blockIdx.x;
    if (w >= n_work) return;

    // (A) fragments of this warpgroup's two 64-row halves from a raw stage, split in registers
    auto load_a = [&](AFrag (&f)[2], int stage) {
        const unsigned char* sa = smem_gen + stage * kStageBytes;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
#pragma unroll
            for (int j = 0; j < kBK / 8; ++j) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = row_base + hf * 64 + (i & 1) * 8, k = j * 8 + kq + (i >> 1) * 4;
                    const float v = A_MN ? *reinterpret_cast<const float*>(sa + (r >> 5) * 4096 + sw128_offset(k, r & 31))
                                         : *reinterpret_cast<const float*>(sa + sw128_offset(r, k));
                    const float h = rn_tf32(v);
                    f[hf].hi[j][i] = __float_as_uint(h);
                    f[hf].corr[j][i] = pack_bf16x2(v - h, h);
                }
            }
    };

    Tile t;
    decode_tile<GROUPED>(w, args, tile_prefix, t);
    int kb0, kb1;
    k_range(t, kb0, kb1);
    int kb = kb0;
    int stage = 0, slot = 0;                                    // ring positions of k-block kb
    uint32_t phase = 0, sphase = 0;
    float acc[2][kAcc];
    AFrag f[2];
    GemmTrace tr;
#ifdef B200MP_GEMM_TRACE
    const long long tr_start = clock64();
#endif
    traced<kTrFullWait>(tr, [&] { bar_wait(bar_full(stage), phase); });
    load_a(f, stage);

    auto release = [&](int st, int sl) {
        if (signal) {
            bar_arrive(bar_empty(st));
            if (!kDirectB) bar_arrive(bar_sempty(sl));
        }
    };
    // epilogue: fragments -> global, rows masked
    auto store_tile = [&](const Tile& tt) {
        const int nt = tt.n0;
        const bool second = nt >= args.n_tiles_c1;
        float* out = second ? args.c2 : args.c;
        const int64_t ldc = second ? args.ldc2 : args.ldc;
        const int col0 = (second ? nt - args.n_tiles_c1 : nt) * BN;
        const float* bias = args.bias ? args.bias + nt * BN : nullptr;
        float* base = out + static_cast<int64_t>(tt.split) * args.m * ldc + tt.m0 * ldc + col0;   // the tile's (0, 0)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = row_base + hf * 64 + h * 8;
                const bool keep = r < tt.rows;
                float* dst = base + r * ldc;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = j * 8 + 2 * kq;
                    float v0 = acc[hf][4 * j + 2 * h], v1 = acc[hf][4 * j + 2 * h + 1];
                    if (bias) {
                        v0 += __ldg(bias + c);
                        v1 += __ldg(bias + c + 1);
                    }
                    if (args.relu) {
                        v0 = fmaxf(v0, 0.0f);
                        v1 = fmaxf(v1, 0.0f);
                    }
                    if (keep) *reinterpret_cast<float2*>(dst + c) = make_float2(v0, v1);
                }
            }
    };
    // One k-block: f holds its A fragments; on return f holds those of the next k-block (false: no more work).
    auto step = [&]() -> bool {
        uint32_t b_hi;
        if (kDirectB) {
            b_hi = smem_base + stage * kStageBytes + kABytes;
        } else {
            traced<kTrFullWait>(tr, [&] { bar_wait(bar_sfull(slot), sphase); });
            b_hi = split_base + slot * 2 * kBBytes;
        }
        const uint32_t b_corr = b_hi + kBBytes;
        // 4 k-steps x (bf16 correction pair, tf32 hi*hi) on each half, small terms first; the k16 bf16 step and the k8
        // tf32 step both advance 32 B along the swizzle row.  Per accumulator the order is that of one m64 tile.
        fence_frag(f[0]);
        fence_frag(f[1]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < kBK / 8; ++j) {
            const uint32_t scale = (kb > kb0 || j > 0) ? 1u : 0u;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                wgmma_bf16<BN>(acc[hf], f[hf].corr[j], smem_desc_sw128(b_corr + j * 32u), scale);
                wgmma_tf32<BN>(acc[hf], f[hf].hi[j], smem_desc_sw128(b_hi + j * 32u), 1u);
            }
        }
        wgmma_commit();
        const int cur_stage = stage, cur_slot = slot;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
        if (!kDirectB && ++slot == kSplitSlots) { slot = 0; sphase ^= 1u; }
        const bool tile_done = ++kb == kb1;
        bool more = true;
        if (tile_done) {
            w += gridDim.x;
            more = w < n_work;
        }
        traced<kTrMmaWait>(tr, [&] { wgmma_wait_all(); });
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        release(cur_stage, cur_slot);
        if (tile_done) {
            traced<kTrEpilogue>(tr, [&] { store_tile(t); });
            if (more) {
                decode_tile<GROUPED>(w, args, tile_prefix, t);
                k_range(t, kb0, kb1);
                kb = kb0;
            }
        }
        if (more) {                                             // next A fragments, possibly the next tile's
            fence_frag(f[0]);
            fence_frag(f[1]);
            traced<kTrFullWait>(tr, [&] { bar_wait(bar_full(stage), phase); });
            load_a(f, stage);
        }
        return more;
    };
    while (step()) {
    }
#ifdef B200MP_GEMM_TRACE
    tr.t[kTrConsumer] += clock64() - tr_start;
#endif
    tr.flush(signal);
}

// w -> (rn_tf32(w), w - rn_tf32(w)) for the (small) weight matrix
__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) {
        const float v = w[i], h = rn_tf32(v);
        hi[i] = h;
        lo[i] = v - h;
    }
}
// (hi, lo) -> pack(bf16(hi), bf16(lo)): the correction operand of a pre-split K-major B, element for element
__global__ void pack_corr_kernel(const float* __restrict__ hi, const float* __restrict__ lo, uint32_t* __restrict__ corr, int64_t n) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) corr[i] = pack_bf16x2(hi[i], lo[i]);
}
// w [rows, cols] -> (rn_tf32(w^T), w^T - rn_tf32(w^T)) [cols, rows], through a 32 x 32 shared-memory tile
__global__ void split_tf32_transposed_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo,
                                             int64_t rows, int64_t cols) {
    __shared__ float tile[32][33];
    const int64_t r0 = static_cast<int64_t>(blockIdx.y) * 32, c0 = static_cast<int64_t>(blockIdx.x) * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = w[r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int64_t c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) {
            const float v = tile[threadIdx.x][i], h = rn_tf32(v);
            hi[c * rows + r] = h;
            lo[c * rows + r] = v - h;
        }
    }
}
// out[i] = sum_s part[s][i], fixed order (deterministic split-K)
__global__ void splitk_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int64_t n, int splits) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) {
        float acc = 0.0f;
        for (int s = 0; s < splits; ++s) acc = __fadd_rn(acc, part[static_cast<int64_t>(s) * n + i]);
        out[i] = acc;
    }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// 2-D fp32 row-major [rows, cols] tensor, zero fill out of bounds.
//   K-major operand  (mn = false): box = [box_mn rows, 32 cols], 128B swizzle (the wgmma K-major layout);
//   MN-major operand (mn = true) : box = [32 k-rows, box_mn cols], unswizzled (transposed while it is split),
//                                  except box_mn = 32 (an MN-major A, loaded as 32-column boxes): 128B swizzle.
static int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, bool mn, int box_mn) {
    const CUtensorMapSwizzle swz = (mn && box_mn != 32) ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
    const int box_cols = mn ? box_mn : kBK;
    const int box_rows = mn ? kBK : box_mn;
    EncodeTiledFn fn = encode_fn();
    // cuTensorMapEncodeTiled is a DRIVER call: it needs a current context.  On a fresh thread (the
    // autograd engine's backward thread) no runtime call may have bound the primary context yet.
    cudaFree(nullptr);
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point not available");
        return B200MP_ERR_CUDA;
    }
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 4};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box_mn=%d", static_cast<int>(r),
                  static_cast<long long>(rows), static_cast<long long>(cols), static_cast<long long>(ld), box_mn);
        return B200MP_ERR_CUDA;
    }
    return B200MP_OK;
}

template <int BN, bool A_MN, bool B_MN, bool B_PRE, bool GROUPED = false>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& ta2, const CUtensorMap& tbh, const CUtensorMap& tbl,
                       const GemmArgs& args, int n_work, cudaStream_t stream) {
    constexpr size_t smem = GemmPlan<BN, B_MN, B_PRE>::kSmem;
    auto kfn = gemm_tf32x3_kernel<BN, A_MN, B_MN, B_PRE, GROUPED>;
    B200MP_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    const int grid = n_work < num_sms() ? n_work : num_sms();
    kfn<<<grid, kGemmThreads, smem, stream>>>(ta, ta2, tbh, tbl, args);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}
// BN = 64 only for a 64-wide output, else 128 (every supported width is then a multiple of it)
template <bool A_MN, bool B_MN, bool B_PRE>
static int launch_bn(int bn, const CUtensorMap& ta, const CUtensorMap& ta2, const CUtensorMap& tbh, const CUtensorMap& tbl,
                     const GemmArgs& args, cudaStream_t s) {
    const int n_work = args.n_tiles_m * args.n_tiles_n * args.n_splits;
    return bn == 64 ? launch_gemm<64, A_MN, B_MN, B_PRE>(ta, ta2, tbh, tbl, args, n_work, s)
                    : launch_gemm<128, A_MN, B_MN, B_PRE>(ta, ta2, tbh, tbl, args, n_work, s);
}

// Correction operand of a pre-split K-major B, packed once per call from (b_hi, b_lo) into stream-ordered scratch, so
// that TMA can stage it next to hi with no preparation pass in the kernel.  Freed in stream order when it goes out of
// scope, after the launch that reads it.  The scratch comes from a memory pool of the library's own per device that
// keeps what it has mapped (the default pool would hand memory back at every synchronisation and map it again on the
// next call, which stalls the stream for milliseconds).
static cudaMemPool_t corr_pool(int dev) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    std::lock_guard<std::mutex> lock(mu);
    if (dev < 0 || dev >= 64) return nullptr;
    if (!pools[dev]) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        cudaMemPool_t pool = nullptr;
        if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
        uint64_t keep = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        pools[dev] = pool;
    }
    return pools[dev];
}
struct CorrB {
    uint32_t* p = nullptr;
    cudaStream_t s = nullptr;
    ~CorrB() {
        if (p) cudaFreeAsync(p, s);
    }
};
static int pack_corr(const float* hi, const float* lo, int64_t n, cudaStream_t s, CorrB& out) {
    out.s = s;
    int dev = 0;
    B200MP_CUDA(cudaGetDevice(&dev));
    cudaMemPool_t pool = corr_pool(dev);
    if (!pool) {
        set_error("gemm: cannot create the correction-operand memory pool on device %d", dev);
        return B200MP_ERR_CUDA;
    }
    B200MP_CUDA(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&out.p), static_cast<size_t>(n) * 4, pool, s));
    pack_corr_kernel<<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, s>>>(hi, lo, out.p, n);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

static bool ok16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static bool width_ok(int64_t w) { return w == 64 || w == 128 || (w > 0 && w % 256 == 0); }
static int tile_n(int64_t w) { return w == 64 ? 64 : 128; }

// [c1 | c2][M, n1 + n2] = [a1 | a2][M, k1 + k2] . B (+ bias, relu), B K-major ([n_out, k_red]) or MN-major
// ([k_red, n_out]); b_lo == nullptr: b_hi is the unsplit matrix and the kernel splits the B tiles itself
static int run_pair(const float* a1, int64_t k1, const float* a2, int64_t k2, const float* b_hi, const float* b_lo, float* c1,
                    int64_t n1, float* c2, int64_t n2, const float* bias, int relu, int64_t m, bool b_mn, cudaStream_t s) {
    const int64_t k_red = k1 + k2, n_out = n1 + n2;
    const int64_t b_rows = b_mn ? k_red : n_out, b_cols = b_mn ? n_out : k_red;
    const int bn = (n1 == 64 && n2 == 0) ? 64 : 128;
    CUtensorMap ta, ta2, tbh, tbl;
    int rc;
    CorrB corr;
    const float* b_second = b_lo ? b_lo : b_hi;                 // K-major pre-split: the packed correction, else lo / raw
    if (b_lo && !b_mn) {
        if ((rc = pack_corr(b_hi, b_lo, b_rows * b_cols, s, corr))) return rc;
        b_second = reinterpret_cast<const float*>(corr.p);
    }
    if ((rc = make_map(&ta, a1, m, k1, k1, false, kBM))) return rc;
    if ((rc = make_map(&ta2, a2 ? a2 : a1, m, a2 ? k2 : k1, a2 ? k2 : k1, false, kBM))) return rc;
    if ((rc = make_map(&tbh, b_hi, b_rows, b_cols, b_cols, b_mn, bn))) return rc;
    if ((rc = make_map(&tbl, b_second, b_rows, b_cols, b_cols, b_mn, bn))) return rc;
    const int kb = static_cast<int>(k_red / kBK);
    GemmArgs args{};
    args.c = c1;
    args.c2 = c2;
    args.bias = bias;
    args.m = m;
    args.ldc = n1;
    args.ldc2 = n2;
    args.n_tiles_m = static_cast<int>(ceil_div(m, kBM));
    args.n_tiles_n = static_cast<int>(n_out / bn);
    args.n_tiles_c1 = static_cast<int>(n1 / bn);
    args.k_blocks = args.k_blocks_per_split = kb;
    args.n_splits = 1;
    args.k_blocks_a1 = static_cast<int>(k1 / kBK);
    args.relu = relu;
    if (b_lo) return b_mn ? launch_bn<false, true, true>(bn, ta, ta2, tbh, tbl, args, s) : launch_bn<false, false, true>(bn, ta, ta2, tbh, tbl, args, s);
    return b_mn ? launch_bn<false, true, false>(bn, ta, ta2, tbh, tbl, args, s) : launch_bn<false, false, false>(bn, ta, ta2, tbh, tbl, args, s);
}

// gw[N,K] = g[M,N]^T . x[M,K]: both operands MN-major as stored, split-K over the M rows
static int run_grad_weight(const float* g, const float* x, float* gw, int64_t m, int64_t n, int64_t k, void* workspace,
                           int64_t workspace_bytes, cudaStream_t s) {
    const int bn = tile_n(k);
    const int tiles = static_cast<int>(ceil_div(n, kBM) * (k / bn));
    const int64_t kblocks = ceil_div(m, kBK);
    if (kblocks > 0x7fffffffLL) return B200MP_ERR_UNSUPPORTED;
    int splits = num_sms() / tiles;
    if (splits < 1) splits = 1;
    if (splits > kblocks) splits = static_cast<int>(kblocks);
    const int kbps = static_cast<int>(ceil_div(kblocks, splits));
    splits = static_cast<int>(ceil_div(kblocks, kbps));            // every split non-empty
    if (static_cast<int64_t>(splits) * n * k * 4 > workspace_bytes) {
        set_error("linear_grad_weight_tf32x3: workspace too small");
        return B200MP_ERR_WORKSPACE;
    }
    CUtensorMap ta, tb;
    int rc;
    if ((rc = make_map(&ta, g, m, n, n, true, 32))) return rc;     // A[m' = n-index, k' = row]: stored [K' rows][M' cols]
    if ((rc = make_map(&tb, x, m, k, k, true, bn))) return rc;
    GemmArgs args{};
    args.c = static_cast<float*>(workspace);
    args.m = n;
    args.ldc = k;
    args.n_tiles_m = static_cast<int>(ceil_div(n, kBM));
    args.n_tiles_n = args.n_tiles_c1 = static_cast<int>(k / bn);
    args.k_blocks = static_cast<int>(kblocks);
    args.k_blocks_per_split = kbps;
    args.n_splits = splits;
    args.k_blocks_a1 = static_cast<int>(kblocks);
    if ((rc = launch_bn<true, true, false>(bn, ta, ta, tb, tb, args, s))) return rc;
    const int64_t total = n * k;
    splitk_reduce_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, s>>>(static_cast<const float*>(workspace), gw,
                                                                                      total, splits);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}
}  // namespace b200mp

using namespace b200mp;

#ifdef B200MP_GEMM_TRACE
// trace build only (not part of the C ABI): copy the kTrSlots clock64 totals to out, then zero them if reset
extern "C" int b200mp_gemm_trace_read(unsigned long long* out, int n, int reset) {
    B200MP_CHECK_ARG(out && n == kTrSlots);
    B200MP_CUDA(cudaDeviceSynchronize());
    B200MP_CUDA(cudaMemcpyFromSymbol(out, g_gemm_trace, sizeof(unsigned long long) * kTrSlots));
    if (reset) {
        void* p = nullptr;
        B200MP_CUDA(cudaGetSymbolAddress(&p, g_gemm_trace));
        B200MP_CUDA(cudaMemset(p, 0, sizeof(unsigned long long) * kTrSlots));
    }
    return B200MP_OK;
}
#endif

extern "C" int b200mp_split_tf32(const float* w, float* w_hi, float* w_lo, int64_t n, void* stream) {
    B200MP_CHECK_ARG(n >= 0);
    if (n == 0) return B200MP_OK;
    B200MP_CHECK_ARG(w && w_hi && w_lo);
    split_tf32_kernel<<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, static_cast<cudaStream_t>(stream)>>>(w, w_hi, w_lo, n);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_split_tf32_transposed(const float* w, float* wt_hi, float* wt_lo, int64_t rows, int64_t cols, void* stream) {
    B200MP_CHECK_ARG(rows >= 0 && cols >= 0);
    if (rows == 0 || cols == 0) return B200MP_OK;
    B200MP_CHECK_ARG(w && wt_hi && wt_lo && ceil_div(rows, 32) <= 65535);
    const dim3 grid(static_cast<unsigned>(ceil_div(cols, 32)), static_cast<unsigned>(ceil_div(rows, 32)));
    split_tf32_transposed_kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(w, wt_hi, wt_lo, rows, cols);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

// y[M,N] = x[M,K] . w[N,K]^T
extern "C" int b200mp_linear_tf32x3(const float* x, const float* w_hi, const float* w_lo, float* y, int64_t m, int64_t n,
                                    int64_t k, void* stream) {
    B200MP_CHECK_ARG(m >= 0 && n > 0 && k > 0);
    if (m == 0) return B200MP_OK;
    B200MP_CHECK_ARG(x && w_hi && y && ok16(x) && ok16(w_hi) && ok16(w_lo) && ok16(y));
    if (k % 32 != 0 || !width_ok(n) || m > 0x7fffffffLL) {
        set_error("linear_tf32x3: unsupported shape m=%lld n=%lld k=%lld", (long long)m, (long long)n, (long long)k);
        return B200MP_ERR_UNSUPPORTED;
    }
    return run_pair(x, k, nullptr, 0, w_hi, w_lo, y, n, nullptr, 0, nullptr, 0, m, false, static_cast<cudaStream_t>(stream));
}

// gx[M,K] = g[M,N] . w[N,K]   (B = w read MN-major exactly as stored: [K' = n rows][N' = k cols])
extern "C" int b200mp_linear_grad_input_tf32x3(const float* g, const float* w_hi, const float* w_lo, float* gx, int64_t m,
                                               int64_t n, int64_t k, void* stream) {
    B200MP_CHECK_ARG(m >= 0 && n > 0 && k > 0);
    if (m == 0) return B200MP_OK;
    B200MP_CHECK_ARG(g && w_hi && gx && ok16(g) && ok16(w_hi) && ok16(w_lo) && ok16(gx));
    if (n % 32 != 0 || !width_ok(k) || m > 0x7fffffffLL) {
        set_error("linear_grad_input_tf32x3: unsupported shape m=%lld n=%lld k=%lld", (long long)m, (long long)n, (long long)k);
        return B200MP_ERR_UNSUPPORTED;
    }
    return run_pair(g, n, nullptr, 0, w_hi, w_lo, gx, k, nullptr, 0, nullptr, 0, m, true, static_cast<cudaStream_t>(stream));
}

extern "C" int64_t b200mp_linear_grad_weight_workspace_bytes(int64_t m, int64_t n, int64_t k) {
    if (m < 0 || n <= 0 || k <= 0) return B200MP_ERR_INVALID_ARG;
    return static_cast<int64_t>(num_sms()) * n * k * 4 + 256;
}

extern "C" int b200mp_linear_grad_weight_tf32x3(const float* g, const float* x, float* gw, int64_t m, int64_t n, int64_t k,
                                                void* workspace, int64_t workspace_bytes, void* stream) {
    B200MP_CHECK_ARG(m >= 0 && n > 0 && k > 0);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (m == 0) {
        B200MP_CUDA(cudaMemsetAsync(gw, 0, sizeof(float) * n * k, s));
        return B200MP_OK;
    }
    B200MP_CHECK_ARG(g && x && gw && workspace && ok16(g) && ok16(x) && ok16(gw) && ok16(workspace));
    if (n % 128 != 0 || !width_ok(k)) {
        set_error("linear_grad_weight_tf32x3: unsupported shape m=%lld n=%lld k=%lld", (long long)m, (long long)n, (long long)k);
        return B200MP_ERR_UNSUPPORTED;
    }
    return run_grad_weight(g, x, gw, m, n, k, workspace, workspace_bytes, s);
}

extern "C" int b200mp_gemm_pair_tf32x3(const float* a1, int64_t k1, const float* a2, int64_t k2, const float* b_hi,
                                       const float* b_lo, int b_layout, const float* bias, int relu, float* c1, int64_t n1,
                                       float* c2, int64_t n2, int64_t m, void* stream) {
    B200MP_CHECK_ARG(m >= 0 && k1 > 0 && k2 >= 0 && n1 > 0 && n2 >= 0 && (b_layout == 0 || b_layout == 1));
    if (m == 0) return B200MP_OK;
    B200MP_CHECK_ARG(a1 && b_hi && c1 && ok16(a1) && ok16(a2) && ok16(b_hi) && ok16(b_lo) && ok16(c1) && ok16(c2));
    B200MP_CHECK_ARG((k2 == 0) == (a2 == nullptr) && (n2 == 0) == (c2 == nullptr));
    if (k1 % 32 != 0 || k2 % 32 != 0 || n1 % 128 != 0 || n2 % 128 != 0 || m > 0x7fffffffLL) {
        set_error("gemm_pair_tf32x3: unsupported shape m=%lld k=%lld+%lld n=%lld+%lld (k %% 32, n %% 128)", (long long)m,
                  (long long)k1, (long long)k2, (long long)n1, (long long)n2);
        return B200MP_ERR_UNSUPPORTED;
    }
    return run_pair(a1, k1, a2, k2, b_hi, b_lo, c1, n1, c2, n2, bias, relu, m, b_layout == 1, static_cast<cudaStream_t>(stream));
}

// out[ptr[r] : ptr[r+1]] = a[ptr[r] : ptr[r+1]] . B_r for every segment r in ONE persistent launch: work items are
// (segment, 256-row tile inside the segment, 128-column tile); the tile -> segment map is rebuilt in shared memory from
// the device-resident ptr, so the segment sizes never travel to the host.
extern "C" int b200mp_segment_matmul_tf32x3(const float* a, const int64_t* ptr, int64_t n_seg, const float* b_hi, const float* b_lo,
                                            int b_layout, float* c, int64_t m, int64_t k, int64_t n, void* stream) {
    B200MP_CHECK_ARG(m >= 0 && k > 0 && n > 0 && n_seg > 0 && (b_layout == 0 || b_layout == 1));
    if (m == 0) return B200MP_OK;
    B200MP_CHECK_ARG(a && ptr && b_hi && b_lo && c && ok16(a) && ok16(b_hi) && ok16(b_lo) && ok16(c));
    if (k % 32 != 0 || n % 128 != 0 || n_seg > kMaxSegments || m > 0x7fffffffLL) {
        set_error("segment_matmul_tf32x3: unsupported shape m=%lld k=%lld n=%lld segments=%lld (k %% 32, n %% 128, <= 120 segments)",
                  (long long)m, (long long)k, (long long)n, (long long)n_seg);
        return B200MP_ERR_UNSUPPORTED;
    }
    const bool b_mn = b_layout == 1;                       // 1: B_r = w[r] [K, N] row-major (out = a w[r]); 0: B_r = w[r] [N, K] (out = a w[r]^T)
    const int64_t b_rows = n_seg * (b_mn ? k : n), b_cols = b_mn ? n : k;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    CUtensorMap ta, tbh, tbl;
    int rc;
    CorrB corr;
    const float* b_second = b_lo;                               // layout 0 (K-major): the packed correction
    if (!b_mn) {
        if ((rc = pack_corr(b_hi, b_lo, b_rows * b_cols, s, corr))) return rc;
        b_second = reinterpret_cast<const float*>(corr.p);
    }
    if ((rc = make_map(&ta, a, m, k, k, false, kBM))) return rc;
    if ((rc = make_map(&tbh, b_hi, b_rows, b_cols, b_cols, b_mn, 128))) return rc;
    if ((rc = make_map(&tbl, b_second, b_rows, b_cols, b_cols, b_mn, 128))) return rc;
    const int kb = static_cast<int>(k / kBK);
    GemmArgs args{};
    args.c = c;
    args.m = m;
    args.ldc = n;
    args.n_tiles_n = args.n_tiles_c1 = static_cast<int>(n / 128);
    args.k_blocks = args.k_blocks_per_split = args.k_blocks_a1 = kb;
    args.n_splits = 1;
    args.seg_ptr = ptr;
    args.n_seg = static_cast<int>(n_seg);
    args.b_seg_rows = static_cast<int>(b_mn ? k : n);
    // upper bound of the work list: every segment adds at most one partial tile
    const int n_work = static_cast<int>((ceil_div(m, kBM) + n_seg) * args.n_tiles_n);
    return b_mn ? launch_gemm<128, false, true, true, true>(ta, ta, tbh, tbl, args, n_work, s)
                : launch_gemm<128, false, false, true, true>(ta, ta, tbh, tbl, args, n_work, s);
}
