// common.cuh -- shared helpers for the b200mp kernels (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <type_traits>

#include "../../include/b200mp.h"

namespace b200mp {

void set_error(const char* fmt, ...);

#define B200MP_CHECK_ARG(cond)                                                          \
    do {                                                                                \
        if (!(cond)) {                                                                  \
            ::b200mp::set_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, #cond); \
            return B200MP_ERR_INVALID_ARG;                                              \
        }                                                                               \
    } while (0)

#define B200MP_CUDA(call)                                                                       \
    do {                                                                                        \
        cudaError_t e__ = (call);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            ::b200mp::set_error("%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            (void)cudaGetLastError(); /* do not leave the error pending for the caller's next CUDA call */ \
            return B200MP_ERR_CUDA;                                                             \
        }                                                                                       \
    } while (0)

#define B200MP_LAUNCH_CHECK() B200MP_CUDA(cudaGetLastError())

constexpr int kSMs = 132;  // H100 SXM (fallback only: the device attribute is queried first)

inline int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = kSMs;
    }
    return n;
}

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Calls fn(T{}, I{}) for the supported (value dtype, index dtype) pairs: fp32 or bf16 values, int32 or int64 indices.
template <typename F>
int dispatch_val_idx(int val_dtype, int idx_dtype, const char* what, F&& fn) {
    if (val_dtype == B200MP_F32 && idx_dtype == B200MP_I32) return fn(float{}, int32_t{});
    if (val_dtype == B200MP_F32 && idx_dtype == B200MP_I64) return fn(float{}, int64_t{});
    if (val_dtype == B200MP_BF16 && idx_dtype == B200MP_I32) return fn(__nv_bfloat16{}, int32_t{});
    if (val_dtype == B200MP_BF16 && idx_dtype == B200MP_I64) return fn(__nv_bfloat16{}, int64_t{});
    set_error("%s: unsupported dtype combination val=%d idx=%d", what, val_dtype, idx_dtype);
    return B200MP_ERR_UNSUPPORTED;
}

// Lane-group shape of a row of n_vec 16-byte vectors: G = the smallest power of two >= n_vec, capped at a warp, and
// VPL = vectors per lane, up to MAX_VPL (wider rows are walked by the kernel's own vbase loop).  Calls
// launch(integral_constant<int, G>, integral_constant<int, VPL>).
template <int MAX_VPL, typename F>
void lane_group_shape(int n_vec, F&& launch) {
    static_assert(MAX_VPL == 1 || MAX_VPL == 2 || MAX_VPL == 4, "VPL is 1, 2 or 4");
    using std::integral_constant;
    if (n_vec <= 1) launch(integral_constant<int, 1>{}, integral_constant<int, 1>{});
    else if (n_vec <= 2) launch(integral_constant<int, 2>{}, integral_constant<int, 1>{});
    else if (n_vec <= 4) launch(integral_constant<int, 4>{}, integral_constant<int, 1>{});
    else if (n_vec <= 8) launch(integral_constant<int, 8>{}, integral_constant<int, 1>{});
    else if (n_vec <= 16) launch(integral_constant<int, 16>{}, integral_constant<int, 1>{});
    else if constexpr (MAX_VPL == 1) launch(integral_constant<int, 32>{}, integral_constant<int, 1>{});
    else if (n_vec <= 32) launch(integral_constant<int, 32>{}, integral_constant<int, 1>{});
    else if constexpr (MAX_VPL == 2) launch(integral_constant<int, 32>{}, integral_constant<int, 2>{});
    else if (n_vec <= 64) launch(integral_constant<int, 32>{}, integral_constant<int, 2>{});
    else launch(integral_constant<int, 32>{}, integral_constant<int, 4>{});
}

// log2 of lane_group_shape's G, for kernels that take the group width at run time.
inline int lane_group_log2(int n_vec) {
    int lg = 0;
    lane_group_shape<1>(n_vec, [&](auto G, auto) { lg = __builtin_ctz(decltype(G)::value); });
    return lg;
}

// Independent edges in flight per lane for VPL vectors per lane: about 4 sixteen-byte row loads.
template <int VPL>
constexpr int unroll_for_vpl() { return VPL >= 4 ? 1 : 4 / VPL; }

// ---------------------------------------------------------------- 128-bit vector helpers
struct __align__(16) Vec16 {
    uint32_t w[4];
};

// Read-only 128-bit load of gathered feature rows (may be re-read by other rows: keep in L2,
// do not pollute L1 -- every row is touched once per warp).
__device__ __forceinline__ Vec16 ldg_row16(const void* p) {
    Vec16 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p));
    return v;
}
// Streaming 128-bit load (data read exactly once: evict first).
__device__ __forceinline__ Vec16 ldg_stream16(const void* p) {
    Vec16 v;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p));
    return v;
}
// cp.async (LDGSTS) into a LANE-PRIVATE shared-memory slot: the gathered row vector a lane will consume itself, fetched one
// loop iteration ahead without holding registers (the issuing thread's own wait_group makes it visible to itself).
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// Streaming 128-bit store (output rows are written once and not re-read by the kernel).
__device__ __forceinline__ void stg_stream16(void* p, const Vec16& v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]),
                 "r"(v.w[2]), "r"(v.w[3])
                 : "memory");
}

template <typename T>
struct ElemTraits;
template <>
struct ElemTraits<float> {
    static constexpr int kPerVec = 4;  // elements per 16 B
    __device__ static __forceinline__ void unpack(const Vec16& v, float (&f)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(v.w[i]);
    }
    __device__ static __forceinline__ Vec16 pack(const float (&f)[4]) {
        Vec16 v;
#pragma unroll
        for (int i = 0; i < 4; ++i) v.w[i] = __float_as_uint(f[i]);
        return v;
    }
    __device__ static __forceinline__ float to_float(float x) { return x; }
    __device__ static __forceinline__ float from_float(float x) { return x; }
};
template <>
struct ElemTraits<__nv_bfloat16> {
    static constexpr int kPerVec = 8;
    __device__ static __forceinline__ void unpack(const Vec16& v, float (&f)[8]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            // bf16 -> fp32 is a 16-bit shift: low half first (little endian)
            f[2 * i] = __uint_as_float(v.w[i] << 16);
            f[2 * i + 1] = __uint_as_float(v.w[i] & 0xffff0000u);
        }
    }
    __device__ static __forceinline__ Vec16 pack(const float (&f)[8]) {
        Vec16 v;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __nv_bfloat162 p = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
            v.w[i] = *reinterpret_cast<uint32_t*>(&p);
        }
        return v;
    }
    __device__ static __forceinline__ float to_float(__nv_bfloat16 x) { return __bfloat162float(x); }
    __device__ static __forceinline__ __nv_bfloat16 from_float(float x) { return __float2bfloat16_rn(x); }
};

// v rounded to the storage dtype T and back (a no-op for fp32): where the reference materialises a T tensor.
template <typename T>
__device__ __forceinline__ float round_to(float v) {
    return ElemTraits<T>::to_float(ElemTraits<T>::from_float(v));
}

// A chunk's fp32 partial of one 16-byte vector (EPV elements) as EPV / 4 float4 stores.
template <int EPV>
__device__ __forceinline__ void store_partial(float* p, const float (&acc)[EPV]) {
#pragma unroll
    for (int q = 0; q < EPV / 4; ++q)
        *reinterpret_cast<float4*>(p + 4 * q) = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
}

// ---------------------------------------------------------------- reductions
// ATen amax/amin propagate NaN; fmaxf/fminf do not, so spell the comparison out.
template <int RED>
__device__ __forceinline__ float red_identity() {
    if (RED == B200MP_MIN) return __int_as_float(0x7f800000);   // +inf
    if (RED == B200MP_MAX) return __int_as_float(0xff800000);   // -inf
    if (RED == B200MP_MUL) return 1.0f;
    return 0.0f;
}
template <int RED>
__device__ __forceinline__ float red_combine(float acc, float v) {
    if (RED == B200MP_MIN) return (v < acc || v != v) ? v : acc;
    if (RED == B200MP_MAX) return (v > acc || v != v) ? v : acc;
    if (RED == B200MP_MUL) return __fmul_rn(acc, v);
    return __fadd_rn(acc, v);  // explicit: never contracted into an FMA with the weight product
}

template <typename I>
__device__ __forceinline__ I ldg_idx(const I* p) {
    return __ldg(p);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// splitmix64's finaliser on seed + key * golden ratio (mod 2^64): the counter-based generator of graclus's colours
// (cluster.cu) and of the random walks' draws (random_walk.cu).
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long seed, unsigned long long key) {
    unsigned long long z = seed + key * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

}  // namespace b200mp
