// scatter.cu -- the COO fallback: out[index[e],:] (+)= src[e,:] for an UNSORTED index, using
// global atomics (the only place the engine uses them), and the row gather used by the unfused
// compatibility path.  Not deterministic for fp32 sums (order of atomics); the CSR path is.
#include "common.cuh"

namespace b200mp {

constexpr int kT = 256;

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    // sm_90+: one 16-byte reduction instead of four 4-byte ones
    asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
    if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));  // sign bit clear (-0.0 goes the other way)
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_min_f32(float* addr, float v) {
    if (__float_as_int(v) >= 0) atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_mul_f32(float* addr, float v) {
    unsigned int* a = reinterpret_cast<unsigned int*>(addr);
    unsigned int old = *a, assumed;
    do {
        assumed = old;
        old = atomicCAS(a, assumed, __float_as_uint(__fmul_rn(__uint_as_float(assumed), v)));
    } while (assumed != old);
}

__global__ void fill_f32_kernel(float* p, int64_t n, float v) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        p[i] = v;
}

template <typename I>
__global__ void scatter_add_v4_kernel(const float* __restrict__ src, const I* __restrict__ index,
                                      float* __restrict__ out, float* __restrict__ count, int64_t n_src,
                                      int n_vec, int64_t n_rows) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t e = t / n_vec;
    const int v = static_cast<int>(t - e * n_vec);
    if (e >= n_src) return;
    const int64_t d = index[e];
    if (static_cast<uint64_t>(d) >= static_cast<uint64_t>(n_rows)) return;   // out-of-range rows are dropped, never written
    const float4 s = __ldcs(reinterpret_cast<const float4*>(src) + e * n_vec + v);
    red_add_v4(out + (d * n_vec + v) * 4, s.x, s.y, s.z, s.w);
    if (count && v == 0) atomicAdd(count + d, 1.0f);
}

template <typename I, int RED>
__global__ void scatter_scalar_kernel(const float* __restrict__ src, const I* __restrict__ index,
                                      float* __restrict__ out, float* __restrict__ count, int64_t n_src,
                                      int64_t feat, int64_t n_rows) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t e = t / feat;
    const int64_t f = t - e * feat;
    if (e >= n_src) return;
    const int64_t d = index[e];
    if (static_cast<uint64_t>(d) >= static_cast<uint64_t>(n_rows)) return;
    const float s = src[t];
    float* o = out + d * feat + f;
    if (RED == B200MP_SUM) atomicAdd(o, s);
    else if (RED == B200MP_MAX) atomic_max_f32(o, s);
    else if (RED == B200MP_MIN) atomic_min_f32(o, s);
    else atomic_mul_f32(o, s);
    if (count && f == 0) atomicAdd(count + d, 1.0f);
}

// mean: out /= max(count, 1); min/max: rows with count == 0 become 0 (_scatter.py:72-100)
template <int RED>
__global__ void scatter_fixup_kernel(float* __restrict__ out, const float* __restrict__ count, int64_t n_rows,
                                     int64_t feat, bool is_mean) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_rows * feat) return;
    const float c = count[t / feat];
    if (RED == B200MP_SUM) {
        if (is_mean) out[t] = __fdiv_rn(out[t], fmaxf(c, 1.0f));
    } else if (c == 0.0f) {
        out[t] = 0.0f;
    }
}

template <typename T, typename I>
__global__ void gather_rows_vec_kernel(const T* __restrict__ x, const I* __restrict__ index,
                                       const float* __restrict__ scale, T* __restrict__ out, int64_t n_out,
                                       int n_vec) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t e = t / n_vec;
    const int v = static_cast<int>(t - e * n_vec);
    if (e >= n_out) return;
    const int64_t r = index[e];
    Vec16 d = ldg_row16(reinterpret_cast<const char*>(x) + (static_cast<size_t>(r) * n_vec + v) * 16);
    if (scale) {
        float f[EPV];
        ElemTraits<T>::unpack(d, f);
        const float s = scale[e];
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = __fmul_rn(s, f[i]);
        d = ElemTraits<T>::pack(f);
    }
    stg_stream16(reinterpret_cast<char*>(out) + (static_cast<size_t>(e) * n_vec + v) * 16, d);
}
template <typename T, typename I>
__global__ void gather_rows_scalar_kernel(const T* __restrict__ x, const I* __restrict__ index,
                                          const float* __restrict__ scale, T* __restrict__ out, int64_t n_out,
                                          int64_t feat) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t e = t / feat;
    if (e >= n_out) return;
    const int64_t f = t - e * feat;
    float v = ElemTraits<T>::to_float(x[static_cast<int64_t>(index[e]) * feat + f]);
    if (scale) v = __fmul_rn(scale[e], v);
    out[t] = ElemTraits<T>::from_float(v);
}

inline unsigned blocks_for(int64_t n) { return static_cast<unsigned>(n <= 0 ? 1 : ceil_div(n, kT)); }

template <typename I>
int scatter_typed(const float* src, const void* index_, float* out, float* count, int64_t n_src, int64_t n_rows,
                  int64_t feat, int reduce, cudaStream_t s) {
    const I* index = static_cast<const I*>(index_);
    const int64_t n_out = n_rows * feat;
    const bool need_count = reduce == B200MP_MEAN || reduce == B200MP_MIN || reduce == B200MP_MAX;
    if (need_count && !count) {
        set_error("scatter_coo: reduce %d needs the count scratch", reduce);
        return B200MP_ERR_INVALID_ARG;
    }
    float init = 0.0f;
    if (reduce == B200MP_MIN) init = __builtin_inff();
    if (reduce == B200MP_MAX) init = -__builtin_inff();
    if (reduce == B200MP_MUL) init = 1.0f;
    unsigned fb = blocks_for(n_out);
    if (fb > static_cast<unsigned>(num_sms()) * 16u) fb = static_cast<unsigned>(num_sms()) * 16u;
    if (init == 0.0f) B200MP_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * n_out, s));
    else fill_f32_kernel<<<fb, kT, 0, s>>>(out, n_out, init);
    if (need_count) B200MP_CUDA(cudaMemsetAsync(count, 0, sizeof(float) * n_rows, s));
    float* cnt = need_count ? count : nullptr;
    if (n_src > 0) {
        const bool v4 = (reduce == B200MP_SUM || reduce == B200MP_MEAN) && feat % 4 == 0 && aligned16(src) && aligned16(out);
        if (v4) {
            const int n_vec = static_cast<int>(feat / 4);
            scatter_add_v4_kernel<I><<<blocks_for(n_src * n_vec), kT, 0, s>>>(src, index, out, cnt, n_src, n_vec, n_rows);
        } else if (reduce == B200MP_SUM || reduce == B200MP_MEAN) {
            scatter_scalar_kernel<I, B200MP_SUM><<<blocks_for(n_src * feat), kT, 0, s>>>(src, index, out, cnt, n_src, feat, n_rows);
        } else if (reduce == B200MP_MAX) {
            scatter_scalar_kernel<I, B200MP_MAX><<<blocks_for(n_src * feat), kT, 0, s>>>(src, index, out, cnt, n_src, feat, n_rows);
        } else if (reduce == B200MP_MIN) {
            scatter_scalar_kernel<I, B200MP_MIN><<<blocks_for(n_src * feat), kT, 0, s>>>(src, index, out, cnt, n_src, feat, n_rows);
        } else {
            scatter_scalar_kernel<I, B200MP_MUL><<<blocks_for(n_src * feat), kT, 0, s>>>(src, index, out, cnt, n_src, feat, n_rows);
        }
        B200MP_LAUNCH_CHECK();
    }
    if (reduce == B200MP_MEAN) scatter_fixup_kernel<B200MP_SUM><<<blocks_for(n_out), kT, 0, s>>>(out, count, n_rows, feat, true);
    else if (reduce == B200MP_MIN || reduce == B200MP_MAX) scatter_fixup_kernel<B200MP_MAX><<<blocks_for(n_out), kT, 0, s>>>(out, count, n_rows, feat, false);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename T, typename I>
int gather_typed(const void* x, const void* index, const float* scale, void* out, int64_t n_out, int64_t feat,
                 cudaStream_t s) {
    const size_t row_bytes = static_cast<size_t>(feat) * sizeof(T);
    if (row_bytes % 16 == 0 && aligned16(x) && aligned16(out)) {
        const int n_vec = static_cast<int>(row_bytes / 16);
        gather_rows_vec_kernel<T, I><<<blocks_for(n_out * n_vec), kT, 0, s>>>(
            static_cast<const T*>(x), static_cast<const I*>(index), scale, static_cast<T*>(out), n_out, n_vec);
    } else {
        gather_rows_scalar_kernel<T, I><<<blocks_for(n_out * feat), kT, 0, s>>>(
            static_cast<const T*>(x), static_cast<const I*>(index), scale, static_cast<T*>(out), n_out, feat);
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_scatter_coo(const float* src, const void* index, float* out, float* count, int64_t n_src,
                                  int64_t n_rows, int64_t feat, int reduce, int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_src >= 0 && n_rows >= 0 && feat >= 0);
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(out);
    B200MP_CHECK_ARG(n_src == 0 || (src && index));
    B200MP_CHECK_ARG(reduce >= B200MP_SUM && reduce <= B200MP_MUL);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (idx_dtype == B200MP_I32) return scatter_typed<int32_t>(src, index, out, count, n_src, n_rows, feat, reduce, s);
    if (idx_dtype == B200MP_I64) return scatter_typed<int64_t>(src, index, out, count, n_src, n_rows, feat, reduce, s);
    set_error("bad idx_dtype %d", idx_dtype);
    return B200MP_ERR_UNSUPPORTED;
}

// out[index[e], :] += src[e, :] into an EXISTING out (no initialisation): the return leg of the
// halo exchange (gradient rows of remote sources added into their owner's rows).
extern "C" int b200mp_index_add_rows(const float* src, const void* index, float* out, int64_t n_src, int64_t feat,
                                     int idx_dtype, void* stream) {
    B200MP_CHECK_ARG(n_src >= 0 && feat >= 0);
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(src && index && out);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool v4 = feat % 4 == 0 && aligned16(src) && aligned16(out);
    if (idx_dtype == B200MP_I32) {
        if (v4) scatter_add_v4_kernel<int32_t><<<blocks_for(n_src * (feat / 4)), kT, 0, s>>>(src, static_cast<const int32_t*>(index), out, nullptr, n_src, static_cast<int>(feat / 4), INT64_MAX);
        else scatter_scalar_kernel<int32_t, B200MP_SUM><<<blocks_for(n_src * feat), kT, 0, s>>>(src, static_cast<const int32_t*>(index), out, nullptr, n_src, feat, INT64_MAX);
    } else if (idx_dtype == B200MP_I64) {
        if (v4) scatter_add_v4_kernel<int64_t><<<blocks_for(n_src * (feat / 4)), kT, 0, s>>>(src, static_cast<const int64_t*>(index), out, nullptr, n_src, static_cast<int>(feat / 4), INT64_MAX);
        else scatter_scalar_kernel<int64_t, B200MP_SUM><<<blocks_for(n_src * feat), kT, 0, s>>>(src, static_cast<const int64_t*>(index), out, nullptr, n_src, feat, INT64_MAX);
    } else {
        set_error("bad idx_dtype %d", idx_dtype);
        return B200MP_ERR_UNSUPPORTED;
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_gather_rows(const void* x, const void* index, const float* scale, void* out, int64_t n_out,
                                  int64_t feat, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_out >= 0 && feat >= 0);
    if (n_out == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(x && index && out);
    return dispatch_val_idx(val_dtype, idx_dtype, "gather_rows", [&](auto tv, auto ti) {
        return gather_typed<decltype(tv), decltype(ti)>(x, index, scale, out, n_out, feat, static_cast<cudaStream_t>(stream));
    });
}
