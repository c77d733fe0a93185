// head_dot.cu -- the node-level attention terms of GATConv in one pass over the projected features.
//
// The reference computes  alpha_src = (x_src * att_src).sum(-1),  alpha_dst = (x_dst * att_dst).sum(-1)
// (nn/conv/gat_conv.py:330-331) as a broadcast multiply that materialises [N, H, C] and a reduction over C,
// and autograd replays the pattern twice more in the backward (grad of the product w.r.t. x and w.r.t. att).
// On config 3 (N = 2.4 M, H*C = 128, bf16) those ten elementwise / reduce launches cost ~10 ms of a 40 ms step.
//
//   forward   s_a[n,h] = sum_c x[n,h,c] * att_a[h,c]   (and s_b with att_b from the same read of x)      fp32 out
//   backward  grad_x[n,h,c] = g_a[n,h] * att_a[h,c] + g_b[n,h] * att_b[h,c]  (+ add[n,h,c], e.g. the attention's grad_v)
//             grad_att_a[h,c] = sum_n g_a[n,h] * x[n,h,c]     -> per-CTA partial rows, folded by b200mp_column_sum
//
// Layout: a thread owns ONE 16-byte vector position v of the row (its att values stay in registers) and walks rows
// r0, r0 + R, ... with R = blockDim / n_vec rows per step; the LPH = chan * sizeof(T) / 16 lanes of a head are adjacent
// and aligned, so the per-head sums are xor-shuffles.  HBM-bound: x is read once in each direction.
#include "common.cuh"

namespace b200mp {

constexpr int kHdT = 256;

template <typename T>
__global__ void __launch_bounds__(kHdT)
head_dot_kernel(const T* __restrict__ x, const float* __restrict__ att_a, const float* __restrict__ att_b,
                float* __restrict__ s_a, float* __restrict__ s_b, int64_t n_rows, int n_vec, int heads, int lph) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const int rows_per_step = kHdT / n_vec;
    const int v = threadIdx.x % n_vec, rl = threadIdx.x / n_vec;
    const bool active = rl < rows_per_step;                    // (kHdT % n_vec threads of the last warp carry no row)
    float wa[EPV], wb[EPV];
#pragma unroll
    for (int i = 0; i < EPV; ++i) {
        wa[i] = att_a[v * EPV + i];
        wb[i] = att_b ? att_b[v * EPV + i] : 0.f;
    }
    const int head = v / lph;
    const bool writer = (v % lph) == 0;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    // every thread of the CTA takes the same number of trips (full-mask shuffles); the LPH lanes of a head are adjacent,
    // aligned (lph divides n_vec and 32) and belong to the same row
    const int64_t stride = static_cast<int64_t>(gridDim.x) * rows_per_step;
    for (int64_t r0 = static_cast<int64_t>(blockIdx.x) * rows_per_step; r0 < n_rows; r0 += stride) {
        const int64_t r = r0 + rl;
        const bool valid = active && r < n_rows;
        float f[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = 0.f;
        if (valid)
            ElemTraits<T>::unpack(ldg_stream16(reinterpret_cast<const char*>(x) + static_cast<size_t>(r) * row_bytes + static_cast<size_t>(v) * 16), f);
        float da = 0.f, db = 0.f;
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            da = fmaf(f[i], wa[i], da);
            db = fmaf(f[i], wb[i], db);
        }
        for (int o = 1; o < lph; o <<= 1) {
            da += __shfl_xor_sync(0xffffffffu, da, o);
            db += __shfl_xor_sync(0xffffffffu, db, o);
        }
        if (valid && writer) {
            s_a[r * heads + head] = da;
            if (s_b) s_b[r * heads + head] = db;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kHdT)
head_dot_backward_kernel(const T* __restrict__ x, const float* __restrict__ att_a, const float* __restrict__ att_b,
                         const float* __restrict__ g_a, const float* __restrict__ g_b, const T* __restrict__ add,
                         T* __restrict__ grad_x, float* __restrict__ part_a, float* __restrict__ part_b,
                         int64_t n_rows, int n_vec, int heads, int lph) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    __shared__ float red[2][kHdT][EPV + 1];
    const int rows_per_step = kHdT / n_vec;
    const int v = threadIdx.x % n_vec, rl = threadIdx.x / n_vec;
    const bool active = rl < rows_per_step;
    float wa[EPV], wb[EPV], acc_a[EPV], acc_b[EPV];
#pragma unroll
    for (int i = 0; i < EPV; ++i) {
        wa[i] = att_a[v * EPV + i];
        wb[i] = att_b ? att_b[v * EPV + i] : 0.f;
        acc_a[i] = acc_b[i] = 0.f;
    }
    const int head = v / lph;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    if (active) {
        for (int64_t r = static_cast<int64_t>(blockIdx.x) * rows_per_step + rl; r < n_rows; r += static_cast<int64_t>(gridDim.x) * rows_per_step) {
            const size_t off = static_cast<size_t>(r) * row_bytes + static_cast<size_t>(v) * 16;
            const float ga = g_a[r * heads + head], gb = g_b ? g_b[r * heads + head] : 0.f;
            float f[EPV], o[EPV];
            ElemTraits<T>::unpack(ldg_stream16(reinterpret_cast<const char*>(x) + off), f);
            if (add) {
                ElemTraits<T>::unpack(ldg_stream16(reinterpret_cast<const char*>(add) + off), o);
            } else {
#pragma unroll
                for (int i = 0; i < EPV; ++i) o[i] = 0.f;
            }
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                o[i] = fmaf(ga, wa[i], fmaf(gb, wb[i], o[i]));
                acc_a[i] = fmaf(ga, f[i], acc_a[i]);
                acc_b[i] = fmaf(gb, f[i], acc_b[i]);
            }
            if (grad_x) stg_stream16(reinterpret_cast<char*>(grad_x) + off, ElemTraits<T>::pack(o));
        }
    }
    // fold the CTA's row groups in fixed order: one partial row [n_vec * EPV] per CTA and per attention vector
#pragma unroll
    for (int i = 0; i < EPV; ++i) {
        red[0][threadIdx.x][i] = acc_a[i];
        red[1][threadIdx.x][i] = acc_b[i];
    }
    __syncthreads();
    if (threadIdx.x < n_vec) {
        for (int i = 0; i < EPV; ++i) {
            float ta = 0.f, tb = 0.f;
            for (int g = 0; g < rows_per_step; ++g) {
                ta += red[0][g * n_vec + threadIdx.x][i];
                tb += red[1][g * n_vec + threadIdx.x][i];
            }
            const size_t o = static_cast<size_t>(blockIdx.x) * n_vec * EPV + static_cast<size_t>(threadIdx.x) * EPV + i;
            part_a[o] = ta;
            if (part_b) part_b[o] = tb;
        }
    }
}

static bool head_dot_shape_ok(int64_t heads, int64_t chan, int val_dtype) {
    const int64_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    if (val_dtype != B200MP_BF16 && val_dtype != B200MP_F32) return false;
    if (heads < 1 || chan < 1 || (chan * es) % 16 != 0) return false;
    const int64_t lph = chan * es / 16;
    if (lph > 32 || (lph & (lph - 1)) != 0) return false;
    return heads * lph <= kHdT;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_head_dot_supported(int64_t heads, int64_t chan, int val_dtype) {
    return head_dot_shape_ok(heads, chan, val_dtype) ? 1 : 0;
}

extern "C" int64_t b200mp_head_dot_parts(int64_t n_rows, int64_t heads, int64_t chan, int val_dtype) {
    if (!head_dot_shape_ok(heads, chan, val_dtype) || n_rows <= 0) return 0;
    const int64_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    const int64_t n_vec = heads * chan * es / 16, rps = kHdT / n_vec;
    const int64_t want = ceil_div(n_rows, rps);
    int sms = kSMs;
    b200mp_device_info(&sms, nullptr, nullptr, nullptr);
    const int64_t cap = static_cast<int64_t>(sms) * 8;
    return want < cap ? want : cap;
}

extern "C" int b200mp_head_dot(const void* x, const float* att_a, const float* att_b, float* s_a, float* s_b,
                               int64_t n_rows, int64_t heads, int64_t chan, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0);
    B200MP_CHECK_ARG(head_dot_shape_ok(heads, chan, val_dtype));
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(x && att_a && s_a && (!att_b == !s_b) && aligned16(x));
    const int64_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    const int lph = static_cast<int>(chan * es / 16), n_vec = static_cast<int>(heads) * lph;
    const unsigned blocks = static_cast<unsigned>(b200mp_head_dot_parts(n_rows, heads, chan, val_dtype));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (val_dtype == B200MP_BF16)
        head_dot_kernel<__nv_bfloat16><<<blocks, kHdT, 0, s>>>(static_cast<const __nv_bfloat16*>(x), att_a, att_b, s_a, s_b, n_rows, n_vec,
                                                              static_cast<int>(heads), lph);
    else
        head_dot_kernel<float><<<blocks, kHdT, 0, s>>>(static_cast<const float*>(x), att_a, att_b, s_a, s_b, n_rows, n_vec,
                                                      static_cast<int>(heads), lph);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

extern "C" int b200mp_head_dot_backward(const void* x, const float* att_a, const float* att_b, const float* g_a,
                                        const float* g_b, const void* add, void* grad_x, float* part_a, float* part_b,
                                        int64_t n_parts, int64_t n_rows, int64_t heads, int64_t chan, int val_dtype,
                                        void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0);
    B200MP_CHECK_ARG(head_dot_shape_ok(heads, chan, val_dtype));
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(x && att_a && g_a && part_a && (!att_b == !g_b) && (!att_b == !part_b));
    B200MP_CHECK_ARG(aligned16(x) && aligned16(add) && aligned16(grad_x));
    B200MP_CHECK_ARG(n_parts == b200mp_head_dot_parts(n_rows, heads, chan, val_dtype));
    const int64_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    const int lph = static_cast<int>(chan * es / 16), n_vec = static_cast<int>(heads) * lph;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (val_dtype == B200MP_BF16)
        head_dot_backward_kernel<__nv_bfloat16><<<static_cast<unsigned>(n_parts), kHdT, 0, s>>>(
            static_cast<const __nv_bfloat16*>(x), att_a, att_b, g_a, g_b, static_cast<const __nv_bfloat16*>(add),
            static_cast<__nv_bfloat16*>(grad_x), part_a, part_b, n_rows, n_vec, static_cast<int>(heads), lph);
    else
        head_dot_backward_kernel<float><<<static_cast<unsigned>(n_parts), kHdT, 0, s>>>(
            static_cast<const float*>(x), att_a, att_b, g_a, g_b, static_cast<const float*>(add), static_cast<float*>(grad_x),
            part_a, part_b, n_rows, n_vec, static_cast<int>(heads), lph);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}
