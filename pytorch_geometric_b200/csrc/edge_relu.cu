// edge_relu.cu -- GINEConv's message relu(x_j + e_ji) fused into the CSR gather-reduce, and its backward.
//
//   out[i,:] = REDUCE_{e in [rowptr[i], rowptr[i+1])} relu(x[col[e],:] + a[eid(e),:])     REDUCE = sum | mean
//   eid(e)   = perm[e] (CSR slot -> the caller's edge id), or e for an adopted CSR (perm == NULL)
//
// The edge rows `a` are read through perm, in the caller's order: they are never copied into CSR order.  x + a is
// rounded to the storage dtype before the ReLU (the reference adds in that dtype), the ReLU keeps NaN (relu(NaN) =
// NaN, which fmaxf would turn into 0), and the sum is accumulated in fp32 in CSR order.
//
// ReLU mask (training only): one bit per (edge, feature) in CSR order, mask_bytes = ceil(feat / 8) bytes per edge;
// bit f % 8 of byte mask[e * mask_bytes + f / 8] is set iff !(x + a <= 0) -- threshold_backward's rule on the
// ReLU's output: 0 at x + a == 0, passed through at NaN.  An fp32 16-byte vector owns a nibble (two vectors per
// byte, combined with one shuffle), a bf16 vector a whole byte.  The two backward sweeps read the bits instead of
// any [E, F] intermediate:
//   grad_x[j,:]       = sum_{t in rowT(j)} bit(t2csr[t]) ? valT[t] * g[colT[t],:] : 0        (transposed CSR)
//   grad_a[eid(e),:]  = bit(e) ? g[i,:] / (mean ? max(deg_i, 1) : 1) : 0                    (destination CSR)
//
// Mapping as in csr_reduce.cuh: a lane group of G lanes per row, VPL 16-byte vectors per lane, rows longer than the
// plan's chunk split into chunks whose fp32 partials csr_combine_kernel folds in chunk order.
#include "csr_reduce.cuh"

namespace b200mp {

// Byte offset and bit shift of 16-byte vector v's first feature inside an edge's mask row.
template <typename T>
__device__ __forceinline__ int mask_byte(int v) { return ElemTraits<T>::kPerVec == 8 ? v : (v >> 1); }
template <typename T>
__device__ __forceinline__ int mask_shift(int v) { return ElemTraits<T>::kPerVec == 8 ? 0 : (v & 1) * 4; }

// Write the bits of vector v (bit i = feature 4v + i / 8v + i).  fp32: lanes lig and lig ^ 1 (same group, so both
// reach this call) hold the two nibbles of one byte; the even lane writes it.  `bits` must be 0 when !valid.
template <typename T, int G>
__device__ __forceinline__ void store_mask(uint8_t* mrow, int v, unsigned bits, int lig, bool valid) {
    if (ElemTraits<T>::kPerVec == 8 || G == 1) {
        if (valid) mrow[mask_byte<T>(v)] = static_cast<uint8_t>(bits);
    } else {
        const unsigned lane = threadIdx.x & 31;
        const unsigned other = __shfl_xor_sync(3u << (lane & ~1u), bits, 1);
        if (!(lig & 1) && valid) mrow[v >> 1] = static_cast<uint8_t>(bits | (other << 4));
    }
}

// Epilogue of a row or chunk: fp32 partial for a chunk, finalised row otherwise.
template <typename T, int EPV>
__device__ __forceinline__ void store_acc(const float (&acc)[EPV], bool is_chunk, int64_t item, int64_t row, int v,
                                          int n_vec, int64_t deg, bool is_mean, const LongRowPlan& plan, T* out) {
    if (is_chunk) {
        store_partial<EPV>(plan.partials + (static_cast<size_t>(item) * n_vec + v) * EPV, acc);
    } else {
        float f[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = finalize<B200MP_SUM>(acc[i], deg, is_mean, false);
        stg_stream16(reinterpret_cast<char*>(out) + (static_cast<size_t>(row) * n_vec + v) * 16, ElemTraits<T>::pack(f));
    }
}

// ---------------------------------------------------------------- forward
template <typename T, typename I, int G, int VPL, int UNR>
__global__ void __launch_bounds__(128)
edge_relu_reduce_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const I* __restrict__ perm,
                        const T* __restrict__ x, const T* __restrict__ a, T* __restrict__ out,
                        uint8_t* __restrict__ mask, int64_t n_rows, int n_vec, int64_t mask_bytes, bool is_mean,
                        LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // uniform per group
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = reinterpret_cast<const char*>(x);
    const char* ab = reinterpret_cast<const char*>(a);

    for (int vbase = 0; vbase < n_vec; vbase += G * VPL) {
        float acc[VPL][EPV];
        bool vvalid[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            vvalid[k] = (vbase + lig + k * G) < n_vec;
#pragma unroll
            for (int i = 0; i < EPV; ++i) acc[k][i] = 0.0f;
        }
        const size_t voff = static_cast<size_t>(vbase + lig) * 16;
        for (int64_t e = begin; e < end; e += UNR) {
            Vec16 xv[UNR][VPL], av[UNR][VPL];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
                    const int64_t c = static_cast<int64_t>(ldg_idx(col + e + u));
                    const int64_t id = perm ? static_cast<int64_t>(ldg_idx(perm + e + u)) : e + u;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (vvalid[k]) {
                            xv[u][k] = ldg_row16(xb + c * row_bytes + voff + static_cast<size_t>(k) * G * 16);
                            av[u][k] = ldg_stream16(ab + id * row_bytes + voff + static_cast<size_t>(k) * G * 16);
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (e + u < end) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        unsigned bits = 0;
                        if (vvalid[k]) {
                            float fx[EPV], fa[EPV];
                            ElemTraits<T>::unpack(xv[u][k], fx);
                            ElemTraits<T>::unpack(av[u][k], fa);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) {
                                const float s = round_to<T>(__fadd_rn(fx[i], fa[i]));
                                const bool on = !(s <= 0.0f);
                                bits |= static_cast<unsigned>(on) << i;
                                acc[k][i] = __fadd_rn(acc[k][i], on ? s : 0.0f);
                            }
                        }
                        if (mask)
                            store_mask<T, G>(mask + static_cast<size_t>(e + u) * mask_bytes, vbase + lig + k * G, bits,
                                             lig, vvalid[k]);
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k)
            if (vvalid[k]) store_acc<T, EPV>(acc[k], is_chunk, item, row, vbase + lig + k * G, n_vec, end - begin, is_mean, plan, out);
    }
}

// Rows that are not a whole number of aligned 16-byte vectors: one warp per work item, lane = feature, bits by ballot.
template <typename T, typename I>
__global__ void __launch_bounds__(256)
edge_relu_reduce_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const I* __restrict__ perm,
                               const T* __restrict__ x, const T* __restrict__ a, T* __restrict__ out,
                               uint8_t* __restrict__ mask, int64_t n_rows, int64_t feat, int64_t mask_bytes,
                               bool is_mean, LongRowPlan plan) {
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // warp-uniform
    for (int64_t f0 = 0; f0 < feat; f0 += 32) {
        const int64_t f = f0 + lane;
        const bool fv = f < feat;
        float acc = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = static_cast<int64_t>(ldg_idx(col + e));
            const int64_t id = perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e;
            bool on = false;
            if (fv) {
                const float s = round_to<T>(__fadd_rn(ElemTraits<T>::to_float(x[c * feat + f]),
                                                      ElemTraits<T>::to_float(a[id * feat + f])));
                on = !(s <= 0.0f);
                acc = __fadd_rn(acc, on ? s : 0.0f);
            }
            if (mask) {
                const unsigned b = __ballot_sync(0xffffffffu, on);
                if (lane < 4 && f0 + 8 * lane < feat)
                    mask[e * mask_bytes + f0 / 8 + lane] = static_cast<uint8_t>(b >> (8 * lane));
            }
        }
        if (!fv) continue;
        if (is_chunk) plan.partials[item * feat + f] = acc;
        else out[row * feat + f] = ElemTraits<T>::from_float(finalize<B200MP_SUM>(acc, end - begin, is_mean, false));
    }
}

// ---------------------------------------------------------------- backward: grad_x over the transposed CSR
template <typename T, typename I, int G, int VPL, int UNR>
__global__ void __launch_bounds__(128)
edge_relu_grad_x_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t, const I* __restrict__ t2csr,
                        const float* __restrict__ val_t, const T* __restrict__ g, const uint8_t* __restrict__ mask,
                        T* __restrict__ grad_x, int64_t n_src, int n_vec, int64_t mask_bytes, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr_t, n_src, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* gb = reinterpret_cast<const char*>(g);

    for (int vbase = 0; vbase < n_vec; vbase += G * VPL) {
        float acc[VPL][EPV];
        bool vvalid[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            vvalid[k] = (vbase + lig + k * G) < n_vec;
#pragma unroll
            for (int i = 0; i < EPV; ++i) acc[k][i] = 0.0f;
        }
        const size_t voff = static_cast<size_t>(vbase + lig) * 16;
        for (int64_t t = begin; t < end; t += UNR) {
            Vec16 gv[UNR][VPL];
            unsigned mb[UNR][VPL];
            float w[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                w[u] = 1.0f;
                if (t + u < end) {
                    const int64_t d = static_cast<int64_t>(ldg_idx(col_t + t + u));
                    const int64_t s = static_cast<int64_t>(ldg_idx(t2csr + t + u));
                    if (val_t) w[u] = __ldg(val_t + t + u);
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (vvalid[k]) {
                            const int v = vbase + lig + k * G;
                            gv[u][k] = ldg_row16(gb + d * row_bytes + voff + static_cast<size_t>(k) * G * 16);
                            mb[u][k] = static_cast<unsigned>(__ldg(mask + s * mask_bytes + mask_byte<T>(v))) >> mask_shift<T>(v);
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                if (t + u < end) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (vvalid[k]) {
                            float f[EPV];
                            ElemTraits<T>::unpack(gv[u][k], f);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) {
                                const float m = val_t ? __fmul_rn(w[u], f[i]) : f[i];
                                acc[k][i] = __fadd_rn(acc[k][i], ((mb[u][k] >> i) & 1u) ? m : 0.0f);
                            }
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k)
            if (vvalid[k]) store_acc<T, EPV>(acc[k], is_chunk, item, row, vbase + lig + k * G, n_vec, end - begin, false, plan, grad_x);
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(256)
edge_relu_grad_x_scalar_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t, const I* __restrict__ t2csr,
                               const float* __restrict__ val_t, const T* __restrict__ g, const uint8_t* __restrict__ mask,
                               T* __restrict__ grad_x, int64_t n_src, int64_t feat, int64_t mask_bytes, LongRowPlan plan) {
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr_t, n_src, plan, row, begin, end, is_chunk)) return;
    for (int64_t f = lane; f < feat; f += 32) {
        float acc = 0.0f;
        for (int64_t t = begin; t < end; ++t) {
            const int64_t d = static_cast<int64_t>(ldg_idx(col_t + t));
            const int64_t s = static_cast<int64_t>(ldg_idx(t2csr + t));
            if ((__ldg(mask + s * mask_bytes + f / 8) >> (f % 8)) & 1) {
                const float gf = ElemTraits<T>::to_float(g[d * feat + f]);
                acc = __fadd_rn(acc, val_t ? __fmul_rn(__ldg(val_t + t), gf) : gf);
            }
        }
        if (is_chunk) plan.partials[item * feat + f] = acc;
        else grad_x[row * feat + f] = ElemTraits<T>::from_float(acc);
    }
}

// ---------------------------------------------------------------- backward: grad_a over the destination CSR
// Every CSR slot is written exactly once (chunks of hub rows only split the work), in the caller's edge order.
template <typename T, typename I, int G, int VPL>
__global__ void __launch_bounds__(128)
edge_relu_grad_edge_kernel(const I* __restrict__ rowptr, const I* __restrict__ perm, const T* __restrict__ g,
                           const uint8_t* __restrict__ mask, T* __restrict__ grad_a, int64_t n_rows, int n_vec,
                           int64_t mask_bytes, bool is_mean, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const int64_t deg = static_cast<int64_t>(__ldg(rowptr + row + 1)) - static_cast<int64_t>(__ldg(rowptr + row));
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    char* ob = reinterpret_cast<char*>(grad_a);

    for (int vbase = 0; vbase < n_vec; vbase += G * VPL) {
        float gs[VPL][EPV];
        bool vvalid[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int v = vbase + lig + k * G;
            vvalid[k] = v < n_vec;
            if (vvalid[k]) {
                ElemTraits<T>::unpack(ldg_row16(reinterpret_cast<const char*>(g) + static_cast<size_t>(row) * row_bytes +
                                                static_cast<size_t>(v) * 16), gs[k]);
#pragma unroll
                for (int i = 0; i < EPV; ++i) gs[k][i] = round_to<T>(finalize<B200MP_SUM>(gs[k][i], deg, is_mean, false));
            }
        }
#pragma unroll 4
        for (int64_t e = begin; e < end; ++e) {
            const int64_t id = perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e;
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (!vvalid[k]) continue;
                const int v = vbase + lig + k * G;
                const unsigned bits = static_cast<unsigned>(__ldg(mask + e * mask_bytes + mask_byte<T>(v))) >> mask_shift<T>(v);
                float f[EPV];
#pragma unroll
                for (int i = 0; i < EPV; ++i) f[i] = ((bits >> i) & 1u) ? gs[k][i] : 0.0f;
                stg_stream16(ob + id * row_bytes + static_cast<size_t>(v) * 16, ElemTraits<T>::pack(f));
            }
        }
    }
}

template <typename T, typename I>
__global__ void __launch_bounds__(256)
edge_relu_grad_edge_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ perm, const T* __restrict__ g,
                                  const uint8_t* __restrict__ mask, T* __restrict__ grad_a, int64_t n_rows, int64_t feat,
                                  int64_t mask_bytes, bool is_mean, LongRowPlan plan) {
    const int lane = threadIdx.x & 31;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const int64_t deg = static_cast<int64_t>(rowptr[row + 1]) - static_cast<int64_t>(rowptr[row]);
    for (int64_t f = lane; f < feat; f += 32) {
        const float gs = round_to<T>(finalize<B200MP_SUM>(ElemTraits<T>::to_float(g[row * feat + f]), deg, is_mean, false));
        for (int64_t e = begin; e < end; ++e) {
            const int64_t id = perm ? static_cast<int64_t>(ldg_idx(perm + e)) : e;
            const bool on = (__ldg(mask + e * mask_bytes + f / 8) >> (f % 8)) & 1;
            grad_a[id * feat + f] = ElemTraits<T>::from_float(on ? gs : 0.0f);
        }
    }
}

// ---------------------------------------------------------------- host-side dispatch
inline bool edge_relu_vec_ok(int64_t feat, size_t elem, const void* p0, const void* p1, const void* p2,
                             const LongRowPlan& plan) {
    return (feat * elem) % 16 == 0 && aligned16(p0) && aligned16(p1) && aligned16(p2) &&
           (plan.n_chunks == 0 || aligned16(plan.partials));
}

template <typename T, typename I>
int edge_relu_forward_typed(const void* rowptr_, const void* col_, const void* perm_, const void* x_, const void* a_,
                            void* out_, uint8_t* mask, int64_t n_rows, int64_t feat, int64_t mask_bytes, bool is_mean,
                            LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const I* perm = static_cast<const I*>(perm_);
    const T* x = static_cast<const T*>(x_);
    const T* a = static_cast<const T*>(a_);
    T* out = static_cast<T*>(out_);
    const int64_t items = plan.n_chunks + n_rows;
    if (edge_relu_vec_ok(feat, sizeof(T), x, a, out, plan)) {
        const int n_vec = static_cast<int>(feat * sizeof(T) / 16);
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            edge_relu_reduce_kernel<T, I, G(), VPL(), unroll_for_vpl<VPL()>()>
                <<<static_cast<unsigned>(ceil_div(items, 128 / G())), 128, 0, stream>>>(
                    rowptr, col, perm, x, a, out, mask, n_rows, n_vec, mask_bytes, is_mean, plan);
        });
    } else {
        edge_relu_reduce_scalar_kernel<T, I><<<static_cast<unsigned>(ceil_div(items, 8)), 256, 0, stream>>>(
            rowptr, col, perm, x, a, out, mask, n_rows, feat, mask_bytes, is_mean, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
            rowptr, out, feat, is_mean, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int edge_relu_grad_x_typed(const void* rowptr_t_, const void* col_t_, const void* t2csr_, const float* val_t,
                           const void* g_, const uint8_t* mask, void* grad_x_, int64_t n_src, int64_t feat,
                           int64_t mask_bytes, LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr_t = static_cast<const I*>(rowptr_t_);
    const I* col_t = static_cast<const I*>(col_t_);
    const I* t2csr = static_cast<const I*>(t2csr_);
    const T* g = static_cast<const T*>(g_);
    T* grad_x = static_cast<T*>(grad_x_);
    const int64_t items = plan.n_chunks + n_src;
    if (edge_relu_vec_ok(feat, sizeof(T), g, grad_x, nullptr, plan)) {
        const int n_vec = static_cast<int>(feat * sizeof(T) / 16);
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            edge_relu_grad_x_kernel<T, I, G(), VPL(), unroll_for_vpl<VPL()>()>
                <<<static_cast<unsigned>(ceil_div(items, 128 / G())), 128, 0, stream>>>(
                    rowptr_t, col_t, t2csr, val_t, g, mask, grad_x, n_src, n_vec, mask_bytes, plan);
        });
    } else {
        edge_relu_grad_x_scalar_kernel<T, I><<<static_cast<unsigned>(ceil_div(items, 8)), 256, 0, stream>>>(
            rowptr_t, col_t, t2csr, val_t, g, mask, grad_x, n_src, feat, mask_bytes, plan);
    }
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        csr_combine_kernel<T, I, B200MP_SUM><<<static_cast<unsigned>(plan.n_long), 256, 0, stream>>>(
            rowptr_t, grad_x, feat, false, false, plan, nullptr);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int edge_relu_grad_edge_typed(const void* rowptr_, const void* perm_, const void* g_, const uint8_t* mask,
                              void* grad_a_, int64_t n_rows, int64_t feat, int64_t mask_bytes, bool is_mean,
                              LongRowPlan plan, cudaStream_t stream) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* perm = static_cast<const I*>(perm_);
    const T* g = static_cast<const T*>(g_);
    T* grad_a = static_cast<T*>(grad_a_);
    const int64_t items = plan.n_chunks + n_rows;
    if (edge_relu_vec_ok(feat, sizeof(T), g, grad_a, nullptr, plan)) {
        const int n_vec = static_cast<int>(feat * sizeof(T) / 16);
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            edge_relu_grad_edge_kernel<T, I, G(), VPL()><<<static_cast<unsigned>(ceil_div(items, 128 / G())), 128, 0,
                                                           stream>>>(rowptr, perm, g, mask, grad_a, n_rows, n_vec,
                                                                     mask_bytes, is_mean, plan);
        });
    } else {
        edge_relu_grad_edge_scalar_kernel<T, I><<<static_cast<unsigned>(ceil_div(items, 8)), 256, 0, stream>>>(
            rowptr, perm, g, mask, grad_a, n_rows, feat, mask_bytes, is_mean, plan);
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_edge_relu_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                                    const void* edge_rows, void* out, void* mask, int64_t n_rows, int64_t n_cols,
                                    int64_t n_edges, int64_t feat, int reduce, const int64_t* long_rows,
                                    const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                    float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_cols >= 0 && n_edges >= 0 && feat >= 0);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out);
    B200MP_CHECK_ARG(n_edges == 0 || (col && x && edge_rows));
    return dispatch_val_idx(val_dtype, idx_dtype, "edge_relu_csr", [&](auto tv, auto ti) {
        return edge_relu_forward_typed<decltype(tv), decltype(ti)>(
            rowptr, col, perm, x, edge_rows, out, static_cast<uint8_t*>(mask), n_rows, feat, (feat + 7) / 8,
            reduce == B200MP_MEAN, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_edge_relu_backward_x(const void* rowptr_t, const void* col_t, const void* t2csr,
                                           const float* val_t, const void* grad_out, const void* mask, void* grad_x,
                                           int64_t n_src, int64_t feat, const int64_t* long_rows,
                                           const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                           int64_t chunk, float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_src >= 0 && feat >= 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_src == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr_t && grad_x);
    return dispatch_val_idx(val_dtype, idx_dtype, "edge_relu_backward_x", [&](auto tv, auto ti) {
        return edge_relu_grad_x_typed<decltype(tv), decltype(ti)>(rowptr_t, col_t, t2csr, val_t, grad_out,
                                                                static_cast<const uint8_t*>(mask), grad_x, n_src, feat,
                                                                (feat + 7) / 8, plan, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_edge_relu_backward_edge(const void* rowptr, const void* perm, const void* grad_out,
                                              const void* mask, void* grad_edge_rows, int64_t n_rows, int64_t feat,
                                              int reduce, const int64_t* long_rows, const int64_t* chunk_ptr,
                                              int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype,
                                              int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && feat >= 0);
    B200MP_CHECK_ARG(reduce == B200MP_SUM || reduce == B200MP_MEAN);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, nullptr, false)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && grad_out && grad_edge_rows);
    return dispatch_val_idx(val_dtype, idx_dtype, "edge_relu_backward_edge", [&](auto tv, auto ti) {
        return edge_relu_grad_edge_typed<decltype(tv), decltype(ti)>(rowptr, perm, grad_out,
                                                                   static_cast<const uint8_t*>(mask), grad_edge_rows,
                                                                   n_rows, feat, (feat + 7) / 8, reduce == B200MP_MEAN,
                                                                   plan, static_cast<cudaStream_t>(stream));
    });
}
