// gat.cu -- fused GAT attention + aggregation over the destination-sorted CSR.
//
// Reference (nn/conv/gat_conv.py:387-409, utils/_softmax.py:82-88): alpha_j + alpha_i gathers,
// leaky_relu, scatter-max, exp, scatter-sum, two more gathers, a division, an [E,H,C] message
// tensor and a scatter-add -- about twelve kernels and three E x H x C materialisations.
// Here: ONE sweep.  Forward keeps a running (max, sum, weighted accumulator) per head in
// registers (online softmax), so every source row is read exactly once:
//     HBM bytes per edge = H*C*s (row) + H*4 (a_src gather) + idx;   per node = H*C*s + 3*H*4.
// Power-law hubs: rows longer than `chunk` edges are cut into chunks (the same plan as the
// gather-reduce kernel); every chunk produces a partial (max, sum, accumulator) state and
// gat_combine_kernel merges the states of a row with the usual exp(m_c - M) rescaling.
// Backward is three sweeps with the attention recomputed from the saved per-(node, head) max and
// denominator instead of storing alpha [E,H]:
//   row dots   D[i,h] = <g[i,h,:], out[i,h,:]>                       (thread per (node, head))
//   edge sweep grad_pre[e,h] = alpha_e (<g_i, xh_j> - D_i) leaky'    (thread per (edge, head): no row is
//              walked serially), grad_a_dst = segmented sum of grad_pre (chunked gather-reduce kernel)
//   source sweep on the transposed CSR: grad_xh[j,h,:] = sum_e alpha_e g[d_e,h,:], grad_a_src.
#include "csr_dispatch.cuh"

namespace b200mp {

constexpr int kGatT = 256;

__device__ __forceinline__ float leaky(float v, float slope) { return v > 0.0f ? v : v * slope; }

// ---------------------------------------------------------------- forward, vectorised
// Lane group of G lanes per work item (a CSR row, or one chunk of a hub row); lane owns VPL 16-byte
// vectors; every vector lies inside one head (C % EPV == 0).
template <typename T, typename I, int G, int VPL>
__global__ void __launch_bounds__(kGatT)
gat_fwd_vec_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const T* __restrict__ xh,
                   const float* __restrict__ a_src, const float* __restrict__ a_dst, T* __restrict__ out,
                   float* __restrict__ row_max, float* __restrict__ row_den, int64_t n_rows, int heads,
                   int chan, int n_vec, float slope, LongRowPlan plan, float* __restrict__ part_ms) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int UNR = VPL == 1 ? 4 : 2;
    const int lig = threadIdx.x & (G - 1);
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / G;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(n_vec) * 16;
    const char* xb = reinterpret_cast<const char*>(xh);

    int head[VPL];
    bool valid[VPL];
    float ad[VPL], m[VPL], s[VPL], acc[VPL][EPV];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int v = lig + k * G;
        valid[k] = v < n_vec;
        head[k] = valid[k] ? (v * EPV) / chan : 0;
        ad[k] = valid[k] ? __ldg(a_dst + row * heads + head[k]) : 0.0f;
        m[k] = -__builtin_inff();
        s[k] = 0.0f;
#pragma unroll
        for (int i = 0; i < EPV; ++i) acc[k][i] = 0.0f;
    }
    for (int64_t e = begin; e < end; e += UNR) {
        Vec16 buf[UNR][VPL];
        float as[UNR][VPL];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            if (e + u < end) {
                const int64_t c = col[e + u];
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    if (valid[k]) {
                        buf[u][k] = ldg_row16(xb + static_cast<size_t>(c) * row_bytes + static_cast<size_t>(lig + k * G) * 16);
                        as[u][k] = __ldg(a_src + c * heads + head[k]);
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            if (e + u < end) {
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    if (valid[k]) {
                        const float l = leaky(as[u][k] + ad[k], slope);
                        const float mn = fmaxf(m[k], l);
                        const float sc = expf(m[k] - mn);      // 0 on the first edge (m = -inf)
                        const float p = expf(l - mn);
                        s[k] = fmaf(s[k], sc, p);
                        float f[EPV];
                        ElemTraits<T>::unpack(buf[u][k], f);
#pragma unroll
                        for (int i = 0; i < EPV; ++i) acc[k][i] = fmaf(acc[k][i], sc, p * f[i]);
                        m[k] = mn;
                    }
                }
            }
        }
    }
    if (is_chunk) {
        // partial state of this chunk: accumulator (fp32, relative to the chunk max), max and sum per head
        float* pbase = plan.partials + static_cast<size_t>(item) * n_vec * EPV;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (!valid[k]) continue;
            const int v = lig + k * G;
            float* p = pbase + static_cast<size_t>(v) * EPV;
#pragma unroll
            for (int i = 0; i < EPV; ++i) p[i] = acc[k][i];
            if ((v * EPV) % chan == 0) {
                part_ms[(item * heads + head[k]) * 2 + 0] = m[k];
                part_ms[(item * heads + head[k]) * 2 + 1] = s[k];
            }
        }
        return;
    }
    char* ob = reinterpret_cast<char*>(out) + static_cast<size_t>(row) * row_bytes;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        if (!valid[k]) continue;
        const int v = lig + k * G;
        const float den = s[k] + 1e-16f;                       // _softmax.py:87 "+ 1e-16"
        float f[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = (end > begin) ? acc[k][i] / den : 0.0f;
        stg_stream16(ob + static_cast<size_t>(v) * 16, ElemTraits<T>::pack(f));
        if ((v * EPV) % chan == 0) {                           // first vector of its head
            row_max[row * heads + head[k]] = (end > begin) ? m[k] : 0.0f;
            row_den[row * heads + head[k]] = den;
        }
    }
}

// Merge the chunk states of every hub row: M = max_c m_c; S = sum_c s_c e^{m_c-M}; out = sum_c acc_c e^{m_c-M} / (S + 1e-16)
template <typename T>
__global__ void __launch_bounds__(256)
gat_combine_kernel(T* __restrict__ out, float* __restrict__ row_max, float* __restrict__ row_den, int heads, int chan,
                   LongRowPlan plan, const float* __restrict__ part_ms) {
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t hc = static_cast<int64_t>(heads) * chan;
    for (int64_t f = threadIdx.x; f < hc; f += blockDim.x) {
        const int h = static_cast<int>(f / chan);
        float M = -__builtin_inff();
        for (int64_t c = c0; c < c1; ++c) M = fmaxf(M, part_ms[(c * heads + h) * 2]);
        float S = 0.0f, acc = 0.0f;
        for (int64_t c = c0; c < c1; ++c) {
            const float sc = expf(part_ms[(c * heads + h) * 2] - M);
            S = fmaf(part_ms[(c * heads + h) * 2 + 1], sc, S);
            acc = fmaf(plan.partials[c * hc + f], sc, acc);
        }
        const float den = S + 1e-16f;
        out[row * hc + f] = ElemTraits<T>::from_float(acc / den);
        if (f % chan == 0) {
            row_max[row * heads + h] = M;
            row_den[row * heads + h] = den;
        }
    }
}

// ---------------------------------------------------------------- forward, generic (any H, C)
// One thread per (destination, head): exact two-pass softmax statistics, then CC channels at a time.
template <typename T, typename I, int CC>
__global__ void __launch_bounds__(kGatT)
gat_fwd_scalar_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, const T* __restrict__ xh,
                      const float* __restrict__ a_src, const float* __restrict__ a_dst, T* __restrict__ out,
                      float* __restrict__ row_max, float* __restrict__ row_den, int64_t n_rows, int heads,
                      int chan, float slope) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_rows * heads) return;
    const int64_t row = t / heads;
    const int h = static_cast<int>(t - row * heads);
    const int64_t begin = rowptr[row], end = rowptr[row + 1];
    const float ad = a_dst[t];
    float m = -__builtin_inff();
    for (int64_t e = begin; e < end; ++e) m = fmaxf(m, leaky(__ldg(a_src + static_cast<int64_t>(col[e]) * heads + h) + ad, slope));
    float s = 0.0f;
    for (int64_t e = begin; e < end; ++e) s += expf(leaky(__ldg(a_src + static_cast<int64_t>(col[e]) * heads + h) + ad, slope) - m);
    const float den = s + 1e-16f;
    row_max[t] = end > begin ? m : 0.0f;
    row_den[t] = den;
    const int64_t hc = static_cast<int64_t>(heads) * chan;
    for (int c0 = 0; c0 < chan; c0 += CC) {
        float acc[CC];
#pragma unroll
        for (int i = 0; i < CC; ++i) acc[i] = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t c = col[e];
            const float p = expf(leaky(__ldg(a_src + c * heads + h) + ad, slope) - m) / den;
            const T* xr = xh + c * hc + static_cast<int64_t>(h) * chan + c0;
#pragma unroll
            for (int i = 0; i < CC; ++i)
                if (c0 + i < chan) acc[i] = fmaf(p, ElemTraits<T>::to_float(xr[i]), acc[i]);
        }
        T* orow = out + row * hc + static_cast<int64_t>(h) * chan + c0;
#pragma unroll
        for (int i = 0; i < CC; ++i)
            if (c0 + i < chan) orow[i] = ElemTraits<T>::from_float(acc[i]);
    }
}

// alpha[e,h] in CSR order from the saved statistics (return_attention_weights, gat_conv.py:374-383);
// thread per (edge, head) -- dst_of_edge = ptr2index(rowptr)
template <typename I>
__global__ void __launch_bounds__(kGatT)
gat_alpha_kernel(const I* __restrict__ dst_of_edge, const I* __restrict__ col, const float* __restrict__ a_src,
                 const float* __restrict__ a_dst, const float* __restrict__ row_max,
                 const float* __restrict__ row_den, float* __restrict__ alpha, int64_t n_edges, int heads,
                 float slope) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_edges * heads) return;
    const int64_t e = t / heads;
    const int h = static_cast<int>(t - e * heads);
    const int64_t i = dst_of_edge[e];
    alpha[t] = expf(leaky(__ldg(a_src + static_cast<int64_t>(col[e]) * heads + h) + a_dst[i * heads + h], slope) -
                    row_max[i * heads + h]) / row_den[i * heads + h];
}

// ---------------------------------------------------------------- backward
// D[i,h] = <g[i,h,:], out[i,h,:]>
template <typename T>
__global__ void __launch_bounds__(kGatT)
gat_bwd_rowdot_kernel(const T* __restrict__ out, const T* __restrict__ grad_out, float* __restrict__ rowdot,
                      int64_t n_rows, int heads, int chan) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_rows * heads) return;
    const T* g = grad_out + t * chan;
    const T* o = out + t * chan;
    float D = 0.0f;
    for (int c = 0; c < chan; ++c) D = fmaf(ElemTraits<T>::to_float(g[c]), ElemTraits<T>::to_float(o[c]), D);
    rowdot[t] = D;
}
// thread (e,h): alpha, dot = <g[i,h,:], xh[j,h,:]>, grad_pre = alpha (dot - D[i,h]) leaky'(pre)
template <typename T, typename I>
__global__ void __launch_bounds__(kGatT)
gat_bwd_edge_kernel(const I* __restrict__ dst_of_edge, const I* __restrict__ col, const T* __restrict__ xh,
                    const float* __restrict__ a_src, const float* __restrict__ a_dst,
                    const float* __restrict__ row_max, const float* __restrict__ row_den,
                    const float* __restrict__ rowdot, const T* __restrict__ grad_out, float* __restrict__ grad_pre,
                    int64_t n_edges, int heads, int chan, float slope) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_edges * heads) return;
    const int64_t e = t / heads;
    const int h = static_cast<int>(t - e * heads);
    const int64_t i = dst_of_edge[e], j = col[e];
    const int64_t hc = static_cast<int64_t>(heads) * chan;
    const float pre = __ldg(a_src + j * heads + h) + __ldg(a_dst + i * heads + h);
    const float alpha = expf(leaky(pre, slope) - __ldg(row_max + i * heads + h)) / __ldg(row_den + i * heads + h);
    const T* g = grad_out + i * hc + static_cast<int64_t>(h) * chan;
    const T* xr = xh + j * hc + static_cast<int64_t>(h) * chan;
    float dot = 0.0f;
    for (int c = 0; c < chan; ++c) dot = fmaf(ElemTraits<T>::to_float(g[c]), ElemTraits<T>::to_float(xr[c]), dot);
    grad_pre[t] = alpha * (dot - __ldg(rowdot + i * heads + h)) * (pre > 0.0f ? 1.0f : slope);
}

// thread (j,h) on the transposed CSR: grad_xh[j,h,:] = sum_e alpha_e * g[d_e,h,:];
// grad_a_src[j,h] = sum_e grad_pre[csr_slot(e), h].
template <typename T, typename I, int CC>
__global__ void __launch_bounds__(kGatT)
gat_bwd_src_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t, const I* __restrict__ t2csr,
                   const float* __restrict__ a_src, const float* __restrict__ a_dst,
                   const float* __restrict__ row_max, const float* __restrict__ row_den,
                   const T* __restrict__ grad_out, const float* __restrict__ grad_pre,
                   T* __restrict__ grad_xh, float* __restrict__ grad_a_src, int64_t n_src, int heads, int chan,
                   float slope) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_src * heads) return;
    const int64_t j = t / heads;
    const int h = static_cast<int>(t - j * heads);
    const int64_t hc = static_cast<int64_t>(heads) * chan;
    const int64_t begin = rowptr_t[j], end = rowptr_t[j + 1];
    const float as = a_src[t];
    float sum = 0.0f;
    for (int64_t e = begin; e < end; ++e) sum += __ldg(grad_pre + static_cast<int64_t>(t2csr[e]) * heads + h);
    grad_a_src[t] = sum;
    for (int c0 = 0; c0 < chan; c0 += CC) {
        float acc[CC];
#pragma unroll
        for (int i = 0; i < CC; ++i) acc[i] = 0.0f;
        for (int64_t e = begin; e < end; ++e) {
            const int64_t d = col_t[e];
            const float alpha = expf(leaky(as + __ldg(a_dst + d * heads + h), slope) - __ldg(row_max + d * heads + h)) /
                                __ldg(row_den + d * heads + h);
            const T* g = grad_out + d * hc + static_cast<int64_t>(h) * chan + c0;
#pragma unroll
            for (int i = 0; i < CC; ++i)
                if (c0 + i < chan) acc[i] = fmaf(alpha, ElemTraits<T>::to_float(g[i]), acc[i]);
        }
        T* gx = grad_xh + j * hc + static_cast<int64_t>(h) * chan + c0;
#pragma unroll
        for (int i = 0; i < CC; ++i)
            if (c0 + i < chan) gx[i] = ElemTraits<T>::from_float(acc[i]);
    }
}

template <typename T, typename I>
int gat_fwd_typed(const void* rowptr_, const void* col_, const void* dst_of_edge, const void* xh_, const float* a_src,
                  const float* a_dst, void* out_, float* row_max, float* row_den, float* alpha_out, int64_t n_rows,
                  int64_t n_edges, int64_t heads, int64_t chan, float slope, LongRowPlan plan, float* part_ms,
                  cudaStream_t s) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const T* xh = static_cast<const T*>(xh_);
    T* out = static_cast<T*>(out_);
    const size_t row_bytes = static_cast<size_t>(heads * chan) * sizeof(T);
    const bool vec_ok = row_bytes % 16 == 0 && chan % EPV == 0 && aligned16(xh) && aligned16(out) && row_bytes / 16 <= 128;
    if (vec_ok) {
        const int n_vec = static_cast<int>(row_bytes / 16);
        const int64_t items = plan.n_chunks + n_rows;
        lane_group_shape<4>(n_vec, [&](auto G, auto VPL) {
            gat_fwd_vec_kernel<T, I, G(), VPL()><<<static_cast<unsigned>(ceil_div(items, kGatT / G())), kGatT, 0, s>>>(
                rowptr, col, xh, a_src, a_dst, out, row_max, row_den, n_rows, static_cast<int>(heads),
                static_cast<int>(chan), n_vec, slope, plan, part_ms);
        });
        B200MP_LAUNCH_CHECK();
        if (plan.n_long > 0) {
            gat_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), 256, 0, s>>>(out, row_max, row_den, static_cast<int>(heads),
                                                                                      static_cast<int>(chan), plan, part_ms);
            B200MP_LAUNCH_CHECK();
        }
    } else {
        gat_fwd_scalar_kernel<T, I, 8><<<static_cast<unsigned>(ceil_div(n_rows * heads, kGatT)), kGatT, 0, s>>>(
            rowptr, col, xh, a_src, a_dst, out, row_max, row_den, n_rows, static_cast<int>(heads),
            static_cast<int>(chan), slope);
        B200MP_LAUNCH_CHECK();
    }
    if (alpha_out && n_edges > 0) {
        gat_alpha_kernel<I><<<static_cast<unsigned>(ceil_div(n_edges * heads, kGatT)), kGatT, 0, s>>>(
            static_cast<const I*>(dst_of_edge), col, a_src, a_dst, row_max, row_den, alpha_out, n_edges,
            static_cast<int>(heads), slope);
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I>
int gat_bwd_typed(const void* rowptr, const void* col, const void* dst_of_edge, const void* rowptr_t, const void* col_t,
                  const void* t2csr, const void* xh, const float* a_src, const float* a_dst, const float* row_max,
                  const float* row_den, const void* out, const void* grad_out, float* grad_pre, float* rowdot,
                  void* grad_xh, float* grad_a_src, float* grad_a_dst, int64_t n_rows, int64_t n_src, int64_t n_edges,
                  int64_t heads, int64_t chan, float slope, LongRowPlan plan, cudaStream_t s) {
    if (n_rows > 0) {
        gat_bwd_rowdot_kernel<T><<<static_cast<unsigned>(ceil_div(n_rows * heads, kGatT)), kGatT, 0, s>>>(
            static_cast<const T*>(out), static_cast<const T*>(grad_out), rowdot, n_rows, static_cast<int>(heads),
            static_cast<int>(chan));
        if (n_edges > 0)
            gat_bwd_edge_kernel<T, I><<<static_cast<unsigned>(ceil_div(n_edges * heads, kGatT)), kGatT, 0, s>>>(
                static_cast<const I*>(dst_of_edge), static_cast<const I*>(col), static_cast<const T*>(xh), a_src, a_dst,
                row_max, row_den, rowdot, static_cast<const T*>(grad_out), grad_pre, n_edges, static_cast<int>(heads),
                static_cast<int>(chan), slope);
        B200MP_LAUNCH_CHECK();
        // grad_a_dst[i,h] = sum over the CSR row of grad_pre[e,h]: the (chunked) segmented reduce
        const int rc = csr_reduce_auto<float, I, false>(static_cast<const I*>(rowptr), static_cast<const I*>(nullptr), nullptr,
                                                        grad_pre, grad_a_dst, n_rows, heads, B200MP_SUM, false, plan,
                                                        nullptr, s);
        if (rc) return rc;
    }
    if (n_src > 0)
        gat_bwd_src_kernel<T, I, 8><<<static_cast<unsigned>(ceil_div(n_src * heads, kGatT)), kGatT, 0, s>>>(
            static_cast<const I*>(rowptr_t), static_cast<const I*>(col_t), static_cast<const I*>(t2csr), a_src,
            a_dst, row_max, row_den, static_cast<const T*>(grad_out), grad_pre, static_cast<T*>(grad_xh),
            grad_a_src, n_src, static_cast<int>(heads), static_cast<int>(chan), slope);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_gat_fused_csr(const void* rowptr, const void* col, const void* dst_of_edge, const void* xh,
                                    const float* a_src, const float* a_dst, void* out, float* row_max, float* row_den,
                                    float* alpha_out, int64_t n_rows, int64_t n_edges, int64_t heads, int64_t chan,
                                    float slope, const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                    int64_t n_chunks, int64_t chunk, float* part_acc, float* part_ms, int idx_dtype,
                                    int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_edges >= 0 && heads > 0 && chan > 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, part_acc, true)) return rc;
    B200MP_CHECK_ARG(n_long_rows == 0 || part_ms);
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && a_dst && out && row_max && row_den);
    B200MP_CHECK_ARG(!alpha_out || dst_of_edge);
    return dispatch_val_idx(val_dtype, idx_dtype, "gat_fused_csr", [&](auto tv, auto ti) {
        return gat_fwd_typed<decltype(tv), decltype(ti)>(rowptr, col, dst_of_edge, xh, a_src, a_dst, out, row_max,
                                                         row_den, alpha_out, n_rows, n_edges, heads, chan, slope, plan,
                                                         part_ms, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int b200mp_gat_fused_csr_backward(const void* rowptr, const void* col, const void* dst_of_edge,
                                             const void* rowptr_t, const void* col_t, const void* t2csr, const void* xh,
                                             const float* a_src, const float* a_dst, const float* row_max,
                                             const float* row_den, const void* out, const void* grad_out,
                                             float* grad_pre, float* rowdot, void* grad_xh, float* grad_a_src,
                                             float* grad_a_dst, int64_t n_rows, int64_t n_src, int64_t n_edges,
                                             int64_t heads, int64_t chan, float slope, const int64_t* long_rows,
                                             const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                             int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                             void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_src >= 0 && n_edges >= 0 && heads > 0 && chan > 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    B200MP_CHECK_ARG(rowptr && rowptr_t && grad_xh && grad_a_src && grad_a_dst && rowdot);
    B200MP_CHECK_ARG(n_edges == 0 || (dst_of_edge && grad_pre));
    return dispatch_val_idx(val_dtype, idx_dtype, "gat_fused_csr_backward", [&](auto tv, auto ti) {
        return gat_bwd_typed<decltype(tv), decltype(ti)>(rowptr, col, dst_of_edge, rowptr_t, col_t, t2csr, xh, a_src,
                                                         a_dst, row_max, row_den, out, grad_out, grad_pre, rowdot,
                                                         grad_xh, grad_a_src, grad_a_dst, n_rows, n_src, n_edges, heads,
                                                         chan, slope, plan, static_cast<cudaStream_t>(stream));
    });
}
