// attention.cu -- fused edge-softmax attention + weighted aggregation over a destination-sorted CSR, forward
// and backward, for the three score functions of the reference's attention convolutions:
//
//   ATTN_GAT    s_e,h = leaky_relu(a_src[j,h] + a_dst[i,h] (+ a_edge[e,h]))        GATConv     gat_conv.py:387-409
//   ATTN_GATV2  s_e,h = sum_c att[h,c] leaky_relu(x_l[j,h,c] + x_r[i,h,c])         GATv2Conv   gatv2_conv.py:358-378
//   ATTN_DOT    s_e,h = scale * <q[i,h,:], k[j,h,:]>                               TransformerConv transformer_conv.py:263-275
//
//   alpha = softmax over the in-edges of i (utils/_softmax.py:82-88: exp(s - max) / (sum + 1e-16)),
//   out[i,h,:] = sum_e alpha_e,h v[j,h,:]        (v = xh / x_l / value rows)
//
// The reference runs ~12 kernels and materialises three [E,H,C] tensors; here every pass reads each gathered row
// once with 128-bit loads and nothing of size E x H x C is ever written.
//
// Mapping.  One WARP per work item (a CSR row, or one 512-edge chunk of a hub row -- the plan of csr_reduce.cuh).
// A row of H*C elements is cut into 16-byte vectors; G = next power of two >= #vectors lanes cover it (VPL = 2
// vectors per lane above 32 vectors), and the S = 32/G lane groups of the warp walk DIFFERENT EDGES OF THE SAME ROW
// (edge e0 + u*S + sub), so a warp never idles on the shorter of two unrelated power-law rows; their partial
// (max, sum, accumulator) states are merged by shuffles at the end with the usual exp(m - M) rescaling.  A head
// spans LPH = C / (elements per vector) neighbouring lanes; per-head dot products (GATv2 / dot scores, and
// <grad_out, v> in the backward) are reduced over those lanes with xor-shuffles.
//
// Backward, two sweeps, attention recomputed from the saved per-(row, head) max and denominator:
//   destination sweep (CSR):  D[i,h] = <g[i,h,:], out[i,h,:]> in registers, then per edge
//        gs_e,h = alpha_e,h (<g[i,h,:], v[j,h,:]> - D[i,h])         (softmax backward)
//        GAT:   gp = gs * leaky'(pre);  grad_a_dst[i,h] += gp;  pair[e,h] = (alpha, gp)
//        GATv2: grad_x_r[i,h,c] += gs att[h,c] leaky'(z);  grad_att[h,c] += gs leaky(z);  pair = (alpha, gs)
//        DOT:   grad_q[i,h,:] += gs scale k[j,h,:];  pair = (alpha, gs scale)
//   source sweep (transposed CSR, t2csr[e] = CSR slot of transposed slot e):
//        grad_v[j,h,:] = sum_e alpha_e g[d_e,h,:]  (+ GATv2: gs att leaky'(z));  GAT: grad_a_src[j,h] = sum gp;
//        DOT: grad_k[j,h,:] = sum_e gs' q[d_e,h,:]
//   `pair` ([E, H, 2] fp32, CSR order) is the only per-edge scratch: 64 B per edge at H = 8, one 64-byte gather
//   per edge in the source sweep instead of re-gathering a_dst / max / den and recomputing exp.
// HBM-bound; algorithmic bytes per edge (DESIGN.md): forward H*C*s (+ H*C*s for DOT's key row) + H*4 (GAT a_src)
// + idx; destination sweep the same + H*8 (pair write); source sweep H*C*s (g row) (+ H*C*s for GATv2 x_r / DOT q)
// + H*8 (pair) + 2 idx.
#include "csr_reduce.cuh"

namespace b200mp {

enum { ATTN_GAT = 0, ATTN_GATV2 = 1, ATTN_DOT = 2 };

int get_option_attn_staged();   // b200mp_set_option("attn_staged", 0 | 1): cp.async-staged forward (default 1)

constexpr int kAttnT = 128;   // 4 warps = 4 work items per CTA

struct AttnArgs {
    const char* v;            // value rows   [n_src, *]  (GAT xh, GATv2 x_l, DOT value)
    const char* k;            // DOT key rows [n_src, *]
    const char* q;            // GATv2 x_r / DOT query rows [n_dst, *]
    const float* s_src;       // GAT a_src [n_src, H]
    const float* s_dst;       // GAT a_dst [n_dst, H]
    const float* att;         // GATv2 att [H*C]
    const float* s_edge;      // GAT optional additive score [E, H] in CSR order (edge_dim)
    const char* ee;           // GATv2 / DOT optional per-edge feature rows [E, H*C] in CSR order (edge_dim): GATv2 adds them
                              // inside the leaky_relu (gatv2_conv.py:358-360), DOT to the key AND the value (transformer_conv.py:258-272)
    char* grad_ee;            // backward: their gradient [E, H*C] (written by the destination sweep, read by GATv2's source sweep)
    size_t v_stride, k_stride, q_stride;   // row strides in BYTES (k and v may be halves of one [N, 2HC] matrix)
    int heads, chan, n_vec, lph;
    float slope, scale;
    // attention dropout (gat_conv.py:404 `alpha = F.dropout(alpha, p, training)`): edge e, head h is dropped when
    // hash(seed, e * H + h) < thresh; kept coefficients are scaled by 1 / (1 - p).  thresh = 0: no dropout.
    uint32_t drop_thresh;
    float drop_scale;
    unsigned long long drop_seed;
};

// The same (edge, head) decision in the forward and in both backward sweeps: counter-based (splitmix64 of the CSR slot
// and head), no state, no [E, H] mask tensor.  torch's Philox stream cannot be reproduced from inside a fused sweep;
// tests compare against the unfused formula with THIS mask (read back through the returned attention coefficients).
__device__ __forceinline__ float drop_factor(const AttnArgs& a, int64_t e, int head) {
    if (a.drop_thresh == 0u) return 1.0f;
    unsigned long long z = a.drop_seed + static_cast<unsigned long long>(e * a.heads + head) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return static_cast<uint32_t>(z >> 32) >= a.drop_thresh ? a.drop_scale : 0.0f;
}

__device__ __forceinline__ float leaky_f(float v, float slope) { return v > 0.0f ? v : v * slope; }

// e^x as ONE multiply + ONE MUFU (ex2.approx: max relative error 2^-22.5, far inside the 1e-5 bar): the sweeps execute
// two exponentials per edge and lane, and libm's expf costs ~8 issue slots each on kernels that are issue/latency bound.
__device__ __forceinline__ float fexp(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
    return y;
}

__device__ __forceinline__ float head_sum(float v, int lph) {
    for (int o = lph >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// merge (m, s) softmax states: returns the two rescale factors
__device__ __forceinline__ void merge_ms(float m1, float m2, float& M, float& c1, float& c2) {
    M = fmaxf(m1, m2);
    c1 = (m1 == -__builtin_inff()) ? 0.0f : fexp(m1 - M);
    c2 = (m2 == -__builtin_inff()) ? 0.0f : fexp(m2 - M);
}

// ------------------------------------------------------------------------------------------------ forward
// STAGED (VPL == 1, G >= 8): the row vectors (and GAT's a_src scalars) of iteration t + 1 are in flight as cp.async
// copies into lane-private shared-memory slots while iteration t is computed -- twice the rows in flight per warp at the
// same register budget (the sweeps are latency-bound: most stalls wait on the gathered rows).
// BT = threads per CTA.  32 (one warp = one work item per CTA) for the staged kernels: a 4-warp CTA holds its slots until
// the longest of its four power-law rows is done, which wastes occupancy.
// VAR: 0 = rows gathered into registers, 1 = STAGED (cp.async slots), 2 = EDGE (register form + per-edge feature rows a.ee).
template <typename T, typename I, int G, int VPL, int MODE, int VAR = 0, int BT = kAttnT>
__global__ void __launch_bounds__(BT, (VPL == 1 ? (VAR == 2 ? 6 : 8) : 5) * (kAttnT / BT))       // <= 64 registers: 32 warps / SM
attn_fwd_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AttnArgs a, T* __restrict__ out,
                float* __restrict__ row_max, float* __restrict__ row_den, int64_t n_rows, LongRowPlan plan,
                float* __restrict__ part_ms) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int S = 32 / G;
    constexpr int UNR = VPL == 1 ? 4 : 2;
    constexpr bool STAGED = VAR == 1, EDGE = VAR == 2 && MODE != ATTN_GAT;
    const int lane = threadIdx.x & 31;
    const int lig = lane & (G - 1);
    const int sub = lane / G;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) return;   // warp-uniform

    int head[VPL];
    bool valid[VPL];
    float sd[VPL], m[VPL], s[VPL], acc[VPL][EPV], qv[VPL][EPV], av[VPL][EPV];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int v = lig + k * G;
        valid[k] = v < a.n_vec;
        head[k] = valid[k] ? (v * EPV) / a.chan : 0;
        m[k] = -__builtin_inff();
        s[k] = 0.0f;
        sd[k] = 0.0f;
#pragma unroll
        for (int i = 0; i < EPV; ++i) acc[k][i] = qv[k][i] = av[k][i] = 0.0f;
        if (!valid[k]) continue;
        if (MODE == ATTN_GAT) sd[k] = __ldg(a.s_dst + row * a.heads + head[k]);
        if (MODE != ATTN_GAT) ElemTraits<T>::unpack(ldg_row16(a.q + static_cast<size_t>(row) * a.q_stride + static_cast<size_t>(v) * 16), qv[k]);
        if (MODE == ATTN_GATV2) {
#pragma unroll
            for (int i = 0; i < EPV; ++i) av[k][i] = __ldg(a.att + v * EPV + i);
        }
    }

    if constexpr (STAGED) {
        static_assert(VPL == 1 && S * UNR <= 32, "staged path: one vector per lane, an iteration inside one index batch");
        extern __shared__ __align__(16) unsigned char attn_stage[];
        constexpr int D = 2;                                        // slots: iteration t and t + 1
        constexpr int NV = MODE == ATTN_DOT ? 2 : 1;                // value (+ key) vector per edge
        constexpr int PER = S * UNR;                                // edges per iteration of the warp
        unsigned char* vslots = attn_stage + static_cast<size_t>(threadIdx.x) * 16;
        float* sslots = reinterpret_cast<float*>(attn_stage + static_cast<size_t>(D) * UNR * NV * BT * 16) + threadIdx.x;
        auto vslot = [&](int d, int u, int v) { return vslots + static_cast<size_t>((d * UNR + u) * NV + v) * (BT * 16); };
        auto sslot = [&](int d, int u) { return sslots + (d * UNR + u) * BT; };
        const int deg = static_cast<int>(end - begin);
        const int n_it = (deg + PER - 1) / PER;
        const size_t off = static_cast<size_t>(lig) * 16;
        int cb = 0;                                                 // index batch held in c0 (c1 = the next one)
        I c0 = (lane < deg) ? ldg_idx(col + begin + lane) : I(0);
        I c1 = (32 + lane < deg) ? ldg_idx(col + begin + 32 + lane) : I(0);
        auto issue = [&](int t) {
            const int d = t & (D - 1);
            const I creg = ((t * PER) >> 5) == cb ? c0 : c1;        // warp-uniform choice
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int j = t * PER + u * S + sub;
                const int64_t c = static_cast<int64_t>(__shfl_sync(0xffffffffu, creg, j & 31));
                if (j < deg && valid[0]) {
                    cp_async16(vslot(d, u, 0), a.v + static_cast<size_t>(c) * a.v_stride + off);
                    if (MODE == ATTN_DOT) cp_async16(vslot(d, u, 1), a.k + static_cast<size_t>(c) * a.k_stride + off);
                    if (MODE == ATTN_GAT) cp_async4(sslot(d, u), a.s_src + c * a.heads + head[0]);
                }
            }
            cp_async_commit();
        };
        // invariant: issue(t) needs index batch (t * PER) >> 5 in {cb, cb + 1} (PER divides 32, so an iteration never
        // straddles a batch); once the issue stream has moved on to batch cb + 1, batch cb is dead: rotate and fetch
        // batch cb + 2, a whole batch before it is needed
        if (n_it > 0) issue(0);
        for (int t = 0; t < n_it; ++t) {
            if (t + 1 < n_it) {
                issue(t + 1);
                if ((((t + 1) * PER) >> 5) > cb) {
                    c0 = c1;
                    ++cb;
                    c1 = ((cb + 1) * 32 + lane < deg) ? ldg_idx(col + begin + (cb + 1) * 32 + lane) : I(0);
                }
            } else {
                cp_async_commit();
            }
            cp_async_wait<1>();
            const int d = t & (D - 1);
            if constexpr (MODE == ATTN_GAT) {
                // GAT scores need no feature data: take the stage's UNR logits first, move the running max ONCE and rescale
                // the accumulators once per stage instead of once per edge (the sweep is issue-bound after the staging)
                float lg[UNR];
                float mb = m[0];
                bool any = false;
#pragma unroll
                for (int u = 0; u < UNR; ++u) {
                    const int j = t * PER + u * S + sub;
                    lg[u] = -__builtin_inff();
                    if (j < deg && valid[0]) {
                        float sc = *sslot(d, u);
                        if (a.s_edge) sc += __ldg(a.s_edge + (begin + j) * a.heads + head[0]);
                        lg[u] = leaky_f(sc + sd[0], a.slope);
                        mb = fmaxf(mb, lg[u]);
                        any = true;
                    }
                }
                if (any) {                                          // (a lane group whose edges are exhausted keeps m = -inf)
                    const float rs = fexp(m[0] - mb);               // 0 on the first stage (m = -inf)
                    s[0] *= rs;
#pragma unroll
                    for (int i = 0; i < EPV; ++i) acc[0][i] *= rs;
                    m[0] = mb;
#pragma unroll
                    for (int u = 0; u < UNR; ++u) {
                        const int j = t * PER + u * S + sub;
                        if (j < deg) {
                            float f[EPV];
                            ElemTraits<T>::unpack(*reinterpret_cast<const Vec16*>(vslot(d, u, 0)), f);
                            const float p = fexp(lg[u] - mb);
                            s[0] += p;                              // the softmax denominator ignores dropout
                            const float pk = p * drop_factor(a, begin + j, head[0]);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) acc[0][i] = fmaf(pk, f[i], acc[0][i]);
                        }
                    }
                }
            } else {
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int j = t * PER + u * S + sub;
                const bool ev = j < deg;
                float f[EPV], l = 0.0f;
                if (ev && valid[0]) {
                    ElemTraits<T>::unpack(*reinterpret_cast<const Vec16*>(vslot(d, u, 0)), f);
                    if (MODE == ATTN_GAT) {
                        float sc = *sslot(d, u);
                        if (a.s_edge) sc += __ldg(a.s_edge + (begin + j) * a.heads + head[0]);
                        l = leaky_f(sc + sd[0], a.slope);
                    }
                    if (MODE == ATTN_GATV2) {
#pragma unroll
                        for (int i = 0; i < EPV; ++i) l = fmaf(av[0][i], leaky_f(f[i] + qv[0][i], a.slope), l);
                    }
                    if (MODE == ATTN_DOT) {
                        float kf[EPV];
                        ElemTraits<T>::unpack(*reinterpret_cast<const Vec16*>(vslot(d, u, 1)), kf);
#pragma unroll
                        for (int i = 0; i < EPV; ++i) l = fmaf(qv[0][i], kf[i], l);
                    }
                }
                if (MODE != ATTN_GAT) {
                    l = head_sum(l, a.lph);
                    if (MODE == ATTN_DOT) l *= a.scale;
                }
                if (ev && valid[0]) {
                    const float mn = fmaxf(m[0], l);
                    const float rs = fexp(m[0] - mn);
                    const float p = fexp(l - mn);
                    s[0] = fmaf(s[0], rs, p);                           // the softmax denominator ignores dropout
                    const float pk = p * drop_factor(a, begin + j, head[0]);
#pragma unroll
                    for (int i = 0; i < EPV; ++i) acc[0][i] = fmaf(acc[0][i], rs, pk * f[i]);
                    m[0] = mn;
                }
            }
            }
        }
        cp_async_wait<0>();
    } else {
    // Column indices are loaded by the whole warp, 32 edges at a time (coalesced, one batch ahead of the row loads so
    // the index latency is off the critical path) and handed to the lane groups by shuffle.
    I c_next = (begin + lane < end) ? ldg_idx(col + begin + lane) : I(0);
    for (int64_t b0 = begin; b0 < end; b0 += 32) {
        const I c_cur = c_next;
        const int nb = static_cast<int>(end - b0 < 32 ? end - b0 : 32);
        c_next = (b0 + 32 + lane < end) ? ldg_idx(col + b0 + 32 + lane) : I(0);
        for (int j0 = 0; j0 < nb; j0 += S * UNR) {
            Vec16 vb[UNR][VPL], kb[UNR][VPL], eb[UNR][VPL];
            float sc[UNR][VPL];
            bool ev[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int j = j0 + u * S + sub;
                ev[u] = j < nb;
                const int64_t c = static_cast<int64_t>(__shfl_sync(0xffffffffu, c_cur, j & 31));
                if (ev[u]) {
                    const int64_t e = b0 + j;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (!valid[k]) continue;
                        const size_t off = static_cast<size_t>(lig + k * G) * 16;
                        vb[u][k] = ldg_row16(a.v + static_cast<size_t>(c) * a.v_stride + off);
                        if (EDGE) eb[u][k] = ldg_stream16(a.ee + static_cast<size_t>(e) * (static_cast<size_t>(a.n_vec) * 16) + off);
                        if (MODE == ATTN_DOT) kb[u][k] = ldg_row16(a.k + static_cast<size_t>(c) * a.k_stride + off);
                        if (MODE == ATTN_GAT) {
                            sc[u][k] = __ldg(a.s_src + c * a.heads + head[k]);
                            if (a.s_edge) sc[u][k] += __ldg(a.s_edge + e * a.heads + head[k]);
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                float f[VPL][EPV], l[VPL];
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    l[k] = 0.0f;
                    if (ev[u] && valid[k]) {
                        float ef[EPV];
                        ElemTraits<T>::unpack(vb[u][k], f[k]);
                        if (EDGE) {
                            ElemTraits<T>::unpack(eb[u][k], ef);
                        } else {
#pragma unroll
                            for (int i = 0; i < EPV; ++i) ef[i] = 0.0f;
                        }
                        if (MODE == ATTN_GAT) l[k] = leaky_f(sc[u][k] + sd[k], a.slope);
                        if (MODE == ATTN_GATV2) {
#pragma unroll
                            for (int i = 0; i < EPV; ++i) l[k] = fmaf(av[k][i], leaky_f(f[k][i] + qv[k][i] + ef[i], a.slope), l[k]);
                        }
                        if (MODE == ATTN_DOT) {
                            float kf[EPV];
                            ElemTraits<T>::unpack(kb[u][k], kf);
#pragma unroll
                            for (int i = 0; i < EPV; ++i) {
                                l[k] = fmaf(qv[k][i], kf[i] + ef[i], l[k]);      // key_j + e
                                f[k][i] += ef[i];                                // value_j + e
                            }
                        }
                    }
                }
                if (MODE != ATTN_GAT) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        l[k] = head_sum(l[k], a.lph);                   // executed by the whole warp
                        if (MODE == ATTN_DOT) l[k] *= a.scale;
                    }
                }
                if (ev[u]) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (!valid[k]) continue;
                        const float mn = fmaxf(m[k], l[k]);
                        const float rs = fexp(m[k] - mn);               // 0 on the first edge (m = -inf)
                        const float p = fexp(l[k] - mn);
                        s[k] = fmaf(s[k], rs, p);
                        const float pk = p * drop_factor(a, b0 + j0 + u * S + sub, head[k]);
#pragma unroll
                        for (int i = 0; i < EPV; ++i) acc[k][i] = fmaf(acc[k][i], rs, pk * f[k][i]);
                        m[k] = mn;
                    }
                }
            }
        }
    }
    }   // !STAGED
    // merge the S lane groups (they walked disjoint edges of the same row)
#pragma unroll
    for (int o = G; o < 32; o <<= 1) {
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const float m2 = __shfl_xor_sync(0xffffffffu, m[k], o);
            const float s2 = __shfl_xor_sync(0xffffffffu, s[k], o);
            float M, c1, c2;
            merge_ms(m[k], m2, M, c1, c2);
            s[k] = s[k] * c1 + s2 * c2;
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                const float a2 = __shfl_xor_sync(0xffffffffu, acc[k][i], o);
                acc[k][i] = acc[k][i] * c1 + a2 * c2;
            }
            m[k] = M;
        }
    }
    if (sub != 0) return;
    const size_t row_bytes = static_cast<size_t>(a.n_vec) * 16;
    if (is_chunk) {
        float* pbase = plan.partials + static_cast<size_t>(item) * a.n_vec * EPV;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (!valid[k]) continue;
            const int v = lig + k * G;
            float* p = pbase + static_cast<size_t>(v) * EPV;
#pragma unroll
            for (int i = 0; i < EPV; ++i) p[i] = acc[k][i];
            if ((v * EPV) % a.chan == 0) {
                part_ms[(item * a.heads + head[k]) * 2 + 0] = m[k];
                part_ms[(item * a.heads + head[k]) * 2 + 1] = s[k];
            }
        }
        return;
    }
    char* ob = reinterpret_cast<char*>(out) + static_cast<size_t>(row) * row_bytes;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        if (!valid[k]) continue;
        const int v = lig + k * G;
        const float den = s[k] + 1e-16f;                           // _softmax.py:87 "+ 1e-16"
        float f[EPV];
#pragma unroll
        for (int i = 0; i < EPV; ++i) f[i] = (end > begin) ? acc[k][i] / den : 0.0f;
        stg_stream16(ob + static_cast<size_t>(v) * 16, ElemTraits<T>::pack(f));
        if ((v * EPV) % a.chan == 0) {
            row_max[row * a.heads + head[k]] = (end > begin) ? m[k] : 0.0f;
            row_den[row * a.heads + head[k]] = den;
        }
    }
}

// Merge the chunk states of every hub row: M = max_c m_c; S = sum_c s_c e^{m_c-M}; out = sum_c acc_c e^{m_c-M} / (S + 1e-16).
// One CTA per hub row; the chunks are dealt to blockDim / W thread slices (W = features padded to a power of two), every
// slice merges its chunks online, the slices are folded through shared memory: the largest hub of the products-shaped
// graph has 5566 chunks, which a single thread per feature used to walk serially (1.9 ms of an 18 ms forward).
constexpr int kCombineT = 1024;
template <typename T>
__global__ void __launch_bounds__(kCombineT)
attn_combine_kernel(T* __restrict__ out, float* __restrict__ row_max, float* __restrict__ row_den, int heads, int chan,
                    LongRowPlan plan, const float* __restrict__ part_ms, int W) {
    __shared__ float sm[3 * kCombineT];
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int64_t hc = static_cast<int64_t>(heads) * chan;
    const int n_slices = kCombineT / W;
    const int slice = threadIdx.x / W;
    for (int64_t f0 = 0; f0 < hc; f0 += W) {
        const int64_t f = f0 + (threadIdx.x % W);
        const bool fv = f < hc && slice < n_slices;
        const int h = fv ? static_cast<int>(f / chan) : 0;
        float M = -__builtin_inff(), S = 0.0f, acc = 0.0f;
        if (fv) {
            for (int64_t c = c0 + slice; c < c1; c += n_slices) {
                const float mc = part_ms[(c * heads + h) * 2], sc = part_ms[(c * heads + h) * 2 + 1];
                const float Mn = fmaxf(M, mc);
                const float r0 = (M == -__builtin_inff()) ? 0.0f : fexp(M - Mn);
                const float r1 = (mc == -__builtin_inff()) ? 0.0f : fexp(mc - Mn);
                S = S * r0 + sc * r1;
                acc = acc * r0 + plan.partials[c * hc + f] * r1;
                M = Mn;
            }
        }
        sm[threadIdx.x] = M;
        sm[kCombineT + threadIdx.x] = S;
        sm[2 * kCombineT + threadIdx.x] = acc;
        __syncthreads();
        if (fv && slice == 0) {
            for (int sl = 1; sl < n_slices; ++sl) {
                const int t = sl * W + (threadIdx.x % W);
                const float m2 = sm[t], s2 = sm[kCombineT + t], a2 = sm[2 * kCombineT + t];
                float Mn, r0, r1;
                merge_ms(M, m2, Mn, r0, r1);
                S = S * r0 + s2 * r1;
                acc = acc * r0 + a2 * r1;
                M = Mn;
            }
            const float den = S + 1e-16f;
            out[row * hc + f] = ElemTraits<T>::from_float(acc / den);
            if (f % chan == 0) {
                row_max[row * heads + h] = M;
                row_den[row * heads + h] = den;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ backward, destination sweep
// Also the alpha writer of the forward (ALPHA_ONLY: alpha[e,h] from the saved statistics, nothing else).
template <typename T, typename I, int G, int VPL, int MODE, bool ALPHA_ONLY, int VAR = 0>      // VAR: see attn_fwd_kernel
__global__ void __launch_bounds__(kAttnT)
attn_bwd_dst_kernel(const I* __restrict__ rowptr, const I* __restrict__ col, AttnArgs a, const float* __restrict__ row_max,
                    const float* __restrict__ row_den, const T* __restrict__ out, const T* __restrict__ grad_out,
                    float* __restrict__ pair, float* __restrict__ alpha_out, T* __restrict__ grad_q,
                    float* __restrict__ grad_s_dst, float* __restrict__ gatt_part, int64_t n_rows, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int S = 32 / G;
    constexpr int UNR = VPL == 1 ? 4 : 2;
    constexpr bool STAGED = VAR == 1, EDGE = VAR == 2 && MODE != ATTN_GAT;
    const int lane = threadIdx.x & 31;
    const int lig = lane & (G - 1);
    const int sub = lane / G;
    const int64_t n_items = plan.n_chunks + n_rows;
    const int64_t warps_total = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
    const size_t row_bytes = static_cast<size_t>(a.n_vec) * 16;

    int head[VPL];
    bool valid[VPL];
    float av[VPL][EPV], gatt[VPL][EPV];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int v = lig + k * G;
        valid[k] = v < a.n_vec;
        head[k] = valid[k] ? (v * EPV) / a.chan : 0;
#pragma unroll
        for (int i = 0; i < EPV; ++i) {
            gatt[k][i] = 0.0f;
            av[k][i] = (MODE == ATTN_GATV2 && valid[k]) ? __ldg(a.att + v * EPV + i) : 0.0f;
        }
    }

    // GATv2 accumulates grad_att over every edge: grid-stride loop over the items (other modes: one item per warp)
    for (int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; item < n_items; item += warps_total) {
        int64_t row, begin, end;
        bool is_chunk;
        if (!decode_item(item, rowptr, n_rows, plan, row, begin, end, is_chunk)) continue;

        float sd[VPL], mrow[VPL], inv_den[VPL], D[VPL], gv[VPL][EPV], qv[VPL][EPV], gq[VPL][EPV], gsd[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int v = lig + k * G;
            sd[k] = mrow[k] = inv_den[k] = D[k] = gsd[k] = 0.0f;
#pragma unroll
            for (int i = 0; i < EPV; ++i) gv[k][i] = qv[k][i] = gq[k][i] = 0.0f;
            if (!valid[k]) continue;
            mrow[k] = __ldg(row_max + row * a.heads + head[k]);
            inv_den[k] = 1.0f / __ldg(row_den + row * a.heads + head[k]);
            if (MODE == ATTN_GAT) sd[k] = __ldg(a.s_dst + row * a.heads + head[k]);
            if (MODE != ATTN_GAT) ElemTraits<T>::unpack(ldg_row16(a.q + static_cast<size_t>(row) * a.q_stride + static_cast<size_t>(v) * 16), qv[k]);
            if (!ALPHA_ONLY) {
                float of[EPV];
                ElemTraits<T>::unpack(ldg_row16(reinterpret_cast<const char*>(grad_out) + static_cast<size_t>(row) * row_bytes + static_cast<size_t>(v) * 16), gv[k]);
                ElemTraits<T>::unpack(ldg_row16(reinterpret_cast<const char*>(out) + static_cast<size_t>(row) * row_bytes + static_cast<size_t>(v) * 16), of);
#pragma unroll
                for (int i = 0; i < EPV; ++i) D[k] = fmaf(gv[k][i], of[i], D[k]);
            }
        }
        if (!ALPHA_ONLY) {
#pragma unroll
            for (int k = 0; k < VPL; ++k) D[k] = head_sum(D[k], a.lph);
        }

        // one edge of this lane group: vbv / kbv = the gathered value (/ key) vectors, scv = GAT's a_src(+a_edge) scalars
        // ebv (EDGE): the edge's feature vectors -- GATv2: z = x_l[j] + x_r[i] + e; DOT: key_j + e and value_j + e
        auto process = [&](int64_t e, bool evu, const Vec16* vbv, const Vec16* kbv, const float* scv, const Vec16* ebv) {
            float f[VPL][EPV], kf[VPL][EPV], ef[VPL][EPV], l[VPL], dot[VPL];
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                l[k] = dot[k] = 0.0f;
#pragma unroll
                for (int i = 0; i < EPV; ++i) f[k][i] = kf[k][i] = ef[k][i] = 0.0f;
                if (evu && valid[k]) {
                    if (!ALPHA_ONLY || MODE == ATTN_GATV2) ElemTraits<T>::unpack(vbv[k], f[k]);
                    if (EDGE) ElemTraits<T>::unpack(ebv[k], ef[k]);
                    if (MODE == ATTN_GAT) l[k] = scv[k] + sd[k];                         // pre-activation
                    if (MODE == ATTN_GATV2) {
#pragma unroll
                        for (int i = 0; i < EPV; ++i) l[k] = fmaf(av[k][i], leaky_f(f[k][i] + qv[k][i] + ef[k][i], a.slope), l[k]);
                    }
                    if (MODE == ATTN_DOT) {
                        ElemTraits<T>::unpack(kbv[k], kf[k]);
#pragma unroll
                        for (int i = 0; i < EPV; ++i) {
                            kf[k][i] += ef[k][i];                                        // key_j + e
                            f[k][i] += ef[k][i];                                         // value_j + e
                            l[k] = fmaf(qv[k][i], kf[k][i], l[k]);
                        }
                    }
                    if (!ALPHA_ONLY) {
#pragma unroll
                        for (int i = 0; i < EPV; ++i) dot[k] = fmaf(gv[k][i], f[k][i], dot[k]);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (MODE != ATTN_GAT) {
                    l[k] = head_sum(l[k], a.lph);
                    if (MODE == ATTN_DOT) l[k] *= a.scale;
                }
                if (!ALPHA_ONLY) dot[k] = head_sum(dot[k], a.lph);
            }
            if (!evu) return;
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (!valid[k]) continue;
                const float score = MODE == ATTN_GAT ? leaky_f(l[k], a.slope) : l[k];
                const float alpha = fexp(score - mrow[k]) * inv_den[k];
                const bool first = ((lig + k * G) * EPV) % a.chan == 0;
                const float keep = drop_factor(a, e, head[k]);           // 0 or 1 / (1 - p); 1 without dropout
                if (ALPHA_ONLY) {
                    if (first) alpha_out[e * a.heads + head[k]] = alpha * keep;    // the reference returns the dropped alpha
                    continue;
                }
                // out = sum_e keep_e alpha_e v_e, D = <g, out>:  d/d score_e = alpha_e (keep_e <g, v_e> - D)
                float gs = alpha * (keep * dot[k] - D[k]);
                if (MODE == ATTN_GAT) {
                    gs *= (l[k] > 0.0f ? 1.0f : a.slope);
                    if (first) gsd[k] += gs;
                }
                float ge[EPV];                                           // EDGE: gradient of the edge's feature vector
                if (MODE == ATTN_GATV2) {
#pragma unroll
                    for (int i = 0; i < EPV; ++i) {
                        const float z = f[k][i] + qv[k][i] + ef[k][i];
                        ge[i] = gs * av[k][i] * (z > 0.0f ? 1.0f : a.slope);
                        gq[k][i] += ge[i];
                        gatt[k][i] = fmaf(gs, leaky_f(z, a.slope), gatt[k][i]);
                    }
                }
                if (MODE == ATTN_DOT) {
                    gs *= a.scale;
#pragma unroll
                    for (int i = 0; i < EPV; ++i) {
                        gq[k][i] = fmaf(gs, kf[k][i], gq[k][i]);
                        ge[i] = fmaf(alpha * keep, gv[k][i], gs * qv[k][i]);      // through the value and through the key
                    }
                }
                if (EDGE)
                    stg_stream16(a.grad_ee + static_cast<size_t>(e) * row_bytes + static_cast<size_t>(lig + k * G) * 16, ElemTraits<T>::pack(ge));
                if (first) *reinterpret_cast<float2*>(pair + (e * a.heads + head[k]) * 2) = make_float2(alpha * keep, gs);
            }
        };

        if constexpr (STAGED) {
            // cp.async-staged gather (see attn_fwd_kernel): iteration t + 1 in flight in lane-private shared-memory slots
            static_assert(VPL == 1 && S * UNR <= 32, "staged path: one vector per lane");
            extern __shared__ __align__(16) unsigned char attn_stage[];
            constexpr int D = 2, NV = MODE == ATTN_DOT ? 2 : 1, PER = S * UNR;
            unsigned char* vslots = attn_stage + static_cast<size_t>(threadIdx.x) * 16;
            float* sslots = reinterpret_cast<float*>(attn_stage + static_cast<size_t>(D) * UNR * NV * kAttnT * 16) + threadIdx.x;
            auto vslot = [&](int d, int u, int v) { return vslots + static_cast<size_t>((d * UNR + u) * NV + v) * (kAttnT * 16); };
            auto sslot = [&](int d, int u) { return sslots + (d * UNR + u) * kAttnT; };
            const int deg = static_cast<int>(end - begin);
            const int n_it = (deg + PER - 1) / PER;
            const size_t off = static_cast<size_t>(lig) * 16;
            int cb = 0;
            I c0 = (lane < deg) ? ldg_idx(col + begin + lane) : I(0);
            I c1 = (32 + lane < deg) ? ldg_idx(col + begin + 32 + lane) : I(0);
            auto issue = [&](int t) {
                const int d = t & (D - 1);
                const I creg = ((t * PER) >> 5) == cb ? c0 : c1;
#pragma unroll
                for (int u = 0; u < UNR; ++u) {
                    const int j = t * PER + u * S + sub;
                    const int64_t c = static_cast<int64_t>(__shfl_sync(0xffffffffu, creg, j & 31));
                    if (j < deg && valid[0]) {
                        if (!ALPHA_ONLY || MODE == ATTN_GATV2) cp_async16(vslot(d, u, 0), a.v + static_cast<size_t>(c) * a.v_stride + off);
                        if (MODE == ATTN_DOT) cp_async16(vslot(d, u, 1), a.k + static_cast<size_t>(c) * a.k_stride + off);
                        if (MODE == ATTN_GAT) cp_async4(sslot(d, u), a.s_src + c * a.heads + head[0]);
                    }
                }
                cp_async_commit();
            };
            if (n_it > 0) issue(0);
            for (int t = 0; t < n_it; ++t) {
                if (t + 1 < n_it) {
                    issue(t + 1);
                    if ((((t + 1) * PER) >> 5) > cb) {
                        c0 = c1;
                        ++cb;
                        c1 = ((cb + 1) * 32 + lane < deg) ? ldg_idx(col + begin + (cb + 1) * 32 + lane) : I(0);
                    }
                } else {
                    cp_async_commit();
                }
                cp_async_wait<1>();
                const int d = t & (D - 1);
#pragma unroll
                for (int u = 0; u < UNR; ++u) {
                    const int j = t * PER + u * S + sub;
                    const bool evu = j < deg;
                    const int64_t e = begin + j;
                    Vec16 v0 = {}, k0 = {};
                    float sc0 = 0.0f;
                    if (evu && valid[0]) {
                        if (!ALPHA_ONLY || MODE == ATTN_GATV2) v0 = *reinterpret_cast<const Vec16*>(vslot(d, u, 0));
                        if (MODE == ATTN_DOT) k0 = *reinterpret_cast<const Vec16*>(vslot(d, u, 1));
                        if (MODE == ATTN_GAT) {
                            sc0 = *sslot(d, u);
                            if (a.s_edge) sc0 += __ldg(a.s_edge + e * a.heads + head[0]);
                        }
                    }
                    process(e, evu, &v0, &k0, &sc0, nullptr);
                }
            }
            cp_async_wait<0>();
        } else {
        I c_next = (begin + lane < end) ? ldg_idx(col + begin + lane) : I(0);
        for (int64_t b0 = begin; b0 < end; b0 += 32) {
            const I c_cur = c_next;
            const int nb = static_cast<int>(end - b0 < 32 ? end - b0 : 32);
            c_next = (b0 + 32 + lane < end) ? ldg_idx(col + b0 + 32 + lane) : I(0);
            for (int j0 = 0; j0 < nb; j0 += S * UNR) {
                Vec16 vb[UNR][VPL], kb[UNR][VPL], eb[UNR][VPL];
                float sc[UNR][VPL];
                bool ev[UNR];
#pragma unroll
                for (int u = 0; u < UNR; ++u) {
                    const int jj = j0 + u * S + sub;
                    const int64_t e = b0 + jj;
                    ev[u] = jj < nb;
                    const int64_t c = static_cast<int64_t>(__shfl_sync(0xffffffffu, c_cur, jj & 31));
#pragma unroll
                    for (int k = 0; k < VPL; ++k) sc[u][k] = 0.0f;
                    if (ev[u]) {
#pragma unroll
                        for (int k = 0; k < VPL; ++k) {
                            if (!valid[k]) continue;
                            const size_t off = static_cast<size_t>(lig + k * G) * 16;
                            if (!ALPHA_ONLY || MODE == ATTN_GATV2) vb[u][k] = ldg_row16(a.v + static_cast<size_t>(c) * a.v_stride + off);
                            if (EDGE) eb[u][k] = ldg_stream16(a.ee + static_cast<size_t>(e) * row_bytes + off);
                            if (MODE == ATTN_DOT) kb[u][k] = ldg_row16(a.k + static_cast<size_t>(c) * a.k_stride + off);
                            if (MODE == ATTN_GAT) {
                                sc[u][k] = __ldg(a.s_src + c * a.heads + head[k]);
                                if (a.s_edge) sc[u][k] += __ldg(a.s_edge + e * a.heads + head[k]);
                            }
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UNR; ++u) process(b0 + j0 + u * S + sub, ev[u], vb[u], kb[u], sc[u], eb[u]);
            }
        }
        }   // !STAGED
        if (ALPHA_ONLY) continue;
        // sum the lane groups' per-row partial gradients
#pragma unroll
        for (int o = G; o < 32; o <<= 1) {
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (MODE == ATTN_GAT) gsd[k] += __shfl_xor_sync(0xffffffffu, gsd[k], o);
                if (MODE != ATTN_GAT) {
#pragma unroll
                    for (int i = 0; i < EPV; ++i) gq[k][i] += __shfl_xor_sync(0xffffffffu, gq[k][i], o);
                }
            }
        }
        if (sub != 0) continue;
        if (MODE == ATTN_GAT) {
            // per-row (or per-chunk) sum of grad_pre; chunk partials are folded by attn_sum_combine_kernel
            float* dstp = is_chunk ? plan.partials + static_cast<size_t>(item) * a.heads : grad_s_dst + row * a.heads;
#pragma unroll
            for (int k = 0; k < VPL; ++k)
                if (valid[k] && ((lig + k * G) * EPV) % a.chan == 0) dstp[head[k]] = gsd[k];
        } else {
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                if (!valid[k]) continue;
                const int v = lig + k * G;
                if (is_chunk) {
                    float* p = plan.partials + (static_cast<size_t>(item) * a.n_vec + v) * EPV;
#pragma unroll
                    for (int i = 0; i < EPV; ++i) p[i] = gq[k][i];
                } else {
                    stg_stream16(reinterpret_cast<char*>(grad_q) + static_cast<size_t>(row) * row_bytes + static_cast<size_t>(v) * 16,
                                 ElemTraits<T>::pack(gq[k]));
                }
            }
        }
    }
    if (MODE == ATTN_GATV2 && !ALPHA_ONLY) {
        // fold grad_att: lane groups by shuffle, warps through shared memory, one partial row per CTA
        __shared__ float sm[kAttnT / 32][64 * 8];
#pragma unroll
        for (int o = G; o < 32; o <<= 1)
#pragma unroll
            for (int k = 0; k < VPL; ++k)
#pragma unroll
                for (int i = 0; i < EPV; ++i) gatt[k][i] += __shfl_xor_sync(0xffffffffu, gatt[k][i], o);
        const int w = threadIdx.x >> 5;
        if (sub == 0) {
#pragma unroll
            for (int k = 0; k < VPL; ++k)
                if (valid[k])
#pragma unroll
                    for (int i = 0; i < EPV; ++i) sm[w][(lig + k * G) * EPV + i] = gatt[k][i];
        }
        __syncthreads();
        const int hc = a.heads * a.chan;
        for (int f = threadIdx.x; f < hc; f += blockDim.x) {
            float t = 0.0f;
            for (int ww = 0; ww < kAttnT / 32; ++ww) t += sm[ww][f];
            gatt_part[static_cast<size_t>(blockIdx.x) * hc + f] = t;
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward, source sweep
template <typename T, typename I, int G, int VPL, int MODE, int VAR = 0, int BT = kAttnT>      // VAR: see attn_fwd_kernel
__global__ void __launch_bounds__(BT)          // no register cap: capping at 64 serialised the row loads (8.0 -> 14.8 ms)
attn_bwd_src_kernel(const I* __restrict__ rowptr_t, const I* __restrict__ col_t, const I* __restrict__ t2csr, AttnArgs a,
                    const T* __restrict__ grad_out, const float* __restrict__ pair, T* __restrict__ grad_v,
                    T* __restrict__ grad_k, float* __restrict__ grad_s_src, int64_t n_src, LongRowPlan plan) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    constexpr int S = 32 / G;
    constexpr int UNR = VPL == 1 ? 4 : 2;
    constexpr bool STAGED = VAR == 1, EDGE = VAR == 2 && MODE == ATTN_GATV2;   // (DOT: no edge term on this side)
    const int lane = threadIdx.x & 31;
    const int lig = lane & (G - 1);
    const int sub = lane / G;
    const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    int64_t row, begin, end;
    bool is_chunk;
    if (!decode_item(item, rowptr_t, n_src, plan, row, begin, end, is_chunk)) return;
    const size_t row_bytes = static_cast<size_t>(a.n_vec) * 16;
    const char* gb = reinterpret_cast<const char*>(grad_out);

    int head[VPL];
    bool valid[VPL];
    float accv[VPL][EPV], acck[VPL][EPV], xl[VPL][EPV], av[VPL][EPV], gss[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int v = lig + k * G;
        valid[k] = v < a.n_vec;
        head[k] = valid[k] ? (v * EPV) / a.chan : 0;
        gss[k] = 0.0f;
#pragma unroll
        for (int i = 0; i < EPV; ++i) accv[k][i] = acck[k][i] = xl[k][i] = av[k][i] = 0.0f;
        if (MODE == ATTN_GATV2 && valid[k]) {
            ElemTraits<T>::unpack(ldg_row16(a.v + static_cast<size_t>(row) * a.v_stride + static_cast<size_t>(v) * 16), xl[k]);
#pragma unroll
            for (int i = 0; i < EPV; ++i) av[k][i] = __ldg(a.att + v * EPV + i);
        }
    }
    // one out-edge: gv = the destination's gradient row vector, qv_ = its x_r / query row vector, pr = (alpha, grad_score)
    auto consume = [&](const Vec16* gv, const Vec16* qv_, const float2* pr) {
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (!valid[k]) continue;
            float g[EPV];
            ElemTraits<T>::unpack(gv[k], g);
            const float alpha = pr[k].x, gs = pr[k].y;
#pragma unroll
            for (int i = 0; i < EPV; ++i) accv[k][i] = fmaf(alpha, g[i], accv[k][i]);
            if (MODE == ATTN_GAT) gss[k] += gs;
            if (MODE != ATTN_GAT) {
                float qf[EPV];
                ElemTraits<T>::unpack(qv_[k], qf);
                if (MODE == ATTN_GATV2 && EDGE) {
                    // qv_ holds the edge's grad_ee row (= gs att leaky'(x_l + x_r + e), written by the destination sweep):
                    // the same quantity flows into x_l[j]
#pragma unroll
                    for (int i = 0; i < EPV; ++i) accv[k][i] += qf[i];
                } else if (MODE == ATTN_GATV2) {
#pragma unroll
                    for (int i = 0; i < EPV; ++i) accv[k][i] = fmaf(gs * av[k][i], ((xl[k][i] + qf[i]) > 0.0f ? 1.0f : a.slope), accv[k][i]);
                } else {
#pragma unroll
                    for (int i = 0; i < EPV; ++i) acck[k][i] = fmaf(gs, qf[i], acck[k][i]);
                }
            }
        }
    };
    if constexpr (STAGED) {
        static_assert(VPL == 1 && S * UNR <= 32, "staged path: one vector per lane");
        extern __shared__ __align__(16) unsigned char attn_stage[];
        constexpr int D = 2, NV = MODE == ATTN_GAT ? 1 : 2, PER = S * UNR;
        unsigned char* vslots = attn_stage + static_cast<size_t>(threadIdx.x) * 16;
        float2* pslots = reinterpret_cast<float2*>(attn_stage + static_cast<size_t>(D) * UNR * NV * BT * 16) + threadIdx.x;
        auto vslot = [&](int d, int u, int v) { return vslots + static_cast<size_t>((d * UNR + u) * NV + v) * (BT * 16); };
        auto pslot = [&](int d, int u) { return pslots + (d * UNR + u) * BT; };
        const int deg = static_cast<int>(end - begin);
        const int n_it = (deg + PER - 1) / PER;
        const size_t off = static_cast<size_t>(lig) * 16;
        int cb = 0;
        I d0 = 0, p0 = 0, d1 = 0, p1 = 0;
        if (lane < deg) { d0 = ldg_idx(col_t + begin + lane); p0 = ldg_idx(t2csr + begin + lane); }
        if (32 + lane < deg) { d1 = ldg_idx(col_t + begin + 32 + lane); p1 = ldg_idx(t2csr + begin + 32 + lane); }
        auto issue = [&](int t) {
            const int d = t & (D - 1);
            const bool cur = ((t * PER) >> 5) == cb;
            const I dreg = cur ? d0 : d1, preg = cur ? p0 : p1;
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int j = t * PER + u * S + sub;
                const int64_t dd = static_cast<int64_t>(__shfl_sync(0xffffffffu, dreg, j & 31));
                const int64_t pp = static_cast<int64_t>(__shfl_sync(0xffffffffu, preg, j & 31));
                if (j < deg && valid[0]) {
                    cp_async16(vslot(d, u, 0), gb + static_cast<size_t>(dd) * row_bytes + off);
                    if (MODE != ATTN_GAT) cp_async16(vslot(d, u, 1), a.q + static_cast<size_t>(dd) * a.q_stride + off);
                    cp_async8(pslot(d, u), reinterpret_cast<const float2*>(pair) + pp * a.heads + head[0]);
                }
            }
            cp_async_commit();
        };
        if (n_it > 0) issue(0);
        for (int t = 0; t < n_it; ++t) {
            if (t + 1 < n_it) {
                issue(t + 1);
                if ((((t + 1) * PER) >> 5) > cb) {
                    d0 = d1;
                    p0 = p1;
                    ++cb;
                    d1 = p1 = 0;
                    if ((cb + 1) * 32 + lane < deg) {
                        d1 = ldg_idx(col_t + begin + (cb + 1) * 32 + lane);
                        p1 = ldg_idx(t2csr + begin + (cb + 1) * 32 + lane);
                    }
                }
            } else {
                cp_async_commit();
            }
            cp_async_wait<1>();
            const int d = t & (D - 1);
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int j = t * PER + u * S + sub;
                if (j < deg && valid[0]) {
                    const Vec16 g0 = *reinterpret_cast<const Vec16*>(vslot(d, u, 0));
                    Vec16 q0 = {};
                    if (MODE != ATTN_GAT) q0 = *reinterpret_cast<const Vec16*>(vslot(d, u, 1));
                    const float2 pr0 = *pslot(d, u);
                    consume(&g0, &q0, &pr0);
                }
            }
        }
        cp_async_wait<0>();
    } else {
    I d_next = 0, p_next = 0;
    if (begin + lane < end) {
        d_next = ldg_idx(col_t + begin + lane);
        p_next = ldg_idx(t2csr + begin + lane);
    }
    for (int64_t b0 = begin; b0 < end; b0 += 32) {
        const I d_cur = d_next, p_cur = p_next;
        const int nb = static_cast<int>(end - b0 < 32 ? end - b0 : 32);
        d_next = p_next = 0;
        if (b0 + 32 + lane < end) {
            d_next = ldg_idx(col_t + b0 + 32 + lane);
            p_next = ldg_idx(t2csr + b0 + 32 + lane);
        }
        for (int j0 = 0; j0 < nb; j0 += S * UNR) {
            Vec16 gbuf[UNR][VPL], qb[UNR][VPL];
            float2 pr[UNR][VPL];
            bool ev[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int jj = j0 + u * S + sub;
                ev[u] = jj < nb;
                const int64_t d = static_cast<int64_t>(__shfl_sync(0xffffffffu, d_cur, jj & 31));
                const int64_t p = static_cast<int64_t>(__shfl_sync(0xffffffffu, p_cur, jj & 31));
                if (ev[u]) {
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        if (!valid[k]) continue;
                        const size_t off = static_cast<size_t>(lig + k * G) * 16;
                        gbuf[u][k] = ldg_row16(gb + static_cast<size_t>(d) * row_bytes + off);
                        if (EDGE) qb[u][k] = ldg_row16(a.grad_ee + static_cast<size_t>(p) * row_bytes + off);
                        else if (MODE != ATTN_GAT) qb[u][k] = ldg_row16(a.q + static_cast<size_t>(d) * a.q_stride + off);
                        pr[u][k] = __ldg(reinterpret_cast<const float2*>(pair) + p * a.heads + head[k]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u)
                if (ev[u]) consume(gbuf[u], qb[u], pr[u]);
        }
    }
    }   // !STAGED
#pragma unroll
    for (int o = G; o < 32; o <<= 1) {
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (MODE == ATTN_GAT) gss[k] += __shfl_xor_sync(0xffffffffu, gss[k], o);
#pragma unroll
            for (int i = 0; i < EPV; ++i) {
                accv[k][i] += __shfl_xor_sync(0xffffffffu, accv[k][i], o);
                if (MODE == ATTN_DOT) acck[k][i] += __shfl_xor_sync(0xffffffffu, acck[k][i], o);
            }
        }
    }
    if (sub != 0) return;
    // chunk partial layout per chunk: [H*C (grad_v) | H*C (grad_k, DOT) | H (grad_s_src, GAT)] fp32
    const size_t hc = static_cast<size_t>(a.n_vec) * EPV;
    const size_t pw = hc * (MODE == ATTN_DOT ? 2 : 1) + (MODE == ATTN_GAT ? a.heads : 0);
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        if (!valid[k]) continue;
        const int v = lig + k * G;
        const bool first = (v * EPV) % a.chan == 0;
        if (is_chunk) {
            float* p = plan.partials + static_cast<size_t>(item) * pw;
#pragma unroll
            for (int i = 0; i < EPV; ++i) p[static_cast<size_t>(v) * EPV + i] = accv[k][i];
            if (MODE == ATTN_DOT) {
#pragma unroll
                for (int i = 0; i < EPV; ++i) p[hc + static_cast<size_t>(v) * EPV + i] = acck[k][i];
            }
            if (MODE == ATTN_GAT && first) p[hc + head[k]] = gss[k];
        } else {
            stg_stream16(reinterpret_cast<char*>(grad_v) + static_cast<size_t>(row) * a.v_stride + static_cast<size_t>(v) * 16, ElemTraits<T>::pack(accv[k]));
            if (MODE == ATTN_DOT)
                stg_stream16(reinterpret_cast<char*>(grad_k) + static_cast<size_t>(row) * a.k_stride + static_cast<size_t>(v) * 16, ElemTraits<T>::pack(acck[k]));
            if (MODE == ATTN_GAT && first) grad_s_src[row * a.heads + head[k]] = gss[k];
        }
    }
}

// Fold fp32 chunk partials [n_chunks, width] of every long row into up to two typed row outputs (w0 / w1 elements at row
// strides s0 / s1 BYTES) and one fp32 output (wf floats per row).  One CTA per long row, chunks dealt to blockDim / W
// thread slices and folded in a fixed order through shared memory (deterministic).
template <typename T>
__global__ void __launch_bounds__(kCombineT)
attn_sum_combine_kernel(LongRowPlan plan, int64_t width, T* __restrict__ o0, int64_t w0, size_t s0, T* __restrict__ o1,
                        int64_t w1, size_t s1, float* __restrict__ of, int64_t wf, int W) {
    __shared__ float sm[kCombineT];
    const int64_t j = blockIdx.x;
    if (j >= plan.n_long) return;
    const int64_t row = plan.long_rows[j];
    const int64_t c0 = plan.chunk_ptr[j], c1 = plan.chunk_ptr[j + 1];
    const int n_slices = kCombineT / W;
    const int slice = threadIdx.x / W;
    for (int64_t f0 = 0; f0 < width; f0 += W) {
        const int64_t f = f0 + (threadIdx.x % W);
        const bool fv = f < width && slice < n_slices;
        float acc = 0.0f;
        if (fv)
            for (int64_t c = c0 + slice; c < c1; c += n_slices) acc += plan.partials[c * width + f];
        sm[threadIdx.x] = acc;
        __syncthreads();
        if (fv && slice == 0) {
            for (int sl = 1; sl < n_slices; ++sl) acc += sm[sl * W + (threadIdx.x % W)];
            if (f < w0) reinterpret_cast<T*>(reinterpret_cast<char*>(o0) + row * s0)[f] = ElemTraits<T>::from_float(acc);
            else if (f < w0 + w1) reinterpret_cast<T*>(reinterpret_cast<char*>(o1) + row * s1)[f - w0] = ElemTraits<T>::from_float(acc);
            else of[row * wf + (f - w0 - w1)] = acc;
        }
        __syncthreads();
    }
}

// grad_att = sum over the per-CTA partial rows (fixed order: deterministic)
__global__ void __launch_bounds__(256)
attn_fold_rows_kernel(const float* __restrict__ part, int64_t n_part, int64_t width, float* __restrict__ out) {
    const int64_t f = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (f >= width) return;
    float acc = 0.0f;
    for (int64_t p = 0; p < n_part; ++p) acc += part[p * width + f];
    out[f] = acc;
}

// ------------------------------------------------------------------------------------------------ host side
inline bool pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }
inline int combine_width(int64_t width) {      // features per slice of the combine kernels: a power of two <= kCombineT
    int w = 1;
    while (w < width && w < kCombineT) w <<= 1;
    return w;
}

template <typename T>
bool attn_vec_ok(int64_t heads, int64_t chan, const AttnArgs& a, const void* out) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const size_t row_bytes = static_cast<size_t>(heads * chan) * sizeof(T);
    if (row_bytes % 16 != 0 || chan % EPV != 0 || row_bytes / 16 > 64) return false;
    const int64_t lph = chan / EPV;
    if (!pow2(lph) || lph > 32) return false;
    if (!aligned16(a.v) || a.v_stride % 16 != 0 || (out && !aligned16(out))) return false;
    if (a.k && (!aligned16(a.k) || a.k_stride % 16 != 0)) return false;
    if (a.q && (!aligned16(a.q) || a.q_stride % 16 != 0)) return false;
    return true;
}

template <typename T, typename I, int MODE>
int attn_forward_typed(const void* rowptr_, const void* col_, AttnArgs a, void* out_, float* row_max, float* row_den,
                       float* alpha_out, int64_t n_rows, int64_t n_edges, LongRowPlan plan, float* part_ms, cudaStream_t s) {
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    T* out = static_cast<T*>(out_);
    const int n_vec = a.n_vec;
    const int64_t items = plan.n_chunks + n_rows;
    const unsigned blocks = static_cast<unsigned>(ceil_div(items, kAttnT / 32));
#define ATTN_FWD_STAGED(G_) attn_fwd_kernel<T, I, G_, 1, MODE, true><<<blocks, kAttnT, stage_bytes, s>>>(rowptr, col, a, out, row_max, row_den, n_rows, plan, part_ms)
#define ATTN_FWD_STAGED1(G_) attn_fwd_kernel<T, I, G_, 1, MODE, true, 32><<<static_cast<unsigned>(items), 32, stage_bytes / (kAttnT / 32), s>>>(rowptr, col, a, out, row_max, row_den, n_rows, plan, part_ms)
    // lane-private cp.async slots: 2 iterations x 4 edges x (value (+ key) vector + a_src scalar) per thread
    const size_t stage_bytes = static_cast<size_t>(2) * 4 * kAttnT * ((MODE == ATTN_DOT ? 2 : 1) * 16 + 4);
    bool edge_done = false;
    if constexpr (MODE != ATTN_GAT) {
        if (a.ee) {                                                            // per-edge feature rows: register form
            lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                attn_fwd_kernel<T, I, G(), VPL(), MODE, 2><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, out, row_max, row_den, n_rows, plan, part_ms);
            });
            edge_done = true;
        }
    }
    if (edge_done) {
    } else if (get_option_attn_staged() == 2 && n_vec > 4 && n_vec <= 32) {          // one-warp CTAs
        if (n_vec <= 8) ATTN_FWD_STAGED1(8);
        else if (n_vec <= 16) ATTN_FWD_STAGED1(16);
        else ATTN_FWD_STAGED1(32);
    } else if (get_option_attn_staged() && n_vec > 4 && n_vec <= 32) {
        if (n_vec <= 8) ATTN_FWD_STAGED(8);
        else if (n_vec <= 16) ATTN_FWD_STAGED(16);
        else ATTN_FWD_STAGED(32);
    } else {
        lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
            attn_fwd_kernel<T, I, G(), VPL(), MODE><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, out, row_max, row_den, n_rows, plan, part_ms);
        });
    }
#undef ATTN_FWD_STAGED1
#undef ATTN_FWD_STAGED
    B200MP_LAUNCH_CHECK();
    if (plan.n_long > 0) {
        attn_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), kCombineT, 0, s>>>(out, row_max, row_den, a.heads, a.chan, plan, part_ms,
                                                                                  combine_width(static_cast<int64_t>(a.heads) * a.chan));
        B200MP_LAUNCH_CHECK();
    }
    if (alpha_out && n_edges > 0) {
        LongRowPlan np = plan;
        np.partials = nullptr;
        bool alpha_done = false;
        if constexpr (MODE != ATTN_GAT) {
            if (a.ee) {
                lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                    attn_bwd_dst_kernel<T, I, G(), VPL(), MODE, true, 2><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, row_max, row_den, nullptr, nullptr, nullptr, alpha_out, nullptr, nullptr, nullptr, n_rows, np);
                });
                alpha_done = true;
            }
        }
        if (!alpha_done) {
            lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                attn_bwd_dst_kernel<T, I, G(), VPL(), MODE, true><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, row_max, row_den, nullptr, nullptr, nullptr, alpha_out, nullptr, nullptr, nullptr, n_rows, np);
            });
        }
        B200MP_LAUNCH_CHECK();
    }
    return B200MP_OK;
}

template <typename T, typename I, int MODE>
int attn_backward_typed(const void* rowptr_, const void* col_, const void* rowptr_t_, const void* col_t_, const void* t2csr_,
                        AttnArgs a, const float* row_max, const float* row_den, const void* out, const void* grad_out,
                        float* pair, void* grad_v, void* grad_k, void* grad_q, float* grad_s_src, float* grad_s_dst,
                        float* grad_att, float* gatt_part, int64_t gatt_rows, int64_t n_rows, int64_t n_src, LongRowPlan plan,
                        LongRowPlan plan_t, cudaStream_t s) {
    constexpr int EPV = ElemTraits<T>::kPerVec;
    const I* rowptr = static_cast<const I*>(rowptr_);
    const I* col = static_cast<const I*>(col_);
    const int n_vec = a.n_vec;
    const int64_t hc = static_cast<int64_t>(n_vec) * EPV;
    if (n_rows > 0) {
        const int64_t items = plan.n_chunks + n_rows;
        unsigned blocks = static_cast<unsigned>(ceil_div(items, kAttnT / 32));
        if (MODE == ATTN_GATV2 && blocks > static_cast<unsigned>(gatt_rows)) blocks = static_cast<unsigned>(gatt_rows);   // persistent
#define ATTN_DST_STAGED(G_) attn_bwd_dst_kernel<T, I, G_, 1, MODE, false, true><<<blocks, kAttnT, dst_stage, s>>>(rowptr, col, a, row_max, row_den, static_cast<const T*>(out), static_cast<const T*>(grad_out), pair, nullptr, static_cast<T*>(grad_q), grad_s_dst, gatt_part, n_rows, plan)
        const size_t dst_stage = static_cast<size_t>(2) * 4 * kAttnT * ((MODE == ATTN_DOT ? 2 : 1) * 16 + 4);
        bool edge_done = false;
        if constexpr (MODE != ATTN_GAT) {
            if (a.ee) {
                lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                    attn_bwd_dst_kernel<T, I, G(), VPL(), MODE, false, 2><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, row_max, row_den, static_cast<const T*>(out), static_cast<const T*>(grad_out), pair, nullptr, static_cast<T*>(grad_q), grad_s_dst, gatt_part, n_rows, plan);
                });
                edge_done = true;
            }
        }
        if (edge_done) {
        } else if (get_option_attn_staged() && n_vec > 4 && n_vec <= 32) {
            if (n_vec <= 8) ATTN_DST_STAGED(8);
            else if (n_vec <= 16) ATTN_DST_STAGED(16);
            else ATTN_DST_STAGED(32);
        } else {
            lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                attn_bwd_dst_kernel<T, I, G(), VPL(), MODE, false><<<blocks, kAttnT, 0, s>>>(rowptr, col, a, row_max, row_den, static_cast<const T*>(out), static_cast<const T*>(grad_out), pair, nullptr, static_cast<T*>(grad_q), grad_s_dst, gatt_part, n_rows, plan);
            });
        }
#undef ATTN_DST_STAGED
        B200MP_LAUNCH_CHECK();
        if (plan.n_long > 0) {
            if (MODE == ATTN_GAT)
                attn_sum_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), kCombineT, 0, s>>>(plan, a.heads, nullptr, 0, 0, nullptr, 0, 0, grad_s_dst, a.heads,
                                                                                              combine_width(a.heads));
            else
                attn_sum_combine_kernel<T><<<static_cast<unsigned>(plan.n_long), kCombineT, 0, s>>>(plan, hc, static_cast<T*>(grad_q), hc, static_cast<size_t>(hc) * sizeof(T), nullptr, 0, 0, nullptr, 0,
                                                                                              combine_width(hc));
            B200MP_LAUNCH_CHECK();
        }
        if (MODE == ATTN_GATV2) {
            attn_fold_rows_kernel<<<static_cast<unsigned>(ceil_div(hc, 256)), 256, 0, s>>>(gatt_part, blocks, hc, grad_att);
            B200MP_LAUNCH_CHECK();
        }
    }
    if (n_src > 0) {
        const int64_t items = plan_t.n_chunks + n_src;
        const unsigned blocks = static_cast<unsigned>(ceil_div(items, kAttnT / 32));
#define ATTN_SRC_STAGED(G_) attn_bwd_src_kernel<T, I, G_, 1, MODE, true><<<blocks, kAttnT, src_stage, s>>>(static_cast<const I*>(rowptr_t_), static_cast<const I*>(col_t_), static_cast<const I*>(t2csr_), a, static_cast<const T*>(grad_out), pair, static_cast<T*>(grad_v), static_cast<T*>(grad_k), grad_s_src, n_src, plan_t)
#define ATTN_SRC_STAGED1(G_) attn_bwd_src_kernel<T, I, G_, 1, MODE, true, 32><<<static_cast<unsigned>(items), 32, src_stage / (kAttnT / 32), s>>>(static_cast<const I*>(rowptr_t_), static_cast<const I*>(col_t_), static_cast<const I*>(t2csr_), a, static_cast<const T*>(grad_out), pair, static_cast<T*>(grad_v), static_cast<T*>(grad_k), grad_s_src, n_src, plan_t)
        const size_t src_stage = static_cast<size_t>(2) * 4 * kAttnT * ((MODE == ATTN_GAT ? 1 : 2) * 16 + 8);
        bool edge_done = false;
        if constexpr (MODE == ATTN_GATV2) {
            if (a.ee) {                                 // x_l's gradient takes the edges' grad_ee rows instead of recomputing them
                lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                    attn_bwd_src_kernel<T, I, G(), VPL(), MODE, 2><<<blocks, kAttnT, 0, s>>>(static_cast<const I*>(rowptr_t_), static_cast<const I*>(col_t_), static_cast<const I*>(t2csr_), a, static_cast<const T*>(grad_out), pair, static_cast<T*>(grad_v), static_cast<T*>(grad_k), grad_s_src, n_src, plan_t);
                });
                edge_done = true;
            }
        }
        if (edge_done) {
        } else if (get_option_attn_staged() == 2 && n_vec > 4 && n_vec <= 32) {
            if (n_vec <= 8) ATTN_SRC_STAGED1(8);
            else if (n_vec <= 16) ATTN_SRC_STAGED1(16);
            else ATTN_SRC_STAGED1(32);
        } else if (get_option_attn_staged() && n_vec > 4 && n_vec <= 32) {
            if (n_vec <= 8) ATTN_SRC_STAGED(8);
            else if (n_vec <= 16) ATTN_SRC_STAGED(16);
            else ATTN_SRC_STAGED(32);
        } else {
            lane_group_shape<2>(n_vec, [&](auto G, auto VPL) {
                attn_bwd_src_kernel<T, I, G(), VPL(), MODE><<<blocks, kAttnT, 0, s>>>(static_cast<const I*>(rowptr_t_), static_cast<const I*>(col_t_), static_cast<const I*>(t2csr_), a, static_cast<const T*>(grad_out), pair, static_cast<T*>(grad_v), static_cast<T*>(grad_k), grad_s_src, n_src, plan_t);
            });
        }
#undef ATTN_SRC_STAGED1
#undef ATTN_SRC_STAGED
        B200MP_LAUNCH_CHECK();
        if (plan_t.n_long > 0) {
            const int64_t w1 = MODE == ATTN_DOT ? hc : 0, wf = MODE == ATTN_GAT ? a.heads : 0;
            attn_sum_combine_kernel<T><<<static_cast<unsigned>(plan_t.n_long), kCombineT, 0, s>>>(
                plan_t, hc + w1 + wf, static_cast<T*>(grad_v), hc, a.v_stride, static_cast<T*>(grad_k), w1, a.k_stride, grad_s_src, wf,
                combine_width(hc + w1 + wf));
            B200MP_LAUNCH_CHECK();
        }
    }
    return B200MP_OK;
}

}  // namespace b200mp

using namespace b200mp;

namespace {

int fill_args(AttnArgs& a, int mode, const void* v, const void* k, const void* q, const float* s_src, const float* s_dst,
              const float* att, const float* s_edge, int64_t v_stride, int64_t k_stride, int64_t q_stride, int64_t heads,
              int64_t chan, float slope, float scale, int val_dtype, float dropout_p, unsigned long long dropout_seed,
              const void* edge_feat, void* grad_edge_feat) {
    const size_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    if (!(dropout_p >= 0.0f && dropout_p < 1.0f)) return 1;
    a.drop_thresh = dropout_p > 0.0f ? static_cast<uint32_t>(fmin(4294967295.0, ceil(static_cast<double>(dropout_p) * 4294967296.0))) : 0u;
    a.drop_scale = dropout_p > 0.0f ? 1.0f / (1.0f - dropout_p) : 1.0f;
    a.drop_seed = dropout_seed;
    const size_t hc_bytes = static_cast<size_t>(heads * chan) * es;
    a.v = static_cast<const char*>(v);
    a.k = static_cast<const char*>(k);
    a.q = static_cast<const char*>(q);
    a.s_src = s_src;
    a.s_dst = s_dst;
    a.att = att;
    a.s_edge = s_edge;
    a.ee = static_cast<const char*>(edge_feat);
    a.grad_ee = static_cast<char*>(grad_edge_feat);
    if (a.ee && (mode == ATTN_GAT || !aligned16(a.ee) || !aligned16(a.grad_ee))) return 1;
    a.v_stride = v_stride > 0 ? static_cast<size_t>(v_stride) * es : hc_bytes;
    a.k_stride = k_stride > 0 ? static_cast<size_t>(k_stride) * es : hc_bytes;
    a.q_stride = q_stride > 0 ? static_cast<size_t>(q_stride) * es : hc_bytes;
    a.heads = static_cast<int>(heads);
    a.chan = static_cast<int>(chan);
    a.n_vec = static_cast<int>(hc_bytes / 16);
    a.lph = static_cast<int>(chan / (16 / es));
    a.slope = slope;
    a.scale = scale;
    if (mode == ATTN_GAT && !(s_src && s_dst)) return 1;
    if (mode == ATTN_GATV2 && !(q && att)) return 1;
    if (mode == ATTN_DOT && !(q && k)) return 1;
    return 0;
}

}  // namespace

// Calls fn(integral_constant<int, MODE>) for the attention mode (checked by the caller to be one of the three).
template <typename F>
int dispatch_attn_mode(int mode, F&& fn) {
    switch (mode) {
        case ATTN_GAT: return fn(std::integral_constant<int, ATTN_GAT>{});
        case ATTN_GATV2: return fn(std::integral_constant<int, ATTN_GATV2>{});
        default: return fn(std::integral_constant<int, ATTN_DOT>{});
    }
}

extern "C" int b200mp_attn_supported(int64_t heads, int64_t chan, int val_dtype) {
    const int64_t es = val_dtype == B200MP_BF16 ? 2 : 4;
    const int64_t epv = 16 / es;
    const int64_t row_bytes = heads * chan * es;
    if (heads <= 0 || chan <= 0 || row_bytes % 16 != 0 || chan % epv != 0 || row_bytes / 16 > 64) return 0;
    const int64_t lph = chan / epv;
    return (lph & (lph - 1)) == 0 && lph <= 32;
}

extern "C" int b200mp_attn_csr_forward(int mode, const void* rowptr, const void* col, const void* v, const void* k,
                                       const void* q, const float* s_src, const float* s_dst, const float* att,
                                       const float* s_edge, int64_t v_stride, int64_t k_stride, int64_t q_stride,
                                       void* out, float* row_max, float* row_den, float* alpha_out, int64_t n_rows,
                                       int64_t n_edges, int64_t heads, int64_t chan, float slope, float scale,
                                       const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                       int64_t n_chunks, int64_t chunk, float* part_acc, float* part_ms, float dropout_p, unsigned long long dropout_seed, const void* edge_feat, int idx_dtype,
                                       int val_dtype, void* stream) {
    B200MP_CHECK_ARG(mode >= ATTN_GAT && mode <= ATTN_DOT);
    B200MP_CHECK_ARG(n_rows >= 0 && n_edges >= 0 && heads > 0 && chan > 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, part_acc, true)) return rc;
    B200MP_CHECK_ARG(n_long_rows == 0 || part_ms);
    if (n_rows == 0) return B200MP_OK;
    B200MP_CHECK_ARG(rowptr && out && row_max && row_den && (n_edges == 0 || (col && v)));
    AttnArgs a;
    if (fill_args(a, mode, v, k, q, s_src, s_dst, att, s_edge, v_stride, k_stride, q_stride, heads, chan, slope, scale, val_dtype, dropout_p, dropout_seed, edge_feat, nullptr)) {
        set_error("attn forward: operands missing for mode %d (or dropout_p outside [0, 1))", mode);
        return B200MP_ERR_INVALID_ARG;
    }
    if (!b200mp_attn_supported(heads, chan, val_dtype) || !aligned16(v) || !aligned16(out) || a.v_stride % 16 || a.k_stride % 16 ||
        a.q_stride % 16 || (k && !aligned16(k)) || (q && !aligned16(q))) {
        set_error("attn forward: shape H=%lld C=%lld not on the vector path (rows must be 16-byte vectors, <= 1 KB, C/vector a power of two)",
                  static_cast<long long>(heads), static_cast<long long>(chan));
        return B200MP_ERR_UNSUPPORTED;
    }
    return dispatch_val_idx(val_dtype, idx_dtype, "attn_csr_forward", [&](auto tv, auto ti) {
        return dispatch_attn_mode(mode, [&](auto m) {
            return attn_forward_typed<decltype(tv), decltype(ti), m()>(rowptr, col, a, out, row_max, row_den, alpha_out,
                                                                       n_rows, n_edges, plan, part_ms,
                                                                       static_cast<cudaStream_t>(stream));
        });
    });
}

extern "C" int64_t b200mp_attn_backward_partial_width(int mode, int64_t heads, int64_t chan, int transposed) {
    /* fp32 elements per chunk of the long-row partial buffers (destination sweep / source sweep) */
    const int64_t hc = heads * chan;
    if (!transposed) return mode == ATTN_GAT ? heads : hc;
    return hc * (mode == ATTN_DOT ? 2 : 1) + (mode == ATTN_GAT ? heads : 0);
}

extern "C" int64_t b200mp_attn_gatt_rows(void) { return static_cast<int64_t>(num_sms()) * 8; }

extern "C" int b200mp_attn_csr_backward(int mode, const void* rowptr, const void* col, const void* rowptr_t, const void* col_t,
                                        const void* t2csr, const void* v, const void* k, const void* q, const float* s_src,
                                        const float* s_dst, const float* att, const float* s_edge, int64_t v_stride,
                                        int64_t k_stride, int64_t q_stride, const float* row_max, const float* row_den,
                                        const void* out, const void* grad_out, float* pair, void* grad_v, void* grad_k,
                                        void* grad_q, float* grad_s_src, float* grad_s_dst, float* grad_att,
                                        float* gatt_part, int64_t n_rows, int64_t n_src, int64_t n_edges, int64_t heads,
                                        int64_t chan, float slope, float scale, const int64_t* long_rows,
                                        const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                        float* partials, const int64_t* long_rows_t, const int64_t* chunk_ptr_t,
                                        int64_t n_long_rows_t, int64_t n_chunks_t, float* partials_t, float dropout_p, unsigned long long dropout_seed, const void* edge_feat, void* grad_edge_feat, int idx_dtype,
                                        int val_dtype, void* stream) {
    B200MP_CHECK_ARG(mode >= ATTN_GAT && mode <= ATTN_DOT);
    B200MP_CHECK_ARG(n_rows >= 0 && n_src >= 0 && n_edges >= 0 && heads > 0 && chan > 0);
    B200MP_CHECK_ARG(rowptr && rowptr_t && grad_v && row_max && row_den && out && grad_out);
    B200MP_CHECK_ARG(n_edges == 0 || (col && col_t && t2csr && pair));
    B200MP_CHECK_ARG(mode != ATTN_GAT || (grad_s_src && grad_s_dst));
    B200MP_CHECK_ARG(mode == ATTN_GAT || grad_q);
    B200MP_CHECK_ARG(mode != ATTN_DOT || grad_k);
    B200MP_CHECK_ARG(mode != ATTN_GATV2 || (grad_att && gatt_part));
    LongRowPlan plan, plan_t;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (int rc = make_plan(plan_t, long_rows_t, chunk_ptr_t, n_long_rows_t, n_chunks_t, chunk, partials_t, true)) return rc;
    AttnArgs a;
    if (fill_args(a, mode, v, k, q, s_src, s_dst, att, s_edge, v_stride, k_stride, q_stride, heads, chan, slope, scale, val_dtype, dropout_p, dropout_seed, edge_feat, grad_edge_feat)) {
        set_error("attn backward: operands missing for mode %d (or dropout_p outside [0, 1))", mode);
        return B200MP_ERR_INVALID_ARG;
    }
    if (!b200mp_attn_supported(heads, chan, val_dtype) || !aligned16(v) || !aligned16(out) || !aligned16(grad_out) || !aligned16(grad_v) ||
        a.v_stride % 16 || a.k_stride % 16 || a.q_stride % 16 || heads * chan > 64 * 8) {
        set_error("attn backward: shape H=%lld C=%lld not on the vector path", static_cast<long long>(heads), static_cast<long long>(chan));
        return B200MP_ERR_UNSUPPORTED;
    }
    return dispatch_val_idx(val_dtype, idx_dtype, "attn_csr_backward", [&](auto tv, auto ti) {
        return dispatch_attn_mode(mode, [&](auto m) {
            return attn_backward_typed<decltype(tv), decltype(ti), m()>(
                rowptr, col, rowptr_t, col_t, t2csr, a, row_max, row_den, out, grad_out, pair, grad_v, grad_k, grad_q,
                grad_s_src, grad_s_dst, grad_att, gatt_part, b200mp_attn_gatt_rows(), n_rows, n_src, plan, plan_t,
                static_cast<cudaStream_t>(stream));
        });
    });
}
