// point.cu -- graph construction on point clouds: k nearest neighbours, radius neighbourhoods, farthest-point
// sampling and nearest-point assignment (pyg_lib.ops knn / radius / fps / nearest, reached through torch.ops.pyg.* in
// nn/pool/__init__.py, nn/conv/{edge,gravnet,x}_conv.py).
//
// Examples.  An example is the range ptr[b]:ptr[b+1] of points; a NULL ptr is one example covering every point.  Query
// y_i belongs to the example b whose range holds i, and its candidates are the x points of example b; when ptr_x has
// fewer examples than ptr_y (or the other way round), the missing trailing examples are empty.  ptr is int32 or int64
// and is read as given (debug mode validates it on the host side).
//
// Distance contract.  Values are fp32 or bf16, widened exactly to fp32 on load, and every sum runs in feature order
// with explicitly rounded operations (no FMA contraction):
//   squared:  d = sum_f (x_f - y_f)^2                    t = __fsub_rn(x_f, y_f), d = __fadd_rn(d, __fmul_rn(t, t))
//   cosine:   d = 1 - dot / (sqrt(|x|^2) sqrt(|y|^2))    each of the three sums as above, IEEE sqrt and division
// so a float32 loop doing one operation at a time reproduces every bit.  A candidate is selected only when its distance
// compares below something (strict <), so a NaN distance (a zero vector under cosine, a non-finite coordinate) or an
// infinite one is never selected.
//
// Sweep.  One thread per query, Q queries (consecutive y indices) per CTA.  The CTA stages its queries' features in
// shared memory transposed ([F][Q], conflict-free), then walks every example its queries touch and, for each, stages
// tiles of that example's x points (widened to fp32) and lets the threads whose query lies in it visit the tile in
// ascending x index, four candidates per pass over the features.  Features too wide for shared memory are read from
// global memory instead (no staging; same arithmetic).  The per-query selector decides what a visit does:
//   k-NN, k <= 32:   a sorted register list of capacity 8 / 16 / 32, inserted by a fully unrolled compare-and-shift
//                    with a strict <; ascending visits then keep ties in ascending x index.
//   k-NN, k > 32:    the same insertion on a list in shared memory ([k][Q]), with half the queries per CTA.
//   radius count:    counts d < r^2 (r^2 formed in fp64, rounded once to fp32) up to max_num_neighbors, skipping
//                    x == y when asked; the CTA leaves the tile loop once every query in it has reached the cap.
//   radius fill:     the same walk, writing each selected x index at its query's offset.
// k-NN writes each query's list into a [2, M k] slab (row, col) and its length; radius counts first.  One single-CTA
// scan turns the lengths into offsets [M + 1]; the caller reads the total back (the one device-to-host copy of a call)
// and, when the slab is not full, compacts it with b200mp_knn_compact, or runs b200mp_radius_fill.
//
// Farthest-point sampling.  One CTA per example keeps the example's coordinates and running min-distance in shared
// memory when they fit (else reads them from global memory and a caller-provided fp32 buffer, both L2-resident at the
// sizes in use).  Each step updates the min-distance to the last pick and takes its argmax, ties to the lowest index,
// by one warp-shuffle and shared-memory reduction with two barriers.  The number of samples of example b is
// ceil(n_b ratio) in fp64 (b200mp_fps_count, scanned into offsets); the start is the example's first point or, given
// a uniform u_b in [0, 1) per example (torch's CUDA generator, drawn on the device), point floor(u_b n_b).
//
// Nearest.  b200mp_nearest is the k-NN sweep with k = 1 and the roles swapped: for each x point, the nearest y point.
//
// -Xptxas -v for sm_90a (CUDA 12.9): every instantiation has no stack frame and no spills.
#include <climits>

#include "common.cuh"

namespace b200mp {

constexpr int kPtMaxK = 128;
constexpr int kPtSmallQ = 128;          // queries per CTA, k <= 32 and radius
constexpr int kPtLargeQ = 64;           // queries per CTA, k > 32
constexpr int kPtMaxTile = 256;         // x points per staged tile
constexpr int64_t kPtTileBytes = 32768; // x tile budget
constexpr int64_t kPtSmemBytes = 200 * 1024;
constexpr int kPtFpsThreads = 512;
constexpr int64_t kPtFpsSmemBytes = 96 * 1024;

__host__ __device__ __forceinline__ int64_t pt_min(int64_t a, int64_t b) { return a < b ? a : b; }

__device__ __forceinline__ float pt_widen(float v) { return v; }
__device__ __forceinline__ float pt_widen(__nv_bfloat16 v) { return __bfloat162float(v); }

__device__ __forceinline__ int64_t pt_ptr(const void* ptr, int is64, int64_t i) {
    return is64 ? static_cast<const int64_t*>(ptr)[i] : static_cast<int64_t>(static_cast<const int32_t*>(ptr)[i]);
}

// Example of point i: the last b < n_ptr - 1 with ptr[b] <= i, or -1 when i lies outside every example.
__device__ __forceinline__ int64_t pt_example_of(const void* ptr, int is64, int64_t n_ptr, int64_t n, int64_t i) {
    if (ptr == nullptr) return i < n ? 0 : -1;
    const int64_t n_ex = n_ptr - 1;
    if (n_ex < 1) return -1;
    int64_t lo = 0, hi = n_ex;  // invariant: answer in [lo, hi)
    if (pt_ptr(ptr, is64, 0) > i) return -1;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (pt_ptr(ptr, is64, mid) <= i) lo = mid;
        else hi = mid;
    }
    return i < pt_ptr(ptr, is64, lo + 1) ? lo : -1;
}

__device__ __forceinline__ void pt_range(const void* ptr, int is64, int64_t n_ptr, int64_t n, int64_t b, int64_t& s,
                                         int64_t& e) {
    s = e = 0;
    if (b < 0) return;
    if (ptr == nullptr) {
        if (b == 0) e = n;
        return;
    }
    if (b + 1 < n_ptr) {
        s = pt_ptr(ptr, is64, b);
        e = pt_ptr(ptr, is64, b + 1);
        if (e < s) e = s;
    }
}

// Squared or cosine distances of NC candidates (x rows at xs apart) to one query (y features ys apart), in feature
// order with explicit rounding.
template <int NC, typename XT, typename YT>
__device__ __forceinline__ void pt_dist(const XT* x, int64_t xs, const YT* y, int64_t ys, int64_t F, bool cosine,
                                        float (&d)[NC]) {
    if (!cosine) {
#pragma unroll
        for (int c = 0; c < NC; ++c) d[c] = 0.0f;
        for (int64_t f = 0; f < F; ++f) {
            const float yv = pt_widen(y[f * ys]);
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const float t = __fsub_rn(pt_widen(x[c * xs + f]), yv);
                d[c] = __fadd_rn(d[c], __fmul_rn(t, t));
            }
        }
        return;
    }
    float dot[NC], nx[NC], ny = 0.0f;
#pragma unroll
    for (int c = 0; c < NC; ++c) dot[c] = nx[c] = 0.0f;
    for (int64_t f = 0; f < F; ++f) {
        const float yv = pt_widen(y[f * ys]);
        ny = __fadd_rn(ny, __fmul_rn(yv, yv));
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const float xv = pt_widen(x[c * xs + f]);
            dot[c] = __fadd_rn(dot[c], __fmul_rn(xv, yv));
            nx[c] = __fadd_rn(nx[c], __fmul_rn(xv, xv));
        }
    }
    const float sy = __fsqrt_rn(ny);
#pragma unroll
    for (int c = 0; c < NC; ++c) d[c] = __fsub_rn(1.0f, __fdiv_rn(dot[c], __fmul_rn(__fsqrt_rn(nx[c]), sy)));
}

struct PtArgs {
    const void* x;
    const void* y;
    const void* ptr_x;
    const void* ptr_y;
    int64_t n_x, n_y, f, n_ptr_x, n_ptr_y;
    int ptr_x64, ptr_y64;
    int cosine;
    int64_t k;              // k-NN: neighbours per query; radius: max_num_neighbors
    float r2;               // radius: the bound on d
    int ignore_same;        // radius: skip x index == y index
    int64_t* out;           // k-NN: slab [2, n_y k]; radius fill: [2, nnz]
    int64_t out_stride;     // row stride of out
    int64_t* offsets;       // [n_y + 1]: lengths at [i + 1] (k-NN, radius count); offsets (radius fill)
    int tile;               // staged x points per tile (0: unstaged)
};

// ------------------------------------------------------------------ selectors
template <int K>
struct PtRegTopK {
    float d[K];
    int32_t j[K];
    __device__ __forceinline__ void init(const PtArgs&, float*, int32_t*, int, int) {
#pragma unroll
        for (int c = 0; c < K; ++c) {
            d[c] = __int_as_float(0x7f800000);
            j[c] = -1;
        }
    }
    __device__ __forceinline__ bool full() const { return false; }
    __device__ __forceinline__ void visit(float v, int64_t idx, int64_t) {
        if (!(v < d[K - 1])) return;
        const int32_t ji = static_cast<int32_t>(idx);
#pragma unroll
        for (int c = K - 1; c > 0; --c) {
            if (v < d[c - 1]) {
                d[c] = d[c - 1];
                j[c] = j[c - 1];
            } else if (v < d[c]) {
                d[c] = v;
                j[c] = ji;
            }
        }
        if (v < d[0]) {
            d[0] = v;
            j[0] = ji;
        }
    }
    __device__ __forceinline__ void finish(const PtArgs& a, int64_t q) {
        int64_t n = 0;
        int64_t* row = a.out + q * a.k;
        int64_t* col = row + a.out_stride;
#pragma unroll
        for (int c = 0; c < K; ++c) {
            if (c < a.k) {
                row[c] = q;
                col[c] = j[c];
                n += j[c] >= 0;
            }
        }
        a.offsets[q + 1] = n;
    }
};

struct PtSmemTopK {
    float* d;
    int32_t* j;
    int stride;
    int k;
    float worst;
    __device__ __forceinline__ void init(const PtArgs& a, float* sd, int32_t* sj, int tid, int q_per_cta) {
        d = sd + tid;
        j = sj + tid;
        stride = q_per_cta;
        k = static_cast<int>(a.k);
        worst = __int_as_float(0x7f800000);
        for (int c = 0; c < k; ++c) {
            d[c * stride] = worst;
            j[c * stride] = -1;
        }
    }
    __device__ __forceinline__ bool full() const { return false; }
    __device__ __forceinline__ void visit(float v, int64_t idx, int64_t) {
        if (!(v < worst)) return;
        int c = k - 1;
        while (c > 0 && v < d[(c - 1) * stride]) {
            d[c * stride] = d[(c - 1) * stride];
            j[c * stride] = j[(c - 1) * stride];
            --c;
        }
        d[c * stride] = v;
        j[c * stride] = static_cast<int32_t>(idx);
        worst = d[(k - 1) * stride];
    }
    __device__ __forceinline__ void finish(const PtArgs& a, int64_t q) {
        int64_t n = 0;
        int64_t* row = a.out + q * a.k;
        int64_t* col = row + a.out_stride;
        for (int c = 0; c < k; ++c) {
            const int32_t jc = j[c * stride];
            row[c] = q;
            col[c] = jc;
            n += jc >= 0;
        }
        a.offsets[q + 1] = n;
    }
};

template <bool FILL>
struct PtRadius {
    int64_t n;
    int64_t cap;
    float r2;
    bool skip_same;
    int64_t base;
    __device__ __forceinline__ void init(const PtArgs& a, float*, int32_t*, int, int) {
        n = 0;
        cap = a.k;
        r2 = a.r2;
        skip_same = a.ignore_same != 0;
        base = 0;
    }
    __device__ __forceinline__ bool full() const { return n >= cap; }
    __device__ __forceinline__ void visit(float v, int64_t idx, int64_t q) {
        if (n < cap && v < r2 && !(skip_same && idx == q)) {
            if constexpr (FILL) {
                out_row[base + n] = q;
                out_col[base + n] = idx;
            }
            ++n;
        }
    }
    int64_t* out_row;
    int64_t* out_col;
    __device__ __forceinline__ void start(const PtArgs& a, int64_t q) {
        if constexpr (FILL) {
            base = a.offsets[q];
            out_row = a.out;
            out_col = a.out + a.out_stride;
        }
    }
    __device__ __forceinline__ void finish(const PtArgs& a, int64_t q) {
        if constexpr (!FILL) a.offsets[q + 1] = n;
    }
};

template <typename S>
__device__ __forceinline__ void pt_start(S&, const PtArgs&, int64_t) {}
template <bool FILL>
__device__ __forceinline__ void pt_start(PtRadius<FILL>& s, const PtArgs& a, int64_t q) { s.start(a, q); }

// ------------------------------------------------------------------ the sweep
// Dynamic shared memory: [k][Q] list (k > 32 only), then y [F][Q] and one x tile [tile][F] when staged.
template <typename T, typename Sel, bool STAGED>
__global__ void __launch_bounds__(kPtSmallQ) point_sweep_kernel(PtArgs a, int list_k) {
    extern __shared__ __align__(16) unsigned char pt_smem[];
    __shared__ long long s_bmin, s_bmax;
    const int tid = threadIdx.x;
    const int Q = blockDim.x;
    const int64_t q0 = static_cast<int64_t>(blockIdx.x) * Q;
    const int64_t q = q0 + tid;
    const bool valid = q < a.n_y;
    const int64_t F = a.f;
    float* sd = reinterpret_cast<float*>(pt_smem);
    int32_t* sj = reinterpret_cast<int32_t*>(sd + static_cast<int64_t>(list_k) * Q);
    float* sy = reinterpret_cast<float*>(sj + static_cast<int64_t>(list_k) * Q);
    float* sx = sy + (STAGED ? F * Q : 0);
    const T* x = static_cast<const T*>(a.x);
    const T* y = static_cast<const T*>(a.y);

    const int64_t my_b = valid ? pt_example_of(a.ptr_y, a.ptr_y64, a.n_ptr_y, a.n_y, q) : -1;
    if (tid == 0) {
        s_bmin = LLONG_MAX;
        s_bmax = -1;
    }
    if constexpr (STAGED) {
        if (valid)
            for (int64_t f = 0; f < F; ++f) sy[f * Q + tid] = pt_widen(y[q * F + f]);
    }
    __syncthreads();
    if (my_b >= 0) {
        atomicMin(&s_bmin, static_cast<long long>(my_b));
        atomicMax(&s_bmax, static_cast<long long>(my_b));
    }
    Sel sel;
    sel.init(a, sd, sj, tid, Q);
    if (valid) pt_start(sel, a, q);
    __syncthreads();
    const int64_t bmin = s_bmin, bmax = s_bmax;

    for (int64_t b = bmin; b <= bmax; ++b) {
        if (!__syncthreads_or(my_b == b)) continue;
        const bool mine = my_b == b;
        int64_t xs, xe;
        pt_range(a.ptr_x, a.ptr_x64, a.n_ptr_x, a.n_x, b, xs, xe);
        if constexpr (STAGED) {
            for (int64_t t0 = xs; t0 < xe; t0 += a.tile) {
                const int nt = static_cast<int>(pt_min(a.tile, xe - t0));
                __syncthreads();
                const T* src = x + t0 * F;
                for (int64_t e = tid; e < nt * F; e += Q) sx[e] = pt_widen(src[e]);
                __syncthreads();
                if (mine && !sel.full()) {
                    int jl = 0;
                    for (; jl + 4 <= nt; jl += 4) {
                        float d[4];
                        pt_dist<4>(sx + jl * F, F, sy + tid, Q, F, a.cosine, d);
#pragma unroll
                        for (int c = 0; c < 4; ++c) sel.visit(d[c], t0 + jl + c, q);
                    }
                    for (; jl < nt; ++jl) {
                        float d[1];
                        pt_dist<1>(sx + jl * F, F, sy + tid, Q, F, a.cosine, d);
                        sel.visit(d[0], t0 + jl, q);
                    }
                }
                if (__syncthreads_and(!mine || sel.full())) break;
            }
        } else if (mine) {
            for (int64_t jx = xs; jx < xe && !sel.full(); ++jx) {
                float d[1];
                pt_dist<1>(x + jx * F, F, y + q * F, 1, F, a.cosine, d);
                sel.visit(d[0], jx, q);
            }
        }
    }
    if (valid) sel.finish(a, q);
}

// offsets[1..n] hold lengths on entry; on exit offsets[0] = 0 and offsets[i + 1] = sum of the first i + 1 lengths.
__global__ void __launch_bounds__(1024) point_scan_kernel(int64_t* offsets, int64_t n) {
    __shared__ long long warp_sums[32];
    const int tid = threadIdx.x;
    const int64_t chunk = (n + blockDim.x - 1) / blockDim.x;
    const int64_t s = pt_min(n, tid * chunk), e = pt_min(n, s + chunk);
    long long sum = 0;
    for (int64_t i = s; i < e; ++i) sum += offsets[i + 1];
    long long inc = sum;
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        long long w = lane < static_cast<int>(blockDim.x >> 5) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long v = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += v;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    long long run = inc - sum + (warp > 0 ? warp_sums[warp - 1] : 0);
    for (int64_t i = s; i < e; ++i) {
        run += offsets[i + 1];
        offsets[i + 1] = run;
    }
    if (tid == 0) offsets[0] = 0;
}

__global__ void point_compact_kernel(const int64_t* slab, const int64_t* offsets, int64_t n_q, int64_t k, int64_t* out,
                                     int64_t nnz) {
    const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (t >= n_q * k) return;
    const int64_t q = t / k, c = t - q * k;
    const int64_t o = offsets[q];
    if (o + c < offsets[q + 1]) {
        out[o + c] = q;
        out[nnz + o + c] = slab[n_q * k + t];
    }
}

// ------------------------------------------------------------------ farthest-point sampling
__global__ void point_fps_count_kernel(const void* ptr, int is64, int64_t n_ptr, int64_t n, double ratio,
                                       int64_t* offsets) {
    const int64_t b = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t n_ex = ptr ? n_ptr - 1 : 1;
    if (b >= n_ex) return;
    int64_t s, e;
    pt_range(ptr, is64, n_ptr, n, b, s, e);
    offsets[b + 1] = static_cast<int64_t>(ceil(static_cast<double>(e - s) * ratio));
}

struct PtBest {
    float v;
    int64_t i;
};
__device__ __forceinline__ bool pt_better(float v, int64_t i, float bv, int64_t bi) {
    return v > bv || (v == bv && i < bi);
}

template <typename T>
__global__ void __launch_bounds__(kPtFpsThreads) point_fps_kernel(const T* src, const void* ptr, int is64, int64_t n_ptr,
                                                                  int64_t n, int64_t F, const float* rnd,
                                                                  const int64_t* offsets, float* dist_ws, int64_t* out,
                                                                  int64_t smem_floats) {
    extern __shared__ __align__(16) unsigned char pt_smem[];
    __shared__ float s_v[kPtFpsThreads / 32];
    __shared__ long long s_i[kPtFpsThreads / 32];
    __shared__ long long s_last;
    const int64_t b = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int64_t s, e;
    pt_range(ptr, is64, n_ptr, n, b, s, e);
    const int64_t nb = e - s, o0 = offsets[b], o1 = offsets[b + 1];
    if (nb <= 0 || o1 <= o0) return;
    const bool staged = nb * (F + 1) <= smem_floats;
    float* sx = reinterpret_cast<float*>(pt_smem);
    float* mind = staged ? sx + nb * F : dist_ws + s;
    const T* gx = src + s * F;
    const float inf = __int_as_float(0x7f800000);
    if (staged)
        for (int64_t t = tid; t < nb * F; t += blockDim.x) sx[t] = pt_widen(gx[t]);
    for (int64_t t = tid; t < nb; t += blockDim.x) mind[t] = inf;
    int64_t last = 0;
    if (rnd) last = pt_min(static_cast<int64_t>(static_cast<double>(rnd[b]) * static_cast<double>(nb)), nb - 1);
    if (tid == 0) out[o0] = s + last;
    __syncthreads();
    for (int64_t m = o0 + 1; m < o1; ++m) {
        float bv = -1.0f;
        int64_t bi = LLONG_MAX;
        for (int64_t t = tid; t < nb; t += blockDim.x) {
            float d[1];
            if (staged) pt_dist<1>(sx + t * F, F, sx + last * F, 1, F, false, d);
            else pt_dist<1>(gx + t * F, F, gx + last * F, 1, F, false, d);
            float v = mind[t];
            if (d[0] < v) {
                v = d[0];
                mind[t] = v;
            }
            if (v > bv) {
                bv = v;
                bi = t;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_down_sync(0xffffffffu, bv, o);
            const long long oi = __shfl_down_sync(0xffffffffu, static_cast<long long>(bi), o);
            if (pt_better(ov, oi, bv, bi)) {
                bv = ov;
                bi = oi;
            }
        }
        if (lane == 0) {
            s_v[warp] = bv;
            s_i[warp] = bi;
        }
        __syncthreads();
        if (warp == 0) {
            const int nw = blockDim.x >> 5;
            bv = lane < nw ? s_v[lane] : -1.0f;
            bi = lane < nw ? s_i[lane] : LLONG_MAX;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_down_sync(0xffffffffu, bv, o);
                const long long oi = __shfl_down_sync(0xffffffffu, static_cast<long long>(bi), o);
                if (pt_better(ov, oi, bv, bi)) {
                    bv = ov;
                    bi = oi;
                }
            }
            if (lane == 0) {
                s_last = bi;
                out[m] = s + bi;
            }
        }
        __syncthreads();
        last = s_last;
    }
}

// ------------------------------------------------------------------ host side
static int pt_check_common(const void* x, const void* y, int64_t n_x, int64_t n_y, int64_t f, const void* ptr_x,
                           int64_t n_ptr_x, const void* ptr_y, int64_t n_ptr_y) {
    B200MP_CHECK_ARG(n_x >= 0 && n_y >= 0 && f >= 1);
    B200MP_CHECK_ARG(n_x < INT32_MAX);
    B200MP_CHECK_ARG(n_x == 0 || x);
    B200MP_CHECK_ARG(n_y == 0 || y);
    B200MP_CHECK_ARG(!ptr_x || n_ptr_x >= 1);
    B200MP_CHECK_ARG(!ptr_y || n_ptr_y >= 1);
    return B200MP_OK;
}

static int pt_scan(int64_t* offsets, int64_t n, cudaStream_t st) {
    point_scan_kernel<<<1, 1024, 0, st>>>(offsets, n);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename T, typename Sel>
static int pt_launch_typed(const PtArgs& a0, int q_per_cta, int list_k, cudaStream_t st) {
    PtArgs a = a0;
    const int64_t list_bytes = static_cast<int64_t>(list_k) * q_per_cta * 8;
    const int64_t y_bytes = a.f * q_per_cta * 4;
    const int64_t tile = pt_min(kPtMaxTile, kPtTileBytes / (a.f * 4));
    const unsigned grid = static_cast<unsigned>(ceil_div(a.n_y, q_per_cta));
    if (tile >= 1 && list_bytes + y_bytes + tile * a.f * 4 <= kPtSmemBytes) {
        a.tile = static_cast<int>(tile);
        const int64_t bytes = list_bytes + y_bytes + tile * a.f * 4;
        auto kern = point_sweep_kernel<T, Sel, true>;
        B200MP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
        kern<<<grid, q_per_cta, bytes, st>>>(a, list_k);
    } else {
        a.tile = 0;
        auto kern = point_sweep_kernel<T, Sel, false>;
        B200MP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(list_bytes)));
        kern<<<grid, q_per_cta, list_bytes, st>>>(a, list_k);
    }
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

template <typename F>
static int pt_dispatch(int val_dtype, const char* what, F&& fn) {
    if (val_dtype == B200MP_F32) return fn(float{});
    if (val_dtype == B200MP_BF16) return fn(__nv_bfloat16{});
    set_error("%s: unsupported value dtype %d", what, val_dtype);
    return B200MP_ERR_UNSUPPORTED;
}

static int pt_knn(PtArgs a, int val_dtype, cudaStream_t st, const char* what) {
    if (a.k < 1 || a.k > kPtMaxK) {
        set_error("%s: k = %lld outside 1..%d", what, static_cast<long long>(a.k), kPtMaxK);
        return B200MP_ERR_UNSUPPORTED;
    }
    B200MP_CHECK_ARG(a.n_y == 0 || (a.out && a.offsets));
    if (a.n_y == 0) {
        if (a.offsets) B200MP_CUDA(cudaMemsetAsync(a.offsets, 0, sizeof(int64_t), st));
        return B200MP_OK;
    }
    const int k = static_cast<int>(a.k);
    const int rc = pt_dispatch(val_dtype, what, [&](auto tv) -> int {
        using T = decltype(tv);
        if (k <= 8) return pt_launch_typed<T, PtRegTopK<8>>(a, kPtSmallQ, 0, st);
        if (k <= 16) return pt_launch_typed<T, PtRegTopK<16>>(a, kPtSmallQ, 0, st);
        if (k <= 32) return pt_launch_typed<T, PtRegTopK<32>>(a, kPtSmallQ, 0, st);
        return pt_launch_typed<T, PtSmemTopK>(a, kPtLargeQ, k, st);
    });
    if (rc) return rc;
    return pt_scan(a.offsets, a.n_y, st);
}

static PtArgs pt_args(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                      int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, int ptr_dtype) {
    PtArgs a{};
    a.x = x;
    a.y = y;
    a.ptr_x = ptr_x;
    a.ptr_y = ptr_y;
    a.n_x = n_x;
    a.n_y = n_y;
    a.f = f;
    a.n_ptr_x = n_ptr_x;
    a.n_ptr_y = n_ptr_y;
    a.ptr_x64 = a.ptr_y64 = ptr_dtype == B200MP_I64;
    return a;
}

}  // namespace b200mp

using namespace b200mp;

extern "C" int b200mp_knn(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                          int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, int64_t k, int cosine, int64_t* slab,
                          int64_t* offsets, int val_dtype, int ptr_dtype, void* stream) {
    if (int rc = pt_check_common(x, y, n_x, n_y, f, ptr_x, n_ptr_x, ptr_y, n_ptr_y)) return rc;
    B200MP_CHECK_ARG(ptr_dtype == B200MP_I32 || ptr_dtype == B200MP_I64);
    PtArgs a = pt_args(x, y, ptr_x, ptr_y, n_x, n_y, f, n_ptr_x, n_ptr_y, ptr_dtype);
    a.cosine = cosine != 0;
    a.k = k;
    a.out = slab;
    a.out_stride = n_y * k;
    a.offsets = offsets;
    return pt_knn(a, val_dtype, static_cast<cudaStream_t>(stream), "knn");
}

extern "C" int b200mp_knn_compact(const int64_t* slab, const int64_t* offsets, int64_t n_y, int64_t k, int64_t* out,
                                  int64_t nnz, void* stream) {
    B200MP_CHECK_ARG(n_y >= 0 && k >= 1 && nnz >= 0);
    if (n_y == 0 || nnz == 0) return B200MP_OK;
    B200MP_CHECK_ARG(slab && offsets && out);
    const int64_t total = n_y * k;
    point_compact_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        slab, offsets, n_y, k, out, nnz);
    B200MP_LAUNCH_CHECK();
    return B200MP_OK;
}

static int pt_radius(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                     int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, float r2, int64_t max_num_neighbors, int ignore_same,
                     int64_t* offsets, int64_t* out, int64_t nnz, int val_dtype, int ptr_dtype, void* stream) {
    if (int rc = pt_check_common(x, y, n_x, n_y, f, ptr_x, n_ptr_x, ptr_y, n_ptr_y)) return rc;
    B200MP_CHECK_ARG(ptr_dtype == B200MP_I32 || ptr_dtype == B200MP_I64);
    B200MP_CHECK_ARG(n_y == 0 || offsets);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool fill = out != nullptr;
    if (n_y == 0) {
        if (!fill && offsets) B200MP_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
        return B200MP_OK;
    }
    if (fill && nnz == 0) return B200MP_OK;
    PtArgs a = pt_args(x, y, ptr_x, ptr_y, n_x, n_y, f, n_ptr_x, n_ptr_y, ptr_dtype);
    a.k = max_num_neighbors > 0 ? max_num_neighbors : 0;
    a.r2 = r2;
    a.ignore_same = ignore_same != 0;
    a.offsets = offsets;
    a.out = out;
    a.out_stride = nnz;
    const int rc = pt_dispatch(val_dtype, "radius", [&](auto tv) -> int {
        using T = decltype(tv);
        if (fill) return pt_launch_typed<T, PtRadius<true>>(a, kPtSmallQ, 0, st);
        return pt_launch_typed<T, PtRadius<false>>(a, kPtSmallQ, 0, st);
    });
    if (rc || fill) return rc;
    return pt_scan(offsets, n_y, st);
}

extern "C" int b200mp_radius_count(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x,
                                   int64_t n_y, int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, float r2,
                                   int64_t max_num_neighbors, int ignore_same_index, int64_t* offsets, int val_dtype,
                                   int ptr_dtype, void* stream) {
    return pt_radius(x, y, ptr_x, ptr_y, n_x, n_y, f, n_ptr_x, n_ptr_y, r2, max_num_neighbors, ignore_same_index,
                     offsets, nullptr, 0, val_dtype, ptr_dtype, stream);
}

extern "C" int b200mp_radius_fill(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x,
                                  int64_t n_y, int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, float r2,
                                  int64_t max_num_neighbors, int ignore_same_index, const int64_t* offsets, int64_t* out,
                                  int64_t nnz, int val_dtype, int ptr_dtype, void* stream) {
    B200MP_CHECK_ARG(nnz == 0 || out);
    int64_t dummy = 0;
    return pt_radius(x, y, ptr_x, ptr_y, n_x, n_y, f, n_ptr_x, n_ptr_y, r2, max_num_neighbors, ignore_same_index,
                     const_cast<int64_t*>(offsets), out ? out : &dummy, nnz, val_dtype, ptr_dtype, stream);
}

extern "C" int b200mp_nearest(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x,
                              int64_t n_y, int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, int64_t* slab,
                              int64_t* offsets, int val_dtype, int ptr_dtype, void* stream) {
    // the k-NN sweep with k = 1 and the roles swapped: x points are the queries, y points the candidates
    if (int rc = pt_check_common(y, x, n_y, n_x, f, ptr_y, n_ptr_y, ptr_x, n_ptr_x)) return rc;
    B200MP_CHECK_ARG(ptr_dtype == B200MP_I32 || ptr_dtype == B200MP_I64);
    PtArgs a = pt_args(y, x, ptr_y, ptr_x, n_y, n_x, f, n_ptr_y, n_ptr_x, ptr_dtype);
    a.k = 1;
    a.out = slab;
    a.out_stride = n_x;
    a.offsets = offsets;
    return pt_knn(a, val_dtype, static_cast<cudaStream_t>(stream), "nearest");
}

extern "C" int b200mp_fps_count(const void* ptr, int64_t n_ptr, int64_t n, double ratio, int64_t* offsets,
                                int ptr_dtype, void* stream) {
    B200MP_CHECK_ARG(n >= 0 && (!ptr || n_ptr >= 1) && offsets);
    B200MP_CHECK_ARG(ratio > 0.0 && ratio <= 1.0);
    B200MP_CHECK_ARG(ptr_dtype == B200MP_I32 || ptr_dtype == B200MP_I64);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t n_ex = ptr ? n_ptr - 1 : 1;
    if (n_ex == 0) {
        B200MP_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
        return B200MP_OK;
    }
    point_fps_count_kernel<<<static_cast<unsigned>(ceil_div(n_ex, 256)), 256, 0, st>>>(ptr, ptr_dtype == B200MP_I64,
                                                                                      n_ptr, n, ratio, offsets);
    B200MP_LAUNCH_CHECK();
    return pt_scan(offsets, n_ex, st);
}

extern "C" int b200mp_fps(const void* src, const void* ptr, int64_t n, int64_t f, int64_t n_ptr, const float* rnd,
                          const int64_t* offsets, float* dist_ws, int64_t* out, int val_dtype, int ptr_dtype,
                          void* stream) {
    B200MP_CHECK_ARG(n >= 0 && f >= 1 && (!ptr || n_ptr >= 1));
    B200MP_CHECK_ARG(ptr_dtype == B200MP_I32 || ptr_dtype == B200MP_I64);
    const int64_t n_ex = ptr ? n_ptr - 1 : 1;
    if (n == 0 || n_ex == 0) return B200MP_OK;
    B200MP_CHECK_ARG(src && offsets && dist_ws && out);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return pt_dispatch(val_dtype, "fps", [&](auto tv) -> int {
        using T = decltype(tv);
        auto kern = point_fps_kernel<T>;
        B200MP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(kPtFpsSmemBytes)));
        kern<<<static_cast<unsigned>(n_ex), kPtFpsThreads, kPtFpsSmemBytes, st>>>(
            static_cast<const T*>(src), ptr, ptr_dtype == B200MP_I64, n_ptr, n, f, rnd, offsets, dist_ws, out,
            kPtFpsSmemBytes / 4);
        B200MP_LAUNCH_CHECK();
        return B200MP_OK;
    });
}
