/*
 * b200mp.h -- C ABI of the H100-native (sm_90a) message-passing aggregation engine.
 *
 * This is the drop-in boundary (SURVEY.md section 8(b), DESIGN.md section 2).  The reference
 * (pyg-team/pytorch_geometric v2.9.0) has no FFI of its own: it late-binds a small set of
 * operator signatures (torch_scatter.*, torch.ops.torch_sparse.spmm_*, pyg_lib.ops.*) and a few
 * Python functions.  Each entry point below states which of those it replaces (file:line under
 * torch_geometric/ of the reference, v2.9.0).  INTEGRATION.md shows the reference-side binding.
 *
 * Conventions
 *  - plain pointers and sizes; no torch types.  All pointers are DEVICE pointers unless the
 *    name ends in _host.  Buffers are caller-owned; nothing is allocated inside.
 *  - feature matrices are row-major, contiguous, [rows, feat]; `val_dtype` selects the element
 *    type (B200MP_F32 / B200MP_BF16); accumulation is always fp32.
 *  - index arrays (`rowptr`, `col`, `index`, `perm`) share one `idx_dtype` per call
 *    (B200MP_I32 / B200MP_I64).  The reference uses int64; int32 halves index traffic and is
 *    what the engine's own graph cache stores when N, E < 2^31.
 *  - edge weights / attention values are always fp32.
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls only
 *    enqueue work; they never synchronise unless documented.
 *  - return value: 0 on success, a negative B200MP_ERR_* code otherwise.  Nothing throws
 *    across the ABI.  A kernel cannot raise: out-of-range indices are undefined behaviour
 *    unless the caller checks them first with b200mp_index_stats() (min / max / sortedness in one
 *    pass); the host-side mirror raises the reference's "valid indices" IndexError
 *    (nn/conv/message_passing.py:269-290) from that result.
 */
#ifndef B200MP_H_
#define B200MP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MP_VERSION "0.1.0"

/* element / index dtypes */
enum { B200MP_F32 = 0, B200MP_BF16 = 1, B200MP_F64 = 2 };
enum { B200MP_I32 = 0, B200MP_I64 = 1 };
/* reductions (same codes as oracle/mp_oracle.c) */
enum { B200MP_SUM = 0, B200MP_MEAN = 1, B200MP_MIN = 2, B200MP_MAX = 3, B200MP_MUL = 4 };
/* errors */
enum {
    B200MP_OK = 0,
    B200MP_ERR_INVALID_ARG = -1,   /* NULL pointer, negative size, misaligned buffer */
    B200MP_ERR_UNSUPPORTED = -2,   /* dtype / reduce combination not implemented */
    B200MP_ERR_CUDA = -3,          /* a CUDA API call or launch failed; see b200mp_last_error() */
    B200MP_ERR_WORKSPACE = -4      /* workspace too small */
};

const char* b200mp_version(void);
const char* b200mp_last_error(void);          /* thread-local, human readable */
int b200mp_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes);
/* Runtime switches for measurements (A/B of kernel variants; the defaults are the measured best).
 *   "spmm_impl"    0 = auto (default), 1 = lane-group-per-row kernel only, 2 = persistent TMA-fed kernel wherever legal
 *   "attn_staged"  2 = cp.async-staged attention sweeps with one-warp CTAs (default), 1 = 4-warp CTAs, 0 = register form;
 *                  0 also turns the multi-aggregation hit-bit path off
 *   "multi_tune"   6 = one-warp CTAs for the multi-aggregation row sweeps (default), 5 = 128-thread CTAs
 *   "gemm_*", "spmm_tune"   tuning knobs of the GEMM / gather kernels (see csrc/core.cu) */
int b200mp_set_option(const char* name, int value);

/* ------------------------------------------------------------------ graph structure (integer work, bit-exact)
 * Replaces: utils/_degree.py:9-31 (degree), index.py:27-37 (ptr2index / index2ptr ==
 * torch._convert_indices_from_coo_to_csr / repeat_interleave), utils/_index_sort.py:10-32 and
 * pyg_lib.ops.index_sort (stable radix sort by key), EdgeIndex.get_csr/get_csc/_sort_by_transpose
 * (edge_index.py:589-696), utils/loop.py:585-657 (add_remaining_self_loops) and :71-131/:382-492
 * (remove_self_loops + add_self_loops), nn/conv/gcn_conv.py:95-113 (gcn_norm). */

/* deg[i] = #(index == i); deg has idx_dtype. */
int b200mp_degree(const void* index, int64_t n_index, int64_t n_nodes, void* deg, int idx_dtype,
                  void* stream);
/* ptr[i] = #(index < i) for a SORTED index; ptr has n_nodes + 1 entries. */
int b200mp_index2ptr(const void* index_sorted, int64_t n_index, int64_t n_nodes, void* ptr,
                     int idx_dtype, void* stream);
/* index[e] = i for ptr[i] <= e < ptr[i+1]. */
int b200mp_ptr2index(const void* ptr, int64_t n_nodes, int64_t n_index, void* index,
                     int idx_dtype, void* stream);
/* min / max / sortedness of an index array in one pass: out_host-less, writes 3 int64 to DEVICE
 * memory stats[3] = {min, max, is_sorted(0/1)} (n_index == 0 -> {0, -1, 1}). */
int b200mp_index_stats(const void* index, int64_t n_index, int64_t* stats, int idx_dtype,
                       void* stream);
/* Stable sort of keys in [0, n_nodes): writes keys_sorted (optional, may be NULL), perm (the
 * stable argsort, idx_dtype) and ptr (optional, n_nodes+1, the CSR pointer of the sorted keys).
 * Workspace size from b200mp_sort_workspace_bytes(). */
int64_t b200mp_sort_workspace_bytes(int64_t n_index, int64_t n_nodes, int idx_dtype);
int b200mp_sort_by_key(const void* keys, int64_t n_index, int64_t n_nodes, void* keys_sorted,
                       void* perm, void* ptr, void* workspace, int64_t workspace_bytes,
                       int idx_dtype, void* stream);
/* out[i] = in[perm[i]] for 4- or 8-byte elements (elem_bytes), perm has idx_dtype. */
int b200mp_permute(const void* in, const void* perm, void* out, int64_t n, int elem_bytes,
                   int idx_dtype, void* stream);
/* Narrowing / widening copy between index dtypes (int64 <-> int32). */
int b200mp_convert_index(const void* in, int in_dtype, void* out, int out_dtype, int64_t n,
                         void* stream);
/* Self-loop handling.  Output order is the reference's: all non-loop edges in input order, then
 * (i,i) for i in [0, n_nodes).  w_in/w_out may be NULL.  mode 0 = add_remaining_self_loops
 * (existing loop weights override fill_value; duplicate loops: the LAST in input order wins,
 * which is the reference's CPU behaviour), mode 1 = remove_self_loops + add_self_loops(fill).
 * n_out_dev (DEVICE int64) receives E' = #nonloops + n_nodes.  row_out/col_out/w_out need
 * n_edges + n_nodes entries.  Workspace from b200mp_self_loops_workspace_bytes(). */
int64_t b200mp_self_loops_workspace_bytes(int64_t n_edges, int64_t n_nodes, int idx_dtype);
int b200mp_self_loops(const void* row, const void* col, const float* w_in, int64_t n_edges,
                      int64_t n_nodes, float fill_value, int mode, void* row_out, void* col_out,
                      float* w_out, int64_t* n_out_dev, void* workspace, int64_t workspace_bytes,
                      int idx_dtype, void* stream);
/* gcn_norm weights on a destination-sorted (CSR over dst) edge list:
 *   deg[i]  = sum of w over the CSR row i, in order (bit-identical to the reference's CPU
 *             scatter_add_, which visits edges in input order, because the sort is stable);
 *   dinv    = deg^-0.5 with inf -> 0;   w_out[e] = dinv[src[e]] * w[e] * dinv[dst(e)].
 * w may be NULL (all ones).  deg_inv_sqrt (n_nodes floats) is an output too. */
int b200mp_gcn_norm_csr(const void* rowptr, const void* src, const float* w, int64_t n_nodes,
                        int64_t n_edges, float* deg_inv_sqrt, float* w_out, int idx_dtype,
                        void* stream);

/* Long-row plan: rows with more than `chunk` edges are split into chunks of `chunk` edges so no
 * warp ever walks a power-law hub alone.  Two calls: count (writes counts_dev[2] =
 * {n_long_rows, n_chunks} to DEVICE memory; the caller reads them back once per graph), then
 * fill: long_rows[n_long_rows] (ascending row ids) and chunk_ptr[n_long_rows + 1] (exclusive scan
 * of ceil(deg / chunk)), both int64.  Workspace from b200mp_csr_plan_workspace_bytes(). */
int b200mp_csr_plan_count(const void* rowptr, int64_t n_rows, int64_t chunk, int64_t* counts_dev,
                          int idx_dtype, void* stream);
int64_t b200mp_csr_plan_workspace_bytes(int64_t n_rows, int64_t n_long_rows, int idx_dtype);
int b200mp_csr_plan_fill(const void* rowptr, int64_t n_rows, int64_t chunk, int64_t n_long_rows,
                         int64_t* long_rows, int64_t* chunk_ptr, void* workspace,
                         int64_t workspace_bytes, int idx_dtype, void* stream);

/* ------------------------------------------------------------------ gather + segmented reduce (the hot path)
 * out[i, :] = REDUCE_{e in [rowptr[i], rowptr[i+1])} val[e] * x[col[e], :]
 * Replaces: MessagePassing._collect/_lift index_select + message + aggregate
 * (nn/conv/message_passing.py:263-333,577-595; collect.jinja:118-139; aggr/base.py:173-185),
 * utils/_spmm.py:12-136, EdgeIndex.matmul (edge_index.py:1903-1970),
 * torch.ops.torch_sparse.spmm_{sum,mean,min,max} (edge_index.py:1798-1810).
 * Semantics are the reference's: empty rows -> 0 for every reduce; mean divides by
 * max(deg, 1); val (fp32, nullable) multiplies before the reduction; the weighted product is
 * rounded before the add (no FMA contraction) so that rows walked by a single lane group in CSR
 * order reproduce the reference's CPU results bit for bit.
 * x: [n_cols, feat], out: [n_rows, feat], both val_dtype.
 * Long rows: pass the plan (long_rows, chunk_ptr, n_long_rows, n_chunks, chunk) and a partials
 * workspace of n_chunks * feat fp32, or n_long_rows = 0 to walk every row with one lane group.
 * bias (nullable, feat fp32) is added to every output row in the epilogue (GCNConv's `out + bias`,
 * gcn_conv.py:265-266, without a second pass over [N, F]).
 * x_halo (nullable): second source segment for node-sharded runs -- column ids >= n_local_cols
 * are read from x_halo[c - n_local_cols, :] (the rows received by the halo all_to_all) so local
 * and remote rows are never concatenated (n_cols = n_local_cols + #halo rows).
 * flags bit 0 (accumulate, sum only, no bias): out[i,:] += result for rows that have edges and
 * rows without edges are left untouched -- adds the halo-edge part after the local-edge sweep.
 * peer_ptrs (nullable, DEVICE array of uint64 addresses, one per GPU) + peer_rows: the source
 * matrix is sharded by contiguous row ranges of peer_rows rows over the GPUs of the box and
 * peer_ptrs[r] is rank r's peer-mapped base address (torch symmetric memory / CUDA IPC); column c
 * is then gathered from peer_ptrs[c / peer_rows] + (c % peer_rows) * row_bytes, i.e. remote rows
 * come straight over NVLink inside this kernel -- the collective is fused into the gather.
 * relu_mask (nullable, with flags bit 0): a [n_rows, feat] matrix of val_dtype; after the accumulate, out[i,f] is
 * zeroed where relu_mask[i,f] <= 0 (rows without edges too) -- the ReLU backward of the producing layer fused into the
 * last writer of its gradient (a layer's input x = relu(pre) is its own mask). */
int b200mp_spmm_csr(const void* rowptr, const void* col, const float* val, const void* x,
                    void* out, int64_t n_rows, int64_t n_cols, int64_t feat, int reduce,
                    const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                    int64_t n_chunks, int64_t chunk, float* partials, const float* bias,
                    const void* x_halo, int64_t n_local_cols, int flags, const void* peer_ptrs,
                    int64_t peer_rows, const void* relu_mask, int idx_dtype, int val_dtype, void* stream);

/* The transposed sweep of GCNConv's backward with its bias gradient: b200mp_spmm_csr's weighted sum over the
 * transposed CSR (rowptr_t, col_t, val_t; reduce sum, val_t required; no bias, halo, peer table, accumulate or
 * relu_mask), out[j, :] = sum_e val_t[e] * x[col_t[e], :], that also returns colsum_out[f] = sum_i x[i, f] in fp32.
 * It needs a square graph in which every row i holds exactly one edge with col_t == i (GCN's self-loops, which the
 * CSR and its transpose both have): the sweep adds the x row of that edge, already loaded for the sum, so the column
 * sum costs no second read of x.  out is bit-identical to b200mp_spmm_csr's.  x: [n_rows, feat].  Long rows: the
 * transposed CSR's plan (long_rows_t, chunk_ptr_t, n_long_rows_t, n_chunks_t, chunk) and partials_t as in
 * b200mp_spmm_csr.  colsum_parts: caller-owned fp32 workspace [n_parts, feat]: one row per CTA of the sweep (a grid
 * of resident CTAs, 8 per SM) and, behind them, the second level of the fold (b200mp_column_sum); pass 16 * #SMs.  The
 * column sum is deterministic on a given device.  Rows that are not whole 16-byte vectors, and rows so wide (above 3072
 * values) that the per-warp column slots pass 48 KB of shared memory, take the plain sweep and b200mp_column_sum. */
int b200mp_spmm_csr_self_colsum(const void* rowptr_t, const void* col_t, const float* val_t, const void* x, void* out,
                                float* colsum_out, int64_t n_rows, int64_t feat, const int64_t* long_rows_t,
                                const int64_t* chunk_ptr_t, int64_t n_long_rows_t, int64_t n_chunks_t, int64_t chunk,
                                float* partials_t, float* colsum_parts, int64_t n_parts, int idx_dtype, int val_dtype,
                                void* stream);

/* Segmented reduce without gather: out[i,:] = REDUCE_{e in [ptr[i], ptr[i+1])} src[e,:].
 * Replaces utils/_segment.py:11-50 (torch._segment_reduce / torch_scatter.segment_csr) and the
 * sorted-index case of utils/_scatter.py:14-138.  Same empty-segment and +-inf -> 0 rules.
 * Long segments (hub destinations): optional long-row plan as in b200mp_spmm_csr (n_long_rows = 0: none). */
int b200mp_segment_csr(const void* ptr, const void* src, void* out, int64_t n_rows, int64_t n_src,
                       int64_t feat, int reduce, const int64_t* long_rows, const int64_t* chunk_ptr,
                       int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                       int idx_dtype, int val_dtype, void* stream);

/* Backward of min/max aggregation (ATen scatter_reduce rule: the gradient is split evenly among
 * tied extrema, and the zero-initialised output counts as one more tie when the extremum is
 * exactly 0 -- see oracle/mp_oracle.c oracle_scatter_backward).  Works on the TRANSPOSED CSR
 * (rows = source nodes, colT[e] = destination of that edge, valT = its weight):
 *   grad_x[j,:] = sum_{e in rowT(j)} [valT[e]*x[j,:] == out[colT[e],:]] * valT[e] * g[colT[e],:] / ties[colT[e],:]
 * ties [n_dst, feat] fp32 is produced by b200mp_minmax_ties on the forward CSR. */
int b200mp_minmax_ties(const void* rowptr, const void* col, const float* val, const void* x,
                       const void* out, float* ties, int64_t n_rows, int64_t feat,
                       int count_self_zero, int idx_dtype, int val_dtype, void* stream);
int b200mp_minmax_backward(const void* rowptr_t, const void* col_t, const float* val_t,
                           const void* x, const void* out, const void* grad_out, const float* ties,
                           void* grad_x, int64_t n_src, int64_t feat, int idx_dtype,
                           int val_dtype, void* stream);

/* Edge-wise dot product (SDDMM): dot[e] = sum_f a[row_of(e), f] * b[col[e], f] over a CSR.
 * This is the gradient of b200mp_spmm_csr(sum) wrt val: a = grad_out, b = x.
 * Replaces the value-gradient branch of _scatter_spmm (edge_index.py:1950-1953). */
int b200mp_sddmm_csr(const void* rowptr, const void* col, const void* a, const void* b, float* dot,
                     int64_t n_rows, int64_t feat, int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ edge-feature message relu(x_j + e_ji)
 * out[i, :] = REDUCE_{e in [rowptr[i], rowptr[i+1])} relu(x[col[e], :] + edge_rows[eid(e), :]), REDUCE = sum | mean,
 * eid(e) = perm[e] (CSR slot -> caller's edge id; NULL for an adopted CSR whose order is the caller's).
 * Replaces: GINEConv.message + aggregate (nn/conv/gin_conv.py:195-204 with message_passing.py:263-333,577-595 and
 * aggr/base.py:173-185): the reference materialises x_j, x_j + edge_attr and its ReLU, three [E, F] tensors.
 * x: [n_cols, feat], edge_rows: [n_edges, feat] in the caller's edge order (read through perm, never permuted), out:
 * [n_rows, feat], all val_dtype.  x + edge_rows is rounded to val_dtype before the ReLU (the reference adds in that
 * dtype); relu(NaN) = NaN; fp32 accumulation in CSR order; mean divides by max(deg, 1); empty rows give 0.
 * Long rows: plan and partials as in b200mp_spmm_csr.  Every CSR slot belongs to a row (rowptr[n_rows] == n_edges).
 * mask (nullable: inference) receives the ReLU mask, n_edges * ceil(feat / 8) bytes in CSR order: bit f % 8 of byte
 * [e * ceil(feat / 8) + f / 8] is set iff !(x + edge_rows <= 0) -- threshold_backward's rule (gradient 0 at 0, passed
 * through at NaN).  The backward entries below read it. */
int b200mp_edge_relu_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                         const void* edge_rows, void* out, void* mask, int64_t n_rows, int64_t n_cols,
                         int64_t n_edges, int64_t feat, int reduce, const int64_t* long_rows,
                         const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                         float* partials, int idx_dtype, int val_dtype, void* stream);
/* grad_x of b200mp_edge_relu_csr over the TRANSPOSED CSR (replaces the index_select backward, an index_add_ with
 * atomics, and the ReLU backward of gin_conv.py:204):
 *   grad_x[j, :] = sum_{t in rowT(j)} mask(t2csr[t]) ? val_t[t] * grad_out[col_t[t], :] : 0
 * t2csr[t] = the CSR slot of transposed slot t; val_t (nullable, fp32) = 1 / max(deg, 1) of the destination for mean.
 * Long source rows: the transposed CSR's plan and partials. */
int b200mp_edge_relu_backward_x(const void* rowptr_t, const void* col_t, const void* t2csr,
                                const float* val_t, const void* grad_out, const void* mask, void* grad_x,
                                int64_t n_src, int64_t feat, const int64_t* long_rows,
                                const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                int64_t chunk, float* partials, int idx_dtype, int val_dtype, void* stream);
/* grad_edge_rows of b200mp_edge_relu_csr, in the caller's edge order (the ReLU backward of gin_conv.py:204):
 *   grad_edge_rows[eid(e), :] = mask(e) ? grad_out[i, :] / (mean ? max(deg_i, 1) : 1) : 0,  e in row i
 * with the quotient rounded to val_dtype.  Every CSR slot is written once; the plan (no partials) splits hub rows. */
int b200mp_edge_relu_backward_edge(const void* rowptr, const void* perm, const void* grad_out,
                                   const void* mask, void* grad_edge_rows, int64_t n_rows, int64_t feat,
                                   int reduce, const int64_t* long_rows, const int64_t* chunk_ptr,
                                   int64_t n_long_rows, int64_t n_chunks, int64_t chunk, int idx_dtype,
                                   int val_dtype, void* stream);

/* ------------------------------------------------------------------ gated message sigmoid(k_i + q_j) * v_j
 * out[i, :] = REDUCE_{e in [rowptr[i], rowptr[i+1])} sigmoid(s_e) * v[col[e], :],  s_e = k[i, :] + q[col[e], :],
 * REDUCE = sum | mean.
 * Replaces: ResGatedGraphConv.message + aggregate (nn/conv/res_gated_graph_conv.py:128-148 with
 * message_passing.py:263-333 and aggr/base.py:173-185): the reference materialises k_i, q_j, v_j, their sum, its
 * sigmoid and the product, six [E, F] tensors.
 * k: [n_rows, feat]; q, v: [n_cols, feat] rows with a shared row stride `ld` >= feat in elements (two tensors, or the
 * two halves of one [n_cols, 2 feat] product); out: [n_rows, feat]; all val_dtype.  s_e, sigmoid(s_e) and the product
 * are each rounded to val_dtype (the reference's add, sigmoid and mul); fp32 accumulation in CSR order; mean divides
 * by max(deg, 1); empty rows give 0.  Long rows: plan and partials ([n_chunks, feat] fp32) as in b200mp_spmm_csr. */
int b200mp_gated_csr(const void* rowptr, const void* col, const void* k, const void* q, const void* v,
                     void* out, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld,
                     int reduce, const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                     int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                     void* stream);
/* grad_k of b200mp_gated_csr over the destination CSR (replaces the autograd of res_gated_graph_conv.py:148 wrt k_i:
 * mul, sigmoid and add backward, then the index_select backward, an index_add_ with atomics):
 *   grad_k[i, :] = g_i * sum_{e in row i} v[col[e], :] * sigmoid'(s_e),  g_i = grad_out[i, :] / (mean ? max(deg_i, 1) : 1)
 * grad_k: [n_rows, feat]; 0 for a row without edges.  Long rows: plan and partials ([n_chunks, feat] fp32). */
int b200mp_gated_backward_dst(const void* rowptr, const void* col, const void* k, const void* q,
                              const void* v, const void* grad_out, void* grad_k, int64_t n_rows,
                              int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld, int reduce,
                              const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                              int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype,
                              int val_dtype, void* stream);
/* grad_q and grad_v of b200mp_gated_csr in ONE sweep over the TRANSPOSED CSR (replaces the autograd of
 * res_gated_graph_conv.py:148 wrt q_j and v_j and its two index_add_ scatters):
 *   grad_v[j, :] = sum_{t in rowT(j)} sigmoid(s_t) * w_t * grad_out[col_t[t], :]
 *   grad_q[j, :] = v[j, :] * sum_{t in rowT(j)} sigmoid'(s_t) * w_t * grad_out[col_t[t], :]
 * s_t = k[col_t[t], :] + q[j, :] rounded to val_dtype; w_t = val_t[t] (nullable, fp32: 1 / max(deg, 1) of the
 * destination for mean) or 1.  grad_q, grad_v: [n_src, feat] rows with q's and v's stride `ld`; 0 for a source
 * without out-edges.  Long source rows: the transposed CSR's plan, partials [n_chunks, 2 feat] fp32. */
int b200mp_gated_backward_src(const void* rowptr_t, const void* col_t, const float* val_t, const void* k,
                              const void* q, const void* v, const void* grad_out, void* grad_q,
                              void* grad_v, int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t feat,
                              int64_t ld, const int64_t* long_rows, const int64_t* chunk_ptr,
                              int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                              int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ crystal-graph message sigmoid(f) * softplus(s)
 * out[i, :] = REDUCE_{e in [rowptr[i], rowptr[i+1])} sigmoid(f_e) * softplus(s_e),  REDUCE = sum | mean, with
 * f_e = u[i, 0:F] + v[col[e], 0:F] (+ c[eid(e), 0:F]) and s_e = u[i, F:2F] + v[col[e], F:2F] (+ c[eid(e), F:2F]).
 * Replaces: CGConv.message + aggregate (nn/conv/cg_conv.py:93-98 with message_passing.py:263-333 and
 * aggr/base.py:173-185): the reference materialises x_i, x_j, their concatenation with edge_attr, both Linear outputs,
 * the sigmoid, the softplus and the product, all [E, *] tensors.  u and v are the per-node column blocks of both
 * Linears (u carries the biases), c the edge_attr block.
 * u: [n_rows, 2F] rows with row stride ld_u >= 2F; v: [n_cols, 2F] rows with stride ld_v >= 2F (u and v may be the
 * two halves of one [N, 4F] product); c: [n_edges, 2F] contiguous in the CALLER's edge order, or NULL; eid(e) =
 * perm[e], or e when perm is NULL (an adopted CSR); out: [n_rows, F]; all val_dtype.  f and s are summed in fp32 and
 * rounded to val_dtype once (the reference's Linear output); sigmoid, softplus (ATen threshold 20) and their product
 * are each rounded to val_dtype; fp32 accumulation in CSR order; mean divides by max(deg, 1); empty rows give 0.
 * Long rows: plan and partials ([n_chunks, F] fp32) as in b200mp_spmm_csr. */
int b200mp_cg_csr(const void* rowptr, const void* col, const void* perm, const void* u, const void* v,
                  const void* c, void* out, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat,
                  int64_t ld_u, int64_t ld_v, int reduce, const int64_t* long_rows,
                  const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                  float* partials, int idx_dtype, int val_dtype, void* stream);
/* grad_u (and grad_c) of b200mp_cg_csr over the destination CSR (replaces the autograd of cg_conv.py:98 wrt x_i and
 * edge_attr: mul, sigmoid, softplus and Linear backward over E rows, then the index_select backward through
 * index_add_ atomics).  With g_i = grad_out[i, :] / (mean ? max(deg_i, 1) : 1):
 *   df_e = g_i * sigmoid'(f_e) * softplus(s_e),  ds_e = g_i * sigmoid(f_e) * softplus'(s_e)
 *   grad_u[i, :] = sum_{e in row i} [df_e | ds_e]   ([n_rows, 2F] rows with stride ld_u; 0 for a row without edges)
 *   grad_c[eid(e), :] = [df_e | ds_e]               ([n_edges, 2F], caller's edge order; NULL: not written;
 *                                                    given only with c)
 * Long rows: plan and partials ([n_chunks, 2F] fp32). */
int b200mp_cg_backward_dst(const void* rowptr, const void* col, const void* perm, const void* u,
                           const void* v, const void* c, const void* grad_out, void* grad_u, void* grad_c,
                           int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int64_t ld_u,
                           int64_t ld_v, int reduce, const int64_t* long_rows, const int64_t* chunk_ptr,
                           int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                           int idx_dtype, int val_dtype, void* stream);
/* grad_v of b200mp_cg_csr by ONE sweep over the TRANSPOSED CSR (replaces the index_select backward wrt x_j):
 *   grad_v[j, :] = sum_{t in rowT(j)} [df_t | ds_t] with g = w_t * grad_out[col_t[t], :]
 * w_t = val_t[t] (nullable, fp32: 1 / max(deg, 1) of the destination for mean) or 1; c is read at perm_t[t], the
 * caller's edge id of transposed slot t.  grad_v: [n_src, 2F] rows with stride ld_v; 0 for a source without
 * out-edges.  When grad_c was written, the segment sum of its rows (b200mp_spmm_csr over rowptr_t with perm_t as the
 * column) gives the same grad_v with fewer bytes.  Long source rows: the transposed CSR's plan, partials
 * [n_chunks, 2F] fp32. */
int b200mp_cg_backward_src(const void* rowptr_t, const void* col_t, const void* perm_t, const float* val_t,
                           const void* u, const void* v, const void* c, const void* grad_out, void* grad_v,
                           int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t feat, int64_t ld_u,
                           int64_t ld_v, const int64_t* long_rows, const int64_t* chunk_ptr,
                           int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                           int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ softmax aggregation (online softmax, one sweep)
 * Per destination i, feature f, in-edge e = (j -> i) in [rowptr[i], rowptr[i+1]), eid(e) = perm[e] or e (perm NULL):
 *   s_e = x[col[e]] + edge_rows[eid(e)] (rounded) | x[col[e]] | edge_rows[eid(e)]
 *   m_e = relu(s_e) + eps (message 1: each step rounded, relu keeps NaN)  |  s_e (message 0)
 *   z_e = t * m_e rounded (t_mode 1: t[0], 2: t[f]) | m_e (t_mode 0)
 *   out[i, f] = sum_e exp(z_e - M) m_e / (sum_e exp(z_e - M) + 1e-16),  M = max_e z_e;  0 for an empty row
 * Replaces: SoftmaxAggregation.forward (nn/aggr/basic.py:196-215) with utils/_softmax.py:60-92 (scatter max, exp,
 * scatter sum, divide, multiply, scatter sum: six [E, F] passes), and GENConv.message (nn/conv/gen_conv.py:231-239).
 * message 1 needs x (edge_rows optional); message 0 takes exactly one of x and edge_rows.  t: [1] or [feat] fp32
 * (read on the device: a learnable t costs no host read; t * m is formed in fp32 and rounded to val_dtype).  x: [n_cols, feat]; edge_rows: [n_edges, feat] in
 * the CALLER's edge order; out: [n_rows, feat]; lse: NULL or [n_rows, feat] fp32 = M + log(S + 1e-16), the only state
 * the backward needs (NaN where M = +inf: the reference's inf - inf).  One exponential per (edge, feature) by a running
 * (M, S, A); fp32 accumulation.  Long rows: plan as in b200mp_spmm_csr, partials [n_chunks, 3 feat] fp32, merged in
 * chunk order by a second launch. */
int b200mp_softmax_aggr_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                            const void* edge_rows, const float* t, void* out, float* lse, int64_t n_rows,
                            int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps, int t_mode,
                            const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                            int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                            void* stream);
/* fp32 workspace elements b200mp_softmax_aggr_backward_dst needs for grad_t. */
int64_t b200mp_softmax_aggr_workspace(int64_t n_rows, int64_t n_chunks, int64_t feat);
/* Destination sweep of the backward (replaces the autograd of basic.py:196-215 / _softmax.py:60-92 / gen_conv.py:231-239
 * over [E, F]).  Recomputes m, z and p_e = exp(z_e - lse_i); with g = grad_out[i], o = out[i]:
 *   grad_m_e = g p_e (1 + t (m_e - o))   (semi_grad: g p_e)        grad_s_e = grad_m_e [s_e > 0 or NaN] (message 1)
 *   grad_edge_rows[eid(e)] = grad_s_e  (NULL: not written)          grad_t[f] = sum_i sum_e g p_e m_e (m_e - o)
 * grad_t: NULL or [feat] fp32 (per-channel sums; the caller sums them for a scalar t), from per-CTA partials folded
 * in fixed order by b200mp_column_sum in `workspace` (b200mp_softmax_aggr_workspace elements).  With grad_t, the
 * feat limit of b200mp_power_mean_backward_dst's grad_p applies (B200MP_ERR_UNSUPPORTED beyond it).  The 1e-16 of the
 * forward's denominator is dropped here: the denominator is >= 1, so it is below fp32 resolution. */
int b200mp_softmax_aggr_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                     const void* edge_rows, const float* t, const void* out, const float* lse,
                                     const void* grad_out, void* grad_edge_rows, float* grad_t, float* workspace,
                                     int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int message,
                                     float eps, int t_mode, int semi_grad, const int64_t* long_rows,
                                     const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                     int idx_dtype, int val_dtype, void* stream);
/* grad_x by ONE sweep over the TRANSPOSED CSR: grad_x[j] = sum_{t in rowT(j)} grad_s_t, gathering grad_out, out and
 * lse of col_t[t] and edge_rows[perm_t[t]] (frozen edge rows) per out-edge.  Needs x.  Used when no grad_edge_rows
 * was written; otherwise the segment sum of grad_edge_rows over the transposed CSR (b200mp_spmm_csr with perm_t as
 * the column) gives grad_x with fewer bytes.  Long source rows: the transposed CSR's plan, partials [n_chunks, feat]. */
int b200mp_softmax_aggr_backward_src(const void* rowptr_t, const void* col_t, const void* perm_t, const void* x,
                                     const void* edge_rows, const float* t, const void* out, const float* lse,
                                     const void* grad_out, void* grad_x, int64_t n_src, int64_t n_dst,
                                     int64_t n_edges, int64_t feat, int message, float eps, int t_mode,
                                     int semi_grad, const int64_t* long_rows, const int64_t* chunk_ptr,
                                     int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                     int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ power-mean aggregation (one sweep)
 * Per destination i, feature f, in-edge e = (j -> i) in [rowptr[i], rowptr[i+1]), eid(e) = perm[e] or e (perm NULL),
 * with m_e formed as in b200mp_softmax_aggr_csr (message 0: x[col[e]] | edge_rows[eid(e)]; message 1:
 * relu(x[col[e]] (+ edge_rows[eid(e)])) + eps, each step rounded):
 *   c_e = clamp(m_e, clamp_min, clamp_max)   y_e = c_e ^ p (rounded)   M_i = sum_e y_e / max(deg_i, 1) (rounded)
 *   out[i, f] = clamp(M_i, clamp_min, clamp_max) ^ (1 / p) (rounded)
 * p_mode 0: no clamp and no pow (a plain mean of the messages); 1: p[0]; 2: p[f].  p is fp32 on the device (a learnable
 * p costs no host read); 1 / p is formed in fp32.  With p: clamp_min > 0 and clamp_max >= clamp_min (+inf: no upper
 * bound); the clamp keeps NaN.  An empty row gives clamp_min ^ (1 / p) with p and 0 without.  c ^ p is
 * ex2.approx(p lg2.approx(c)) (csrc/power_mean.cu states the bound); the sum is fp32 and compensated.
 * Replaces: PowerMeanAggregation.forward (nn/aggr/basic.py:275-293: clamp, pow, scatter mean, clamp, pow over [E, F]),
 * behind GENConv.message (nn/conv/gen_conv.py:231-239) with message 1.
 * x: [n_cols, feat]; edge_rows: [n_edges, feat] in the CALLER's edge order; out: [n_rows, feat]; mean: NULL or
 * [n_rows, feat] fp32 = M, the only state the backward needs.  Long rows: plan as in b200mp_spmm_csr, partials
 * [n_chunks, feat] fp32, summed in chunk order by a second launch. */
int b200mp_power_mean_csr(const void* rowptr, const void* col, const void* perm, const void* x,
                          const void* edge_rows, const float* p, void* out, float* mean, int64_t n_rows,
                          int64_t n_cols, int64_t n_edges, int64_t feat, int message, float eps, int p_mode,
                          float clamp_min, float clamp_max, const int64_t* long_rows, const int64_t* chunk_ptr,
                          int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype,
                          int val_dtype, void* stream);
/* fp32 workspace elements of the power-mean backward: b200mp_power_mean_backward_dst over n_rows destination rows
 * (n_node = 0), or b200mp_power_mean_backward_src over n_rows source rows of the transposed CSR with n_node = n_dst
 * (its node plane). */
int64_t b200mp_power_mean_workspace(int64_t n_node, int64_t n_rows, int64_t n_chunks, int64_t feat);
/* Destination sweep of the backward (replaces the autograd of basic.py:275-293 / gen_conv.py:231-239 over [E, F]).
 * Recomputes m, c and y; with g = grad_out[i], o = out[i] and C_i = clamp(M_i):
 *   G_i = g (1/p) C_i ^ (1/p - 1) / max(deg_i, 1) [clamp_min <= M_i <= clamp_max]   (p_mode 0: g / max(deg_i, 1))
 *   grad_m_e = G_i p c_e ^ (p - 1) [clamp_min <= m_e <= clamp_max]     grad_s_e = grad_m_e [s_e > 0 or NaN] (message 1)
 *   grad_edge_rows[eid(e)] = grad_s_e (NULL: not written)
 *   grad_p[f] = sum_i sum_e G_i y_e ln c_e - sum_i g o ln C_i / p^2     (the second sum includes empty rows)
 * grad_p: NULL or [feat] fp32 (per-channel sums; the caller sums them for a scalar p), from per-CTA partials folded in
 * fixed order by b200mp_column_sum in `workspace` (b200mp_power_mean_workspace(0, n_rows, n_chunks, feat)).  With
 * grad_p, feat is at most about 7,000 on the scalar path and 14,000 on the 16-byte vector path: wider rows return
 * B200MP_ERR_UNSUPPORTED before anything is launched, because each lane group keeps one fp32 row of grad_p partials
 * in shared memory.  b200mp_power_mean_backward_src has the same limit. */
int b200mp_power_mean_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x,
                                   const void* edge_rows, const float* p, const void* out, const float* mean,
                                   const void* grad_out, void* grad_edge_rows, float* grad_p, float* workspace,
                                   int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, int message,
                                   float eps, int p_mode, float clamp_min, float clamp_max, const int64_t* long_rows,
                                   const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                                   int idx_dtype, int val_dtype, void* stream);
/* grad_x (and grad_p) by ONE sweep over the TRANSPOSED CSR: a node kernel first writes G_i of every destination into
 * `workspace` (b200mp_power_mean_workspace(n_dst, n_src, n_chunks, feat)) with the per-row grad_p terms, then
 * grad_x[j] = sum_{t in rowT(j)} grad_s_t gathers one fp32 row of G at col_t[t] and edge_rows[perm_t[t]] (frozen edge
 * rows) per out-edge.  rowptr: the destination CSR's (for the degrees).  Needs x.  Used when no grad_edge_rows was
 * written; otherwise the segment sum of grad_edge_rows over the transposed CSR (b200mp_spmm_csr with perm_t as the
 * column) gives grad_x with fewer bytes.  Long source rows: the transposed CSR's plan, partials [n_chunks, feat]. */
int b200mp_power_mean_backward_src(const void* rowptr, const void* rowptr_t, const void* col_t, const void* perm_t,
                                   const void* x, const void* edge_rows, const float* p, const void* out,
                                   const float* mean, const void* grad_out, void* grad_x, float* grad_p,
                                   float* workspace, int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t feat,
                                   int message, float eps, int p_mode, float clamp_min, float clamp_max,
                                   const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                                   int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                                   void* stream);

/* ------------------------------------------------------------------ quantile aggregation (one selection sweep)
 * Replaces: QuantileAggregation.forward / MedianAggregation (nn/aggr/quantile.py:71-130: a column-wise sort of the
 * [E, F] messages, a stable sort of an expanded int64 [E, F] index and two gathers).  Per destination i (count_i
 * in-edges from offset ptr_i = rowptr[i]), channel f and q = q[k] (fp32 on the device, n_q >= 1):
 *   h = fl32(q fl32(count_i - 1)),  P = fl32(h + fl32(ptr_i))   (quantile.py:88; exact integer offsets once
 *   ptr_i + count_i - 1 >= 2^24, where the reference's fp32 P leaves the group; every rank is then clamped into
 *   [0, count_i - 1], as fl32(count_i - 1) may round up past 2^24)
 *   interpolation 0 linear: l + (r - l) frac   1 lower: floor(P)   2 higher: ceil(P)   3 nearest: rint(P) (half to even)
 *   4 midpoint: 0.5 l + 0.5 r   -- l, r the values of rank floor(P) - ptr_i and ceil(P) - ptr_i, frac = P - floor(P)
 * Ranks order the messages by value (-0.0 == +0.0, NaN above +inf), ties by CSR slot (the caller's order).  Each op
 * rounds as ATen's; bf16 linear writes fp32 (the reference's promotion), every other case the messages' dtype.  An
 * empty row gives fill_value.  out: [n_rows, n_q * feat], row i = [q_0 | q_1 | ...] (quantile.py:125-129).
 * Messages: x [n_cols, feat] gathered through col, or edge_rows [n_edges, feat] in the CALLER's order read through perm
 * (NULL: the slot).  bits: NULL, or the saved state of the backward, b200mp_quantile_bits_words(...) uint32 words
 * [n_edges (caller order), R n_q, ceil(feat / 32)], R = 2 for linear and midpoint (floor picks, then ceil picks) and 1
 * otherwise; zeroed and written here.  plan_*: the destination CSR's long-row plan (b200mp_csr_plan_*): its rows are
 * selected by one CTA per 32 channels; no partials.  csrc/quantile.cu states the algorithm. */
int64_t b200mp_quantile_bits_words(int64_t n_edges, int64_t n_q, int interpolation, int64_t feat);
int b200mp_quantile_csr(const void* rowptr, const void* col, const void* perm, const void* x, const void* edge_rows,
                        const float* q, int64_t n_q, int interpolation, float fill_value, void* out, uint32_t* bits,
                        int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t feat, const int64_t* plan_rows,
                        const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks, int64_t plan_chunk,
                        int idx_dtype, int val_dtype, void* stream);
/* The gradient of the edge rows, written densely in the caller's order (quantile.py's autograd: the sort, gathers and
 * index_select backward): g = grad_out[i, k feat + f] (fp32 for bf16 linear, else the messages' dtype) goes to each
 * picked element as g (lower, higher, nearest), round(0.5 g) (midpoint), or g - g frac and g frac (linear; bf16:
 * round(round(g) - round(g frac)) and round(g frac)); an element's picks are summed over q in order, each add rounded,
 * the floor picks' sum then plus the ceil picks'.  Reads only bits, q and grad_out.  plan_*: the destination CSR's plan
 * (long rows split into chunks; no partials). */
int b200mp_quantile_backward_dst(const void* rowptr, const void* perm, const float* q, int64_t n_q, int interpolation,
                                 const uint32_t* bits, const void* grad_out, void* grad_edge_rows, int64_t n_rows,
                                 int64_t n_edges, int64_t feat, const int64_t* plan_rows,
                                 const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks,
                                 int64_t plan_chunk, int idx_dtype, int val_dtype, void* stream);
/* grad_x of the gathered form by ONE sweep over the TRANSPOSED CSR: grad_x[j] = the fp32 sum, in transposed slot
 * order, of the per-message gradient above over j's out-edges t (message perm_t[t], destination col_t[t]), read only
 * where a bit is set; rounded once to the messages' dtype.  A long source row is summed per plan chunk and the chunk
 * sums are folded in chunk order.  rowptr: the destination CSR's (offsets and counts).
 * plan_*: the transposed CSR's plan, partials [plan_n_chunks, feat] fp32, folded in chunk order. */
int b200mp_quantile_backward_src(const void* rowptr, const void* rowptr_t, const void* col_t, const void* perm_t,
                                 const float* q, int64_t n_q, int interpolation, const uint32_t* bits,
                                 const void* grad_out, void* grad_x, int64_t n_src, int64_t n_dst, int64_t n_edges,
                                 int64_t feat, const int64_t* plan_rows, const int64_t* plan_chunk_ptr,
                                 int64_t plan_n_long, int64_t plan_n_chunks, int64_t plan_chunk, float* plan_partials,
                                 int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ NNConv / ECConv (edge-conditioned message)
 * Replaces: NNConv.message + aggregate (nn/conv/nn_conv.py:96-122: the edge network's [E, F_in F_out] output viewed as
 * one F_in x F_out matrix per edge, a batched x_j product into [E, F_out], then scatter).  With the edge network's last
 * Linear split off, h [E, K] (the output of everything before it, in the CALLER's edge order, read through perm; NULL
 * perm: the slot) and h~_e = [h_e, 1], the sweep writes for destination rows [row_begin, row_end) of the CSR
 *   P[i - row_begin, k F_in + a] = sum_{e = (j -> i)} h~_e[k] x[j, a]     (fp32; mean: / max(deg_i, 1))
 * and out = P W' with W' [(K+1) F_in, F_out] from the last Linear's weight and bias is the caller's GEMM.  Rows
 * without edges give 0.  Supported: K >= 0, F_in >= 1, (K + 1) F_in <= 16384 (dP_i of 64 KiB in shared memory in the
 * backward); else B200MP_ERR_UNSUPPORTED.  reduce: SUM or MEAN.  plan_*: the destination CSR's long-row plan, partials
 * [plan_n_chunks, (K+1) F_in] fp32 folded in chunk order (chunks of rows outside the range are skipped). */
int b200mp_nn_conv_supported(int64_t k, int64_t fin, int val_dtype);
int b200mp_nn_conv_csr(const void* rowptr, const void* col, const void* perm, const void* x, const void* h, float* p,
                       int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t k, int64_t fin, int64_t row_begin,
                       int64_t row_end, int reduce, const int64_t* plan_rows, const int64_t* plan_chunk_ptr,
                       int64_t plan_n_long, int64_t plan_n_chunks, int64_t plan_chunk, float* plan_partials,
                       int idx_dtype, int val_dtype, void* stream);
/* The destination half of the backward (nn_conv.py:119-122 under autograd) for rows [row_begin, row_end): grad_p =
 * dL/dP of those rows, fp32 in P's layout (the caller's G W'^T).  Per edge e = (j -> i), in the caller's order:
 *   grad_h[e, k] = sum_a x[j, a] grad_p[i, k F_in + a]  (k < K)      q[e, a] = sum_{k <= K} h~_e[k] grad_p[i, k F_in + a]
 * each divided by max(deg_i, 1) for mean and rounded once to the value dtype.  grad_h or q may be NULL (not written).
 * grad_x is the segment sum of q's rows over the transposed CSR (b200mp_spmm_csr with perm_t as the column).
 * plan_*: the destination CSR's plan (hub rows split into chunks; no partials: no combine step). */
int b200mp_nn_conv_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x, const void* h,
                                const float* grad_p, void* grad_h, void* q, int64_t n_rows, int64_t n_cols,
                                int64_t n_edges, int64_t k, int64_t fin, int64_t row_begin, int64_t row_end, int reduce,
                                const int64_t* plan_rows, const int64_t* plan_chunk_ptr, int64_t plan_n_long,
                                int64_t plan_n_chunks, int64_t plan_chunk, int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ SplineConv (B-spline basis and weighting)
 * Supported: degree 1..3, S = (degree + 1)^D basis slots per edge with 1 <= S <= 64; the fused sweeps also need
 * K >= 1, F_in >= 1 and K F_in <= 16384 (P_i in shared memory); else B200MP_ERR_UNSUPPORTED.  Values fp32 or bf16. */
int b200mp_spline_supported(int64_t k, int64_t fin, int64_t s, int val_dtype);
/* Replaces pyg_lib.ops.spline_basis (spline_conv.py:151-152).  pseudo [E, D] (val_dtype), kernel_size [D] int64,
 * is_open_spline [D] uint8, all on the device.  Writes basis [E, S] (val_dtype) and weight_index [E, S] (wi_dtype,
 * B200MP_I32 or B200MP_I64): for slot s, with k_d the d-th base-(degree+1) digit of s (dimension 0 fastest) and
 * v_d = pseudo[e, d] * (kernel_size[d] - degree * is_open_spline[d]) in fp32,
 *   weight_index = sum_d ((floor(v_d) + k_d) mod kernel_size[d]) prod_{d' < d} kernel_size[d'],  basis = prod_d B(t_d, k_d)
 * with t_d = v_d - floor(v_d).  The modulo is non-negative and kernel sizes below 1 count as 1, so pseudo outside
 * [0, 1] gives indices in [0, K) (the reference leaves that case undefined). */
int b200mp_spline_basis(const void* pseudo, const int64_t* kernel_size, const uint8_t* is_open_spline, void* basis,
                        void* weight_index, int64_t n_edges, int64_t dim, int degree, int val_dtype, int wi_dtype,
                        void* stream);
/* The basis's backward (pyg_lib.ops.spline_basis under autograd): grad_pseudo [E, D] = sum_s grad_basis[e, s] d basis[e, s]
 * / d pseudo[e, d] in fp32, in slot order, rounded once to val_dtype. */
int b200mp_spline_basis_backward(const void* grad_basis, const void* pseudo, const int64_t* kernel_size,
                                 const uint8_t* is_open_spline, void* grad_pseudo, int64_t n_edges, int64_t dim,
                                 int degree, int val_dtype, void* stream);
/* Replaces pyg_lib.ops.spline_weighting (spline_conv.py:153): out[e] = sum_s basis[e, s] x[e] @ weight[wi[e, s]] for
 * x [E, F_in], weight [K, F_in, F_out], basis and weight_index [E, S] (idx_dtype) -- the standalone, unfused op.
 * A slot whose index lies outside [0, K) contributes nothing. */
int b200mp_spline_weighting(const void* x, const void* weight, const void* basis, const void* weight_index, void* out,
                            int64_t n_edges, int64_t fin, int64_t fout, int64_t k, int64_t s, int idx_dtype,
                            int val_dtype, void* stream);
/* Its backward; each of grad_x [E, F_in], grad_basis [E, S] (val_dtype) and grad_weight [K, F_in, F_out] (fp32) may be
 * NULL (not computed).  grad_weight needs slot_order (the flat slot ids e S + s sorted by weight index, stably) and
 * slot_ptr [K + 1] (where each kernel's slots begin in it), both of idx_dtype; each kernel's slots are summed in that
 * order. */
int b200mp_spline_weighting_backward(const void* grad_out, const void* x, const void* weight, const void* basis,
                                     const void* weight_index, const void* slot_order, const void* slot_ptr,
                                     void* grad_x, void* grad_basis, float* grad_weight, int64_t n_edges, int64_t fin,
                                     int64_t fout, int64_t k, int64_t s, int idx_dtype, int val_dtype, void* stream);
/* Replaces SplineConv.message + aggregate (spline_conv.py:150-153 and the sum / mean scatter) for destination rows
 * [row_begin, row_end) of the CSR: with basis [E, S] (val_dtype) and weight_index [E, S] int32 in the CALLER's edge
 * order, read through perm (NULL: the slot),
 *   P[i - row_begin, k F_in + a] = sum_{e = (j -> i), s : wi[e, s] = k} basis[e, s] x[j, a]   (fp32; mean: / max(deg_i, 1))
 * and out = P weight.view(K F_in, F_out) is the caller's GEMM.  Rows without edges give 0; slots whose index lies outside
 * [0, K) add nothing.  reduce: SUM or MEAN.  plan_*: the destination CSR's long-row plan, partials
 * [plan_n_chunks, K F_in] fp32 folded in chunk order (chunks of rows outside the range are skipped). */
int b200mp_spline_csr(const void* rowptr, const void* col, const void* perm, const void* x, const void* basis,
                      const int32_t* weight_index, float* p, int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t k,
                      int64_t fin, int64_t s, int64_t row_begin, int64_t row_end, int reduce, const int64_t* plan_rows,
                      const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks, int64_t plan_chunk,
                      float* plan_partials, int idx_dtype, int val_dtype, void* stream);
/* The destination half of its backward for rows [row_begin, row_end): grad_p = dL/dP of those rows, fp32 in P's layout
 * (the caller's G weight^T).  Per edge e = (j -> i), in the caller's order, with dP_i divided by max(deg_i, 1) for mean:
 *   grad_basis[e, s] = <dP_i[wi[e, s]], x[j]>        q[e, a] = sum_s basis[e, s] dP_i[wi[e, s], a]
 * rounded once to val_dtype; either may be NULL (not written).  grad_x is the segment sum of q over the transposed CSR.
 * plan_*: the destination CSR's plan (no partials: no combine step). */
int b200mp_spline_backward_dst(const void* rowptr, const void* col, const void* perm, const void* x, const void* basis,
                               const int32_t* weight_index, const float* grad_p, void* grad_basis, void* q,
                               int64_t n_rows, int64_t n_cols, int64_t n_edges, int64_t k, int64_t fin, int64_t s,
                               int64_t row_begin, int64_t row_end, int reduce, const int64_t* plan_rows,
                               const int64_t* plan_chunk_ptr, int64_t plan_n_long, int64_t plan_n_chunks,
                               int64_t plan_chunk, int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ point clouds (k-NN, radius, fps, nearest)
 * Replace pyg_lib.ops.knn / radius / fps / nearest (torch.ops.pyg.*, nn/pool/__init__.py:85,140,199,265,331,375).
 * Points: x [n_x, f], y [n_y, f] row-major (val_dtype, fp32 or bf16, widened exactly to fp32); n_x < 2^31.  Examples:
 * ptr_x [n_ptr_x] / ptr_y [n_ptr_y] (ptr_dtype, one dtype for both) give example b the range ptr[b]:ptr[b+1]; a NULL
 * ptr is one example covering every point, and examples missing at the end of the shorter ptr are empty.
 * Distances: d = sum_f (x_f - y_f)^2, or 1 - dot / (sqrt(|x|^2) sqrt(|y|^2)) under cosine, every sum in feature order with
 * explicitly rounded fp32 operations (no FMA contraction); a candidate is selected only when d compares below something
 * with a strict <, so NaN and infinite distances are never selected.  Outputs are int64; offsets [n + 1] are written as
 * exclusive offsets of the per-query lengths (offsets[n] is the total, the caller's one device-to-host read). */
/* k nearest x points of each query's example, 1 <= k <= 128 (else B200MP_ERR_UNSUPPORTED): slab [2, n_y k] gets, for
 * query i, row i in slab[0, i k + c] and the c-th neighbour in slab[1, i k + c] (distance ascending, ties by ascending x
 * index; -1 past the query's length), and offsets [n_y + 1] the offsets of the lengths.  When offsets[n_y] == n_y k the
 * slab is the [2, nnz] result; otherwise b200mp_knn_compact packs it. */
int b200mp_knn(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y, int64_t f,
               int64_t n_ptr_x, int64_t n_ptr_y, int64_t k, int cosine, int64_t* slab, int64_t* offsets, int val_dtype,
               int ptr_dtype, void* stream);
/* out [2, nnz] = the slab's first offsets[i+1] - offsets[i] entries of each query, queries ascending. */
int b200mp_knn_compact(const int64_t* slab, const int64_t* offsets, int64_t n_y, int64_t k, int64_t* out, int64_t nnz,
                       void* stream);
/* Radius, pass 1: offsets [n_y + 1] of the number of x points of each query's example with d < r2 (squared distance;
 * r2 is the caller's fp64 r * r rounded once to fp32), capped at max_num_neighbors, skipping x index == y index when
 * ignore_same_index is set. */
int b200mp_radius_count(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                        int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, float r2, int64_t max_num_neighbors,
                        int ignore_same_index, int64_t* offsets, int val_dtype, int ptr_dtype, void* stream);
/* Radius, pass 2: out [2, nnz] (nnz = offsets[n_y]) gets (y index, x index) pairs, queries ascending and each query's
 * first max_num_neighbors x points in ascending index order. */
int b200mp_radius_fill(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                       int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, float r2, int64_t max_num_neighbors,
                       int ignore_same_index, const int64_t* offsets, int64_t* out, int64_t nnz, int val_dtype,
                       int ptr_dtype, void* stream);
/* For each x point, the nearest y point of its example (torch-cluster's cluster vector): the k-NN sweep with k = 1 and
 * the roles swapped.  slab [2, n_x] gets (x index, y index or -1), offsets [n_x + 1] the offsets of the lengths (0 or 1):
 * offsets[n_x] < n_x means some x point found no y point. */
int b200mp_nearest(const void* x, const void* y, const void* ptr_x, const void* ptr_y, int64_t n_x, int64_t n_y,
                   int64_t f, int64_t n_ptr_x, int64_t n_ptr_y, int64_t* slab, int64_t* offsets, int val_dtype,
                   int ptr_dtype, void* stream);
/* Farthest-point sampling, pass 1: offsets [B + 1] of ceil(n_b ratio) (fp64) samples per example, 0 < ratio <= 1;
 * B = n_ptr - 1, or 1 when ptr is NULL. */
int b200mp_fps_count(const void* ptr, int64_t n_ptr, int64_t n, double ratio, int64_t* offsets, int ptr_dtype,
                     void* stream);
/* Pass 2: out [offsets[B]] gets each example's samples (global indices) in selection order, examples concatenated.  The
 * start is the example's first point, or point floor(rnd[b] n_b) when rnd [B] (uniform in [0, 1), fp32) is given;
 * each step takes the argmax of the running min squared distance, ties to the lowest index.  dist_ws [n] fp32 is the
 * min-distance of examples too large for shared memory. */
int b200mp_fps(const void* src, const void* ptr, int64_t n, int64_t f, int64_t n_ptr, const float* rnd,
               const int64_t* offsets, float* dist_ws, int64_t* out, int val_dtype, int ptr_dtype, void* stream);

/* ------------------------------------------------------------------ clustering for pooling (graclus, voxel grid)
 * Greedy graph matching: replaces pyg_lib.ops.graclus_cluster (torch.ops.pyg.graclus_cluster, nn/pool/graclus.py:39).
 * rowptr [n + 1] / col (idx_dtype) is the CSR adjacency, n < 2^31; weight (NULL = unweighted) is one value per CSR
 * entry, fp32 / bf16 / fp64 (weight_dtype = B200MP_F32 / B200MP_BF16 / B200MP_F64), only compared after an exact
 * widening to fp64.  cluster [n] int64 gets min(u, v) for each matched pair and u for each singleton.  The matching is
 * a pure function of (graph, weight, seed): rounds of propose / respond / settle with node colours from
 * splitmix64(seed, round * n + u), in one cooperative launch (B200MP_ERR_UNSUPPORTED on a device without cooperative
 * launches), at most 256 rounds, after which unmatched nodes become singletons (csrc/cluster.cu states the rules).
 * ws [2n + 3] int32 is scratch; ws[2n + 2] receives the number of rounds used.  n = 0 launches nothing. */
int b200mp_graclus(const void* rowptr, const void* col, const void* weight, int64_t n, uint64_t seed, int64_t* cluster,
                   int32_t* ws, int idx_dtype, int weight_dtype, void* stream);
/* Regular-grid clustering: replaces pyg_lib.ops.grid_cluster (torch.ops.pyg.grid_cluster, nn/pool/voxel_grid.py:66).
 * pos [n, d] row-major, size / start / end [d], all val_dtype (B200MP_F32 or B200MP_F64).  out [n] int64 gets
 * sum_k trunc((pos[i, k] - start[k]) / size[k]) * prod_{k' < k} (trunc((end[k'] - start[k']) / size[k']) + 1), one IEEE
 * subtract and one IEEE divide per term in val_dtype, converted toward zero (saturating, NaN -> INT64_MIN) and summed
 * with 64-bit wrap-around.  A NULL start / end is the column min / max of pos (NaN propagating), computed on the device
 * into ws, which then holds 514 d elements of val_dtype.  1 <= d <= 65535. */
int b200mp_grid_cluster(const void* pos, const void* size, const void* start, const void* end, int64_t n, int64_t d,
                        int64_t* out, void* ws, int val_dtype, void* stream);

/* ------------------------------------------------------------------ random walks (uniform and node2vec)
 * Replaces pyg_lib.ops.random_walk (torch.ops.pyg.random_walk: nn/models/node2vec.py:64,103, utils/dropout.py:285,
 * transforms/rooted_subgraph.py:171).  rowptr [n + 1] / col [n_edges] is the CSR adjacency, start [n_walks] the first
 * node of each walk, all idx_dtype; n < 2^31 - 1.  out [n_walks, walk_length + 1] (idx_dtype) gets each walk, column 0
 * being start.  p, q: finite and > 0; p = q = 1 gives uniform walks, anything else node2vec's second-order walk by
 * rejection sampling with at most max_trials trials per step before an exact draw.  The walks are a pure function of
 * (graph, start, walk_length, p, q, max_trials, seed); csrc/random_walk.cu states the generator and every rule.  A start
 * outside [0, n) gives a row of -1; a picked node outside [0, n) (or a row with bounds outside [0, n_edges]) ends its
 * walk, the rest of the row being -1.  rows_unsorted [1] int32 (DEVICE; required when p != 1 or q != 1) is 1 when
 * some row of col decreases, which selects a linear scan over a binary search for the neighbour test; with
 * refresh_rows_unsorted it is computed here first (O(n_edges)), otherwise it is read as the caller left it.
 * n_walks = 0 launches nothing. */
int b200mp_random_walk(const void* rowptr, const void* col, const void* start, int64_t n, int64_t n_edges,
                       int64_t n_walks, int64_t walk_length, double p, double q, int64_t max_trials, uint64_t seed,
                       int32_t* rows_unsorted, int refresh_rows_unsorted, void* out, int idx_dtype, void* stream);

/* ------------------------------------------------------------------ COO scatter fallback (atomics)
 * out[index[e], :] (+)= src[e, :] for an UNSORTED index.  Replaces utils/_scatter.py:14-138
 * (aten::scatter_add_ / scatter_reduce_, torch_scatter.scatter).  fp32 only.  `count` is a
 * caller-provided n_rows fp32 scratch (used by mean/min/max to detect empty rows).  out is fully
 * written (initialised inside).  sum uses red.global.add.v4.f32 where feat % 4 == 0. */
int b200mp_scatter_coo(const float* src, const void* index, float* out, float* count,
                       int64_t n_src, int64_t n_rows, int64_t feat, int reduce, int idx_dtype,
                       void* stream);
/* out[index[e], :] += src[e, :] into an EXISTING fp32 out (no initialisation; atomics): the
 * return leg of the multi-GPU halo exchange (aten::index_add_). */
int b200mp_index_add_rows(const float* src, const void* index, float* out, int64_t n_src,
                          int64_t feat, int idx_dtype, void* stream);
/* Gather rows: out[e,:] = x[index[e],:]  (aten::index_select, message_passing.py:263-290) --
 * only used by the unfused compatibility path and by backward of scatter. scale (nullable, one
 * fp32 per row of out) multiplies each gathered row. */
int b200mp_gather_rows(const void* x, const void* index, const float* scale, void* out,
                       int64_t n_out, int64_t feat, int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ segment softmax
 * out[e,h] = exp(src[e,h] - max_g) / (sum_g exp(src - max_g) + 1e-16) over CSR groups.
 * Replaces utils/_softmax.py:12-92 and pyg_lib.ops.softmax_csr.  fp32.  backward:
 * grad_src = out * (grad_out - sum_g(grad_out * out)). */
int b200mp_softmax_csr(const void* ptr, const float* src, float* out, int64_t n_rows,
                       int64_t n_src, int64_t heads, int idx_dtype, void* stream);
int b200mp_softmax_csr_backward(const void* ptr, const float* out, const float* grad_out,
                                float* grad_src, int64_t n_rows, int64_t n_src, int64_t heads,
                                int idx_dtype, void* stream);
/* Edge-parallel pieces of the hub-safe segment softmax (groups longer than the long-row chunk): with
 * d = dst_of_edge[e], row [n_rows, heads] fp32,
 *   op 0: out = exp(a - row[d])   op 1: out = a / (row[d] + 1e-16)   op 2: out = a * b   op 3: out = a * (b - row[d]).
 * The host composes _softmax.py:82-88 as segment-max, op 0, segment-sum, op 1 (backward: op 2, segment-sum,
 * op 3) with b200mp_segment_csr and its long-row plan, so no group is ever walked by a single lane group. */
int b200mp_softmax_edge_op(int op, const float* a, const float* b, const float* row, const void* dst_of_edge,
                           float* out, int64_t n_src, int64_t heads, int idx_dtype, void* stream);


/* ------------------------------------------------------------------ bias gradient
 * out[f] = sum_i x[i, f] (fp32): the gradient of the layer bias that autograd derives for `out + bias`
 * (nn/conv/gcn_conv.py:263-264), as one deterministic two-launch column sum instead of ATen's generic
 * reduction.  partials: caller-owned fp32 workspace [n_parts, feat], n_parts from b200mp_column_sum_parts. */
int64_t b200mp_column_sum_parts(int64_t n_rows);
int b200mp_column_sum(const void* x, float* out, float* partials, int64_t n_parts, int64_t n_rows, int64_t feat,
                      int val_dtype, void* stream);

/* ------------------------------------------------------------------ multi-aggregation (one sweep, k outputs)
 * Replaces FusedAggregation.forward (nn/aggr/fused.py:191-336: one scatter per base reduction plus the
 * shared count) and the [sum, mean, min, max, var, std] members of MultiAggregation (nn/aggr/multi.py):
 * every requested output of row i is derived from ONE walk over rowptr[i]:rowptr[i+1].
 *   col != NULL: gather mode, row e reads x[col[e], :]  (x: [n_src, feat]);
 *   col == NULL: segment mode, x is the destination-sorted message matrix [n_src = E, feat].
 * out_* are nullable [n_rows, feat] tensors of val_dtype (NULL = not requested); ties_min / ties_max
 * (nullable, fp32 [n_rows, feat]) receive the number of edges attaining the extremum, plus one where the
 * extremum is 0 if count_self_zero (ATen's scatter_reduce backward rule) -- what the backward divides by.
 * mean = sum / max(deg,1); var = sumsq / max(deg,1) - mean^2; std = sqrt(max(var,1e-5)), 0 where that is
 * <= sqrt(1e-5) (fused.py:319-323); empty rows give 0 everywhere.  Hub rows: long-row plan of
 * b200mp_csr_plan_* with partials of n_chunks * 6 * feat fp32.
 * hit_mask (nullable; gather mode, fp32, feat % 4 == 0, with a ties plane): uint8 [n_edges, feat / 4] in CSR edge
 * order, bit i of byte (e, v) = x[col[e], 4v + i] equals the row's min, bit 4 + i = equals the row's max -- the
 * comparison the backward needs, taken while the row's sources are still in L2, so that the backward reads one byte
 * per edge and vector instead of the destination's min and max vectors (ask b200mp_multi_aggr_mask_supported). */
int b200mp_multi_aggr_mask_supported(int64_t feat, int val_dtype, int segment_mode);
int b200mp_multi_aggr_csr(const void* rowptr, const void* col, const void* x, void* out_sum, void* out_mean,
                          void* out_min, void* out_max, void* out_var, void* out_std, float* ties_min,
                          float* ties_max, void* hit_mask, int64_t n_rows, int64_t n_src, int64_t feat, int count_self_zero,
                          const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                          int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype,
                          void* stream);
/* Backward of the above in one kernel.  The caller folds the output gradients into per-destination fp32
 * rows (all nullable, [n_dst, feat]):  term_a (added), term_b (multiplies the message value),
 * g_min = grad_min / ties_min with out_min (val_dtype), g_max / out_max likewise; then
 *   grad(x_e) = sum over the destinations d of the value:  term_a[d] + x * term_b[d]
 *               + [x == out_min[d]] * g_min[d] + [x == out_max[d]] * g_max[d].
 * segment_mode != 0: n_items = E messages, idx = dst_of_edge [E] (ptr unused), x / grad_x: [E, feat];
 * segment_mode == 0: n_items = n_src source rows, (ptr, idx) = transposed CSR (rowptr_t, col_t).
 * hit_mask + t2csr (both nullable, gather mode only): the forward's hit bits and the CSR slot of every transposed
 * slot; when given and supported they replace the reads of out_min / out_max (which must still be passed: shapes the
 * masked kernel does not cover compare against them). */
/* Elementwise prologue of the backward: folds the output gradients (nullable, [n_rows, feat] val_dtype) and
 * the saved mean / std / tie counts into term_a, term_b, g_min / ties_min, g_max / ties_max (fp32).
 * cnt = max(rowptr[i+1] - rowptr[i], 1); semi_grad drops the 2 x / cnt term of var / std (basic.py:106-110). */
int b200mp_multi_aggr_prepare_backward(const void* rowptr, const void* g_sum, const void* g_mean,
                                       const void* g_var, const void* g_std, const void* g_min,
                                       const void* g_max, const void* mean, const void* std,
                                       const float* ties_min, const float* ties_max, float* term_a,
                                       float* term_b, float* gmin_out, float* gmax_out, int64_t n_rows,
                                       int64_t feat, int semi_grad, int idx_dtype, int val_dtype, void* stream);
int b200mp_multi_aggr_backward(const void* ptr, const void* idx, const void* x, const float* term_a,
                               const float* term_b, const void* out_min, const float* g_min,
                               const void* out_max, const float* g_max, const void* hit_mask, const void* t2csr,
                               void* grad_x, int64_t n_items, int64_t feat, int segment_mode, int idx_dtype,
                               int val_dtype, void* stream);

/* ------------------------------------------------------------------ PNA: shifted multi-aggregation + degree scalers
 * PNAConv with one pre-layer per tower (nn/conv/pna_conv.py:167-188) sends m_e = u_i + w_e over edge e = (j -> i), with
 * u = x_t Wa_t^T + b_t, w_e = v_j (+ c_e), v = x_t Wb_t^T, c = edge_encoder(edge_attr) Wc_t^T, all towers side by side
 * in one width W = towers * feat.  The sweep collects the statistics of w only (b200mp_multi_aggr_csr in gather mode on
 * v with count_self_zero = 0, or b200mp_pna_edge_stats with edge features); the shift by u, the aggregators and the
 * scalers are per destination.  Replaces: the message's [E, T, 2F or 3F] concatenation and per-tower Linear
 * (pna_conv.py:167-188), MultiAggregation's per-aggregator passes over 3-D messages (nn/aggr/multi.py:157), and
 * DegreeScalerAggregation's degree scatter, per-scaler products and concatenations (nn/aggr/scaler.py:75-109), plus
 * cat([x, out]) (pna_conv.py:169).
 * Aggregator codes: 0 sum, 1 mean, 2 min, 3 max, 4 var, 5 std (at most 6); scaler codes: 0 identity, 1 amplification,
 * 2 attenuation, 3 linear, 4 inverse_linear (at most 5); both lists are host arrays read at the call.
 * avg_deg_lin / avg_deg_log: device fp32 scalars.  stats_dtype: B200MP_F32 or val_dtype (the statistics' dtype;
 * ties are fp32).  u: [n_rows, W] rows of stride u_ld; x: [n_rows, W] (x_t of every tower).
 * Epilogue: out [n_rows, towers, (1 + A S) feat] = cat([x_t, s_1(a_1 .. a_A), .., s_S(a_1 .. a_A)]) per tower, with
 *   sum = deg u + sum w, mean = sum / max(deg, 1), min / max = u + min / max w (0 for an empty row), var / std from the
 *   statistics of w (shift-invariant; std clamps at 1e-5 and is zeroed at <= sqrt(1e-5)), deg rounded to val_dtype. */
int b200mp_pna_epilogue(const void* rowptr, const void* x, const void* u, int64_t u_ld, const void* stat_sum,
                        const void* stat_min, const void* stat_max, const void* stat_var, const int32_t* aggr_host,
                        int n_aggr, const int32_t* scaler_host, int n_scaler, const float* avg_deg_lin,
                        const float* avg_deg_log, void* out, int64_t n_rows, int64_t towers, int64_t feat,
                        int stats_dtype, int idx_dtype, int val_dtype, void* stream);
/* Prologue of the backward: folds grad_out (the epilogue's block) into the rows b200mp_multi_aggr_backward or
 * b200mp_pna_edge_backward read (all nullable, fp32 [n_rows, W]): term_a, term_b, gmin = g_min / ties, gmax = g_max /
 * ties, where ties count the zero-initialised self of the reference's scatter when the SHIFTED extremum is 0; and in
 * closed form grad_u (rows of stride gu_ld) = deg g_sum + [deg > 0] g_mean + g_min ties_w_min / ties + g_max ...,
 * grad_x = the x slot's gradient, avg_part [n_rows, 2] = per-row d L / d avg_deg_lin and d L / d avg_deg_log (the caller
 * sums the rows in a fixed order). */
int b200mp_pna_prologue(const void* rowptr, const void* grad_out, const void* u, int64_t u_ld, const void* stat_sum,
                        const void* stat_min, const void* stat_max, const void* stat_var, const float* ties_min,
                        const float* ties_max, const int32_t* aggr_host, int n_aggr, const int32_t* scaler_host,
                        int n_scaler, const float* avg_deg_lin, const float* avg_deg_log, float* term_a, float* term_b,
                        float* gmin, float* gmax, void* grad_u, int64_t gu_ld, void* grad_x, float* avg_part,
                        int64_t n_rows, int64_t towers, int64_t feat, int stats_dtype, int idx_dtype, int val_dtype,
                        void* stream);
/* Statistics of w_e = v[col[e]] + c[perm[e]] (rounded to val_dtype) over the destination CSR, fp32 [n_rows, width]
 * planes (each nullable): sum, min, max, var (= sum w^2 / cnt - mean^2), and the tie counts of min / max (no self).
 * v: [n_cols, width] rows of stride v_ld; c: [n_edges, width] in the caller's edge order, perm: CSR slot -> caller's
 * edge (nullable = identity).  Hub rows: long-row plan with partials of n_chunks * 6 * width fp32. */
int b200mp_pna_edge_stats(const void* rowptr, const void* col, const void* perm, const void* v, int64_t v_ld,
                          const void* c, float* stat_sum, float* stat_min, float* stat_max, float* stat_var,
                          float* ties_min, float* ties_max, int64_t n_rows, int64_t n_cols, int64_t n_edges,
                          int64_t width, const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                          int64_t n_chunks, int64_t chunk, float* partials, int idx_dtype, int val_dtype, void* stream);
/* Backward of b200mp_pna_edge_stats + the prologue, in ONE sweep over the transposed CSR (rowptr_t, col_t, perm_t =
 * transposed slot -> caller's edge): d L / d w_e = term_a[i] + w_e term_b[i] + [w_e == min w_i] gmin[i] + [w_e == max
 * w_i] gmax[i] is written to grad_c[e] and summed into grad_v[j] (rows of stride gv_ld); either output may be null. */
int b200mp_pna_edge_backward(const void* rowptr_t, const void* col_t, const void* perm_t, const void* v, int64_t v_ld,
                             const void* c, const float* term_a, const float* term_b, const float* stat_min,
                             const float* gmin, const float* stat_max, const float* gmax, void* grad_v, int64_t gv_ld,
                             void* grad_c, int64_t n_src, int64_t n_dst, int64_t n_edges, int64_t width, int idx_dtype,
                             int val_dtype, void* stream);

/* ------------------------------------------------------------------ node-level attention terms
 * s_a[n,h] = sum_c x[n,h,c] * att_a[h,c] (and s_b with att_b from the same read of x; att_b / s_b nullable together):
 * GATConv's alpha_src / alpha_dst = (x * att).sum(-1) (nn/conv/gat_conv.py:330-331) without the [N,H,C] product tensor.
 * x: [n_rows, heads*chan] of val_dtype (fp32 / bf16), att_*: fp32 [heads*chan], s_*: fp32 [n_rows, heads].
 * Supported when chan * sizeof(val) is a multiple of 16 and a power-of-two number (<= 32) of 16-byte vectors, and a row has
 * at most 256 vectors (b200mp_head_dot_supported); other shapes are the caller's business.
 * Backward in one pass: grad_x = g_a (x) att_a + g_b (x) att_b (+ add, nullable: e.g. the attention's own grad_v), and
 * per-CTA partial rows part_* [n_parts, heads*chan] fp32 of grad_att_* = sum_n g_*[n,h] * x[n,h,c] (fold them with
 * b200mp_column_sum; n_parts from b200mp_head_dot_parts).  grad_x nullable (x does not need a gradient). */
int b200mp_head_dot_supported(int64_t heads, int64_t chan, int val_dtype);
int64_t b200mp_head_dot_parts(int64_t n_rows, int64_t heads, int64_t chan, int val_dtype);
int b200mp_head_dot(const void* x, const float* att_a, const float* att_b, float* s_a, float* s_b, int64_t n_rows,
                    int64_t heads, int64_t chan, int val_dtype, void* stream);
int b200mp_head_dot_backward(const void* x, const float* att_a, const float* att_b, const float* g_a, const float* g_b,
                             const void* add, void* grad_x, float* part_a, float* part_b, int64_t n_parts,
                             int64_t n_rows, int64_t heads, int64_t chan, int val_dtype, void* stream);

/* ------------------------------------------------------------------ fused GAT attention + aggregation
 * One sweep over the destination-sorted CSR per (node, head):
 *   logit_e = leaky_relu(a_src[col[e],h] + a_dst[i,h], slope)
 *   alpha_e = softmax over the row;  out[i,h,:] = sum_e alpha_e * xh[col[e],h,:]
 * Replaces GATConv.edge_update + message + aggregate (nn/conv/gat_conv.py:387-409,
 * utils/_softmax.py:82-88) -- 12 kernels and three [E,H,C] tensors in the reference.
 * xh: [n_src, heads*chan] val_dtype; a_src [n_src, heads], a_dst [n_rows, heads] fp32;
 * out: [n_rows, heads*chan] val_dtype; row_max/row_den [n_rows, heads] fp32 (saved for backward);
 * alpha_out (nullable) [n_edges, heads] fp32 in CSR order. */
int b200mp_gat_fused_csr(const void* rowptr, const void* col, const void* dst_of_edge, const void* xh,
                         const float* a_src, const float* a_dst, void* out, float* row_max,
                         float* row_den, float* alpha_out, int64_t n_rows, int64_t n_edges,
                         int64_t heads, int64_t chan, float slope, const int64_t* long_rows,
                         const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                         float* part_acc, float* part_ms, int idx_dtype, int val_dtype, void* stream);
/* (dst_of_edge = ptr2index(rowptr), only needed with alpha_out.  Hub rows: pass the long-row plan of
 * b200mp_csr_plan_* plus part_acc [n_chunks, heads*chan] and part_ms [n_chunks, heads, 2] fp32; every
 * chunk keeps an online-softmax state that is merged with exp(m_c - M) rescaling.)
 *
 * Backward of b200mp_gat_fused_csr, attention recomputed from row_max/row_den:
 *  row dots    rowdot[i,h] = <g[i,h,:], out[i,h,:]>               (scratch [n_rows, heads])
 *  edge sweep  grad_pre[e,h] (CSR order, scratch [n_edges, heads]) -- one thread per (edge, head), so
 *              no row is walked serially -- and grad_a_dst[i,h] = its (chunked) segmented sum
 *              (partials: n_chunks * heads fp32 when the plan is given)
 *  source sweep (rowptr_t/col_t, t2csr[e] = CSR slot of transposed slot e): grad_xh[j,h,:] (the
 *              message term only; the a_src/a_dst terms flow back through the caller's
 *              (xh*att).sum(-1)) and grad_a_src[j,h]. */
int b200mp_gat_fused_csr_backward(const void* rowptr, const void* col, const void* dst_of_edge,
                                  const void* rowptr_t, const void* col_t, const void* t2csr,
                                  const void* xh, const float* a_src, const float* a_dst,
                                  const float* row_max, const float* row_den, const void* out,
                                  const void* grad_out, float* grad_pre, float* rowdot, void* grad_xh,
                                  float* grad_a_src, float* grad_a_dst, int64_t n_rows, int64_t n_src,
                                  int64_t n_edges, int64_t heads, int64_t chan, float slope,
                                  const int64_t* long_rows, const int64_t* chunk_ptr,
                                  int64_t n_long_rows, int64_t n_chunks, int64_t chunk, float* partials,
                                  int idx_dtype, int val_dtype, void* stream);

/* ------------------------------------------------------------------ argmin / argmax outputs (csrc/arg.cu)
 * The (out, arg) operator signatures the reference binds to: torch_scatter.scatter_max / scatter_min
 * (utils/_scatter.py:147-156) and torch.ops.torch_sparse.spmm_min / spmm_max (edge_index.py:1798-1810).
 * `out` is what b200mp_scatter_coo / b200mp_spmm_csr produced (fp32, min or max); these passes find its producer:
 *   b200mp_scatter_arg   arg[i,f] = smallest e with index[e] == i and src[e,f] == out[i,f]; n_src for empty groups
 *   b200mp_spmm_csr_arg  arg[i,f] = first CSR slot e of row i with val[e]*x[col[e],f] == out[i,f]; nnz for empty rows
 * arg: int64 [n_rows, feat]. */
int b200mp_scatter_arg(const float* src, const void* index, const float* out, int64_t* arg, int64_t n_src,
                       int64_t n_rows, int64_t feat, int idx_dtype, void* stream);
int b200mp_spmm_csr_arg(const void* rowptr, const void* col, const float* val, const float* x, const float* out,
                        int64_t* arg, int64_t n_rows, int64_t feat, int64_t nnz, int idx_dtype, void* stream);

/* ------------------------------------------------------------------ fused attention family (csrc/attention.cu)
 * One kernel skeleton for the three score functions of the reference's attention convolutions, forward and
 * backward, over the destination-sorted CSR (alpha = softmax over the in-edges of i, utils/_softmax.py:82-88;
 * out[i,h,:] = sum_e alpha_e,h v[col[e],h,:]):
 *   mode 0 GAT    s = leaky_relu(s_src[j,h] + s_dst[i,h] (+ s_edge[e,h]))       nn/conv/gat_conv.py:387-409
 *   mode 1 GATv2  s = sum_c att[h,c] leaky_relu(v[j,h,c] + q[i,h,c])           nn/conv/gatv2_conv.py:358-378
 *   mode 2 DOT    s = scale <q[i,h,:], k[j,h,:]>                               nn/conv/transformer_conv.py:263-275
 * v (GAT xh / GATv2 x_l / value rows), k (DOT keys): [n_src, heads*chan] val_dtype with row strides v_stride /
 * k_stride in ELEMENTS (0 = heads*chan; k and v may be the halves of one [N, 2*H*C] product); q (GATv2 x_r / DOT
 * queries): [n_rows, heads*chan], stride q_stride; s_src [n_src, heads], s_dst [n_rows, heads], att [heads*chan],
 * s_edge [n_edges, heads] (CSR order, nullable) fp32.  out [n_rows, heads*chan]; row_max / row_den [n_rows, heads]
 * fp32 are saved for the backward; alpha_out (nullable) [n_edges, heads] fp32 in CSR order.
 * dropout_p in [0, 1): attention dropout (gat_conv.py:404, gatv2_conv.py:376, transformer_conv.py:268 -- F.dropout on the
 * normalised coefficients): (edge, head) pairs are dropped by a counter-based hash of (dropout_seed, CSR slot, head) that the
 * forward and the backward evaluate identically (pass the same p and seed to both); kept coefficients are scaled by
 * 1 / (1 - p); alpha_out returns the dropped coefficients like the reference.  0 = no dropout.
 * edge_feat (nullable; GATv2 and dot modes): per-edge feature rows [n_edges, heads*chan] of val_dtype in CSR order, i.e.
 * lin_edge(edge_attr) of `edge_dim` layers: GATv2 adds them inside the leaky_relu (gatv2_conv.py:358-360), the dot mode to
 * the key and to the value (transformer_conv.py:258-272).  The backward writes grad_edge_feat (same shape; required when
 * edge_feat is given).  (GAT's edge_dim term is the scalar s_edge.)
 * Shapes: b200mp_attn_supported(heads, chan, val_dtype) != 0 (rows of whole 16-byte vectors, <= 1 KB, a head =
 * a power-of-two number of vectors), else B200MP_ERR_UNSUPPORTED.  Hub rows: the long-row plan of
 * b200mp_csr_plan_* plus part_acc [n_chunks, heads*chan] and part_ms [n_chunks, heads, 2] fp32.
 *
 * Backward: destination sweep (softmax backward per edge, grad_q / grad_s_dst / grad_att, and the per-edge scratch
 * pair [n_edges, heads, 2] fp32 = (alpha, grad_score) in CSR order -- for GAT pair[...,1] is also the gradient of
 * s_edge) then source sweep on the transposed CSR (t2csr[e] = CSR slot of transposed slot e): grad_v, grad_k (DOT),
 * grad_s_src (GAT).  Long-row partials: partials [n_chunks, b200mp_attn_backward_partial_width(mode,H,C,0)] and
 * partials_t [n_chunks_t, ...(mode,H,C,1)] fp32; gatt_part (GATv2) [b200mp_attn_gatt_rows(), heads*chan] fp32. */
int b200mp_attn_supported(int64_t heads, int64_t chan, int val_dtype);
int b200mp_attn_csr_forward(int mode, const void* rowptr, const void* col, const void* v, const void* k,
                            const void* q, const float* s_src, const float* s_dst, const float* att,
                            const float* s_edge, int64_t v_stride, int64_t k_stride, int64_t q_stride,
                            void* out, float* row_max, float* row_den, float* alpha_out, int64_t n_rows,
                            int64_t n_edges, int64_t heads, int64_t chan, float slope, float scale,
                            const int64_t* long_rows, const int64_t* chunk_ptr, int64_t n_long_rows,
                            int64_t n_chunks, int64_t chunk, float* part_acc, float* part_ms, float dropout_p,
                            unsigned long long dropout_seed, const void* edge_feat, int idx_dtype, int val_dtype,
                            void* stream);
int64_t b200mp_attn_backward_partial_width(int mode, int64_t heads, int64_t chan, int transposed);
int64_t b200mp_attn_gatt_rows(void);
int b200mp_attn_csr_backward(int mode, const void* rowptr, const void* col, const void* rowptr_t,
                             const void* col_t, const void* t2csr, const void* v, const void* k, const void* q,
                             const float* s_src, const float* s_dst, const float* att, const float* s_edge,
                             int64_t v_stride, int64_t k_stride, int64_t q_stride, const float* row_max,
                             const float* row_den, const void* out, const void* grad_out, float* pair,
                             void* grad_v, void* grad_k, void* grad_q, float* grad_s_src, float* grad_s_dst,
                             float* grad_att, float* gatt_part, int64_t n_rows, int64_t n_src, int64_t n_edges,
                             int64_t heads, int64_t chan, float slope, float scale, const int64_t* long_rows,
                             const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks, int64_t chunk,
                             float* partials, const int64_t* long_rows_t, const int64_t* chunk_ptr_t,
                             int64_t n_long_rows_t, int64_t n_chunks_t, float* partials_t, float dropout_p,
                             unsigned long long dropout_seed, const void* edge_feat, void* grad_edge_feat, int idx_dtype,
                             int val_dtype, void* stream);

/* ------------------------------------------------------------------ dense transform on tensor cores
 * fp32-accurate 3xTF32 GEMMs (wgmma + TMA, csrc/gemm_tf32x3.cu) for the layer's
 * Linear (nn/dense/linear.py:121-127: F.linear, run by the reference as strict-fp32 cuBLAS):
 *   b200mp_linear_tf32x3            y [M,N]  = x [M,K] . w[N,K]^T
 *   b200mp_linear_grad_input_tf32x3 gx[M,K]  = g [M,N] . w[N,K]
 *   b200mp_linear_grad_weight_tf32x3 gw[N,K] = g [M,N]^T . x[M,K]   (deterministic split-K)
 * w_hi/w_lo come from b200mp_split_tf32 (w = w_hi + w_lo, w_hi = rn_tf32(w)); w_lo == NULL means w_hi is
 * the UNSPLIT weight and the kernel splits each B tile in shared memory (one L2 read of W per tile instead
 * of two).  All matrices
 * row-major, contiguous, 16-byte aligned.  Shape limits (else B200MP_ERR_UNSUPPORTED and the caller
 * uses a library GEMM): reduction dim % 32 == 0, output width in {64, 128} or a multiple of 256,
 * and for grad_weight N % 128 == 0. */
int b200mp_split_tf32(const float* w, float* w_hi, float* w_lo, int64_t n, void* stream);
/* w [rows, cols] -> wt_hi = rn_tf32(w^T), wt_lo = w^T - wt_hi, both [cols, rows]: the input gradient g . w then runs
 * as the K-major pair form (b_layout 0) on (wt_hi, wt_lo), whose B tiles the kernel reads straight from its TMA stages. */
int b200mp_split_tf32_transposed(const float* w, float* wt_hi, float* wt_lo, int64_t rows, int64_t cols, void* stream);
int b200mp_linear_tf32x3(const float* x, const float* w_hi, const float* w_lo, float* y, int64_t m,
                         int64_t n, int64_t k, void* stream);
int b200mp_linear_grad_input_tf32x3(const float* g, const float* w_hi, const float* w_lo, float* gx,
                                    int64_t m, int64_t n, int64_t k, void* stream);
int64_t b200mp_linear_grad_weight_workspace_bytes(int64_t m, int64_t n, int64_t k);
int b200mp_linear_grad_weight_tf32x3(const float* g, const float* x, float* gw, int64_t m, int64_t n,
                                     int64_t k, void* workspace, int64_t workspace_bytes,
                                     void* stream);

/* Pair form: two A streams accumulate into ONE accumulator,
 * the epilogue adds a bias and applies ReLU, and the output columns may be split over two matrices:
 *     [c1 | c2] [M, n1+n2] = act( [a1 | a2] [M, k1+k2] . B + bias )
 * b_layout 0: B = w [n1+n2, k1+k2] row-major (y = A w^T: SAGEConv's lin_l(agg) + lin_r(x) with w = [W_l | W_r],
 * sage_conv.py:134-141, in one launch instead of two GEMMs and an add); b_layout 1: B = w [k1+k2, n1+n2] row-major
 * (y = A w: both input gradients of such a pair from one read of g, RGCNConv's [H | x] . [W_1;..;W_R; root],
 * rgcn_conv.py:257-280).  a2 / c2 / bias nullable (k2 = 0 / n2 = 0).  k1, k2 % 32 == 0; n1, n2 % 128 == 0;
 * b_lo == NULL: b_hi is the unsplit matrix (the kernel splits B tiles itself). */
int b200mp_gemm_pair_tf32x3(const float* a1, int64_t k1, const float* a2, int64_t k2, const float* b_hi,
                            const float* b_lo, int b_layout, const float* bias, int relu, float* c1, int64_t n1,
                            float* c2, int64_t n2, int64_t m, void* stream);

/* Grouped form: pyg_lib.ops.segment_matmul(inputs, ptr, other) (nn/dense/linear.py:248-255, nn/conv/rgcn_conv.py:288;
 * HeteroLinear, HeteroDictLinear, RGCNConv's sorted-by-type path).
 *     c[ptr[r] : ptr[r+1], :] = a[ptr[r] : ptr[r+1], :] . B_r        for r in [0, n_seg)
 * in ONE persistent launch over (segment, 128-row tile, 128-column tile) work items; ptr [n_seg+1] int64 stays on the
 * device (the tile -> segment map is rebuilt in shared memory), partial tiles at segment ends are stored row-masked.
 * b_layout 1: B_r = w[r] of a [n_seg, K, N] weight (c = a w[r]); b_layout 0: B_r = w[r] of a [n_seg, N, K] weight
 * (c = a w[r]^T: the input gradient of layout 1).  b_hi / b_lo from b200mp_split_tf32 over the whole stack.
 * k % 32 == 0, n % 128 == 0, n_seg <= 120. */
int b200mp_segment_matmul_tf32x3(const float* a, const int64_t* ptr, int64_t n_seg, const float* b_hi,
                                 const float* b_lo, int b_layout, float* c, int64_t m, int64_t k, int64_t n,
                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200MP_H_ */
