// segment.cu -- C ABI for the segmented reduce without gather (b200mp_segment_csr).
#include "csr_dispatch.cuh"

using namespace b200mp;

extern "C" int b200mp_segment_csr(const void* ptr, const void* src, void* out, int64_t n_rows,
                                  int64_t n_src, int64_t feat, int reduce, const int64_t* long_rows,
                                  const int64_t* chunk_ptr, int64_t n_long_rows, int64_t n_chunks,
                                  int64_t chunk, float* partials, int idx_dtype, int val_dtype, void* stream) {
    B200MP_CHECK_ARG(n_rows >= 0 && n_src >= 0 && feat >= 0);
    LongRowPlan plan;
    if (int rc = make_plan(plan, long_rows, chunk_ptr, n_long_rows, n_chunks, chunk, partials, true)) return rc;
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    B200MP_CHECK_ARG(ptr && out);
    B200MP_CHECK_ARG(src || n_src == 0);
    return dispatch_val_idx(val_dtype, idx_dtype, "segment_csr", [&](auto tv, auto ti) {
        using T = decltype(tv);
        using I = decltype(ti);
        return csr_reduce_auto<T, I, false>(static_cast<const I*>(ptr), static_cast<const I*>(nullptr), nullptr,
                                             static_cast<const T*>(src), static_cast<T*>(out), n_rows, feat, reduce,
                                             true, plan, nullptr, static_cast<cudaStream_t>(stream));
    });
}
