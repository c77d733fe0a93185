// csr_dispatch.cuh -- picks the kernel variant for one gather/segment reduce call.
//   wide rows  (512 B <= row_bytes <= 2 KB, 16 B aligned): persistent TMA-fed streaming kernel
//   otherwise : lane-group-per-row kernel (csr_reduce.cuh), scalar fallback for odd widths
// b200mp_set_option("spmm_impl", 1) forces the lane-group kernel (A/B measurements).
#pragma once

#include "csr_reduce.cuh"
#include "csr_tma.cuh"

namespace b200mp {

int get_option_spmm_impl();  // 0 = auto, 1 = lane-group kernel, 2 = TMA kernel where legal

template <typename T, typename I, int RED, bool GATHER>
int csr_reduce_variant(const I* rowptr, const I* col, const float* val, const T* x, T* out, int64_t n_rows,
                       int64_t feat, bool is_mean, bool inf_to_zero, LongRowPlan plan, const float* bias,
                       cudaStream_t stream) {
    if (n_rows == 0 || feat == 0) return B200MP_OK;
    const size_t row_bytes = static_cast<size_t>(feat) * sizeof(T);
    const bool tma_ok = row_bytes % 16 == 0 && row_bytes >= 512 && row_bytes <= 2048 && aligned16(x) &&
                        aligned16(plan.x2) && aligned16(out) && (plan.n_chunks == 0 || aligned16(plan.partials));
    // "auto" is the lane-group kernel: at 48 warps/SM it keeps more rows in flight than the TMA-fed
    // kernel, which is issue-bound at 6 warps/SM.  The TMA variant stays selectable for A/B timing.
    const int impl = get_option_spmm_impl();
    if (tma_ok && impl == 2 && !plan.accumulate && !plan.peers)
        return csr_tma_launch<T, I, RED, GATHER>(rowptr, col, val, x, out, n_rows, feat, is_mean, inf_to_zero, plan,
                                                 bias, stream);
    return csr_reduce_dispatch<T, I, RED, GATHER>(rowptr, col, val, x, out, n_rows, feat, is_mean, inf_to_zero, plan,
                                                  bias, stream);
}

template <typename T, typename I, bool GATHER>
int csr_reduce_auto(const I* rowptr, const I* col, const float* val, const T* x, T* out, int64_t n_rows,
                    int64_t feat, int reduce, bool inf_to_zero, LongRowPlan plan, const float* bias,
                    cudaStream_t stream) {
    switch (reduce) {
        case B200MP_SUM:
            return csr_reduce_variant<T, I, B200MP_SUM, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, false, plan, bias, stream);
        case B200MP_MEAN:
            return csr_reduce_variant<T, I, B200MP_SUM, GATHER>(rowptr, col, val, x, out, n_rows, feat, true, false, plan, bias, stream);
        case B200MP_MIN:
            return csr_reduce_variant<T, I, B200MP_MIN, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, inf_to_zero, plan, bias, stream);
        case B200MP_MAX:
            return csr_reduce_variant<T, I, B200MP_MAX, GATHER>(rowptr, col, val, x, out, n_rows, feat, false, inf_to_zero, plan, bias, stream);
        default:
            set_error("csr_reduce: unsupported reduce %d", reduce);
            return B200MP_ERR_UNSUPPORTED;
    }
}

}  // namespace b200mp
