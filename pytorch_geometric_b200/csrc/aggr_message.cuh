// aggr_message.cuh -- the per-edge message of the softmax- and power-mean-aggregation sweeps (softmax_aggr.cu,
// power_mean.cu): x gathered through col, an edge row in the caller's edge order, or GENConv's relu(x_j + e_ji) + eps
// (nn/conv/gen_conv.py:231-239).
#pragma once

#include "common.cuh"

namespace b200mp {

enum SmForm { kSmX = 0, kSmA = 1, kSmXRelu = 2, kSmXARelu = 3 };   // which rows are read, and the message

template <int FORM>
struct SmForms {
    static constexpr bool kX = FORM != kSmA;
    static constexpr bool kA = FORM == kSmA || FORM == kSmXARelu;
    static constexpr bool kRelu = FORM == kSmXRelu || FORM == kSmXARelu;
};

// The message m and its pre-activation gate `on` from the fp32 loads.
template <typename T, int FORM>
__device__ __forceinline__ float sm_message(float xv, float av, float eps, bool& on) {
    using Fm = SmForms<FORM>;
    const float s = (Fm::kX && Fm::kA) ? round_to<T>(__fadd_rn(xv, av)) : (Fm::kX ? xv : av);
    on = !(s <= 0.0f);
    return Fm::kRelu ? round_to<T>(__fadd_rn(on ? s : 0.0f, eps)) : s;
}

// Message form from the operands: x and / or a, identity or relu + eps.
inline int sm_form(const void* x, const void* a, int message) {
    if (message == 1) return a ? kSmXARelu : kSmXRelu;
    return x ? kSmX : kSmA;
}

}  // namespace b200mp
