// gate_math.cuh -- elementwise helpers shared by the gated message sweeps (gated.cu, cg.cu).
#pragma once

#include "common.cuh"

namespace b200mp {

// sigma(s) and sigma'(s) from t = exp(-|s|) by __expf (ex2.approx) and r = 1 / (1 + t) by __fdividef (rcp.approx): two
// MUFU operations.  sigma = s >= 0 ? r : t * r and sigma' = t * r * r -- never sigma * (1 - sigma), which cancels at
// large |s|.  s = +inf gives 1, 0; s = -inf gives 0, 0; NaN stays NaN (s >= 0 is false, t = NaN).
__device__ __forceinline__ void sigmoid_pair(float s, float& sig, float& dsig) {
    const float t = __expf(-fabsf(s));
    const float r = __fdividef(1.0f, 1.0f + t);
    const float tr = __fmul_rn(t, r);
    sig = s >= 0.0f ? r : tr;
    dsig = __fmul_rn(tr, r);
}

}  // namespace b200mp
