// The gate and the 4-feature lane loads shared by the gated aggregation (gated.cu) and GatedGCN (gatedgcn.cu): one
// definition of the sigmoid, so that both libraries compute the same gate bits for the same pre-activation.
#pragma once

#include <cuda_runtime.h>

namespace pgcn {

// eta = sigmoid(x) and ds = eta (1 - eta), the latter as eta * sigmoid(-x) = eta * (e * eta), e = expf(-x); where e
// overflows, sigmoid(-x) is 1. Explicitly rounded operations: no contraction can differ between instances.
__device__ __forceinline__ float gate(float x, float& ds)
{
    const float e = expf(-x);
    const float eta = __frcp_rn(__fadd_rn(1.0f, e));
    const float em = isinf(e) ? 1.0f : __fmul_rn(e, eta);
    ds = __fmul_rn(eta, em);
    return eta;
}

// The 4 features of this lane in the pass starting at t0: 4 consecutive ones (VEC, one float4) or 4 a warp apart.
// Both lay every feature in the same accumulator slot sequence, so both sum in the same order.
template <bool VEC>
__device__ __forceinline__ void load4(const float* row, int t0, int lane, int f, float (&v)[4])
{
    if constexpr (VEC) {
        const int c = t0 + 4 * lane;
        if (c < f) {
            const float4 u = __ldg(reinterpret_cast<const float4*>(row + c));
            v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w;
        } else {
            v[0] = v[1] = v[2] = v[3] = 0.0f;
        }
    } else {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int c = t0 + lane + 32 * u;
            v[u] = c < f ? __ldg(row + c) : 0.0f;
        }
    }
}

template <bool VEC>
__device__ __forceinline__ void store4(float* row, int t0, int lane, int f, const float (&v)[4])
{
    if constexpr (VEC) {
        const int c = t0 + 4 * lane;
        if (c < f) *reinterpret_cast<float4*>(row + c) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int c = t0 + lane + 32 * u;
            if (c < f) row[c] = v[u];
        }
    }
}

}  // namespace pgcn
