// Edge dropout (include/pgcn_dropout.h): a grid-stride map over the entries of a [nnz, K] array. Per entry it reads the
// 8-byte (global row, global column) pair and the K values, makes one Philox4x32-10 call per 4 heads and writes the K
// values: 8 + 8K bytes of HBM traffic per entry.
#include "../../include/pgcn_dropout.h"
#include "philox.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <string>

namespace pgcn {

struct DropoutArgs {
    const int32_t* pairs;
    int64_t nnz;
    uint32_t threshold;
    float scale;
    const int64_t* state;
    const float* x;            // may equal y: plain loads, no __ldg / __restrict__ on the values
    float* y;
};

constexpr int kDropoutThreads = 256;

// K consecutive floats of entry e: VEC reads and writes them as float2 / float4 vectors (the host checked that every
// operand is 16-byte aligned), else one by one. Same values either way.
template <int K, bool VEC>
__device__ __forceinline__ void load_values(const float* p, float (&v)[K])
{
    if constexpr (VEC && K >= 4) {
#pragma unroll
        for (int q = 0; q < K / 4; ++q) {
            const float4 u = reinterpret_cast<const float4*>(p)[q];
            v[4 * q] = u.x; v[4 * q + 1] = u.y; v[4 * q + 2] = u.z; v[4 * q + 3] = u.w;
        }
    } else if constexpr (VEC && K == 2) {
        const float2 u = *reinterpret_cast<const float2*>(p);
        v[0] = u.x; v[1] = u.y;
    } else {
#pragma unroll
        for (int j = 0; j < K; ++j) v[j] = p[j];
    }
}

template <int K, bool VEC>
__device__ __forceinline__ void store_values(float* p, const float (&v)[K])
{
    if constexpr (VEC && K >= 4) {
#pragma unroll
        for (int q = 0; q < K / 4; ++q)
            reinterpret_cast<float4*>(p)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else if constexpr (VEC && K == 2) {
        *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
    } else {
#pragma unroll
        for (int j = 0; j < K; ++j) p[j] = v[j];
    }
}

template <int K, bool VEC>
__global__ void __launch_bounds__(kDropoutThreads) edge_dropout_kernel(DropoutArgs a)
{
    const uint64_t key = (uint64_t)__ldg(a.state);
    const uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
    const uint32_t c = (uint32_t)__ldg(a.state + 1);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < a.nnz; e += stride) {
        uint32_t gi, gj;
        if constexpr (VEC) {
            const int2 pr = __ldg(reinterpret_cast<const int2*>(a.pairs) + e);
            gi = (uint32_t)pr.x; gj = (uint32_t)pr.y;
        } else {
            gi = (uint32_t)__ldg(a.pairs + 2 * e);
            gj = (uint32_t)__ldg(a.pairs + 2 * e + 1);
        }
        float v[K];
        load_values<K, VEC>(a.x + e * K, v);
#pragma unroll
        for (int q = 0; q < (K + 3) / 4; ++q) {
            uint32_t w[4];
            philox4x32_10(gi, gj, c, (uint32_t)q, k0, k1, w);
#pragma unroll
            for (int j = 0; j < 4 && 4 * q + j < K; ++j)
                v[4 * q + j] *= w[j] >= a.threshold ? a.scale : 0.0f;     // x * 0 keeps NaN a NaN
        }
        store_values<K, VEC>(a.y + e * K, v);
    }
}

}  // namespace pgcn

using namespace pgcn;

namespace {

std::string g_error = "";

int fail(int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_error = buf;
    return code;
}

template <int K>
void launch(const DropoutArgs& a, bool vec, int blocks, cudaStream_t s)
{
    if (vec) edge_dropout_kernel<K, true><<<blocks, kDropoutThreads, 0, s>>>(a);
    else edge_dropout_kernel<K, false><<<blocks, kDropoutThreads, 0, s>>>(a);
}

}  // namespace

extern "C" {

const char* pgcn_dropout_version(void) { return "pgcn_dropout 0.1 (sm_90a, Philox4x32-10 edge dropout)"; }

const char* pgcn_dropout_last_error(void) { return g_error.c_str(); }

int pgcn_edge_dropout(const int32_t* pairs, int64_t nnz, int32_t heads, uint32_t threshold, float scale,
                      const int64_t* state, const float* x, float* y, void* stream)
{
    if (nnz < 0) return fail(PGCN_DROPOUT_ERR_INVALID, "nnz=%lld is negative", (long long)nnz);
    if (heads != 1 && heads != 2 && heads != 4 && heads != 8)
        return fail(PGCN_DROPOUT_ERR_INVALID, "heads=%d: the dropout kernels take 1, 2, 4 or 8 heads", heads);
    if (!std::isfinite(scale)) return fail(PGCN_DROPOUT_ERR_INVALID, "scale is not finite");
    if (nnz > 0 && (!pairs || !state || !x || !y)) return fail(PGCN_DROPOUT_ERR_INVALID, "null pointer");
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(PGCN_DROPOUT_ERR_NOGPU, "no CUDA device (%s): edge dropout has no CPU path", cudaGetErrorString(e));
    }
    if (nnz == 0) return PGCN_DROPOUT_OK;
    int sms = 0;
    e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return fail(PGCN_DROPOUT_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
    // a full SM of 256-thread blocks (2048 threads) on every SM; the grid-stride loop takes the rest
    const int64_t want = (nnz + kDropoutThreads - 1) / kDropoutThreads;
    const int blocks = (int)std::min<int64_t>(want, (int64_t)sms * (2048 / kDropoutThreads));
    const bool vec = (((uintptr_t)pairs | (uintptr_t)x | (uintptr_t)y) & 15) == 0;
    const DropoutArgs a{pairs, nnz, threshold, scale, state, x, y};
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (heads) {
    case 1: launch<1>(a, vec, blocks, s); break;
    case 2: launch<2>(a, vec, blocks, s); break;
    case 4: launch<4>(a, vec, blocks, s); break;
    default: launch<8>(a, vec, blocks, s); break;
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PGCN_DROPOUT_ERR_CUDA, "edge_dropout_kernel launch: %s", cudaGetErrorString(e));
    return PGCN_DROPOUT_OK;
}

}  // extern "C"
