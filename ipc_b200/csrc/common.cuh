// common.cuh -- shared helpers for the ipc_b200 CUDA hot path (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>


#define HD __host__ __device__ __forceinline__
#define DEV __device__ __forceinline__

namespace ipcgpu {

// H100 SXM (the PCIe part has 114).  Only grid sizes and the persistent warp pass's spill buffers derive from it: no kernel needs all of
// its CTAs resident at once (no grid-wide sync or spin-wait), so results are the same on any SM count.
constexpr int kSMs = 132;

// 3x3 row-major register matrix
struct M3 {
    double m[9];
    DEV double& operator()(int i, int j) { return m[3 * i + j]; }
    DEV double operator()(int i, int j) const { return m[3 * i + j]; }
};

DEV double det3(const M3& A)
{
    return A(0, 0) * (A(1, 1) * A(2, 2) - A(1, 2) * A(2, 1))
        - A(0, 1) * (A(1, 0) * A(2, 2) - A(1, 2) * A(2, 0))
        + A(0, 2) * (A(1, 0) * A(2, 1) - A(1, 1) * A(2, 0));
}

// order-preserving map of a non-negative double onto uint64 (for atomicMin on step sizes)
DEV unsigned long long dbl_to_ord(double x) { return (unsigned long long)__double_as_longlong(x); }
DEV double ord_to_dbl(unsigned long long u) { return __longlong_as_double((long long)u); }

template <typename T>
DEV T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
DEV double warp_min(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// The fixed-order sum over a 256-thread CTA of N per-thread values v[0..N): warp shuffles, then the 8 warp sums in warp order starting
// from +0.0; thread c writes the sum of v[c] to out[c].  Every thread of the CTA calls it.  The per-CTA partials of every deterministic
// two-level sum come from here, so they all round alike.
template <int N = 1>
DEV void cta_sum(const double* v, double* out)
{
    __shared__ double sm[N][8];
#pragma unroll
    for (int c = 0; c < N; ++c) {
        const double w = warp_sum(v[c]);
        if ((threadIdx.x & 31) == 0) sm[c][threadIdx.x >> 5] = w;
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += sm[threadIdx.x][w];
        out[threadIdx.x] = s;
    }
}

} // namespace ipcgpu
