// misc.cu -- small per-vertex kernels the Newton driver runs between the hot stages.
#include "common.cuh"
#include "kernels.h"
#include <algorithm>

namespace ipcgpu {

// Optimizer::stepForward (src/TimeStepper/Optimizer.cpp:2919-2938): x = x0 + alpha * p, alpha from the host or (alpha_ord != nullptr) the
// device-resident step of a line search
__global__ void __launch_bounds__(256) k_step_forward(int nV, const double* __restrict__ x0, const double* __restrict__ p, double alpha, double* __restrict__ x,
    const unsigned long long* __restrict__ alpha_ord)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    if (alpha_ord) alpha = ord_to_dbl(*alpha_ord);
#pragma unroll
    for (int c = 0; c < 3; ++c) x[(size_t)c * nV + v] = x0[(size_t)c * nV + v] + alpha * p[3 * (size_t)v + c];
}

void step_forward(int nV, const double* x0, const double* p, double alpha, double* x, cudaStream_t st, const unsigned long long* alpha_ord)
{
    if (nV > 0) k_step_forward<<<(nV + 255) / 256, 256, 0, st>>>(nV, x0, p, alpha, x, alpha_ord);
}

// inertia term of Optimizer::computeEnergyVal (Optimizer.cpp:3227-3239): sum_v |x_v - xtilde_v|^2 m_v / 2 over the vertices [v0, v1)
// (fixed-order two-level sum: per-CTA partials, then k_reduce_sum)
__global__ void __launch_bounds__(256) k_inertia_energy(int v0, int v1, int nV, const double* __restrict__ x, const double* __restrict__ xt, const double* __restrict__ mass,
    double* __restrict__ partials)
{
    const int v = v0 + blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (v < v1) {
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double d = x[(size_t)c * nV + v] - xt[(size_t)c * nV + v];
            s += d * d;
        }
        e = s * mass[v] / 2.0;
    }
    cta_sum(&e, partials + blockIdx.x);
}
// ... and of computeGradient (:3439-3450): g_v += m_v (x_v - xtilde_v) unless v is a projected Dirichlet vertex
__global__ void __launch_bounds__(256) k_inertia_gradient(int nV, const double* __restrict__ x, const double* __restrict__ xt, const double* __restrict__ mass,
    const uint8_t* __restrict__ dbc, int projectDBC, double* __restrict__ g)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    if (dbc && (dbc[v] == 1 || (dbc[v] == 2 && projectDBC))) return;
    const double m = mass[v];
#pragma unroll
    for (int c = 0; c < 3; ++c) g[3 * (size_t)v + c] += m * (x[(size_t)c * nV + v] - xt[(size_t)c * nV + v]);
}
int inertia_energy_blocks(int nV) { return (nV + 255) / 256; }
void inertia_energy(int v0, int v1, int nV, const double* x, const double* xt, const double* mass, double* partials, cudaStream_t st)
{
    if (v1 > v0) k_inertia_energy<<<(v1 - v0 + 255) / 256, 256, 0, st>>>(v0, v1, nV, x, xt, mass, partials);
}
void inertia_gradient(int nV, const double* x, const double* xt, const double* mass, const uint8_t* dbc, int projectDBC, double* g, cudaStream_t st)
{
    if (nV > 0) k_inertia_gradient<<<(nV + 255) / 256, 256, 0, st>>>(nV, x, xt, mass, dbc, projectDBC, g);
}

__global__ void __launch_bounds__(256) k_zero_words(size_t n, unsigned* __restrict__ p)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = 0u;
}
void zero_words(void* p, size_t n_words, cudaStream_t st)
{
    if (n_words) k_zero_words<<<(unsigned)std::min<size_t>((n_words + 255) / 256, (size_t)kSMs * 16), 256, 0, st>>>(n_words, static_cast<unsigned*>(p));
}

} // namespace ipcgpu
