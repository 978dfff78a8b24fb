// timestep.cu -- the time-integration frame of a time step on the device (sm_90a): the inertia target x~ (Optimizer::computeXTilta,
// Optimizer.cpp:1236-1278), the end-of-step update of Optimizer::solve for TIT_BE / TIT_NM (:572-590) and the predictor directions of
// Optimizer::initX options 1-4 (:930-1080).
//   *** compiled with --fmad=false (NOFMA_FILES): every expression keeps the reference's evaluation order and rounds each product and sum
//   separately, so the results are bit-identical to a float64 restatement ***
//
// Layouts are the reference's .data() layouts: velocity is an Eigen::VectorXd, interleaved 3 nV (component 3v + d); acceleration and
// dx_Elastic are Eigen::MatrixXd nV x 3, column-major (SoA, entry d nV + v); V, V_prev and x~ are SoA like every position array.  The
// reference pairs velocity component 3v + d with acceleration(v, d) through its RowMatrixXd maps.
//
// "Dirichlet" is Mesh::isDBCVertex (Mesh.hpp:134): dbc != 0.  The obstacle tail carries that flag, so its predictor is 0 and its x~ is V_prev.
// Every kernel reads the time-integration parameters from device memory (TimeParams), so a replayed graph uses the current dt / beta / gamma.
#include "common.cuh"
#include "kernels.h"
#include <algorithm>

namespace ipcgpu {

DEV bool dbc_vertex(const uint8_t* dbc, int v) { return dbc && dbc[v] != 0; }

// computeXTilta for one coordinate of a non-Dirichlet vertex: xp = V_prev(v, d), vel = velocity[3v + d], acc = acceleration(v, d)
DEV double xtilde_of(const TimeParams& q, int d, double xp, double vel, double acc)
{
    if (q.type == 0) return xp + (vel * q.dt + q.gDtSq[d]);                                           // :1250
    return xp + ((vel * q.dt + q.beta * q.gDtSq[d]) + (0.5 - q.beta) * (q.dtSq * acc));             // :1268
}

static int grid_of(int nV) { return std::max(1, std::min((nV + 255) / 256, kSMs * 8)); }

__global__ void __launch_bounds__(256) k_xtilde(DynamicsArgs p)
{
    const TimeParams q = *p.tp;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x) {
        const bool fixed = dbc_vertex(p.dbc, v);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const size_t i = (size_t)d * p.nV + v;
            const double xp = p.Vprev[i];
            p.xtilde[i] = fixed ? xp : xtilde_of(q, d, xp, p.vel[3 * (size_t)v + d], p.acc[i]);
        }
    }
}

// Optimizer::solve (:572-590): dx_Elastic, velocity, acceleration, V_prev = V, then computeXTilta with the new state.  Every read of x~ is
// the x~ of the step that just finished (each thread reads its own entries before it overwrites them).
__global__ void __launch_bounds__(256) k_end_time_step(DynamicsArgs p)
{
    const TimeParams q = *p.tp;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x) {
        const bool fixed = dbc_vertex(p.dbc, v);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const size_t i = (size_t)d * p.nV + v, k = 3 * (size_t)v + d;
            const double x = p.V[i], xt = p.xtilde[i];
            double vel = p.vel[k], acc;
            p.dxe[i] = x - xt; // dx_Elastic = result.V - xTilta
            if (q.type == 0) {
                const double vn = (x - p.Vprev[i]) / q.dt; // velocity = (V - V_prev) / dt
                acc = (vn - vel) / q.dt;                    // acceleration = (velocity - velocity_prev) / dt
                vel = vn;
            }
            else {
                vel = vel + (q.dt * (1.0 - q.gamma)) * p.acc[i];     // velocity + dt (1 - gamma) acceleration
                acc = (x - xt) / (q.dtSq * q.beta) + q.gravity[d];    // (V - xTilta) / (dtSq beta), rowwise += gravity
                vel = vel + (q.dt * q.gamma) * acc;                   // velocity += dt gamma acceleration
            }
            p.vel[k] = vel;
            p.acc[i] = acc;
            p.Vprev[i] = x; // result.V_prev = result.V
            p.xtilde[i] = fixed ? x : xtilde_of(q, d, x, vel, acc);
        }
    }
}

// initX (:930-1080): the predictor of option 1-4 (0: zero) into the search direction, interleaved, 0 on Dirichlet vertices
__global__ void __launch_bounds__(256) k_predictor(DynamicsArgs p, int option, double* __restrict__ dir)
{
    const TimeParams q = *p.tp;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x) {
        const bool fixed = dbc_vertex(p.dbc, v) || option == 0;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const size_t i = (size_t)d * p.nV + v, k = 3 * (size_t)v + d;
            double r = 0.0;
            if (!fixed) {
                const double dv = q.dt * p.vel[k];
                const bool be = q.type == 0;
                switch (option) {
                case 1: r = dv; break;                                                          // explicit Euler
                case 2: r = be ? dv + q.gDtSq[d] : dv + q.gDtSq[d] / 2.0; break;                 // xHat
                case 3: r = be ? (dv + q.gDtSq[d]) + p.dxe[i] : (dv + q.gDtSq[d] / 2.0) + p.dxe[i] * 2.0; break; // symplectic Euler
                default: r = be ? dv + (q.gDtSq[d] + 0.5 * p.dxe[i]) : (dv + q.gDtSq[d] / 2.0) + p.dxe[i]; break; // uniformly accelerated
                }
            }
            dir[k] = r;
        }
    }
}

void timestep_xtilde(const DynamicsArgs& p, cudaStream_t st)
{
    if (p.nV > 0) k_xtilde<<<grid_of(p.nV), 256, 0, st>>>(p);
}

void timestep_end(const DynamicsArgs& p, cudaStream_t st)
{
    if (p.nV > 0) k_end_time_step<<<grid_of(p.nV), 256, 0, st>>>(p);
}

void timestep_predictor(const DynamicsArgs& p, int option, double* dir, cudaStream_t st)
{
    if (p.nV > 0) k_predictor<<<grid_of(p.nV), 256, 0, st>>>(p, option, dir);
}

} // namespace ipcgpu
