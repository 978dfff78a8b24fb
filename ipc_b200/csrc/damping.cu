// damping.cu -- the last terms of Optimizer::computeEnergyVal / computeGradient / computePrecondMtr that used to stay on the host (sm_90a):
// Rayleigh damping 1/2 d^T D d (Optimizer.cpp:3381-3400, :3519-3540, :3707-3709, D from computeDampingMtr :3723-3734), the Neumann forces
// (:3241-3250, :3452-3461) and the augmented-Lagrangian Dirichlet penalty (AnimScripter.cpp:2286-2344).
//
// D is held once, in the elastic slot order of api_mesh.cu's build_maps: one full 3x3 row-major block per mesh vertex pair (slot_v <= slot_u),
// so it does not depend on the system's sparsity pattern (host- or device-built); slot_off places a block in the CSR.  Every sum is in a
// fixed order (per-CTA partials, then k_reduce_sum; the per-vertex gather walks a slot incidence list built once per mesh): no atomics,
// the results are bitwise reproducible and an eager and a replayed line search take the same Armijo decisions.
#include "common.cuh"
#include "kernels.h"
#include <algorithm>

namespace ipcgpu {

// a projected Dirichlet vertex (Mesh::isProjectDBCVertex, Mesh.hpp:135-143; dbc: 0 NOT_DBC, 1 ZERO, 2 NONZERO)
DEV bool projected(const uint8_t* dbc, int v, int projectDBC) { return dbc && (dbc[v] == 1 || (dbc[v] == 2 && projectDBC)); }

// d_v = x_v - x_prev,v, zeroed on the vertices `zero` names
DEV void displacement(int nV, const double* __restrict__ x, const double* __restrict__ xp, int v, bool zero, double d[3])
{
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = zero ? 0.0 : x[(size_t)c * nV + v] - xp[(size_t)c * nV + v];
}

// ---- damping ---------------------------------------------------------------------------------------------------------------------
// computeDampingMtr's assembly (Energy.cpp:317-330 with projectDBC = 1 -> IglUtils::addBlockToMatrix, IglUtils.hpp:44-80) into slot storage:
// the per-tet blocks of k_elastic_grad_hess (Hessian only, coef, projected) summed in ascending tet order as k_assemble_csr sums them; a block
// with a Dirichlet vertex is dropped, except that the diagonal block of a Dirichlet vertex is SET to the identity (setCoeff, :45-52).  9 threads
// per slot, one per upper entry (diagonal slots: 6); both triangles of a diagonal block are written
__global__ void __launch_bounds__(288) k_damping_assemble(int nSlots, const int* __restrict__ slot_v, const int* __restrict__ slot_u,
    const int* __restrict__ con_ptr, const unsigned* __restrict__ con_src, const double* __restrict__ hblk, const uint8_t* __restrict__ dbc,
    double* __restrict__ D)
{
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int s = (int)(tid / 9), q = (int)(tid - 9ll * s);
    if (s >= nSlots) return;
    const int v = slot_v[s], u = slot_u[s];
    const bool diag = (v == u);
    if (diag && q >= 6) return;
    const bool dropped = projected(dbc, v, 1) || projected(dbc, u, 1);
    int r, c;
    if (diag) { r = (q < 3) ? 0 : (q < 5 ? 1 : 2); c = (q < 3) ? q : (q < 5 ? q - 2 : 2); } // upper entry (r, c), c >= r
    else { r = q / 3; c = q - 3 * r; }
    double h = 0.0;
    if (!dropped) {
        const int b = con_ptr[s], e = con_ptr[s + 1];
#pragma unroll 4
        for (int k = b; k < e; ++k) h += hblk[__ldg(con_src + k) + q];
    }
    else if (diag && r == c) h = 1.0;
    double* B = D + 9 * (size_t)s;
    B[3 * r + c] = h;
    if (diag) B[3 * c + r] = h;
}

// 1/2 d^T D d with every Dirichlet row of d zeroed (:3381-3400): slot s adds (2 - delta_vu) d_v^T B_s d_u; scaled by 1/2 in the reduce
__global__ void __launch_bounds__(256) k_damping_energy(int nSlots, const int* __restrict__ slot_v, const int* __restrict__ slot_u, const double* __restrict__ D,
    int nV, const double* __restrict__ x, const double* __restrict__ xp, const uint8_t* __restrict__ dbc, double* __restrict__ partials)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (s < nSlots) {
        const int v = slot_v[s], u = slot_u[s];
        double dv[3], du[3];
        displacement(nV, x, xp, v, dbc && dbc[v], dv);
        displacement(nV, x, xp, u, dbc && dbc[u], du);
        const double* B = D + 9 * (size_t)s;
#pragma unroll
        for (int r = 0; r < 3; ++r) e += dv[r] * ((B[3 * r] * du[0] + B[3 * r + 1] * du[1]) + B[3 * r + 2] * du[2]);
        if (v != u) e *= 2.0;
    }
    cta_sum(&e, partials + blockIdx.x);
}

// g += D d (:3519-3540), d zeroed on the projected Dirichlet vertices: one thread per vertex gathers its row of the symmetric product over
// the slot incidence list (entry 2s: slot s has the vertex as slot_v, B_s d_u; entry 2s + 1: as slot_u of an off-diagonal slot, B_s^T d_v)
__global__ void __launch_bounds__(256) k_damping_gradient(int nV, const int* __restrict__ inc_ptr, const int* __restrict__ inc, const int* __restrict__ slot_v,
    const int* __restrict__ slot_u, const double* __restrict__ D, const double* __restrict__ x, const double* __restrict__ xp, const uint8_t* __restrict__ dbc,
    int projectDBC, double* __restrict__ g)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    double acc[3] = { 0.0, 0.0, 0.0 };
    const int e = inc_ptr[v + 1];
    for (int k = inc_ptr[v]; k < e; ++k) {
        const int ent = __ldg(inc + k), s = ent >> 1;
        const bool tr = ent & 1;
        const int w = tr ? __ldg(slot_v + s) : __ldg(slot_u + s);
        double d[3];
        displacement(nV, x, xp, w, projected(dbc, w, projectDBC), d);
        const double* B = D + 9 * (size_t)s;
        if (!tr) {
#pragma unroll
            for (int r = 0; r < 3; ++r) acc[r] += (B[3 * r] * d[0] + B[3 * r + 1] * d[1]) + B[3 * r + 2] * d[2];
        }
        else {
#pragma unroll
            for (int r = 0; r < 3; ++r) acc[r] += (B[r] * d[0] + B[3 + r] * d[1]) + B[6 + r] * d[2];
        }
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) g[3 * (size_t)v + r] += acc[r];
}

// addCoeff(dampingMtr, 1.0) (:3707-3709): every block added at its CSR offsets (slot_off, as k_assemble_csr writes them)
__global__ void __launch_bounds__(288) k_damping_hessian(int nSlots, const int* __restrict__ slot_v, const int* __restrict__ slot_u, const int* __restrict__ slot_off,
    const double* __restrict__ D, double* __restrict__ a)
{
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int s = (int)(tid / 9), q = (int)(tid - 9ll * s);
    if (s >= nSlots) return;
    const bool diag = slot_v[s] == slot_u[s];
    if (diag && q >= 6) return;
    int r, c; // row inside the block, column relative to the row's slot offset
    if (diag) { r = (q < 3) ? 0 : (q < 5 ? 1 : 2); c = (q < 3) ? q : (q < 5 ? q - 3 : 0); }
    else { r = q / 3; c = q - 3 * r; }
    a[slot_off[3 * s + r] + c] += D[9 * (size_t)s + 3 * r + (diag ? r + c : c)];
}

// ---- Neumann forces (:3241-3250, :3452-3461): every non-Dirichlet vertex, whatever projectDBC is ------------------------------------
__global__ void __launch_bounds__(256) k_neumann_energy(int nV, const double* __restrict__ x, const double* __restrict__ f, const double* __restrict__ mass,
    const uint8_t* __restrict__ dbc, const double* __restrict__ coef_p, double* __restrict__ partials)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const double coef = *coef_p;
    double e = 0.0;
    if (v < nV && !(dbc && dbc[v])) {
        const double dot = (x[v] * f[3 * (size_t)v] + x[(size_t)nV + v] * f[3 * (size_t)v + 1]) + x[2 * (size_t)nV + v] * f[3 * (size_t)v + 2];
        e = -((coef * mass[v]) * dot);
    }
    cta_sum(&e, partials + blockIdx.x);
}
__global__ void __launch_bounds__(256) k_neumann_gradient(int nV, const double* __restrict__ f, const double* __restrict__ mass, const uint8_t* __restrict__ dbc,
    const double* __restrict__ coef, double* __restrict__ g)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV || (dbc && dbc[v])) return;
    const double cm = *coef * mass[v];
#pragma unroll
    for (int r = 0; r < 3; ++r) g[3 * (size_t)v + r] -= cm * f[3 * (size_t)v + r];
}

// ---- augmented-Lagrangian Dirichlet penalty (AnimScripter.cpp:2286-2344): per target i, vertex vid[i], target t_i, multiplier lambda_i; rho is
// read from device memory, and rho == 0 adds nothing (Optimizer.cpp:3402, :3542, :3711) ----------------------------------------------------
DEV double sq_dist(int nV, const double* __restrict__ x, int v, const double* __restrict__ t, double dx[3])
{
#pragma unroll
    for (int c = 0; c < 3; ++c) dx[c] = x[(size_t)c * nV + v] - t[c];
    return (dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2];
}
__global__ void __launch_bounds__(256) k_dirichlet_energy(int n, const int* __restrict__ vid, const double* __restrict__ tgt, const double* __restrict__ lam,
    int nV, const double* __restrict__ x, const double* __restrict__ mass, const double* __restrict__ rho_p, double* __restrict__ partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double rho = *rho_p;
    double e = 0.0;
    if (i < n && rho != 0.0) { // augmentMDBCEnergy (:2303-2311)
        const int v = vid[i];
        double dx[3];
        const double sq = sq_dist(nV, x, v, tgt + 3 * (size_t)i, dx);
        const double* l = lam + 3 * (size_t)i;
        const double m = mass[v];
        e = rho / 2.0 * m * sq - sqrt(m) * ((l[0] * dx[0] + l[1] * dx[1]) + l[2] * dx[2]);
    }
    cta_sum(&e, partials + blockIdx.x);
}
__global__ void __launch_bounds__(256) k_dirichlet_gradient(int n, const int* __restrict__ vid, const double* __restrict__ tgt, const double* __restrict__ lam,
    int nV, const double* __restrict__ x, const double* __restrict__ mass, const double* __restrict__ rho_p, double* __restrict__ g)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double rho = *rho_p;
    if (i >= n || rho == 0.0) return;
    const int v = vid[i];
    double dx[3];
    sq_dist(nV, x, v, tgt + 3 * (size_t)i, dx);
    const double m = mass[v], sm = sqrt(m);
#pragma unroll
    for (int r = 0; r < 3; ++r) g[3 * (size_t)v + r] = (g[3 * (size_t)v + r] - sm * lam[3 * (size_t)i + r]) + rho * m * dx[r]; // :2314-2321
}
// augmentMDBCHessian (:2323-2336): rho m on the vertex's three diagonal entries, the first stored entry of each upper-triangular row
__global__ void __launch_bounds__(256) k_dirichlet_hessian(int n, const int* __restrict__ vid, const double* __restrict__ mass, const double* __restrict__ rho_p,
    const int* __restrict__ ia, int base, double* __restrict__ a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double rho = *rho_p;
    if (i >= n || rho == 0.0) return;
    const int v = vid[i];
    const double val = rho * mass[v];
#pragma unroll
    for (int r = 0; r < 3; ++r) a[ia[3 * v + r] - base] += val;
}
// updateLambda (:2338-2345)
__global__ void __launch_bounds__(256) k_dirichlet_update_lambda(int n, const int* __restrict__ vid, const double* __restrict__ tgt, int nV, const double* __restrict__ x,
    const double* __restrict__ mass, const double* __restrict__ rho_p, double* __restrict__ lam)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int v = vid[i];
    double dx[3];
    sq_dist(nV, x, v, tgt + 3 * (size_t)i, dx);
    const double w = *rho_p * sqrt(mass[v]);
#pragma unroll
    for (int r = 0; r < 3; ++r) lam[3 * (size_t)i + r] -= w * dx[r];
}
// computeCompletedStepSize (:2286-2300): the squared distances to the targets, then 1 - sqrt(sqNorm / (dist2Tol 1e6))
__global__ void __launch_bounds__(256) k_dirichlet_sqnorm(int n, const int* __restrict__ vid, const double* __restrict__ tgt, int nV, const double* __restrict__ x,
    double* __restrict__ partials)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (i < n) {
        double dx[3];
        e = sq_dist(nV, x, vid[i], tgt + 3 * (size_t)i, dx);
    }
    cta_sum(&e, partials + blockIdx.x);
}
__global__ void k_dirichlet_step(const double* __restrict__ tol_p, double* __restrict__ s)
{
    if (threadIdx.x != 0) return;
    const double dist2Tol = *tol_p; // (device-resident: a new value per time step needs no new capture)
    s[0] = dist2Tol == 0.0 ? 1.0 : 1.0 - sqrt(s[0] / (dist2Tol * 1.0e6));
}
__global__ void k_set_double(double* p, double v)
{
    if (threadIdx.x == 0) p[0] = v;
}

// ---- launchers -----------------------------------------------------------------------------------------------------------------------
static int blocks256(int n) { return (n + 255) / 256; }
static int blocks_slots9(int nSlots) { return (int)(((long long)nSlots * 9 + 287) / 288); }

void damping_assemble(int nSlots, const int* slot_v, const int* slot_u, const int* con_ptr, const unsigned* con_src, const double* hblk, const uint8_t* dbc,
    double* D, cudaStream_t st)
{
    if (nSlots > 0) k_damping_assemble<<<blocks_slots9(nSlots), 288, 0, st>>>(nSlots, slot_v, slot_u, con_ptr, con_src, hblk, dbc, D);
}
int damping_energy_blocks(int nSlots) { return blocks256(nSlots); }
void damping_energy(const DampingArgs& p, double* partials, cudaStream_t st)
{
    if (p.nSlots > 0) k_damping_energy<<<blocks256(p.nSlots), 256, 0, st>>>(p.nSlots, p.slot_v, p.slot_u, p.D, p.nV, p.V, p.Vprev, p.dbc, partials);
}
void damping_gradient(const DampingArgs& p, int projectDBC, double* g, cudaStream_t st)
{
    if (p.nV > 0) k_damping_gradient<<<blocks256(p.nV), 256, 0, st>>>(p.nV, p.inc_ptr, p.inc, p.slot_v, p.slot_u, p.D, p.V, p.Vprev, p.dbc, projectDBC, g);
}
void damping_hessian(const DampingArgs& p, const int* slot_off, double* a, cudaStream_t st)
{
    if (p.nSlots > 0) k_damping_hessian<<<blocks_slots9(p.nSlots), 288, 0, st>>>(p.nSlots, p.slot_v, p.slot_u, slot_off, p.D, a);
}
int vertex_energy_blocks(int n) { return blocks256(n); }
void neumann_energy(int nV, const double* x, const double* f, const double* mass, const uint8_t* dbc, const double* coef, double* partials, cudaStream_t st)
{
    if (nV > 0) k_neumann_energy<<<blocks256(nV), 256, 0, st>>>(nV, x, f, mass, dbc, coef, partials);
}
void neumann_gradient(int nV, const double* f, const double* mass, const uint8_t* dbc, const double* coef, double* g, cudaStream_t st)
{
    if (nV > 0) k_neumann_gradient<<<blocks256(nV), 256, 0, st>>>(nV, f, mass, dbc, coef, g);
}
void dirichlet_energy(const DirichletArgs& p, double* partials, cudaStream_t st)
{
    if (p.n > 0) k_dirichlet_energy<<<blocks256(p.n), 256, 0, st>>>(p.n, p.vid, p.tgt, p.lam, p.nV, p.V, p.mass, p.rho, partials);
}
void dirichlet_gradient(const DirichletArgs& p, double* g, cudaStream_t st)
{
    if (p.n > 0) k_dirichlet_gradient<<<blocks256(p.n), 256, 0, st>>>(p.n, p.vid, p.tgt, p.lam, p.nV, p.V, p.mass, p.rho, g);
}
void dirichlet_hessian(const DirichletArgs& p, const int* ia, int base, double* a, cudaStream_t st)
{
    if (p.n > 0) k_dirichlet_hessian<<<blocks256(p.n), 256, 0, st>>>(p.n, p.vid, p.mass, p.rho, ia, base, a);
}
void dirichlet_update_lambda(const DirichletArgs& p, double* lam, cudaStream_t st)
{
    if (p.n > 0) k_dirichlet_update_lambda<<<blocks256(p.n), 256, 0, st>>>(p.n, p.vid, p.tgt, p.nV, p.V, p.mass, p.rho, lam);
}
void dirichlet_completed_step(const DirichletArgs& p, const double* dist2Tol, double* partials, double* out, cudaStream_t st)
{
    const int nb = blocks256(p.n);
    if (nb > 0) k_dirichlet_sqnorm<<<nb, 256, 0, st>>>(p.n, p.vid, p.tgt, p.nV, p.V, partials);
    reduce_sum(partials, nb, 1.0, out, st);
    k_dirichlet_step<<<1, 32, 0, st>>>(dist2Tol, out);
}
void set_double(double* p, double v, cudaStream_t st) { k_set_double<<<1, 32, 0, st>>>(p, v); }

} // namespace ipcgpu
