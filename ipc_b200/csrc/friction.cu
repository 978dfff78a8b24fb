// friction.cu -- lagged smoothed-static-friction terms of the self-contact pairs (SURVEY 8 f4), sm_90a.
//
// Reference being replaced:
//   Optimizer.cpp:1582-1595                lagged normal force lambda_c = -kappa b'(d_c) 2 sqrt(d_c) * multiplicity
//   SelfCollisionHandler.cpp:2481-2527     computeDistCoordAndTanBasis  ("TODO: parallelize" serial loop)
//   SelfCollisionHandler.cpp:2529-2596     computeFrictionEnergy
//   SelfCollisionHandler.cpp:2598-2735     augmentFrictionGradient      (serial)
//   SelfCollisionHandler.cpp:2745-2987     augmentFrictionHessian       (12x12 makePD per pair + serial CSR add)
//   FrictionUtils.hpp:24-347               bases, closest points, lifts, C1 clamping (SFCLAMPING_ORDER 1, Types.hpp:42)
//
// Design (not a translation).  With w the stencil weights of the relative displacement (relDX = sum_k w_k dx_k), B the 3x2 lagged tangent
// basis and u = B^T relDX, every friction term lives in the 2-dimensional tangent plane:
//     E_c = coef lambda f0(|u|),   g_k = coef lambda f1(|u|)/|u| * w_k B u,   H_kl = w_k w_l * B S B^T,
//     S   = coef lambda [ e_perp (I - uu^T/|u|^2) + e_par uu^T/|u|^2 ],   sliding: e_perp = 1/|u|, e_par = 0;  sticking: e_perp = f1/|u|, e_par = f2.
// The reference forms the 12x12 matrix T^T S T and eigen-decomposes it (makePD); its non-zero spectrum is (sum w^2) * eig(S), so the
// projection is the clamp of the two eigenvalues of S -- done here in closed form on e_perp, e_par.  One thread per pair, ten 3x3 blocks
// w_k w_l M (M = B S B^T is symmetric, so no orientation case) added straight into the CSR rows this rank owns.
#include "repro.cuh"

namespace ipcgpu {

struct FricPair {
    PairStencil s;
    double w[4];
    V3 b0, b1;
    double u0, u1;
};

DEV void fric_weights(int kind, double c0, double c1, double* w)
{
    if (kind == 0) { w[0] = 1.0; w[1] = -1.0 + c0 + c1; w[2] = -c0; w[3] = -c1; }          // PT  FrictionUtils.hpp:48-57
    else if (kind == 1) { w[0] = 1.0 - c0; w[1] = c0; w[2] = c1 - 1.0; w[3] = -c1; }       // EE  :131-140
    else if (kind == 2) { w[0] = 1.0; w[1] = c0 - 1.0; w[2] = -c0; w[3] = 0.0; }           // PE  :183-191
    else { w[0] = 1.0; w[1] = -1.0; w[2] = 0.0; w[3] = 0.0; }                              // PP  :246-252
}

// kUnrolled: the stencil loop unrolled with a guard, so that dx stays in registers (the reproducible mode's staging kernel; the other
// kernels keep the loop they were tuned with)
template <bool kUnrolled = false>
DEV FricPair fric_pair(const FrictionArgs& p, int c)
{
    FricPair f;
    f.s = decode(p.cs[c]);
    const double2 co = p.coord[c];
    fric_weights(f.s.kind, co.x, co.y, f.w);
    const double* B = p.basis + 6 * (size_t)c;
    f.b0 = { B[0], B[1], B[2] };
    f.b1 = { B[3], B[4], B[5] };
    V3 dx[4];
    if (kUnrolled) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (k < f.s.nv) dx[k] = load_vertex(p.V, p.nV, f.s.v[k]) - load_vertex(p.Vt, p.nV, f.s.v[k]);
    }
    else
        for (int k = 0; k < f.s.nv; ++k) dx[k] = load_vertex(p.V, p.nV, f.s.v[k]) - load_vertex(p.Vt, p.nV, f.s.v[k]);
    V3 r; // relDX3D in the reference's own association (FrictionUtils.hpp:48-57, 131-140, 183-191, 246-252)
    if (f.s.kind == 0) r = dx[0] - (dx[1] + co.x * (dx[2] - dx[1]) + co.y * (dx[3] - dx[1]));
    else if (f.s.kind == 1) r = dx[0] + co.x * (dx[1] - dx[0]) - (dx[2] + co.y * (dx[3] - dx[2]));
    else if (f.s.kind == 2) r = dx[0] - (dx[1] + co.x * (dx[2] - dx[1]));
    else r = dx[0] - dx[1];
    f.u0 = dot(r, f.b0);
    f.u1 = dot(r, f.b1);
    return f;
}

DEV V3 unit_or_self(V3 a)
{
    const double z = norm2(a);
    return z > 0.0 ? (1.0 / sqrt(z)) * a : a;
}

// -----------------------------------------------------------------------------------------------------------
// lag: snapshot of the active set + lambda, closest-point coordinates, tangent bases at the current positions
// -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_friction_lag(BarrierArgs p, int4* __restrict__ cs_out, int* __restrict__ n_out, double* __restrict__ lambda,
    double2* __restrict__ coord, double* __restrict__ basis, int capacity, int* __restrict__ bad)
{
    const int n = min(*p.nC, capacity);
    const double kappa = p.kappa_dev ? *p.kappa_dev : p.kappa;
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_out = n;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int4 mm = p.cs[c];
        const PairStencil s = decode(mm);
        V3 x[4];
        load_stencil(s, p.V, p.nV, x);
        const double d = pair_distance(s, x);
        if (!(d > 0.0)) atomicExch(bad, 1);
        double b, db, d2b;
        barrier_all(d, p.dHat, b, db, d2b);
        double lam = db;
        lam *= -kappa * 2.0 * sqrt(d);
        if (mm.x < 0 && mm.w < -1) lam *= (double)(-mm.w); // PP or PE duplication (Optimizer.cpp:1588-1591)
        // no friction against a mesh obstacle: the reference's MeshCO does not implement the friction functions (CollisionObject.h:403-423 throw),
        // Optimizer.cpp:1582-1600 lags the self-contact set only.  A zero normal force switches the pair's E / g / H off.
        for (int k = 0; k < s.nv; ++k)
            if (s.v[k] >= p.nVdof) lam = 0.0;
        double c0 = 0.0, c1 = 0.0;
        V3 b0, b1;
        if (s.kind == 0) {        // PT: FrictionUtils.hpp:24-46
            const V3 r0 = x[2] - x[1], r1 = x[3] - x[1], rel = x[0] - x[1];
            ldlt2(dot(r0, r0), dot(r0, r1), dot(r1, r1), dot(r0, rel), dot(r1, rel), c0, c1);
            b0 = unit_or_self(r0);
            b1 = unit_or_self(cross(cross(r0, r1), r0));
        }
        else if (s.kind == 1) {   // EE: :95-129
            const V3 e20 = x[0] - x[2], e01 = x[1] - x[0], e23 = x[3] - x[2];
            ldlt2(dot(e01, e01), -dot(e23, e01), dot(e23, e23), -dot(e20, e01), dot(e20, e23), c0, c1);
            b0 = unit_or_self(e01);
            b1 = unit_or_self(cross(cross(e01, e23), e01));
        }
        else if (s.kind == 2) {   // PE: :163-181
            const V3 e12 = x[2] - x[1];
            c0 = dot(x[0] - x[1], e12) / dot(e12, e12);
            b0 = unit_or_self(e12);
            b1 = unit_or_self(cross(e12, x[0] - x[1]));
        }
        else {                    // PP: :227-244
            const V3 v01 = x[1] - x[0];
            const V3 xc = cross(V3{ 1.0, 0.0, 0.0 }, v01), yc = cross(V3{ 0.0, 1.0, 0.0 }, v01);
            if (norm2(xc) > norm2(yc)) { b0 = unit_or_self(xc); b1 = unit_or_self(cross(v01, xc)); }
            else { b0 = unit_or_self(yc); b1 = unit_or_self(cross(v01, yc)); }
        }
        cs_out[c] = mm;
        lambda[c] = lam;
        coord[c] = make_double2(c0, c1);
        double* B = basis + 6 * (size_t)c;
        B[0] = b0.x; B[1] = b0.y; B[2] = b0.z; B[3] = b1.x; B[4] = b1.y; B[5] = b1.z;
    }
}

// C1 clamping (FrictionUtils.hpp:278-292)
DEV double f0_SF(double x2, double eps) { return x2 * (-sqrt(x2) / 3.0 + eps) / (eps * eps) + eps / 3.0; }
DEV double f1_SF_div(double x2, double eps) { return (-sqrt(x2) + 2.0 * eps) / (eps * eps); }
DEV double f2_SF(double x2, double eps) { return 2.0 * (eps - sqrt(x2)) / (eps * eps); }

struct FricRange {
    int b, e;
};
DEV FricRange fric_range(const FrictionArgs& p)
{
    const long long n = *p.n;
    if (p.nranks > 1) return { (int)(n * p.rank / p.nranks), (int)(n * (p.rank + 1) / p.nranks) };
    return { 0, (int)n };
}

constexpr int kFricEnergyBlocks = kSMs * 2;
__global__ void __launch_bounds__(256) k_friction_energy(FrictionArgs p, double* __restrict__ partials)
{
    const FricRange r = fric_range(p);
    const double eps = sqrt(p.eps2);
    double val = 0.0;
    for (int c = r.b + blockIdx.x * blockDim.x + threadIdx.x; c < r.e; c += gridDim.x * blockDim.x) {
        const FricPair f = fric_pair(p, c);
        const double x2 = f.u0 * f.u0 + f.u1 * f.u1;
        val += (x2 > p.eps2) ? p.lambda[c] * sqrt(x2) : p.lambda[c] * f0_SF(x2, eps);
    }
    cta_sum(&val, partials + blockIdx.x);
}

// kStage: the contributions go to the staging array under their gradient keys (repro.cuh)
template <bool kStage>
__global__ void __launch_bounds__(128) k_friction_gradient(FrictionArgs p, double* __restrict__ g)
{
    const FricRange r = fric_range(p);
    const double eps = sqrt(p.eps2);
    for (int c = r.b + blockIdx.x * blockDim.x + threadIdx.x; c < r.e; c += gridDim.x * blockDim.x) {
        const FricPair f = fric_pair<kStage>(p, c);
        const double x2 = f.u0 * f.u0 + f.u1 * f.u1;
        double u0 = f.u0, u1 = f.u1;
        if (x2 > p.eps2) { const double n = sqrt(x2); u0 /= n; u1 /= n; }
        else { const double s = f1_SF_div(x2, eps); u0 *= s; u1 *= s; }
        const V3 t = u0 * f.b0 + u1 * f.b1;
        const double cl = p.coef * p.lambda[c];
#pragma unroll
        for (int k = 0; k < 4; ++k) { // (unrolled with a guard: the stencil stays in registers)
            if (k >= f.s.nv) continue;
            const double wk = f.w[k] * cl;
            put_g<kStage>(g, f.s.v[k], gkey_active(c, k), 0, wk * t.x);
            put_g<kStage>(g, f.s.v[k], gkey_active(c, k), 1, wk * t.y);
            put_g<kStage>(g, f.s.v[k], gkey_active(c, k), 2, wk * t.z);
        }
    }
}

// the projected tangent-plane block M = B S B^T of pair f (symmetric, row-major)
DEV void fric_block(const FrictionArgs& p, const FricPair& f, int c, double eps, double* M)
{
    const double x2 = f.u0 * f.u0 + f.u1 * f.u1, xn = sqrt(x2);
    const double cl = p.coef * p.lambda[c];
    // eigenvalues of S across / along the slip direction
    double e_perp, e_par;
    if (x2 > p.eps2) { e_perp = cl / xn; e_par = 0.0; }                 // :2776-2786  c lam (I/|u| - uu^T/|u|^3)
    else {                                                               // :2787-2804
        const double f1 = f1_SF_div(x2, eps), f2 = f2_SF(x2, eps);
        e_perp = cl * f1;
        e_par = (f2 != f1 && x2 != 0.0) ? cl * f2 : e_perp;
    }
    // makePD (IglUtils.hpp:119-133): clamp of the spectrum -- here the two eigenvalues of S
    e_perp = fmax(e_perp, 0.0);
    e_par = fmax(e_par, 0.0);
    // M = B S B^T = e_perp (b0 b0^T + b1 b1^T) + (e_par - e_perp) t t^T,  t = B u / |u|
    {
        V3 t = { 0.0, 0.0, 0.0 };
        if (x2 > 0.0) t = (f.u0 / xn) * f.b0 + (f.u1 / xn) * f.b1;
        const double de = e_par - e_perp;
        const double b0v[3] = { f.b0.x, f.b0.y, f.b0.z }, b1v[3] = { f.b1.x, f.b1.y, f.b1.z }, tv[3] = { t.x, t.y, t.z };
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) M[3 * i + j] = e_perp * (b0v[i] * b0v[j] + b1v[i] * b1v[j]) + de * (tv[i] * tv[j]);
    }
}

__global__ void __launch_bounds__(128) k_friction_hessian(FrictionArgs p, double* __restrict__ a, int* __restrict__ err)
{
    const int n = *p.n;
    const double eps = sqrt(p.eps2);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const FricPair f = fric_pair(p, c);
        bool mine = false; // row-owner rule: a rank adds only the block rows it owns
        for (int k = 0; k < f.s.nv; ++k) mine = mine || (f.s.v[k] >= p.row_lo && f.s.v[k] < p.row_hi);
        if (!mine) continue;
        double M[9];
        fric_block(p, f, c, eps, M);
        for (int bi = 0; bi < f.s.nv; ++bi) {
            for (int bj = bi; bj < f.s.nv; ++bj) {
                const int vi = min(f.s.v[bi], f.s.v[bj]), vj = max(f.s.v[bi], f.s.v[bj]);
                if (vi < p.row_lo || vi >= p.row_hi) continue;
                if (proj_dbc(p.dbc, vi, p.projectDBC) || proj_dbc(p.dbc, vj, p.projectDBC)) continue;
                const double ww = f.w[bi] * f.w[bj];
                for (int r = 0; r < 3; ++r) {
                    const int c0 = (bi == bj) ? r : 0;
                    const int o = csr_find(p.ia, p.ja, p.base, 3 * vi + r, 3 * vj + c0);
                    if (o < 0) { atomicExch(err, 1); continue; }
                    for (int q = c0; q < 3; ++q) atomicAdd(a + o + (q - c0), ww * M[3 * r + q]);
                }
            }
        }
    }
}

// reproducible mode: M and the stencil weights of every pair to hstage (13 doubles per pair), then a per-row gather (repro.cuh) of the blocks
// w_bi w_bj M, one thread per row vertex
__global__ void __launch_bounds__(128) k_friction_hessian_stage(FrictionArgs p)
{
    const int n = *p.n;
    const double eps = sqrt(p.eps2);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const FricPair f = fric_pair<true>(p, c);
        double* out = p.rep.hstage + 13 * (size_t)c;
        fric_block(p, f, c, eps, out);
        for (int k = 0; k < 4; ++k) out[9 + k] = f.w[k];
    }
}
__global__ void __launch_bounds__(128) k_friction_hessian_gather(FrictionArgs p, double* __restrict__ a, int* __restrict__ err)
{
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x)
        repro_gather_row(v, p.rep.h, p.dbc, p.projectDBC, p.ia, p.ja, p.base, a, err, [&](int c, int bi, int bj, double* acc) {
            const double* S = p.rep.hstage + 13 * (size_t)c;
            const double ww = S[9 + bi] * S[9 + bj];
            for (int i = 0; i < 9; ++i) acc[i] += ww * S[i];
        });
}

// -----------------------------------------------------------------------------------------------------------
void friction_lag(const BarrierArgs& p, int4* cs_out, int* n_out, double* lambda, double2* coord, double* basis, int capacity, int* bad, cudaStream_t st)
{
    k_friction_lag<<<kSMs * 4, 128, 0, st>>>(p, cs_out, n_out, lambda, coord, basis, capacity, bad);
}
void friction_energy(const FrictionArgs& p, double* partials, cudaStream_t st) { k_friction_energy<<<kFricEnergyBlocks, 256, 0, st>>>(p, partials); }
int friction_energy_blocks() { return kFricEnergyBlocks; }
void friction_gradient(const FrictionArgs& p, double* g, cudaStream_t st)
{
    if (p.rep.on) {
        k_friction_gradient<true><<<kSMs * 4, 128, 0, st>>>(p, p.rep.stage);
        repro_gather_g(p.nV, p.rep.g, p.rep.stage, 0ull, ~0ull, g, st);
    }
    else k_friction_gradient<false><<<kSMs * 4, 128, 0, st>>>(p, g);
}
void friction_hessian(const FrictionArgs& p, double* a, int* err, cudaStream_t st)
{
    if (p.rep.on) {
        k_friction_hessian_stage<<<kSMs * 4, 128, 0, st>>>(p);
        k_friction_hessian_gather<<<kSMs * 4, 128, 0, st>>>(p, a, err);
    }
    else k_friction_hessian<<<kSMs * 4, 128, 0, st>>>(p, a, err);
}

} // namespace ipcgpu
