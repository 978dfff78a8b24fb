// halfspace.cu -- analytic half-space collision objects (HalfSpace<3>: script tokens `ground` / `halfSpace`, Config.cpp:425-447) on the
// device, sm_90a.
//   *** compiled with --fmad=false (NOFMA_FILES): n.x = (n0 x0 + n1 x1) + n2 x2 rounds like the -ffp-contract=off oracle, so the active set,
//   the crossing count and the step bound are bit-identical to it ***
//
// Reference being replaced (DESIGN.md section 3.12):
//   CollisionObject.h:323-352    computeConstraintSet: SVI vertices, not Dirichlet, codimension 3, d = dist^2 < dHat
//   HalfSpace.cpp:106-111        dist = n.x + D, d = dist^2 (n normalised, D = -n.origin: HalfSpace::init, :42-52)
//   Optimizer.cpp:3254-3267      kappa b(d) (the d <= 0 exit)                     HalfSpace.cpp:121-143  g += kappa b'(d) 2 dist n
//   HalfSpace.cpp:169-213        H += kappa param n n^T iff param = 4 b'' d + 2 b' > 0 (the exact PSD projection of a rank-one block)
//   HalfSpace.cpp:242-269        step bound -dist / (n.p) * slackness over the non-Dirichlet SVI vertices moving towards the plane
//   CollisionObject.h:386-401    isIntersected: d <= 0 over every codimension-3, non-Dirichlet vertex (only dist == 0 or an underflow of dist^2)
//   Optimizer.cpp:1555-1572      lagged lambda = -kappa 2 sqrt(d) b'(d) for planes with friction > 0
//   HalfSpace.cpp:272-380        friction: u = tangential part of (x - x_prev) - velocitydt, quadratic smoothing below eps
//
// Data: plane k holds kPlaneStride doubles [n0 n1 n2 D v0 v1 v2 mu] in device memory (ipcgpu_set_halfspaces), so a scripted motion between
// time steps needs no new capture.  Entries are (plane, vertex) pairs; the active set is a stream compaction of the flags of the flattened
// (plane, SVI index) range, i.e. plane-major and in SVI order inside a plane: the reference's order of activeSet[coI] over coI.  Every
// Hessian contribution is a 3x3 block on the diagonal of the vertex's rows, whose upper part starts each row (the upper-triangular CSR keeps
// the diagonal block of every vertex): no column search.
#include "pair_common.cuh"
#include "kernels.h"
#include <cub/cub.cuh>
#include <algorithm>

namespace ipcgpu {

namespace {

DEV double plane_dist(const double* __restrict__ pl, const double* __restrict__ V, int nV, int v)
{
    return ((pl[0] * V[v] + pl[1] * V[(size_t)nV + v]) + pl[2] * V[(size_t)2 * nV + v]) + pl[3];
}
DEV bool codim3(const int* vCoDim, int v) { return !vCoDim || vCoDim[v] == 3; }
DEV bool is_dbc(const uint8_t* dbc, int v) { return dbc && dbc[v] != 0; }
DEV bool owned(const HalfSpaceArgs& p, int v) { return v >= p.row_lo && v < p.row_hi; }

// ---- active set: flag, scan, scatter ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_hs_flags(HalfSpaceArgs p, double dHat, int* __restrict__ flags)
{
    const int n = p.nP * p.nSV;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int pl = k / p.nSV, v = p.SVI[k - pl * p.nSV];
        int f = 0;
        if (!is_dbc(p.dbc, v) && codim3(p.vCoDim, v)) {
            const double dist = plane_dist(p.par + kPlaneStride * pl, p.V, p.nV, v);
            f = dist * dist < dHat;
        }
        flags[k] = f;
    }
}
// pstart[q] = first entry of plane q in the active list (pstart[nP] = its size)
__global__ void __launch_bounds__(256) k_hs_scatter(HalfSpaceArgs p, const int* __restrict__ flags, const int* __restrict__ offs, int2* __restrict__ act,
    int* __restrict__ n_act, int* __restrict__ pstart, IterState* __restrict__ st)
{
    const int n = p.nP * p.nSV;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int pl = k / p.nSV, sv = k - pl * p.nSV;
        if (flags[k]) act[offs[k]] = make_int2(pl, p.SVI[sv]);
        if (sv == 0) pstart[pl] = offs[k];
        if (k == n - 1) {
            const int total = offs[k] + flags[k];
            pstart[p.nP] = total;
            *n_act = total;
            st->hs_n_active = total;
        }
    }
}

// ---- barrier terms over the active set ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_hs_energy(HalfSpaceArgs p, double dHat, double* __restrict__ partials, int* __restrict__ bad)
{
    const int n = *p.n_act;
    double val = 0.0;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.act[c];
        if (!owned(p, e.y)) continue;
        const double dist = plane_dist(p.par + kPlaneStride * e.x, p.V, p.nV, e.y), d = dist * dist;
        if (d <= 0.0) { atomicExch(bad, 1); continue; }
        double b, db, d2b;
        barrier_all(d, dHat, b, db, d2b);
        val += b;
    }
    cta_sum(&val, partials + blockIdx.x);
}

// reproducible mode (kStage): entry c of plane q at vertex v leaves its vector (3 doubles) or the upper part of its block (6) in rep_stage[c]
// and marks itself in rep_mask[v] / rep_pos; k_hs_repro_add then adds the entries of every vertex in plane order
template <int kWidth>
DEV void hs_stage(const HalfSpaceArgs& p, int c, int2 e, const double* val)
{
    for (int i = 0; i < kWidth; ++i) p.rep_stage[(size_t)kWidth * c + i] = val[i];
    p.rep_pos[kMaxPlanes * (size_t)e.y + e.x] = c;
    atomicOr(p.rep_mask + e.y, 1 << e.x);
}

// kappa_dev != nullptr (the barrier kernels below): kappa is the device-resident one
template <bool kStage>
__global__ void __launch_bounds__(128) k_hs_gradient(HalfSpaceArgs p, double dHat, double kappa, const double* __restrict__ kappa_dev, double* __restrict__ g)
{
    if (kappa_dev) kappa = *kappa_dev;
    const int n = *p.n_act;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.act[c];
        if (!owned(p, e.y)) continue;
        const double* pl = p.par + kPlaneStride * e.x;
        const double dist = plane_dist(pl, p.V, p.nV, e.y), d = dist * dist;
        double b, db, d2b;
        barrier_all(d, dHat, b, db, d2b);
        const double s = kappa * db * 2.0 * dist; // coef * input[cI] * 2.0 * dist (HalfSpace.cpp:138)
        if (kStage) {
            const double val[3] = { s * pl[0], s * pl[1], s * pl[2] };
            hs_stage<3>(p, c, e, val);
        }
        else
            for (int r = 0; r < 3; ++r) atomicAdd(g + 3 * (size_t)e.y + r, s * pl[r]);
    }
}

// upper part of a symmetric 3x3 block M (row-major) onto the diagonal block of vertex v: row 3v+r starts with column 3v+r
template <bool kStage>
DEV void add_diag_block(const HalfSpaceArgs& p, int c, int2 e, const double* M, double* a)
{
    if (kStage) {
        const double val[6] = { M[0], M[1], M[2], M[4], M[5], M[8] };
        hs_stage<6>(p, c, e, val);
    }
    else
        for (int r = 0; r < 3; ++r) {
            const int o = p.ia[3 * e.y + r] - p.base;
            for (int q = r; q < 3; ++q) atomicAdd(a + o + (q - r), M[3 * r + q]);
        }
}

// the entry of the lowest plane of its vertex adds the staged entries of that vertex in plane order, once, and clears the vertex's mask.
// kWidth 3: into g[v]; 6: into the upper part of v's diagonal block of a
template <int kWidth>
__global__ void __launch_bounds__(128) k_hs_repro_add(HalfSpaceArgs p, const int2* __restrict__ list, const int* __restrict__ n_ptr, double* __restrict__ out)
{
    const int n = *n_ptr;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = list[c];
        const int m = p.rep_mask[e.y];
        if (m == 0 || __ffs(m) - 1 != e.x) continue;
        double sum[kWidth];
        for (int i = 0; i < kWidth; ++i) sum[i] = 0.0;
        for (int q = 0; q < kMaxPlanes; ++q) {
            if (!((m >> q) & 1)) continue;
            const double* val = p.rep_stage + (size_t)kWidth * p.rep_pos[kMaxPlanes * (size_t)e.y + q];
            for (int i = 0; i < kWidth; ++i) sum[i] += val[i];
        }
        p.rep_mask[e.y] = 0;
        if (kWidth == 3)
            for (int r = 0; r < 3; ++r) out[3 * (size_t)e.y + r] += sum[r];
        else
            for (int r = 0, i = 0; r < 3; ++r) {
                const int o = p.ia[3 * e.y + r] - p.base;
                for (int q = r; q < 3; ++q, ++i) out[o + (q - r)] += sum[i];
            }
    }
}

template <bool kStage>
__global__ void __launch_bounds__(128) k_hs_hessian(HalfSpaceArgs p, double dHat, double kappa, const double* __restrict__ kappa_dev, int projectDBC,
    double* __restrict__ a)
{
    if (kappa_dev) kappa = *kappa_dev;
    const int n = *p.n_act;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.act[c];
        if (!owned(p, e.y) || proj_dbc(p.dbc, e.y, projectDBC)) continue;
        const double* pl = p.par + kPlaneStride * e.x;
        const double dist = plane_dist(pl, p.V, p.nV, e.y), d = dist * dist;
        double b, db, d2b;
        barrier_all(d, dHat, b, db, d2b);
        const double param = 4.0 * d2b * d + 2.0 * db;
        if (!(param > 0.0)) continue;
        const double s = kappa * param;
        double M[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) M[3 * i + j] = s * (pl[i] * pl[j]);
        add_diag_block<kStage>(p, c, e, M, a);
    }
}

// ---- step bound (replicated: every rank walks all of SVI) --------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_hs_step(HalfSpaceArgs p, const double* __restrict__ dir, double slack, unsigned long long* __restrict__ step_ord)
{
    const int n = p.nP * p.nSV;
    double m = 1.0; // maxStepSizes[svI] = 1.0 (HalfSpace.cpp:255)
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int pl = k / p.nSV, v = p.SVI[k - pl * p.nSV];
        if (is_dbc(p.dbc, v)) continue;
        const double* q = p.par + kPlaneStride * pl;
        const double c = (q[0] * dir[3 * (size_t)v] + q[1] * dir[3 * (size_t)v + 1]) + q[2] * dir[3 * (size_t)v + 2];
        if (c < 0.0) {
            const double dist = plane_dist(q, p.V, p.nV, v);
            m = fmin(m, -dist / c * slack);
        }
    }
    m = warp_min(m);
    if ((threadIdx.x & 31) == 0) atomicMin(step_ord, dbl_to_ord(m > 0.0 ? m : 0.0)); // a bound <= 0 is stored as 0 (no negative ord image)
}
__global__ void k_hs_step_stage(IterState* st)
{
    if (threadIdx.x != 0) return;
    const double a = ord_to_dbl(st->step_ord);
    st->hs_alpha = a;
    if (a == 0.0) st->hs_zero_step = 1;
}

// ---- crossing check: every vertex (not only SVI) -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_hs_crossings(HalfSpaceArgs p, int* __restrict__ count)
{
    int hits = 0;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x) {
        if (!owned(p, v) || is_dbc(p.dbc, v) || !codim3(p.vCoDim, v)) continue;
        for (int pl = 0; pl < p.nP; ++pl) {
            const double dist = plane_dist(p.par + kPlaneStride * pl, p.V, p.nV, v);
            hits += dist * dist <= 0.0; // the reference tests the SQUARED distance: a vertex behind the plane is not caught
        }
    }
    hits = warp_sum(hits);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(count, hits);
}

// ---- friction ------------------------------------------------------------------------------------------------------------
// lag: the active entries of the planes with friction > 0, in order; lambda = -kappa 2 sqrt(d) b'(d)
__global__ void __launch_bounds__(128) k_hs_lag(HalfSpaceArgs p, double dHat, double kappa, const double* __restrict__ kappa_dev, const int* __restrict__ pstart,
    int2* __restrict__ lag, double* __restrict__ lam, int* __restrict__ n_lag, int* __restrict__ bad, IterState* __restrict__ st)
{
    if (kappa_dev) kappa = *kappa_dev;
    const int n = pstart[p.nP];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int m = 0;
        for (int q = 0; q < p.nP; ++q)
            if (p.par[kPlaneStride * q + 7] > 0.0) m += pstart[q + 1] - pstart[q];
        *n_lag = m;
        st->hs_n_lagged = m;
    }
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.act[c];
        if (!(p.par[kPlaneStride * e.x + 7] > 0.0)) continue;
        int skip = 0; // entries of the frictionless planes before this one
        for (int q = 0; q < e.x; ++q)
            if (!(p.par[kPlaneStride * q + 7] > 0.0)) skip += pstart[q + 1] - pstart[q];
        const double dist = plane_dist(p.par + kPlaneStride * e.x, p.V, p.nV, e.y), d = dist * dist;
        if (!(d > 0.0)) atomicExch(bad, 1);
        double b, db, d2b;
        barrier_all(d, dHat, b, db, d2b);
        double l = db;
        l *= -kappa * 2.0 * sqrt(d);
        lag[c - skip] = e;
        lam[c - skip] = l;
    }
}

struct Slip {
    double u[3];   // VProj
    double mag2;   // |VProj|^2
};
DEV Slip slip(const HalfSpaceArgs& p, const double* pl, int v)
{
    double vd[3];
    for (int r = 0; r < 3; ++r) vd[r] = (p.V[(size_t)r * p.nV + v] - p.Vt[(size_t)r * p.nV + v]) - pl[4 + r];
    const double un = (vd[0] * pl[0] + vd[1] * pl[1]) + vd[2] * pl[2];
    Slip s;
    for (int r = 0; r < 3; ++r) s.u[r] = vd[r] - un * pl[r];
    s.mag2 = (s.u[0] * s.u[0] + s.u[1] * s.u[1]) + s.u[2] * s.u[2];
    return s;
}

__global__ void __launch_bounds__(256) k_hs_fric_energy(HalfSpaceArgs p, double eps2, double* __restrict__ partials)
{
    const int n = *p.n_lag;
    const double eps = sqrt(eps2);
    double val = 0.0;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.lag[c];
        if (!owned(p, e.y)) continue;
        const double* pl = p.par + kPlaneStride * e.x;
        const Slip s = slip(p, pl, e.y);
        const double m = pl[7] * p.lam[c];
        val += (s.mag2 > eps2) ? m * (sqrt(s.mag2) - eps * 0.5) : m * s.mag2 / eps * 0.5; // HalfSpace.cpp:289-294
    }
    cta_sum(&val, partials + blockIdx.x);
}

template <bool kStage>
__global__ void __launch_bounds__(128) k_hs_fric_gradient(HalfSpaceArgs p, double eps2, double* __restrict__ g)
{
    const int n = *p.n_lag;
    const double eps = sqrt(eps2);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.lag[c];
        if (!owned(p, e.y)) continue;
        const double* pl = p.par + kPlaneStride * e.x;
        const Slip s = slip(p, pl, e.y);
        const double m = pl[7] * p.lam[c];
        const double f = (s.mag2 > eps2) ? m / sqrt(s.mag2) : m / eps; // HalfSpace.cpp:317-322
        if (kStage) {
            const double val[3] = { f * s.u[0], f * s.u[1], f * s.u[2] };
            hs_stage<3>(p, c, e, val);
        }
        else
            for (int r = 0; r < 3; ++r) atomicAdd(g + 3 * (size_t)e.y + r, f * s.u[r]);
    }
}

template <bool kStage>
__global__ void __launch_bounds__(128) k_hs_fric_hessian(HalfSpaceArgs p, double eps2, int projectDBC, double* __restrict__ a)
{
    const int n = *p.n_lag;
    const double eps = sqrt(eps2);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const int2 e = p.lag[c];
        if (!owned(p, e.y) || proj_dbc(p.dbc, e.y, projectDBC)) continue;
        const double* pl = p.par + kPlaneStride * e.x;
        const Slip s = slip(p, pl, e.y);
        const double m = pl[7] * p.lam[c];
        double M[9];
        if (s.mag2 > eps2) {
            // makePD(-m/|u|^3 u u^T + m/|u| (I - n n^T)) (HalfSpace.cpp:351-357).  u lies in the tangent plane, so the matrix is m/|u| w w^T with
            // w = n x u/|u|: spectrum {0, 0, m/|u|}, and this closed form is its projection (the reference's eigen-solve differs at rounding level)
            const double mag = sqrt(s.mag2);
            const double uh[3] = { s.u[0] / mag, s.u[1] / mag, s.u[2] / mag };
            const double w[3] = { pl[1] * uh[2] - pl[2] * uh[1], pl[2] * uh[0] - pl[0] * uh[2], pl[0] * uh[1] - pl[1] * uh[0] };
            const double k = fmax(m / mag, 0.0);
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) M[3 * i + j] = k * (w[i] * w[j]);
        }
        else { // (I - n n^T) m / eps (:360)
            const double k = m / eps;
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) M[3 * i + j] = ((i == j ? 1.0 : 0.0) - pl[i] * pl[j]) * k;
        }
        add_diag_block<kStage>(p, c, e, M, a);
    }
}

constexpr int kHsEnergyBlocks = kSMs;
int grid_for(long long n, int threads) { return (int)std::max(1LL, std::min((n + threads - 1) / threads, (long long)kSMs * 8)); }

} // namespace

int halfspace_energy_blocks() { return kHsEnergyBlocks; }

size_t halfspace_scan_bytes(int n)
{
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int*)nullptr, (int*)nullptr, n);
    return bytes;
}

cudaError_t halfspace_active_set(const HalfSpaceArgs& p, double dHat, int* flags, int* offs, void* scan_tmp, size_t scan_bytes, int2* act, int* n_act,
    int* pstart, IterState* st_dev, cudaStream_t st)
{
    const int n = p.nP * p.nSV;
    k_hs_flags<<<grid_for(n, 256), 256, 0, st>>>(p, dHat, flags);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, flags, offs, n, st);
    if (e != cudaSuccess) return e;
    k_hs_scatter<<<grid_for(n, 256), 256, 0, st>>>(p, flags, offs, act, n_act, pstart, st_dev);
    return cudaGetLastError();
}
void halfspace_energy(const HalfSpaceArgs& p, double dHat, double* partials, int* bad, cudaStream_t st)
{
    k_hs_energy<<<kHsEnergyBlocks, 256, 0, st>>>(p, dHat, partials, bad);
}
void halfspace_gradient(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, double* g, cudaStream_t st)
{
    if (p.rep_mask) {
        k_hs_gradient<true><<<kSMs, 128, 0, st>>>(p, dHat, kappa, kappa_dev, g);
        k_hs_repro_add<3><<<kSMs, 128, 0, st>>>(p, p.act, p.n_act, g);
    }
    else k_hs_gradient<false><<<kSMs, 128, 0, st>>>(p, dHat, kappa, kappa_dev, g);
}
void halfspace_hessian(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, int projectDBC, double* a, cudaStream_t st)
{
    if (p.rep_mask) {
        k_hs_hessian<true><<<kSMs, 128, 0, st>>>(p, dHat, kappa, kappa_dev, projectDBC, a);
        k_hs_repro_add<6><<<kSMs, 128, 0, st>>>(p, p.act, p.n_act, a);
    }
    else k_hs_hessian<false><<<kSMs, 128, 0, st>>>(p, dHat, kappa, kappa_dev, projectDBC, a);
}
void halfspace_step(const HalfSpaceArgs& p, const double* dir, double slack, IterState* st_dev, cudaStream_t st)
{
    k_hs_step<<<grid_for((long long)p.nP * p.nSV, 256), 256, 0, st>>>(p, dir, slack, &st_dev->step_ord);
    k_hs_step_stage<<<1, 32, 0, st>>>(st_dev);
}
void halfspace_crossings(const HalfSpaceArgs& p, IterState* st_dev, cudaStream_t st)
{
    zero_words(&st_dev->hs_crossings, 1, st);
    k_hs_crossings<<<grid_for(p.nV, 256), 256, 0, st>>>(p, &st_dev->hs_crossings);
}
void halfspace_lag(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, const int* pstart, int2* lag, double* lam, int* n_lag, int* bad,
    IterState* st_dev, cudaStream_t st)
{
    k_hs_lag<<<kSMs, 128, 0, st>>>(p, dHat, kappa, kappa_dev, pstart, lag, lam, n_lag, bad, st_dev);
}
void halfspace_friction_energy(const HalfSpaceArgs& p, double eps2, double* partials, cudaStream_t st)
{
    k_hs_fric_energy<<<kHsEnergyBlocks, 256, 0, st>>>(p, eps2, partials);
}
void halfspace_friction_gradient(const HalfSpaceArgs& p, double eps2, double* g, cudaStream_t st)
{
    if (p.rep_mask) {
        k_hs_fric_gradient<true><<<kSMs, 128, 0, st>>>(p, eps2, g);
        k_hs_repro_add<3><<<kSMs, 128, 0, st>>>(p, p.lag, p.n_lag, g);
    }
    else k_hs_fric_gradient<false><<<kSMs, 128, 0, st>>>(p, eps2, g);
}
void halfspace_friction_hessian(const HalfSpaceArgs& p, double eps2, int projectDBC, double* a, cudaStream_t st)
{
    if (p.rep_mask) {
        k_hs_fric_hessian<true><<<kSMs, 128, 0, st>>>(p, eps2, projectDBC, a);
        k_hs_repro_add<6><<<kSMs, 128, 0, st>>>(p, p.lag, p.n_lag, a);
    }
    else k_hs_fric_hessian<false><<<kSMs, 128, 0, st>>>(p, eps2, projectDBC, a);
}

} // namespace ipcgpu
