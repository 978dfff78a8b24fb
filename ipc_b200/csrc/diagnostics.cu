// diagnostics.cu -- the end-of-step diagnostics of the reference's IP time step on the device (sm_90a):
//
//   Optimizer.cpp:3746-3778   computeSystemEnergy                  system_energy: per component, sum vol psi over its tets, plus
//                                                                  sum m (|V - V_prev|^2 / dtSq / 2 - g.V) over its vertices; the momentum
//                                                                  sum p, p = m / dt (V - V_prev); the angular momentum sum V x p
//   Optimizer.cpp:1619-1691   the read-back after solveSub_IP     constraint_summary: count, min and max of the constraint values (planes,
//                                                                  then the self / obstacle active entries) and |fb|, with
//                                                                  fb = dual + d - sqrt(dual^2 + d^2), dual = -kappa g_b(d)
//   *** compiled with --fmad=false (NOFMA_FILES): every per-entry expression keeps the reference's evaluation order and rounds each product
//   and sum separately; the plane distances round as the half-space kernels (halfspace.cu, also built without contraction) evaluate them ***
//
// Summation order (no value atomics: the same state gives the same bits, eager or replayed):
//   - a segment (DiagSegment, kernels.h) is summed by one 256-thread CTA: thread t adds the entries begin + t, begin + t + 256, ... in that
//     order, then cta_sum (common.cuh) adds the threads in its fixed tree;
//   - a component adds its tet segments in table order starting from +0.0, then its vertex segments the same way, and sysE is the tet sum
//     plus the vertex sum; sysM and sysL add the vertex segments in table order;
//   - the summary adds fb^2 per CTA over a fixed grid-stride assignment, then the kDiagSummaryBlocks partials in the fixed order of one CTA.
// The minimum and maximum are taken on the order-preserving images of the (non-negative) squared distances: exact, in any order.
#include "common.cuh"
#include "contact.cuh"
#include "kernels.h"

namespace ipcgpu {

namespace {

constexpr int kThreads = 256;
static_assert(kDiagSummaryBlocks == 2 * kSMs, "one summary CTA pair per SM");

// one vertex's terms of computeSystemEnergy (:3764-3774) in the reference's Eigen evaluation order: (V.row - V_prev.row).squaredNorm() adds
// the squares left to right; gravity.dot(V.row) is the unrolled 3-term redux g0 x0 + (g1 x1 + g2 x2); p = (m / dt) (x - xp); Eigen's cross
DEV void vertex_terms(const SystemEnergyArgs& p, const TimeParams& q, int v, double* acc)
{
    double x[3], dx[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        x[d] = p.V[(size_t)d * p.nV + v];
        dx[d] = x[d] - p.Vprev[(size_t)d * p.nV + v];
    }
    const double m = p.mass[v];
    const double sq = (dx[0] * dx[0] + dx[1] * dx[1]) + dx[2] * dx[2];
    const double gx = q.gravity[0] * x[0] + (q.gravity[1] * x[1] + q.gravity[2] * x[2]);
    acc[0] += m * (sq / q.dtSq / 2.0 - gx);
    const double mdt = m / q.dt;
    const double pm[3] = { mdt * dx[0], mdt * dx[1], mdt * dx[2] };
#pragma unroll
    for (int d = 0; d < 3; ++d) acc[1 + d] += pm[d];
    acc[4] += x[1] * pm[2] - x[2] * pm[1];
    acc[5] += x[2] * pm[0] - x[0] * pm[2];
    acc[6] += x[0] * pm[1] - x[1] * pm[0];
}

__global__ void __launch_bounds__(kThreads) k_system_energy_segments(SystemEnergyArgs p)
{
    const DiagSegment s = p.seg[blockIdx.x];
    double acc[7] = { 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 };
    if (s.kind == kSegTets) {
        for (int t = s.begin + threadIdx.x; t < s.end; t += kThreads) acc[0] += p.e_per_tet[t];
    }
    else {
        const TimeParams q = *p.tp;
        for (int v = s.begin + threadIdx.x; v < s.end; v += kThreads) vertex_terms(p, q, v, acc);
    }
    cta_sum<7>(acc, p.part + 7 * (size_t)blockIdx.x);
}

// one thread per component: its segments in table order
__global__ void __launch_bounds__(128) k_system_energy_components(SystemEnergyArgs p)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= p.n_comp) return;
    double e_tets = 0.0, e_verts = 0.0, mo[3] = { 0.0, 0.0, 0.0 }, am[3] = { 0.0, 0.0, 0.0 };
    for (int s = p.comp_seg[c]; s < p.comp_seg[c + 1]; ++s) {
        const double* q = p.part + 7 * (size_t)s;
        if (p.seg[s].kind == kSegTets) {
            e_tets += q[0];
            continue;
        }
        e_verts += q[0];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            mo[d] += q[1 + d];
            am[d] += q[4 + d];
        }
    }
    p.out[c] = e_tets + e_verts;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        p.out[p.n_comp + 3 * (size_t)c + d] = mo[d];
        p.out[4 * (size_t)p.n_comp + 3 * (size_t)c + d] = am[d];
    }
}

DEV unsigned long long warp_min_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
DEV unsigned long long warp_max_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// min and max over a 256-thread CTA: the results in thread 0's lo / hi
DEV void cta_min_max(unsigned long long& lo, unsigned long long& hi)
{
    __shared__ unsigned long long sm[2][8];
    lo = warp_min_u64(lo);
    hi = warp_max_u64(hi);
    if ((threadIdx.x & 31) == 0) {
        sm[0][threadIdx.x >> 5] = lo;
        sm[1][threadIdx.x >> 5] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < 8; ++w) {
            lo = min(lo, sm[0][w]);
            hi = max(hi, sm[1][w]);
        }
}

// entry i: the planes' active entries first (d as k_hs_energy evaluates it), then the self / obstacle active entries
__global__ void __launch_bounds__(kThreads) k_summary_entries(SummaryArgs p)
{
    const int n_pl = p.n_act ? *p.n_act : 0, n = n_pl + *p.nC;
    const double kappa = p.kappa_dev ? *p.kappa_dev : p.kappa;
    double fb2 = 0.0;
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        double d;
        if (i < n_pl) {
            const int2 e = p.act[i];
            const double* pl = p.par + kPlaneStride * e.x;
            const double dist = ((pl[0] * p.V[e.y] + pl[1] * p.V[(size_t)p.nV + e.y]) + pl[2] * p.V[(size_t)2 * p.nV + e.y]) + pl[3];
            d = dist * dist;
        }
        else d = p.val[i - n_pl];
        double b, db, d2b;
        barrier_all(d, p.dHat, b, db, d2b); // compute_g_b (:1685)
        const double dual = db * -kappa;
        const double fb = dual + d - sqrt(dual * dual + d * d); // :1688-1691
        fb2 += fb * fb;
        lo = min(lo, dbl_to_ord(d));
        hi = max(hi, dbl_to_ord(d));
    }
    cta_sum(&fb2, p.part + blockIdx.x);
    cta_min_max(lo, hi);
    if (threadIdx.x == 0) {
        p.part_ord[2 * blockIdx.x] = lo;
        p.part_ord[2 * blockIdx.x + 1] = hi;
    }
}

// out = { n, d_min, d_max, |fb| }; n == 0 leaves the other three 0 ("no collision in this time step", :1749-1752)
__global__ void __launch_bounds__(kThreads) k_summary_finish(SummaryArgs p)
{
    __shared__ double tot;
    const int n = (p.n_act ? *p.n_act : 0) + *p.nC;
    double s = 0.0;
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int b = threadIdx.x; b < kDiagSummaryBlocks; b += kThreads) {
        s += p.part[b];
        lo = min(lo, p.part_ord[2 * b]);
        hi = max(hi, p.part_ord[2 * b + 1]);
    }
    cta_sum(&s, &tot);
    cta_min_max(lo, hi);
    __syncthreads();
    if (threadIdx.x == 0) {
        p.out[0] = (double)n;
        p.out[1] = n ? ord_to_dbl(lo) : 0.0;
        p.out[2] = n ? ord_to_dbl(hi) : 0.0;
        p.out[3] = n ? sqrt(tot) : 0.0;
    }
}

} // namespace

void system_energy(const SystemEnergyArgs& p, cudaStream_t st)
{
    if (p.n_seg > 0) k_system_energy_segments<<<p.n_seg, kThreads, 0, st>>>(p);
    k_system_energy_components<<<(p.n_comp + 127) / 128, 128, 0, st>>>(p);
}

void constraint_summary(const SummaryArgs& p, cudaStream_t st)
{
    k_summary_entries<<<kDiagSummaryBlocks, kThreads, 0, st>>>(p);
    k_summary_finish<<<1, kThreads, 0, st>>>(p);
}

} // namespace ipcgpu
