// barrier.cu -- per-pair barrier energy / gradient / PSD-projected Hessian over the active constraint set (sm_90a).
//
// Reference being replaced: SelfCollisionHandler<3>::evaluateConstraints (:64-81), leftMultiplyConstraintJacobianT
// (:84-148, serial "TODO: parallelize"), augmentIPHessian (:418-561, serial CSR add), augmentParaEEGradient/Hessian
// (:2990-3201) and the composition in Optimizer.cpp:3290-3353, 3492-3502, 3693-3695.
//
//  * one thread per pair; the squared distance, its gradient and Hessian come from contact.cuh;
//  * makePD on the 6/9/12-square block (IglUtils.hpp:119-137) is a cyclic Jacobi eigen-solver whose three
//    12x12 work matrices live in shared memory, element-major / lane-minor (element e of lane t at e*32+t), so every
//    access of a warp is conflict-free even though p,q are data dependent per sweep position only;
//  * gradients and CSR values are accumulated with FP64 red.global.add (pair counts are orders of magnitude below the
//    tet count; the elastic path stays deterministic, the barrier scatter is order-free to ~1 ulp of the sum).
#include "repro.cuh"
#include <algorithm>

namespace ipcgpu {

// distance + gradient (12) [+ Hessian through puth]
template <typename PutH>
__device__ inline double pair_derivs(const PairStencil& s, const V3* x, double* g, bool want_h, PutH puth)
{
    if (s.kind == 3) {
        V3 r = 2.0 * (x[0] - x[1]);
        g[0] = r.x; g[1] = r.y; g[2] = r.z; g[3] = -r.x; g[4] = -r.y; g[5] = -r.z;
        if (want_h)
            for (int i = 0; i < 6; ++i)
                for (int j = 0; j < 6; ++j) puth(i, j, (i == j) ? 2.0 : ((i % 3 == j % 3) ? -2.0 : 0.0));
        return norm2(x[0] - x[1]);
    }
    Diff D;
    if (s.kind == 0) plane_dist(x[0] - x[1], x[2] - x[1], x[3] - x[1], D);
    else if (s.kind == 1) plane_dist(x[2] - x[0], x[1] - x[0], x[3] - x[2], D);
    else line_dist(x[0] - x[1], x[2] - x[1], D);
    diff_to_vertices(D, s.kind, s.nv, true, want_h, [&](int i, double v) { g[i] = v; }, puth);
    return D.val;
}

// mollifier e(x) on the 4-vertex edge stencil: value, gradient (12), Hessian via puth   [:2851-2912]
template <typename PutH>
__device__ inline double mollifier(const V3* ex, double eps_x, double* eg, bool want_h, PutH puth)
{
    Diff C;
    cross_norm(ex[1] - ex[0], ex[3] - ex[2], C);
    if (!(C.val < eps_x)) {
        for (int i = 0; i < 12; ++i) eg[i] = 0.0;
        if (want_h)
            for (int i = 0; i < 12; ++i)
                for (int j = 0; j < 12; ++j) puth(i, j, 0.0);
        return 1.0;
    }
    const double inv = 1.0 / eps_x;
    const double qg = 2.0 * inv * (-inv * C.val + 1.0);
    const double qH = -2.0 / (eps_x * eps_x);
    double cg[12];
    diff_to_vertices(C, 3, 4, true, false, [&](int i, double v) { cg[i] = v; }, [](int, int, double) {});
    for (int i = 0; i < 12; ++i) eg[i] = cg[i] * qg;
    if (want_h)
        diff_to_vertices(C, 3, 4, false, true, [](int, double) {}, [&](int i, int j, double v) { puth(i, j, v * qg + (qH * cg[i]) * cg[j]); });
    const double r = C.val / eps_x;
    return (-r + 2.0) * r;
}

// The list sizes live on the device (the constraint set is built there and nothing is read back inside an iteration), so every
// kernel below is a grid-stride loop over [0, n) with n taken from device memory.  Item i of a rank's share: the first (ce - cb)
// items are entries [cb, ce) of the active list, the rest entries [pb, pe) of the mollified list.
struct ListRange {
    int cb, ce, pb, pe;
};
DEV ListRange list_range(const BarrierArgs& p, bool whole)
{
    const long long nC = *p.nC, nP = *p.nP;
    ListRange r;
    if (p.share && !whole) {
        r.cb = (int)(nC * p.rank / p.nranks); r.ce = (int)(nC * (p.rank + 1) / p.nranks);
        r.pb = (int)(nP * p.rank / p.nranks); r.pe = (int)(nP * (p.rank + 1) / p.nranks);
    }
    else { r.cb = 0; r.ce = (int)nC; r.pb = 0; r.pe = (int)nP; }
    return r;
}

// -----------------------------------------------------------------------------------------------------------
// energy: kappa * sum( mult*b(d) ) + kappa * sum( e*b(d) )      (Optimizer.cpp:3290-3353)
// -----------------------------------------------------------------------------------------------------------
constexpr int kBarrierEnergyBlocks = kSMs * 2;
__global__ void __launch_bounds__(256) k_barrier_energy(BarrierArgs p, double* __restrict__ partials, int* __restrict__ bad)
{
    const ListRange lr = list_range(p, false);
    const int nA = lr.ce - lr.cb, n = nA + (lr.pe - lr.pb);
    double val = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const bool is_para = i >= nA;
        const int c = is_para ? lr.pb + (i - nA) : lr.cb + i;
        const int4 mm = is_para ? p.para[c] : p.cs[c];
        const PairStencil s = decode(mm);
        V3 x[4];
        load_stencil(s, p.V, p.nV, x);
        const double d = pair_distance(s, x);
        if (!(d > 0.0)) atomicExch(bad, 1);
        else {
            double b, db, d2b;
            barrier_all(d, p.dHat, b, db, d2b);
            if (!is_para) val += (mm.x < 0 && mm.w < -1) ? b * (double)(-mm.w) : b;
            else {
                int ev[4];
                V3 ex[4];
                const double eps_x = load_para_edges(mm, p.para_e[c], p.SE, p.V, p.Vrest, p.nV, ev, ex);
                double eg[12];
                const double e = mollifier(ex, eps_x, eg, false, [](int, int, double) {});
                val += b * e;
            }
        }
    }
    cta_sum(&val, partials + blockIdx.x);
}

// -----------------------------------------------------------------------------------------------------------
// gradient: g += kappa*mult*b'(d) grad d   (+ para-EE: kappa*b*grad e + kappa*e*b' grad d)
// -----------------------------------------------------------------------------------------------------------
// kDevKappa: kappa is the device-resident one (BarrierArgs::kappa_dev).  A template parameter rather than a run-time test, and read where
// p.kappa was, so that the host-kappa instantiations compile to the same code (registers, spills) as without the device kappa
template <bool kDevKappa>
DEV double barrier_kappa(const BarrierArgs& p) { return kDevKappa ? *p.kappa_dev : p.kappa; }

// kStage: the contributions go to the staging array under their gradient keys (repro.cuh).  kParaOnly: the mollified list alone, the
// reference's augmentParaEEGradient (:2990-3045)
template <bool kDevKappa, bool kStage, bool kParaOnly = false>
__global__ void __launch_bounds__(128) k_barrier_gradient(BarrierArgs p, double* __restrict__ g)
{
    const ListRange lr = list_range(p, false);
    const int nA = kParaOnly ? 0 : lr.ce - lr.cb, n = nA + (lr.pe - lr.pb);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const bool is_para = i >= nA;
    const int c = is_para ? lr.pb + (i - nA) : lr.cb + i;
    const int4 mm = is_para ? p.para[c] : p.cs[c];
    const PairStencil s = decode(mm);
    V3 x[4];
    load_stencil(s, p.V, p.nV, x);
    double gd[12];
    const double d = pair_derivs(s, x, gd, false, [](int, int, double) {});
    double b, db, d2b;
    barrier_all(d, p.dHat, b, db, d2b);
    double w;
    if (!is_para) w = barrier_kappa<kDevKappa>(p) * s.mult * db;
    else {
        int ev[4];
        V3 ex[4];
        const double eps_x = load_para_edges(mm, p.para_e[c], p.SE, p.V, p.Vrest, p.nV, ev, ex);
        double eg[12];
        const double e = mollifier(ex, eps_x, eg, false, [](int, int, double) {});
        for (int k = 0; k < 4; ++k)
            for (int q = 0; q < 3; ++q) put_g<kStage>(g, ev[k], gkey_para_edge(p.rep.cap, c, k), q, barrier_kappa<kDevKappa>(p) * b * eg[3 * k + q]);
        w = barrier_kappa<kDevKappa>(p) * e * db; // slot 3 is -1 (or a vertex id): multiplicity 1
    }
    for (int k = 0; k < s.nv; ++k)
        for (int q = 0; q < 3; ++q) put_g<kStage>(g, s.v[k], is_para ? gkey_para_dist(p.rep.cap, c, k) : gkey_active(c, k), q, w * gd[3 * k + q]);
    }
}

// -----------------------------------------------------------------------------------------------------------
// the reference's own two-step form of the gradient (Optimizer.cpp:3492-3499): evaluateConstraints (:64-81) hands the squared
// distances of the active set to the host, which maps them through b'(d) and passes them back to leftMultiplyConstraintJacobianT
// (:84-148): out += coef * mult_c * input_c * grad d_c.  Active set only (the mollified pairs go through augmentParaEEGradient).
// -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_evaluate_constraints(BarrierArgs p, double* __restrict__ val)
{
    const int n = *p.nC;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) val[c] = pair_distance(p.cs[c], p.V, p.nV);
}
template <bool kStage>
__global__ void __launch_bounds__(128) k_constraint_jacobian_t(BarrierArgs p, const double* __restrict__ input, double coef, double* __restrict__ g)
{
    const ListRange lr = list_range(p, false);
    for (int c = lr.cb + blockIdx.x * blockDim.x + threadIdx.x; c < lr.ce; c += gridDim.x * blockDim.x) {
        const PairStencil s = decode(p.cs[c]);
        V3 x[4];
        load_stencil(s, p.V, p.nV, x);
        double gd[12];
        pair_derivs(s, x, gd, false, [](int, int, double) {});
        const double w = coef * s.mult * input[c];
        for (int k = 0; k < s.nv; ++k)
            for (int q = 0; q < 3; ++q) put_g<kStage>(g, s.v[k], gkey_active(c, k), q, w * gd[3 * k + q]);
    }
}

// -----------------------------------------------------------------------------------------------------------
// Hessian: makePD( kappa*mult*(b'' g g^T + b' H_d) ) scattered into the CSR (upper triangle)
//   pass 1 (thread per pair)  : unprojected block, zero-padded to 12x12, to global memory (144 contiguous doubles per pair)
//   pass 2 (warp per pair)    : parallel-order Jacobi eigen-solver on the 12x12 (6 disjoint rotations per round, 11 rounds
//                               per sweep, the round-robin tournament schedule), clamp, rebuild, red.add into the CSR
// -----------------------------------------------------------------------------------------------------------
DEV bool owns_row(const BarrierArgs& p, int v) { return v >= p.row_lo && v < p.row_hi; }

// kFixedSlot (reproducible mode, one rank): the pair of list position c (active, then mollified) keeps slot c, so that the slot order is the
// list order; *n_owned = the number of pairs
template <bool kDevKappa, bool kFixedSlot>
__global__ void __launch_bounds__(64) k_barrier_hessian_build(BarrierArgs p, double* __restrict__ Hraw, int* __restrict__ rows_out, int* __restrict__ n_owned,
    int capacity, int* __restrict__ flags)
{
    const int nC = *p.nC, nTot = nC + *p.nP;
    if (kFixedSlot && blockIdx.x == 0 && threadIdx.x == 0) *n_owned = min(nTot, capacity);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < nTot; c += gridDim.x * blockDim.x) {
    // the matrix is assembled in thread-local memory (interleaved across the warp by the hardware: every access is one coalesced
    // transaction) and shipped to its pair-major slot once at the end; read-modify-write straight on the 1152-byte-strided slots
    // cost 32 sectors per warp access
    const bool is_para = c >= nC;
    const int4 mm = is_para ? p.para[c - nC] : p.cs[c];
    const PairStencil s = decode(mm);
    int rows[4];
    {   // row ownership (multi-rank): this rank assembles the pair only if it owns a row of its stencil.  The rows are hessian_rows',
        // written out: the call raises this kernel's spill loads
        bool mine = false;
        if (!is_para) {
            for (int k = 0; k < 4; ++k) rows[k] = (k < s.nv) ? s.v[k] : -1;
        }
        else para_edge_stencil(mm, p.para_e[c - nC], p.SE, rows);
        for (int k = 0; k < 4; ++k) mine = mine || (rows[k] >= 0 && owns_row(p, rows[k]));
        if (!mine) continue;
    }
    double H[144];
#define HE(i, j) H[(i) * 12 + (j)]
    for (int i = 0; i < 144; ++i) H[i] = 0.0;
    V3 x[4];
    load_stencil(s, p.V, p.nV, x);
    if (!is_para) {
        const int n = 3 * s.nv;
        double gd[12];
        const double d = pair_derivs(s, x, gd, true, [&](int i, int j, double v) { HE(i, j) = v; });
        double b, db, d2b;
        barrier_all(d, p.dHat, b, db, d2b);
        const double coef = barrier_kappa<kDevKappa>(p) * s.mult;
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) HE(i, j) = ((coef * d2b) * gd[i]) * gd[j] + (coef * db) * HE(i, j);
    }
    else {
        // mollified pair on the two-edge stencil (:3049-3173)
        int ev[4];
        V3 ex[4];
        const double eps_x = load_para_edges(mm, p.para_e[c - nC], p.SE, p.V, p.Vrest, p.nV, ev, ex);
        double gd0[12], gd[12], eg[12];
        double AE[144], VE[144]; // distance Hessian on its own stencil / embedded in the edge stencil
        const double d = pair_derivs(s, x, gd0, true, [&](int i, int j, double v) { AE[i * 12 + j] = v; });
        int map[4];
        for (int k = 0; k < s.nv; ++k) {
            map[k] = -1;
            for (int i = 0; i < 4; ++i)
                if (ev[i] == s.v[k]) map[k] = i;
        }
        for (int i = 0; i < 12; ++i) gd[i] = 0.0;
        for (int i = 0; i < 144; ++i) VE[i] = 0.0;
        for (int k = 0; k < s.nv; ++k) {
            if (map[k] < 0) continue;
            for (int i = 0; i < 3; ++i) gd[3 * map[k] + i] = gd0[3 * k + i];
            for (int l = 0; l < s.nv; ++l) {
                if (map[l] < 0) continue;
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j) VE[(3 * map[k] + i) * 12 + 3 * map[l] + j] = AE[(3 * k + i) * 12 + 3 * l + j];
            }
        }
        double b, db, d2b;
        barrier_all(d, p.dHat, b, db, d2b);
        const double e = mollifier(ex, eps_x, eg, true, [&](int i, int j, double v) { HE(i, j) = v; });
        const double k = barrier_kappa<kDevKappa>(p);
        for (int i = 0; i < 12; ++i)
            for (int j = 0; j < 12; ++j)
                HE(i, j) = ((k * db) * gd[i]) * eg[j] + ((k * db) * gd[j]) * eg[i] + (k * b) * HE(i, j) + ((k * e * d2b) * gd[i]) * gd[j] + (k * e * db) * VE[i * 12 + j];
    }
    // compacted output slot (one atomic per warp iteration)
    int slot = c;
    if (!kFixedSlot) {
        const unsigned m = __activemask();
        const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(n_owned, __popc(m));
        base = __shfl_sync(m, base, leader);
        slot = base + __popc(m & ((1u << lane) - 1u));
    }
    if (slot >= capacity) {
        atomicExch(flags + FLAG_SET_CAPACITY, 1);
        continue;
    }
    for (int q = 0; q < 4; ++q) rows_out[4 * (size_t)slot + q] = rows[q];
    double2* out = reinterpret_cast<double2*>(Hraw + (size_t)slot * 144);
    for (int i = 0; i < 72; ++i) out[i] = make_double2(H[2 * i], H[2 * i + 1]);
    }
#undef HE
}

// -----------------------------------------------------------------------------------------------------------
// PSD projection of the 12x12 pair Hessians (IglUtils::makePD, IglUtils.hpp:112-133).
//
// (1) Reduction 12 -> 9.  Every pair energy depends on vertex differences only, so H (1,1,1,1)^T (x) e_k = 0 for k = 1..3 (unused
// vertex blocks are zero, which keeps this true for the 2- and 3-vertex stencils).  With Q = Q4 (x) I3, Q4 the 3x4 Helmert matrix
// (orthonormal rows orthogonal to (1,1,1,1)), range(H) lies in range(Q^T), hence H = Q^T M Q with M = Q H Q^T (9x9) and, Q^T having
// orthonormal columns, makePD(H) = Q^T makePD(M) Q exactly.  A 9x9 (padded to 10x10) eigenproblem costs half a 12x12 one.
//
// (2) Parallel-order cyclic Jacobi held entirely in registers.  Five lanes share one matrix: lane k owns the columns sitting at
// ring positions 2k ("top") and 2k+1 ("bottom") of A and of the eigenvector accumulator V, so the column half of a rotation is
// lane-local and the row half only needs the five (c, s) pairs of the round.  Between rounds the columns travel round a Brent-Luk
// tournament ring (position 0 fixed, tops move one lane up, bottoms one lane down) and the rows of A follow the same permutation,
// which costs nothing because every moved value passes through a shuffle whose destination register is chosen at compile time.
// After 9 rounds (one sweep) the ring is back where it started.  Six matrices per warp (30 lanes).  A matrix that has converged
// freezes (c = 1, s = 0), so its result does not depend on its neighbours in the warp.
//
// Output: makePD(M) (81 doubles, row-major 9x9) over the first 81 entries of the pair's 144-double slot; the scatter kernel applies
// Q^T . Q on the fly.
constexpr int kProjWarps = 4;   // warps per CTA
constexpr int kProjN = 10;      // padded matrix order
constexpr int kProjG = 5;       // lanes per matrix
constexpr int kProjPerWarp = 6; // matrices per warp
__host__ __device__ constexpr int ring_next(int i) // where the row/column at position i sits after one round
{
    return i == 0 ? 0 : i == 1 ? 2 : i == kProjN - 2 ? kProjN - 1 : (i % 2 == 0) ? i + 2 : i - 2;
}
// Helmert rows: q0 = (1,-1,0,0)/sqrt2, q1 = (1,1,-2,0)/sqrt6, q2 = (1,1,1,-3)/sqrt12
DEV double helmert(int a, int c)
{
    const double r2 = 0.70710678118654752440, r6 = 0.40824829046386301637, r12 = 0.28867513459481288225;
    if (a == 0) return c == 0 ? r2 : (c == 1 ? -r2 : 0.0);
    if (a == 1) return c <= 1 ? r6 : (c == 2 ? -2.0 * r6 : 0.0);
    return c <= 2 ? r12 : -3.0 * r12;
}
// column j (< 9) of M = Q H Q^T, rows 0..8 (row 9 of the padded matrix is zero)
DEV void reduced_column(const double* __restrict__ H0, int j, double* col /* 10 */)
{
    const int b = j / 3, s = j - 3 * b;
    double w[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) w[i] = 0.0;
#pragma unroll
    for (int dd = 0; dd < 4; ++dd) {
        const double q = helmert(b, dd);
        const double* row = H0 + (3 * dd + s) * 12; // H is symmetric: row 3d+s stands for column 3d+s
#pragma unroll
        for (int i = 0; i < 12; ++i) w[i] += q * row[i];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            double v = 0.0;
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) v += helmert(a, cc) * w[3 * cc + r];
            col[3 * a + r] = v;
        }
    col[9] = 0.0;
}

__global__ void __launch_bounds__(32 * kProjWarps) k_barrier_hessian_project(const int* __restrict__ n_ptr, int capacity, double* __restrict__ H, int* __restrict__ psd)
{
    constexpr int N = kProjN, G = kProjG;
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int grp = lane / G, k = lane - G * grp, base = G * grp;
    const int n = min(*n_ptr, capacity);
    const int nwarps = gridDim.x * kProjWarps;
    for (int warp = blockIdx.x * kProjWarps + (threadIdx.x >> 5); warp * kProjPerWarp < n; warp += nwarps) { // warp-uniform trip count
    const int c = warp * kProjPerWarp + grp;
    bool live = grp < kProjPerWarp && c < n;
    double AT[N], AB[N], VT[N], VB[N];
    double* H0 = H + (size_t)(live ? c : 0) * 144;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        AT[i] = (i == 2 * k) ? 1.0 : 0.0;
        AB[i] = (i == 2 * k + 1) ? 1.0 : 0.0;
        VT[i] = (i == 2 * k) ? 1.0 : 0.0;
        VB[i] = (i == 2 * k + 1) ? 1.0 : 0.0;
    }
    if (live) {
        reduced_column(H0, 2 * k, AT);
        if (2 * k + 1 < 9) reduced_column(H0, 2 * k + 1, AB);
        else {
#pragma unroll
            for (int i = 0; i < N; ++i) AB[i] = 0.0; // the padding column
        }
    }
    __syncwarp(); // every lane has read H before anything is written back
    auto group_sum = [&](double v) {
        double t = 0.0;
#pragma unroll
        for (int m = 0; m < G; ++m) t += __shfl_sync(full, v, base + m);
        return t; // same order on every lane of the group
    };
    bool done = !live;
    for (int sweep = 0; sweep < 30; ++sweep) {
        // convergence of each matrix: off-diagonal mass against diagonal mass
        {
            double off = 0.0, dg = 0.0;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const double t2 = AT[i] * AT[i], b2 = AB[i] * AB[i];
                off += ((i == 2 * k) ? 0.0 : t2) + ((i == 2 * k + 1) ? 0.0 : b2);
                dg += ((i == 2 * k) ? t2 : 0.0) + ((i == 2 * k + 1) ? b2 : 0.0);
            }
            const double offg = group_sum(off), dgg = group_sum(dg);
            if (offg <= 2e-26 * dgg || offg <= 1e-300) done = true;
        }
        if (__all_sync(full, done)) break;
        for (int r = 0; r < N - 1; ++r) {
            double app = 0.0, aqq = 0.0, apq = 0.0;
#pragma unroll
            for (int m = 0; m < G; ++m)
                if (k == m) {
                    app = AT[2 * m];
                    aqq = AB[2 * m + 1];
                    apq = AB[2 * m];
                }
            double cc = 1.0, ss = 0.0;
            if (!done && apq != 0.0) {
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
                cc = 1.0 / sqrt(t * t + 1.0);
                ss = t * cc;
            }
            // columns (own pair): col_p' = c col_p - s col_q, col_q' = s col_p + c col_q, for A and V
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const double a0 = AT[i], a1 = AB[i], v0 = VT[i], v1 = VB[i];
                AT[i] = cc * a0 - ss * a1;
                AB[i] = ss * a0 + cc * a1;
                VT[i] = cc * v0 - ss * v1;
                VB[i] = ss * v0 + cc * v1;
            }
            // rows (all pairs of the round)
#pragma unroll
            for (int m = 0; m < G; ++m) {
                const double cm = __shfl_sync(full, cc, base + m), sm = __shfl_sync(full, ss, base + m);
                const double t0 = AT[2 * m], t1 = AT[2 * m + 1], b0 = AB[2 * m], b1 = AB[2 * m + 1];
                AT[2 * m] = cm * t0 - sm * t1;
                AT[2 * m + 1] = sm * t0 + cm * t1;
                AB[2 * m] = cm * b0 - sm * b1;
                AB[2 * m + 1] = sm * b0 + cm * b1;
            }
            // ring move
            double nAT[N], nAB[N];
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const double upA = __shfl_up_sync(full, (k == 0) ? AB[i] : AT[i], 1);
                const double dnA = __shfl_down_sync(full, AB[i], 1);
                nAT[ring_next(i)] = (k == 0) ? AT[i] : upA;
                nAB[ring_next(i)] = (k == G - 1) ? AT[i] : dnA;
                const double upV = __shfl_up_sync(full, (k == 0) ? VB[i] : VT[i], 1);
                const double dnV = __shfl_down_sync(full, VB[i], 1);
                const double vt = VT[i];
                VT[i] = (k == 0) ? vt : upV;
                VB[i] = (k == G - 1) ? vt : dnV;
            }
#pragma unroll
            for (int i = 0; i < N; ++i) {
                AT[i] = nAT[i];
                AB[i] = nAB[i];
            }
        }
    }
    // clamp the negative eigenvalues and rebuild: makePD(M) = sum_{lambda > 0} lambda v v^T  (IglUtils.hpp:123-131)
    double lt = 0.0, lb = 0.0;
#pragma unroll
    for (int m = 0; m < G; ++m)
        if (k == m) {
            lt = AT[2 * m];
            lb = AB[2 * m + 1];
        }
    // IglUtils.hpp:123-125: "if (eigenvalues()[0] >= 0.0) return;" -- a block without a negative eigenvalue is handed back untouched.
    // The raw 12x12 input then stays in its slot (nothing is written below) and the scatter kernel reads it directly.
    {
        double lmin = fmin(lt, lb);
#pragma unroll
        for (int m = 0; m < G; ++m) lmin = fmin(lmin, __shfl_sync(full, fmin(lt, lb), base + m));
        const bool unchanged = lmin >= 0.0;
        if (live && k == 0) psd[c] = unchanged ? 1 : 0;
        if (unchanged) live = false; // (group-uniform) keep the shuffles below convergent, skip the stores
    }
    lt = fmax(lt, 0.0);
    lb = fmax(lb, 0.0);
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        const double wt = lt * VT[i], wb = lb * VB[i];
#pragma unroll
        for (int j = i; j < 9; ++j) {
            const double tot = group_sum(wt * VT[j] + wb * VB[j]);
            if (live && k == ((i * 9 + j) % G)) {
                H0[i * 9 + j] = tot;
                H0[j * 9 + i] = tot;
            }
        }
    }
    __syncwarp();
    }
}

// entry (i, j) of a pair slot's projected Hessian: the raw 12x12 where makePD returned its input (psd flag), else
// (Q^T M Q)[i][j] = sum_{a,b} Q4[a][bi] Q4[b][bj] M[3a+r][3b+q] from the 9x9 M that k_barrier_hessian_project left in the slot
DEV double pair_hessian_entry(const double* __restrict__ H0, bool raw, int i, int j)
{
    if (raw) return H0[i * 12 + j];
    const int bi = i / 3, r = i % 3, bj = j / 3, q = j % 3;
    double v = 0.0;
#pragma unroll
    for (int ka = 0; ka < 3; ++ka) {
        const double qa = helmert(ka, bi);
#pragma unroll
        for (int kb = 0; kb < 3; ++kb) v += (qa * helmert(kb, bj)) * H0[(3 * ka + r) * 9 + 3 * kb + q];
    }
    return v;
}

// scatter of the projected pair Hessians into the CSR values (upper-triangular 3x3 blocks, LinSysSolver.hpp:207-265)
constexpr int kScatWarps = 8;
__global__ void __launch_bounds__(32 * kScatWarps) k_barrier_hessian_scatter(BarrierArgs p, const int* __restrict__ n_ptr, int capacity, const double* __restrict__ H,
    const int* __restrict__ rows_in, const int* __restrict__ psd, double* __restrict__ a, int* __restrict__ err)
{
    __shared__ int sOff[kScatWarps][48];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int n = min(*n_ptr, capacity);
    for (int c = blockIdx.x * kScatWarps + wib; c < n; c += gridDim.x * kScatWarps) {
    const double* H0 = H + (size_t)c * 144;
    const bool raw = psd[c] != 0;
    // CSR offsets of the 16 vertex blocks x 3 rows (upper-triangular blocks only); -1 = skip, -2 = missing in the pattern
    int rows[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) rows[q] = rows_in[4 * (size_t)c + q];
    for (int t = lane; t < 48; t += 32) {
        const int bi = t / 12, bj = (t / 3) % 4, r = t % 3;
        int o = -1;
        const int vi = rows[bi], vj = rows[bj];
        if (upper_block(rows, bi, bj) && owns_row(p, vi) && !proj_dbc(p.dbc, vi, p.projectDBC) && !proj_dbc(p.dbc, vj, p.projectDBC)) {
            const int c0 = (vi == vj) ? r : 0;
            o = csr_find(p.ia, p.ja, p.base, 3 * vi + r, 3 * vj + c0);
            if (o < 0) o = -2;
            else o -= c0; // so that column q of the block lands at o + q
        }
        sOff[wib][t] = o;
    }
    __syncwarp();
#pragma unroll
    for (int kk = 0; kk < 5; ++kk) {
        const int e = lane + 32 * kk;
        if (e < 144) {
            const int i = e / 12, j = e % 12;
            const int bi = i / 3, r = i % 3, bj = j / 3, q = j % 3;
            const int o = sOff[wib][(bi * 4 + bj) * 3 + r];
            if (o == -2) atomicExch(err, 1);
            else if (o != -1) {
                if (rows[bi] == rows[bj] && q < r) continue; // strictly lower part of a diagonal block
                atomicAdd(a + o + q, pair_hessian_entry(H0, raw, i, j));
            }
        }
    }
    __syncwarp(); // sOff is reused by the next slot of this warp
    }
}

// reproducible mode: the scatter above as a per-row gather (repro.cuh), one thread per row vertex; slot c holds list entry c
__global__ void __launch_bounds__(128) k_barrier_hessian_gather(BarrierArgs p, const int* __restrict__ n_ptr, int capacity, const double* __restrict__ H,
    const int* __restrict__ psd, double* __restrict__ a, int* __restrict__ err)
{
    const int n = min(*n_ptr, capacity);
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < p.nV; v += gridDim.x * blockDim.x)
        repro_gather_row(v, p.rep.h, p.dbc, p.projectDBC, p.ia, p.ja, p.base, a, err, [&](int c, int bi, int bj, double* acc) {
            if (c >= n) return;
            const double* H0 = H + (size_t)c * 144;
            const bool raw = psd[c] != 0;
            for (int r = 0; r < 3; ++r)
                for (int q = 0; q < 3; ++q) acc[3 * r + q] += pair_hessian_entry(H0, raw, 3 * bi + r, 3 * bj + q);
        });
}

// -----------------------------------------------------------------------------------------------------------
void barrier_energy(const BarrierArgs& p, double* partials, int* bad, cudaStream_t st)
{
    k_barrier_energy<<<kBarrierEnergyBlocks, 256, 0, st>>>(p, partials, bad);
}
int barrier_energy_blocks() { return kBarrierEnergyBlocks; }
void barrier_gradient(const BarrierArgs& p, double* g, cudaStream_t st)
{
    if (p.rep.on) {
        if (p.kappa_dev) k_barrier_gradient<true, true><<<kSMs * 4, 128, 0, st>>>(p, p.rep.stage);
        else k_barrier_gradient<false, true><<<kSMs * 4, 128, 0, st>>>(p, p.rep.stage);
        repro_gather_g(p.nV, p.rep.g, p.rep.stage, 0ull, kAllKeys, g, st);
    }
    else if (p.kappa_dev) k_barrier_gradient<true, false><<<kSMs * 4, 128, 0, st>>>(p, g);
    else k_barrier_gradient<false, false><<<kSMs * 4, 128, 0, st>>>(p, g);
}
void evaluate_constraints(const BarrierArgs& p, double* val, cudaStream_t st) { k_evaluate_constraints<<<kSMs * 2, 256, 0, st>>>(p, val); }
void constraint_jacobian_t(const BarrierArgs& p, const double* input, double coef, double* g, cudaStream_t st)
{
    if (p.rep.on) {
        k_constraint_jacobian_t<true><<<kSMs * 4, 128, 0, st>>>(p, input, coef, p.rep.stage);
        repro_gather_g(p.nV, p.rep.g, p.rep.stage, 0ull, para_keys(p.rep.cap), g, st); // the active list's contributions
    }
    else k_constraint_jacobian_t<false><<<kSMs * 4, 128, 0, st>>>(p, input, coef, g);
}
void para_gradient(const BarrierArgs& p, double* g, cudaStream_t st)
{
    if (p.rep.on) {
        if (p.kappa_dev) k_barrier_gradient<true, true, true><<<kSMs, 128, 0, st>>>(p, p.rep.stage);
        else k_barrier_gradient<false, true, true><<<kSMs, 128, 0, st>>>(p, p.rep.stage);
        repro_gather_g(p.nV, p.rep.g, p.rep.stage, para_keys(p.rep.cap), kAllKeys, g, st); // the mollified list's contributions
    }
    else if (p.kappa_dev) k_barrier_gradient<true, false, true><<<kSMs, 128, 0, st>>>(p, g);
    else k_barrier_gradient<false, false, true><<<kSMs, 128, 0, st>>>(p, g);
}
void barrier_hessian_build_project(const BarrierArgs& p, int* flags, double* Hraw, int* rows, int* psd, int* n_owned, int capacity, cudaStream_t st)
{
    cudaMemsetAsync(n_owned, 0, sizeof(int), st);
    if (p.rep.on) {
        if (p.kappa_dev) k_barrier_hessian_build<true, true><<<kSMs * 8, 64, 0, st>>>(p, Hraw, rows, n_owned, capacity, flags);
        else k_barrier_hessian_build<false, true><<<kSMs * 8, 64, 0, st>>>(p, Hraw, rows, n_owned, capacity, flags);
    }
    else if (p.kappa_dev) k_barrier_hessian_build<true, false><<<kSMs * 8, 64, 0, st>>>(p, Hraw, rows, n_owned, capacity, flags);
    else k_barrier_hessian_build<false, false><<<kSMs * 8, 64, 0, st>>>(p, Hraw, rows, n_owned, capacity, flags);
    k_barrier_hessian_project<<<kSMs * 4, 32 * kProjWarps, 0, st>>>(n_owned, capacity, Hraw, psd);
}
void barrier_hessian_scatter(const BarrierArgs& p, double* a, int* flags, const double* Hraw, const int* rows, const int* psd, const int* n_owned, int capacity, cudaStream_t st)
{
    if (p.rep.on) k_barrier_hessian_gather<<<kSMs * 4, 128, 0, st>>>(p, n_owned, capacity, Hraw, psd, a, flags + FLAG_PATTERN);
    else k_barrier_hessian_scatter<<<kSMs * 4, 32 * kScatWarps, 0, st>>>(p, n_owned, capacity, Hraw, rows, psd, a, flags + FLAG_PATTERN);
}

} // namespace ipcgpu
