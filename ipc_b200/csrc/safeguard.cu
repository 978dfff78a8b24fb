// safeguard.cu -- line-search safeguards on the device (sm_90a): element inversion check and intersection check (edge-triangle, and
// codimension-0 point in tetrahedron).
//   *** compiled with --fmad=false (NOFMA_FILES): the floating-point decisions (filter, full-pivot solve) round like the CPU oracle ***
//
// Reference being replaced (SURVEY 8(f) rank 2: "a whole line-search trial is one stream with no host round trip"):
//   Mesh<3>::checkInversion(bool mute)                         src/Mesh.cpp:715-763
//   SelfCollisionHandler<3>::checkEdgeTriIntersectionIfAny     src/CollisionObject/SelfCollisionHandler.cpp:3254-3337
//   IglUtils::segTriIntersect (USE_PREDICATES, CMakeLists:139) src/Utils/IglUtils.hpp:214-265
//   IglUtils::pointInsideTetrahedron (USE_PREDICATES)          src/Utils/IglUtils.hpp:276-294
//   SpatialHash::queryTriangleForEdges                         src/Utils/SpatialHash.hpp:526-556   (here: the sort-based grid of broadphase.cuh)
//
// igl::predicates::orient3d is an exact predicate (Shewchuk).  Device version: the usual floating-point filter; inputs it cannot decide
// (a handful per million tests) go through an exact evaluation with floating-point expansions held in thread-local memory
// (two-sum, two-product via the explicit fma intrinsic, grow-expansion, scale-expansion -- Shewchuk 1997, figs. 6, 7, 13).
#include "broadphase.cuh"
#include "abi.h"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <vector>

namespace ipcgpu {

// ---- exact arithmetic on expansions ------------------------------------------------------------------------------------------
DEV void two_sum(double a, double b, double& x, double& y)
{
    x = a + b;
    const double bv = x - a, av = x - bv;
    y = (a - av) + (b - bv);
}
DEV void two_prod(double a, double b, double& x, double& y)
{
    x = a * b;
    y = __fma_rn(a, b, -x); // exact rounding error of the product
}
// h (n components, nonoverlapping, increasing magnitude) += b, in place; returns the new length (<= n + 1); zeros are dropped
__device__ __noinline__ int grow_inplace(int n, double* h, double b)
{
    double q = b;
    int m = 0;
    for (int i = 0; i < n; ++i) {
        double s, r;
        two_sum(q, h[i], s, r); // h[i] is read before h[m] (m <= i) is written
        if (r != 0.0) h[m++] = r;
        q = s;
    }
    if (q != 0.0 || m == 0) h[m++] = q;
    return m;
}
// h = e + f (h must not alias f; capacity ne + nf)
DEV int expansion_sum(int ne, const double* e, int nf, const double* f, double* h)
{
    int n = ne;
    for (int i = 0; i < ne; ++i) h[i] = e[i];
    for (int j = 0; j < nf; ++j) n = grow_inplace(n, h, f[j]);
    return n;
}
// h = e * b (h must not alias e; capacity 2 n)
__device__ __noinline__ int scale_expansion(int n, const double* e, double b, double* h)
{
    double q, hh;
    two_prod(e[0], b, q, hh);
    int m = 0;
    if (hh != 0.0) h[m++] = hh;
    for (int i = 1; i < n; ++i) {
        double t1, t0, s, r;
        two_prod(e[i], b, t1, t0);
        two_sum(q, t0, s, r);
        if (r != 0.0) h[m++] = r;
        two_sum(t1, s, q, r);
        if (r != 0.0) h[m++] = r;
    }
    if (q != 0.0 || m == 0) h[m++] = q;
    return m;
}
// x*y - z*w exactly (<= 4 components)
DEV int prod_diff(double x, double y, double z, double w, double* h)
{
    double a1, a0, b1, b0;
    two_prod(x, y, a1, a0);
    two_prod(z, w, b1, b0);
    h[0] = a0;
    h[1] = a1;
    int n = grow_inplace(2, h, -b0);
    return grow_inplace(n, h, -b1);
}
// exact sign of the 4x4 orientation determinant on the untranslated coordinates (cofactor expansion along z)
__device__ __noinline__ int orient3d_exact(const double* pa, const double* pb, const double* pc, const double* pd)
{
    double ab[4], bc[4], cd[4], da[4], ac[4], bd[4];
    const int nab = prod_diff(pa[0], pb[1], pb[0], pa[1], ab), nbc = prod_diff(pb[0], pc[1], pc[0], pb[1], bc), ncd = prod_diff(pc[0], pd[1], pd[0], pc[1], cd);
    const int nda = prod_diff(pd[0], pa[1], pa[0], pd[1], da), nac = prod_diff(pa[0], pc[1], pc[0], pa[1], ac), nbd = prod_diff(pb[0], pd[1], pd[0], pb[1], bd);
    double nac_[4], nbd_[4], t[12], cda[12], dab[12], abc[12], bcd[12];
    for (int i = 0; i < nac; ++i) nac_[i] = -ac[i];
    for (int i = 0; i < nbd; ++i) nbd_[i] = -bd[i];
    int nt = expansion_sum(ncd, cd, nda, da, t);
    const int ncda = expansion_sum(nt, t, nac, ac, cda);
    nt = expansion_sum(nda, da, nab, ab, t);
    const int ndab = expansion_sum(nt, t, nbd, bd, dab);
    nt = expansion_sum(nab, ab, nbc, bc, t);
    const int nabc = expansion_sum(nt, t, nac, nac_, abc);
    nt = expansion_sum(nbc, bc, ncd, cd, t);
    const int nbcd = expansion_sum(nt, t, nbd, nbd_, bcd);
    double adet[24], bdet[24], cdet[24], ddet[24], det[96];
    const int na = scale_expansion(nbcd, bcd, pa[2], adet), nb = scale_expansion(ncda, cda, -pb[2], bdet);
    const int nc = scale_expansion(ndab, dab, pc[2], cdet), nd = scale_expansion(nabc, abc, -pd[2], ddet);
    int n = expansion_sum(na, adet, nb, bdet, det);
    for (int j = 0; j < nc; ++j) n = grow_inplace(n, det, cdet[j]);
    for (int j = 0; j < nd; ++j) n = grow_inplace(n, det, ddet[j]);
    const double top = det[n - 1]; // the largest-magnitude component carries the sign
    return (top > 0.0) - (top < 0.0);
}
// sign of orient3d(pa, pb, pc, pd): +1 / 0 / -1
DEV int orient3d(const double* pa, const double* pb, const double* pc, const double* pd)
{
    const double adx = pa[0] - pd[0], bdx = pb[0] - pd[0], cdx = pc[0] - pd[0];
    const double ady = pa[1] - pd[1], bdy = pb[1] - pd[1], cdy = pc[1] - pd[1];
    const double adz = pa[2] - pd[2], bdz = pb[2] - pd[2], cdz = pc[2] - pd[2];
    const double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy, cdxady = cdx * ady, adxcdy = adx * cdy, adxbdy = adx * bdy, bdxady = bdx * ady;
    const double det = adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy) + cdz * (adxbdy - bdxady);
    const double permanent = (fabs(bdxcdy) + fabs(cdxbdy)) * fabs(adz) + (fabs(cdxady) + fabs(adxcdy)) * fabs(bdz) + (fabs(adxbdy) + fabs(bdxady)) * fabs(cdz);
    const double errbound = 1.7763568394002505e-15 * permanent; // 16 eps: wider than Shewchuk's (7 + 56 eps) eps, see the oracle
    if (det > errbound) return 1;
    if (-det > errbound) return -1;
    return orient3d_exact(pa, pb, pc, pd);
}

// x = M^-1 b, Gaussian elimination with full pivoting in Eigen::FullPivLU's order (first maximum in column-major order of the
// remaining corner), rank threshold eps * 3 * max pivot; m is the 3x3 in rows
DEV void full_piv_solve3(double (&m)[3][3], const double* b, double* x)
{
    int cq[3] = { 0, 1, 2 };
    double rhs[3] = { b[0], b[1], b[2] };
    double maxpiv = 0.0;
    int nz = 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (k >= nz) break;
        int pr = k, pc = k;
        double big = -1.0;
        for (int j = k; j < 3; ++j)
            for (int i = k; i < 3; ++i)
                if (fabs(m[i][j]) > big) { big = fabs(m[i][j]); pr = i; pc = j; }
        if (big == 0.0) { nz = k; break; }
        maxpiv = fmax(maxpiv, big);
        if (pr != k) {
            for (int j = 0; j < 3; ++j) { const double t = m[k][j]; m[k][j] = m[pr][j]; m[pr][j] = t; }
            const double t = rhs[k]; rhs[k] = rhs[pr]; rhs[pr] = t;
        }
        if (pc != k) {
            for (int i = 0; i < 3; ++i) { const double t = m[i][k]; m[i][k] = m[i][pc]; m[i][pc] = t; }
            const int t = cq[k]; cq[k] = cq[pc]; cq[pc] = t;
        }
        for (int i = k + 1; i < 3; ++i) m[i][k] /= m[k][k];
        for (int i = k + 1; i < 3; ++i)
            for (int j = k + 1; j < 3; ++j) m[i][j] -= m[i][k] * m[k][j];
    }
    int rank = 0;
    for (int k = 0; k < nz; ++k)
        if (fabs(m[k][k]) > maxpiv * 2.220446049250313e-16 * 3.0) ++rank;
    for (int i = 1; i < 3; ++i)
        for (int j = 0; j < i; ++j) rhs[i] -= m[i][j] * rhs[j];
    double y[3] = { 0.0, 0.0, 0.0 };
    for (int i = rank - 1; i >= 0; --i) {
        double s = rhs[i];
        for (int j = i + 1; j < rank; ++j) s -= m[i][j] * y[j];
        y[i] = s / m[i][i];
    }
    x[0] = x[1] = x[2] = 0.0;
    for (int k = 0; k < 3; ++k) x[cq[k]] = y[k];
}

// IglUtils::segTriIntersect (IglUtils.hpp:214-265)
DEV bool seg_tri_intersect(const double* ve0, const double* ve1, const double* vt0, const double* vt1, const double* vt2)
{
    const int o1 = orient3d(vt0, vt1, vt2, ve0), o2 = orient3d(vt0, vt1, vt2, ve1);
    if (o1 == 0 || o2 == 0) return false; // coplanar: caught through d(EE) = 0 or d(PT) = 0
    if (o1 == o2) return false;           // the edge is on one side of the triangle's plane
    double m[3][3], b[3], uvt[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        m[i][0] = vt1[i] - vt0[i];
        m[i][1] = vt2[i] - vt0[i];
        m[i][2] = ve0[i] - ve1[i];
        b[i] = ve0[i] - vt0[i];
    }
    full_piv_solve3(m, b, uvt);
    return uvt[0] >= 0.0 && uvt[1] >= 0.0 && uvt[0] + uvt[1] <= 1.0 && uvt[2] >= 0.0 && uvt[2] <= 1.0;
}

// ---- kernels ---------------------------------------------------------------------------------------------------------------
// one warp per query triangle (kPairQueriesPerWarp in a row): scan the edge grid for boxes that overlap the triangle's box, run the
// exact test on the lanes that hold a candidate, count the triangles with at least one intersecting edge (the reference stops at
// the first per triangle: same count)
__global__ void __launch_bounds__(256) k_tri_edge_intersect(SurfArgs s, const Grid* __restrict__ gp, SortedGrid eg, const Box* __restrict__ tboxes, int first, int last,
    int* __restrict__ n_hit)
{
    const int lane = threadIdx.x & 31;
    const Grid g = *gp;
    const int q0 = first + (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * kPairQueriesPerWarp;
    for (int f = q0; f < min(q0 + kPairQueriesPerWarp, last); ++f) {
        const int tv[3] = { s.SF[f], s.SF[(size_t)s.nSF + f], s.SF[(size_t)2 * s.nSF + f] };
        double t[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) t[k][c] = __ldg(s.V + (size_t)c * s.nV + tv[k]);
        const int cod_f = s.vCoDim ? s.vCoDim[tv[0]] : 3;
        const bool tri_dbc = s.dbc && s.dbc[tv[0]] && s.dbc[tv[1]] && s.dbc[tv[2]];
        bool any = false;
        warp_scan_candidates(g, eg, tboxes[f], lane, [&](bool hit, int e) {
            if (!hit || any) return;
            const int e0 = s.SE[2 * e], e1 = s.SE[2 * e + 1];
            if (e0 == tv[0] || e0 == tv[1] || e0 == tv[2] || e1 == tv[0] || e1 == tv[1] || e1 == tv[2]) return;
            const int cod_e = s.vCoDim ? s.vCoDim[e0] : 3;
            // mesh against itself: :3281-3284; mesh against the obstacle: every pair (MeshCO.cpp:2611-2678); inside the obstacle: none
            const bool oT = obstacle_vertex(s, tv[0]), oE = obstacle_vertex(s, e0);
            if (oT && oE) return;
            if (!oT && !oE && ((cod_f < 3 && cod_e < 3) || (tri_dbc && s.dbc[e0] && s.dbc[e1]))) return;
            double p0[3], p1[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                p0[c] = __ldg(s.V + (size_t)c * s.nV + e0);
                p1[c] = __ldg(s.V + (size_t)c * s.nV + e1);
            }
            if (seg_tri_intersect(p0, p1, t[0], t[1], t[2])) any = true;
        });
        if (__any_sync(0xffffffffu, any) && lane == 0) atomicAdd(n_hit, 1);
    }
}

// ---- codimension-0 points inside tetrahedra (second half of checkEdgeTriIntersectionIfAny, SelfCollisionHandler.cpp:3301-3337) -----------
// IglUtils::pointInsideTetrahedron (IglUtils.hpp:276-294, USE_PREDICATES): four exact orientations in the reference's argument order, each
// "not negative".  A point on a face, an edge or a vertex is inside; a zero-volume tet holds every point of its box that passes the four
// (degenerate) orientations; an inverted tet holds no interior point.
DEV bool point_in_tet(const double* p, const double (&t)[4][3])
{
    return orient3d(t[0], t[2], t[1], p) >= 0 && orient3d(t[0], t[3], t[2], p) >= 0 && orient3d(t[0], t[1], t[3], p) >= 0 && orient3d(t[1], t[2], t[3], p) >= 0;
}

DEV int point_cell(const PointGrid& g, int a, double x) { return min(max((int)floor((x - g.o[a]) * g.inv_h), 0), g.n[a] - 1); }

// one CTA: the box of the points, then a cubic-cell grid with at most max(8, min(n, 2^20)) cells (bisection on the cell edge).  The
// floor of (x - o) * inv_h is monotone in x, so a point inside a tetrahedron's box lies in a cell of the box's cell range.
__global__ void __launch_bounds__(1024) k_pit_grid(const double* __restrict__ V, int nV, const int* __restrict__ pts, int n, PointGrid* __restrict__ gout)
{
    __shared__ double s_lo[32][3], s_hi[32][3];
    double lo[3] = { INFINITY, INFINITY, INFINITY }, hi[3] = { -INFINITY, -INFINITY, -INFINITY };
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int v = pts[i];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double x = __ldg(V + (size_t)a * nV + v);
            lo[a] = fmin(lo[a], x);
            hi[a] = fmax(hi[a], x);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = warp_min(lo[a]);
        hi[a] = -warp_min(-hi[a]);
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
        for (int a = 0; a < 3; ++a) { s_lo[w][a] = lo[a]; s_hi[w][a] = hi[a]; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    PointGrid g;
    for (int a = 0; a < 3; ++a) {
        g.lo[a] = s_lo[0][a];
        g.hi[a] = s_hi[0][a];
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) { g.lo[a] = fmin(g.lo[a], s_lo[k][a]); g.hi[a] = fmax(g.hi[a], s_hi[k][a]); }
        g.o[a] = g.lo[a];
    }
    const double target = (double)max(8, min(n, (int)kGridCells));
    const double ext = fmax(g.hi[0] - g.lo[0], fmax(g.hi[1] - g.lo[1], g.hi[2] - g.lo[2]));
    auto cells = [&](double h) { return (floor((g.hi[0] - g.lo[0]) / h) + 1.0) * (floor((g.hi[1] - g.lo[1]) / h) + 1.0) * (floor((g.hi[2] - g.lo[2]) / h) + 1.0); };
    double h = 1.0;
    if (ext > 0.0) {
        double a = 0.0;
        h = ext;
        for (int it = 0; it < 64; ++it) { // smallest edge (to rounding) with cells(h) <= target
            const double mid = 0.5 * (a + h);
            if (cells(mid) <= target) h = mid;
            else a = mid;
        }
    }
    g.inv_h = 1.0 / h;
    for (int a = 0; a < 3; ++a) g.n[a] = min((int)floor((g.hi[a] - g.lo[a]) * g.inv_h) + 1, (int)kGridCells);
    *gout = g;
}

__global__ void __launch_bounds__(256) k_pit_keys(const double* __restrict__ V, int nV, const int* __restrict__ pts, int n, const PointGrid* __restrict__ gp,
    unsigned* __restrict__ key, int* __restrict__ id)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const PointGrid g = *gp;
    const int v = pts[i];
    int c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = point_cell(g, a, __ldg(V + (size_t)a * nV + v));
    key[i] = (unsigned)(((long long)c[2] * g.n[1] + c[1]) * g.n[0] + c[0]);
    id[i] = v;
}

// one thread per tetrahedron [t_begin, t_end) (every tet: no Dirichlet and no mu / lambda filter, the reference loops over all of F): the
// rows of cells its box covers are consecutive key ranges of the sorted points, found by binary search; every point in them that lies in
// the tet's box (inclusive, as the reference compares) gets the exact test.  Counts (point, tet) pairs.
__global__ void __launch_bounds__(256) k_points_in_tets(ElasticArgs p, const PointGrid* __restrict__ gp, const unsigned* __restrict__ key, const int* __restrict__ id, int n,
    int* __restrict__ n_hit)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int hits = 0;
    if (t < p.t_end - p.t_begin) {
        const int tt = p.t_begin + t;
        const PointGrid g = *gp;
        double x[4][3], lo[3], hi[3];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int v = __ldg(p.T + (size_t)k * p.nT + tt);
#pragma unroll
            for (int a = 0; a < 3; ++a) x[k][a] = __ldg(p.V + (size_t)a * p.nV + v);
        }
        bool miss = false;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            lo[a] = fmin(fmin(x[0][a], x[1][a]), fmin(x[2][a], x[3][a]));
            hi[a] = fmax(fmax(x[0][a], x[1][a]), fmax(x[2][a], x[3][a]));
            miss = miss || lo[a] > g.hi[a] || hi[a] < g.lo[a];
        }
        if (!miss) {
            int c0[3], c1[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) { c0[a] = point_cell(g, a, lo[a]); c1[a] = point_cell(g, a, hi[a]); }
            for (int iz = c0[2]; iz <= c1[2]; ++iz)
                for (int iy = c0[1]; iy <= c1[1]; ++iy) {
                    const unsigned row = (unsigned)(((long long)iz * g.n[1] + iy) * g.n[0]);
                    int j = 0, e = n;
                    { // lower bound of the row's first cell
                        int l = 0, r = n;
                        while (l < r) { const int m = (l + r) >> 1; if (__ldg(key + m) < row + c0[0]) l = m + 1; else r = m; }
                        j = l;
                    }
                    { // upper bound of its last cell
                        int l = j, r = n;
                        while (l < r) { const int m = (l + r) >> 1; if (__ldg(key + m) <= row + c1[0]) l = m + 1; else r = m; }
                        e = l;
                    }
                    for (; j < e; ++j) {
                        const int v = __ldg(id + j);
                        double q[3];
#pragma unroll
                        for (int a = 0; a < 3; ++a) q[a] = __ldg(p.V + (size_t)a * p.nV + v);
                        if (lo[0] <= q[0] && lo[1] <= q[1] && lo[2] <= q[2] && hi[0] >= q[0] && hi[1] >= q[1] && hi[2] >= q[2] && point_in_tet(q, x)) ++hits;
                    }
                }
        }
    }
    const int tot = warp_sum(hits);
    if (tot && (threadIdx.x & 31) == 0) atomicAdd(n_hit, tot);
}

// Mesh::checkInversion: tets with mu, lambda != 0 whose current edge matrix has a negative determinant
__global__ void __launch_bounds__(256) k_count_inverted(ElasticArgs p, int* __restrict__ n_inv)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    bool inv = false;
    if (t < p.t_end - p.t_begin) {
        const int tt = p.t_begin + t;
        if (__ldg(p.mu + tt) != 0.0 && __ldg(p.lam + tt) != 0.0) {
            int v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = __ldg(p.T + (size_t)k * p.nT + tt);
            double e[3][3];
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
                for (int c = 0; c < 3; ++c) e[k][c] = __ldg(p.V + (size_t)c * p.nV + v[k + 1]) - __ldg(p.V + (size_t)c * p.nV + v[0]);
            // determinant of the matrix whose COLUMNS are e[0], e[1], e[2] (cofactors along the first row)
            const double det = e[0][0] * (e[1][1] * e[2][2] - e[2][1] * e[1][2]) - e[1][0] * (e[0][1] * e[2][2] - e[2][1] * e[0][2])
                + e[2][0] * (e[0][1] * e[1][2] - e[1][1] * e[0][2]);
            inv = det < 0.0;
        }
    }
    const unsigned m = __ballot_sync(0xffffffffu, inv);
    if (m && (threadIdx.x & 31) == 0) atomicAdd(n_inv, __popc(m));
}

} // namespace ipcgpu

using namespace ipcgpu;

// enqueue the inversion count of this rank's tets into IterState::checks[0]
int safeguard_inversion(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->stream;
    int* cnt = &ctx->iter.p->checks[0];
    if (cudaMemsetAsync(cnt, 0, sizeof(int), st) != cudaSuccess) return IPCGPU_ERR_CUDA;
    const ElasticArgs p = ctx->eargs();
    const int n = p.t_end - p.t_begin;
    if (n > 0) k_count_inverted<<<nblk(n, 256), 256, 0, st>>>(p, cnt);
    ++ctx->launches;
    return cudaGetLastError() == cudaSuccess ? 0 : IPCGPU_ERR_CUDA;
}

// the codimension-0 vertices (vCoDim == 0) and the workspace of their grid; none (or no vCoDim) leaves the check as it was
int safeguard_set_points(ipcgpu_ctx* ctx, const int* vCoDim)
{
    PointTetWork& w = ctx->pit;
    std::vector<int> pts;
    if (vCoDim)
        for (int v = 0; v < ctx->nV; ++v)
            if (vCoDim[v] == 0) pts.push_back(v);
    w.n = (int)pts.size();
    if (w.n == 0) return 0;
    size_t bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, w.n, 0, 24, ctx->stream) != cudaSuccess)
        return IPCGPU_ERR_CUDA;
    w.sort_bytes = bytes;
    const bool ok = w.pts.upload(pts.data(), pts.size(), ctx->stream) && w.id.reserve(w.n) && w.id_sorted.reserve(w.n) && w.key.reserve(w.n) && w.key_sorted.reserve(w.n)
        && w.grid.reserve(1) && w.sort_tmp.reserve(std::max<size_t>(bytes, 1));
    if (!ok) {
        ctx->err = "point-in-tetrahedron workspace allocation failed";
        return IPCGPU_ERR_CUDA;
    }
    return cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : IPCGPU_ERR_CUDA; // (pts came from pageable host memory)
}

// enqueue the intersection count into IterState::checks[1]: the edge-triangle pairs (this rank's share of the triangles) plus the
// (codimension-0 point, tetrahedron) pairs of the point-in-tetrahedron test (this rank's tets).  The static grid is rebuilt at the current
// positions with zero inflation (the reference rebuilds its hash before the check as well, Optimizer.cpp:2720); so is the point grid.
int safeguard_intersections(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->stream;
    ContactWork& w = ctx->cw;
    const SurfArgs s = surf_args(ctx);
    int* cnt = &ctx->iter.p->checks[1];
    if (cudaMemsetAsync(cnt, 0, sizeof(int), st) != cudaSuccess) return IPCGPU_ERR_CUDA;
    if (s.nSF > 0 && s.nSE > 0) {
        int rc = boxes_and_grid(ctx, 0.0, false);
        if (rc) return rc;
        const SortedGrid eg = edge_grid(ctx);
        const int f0 = (int)((long long)s.nSF * ctx->rank / ctx->nranks), f1 = (int)((long long)s.nSF * (ctx->rank + 1) / ctx->nranks);
        if (f1 > f0) k_tri_edge_intersect<<<nblk(f1 - f0, 8 * kPairQueriesPerWarp), 256, 0, st>>>(s, w.grid.p, eg, w.tbox.p, f0, f1, cnt);
        ++ctx->launches;
        if (cudaGetLastError() != cudaSuccess) return IPCGPU_ERR_CUDA;
    }
    PointTetWork& pw = ctx->pit;
    const ElasticArgs p = ctx->eargs();
    if (pw.n == 0 || p.t_end <= p.t_begin) return 0;
    k_pit_grid<<<1, 1024, 0, st>>>(ctx->V.p, ctx->nV, pw.pts.p, pw.n, pw.grid.p);
    k_pit_keys<<<nblk(pw.n, 256), 256, 0, st>>>(ctx->V.p, ctx->nV, pw.pts.p, pw.n, pw.grid.p, pw.key.p, pw.id.p);
    size_t bytes = pw.sort_bytes;
    if (cub::DeviceRadixSort::SortPairs(pw.sort_tmp.p, bytes, pw.key.p, pw.key_sorted.p, pw.id.p, pw.id_sorted.p, pw.n, 0, 24, st) != cudaSuccess) return IPCGPU_ERR_CUDA;
    k_points_in_tets<<<nblk(p.t_end - p.t_begin, 256), 256, 0, st>>>(p, pw.grid.p, pw.key_sorted.p, pw.id_sorted.p, pw.n, cnt);
    ctx->launches += 4; // (the sort counts as one)
    return cudaGetLastError() == cudaSuccess ? 0 : IPCGPU_ERR_CUDA;
}
