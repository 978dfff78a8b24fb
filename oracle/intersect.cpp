/* oracle/intersect.cpp -- TEST INFRASTRUCTURE ONLY (CPU restatement; never linked into or called by the product path).
 *
 * Line-search safeguards of the reference (SURVEY 8(f) rank 2):
 *   SelfCollisionHandler<3>::checkEdgeTriIntersectionIfAny   src/CollisionObject/SelfCollisionHandler.cpp:3254-3340
 *   IglUtils::segTriIntersect                                 src/Utils/IglUtils.hpp:214-265   (USE_PREDICATES branch: CMakeLists.txt:139)
 *   Mesh<3>::checkInversion                                   src/Mesh.cpp:715-763
 *
 * igl::predicates::orient3d (libigl -> Shewchuk's predicates, not in /root/reference) is an EXACT predicate: any correct exact
 * evaluation returns the same sign, so it is restated here from the published method (J. R. Shewchuk, "Adaptive Precision
 * Floating-Point Arithmetic and Fast Robust Geometric Predicates", 1997): a floating-point filter with a forward error bound, then
 * the determinant evaluated exactly with floating-point expansions (two-sum / two-product, grow-expansion, scale-expansion).
 * Pinned by tests/test_oracle_intersect.py against exact rational arithmetic (Python fractions) incl. exactly coplanar inputs.
 * Eigen's fullPivLu (IglUtils.hpp:258) is restated as Gaussian elimination with full pivoting in Eigen's pivot order
 * (first maximum in column-major order of the remaining corner), rank threshold 3 eps * max pivot, and both triangular solves by columns
 * as Eigen 3.4 runs them; pinned by tests/test_safeguard_regimes.py to a Python restatement of the same operations, bit for bit.
 */
#include "oracle.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

inline void two_sum(double a, double b, double& x, double& y)
{
    x = a + b;
    const double bv = x - a, av = x - bv;
    y = (a - av) + (b - bv);
}
inline void two_prod(double a, double b, double& x, double& y)
{
    x = a * b;
    y = std::fma(a, b, -x); /* exact error of the product */
}

/* e (nonoverlapping, increasing magnitude) + b -> h ; zero components dropped */
int grow_expansion(int n, const double* e, double b, double* h)
{
    double q = b;
    int m = 0;
    for (int i = 0; i < n; ++i) {
        double s, r;
        two_sum(q, e[i], s, r);
        if (r != 0.0) h[m++] = r;
        q = s;
    }
    if (q != 0.0 || m == 0) h[m++] = q;
    return m;
}
/* e + f -> h (h may not alias e or f); repeated grow-expansion (Shewchuk fig. 7): valid for any nonoverlapping inputs */
int expansion_sum(int ne, const double* e, int nf, const double* f, double* h)
{
    std::vector<double> tmp(e, e + ne), nxt((size_t)ne + nf + 1);
    int n = ne;
    for (int j = 0; j < nf; ++j) {
        n = grow_expansion(n, tmp.data(), f[j], nxt.data());
        tmp.assign(nxt.begin(), nxt.begin() + n);
        nxt.resize((size_t)n + nf + 1);
    }
    std::memcpy(h, tmp.data(), sizeof(double) * n);
    return n;
}
/* e * b -> h (up to 2n components), Shewchuk fig. 13 */
int scale_expansion(int n, const double* e, double b, double* h)
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
        /* fast-two-sum(t1, s) is valid here (|t1| >= |s| by construction), but two_sum is always valid */
        two_sum(t1, s, q, r);
        if (r != 0.0) h[m++] = r;
    }
    if (q != 0.0 || m == 0) h[m++] = q;
    return m;
}
/* x*y - z*w exactly, 4 components */
int prod_diff(double x, double y, double z, double w, double* h)
{
    double a1, a0, b1, b0;
    two_prod(x, y, a1, a0);
    two_prod(z, w, b1, b0);
    const double e[2] = { a0, a1 }, f[2] = { -b0, -b1 };
    return expansion_sum(2, e, 2, f, h);
}

/* exact sign of det [a-d; b-d; c-d] via the 4x4 cofactor expansion on the UNtranslated coordinates.  The four scaled terms are summed in
 * the device's order (adet + bdet, then every component of cdet and of ddet grown in); lens (nullable) receives the component counts the
 * device's fixed buffers must hold: cda, dab, abc, bcd, the longest pairwise sum before them, adet, bdet, cdet, ddet, the longest running
 * sum and the final sum (orc_orient3d_trace) */
int orient3d_exact(const double* pa, const double* pb, const double* pc, const double* pd, int* lens = nullptr)
{
    double ab[4], bc[4], cd[4], da[4], ac[4], bd[4];
    const int nab = prod_diff(pa[0], pb[1], pb[0], pa[1], ab), nbc = prod_diff(pb[0], pc[1], pc[0], pb[1], bc), ncd = prod_diff(pc[0], pd[1], pd[0], pc[1], cd);
    const int nda = prod_diff(pd[0], pa[1], pa[0], pd[1], da), nac = prod_diff(pa[0], pc[1], pc[0], pa[1], ac), nbd = prod_diff(pb[0], pd[1], pd[0], pb[1], bd);
    double t[16], cda[16], dab[16], abc[16], bcd[16], nac_[4], nbd_[4];
    for (int i = 0; i < nac; ++i) nac_[i] = -ac[i];
    for (int i = 0; i < nbd; ++i) nbd_[i] = -bd[i];
    int nt = expansion_sum(ncd, cd, nda, da, t), ntmax = nt;
    const int ncda = expansion_sum(nt, t, nac, ac, cda);
    nt = expansion_sum(nda, da, nab, ab, t), ntmax = std::max(ntmax, nt);
    const int ndab = expansion_sum(nt, t, nbd, bd, dab);
    nt = expansion_sum(nab, ab, nbc, bc, t), ntmax = std::max(ntmax, nt);
    const int nabc = expansion_sum(nt, t, nac, nac_, abc);
    nt = expansion_sum(nbc, bc, ncd, cd, t), ntmax = std::max(ntmax, nt);
    const int nbcd = expansion_sum(nt, t, nbd, nbd_, bcd);
    double adet[32], bdet[32], cdet[32], ddet[32], det[128], nxt[128];
    const int na = scale_expansion(nbcd, bcd, pa[2], adet), nb = scale_expansion(ncda, cda, -pb[2], bdet);
    const int nc = scale_expansion(ndab, dab, pc[2], cdet), nd = scale_expansion(nabc, abc, -pd[2], ddet);
    int n = expansion_sum(na, adet, nb, bdet, det), nmax = n;
    for (int j = 0; j < nc + nd; ++j) {
        n = grow_expansion(n, det, j < nc ? cdet[j] : ddet[j - nc], nxt);
        std::memcpy(det, nxt, sizeof(double) * n);
        nmax = std::max(nmax, n);
    }
    if (lens) {
        const int l[11] = { ncda, ndab, nabc, nbcd, ntmax, na, nb, nc, nd, nmax, n };
        std::memcpy(lens, l, sizeof(l));
    }
    const double top = det[n - 1]; /* the largest-magnitude component carries the sign */
    return (top > 0.0) - (top < 0.0);
}

/* the floating-point filter: +1 / -1 when it decides, 2 when the input goes to the exact stage */
int orient3d_filter(const double* pa, const double* pb, const double* pc, const double* pd)
{
    const double adx = pa[0] - pd[0], bdx = pb[0] - pd[0], cdx = pc[0] - pd[0];
    const double ady = pa[1] - pd[1], bdy = pb[1] - pd[1], cdy = pc[1] - pd[1];
    const double adz = pa[2] - pd[2], bdz = pb[2] - pd[2], cdz = pc[2] - pd[2];
    const double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy, cdxady = cdx * ady, adxcdy = adx * cdy, adxbdy = adx * bdy, bdxady = bdx * ady;
    const double det = adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy) + cdz * (adxbdy - bdxady);
    const double permanent = (std::fabs(bdxcdy) + std::fabs(cdxbdy)) * std::fabs(adz) + (std::fabs(cdxady) + std::fabs(adxcdy)) * std::fabs(bdz)
        + (std::fabs(adxbdy) + std::fabs(bdxady)) * std::fabs(cdz);
    /* Shewchuk's stage-A bound is (7 + 56 eps) eps * permanent with eps = 2^-53; a wider filter (16 eps) only sends more inputs to the
     * exact stage and keeps the argument independent of the evaluation order above */
    const double errbound = 1.7763568394002505e-15 * permanent;
    if (det > errbound) return 1;
    if (-det > errbound) return -1;
    return 2;
}

} // namespace

extern "C" {

/* sign (+1 / 0 / -1) of orient3d(pa, pb, pc, pd) in Shewchuk's convention (positive when pd lies below the plane pa pb pc) */
int orc_orient3d(const double* pa, const double* pb, const double* pc, const double* pd)
{
    const int f = orient3d_filter(pa, pb, pc, pd);
    return f != 2 ? f : orient3d_exact(pa, pb, pc, pd);
}
int orc_orient3d_exact(const double* pa, const double* pb, const double* pc, const double* pd) { return orient3d_exact(pa, pb, pc, pd); }
/* orc_orient3d with the path it took: info[0] = 1 when the filter decided (info[1..11] = 0), else 0 and info[1..11] the component counts of
 * the exact stage (cda, dab, abc, bcd, longest pairwise sum, adet, bdet, cdet, ddet, longest running sum, final sum) */
int orc_orient3d_trace(const double* pa, const double* pb, const double* pc, const double* pd, int* info)
{
    std::memset(info, 0, 12 * sizeof(int));
    const int f = orient3d_filter(pa, pb, pc, pd);
    if (f != 2) {
        info[0] = 1;
        return f;
    }
    return orient3d_exact(pa, pb, pc, pd, info + 1);
}

/* x = M^-1 b by Gaussian elimination with full pivoting (Eigen::FullPivLU order); M column-major 3x3.  returns the rank */
static int full_piv_solve3(const double* Mcm, const double* b, double* x)
{
    double m[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[i][j] = Mcm[3 * j + i];
    int rp[3] = { 0, 1, 2 }, cq[3] = { 0, 1, 2 };
    double rhs[3] = { b[0], b[1], b[2] };
    double maxpiv = 0.0;
    int nz = 3;
    for (int k = 0; k < 3; ++k) {
        int pr = k, pc = k;
        double big = -1.0;
        for (int j = k; j < 3; ++j)      /* column-major visit, first maximum wins */
            for (int i = k; i < 3; ++i)
                if (std::fabs(m[i][j]) > big) { big = std::fabs(m[i][j]); pr = i; pc = j; }
        if (big == 0.0) { nz = k; break; }
        maxpiv = std::max(maxpiv, big);
        if (pr != k) { for (int j = 0; j < 3; ++j) std::swap(m[k][j], m[pr][j]); std::swap(rhs[k], rhs[pr]); std::swap(rp[k], rp[pr]); }
        if (pc != k) { for (int i = 0; i < 3; ++i) std::swap(m[i][k], m[i][pc]); std::swap(cq[k], cq[pc]); }
        for (int i = k + 1; i < 3; ++i) m[i][k] /= m[k][k];
        for (int i = k + 1; i < 3; ++i)
            for (int j = k + 1; j < 3; ++j) m[i][j] -= m[i][k] * m[k][j];
    }
    /* rank with Eigen's default threshold: pivots <= eps * 3 * maxpivot count as zero */
    int rank = 0;
    for (int k = 0; k < nz; ++k)
        if (std::fabs(m[k][k]) > maxpiv * 2.220446049250313e-16 * 3.0) ++rank;
    /* both triangular solves by columns, as Eigen's triangular_solve_vector does for a column-major block (FullPivLU::_solve_impl passes
     * runtime-sized blocks, so nothing is unrolled): a solved entry is subtracted from every row above/below it at once, and an entry that is
     * exactly zero is skipped.  Row 0 of the back substitution thus rounds as (r0 - U02 y2) - U01 y1. */
    for (int j = 0; j < 3; ++j) /* forward: unit lower */
        if (rhs[j] != 0.0)
            for (int i = j + 1; i < 3; ++i) rhs[i] -= rhs[j] * m[i][j];
    for (int j = rank - 1; j >= 0; --j) /* back substitution on the leading rank x rank block */
        if (rhs[j] != 0.0) {
            rhs[j] /= m[j][j];
            for (int i = 0; i < j; ++i) rhs[i] -= rhs[j] * m[i][j];
        }
    x[0] = x[1] = x[2] = 0.0;
    for (int k = 0; k < rank; ++k) x[cq[k]] = rhs[k];
    return rank;
}

/* IglUtils::segTriIntersect (IglUtils.hpp:214-265, USE_PREDICATES) with the path it took: exit 0 = an endpoint in the triangle's plane,
 * 1 = both endpoints on one side, 2 = solved (rank and uvt filled; both nullable) */
int orc_seg_tri_trace(const double* ve0, const double* ve1, const double* vt0, const double* vt1, const double* vt2, int* exit, int* rank, double* uvt)
{
    const int o1 = orc_orient3d(vt0, vt1, vt2, ve0), o2 = orc_orient3d(vt0, vt1, vt2, ve1);
    *exit = (o1 == 0 || o2 == 0) ? 0 : (o1 == o2 ? 1 : 2);
    if (*exit != 2) return 0; /* coplanar: detected through d(EE) = 0 or d(PT) = 0 instead; or the edge is on one side of the plane */
    double M[9], b[3], x[3];
    for (int i = 0; i < 3; ++i) {
        M[i] = vt1[i] - vt0[i];
        M[3 + i] = vt2[i] - vt0[i];
        M[6 + i] = ve0[i] - ve1[i];
        b[i] = ve0[i] - vt0[i];
    }
    const int r = full_piv_solve3(M, b, x);
    if (rank) *rank = r;
    if (uvt) std::memcpy(uvt, x, sizeof(x));
    return (x[0] >= 0.0 && x[1] >= 0.0 && x[0] + x[1] <= 1.0 && x[2] >= 0.0 && x[2] <= 1.0) ? 1 : 0;
}
int orc_seg_tri_intersect(const double* ve0, const double* ve1, const double* vt0, const double* vt1, const double* vt2)
{
    int exit;
    return orc_seg_tri_trace(ve0, ve1, vt0, vt1, vt2, &exit, nullptr, nullptr);
}

/* SelfCollisionHandler::checkEdgeTriIntersectionIfAny (:3254-3296): 1 = intersection free.  The candidate edges of a triangle come from a
 * uniform grid over the edges' boxes (any superset of the truly intersecting pairs gives the same answer: a pair whose boxes are disjoint
 * cannot intersect).  hits (nullable) receives the number of intersected triangles (the reference stops at the first per triangle),
 * tri_flags (nullable) which ones. */
int orc_intersection_free(const orc_surf* s, double cell, int* hits, int* tri_flags /* nSF, nullable */, int nthreads)
{
    const int nV = s->nV;
    auto X = [&](int v, int c) { return s->V[(size_t)c * nV + v]; };
    double lo[3] = { 1e300, 1e300, 1e300 }, hi[3] = { -1e300, -1e300, -1e300 };
    for (int e = 0; e < 2 * s->nSE; ++e)
        for (int c = 0; c < 3; ++c) { lo[c] = std::min(lo[c], X(s->SE[e], c)); hi[c] = std::max(hi[c], X(s->SE[e], c)); }
    if (s->nSE == 0 || s->nSF == 0) { if (hits) *hits = 0; return 1; }
    if (!(cell > 0.0)) cell = 1.0;
    int n[3];
    for (int c = 0; c < 3; ++c) n[c] = std::max(1, std::min(512, (int)std::floor((hi[c] - lo[c]) / cell) + 1));
    double inv[3];
    for (int c = 0; c < 3; ++c) inv[c] = n[c] / std::max(hi[c] - lo[c], 1e-300) * (1.0 - 1e-12);
    auto cellc = [&](double x, int c) { return std::min(n[c] - 1, std::max(0, (int)std::floor((x - lo[c]) * inv[c]))); };
    const size_t ncell = (size_t)n[0] * n[1] * n[2];
    std::vector<int> start(ncell + 1, 0);
    auto erange = [&](int e, int* a, int* b) {
        for (int c = 0; c < 3; ++c) {
            const double x0 = X(s->SE[2 * e], c), x1 = X(s->SE[2 * e + 1], c);
            a[c] = cellc(std::min(x0, x1), c);
            b[c] = cellc(std::max(x0, x1), c);
        }
    };
    for (int e = 0; e < s->nSE; ++e) {
        int a[3], b[3];
        erange(e, a, b);
        for (int k = a[2]; k <= b[2]; ++k)
            for (int j = a[1]; j <= b[1]; ++j)
                for (int i = a[0]; i <= b[0]; ++i) ++start[((size_t)k * n[1] + j) * n[0] + i + 1];
    }
    for (size_t q = 0; q < ncell; ++q) start[q + 1] += start[q];
    std::vector<int> items(start[ncell]), cur(start.begin(), start.end() - 1);
    for (int e = 0; e < s->nSE; ++e) {
        int a[3], b[3];
        erange(e, a, b);
        for (int k = a[2]; k <= b[2]; ++k)
            for (int j = a[1]; j <= b[1]; ++j)
                for (int i = a[0]; i <= b[0]; ++i) items[cur[((size_t)k * n[1] + j) * n[0] + i]++] = e;
    }
    int total = 0;
#pragma omp parallel for schedule(dynamic, 256) num_threads(nthreads > 0 ? nthreads : 1) reduction(+ : total)
    for (int f = 0; f < s->nSF; ++f) {
        const int tv[3] = { s->SF[f], s->SF[(size_t)s->nSF + f], s->SF[(size_t)2 * s->nSF + f] };
        double t[3][3], tlo[3], thi[3];
        int a[3], b[3];
        for (int c = 0; c < 3; ++c) {
            for (int k = 0; k < 3; ++k) t[k][c] = X(tv[k], c);
            tlo[c] = std::min(t[0][c], std::min(t[1][c], t[2][c]));
            thi[c] = std::max(t[0][c], std::max(t[1][c], t[2][c]));
            a[c] = cellc(tlo[c], c);
            b[c] = cellc(thi[c], c);
        }
        const int cod_f = s->vCoDim ? s->vCoDim[tv[0]] : 3;
        bool hit = false;
        for (int k = a[2]; k <= b[2] && !hit; ++k)
            for (int j = a[1]; j <= b[1] && !hit; ++j)
                for (int i = a[0]; i <= b[0] && !hit; ++i) {
                    const size_t q = ((size_t)k * n[1] + j) * n[0] + i;
                    for (int it = start[q]; it < start[q + 1] && !hit; ++it) {
                        const int e = items[it], e0 = s->SE[2 * e], e1 = s->SE[2 * e + 1];
                        if (e0 == tv[0] || e0 == tv[1] || e0 == tv[2] || e1 == tv[0] || e1 == tv[1] || e1 == tv[2]) continue;
                        const int cod_e = s->vCoDim ? s->vCoDim[e0] : 3;
                        const bool alldbc = s->dbc && s->dbc[e0] && s->dbc[e1] && s->dbc[tv[0]] && s->dbc[tv[1]] && s->dbc[tv[2]];
                        if ((cod_f < 3 && cod_e < 3) || alldbc) continue;
                        const double p0[3] = { X(e0, 0), X(e0, 1), X(e0, 2) }, p1[3] = { X(e1, 0), X(e1, 1), X(e1, 2) };
                        bool sep = false;
                        for (int c = 0; c < 3; ++c) sep = sep || std::min(p0[c], p1[c]) > thi[c] || std::max(p0[c], p1[c]) < tlo[c];
                        if (sep) continue;
                        if (orc_seg_tri_intersect(p0, p1, t[0], t[1], t[2])) hit = true;
                    }
                }
        total += hit ? 1 : 0;
        if (tri_flags) tri_flags[f] = hit ? 1 : 0;
    }
    if (hits) *hits = total;
    return total == 0 ? 1 : 0;
}

/* Mesh::checkInversion(bool mute) (Mesh.cpp:745-763): number of tets with mu, lambda != 0 whose current edge matrix has det < 0 */
int orc_count_inverted(const orc_mesh* m)
{
    int cnt = 0;
    for (int t = 0; t < m->nT; ++t) {
        if (!(m->mu[t] != 0.0 && m->lam[t] != 0.0)) continue;
        int v[4];
        for (int k = 0; k < 4; ++k) v[k] = m->T[(size_t)k * m->nT + t];
        double e[3][3];
        for (int k = 0; k < 3; ++k)
            for (int c = 0; c < 3; ++c) e[k][c] = m->V[(size_t)c * m->nV + v[k + 1]] - m->V[(size_t)c * m->nV + v[0]];
        /* determinant of the matrix with COLUMNS e[0], e[1], e[2] (3x3 cofactor expansion along the first row, Eigen's formula for 3x3) */
        const double det = e[0][0] * (e[1][1] * e[2][2] - e[2][1] * e[1][2]) - e[1][0] * (e[0][1] * e[2][2] - e[2][1] * e[0][2]) + e[2][0] * (e[0][1] * e[1][2] - e[1][1] * e[0][2]);
        if (det < 0.0) ++cnt;
    }
    return cnt;
}
}
