"""Generates tests/golden/safeguard_regimes_golden.npz: a soup of disjoint stencils at the places where the line-search safeguards
(orient3d, segTriIntersect, pointInsideTetrahedron, checkInversion -- csrc/safeguard.cu, DESIGN 3.6) change their decision, with every
decision evaluated from the stored doubles alone.

Specification of each decision:
  exact      every orient3d sign (Fraction arithmetic on the stored doubles): both exits of segTriIntersect and all of
             pointInsideTetrahedron (with its inclusive box test), and the exact u, v, t of the segment-triangle system with their margin
             min(u, v, 1 - u - v, t, 1 - t)
  restated   the double arithmetic of the reference, in a fixed order without fused operations: Eigen 3.4's FullPivLU solve of
             segTriIntersect (pivot = first maximum in column-major order of the remaining corner, rank threshold 3 eps * max pivot, both
             triangular solves by columns with exactly zero entries skipped, as triangular_solve_vector runs them on the runtime-sized
             blocks _solve_impl passes), and the 3x3 determinant of checkInversion (Mesh.cpp:745-763)
  recorded   the same solve with a row-oriented back substitution (s = r0; s -= U01 y1; s -= U02 y2), and the exact sign of each
             inversion determinant where the double sign differs from it

Stencils (each kind has its own families, FAMILIES):
  orient  points a, b, c, d: the query orient3d(a, b, c, d).  On the device it is read through two tets, (a, c, b, p+) and (a, b, c, p-)
          with apexes on either side of the plane, and d as a codimension-0 point: pointInsideTetrahedron's first orientation is
          orient3d(a, b, c, d) for the first tet and its negative for the second.  o_pit holds both exact outcomes.
  segtri  an edge e0 e1 and a triangle t0 t1 t2 (one surface triangle, one surface edge).
  pit     a tet and several codimension-0 points.
  inv     one tet (checkInversion).
Placement: stencils are sorted by their extent and laid along x with gaps of their extent, so that no two boxes meet and no stencil sits
at a coordinate large against its own size (offset families add their offset in y and z).  Exactly-zero families use dyadic data that
the placement translates exactly.  Scales stay within 1e-8 ... 1e8: the expansion arithmetic, like Shewchuk's, is exact only where no
product underflows.
Run:  python tests/golden/gen_safeguard_regimes_golden.py
"""
import math
import os
from fractions import Fraction as Fr

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "safeguard_regimes_golden.npz")
SEED = 20261017
EPS = 2.0 ** -52
FAMILIES = {
    "orient": ("generic", "coplanar_dyadic", "ulp_off", "near_coplanar", "offset", "scale", "degenerate", "long_expansion"),
    "segtri": ("interior", "through_edge", "through_vertex", "boundary_ulp", "endpoint_in_plane", "endpoint_ulp", "coplanar_segment",
               "near_parallel", "sliver", "box_touch", "order_sensitive"),
    "pit": ("dyadic_boundary", "manybit_boundary", "inverted_flat", "small_offset", "box_boundary", "grid_coplanar", "grid_single",
            "grid_duplicate"),
    "inv": ("zero", "signed_zero", "one_ulp", "near_flat_offset"),
}
# pit families the tests also run as a scene of their own (the point grid of k_pit_grid sees only their points)
ALONE = ("grid_coplanar", "grid_single", "grid_duplicate")


# ---- exact and restated arithmetic --------------------------------------------------------------------------------------------------
def orient_exact(a, b, c, d):
    ad, bd, cd = ([Fr(float(x)) - Fr(float(y)) for x, y in zip(p, d)] for p in (a, b, c))
    det = ad[2] * (bd[0] * cd[1] - cd[0] * bd[1]) + bd[2] * (cd[0] * ad[1] - ad[0] * cd[1]) + cd[2] * (ad[0] * bd[1] - bd[0] * ad[1])
    return (det > 0) - (det < 0)


def orient_filter(a, b, c, d):
    """the floating-point filter of the device and the oracle: +1 / -1 decided, 2 undecided"""
    a, b, c, d = ([float(x) for x in p] for p in (a, b, c, d))
    adx, bdx, cdx = a[0] - d[0], b[0] - d[0], c[0] - d[0]
    ady, bdy, cdy = a[1] - d[1], b[1] - d[1], c[1] - d[1]
    adz, bdz, cdz = a[2] - d[2], b[2] - d[2], c[2] - d[2]
    bdxcdy, cdxbdy, cdxady, adxcdy, adxbdy, bdxady = bdx * cdy, cdx * bdy, cdx * ady, adx * cdy, adx * bdy, bdx * ady
    det = adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy) + cdz * (adxbdy - bdxady)
    perm = (abs(bdxcdy) + abs(cdxbdy)) * abs(adz) + (abs(cdxady) + abs(adxcdy)) * abs(bdz) + (abs(adxbdy) + abs(bdxady)) * abs(cdz)
    err = 1.7763568394002505e-15 * perm
    return 1 if det > err else (-1 if -det > err else 2)


def point_in_tet_exact(p, t):
    """IglUtils::pointInsideTetrahedron after the inclusive box test of the check"""
    t = np.asarray(t)
    if np.any(p < t.min(0)) or np.any(p > t.max(0)):
        return 0
    return int(orient_exact(t[0], t[2], t[1], p) >= 0 and orient_exact(t[0], t[3], t[2], p) >= 0 and orient_exact(t[0], t[1], t[3], p) >= 0
               and orient_exact(t[1], t[2], t[3], p) >= 0)


def full_piv_lu_solve(Mrows, b, row_order=False):
    """Eigen 3.4 FullPivLU<Matrix3d>::solve in IEEE doubles (Python floats: no fused operations); returns (x, rank)"""
    m = [[float(x) for x in r] for r in Mrows]
    r = [float(x) for x in b]
    cq, maxpiv, nz = [0, 1, 2], 0.0, 3
    for k in range(3):
        big, pr, pc = -1.0, k, k
        for j in range(k, 3):
            for i in range(k, 3):
                if abs(m[i][j]) > big:
                    big, pr, pc = abs(m[i][j]), i, j
        if big == 0.0:
            nz = k
            break
        maxpiv = max(maxpiv, big)
        m[k], m[pr] = m[pr], m[k]
        r[k], r[pr] = r[pr], r[k]
        for row in m:
            row[k], row[pc] = row[pc], row[k]
        cq[k], cq[pc] = cq[pc], cq[k]
        for i in range(k + 1, 3):
            m[i][k] = m[i][k] / m[k][k]
        for i in range(k + 1, 3):
            for j in range(k + 1, 3):
                m[i][j] = m[i][j] - m[i][k] * m[k][j]
    rank = sum(1 for k in range(nz) if abs(m[k][k]) > maxpiv * 2.220446049250313e-16 * 3.0)
    for j in range(3):  # unit lower, by columns (every order rounds the same here)
        if r[j] != 0.0:
            for i in range(j + 1, 3):
                r[i] = r[i] - r[j] * m[i][j]
    if row_order:
        y = [0.0, 0.0, 0.0]
        for i in range(rank - 1, -1, -1):
            s = r[i]
            for j in range(i + 1, rank):
                s = s - m[i][j] * y[j]
            y[i] = s / m[i][i]
        r = y
    else:
        for j in range(rank - 1, -1, -1):
            if r[j] != 0.0:
                r[j] = r[j] / m[j][j]
                for i in range(j):
                    r[i] = r[i] - r[j] * m[i][j]
    x = [0.0, 0.0, 0.0]
    for k in range(rank):
        x[cq[k]] = r[k]
    return x, rank


def seg_tri_system(e0, e1, t0, t1, t2):
    M = [[t1[i] - t0[i], t2[i] - t0[i], e0[i] - e1[i]] for i in range(3)]
    return M, [e0[i] - t0[i] for i in range(3)]


def accept(x):
    return x[0] >= 0.0 and x[1] >= 0.0 and x[0] + x[1] <= 1.0 and x[2] >= 0.0 and x[2] <= 1.0


def seg_tri(e0, e1, t0, t1, t2):
    """exact exit (0 an endpoint in the plane, 1 one side, 2 crossing) and everything the fixture stores about the solve"""
    o1, o2 = orient_exact(t0, t1, t2, e0), orient_exact(t0, t1, t2, e1)
    ex = 0 if (o1 == 0 or o2 == 0) else (1 if o1 == o2 else 2)
    out = dict(exit=ex, rank=-1, uvt=[np.nan] * 3, dec=0, dec_row=0, dec_exact=0, margin=np.nan, band=np.nan)
    if ex != 2:
        return out
    M, b = seg_tri_system([float(x) for x in e0], [float(x) for x in e1], [float(x) for x in t0], [float(x) for x in t1], [float(x) for x in t2])
    x, rank = full_piv_lu_solve(M, b)
    xr, _ = full_piv_lu_solve(M, b, row_order=True)
    # exact u, v, t (the exact system is regular: the edge crosses the plane of a nondegenerate triangle)
    Me = [[Fr(v) for v in row] for row in M]
    be = [Fr(v) for v in b]

    def det3(A):
        return (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
                + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]))

    D = det3(Me)
    xe = []
    for k in range(3):
        A = [row[:] for row in Me]
        for i in range(3):
            A[i][k] = be[i]
        xe.append(det3(A) / D)
    margin = min(xe[0], xe[1], 1 - xe[0] - xe[1], xe[2], 1 - xe[2])
    Mf = np.array(M)
    inv = np.linalg.inv(Mf) if np.linalg.cond(Mf) < 1e300 else np.full((3, 3), np.inf)
    nrm = lambda A: float(np.max(np.sum(np.abs(A), axis=-1))) if np.ndim(A) == 2 else float(np.max(np.abs(A)))
    band = 64.0 * EPS * nrm(inv) * (nrm(Mf) * nrm(np.array([float(v) for v in xe])) + nrm(np.array(b)))
    out.update(rank=rank, uvt=x, dec=int(accept(x)), dec_row=int(accept(xr)), dec_exact=int(margin >= 0), margin=float(margin), band=band)
    return out


def inv_det_double(t):
    """Mesh::checkInversion's determinant of the edge matrix with columns e0, e1, e2, in IEEE doubles"""
    e = [[float(t[k + 1][c]) - float(t[0][c]) for c in range(3)] for k in range(3)]
    return e[0][0] * (e[1][1] * e[2][2] - e[2][1] * e[1][2]) - e[1][0] * (e[0][1] * e[2][2] - e[2][1] * e[0][2]) + e[2][0] * (e[0][1] * e[1][2] - e[1][1] * e[0][2])


def inv_det_sign_exact(t):
    e = [[Fr(float(t[k + 1][c])) - Fr(float(t[0][c])) for c in range(3)] for k in range(3)]
    d = e[0][0] * (e[1][1] * e[2][2] - e[2][1] * e[1][2]) - e[1][0] * (e[0][1] * e[2][2] - e[2][1] * e[0][2]) + e[2][0] * (e[0][1] * e[1][2] - e[1][1] * e[0][2])
    return (d > 0) - (d < 0)


# ---- stencil builders: f(rng, c) -> points, c the stencil's centre (an exactly representable dyadic point) -------------------------------
def dy(rng, n, den=64, lim=1.0):
    """dyadic numbers k / den in [-lim, lim]"""
    return rng.integers(-int(lim * den), int(lim * den) + 1, size=n) / den


def ulp(x, ax, up):
    """x with coordinate ax (or the next nonzero one: a step off 0 would be subnormal, where the expansion arithmetic is not exact) moved by
    one ulp"""
    x = x.copy()
    while x[ax] == 0:
        ax = (ax + 1) % 3
    x[ax] = np.nextafter(x[ax], np.inf if up else -np.inf)
    return x


def unit(rng):
    v = rng.standard_normal(3)
    return v / np.linalg.norm(v)


def tri_in_plane(rng, c, s):
    """a well-shaped triangle of size s around c with full-mantissa coordinates"""
    return [c + s * rng.uniform(-1, 1, 3) for _ in range(3)]


def normal(a, b, c):
    n = np.cross(b - a, c - a)
    return n / np.linalg.norm(n)


def orient_stencil(a, b, c, d, s):
    """(a, b, c, d) plus apexes p+ / p- well off the plane on the positive / negative side of orient3d(a, b, c, .)"""
    cen = (a + b + c) / 3.0
    n = np.cross(b - a, c - a)
    nn = np.linalg.norm(n)
    n = n / nn if nn > 0 else np.array([0.0, 0.0, 1.0])
    pp, pm = cen + s * n, cen - s * n
    if orient_exact(a, b, c, pp) < 0:
        pp, pm = pm, pp
    return np.array([a, b, c, d, pp, pm])


def build():
    rng0 = np.random.default_rng(SEED)
    specs = []  # (kind, family, extent, offset, builder)

    def add(kind, fam, extent, fn, offset=0.0):
        specs.append((kind, FAMILIES[kind].index(fam), float(extent), float(offset), fn, int(rng0.integers(2 ** 62))))

    # -- orientation families ------------------------------------------------------------------------------------------------------
    for _ in range(12):
        def f(rng, c):
            a, b, cc = tri_in_plane(rng, c, 1.0)
            d = (a + b + cc) / 3 + 0.3 * rng.standard_normal(3)
            return orient_stencil(a, b, cc, d, 1.0)
        add("orient", "generic", 4.0, f)
    for k in range(24):
        def f(rng, c):
            while True:
                a, b, cc = (c + dy(rng, 3, 16) for _ in range(3))
                if orient_exact(a, b, cc, c + np.array([0.1, 0.2, 0.3])) != 0 or orient_exact(a, b, cc, c + np.array([0.3, -0.1, 0.7])) != 0:
                    break
            u, v = rng.integers(1, 4, 2) / 8.0
            d = a + u * (b - a) + v * (cc - a)
            assert orient_exact(a, b, cc, d) == 0
            return orient_stencil(a, b, cc, d, 1.0)
        add("orient", "coplanar_dyadic", 4.0, f)
    for k in range(24):
        def f(rng, c, k=k):
            while True:
                a, b, cc = (c + dy(rng, 3, 16) for _ in range(3))
                if np.linalg.norm(np.cross(b - a, cc - a)) > 0.3:
                    break
            d = a + 0.25 * (b - a) + 0.375 * (cc - a)
            ax, sgn = k % 3, (1 if (k // 3) % 2 == 0 else -1)
            d = ulp(d, ax, sgn > 0)
            return orient_stencil(a, b, cc, d, 1.0)
        add("orient", "ulp_off", 4.0, f)

    def near_coplanar(s, need_undecided=True):
        def f(rng, c):
            for _ in range(200):  # (where the offset's rounding moves d off the plane by more than the filter's bound, the last try is kept)
                a, b, cc = tri_in_plane(rng, c, s)
                u, v = rng.uniform(0.2, 0.4, 2)
                d = a + u * (b - a) + v * (cc - a)
                if not need_undecided or (orient_filter(a, b, cc, d) == 2 and orient_exact(a, b, cc, d) != 0):
                    break
            return orient_stencil(a, b, cc, d, s)
        return f
    for _ in range(30):
        add("orient", "near_coplanar", 4.0, near_coplanar(1.0))
    for k in range(30):
        s, off = 10.0 ** (-3 + 3 * (k % 5) / 4), 10.0 ** (3 + (k // 5) % 4)
        add("orient", "offset", 4 * s, near_coplanar(s), offset=off)
    for k in range(30):
        s = 10.0 ** (-8 + 16 * (k % 10) / 9)
        add("orient", "scale", 4 * s, near_coplanar(s))
    for k in range(12):
        def f(rng, c, k=k):
            a, b, cc = (c + dy(rng, 3, 16) for _ in range(3))
            if k % 3 == 0:
                b = a.copy()                      # repeated point
            elif k % 3 == 1:
                cc = a + 0.5 * (b - a)            # collinear (exact: dyadic)
            else:
                b, cc = a.copy(), a.copy()        # all three equal
            d = c + dy(rng, 3, 16)
            if k % 2:
                d = a.copy()
            return orient_stencil(a, b, cc, d, 1.0)
        add("orient", "degenerate", 4.0, f)

    def long_expansion(rng, c):
        """coordinates whose mantissa bits are spread over many exponents, d in the plane up to rounding: the exact stage runs with long
        expansions"""
        best, bl = None, -1
        for _ in range(40):
            pts = []
            for _ in range(3):
                p = c + np.array([rng.uniform(0.5, 1) * 2.0 ** rng.integers(-1, 1) + rng.uniform(-1, 1) * 2.0 ** rng.integers(-40, -20)
                                  for _ in range(3)]) * rng.choice([-1, 1], 3)
                pts.append(p)
            a, b, cc = pts
            u, v = rng.uniform(0.2, 0.4, 2)
            d = a + u * (b - a) + v * (cc - a)
            d = d + np.array([rng.uniform(-1, 1) * 2.0 ** rng.integers(-60, -50) for _ in range(3)])
            if best is None:
                best = orient_stencil(a, b, cc, d, 1.0)
            if orient_filter(a, b, cc, d) != 2:
                continue
            bits = sum(len(set(np.frexp(np.array(p))[1])) for p in (a, b, cc, d))
            if bits > bl:
                best, bl = orient_stencil(a, b, cc, d, 1.0), bits
        return best
    for _ in range(24):
        add("orient", "long_expansion", 6.0, long_expansion)

    # -- segTriIntersect families ----------------------------------------------------------------------------------------------------
    for k in range(8):
        def f(rng, c, k=k):
            t = tri_in_plane(rng, c, 1.0)
            n = normal(*t)
            u, v = rng.uniform(0.2, 0.35, 2) if k < 6 else rng.uniform(0.6, 0.8, 2)  # 6 hits, 2 misses
            p = t[0] + u * (t[1] - t[0]) + v * (t[2] - t[0])
            w = n + 0.3 * unit(rng)
            return np.array([p - 0.7 * w, p + 0.9 * w, *t])
        add("segtri", "interior", 6.0, f)

    def through(kind_pt):
        def f(rng, c):
            while True:
                t = [c + dy(rng, 3, 8) for _ in range(3)]
                if np.linalg.norm(np.cross(t[1] - t[0], t[2] - t[0])) > 0.4:
                    break
            s = rng.integers(1, 8) / 8.0
            if kind_pt == "edge":
                which = rng.integers(3)   # u = 0, v = 0 or u + v = 1 exactly
                p = [t[0] + s * (t[2] - t[0]), t[0] + s * (t[1] - t[0]), t[1] + s * (t[2] - t[1])][which]
            else:
                p = t[rng.integers(3)].copy()
            w = unit(rng)   # full-mantissa direction: the solve rounds
            if abs(w @ normal(*t)) < 0.2:
                w = w + normal(*t)
            l0, l1 = rng.uniform(0.3, 1.0, 2)
            return np.array([p - l0 * w, p + l1 * w, *t])
        return f
    for _ in range(60):
        add("segtri", "through_edge", 8.0, through("edge"))
    for _ in range(40):
        add("segtri", "through_vertex", 8.0, through("vertex"))
    for k in range(40):
        def f(rng, c, k=k):
            st = through("edge" if k % 2 else "vertex")(rng, c)
            i, ax = 2 + rng.integers(3), rng.integers(3)   # one ulp inside or outside: a triangle vertex moves
            st[i] = ulp(st[i], ax, k % 4 < 2)
            return st
        add("segtri", "boundary_ulp", 8.0, f)
    for k in range(12):
        def f(rng, c, k=k):
            while True:
                t = [c + dy(rng, 3, 8) for _ in range(3)]
                if np.linalg.norm(np.cross(t[1] - t[0], t[2] - t[0])) > 0.4:
                    break
            u, v = (rng.integers(1, 3, 2) / 8.0) if k % 2 == 0 else (rng.integers(5, 8, 2) / 8.0)
            p = t[0] + u * (t[1] - t[0]) + v * (t[2] - t[0])   # exactly in the plane (inside the triangle or not)
            q = p + normal(*t) * (1 if k % 4 < 2 else -1) * 0.75
            return np.array([p, q, *t] if k % 3 else [q, p, *t])
        add("segtri", "endpoint_in_plane", 8.0, f)
    for k in range(24):
        def f(rng, c, k=k):
            while True:
                t = [c + dy(rng, 3, 8) for _ in range(3)]
                if np.linalg.norm(np.cross(t[1] - t[0], t[2] - t[0])) > 0.4:
                    break
            u, v = rng.integers(1, 3, 2) / 8.0
            p = t[0] + u * (t[1] - t[0]) + v * (t[2] - t[0])
            q = p + normal(*t) * (1 if k % 2 else -1) * rng.uniform(0.5, 1.0)
            ax = rng.integers(3)
            p = ulp(p, ax, k % 4 < 2)   # exact t about 0 (or 1 below)
            return np.array([p, q, *t] if k % 8 < 4 else [q, p, *t])
        add("segtri", "endpoint_ulp", 8.0, f)
    for k in range(6):
        def f(rng, c, k=k):
            t = [c + dy(rng, 3, 8) for _ in range(3)]
            u0, v0, u1, v1 = rng.integers(-2, 9, 4) / 8.0
            p, q = t[0] + u0 * (t[1] - t[0]) + v0 * (t[2] - t[0]), t[0] + u1 * (t[1] - t[0]) + v1 * (t[2] - t[0])
            return np.array([p, q, *t])
        add("segtri", "coplanar_segment", 12.0, f)
    for k in range(28):
        def f(rng, c, k=k):
            r = 10.0 ** (-2 - 16 * (k % 14) / 13)          # normal component over length: 1e-2 ... 1e-18 (rank 2 below ~3e-16)
            if k < 14:                                     # plane z = const: the endpoints' heights are exact
                t = [c + np.array([*rng.uniform(-1, 1, 2), 0.0]) for _ in range(3)]
                n = np.array([0.0, 0.0, 1.0])
            else:
                t = tri_in_plane(rng, c, 1.0)
                n = normal(*t)
            cen = (t[0] + t[1] + t[2]) / 3.0
            w = np.cross(n, unit(rng))
            w = w / np.linalg.norm(w)
            p = cen + 0.1 * rng.uniform(-1, 1) * w
            return np.array([p - w + r * n, p + w - r * n, *t])
        add("segtri", "near_parallel", 6.0, f)
    for k in range(16):
        def f(rng, c, k=k):
            asp = 10.0 ** (-1 - 7 * (k % 8) / 7)           # aspect 1e-1 ... 1e-8
            L = unit(rng)
            h = np.cross(L, unit(rng))
            h = h / np.linalg.norm(h)
            t = [c - L, c + L, c + rng.uniform(-0.5, 0.5) * L + asp * h]
            n = normal(*t)
            s = rng.uniform(0.1, 0.9) * asp if k < 8 else (-1 if k % 2 else 1) * rng.uniform(0, 1) * asp * 1e-3
            p = c + rng.uniform(-0.3, 0.3) * L + s * h
            return np.array([p - 0.5 * n, p + 0.5 * n, *t])
        add("segtri", "sliver", 6.0, f)
    for k in range(8):
        def f(rng, c, k=k):
            t = [c + np.array(v) for v in ([0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.5, 0.0])]
            if k % 2 == 0:   # the edge's box is the plane x = 1 of the triangle's box: through the vertex (1, 0, 0)
                e0, e1 = c + np.array([1.0, -0.25, -0.5]), c + np.array([1.0, 0.25, 0.5])
            else:            # through the point (0.5, 0.25, 0) of the edge t1 t2, box face y = 0.5 touched from above
                e0, e1 = c + np.array([0.375, 0.5, -0.5]), c + np.array([0.625, 0.0, 0.5])
            if k >= 4:       # corner touch: the boxes share only the edge x = 1, y = 0.5 (z = 0) of the triangle's box; no intersection
                e0, e1 = c + np.array([1.0, 0.5, 2.0 ** -40 if k % 2 else -0.5]), c + np.array([1.5, 1.0, 1.0 if k % 2 else 0.0])
            return np.array([e0, e1, *t])
        add("segtri", "box_touch", 6.0, f)

    for _ in range(16):
        def f(rng, c):
            """full-mantissa triangle, an edge through a rounded point of a triangle edge or a vertex, kept where the row-oriented back
            substitution decides otherwise than Eigen's column order"""
            for _ in range(5000):
                t = [c + rng.uniform(-1, 1, 3) for _ in range(3)]
                sp = rng.uniform(0, 1)
                p = [t[0] + sp * (t[2] - t[0]), t[0] + sp * (t[1] - t[0]), t[1] + sp * (t[2] - t[1]), t[0], t[1], t[2]][rng.integers(6)]
                w = rng.standard_normal(3)
                e0, e1 = p - rng.uniform(0.3, 1) * w, p + rng.uniform(0.3, 1) * w
                M, b = seg_tri_system(e0, e1, *t)
                if accept(full_piv_lu_solve(M, b)[0]) != accept(full_piv_lu_solve(M, b, row_order=True)[0]):
                    break
            return np.array([e0, e1, *t])
        add("segtri", "order_sensitive", 8.0, f)

    # -- pointInsideTetrahedron families ----------------------------------------------------------------------------------------------
    def tet_points_boundary(t, rng, dyadic):
        """vertices, edge points, face points (exact for dyadic data, rounded otherwise), one ulp in and out, an interior point"""
        q = [t[rng.integers(4)].copy()]
        i, j = rng.choice(4, 2, replace=False)
        q.append(t[i] + 0.5 * (t[j] - t[i]) if dyadic else t[i] + rng.uniform(0.1, 0.9) * (t[j] - t[i]))
        i, j, k = rng.choice(4, 3, replace=False)
        fp = t[i] + 0.25 * (t[j] - t[i]) + 0.5 * (t[k] - t[i]) if dyadic else t[i] + rng.uniform(0.1, 0.4) * (t[j] - t[i]) + rng.uniform(0.1, 0.4) * (t[k] - t[i])
        q.append(fp)
        for sgn in (1, -1):
            q.append(ulp(fp, rng.integers(3), sgn > 0))
        q.append(t.mean(0))
        return np.array(q)

    def good_tet(rng, c, s, dyadic):
        while True:
            t = np.array([c + (dy(rng, 3, 8) * s if dyadic else s * rng.uniform(-1, 1, 3)) for _ in range(4)])
            if abs(np.linalg.det(t[1:] - t[0])) > 0.05 * s ** 3:
                if orient_exact(t[0], t[2], t[1], t[3]) < 0:
                    t[[1, 2]] = t[[2, 1]]
                return t
    for _ in range(16):
        def f(rng, c):
            t = good_tet(rng, c, 1.0, True)
            return t, tet_points_boundary(t, rng, True)
        add("pit", "dyadic_boundary", 4.0, f)
    for _ in range(16):
        def f(rng, c):
            t = good_tet(rng, c, 1.0, False)
            return t, tet_points_boundary(t, rng, False)
        add("pit", "manybit_boundary", 4.0, f)
    for k in range(8):
        def f(rng, c, k=k):
            t = good_tet(rng, c, 1.0, True)
            if k % 2:
                t[[1, 2]] = t[[2, 1]]            # inverted: no interior point is inside
            else:
                t[3] = t[0] + 0.5 * (t[1] - t[0]) + 0.25 * (t[2] - t[0])   # flat: points of the plane within the box may pass
            q = tet_points_boundary(t, rng, True)
            return t, np.concatenate([q, [t[0] + 0.25 * (t[1] - t[0]) + 0.25 * (t[2] - t[0])]])
        add("pit", "inverted_flat", 4.0, f)
    for k in range(12):
        s, off = 1e-6 * (1 + k % 3), [0.0, 1.0, 1e3][k % 3 if k < 9 else 2]
        def f(rng, c, s=s):
            t = good_tet(rng, c, s, False)
            return t, tet_points_boundary(t, rng, False)
        add("pit", "small_offset", 4e-6 * (1 + k % 3), f, offset=off)
    for k in range(8):
        def f(rng, c, k=k):
            t = np.array([c, c + [1.0, 0, 0], c + [0, 1.0, 0], c + [0, 0, 1.0]])   # axis-aligned faces lie in the box's faces
            q = [c + [0.25, 0.25, 0.0], c + [0.0, 0.5, 0.25], c + [1.0, 1.0, 0.0], c + [1.0, 1.0, 1.0], c + [0.5, 0.5, 0.0],
                 c + [0.5, 0.5, 2.0 ** -30], c + [-0.0, 0.0, 0.0] + [0.0, 0.0, -(2.0 ** -30)], c + [0.25, 0.25, 0.5]]
            return t, np.array(q)
        add("pit", "box_boundary", 4.0, f)
    for k in range(6):   # every point of this family has the same z: the point grid has zero extent on z when run alone
        def f(rng, c, k=k):
            t = good_tet(rng, c, 1.0, True)
            zc = c[2]
            q = [np.array([*(c[:2] + dy(rng, 2, 8, 0.75)), zc]) for _ in range(5)]
            return t, np.array(q)
        add("pit", "grid_coplanar", 4.0, f)
    def f_single(rng, c):
        t = good_tet(rng, c, 1.0, True)
        return t, np.array([t[0] + 0.25 * (t[1] - t[0]) + 0.5 * (t[2] - t[0])])   # exactly on a face
    add("pit", "grid_single", 4.0, f_single)
    for k in range(4):
        def f(rng, c):
            t = good_tet(rng, c, 1.0, True)
            p = t[0] + 0.25 * (t[1] - t[0]) + 0.25 * (t[2] - t[0]) + 0.25 * (t[3] - t[0])
            return t, np.array([p, p, p, t[1], t[1]])
        add("pit", "grid_duplicate", 4.0, f)

    # -- inversion families ------------------------------------------------------------------------------------------------------------
    for k in range(8):
        def f(rng, c, k=k):
            a, b, cc = (c + dy(rng, 3, 8) for _ in range(3))
            d = a + 0.5 * (b - a) + 0.25 * (cc - a) if k % 2 else a + 0.75 * (b - a)
            return np.array([a, b, cc, d])
        add("inv", "zero", 4.0, f)
    for k in range(4):
        def f(rng, c, k=k):
            # flat tets in z = 0 with signed zeros: e_z = -0.0 - 0.0 = -0.0 and the cofactor terms are signed zeros.  With e00, e20 < 0 the
            # double determinant is -0.0, otherwise +0.0 (y and z are set literally: adding a centre would turn -0.0 into +0.0)
            sx = -1.0 if k % 2 == 0 else 1.0
            t = np.array([[0.0, 0.0, 0.0], [sx, 0.0, -0.0], [0.0, 1.0, -0.0], [0.5 * sx, 0.5, -0.0]])
            t[:, 0] = t[:, 0] + c[0]
            want = np.copysign(0.0, sx)
            assert inv_det_double(t) == 0 and np.signbit(inv_det_double(t)) == np.signbit(want)
            return t
        add("inv", "signed_zero", 4.0, f)
    for k in range(8):
        def f(rng, c, k=k):
            h = (1 if k % 2 else -1) * 2.0 ** -(40 + 2 * (k // 2))
            t = np.array([c, c + [1.0, 0, 0], c + [0, 1.0, 0], c + [0.25, 0.25, h]])
            return t
        add("inv", "one_ulp", 4.0, f)
    for k in range(24):
        off = 10.0 ** (3 + k % 4)
        def f(rng, c):
            while True:
                a, b, cc = tri_in_plane(rng, c, 1e-3)
                u, v = rng.uniform(0.2, 0.4, 2)
                d = a + u * (b - a) + v * (cc - a)
                t = np.array([a, b, cc, d])
                dd = inv_det_double(t)
                if (dd > 0) - (dd < 0) != inv_det_sign_exact(t) or rng.random() < 0.3:
                    return t
        add("inv", "near_flat_offset", 4e-3, f, offset=off)

    # -- placement ---------------------------------------------------------------------------------------------------------------------
    order = sorted(range(len(specs)), key=lambda s: specs[s][2])
    cursor = 0.0
    placed = [None] * len(specs)
    for s in order:
        kind, fam, ext, off, fn, seed = specs[s]
        q = 2.0 ** math.ceil(math.log2(ext))
        cx = math.ceil((cursor + 1.5 * ext) / q) * q
        cursor = cx + 1.5 * ext
        placed[s] = fn(np.random.default_rng(seed), np.array([cx, off, off]))
    return specs, placed


def evaluate(specs, placed):
    out = {}
    for kind in FAMILIES:
        idx = [s for s in range(len(specs)) if specs[s][0] == kind]
        out[f"{kind}_family"] = np.array([specs[s][1] for s in idx], np.int32)
        if kind == "orient":
            P = np.array([placed[s] for s in idx])
            out["orient_pts"] = P
            out["orient_sign"] = np.array([orient_exact(*p[:4]) for p in P], np.int32)
            out["orient_filter"] = np.array([orient_filter(*p[:4]) for p in P], np.int32)
            out["orient_pit"] = np.array([[point_in_tet_exact(p[3], [p[0], p[2], p[1], p[4]]), point_in_tet_exact(p[3], [p[0], p[1], p[2], p[5]])]
                                          for p in P], np.int32)
        elif kind == "segtri":
            P = np.array([placed[s] for s in idx])
            out["segtri_pts"] = P
            r = [seg_tri(*p) for p in P]
            for key in ("exit", "rank", "dec", "dec_row", "dec_exact"):
                out[f"segtri_{key}"] = np.array([x[key] for x in r], np.int32)
            for key in ("uvt", "margin", "band"):
                out[f"segtri_{key}"] = np.array([x[key] for x in r], np.float64)
        elif kind == "pit":
            out["pit_tets"] = np.array([placed[s][0] for s in idx])
            q = [placed[s][1] for s in idx]
            out["pit_pts"] = np.concatenate(q)
            out["pit_owner"] = np.concatenate([np.full(len(x), k, np.int32) for k, x in enumerate(q)])
            out["pit_in"] = np.array([point_in_tet_exact(p, out["pit_tets"][o]) for p, o in zip(out["pit_pts"], out["pit_owner"])], np.int32)
        else:
            T = np.array([placed[s] for s in idx])
            out["inv_tets"] = T
            out["inv_det"] = np.array([inv_det_double(t) for t in T])
            out["inv_sign_exact"] = np.array([inv_det_sign_exact(t) for t in T], np.int32)
    return out


def main():
    specs, placed = build()
    out = evaluate(specs, placed)
    np.savez_compressed(OUT, **out)
    st = out
    print("orient", len(st["orient_family"]), "undecided", int((st["orient_filter"] == 2).sum()), "zero", int((st["orient_sign"] == 0).sum()))
    print("segtri", len(st["segtri_family"]), "exits", np.bincount(st["segtri_exit"]).tolist(), "rank2", int((st["segtri_rank"] == 2).sum()),
          "row/col order decisions differ", int((st["segtri_dec"] != st["segtri_dec_row"]).sum()),
          "double vs exact differ", int((st["segtri_dec"] != st["segtri_dec_exact"]).sum()))
    print("pit", len(st["pit_family"]), "points", len(st["pit_pts"]), "inside", int(st["pit_in"].sum()))
    print("inv", len(st["inv_family"]), "double sign != exact", int((np.sign(st["inv_det"]) != st["inv_sign_exact"]).sum()))


if __name__ == "__main__":
    main()
