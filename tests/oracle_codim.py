"""Test helpers for codimensional scenes: the oracle's point-in-tetrahedron count, its exact-rational restatement, and scenes modelled on
the reference's codimensional examples (17_pinCushionBall, 18_pointRollerBall / 18_segRollerBall, coDimUnitTests/*PlaneDrop)."""
import os
from fractions import Fraction

import numpy as np
from scipy.spatial import cKDTree

import oracle as orc
from ipc_b200 import codim, mesh as M
from ipc_b200.scenes import shape_transform

MESHES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "meshes")


def points_in_tets(V, T, pts, nthreads=1):
    """Second half of SelfCollisionHandler::checkEdgeTriIntersectionIfAny (:3301-3337) on the host: (point, tet) pairs with the
    codimension-0 point inside the tet, every tet against every point, no filter.  A pair counts when the tet's box holds the point
    (inclusive) and none of the four orientations of IglUtils::pointInsideTetrahedron (IglUtils.hpp:276-294, in its argument order) is
    negative, each decided by the oracle's exact orc_orient3d.  The candidate pairs come from a k-d tree over the points queried with a
    cube that covers each tet's box; the box test and the orientations decide (V (n, 3), T (m, 4), pts vertex ids)."""
    V = np.ascontiguousarray(V, dtype=np.float64)
    T = np.asarray(T, dtype=np.int64).reshape(-1, 4)
    pts = np.asarray(pts, dtype=np.int64).ravel()
    if len(pts) == 0 or len(T) == 0:
        return 0
    X = V[T]
    lo, hi = X.min(1), X.max(1)
    c = 0.5 * (lo + hi)
    r = 0.5 * (hi - lo).max(1)
    r = r + 1e-12 * (np.abs(c).max(1) + r) + 1e-300  # the cube c +- r covers the box despite the rounding of c and r
    lists = cKDTree(V[pts]).query_ball_point(c, r, p=np.inf, workers=max(int(nthreads), 1))
    n_per = np.fromiter((len(x) for x in lists), dtype=np.int64, count=len(lists))
    if n_per.sum() == 0:
        return 0
    ti = np.repeat(np.arange(len(T)), n_per)
    pv = pts[np.concatenate([np.asarray(x, dtype=np.int64) for x in lists if len(x)])]
    P = V[pv]
    inbox = np.all((lo[ti] <= P) & (hi[ti] >= P), axis=1)
    n = 0
    for t, v in zip(ti[inbox], pv[inbox]):
        x, q = X[t], V[v]
        if (orc.orient3d(x[0], x[2], x[1], q) != -1 and orc.orient3d(x[0], x[3], x[2], q) != -1 and orc.orient3d(x[0], x[1], x[3], q) != -1
                and orc.orient3d(x[1], x[2], x[3], q) != -1):
            n += 1
    return n


def orient3d_exact(a, b, c, d):
    """sign of det [a - d; b - d; c - d] in rationals"""
    a, b, c, d = ([Fraction(float(x)) for x in p] for p in (a, b, c, d))
    r = [[a[k] - d[k] for k in range(3)], [b[k] - d[k] for k in range(3)], [c[k] - d[k] for k in range(3)]]
    det = r[0][0] * (r[1][1] * r[2][2] - r[1][2] * r[2][1]) - r[0][1] * (r[1][0] * r[2][2] - r[1][2] * r[2][0]) + r[0][2] * (r[1][0] * r[2][1] - r[1][1] * r[2][0])
    return (det > 0) - (det < 0)


def points_in_tets_exact(V, T, pts):
    """the reference's loop (SelfCollisionHandler.cpp:3301-3337) with exact orientations: inclusive box, then four orientations >= 0"""
    n = 0
    for t in np.asarray(T).reshape(-1, 4):
        x = [V[k] for k in t]
        lo, hi = np.min(x, axis=0), np.max(x, axis=0)
        for v in pts:
            p = V[v]
            if not (np.all(lo <= p) and np.all(hi >= p)):
                continue
            if (orient3d_exact(x[0], x[2], x[1], p) >= 0 and orient3d_exact(x[0], x[3], x[2], p) >= 0 and orient3d_exact(x[0], x[1], x[3], p) >= 0
                    and orient3d_exact(x[1], x[2], x[3], p) >= 0):
                n += 1
    return n


def crafted_soup():
    """(V (n, 3), T (m, 4), pts): the degenerate point-in-tet cases as one soup of independent tets and points"""
    tets, points = [], []
    base = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])

    def tet(X, off):
        tets.append(np.asarray(X, dtype=np.float64) + off)

    def pt(p, off):
        points.append(np.asarray(p, dtype=np.float64) + off)

    for k, (X, P) in enumerate([
        (base, [[0.25, 0.25, 0.0]]),                                   # on a face
        (base, [[0.5, 0.0, 0.0]]),                                     # on an edge
        (base, [[0.0, 0.0, 1.0]]),                                     # on a vertex
        (base, [[0.1, 0.1, np.nextafter(0.0, 1.0)]]),                  # one ulp inside a face
        (base, [[0.1, 0.1, np.nextafter(0.0, -1.0)]]),                 # one ulp outside a face (outside the box as well)
        (base, [[0.5, 0.5, np.nextafter(0.0, 1.0)]]),                  # in the box, one ulp off the slanted face: outside (x + y + z > 1)
        (base, [[0.9, 0.9, 0.9]]),                                     # in the box, outside the tet
        (base, [[1.0, 1.0, 0.0]]),                                     # on the box boundary, outside the tet
        (base[[0, 2, 1, 3]], [[0.1, 0.1, 0.1]]),                       # inverted tet, interior point
        (base[[0, 2, 1, 3]], [[0.0, 0.0, 0.0]]),                       # inverted tet, its vertex
        ([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], [[0.25, 0.25, 0.0]]),  # zero-volume tet, point in its plane
        ([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], [[0.25, 0.25, 1e-300]]),  # zero-volume tet, point in its box (zero z extent: outside)
    ]):
        off = np.array([3.0 * k, 0.0, 0.0])
        tet(X, off)
        for p in P:
            pt(p, off)
    # the floating-point filter cannot decide: a face plane through points with many bits, and a point on it to the last bit
    a = np.array([0.1, 0.2, 0.3]); b = np.array([1.1, 0.7, 0.3]); c = np.array([0.3, 1.3, 0.7]); dd = np.array([0.5, 0.6, 1.9])
    off = np.array([40.0, 0.0, 0.0])
    tet([a, b, c, dd], off)
    for s in (0.5, 0.25):
        pt(a + s * (b - a), off)  # on the edge a-b up to rounding of the sum and the offset
    pt((a + b + c) / 3.0, off)    # on the face a b c up to rounding
    pt((a + b + c + dd) / 4.0, off)
    V = np.concatenate([np.concatenate(tets), np.asarray(points)])
    nt = len(tets)
    T = np.arange(4 * nt, dtype=np.int32).reshape(nt, 4)
    pts = np.arange(4 * nt, len(V), dtype=np.int32)
    return V, T, pts


# ---- scenes ---------------------------------------------------------------------------------------------------------------------
def _ball(res, radius, center):
    V, T = M.ball_tets(res, radius=radius, center=center)
    return dict(codim=3, V=V, T=T)


def pin_cushion(res=6, n=9):
    """17_pinCushionBall-like: a ball on an n x n bed of vertical segments (segMeshes/edge.seg rotated 90 degrees about z, scaled), the
    segments scripted (Dirichlet)"""
    Ve, Ee = codim.read_seg(os.path.join(MESHES, "edge.seg"))
    comps = [_ball(res, 0.45, (0.0, 0.56, 0.0))]
    for i in range(n):
        for k in range(n):
            V = shape_transform(Ve, translate=(-0.4 + 0.8 * i / (n - 1), 0.0, -0.4 + 0.8 * k / (n - 1)), rotate_deg=(0, 0, 90), scale=(0.1, 0.1, 0.1))
            comps.append(dict(codim=1, V=V, E=Ee, dbc=True))
    return codim.codim_scene(comps, density=1000.0, YM=1e4, PR=0.4)


def point_roller(res=6):
    """18_pointRollerBall-like: two point cylinders (cylinder.pt -> cylinder.obj's vertices) under a ball, scripted"""
    Vc = codim.read_pt(os.path.join(MESHES, "cylinder.pt"))
    cyl = [shape_transform(Vc, translate=t, rotate_deg=r, scale=(0.5, 0.5, 0.5)) for t, r in (((0.0, -0.1, 0.0), (0, 0, 0)), ((0.5, -0.1, 0.5), (0, 90, 0)))]
    top = max((c[np.argmax(c[:, 1])] for c in cyl), key=lambda q: q[1])  # the ball's lowest vertex 0.01 above the highest point
    comps = [_ball(res, 0.3, (top[0], top[1] + 0.31, top[2]))] + [dict(codim=0, V=c, dbc=True) for c in cyl]
    return codim.codim_scene(comps, density=500.0, YM=1e4, PR=0.4)


def plane_drop(kind, n=6):
    """coDimUnitTests mat40x40_pointPlaneDrop / _segPlaneDrop-like: a tet mat over the point plane (pointPlane.obj as points) or the segment
    plane (segPlane.seg), the plane scripted"""
    Vm, Tm = M.grid_tets(n, 2, n, h=1.0 / n, origin=(0.1, 0.015, 0.1))
    if kind == "point":
        Vp = codim.read_pt(os.path.join(MESHES, "pointPlane.pt"))
        comp = dict(codim=0, V=shape_transform(Vp, scale=(0.3, 0.3, 0.3)), dbc=True)
    else:
        Vp, Ep = codim.read_seg(os.path.join(MESHES, "segPlane.seg"))
        comp = dict(codim=1, V=shape_transform(Vp, scale=(0.3, 0.3, 0.3)), E=Ep, dbc=True)
    return codim.codim_scene([dict(codim=3, V=Vm, T=Tm), comp], density=1000.0, YM=1e4, PR=0.4)
