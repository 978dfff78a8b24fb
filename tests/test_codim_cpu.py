"""Codimensional scene input (ipc_b200/codim.py) against hand-computed cases, and the host point-in-tetrahedron count (oracle_codim, on the
oracle's exact orient3d) against exact rational arithmetic (no GPU)."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as orc
import oracle_codim as oc
from ipc_b200 import codim, mesh as M
from ipc_b200.scenes import shape_transform


def small_scene(density=2.0):
    """one tet, one triangle, two segments sharing a vertex, two loose points"""
    Vt = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    Vf = np.array([[2.0, 0.0, 0.0], [3.0, 0.0, 0.0], [2.0, 2.0, 0.0]])
    Ve = np.array([[0.0, 3.0, 0.0], [0.0, 3.0, 2.0], [0.0, 3.0, 3.0]])
    Vp = np.array([[5.0, 5.0, 5.0], [6.0, 5.0, 5.0]])
    comps = [dict(codim=3, V=Vt, T=[[0, 1, 2, 3]]), dict(codim=2, V=Vf, F=[[0, 1, 2]]), dict(codim=1, V=Ve, E=[[1, 0], [1, 2]], dbc=True),
             dict(codim=0, V=Vp)]
    return codim.codim_scene(comps, density=density), comps


def test_scene_arrays():
    m, _ = small_scene()
    assert list(m.componentNodeRange) == [0, 4, 7, 10, 12] and list(m.componentCoDim) == [3, 2, 1, 0]
    assert list(m.vCoDim) == [3] * 4 + [2] * 3 + [1] * 3 + [0] * 2
    assert list(m.dbc) == [0] * 7 + [1] * 3 + [0] * 2
    # SF: the tet's boundary faces, then the triangle; SFEdges: the triangles' edges in set order (first-seen orientation), then CE
    assert m.SF.shape == (5, 3) and list(m.SF[-1]) == [4, 5, 6]
    tri_edges = M.surface_edges(m.SF)
    assert [tuple(e) for e in m.SFEdges] == [tuple(e) for e in tri_edges] + [(8, 7), (8, 9)]
    assert (4, 5) in [tuple(e) for e in tri_edges] and (6, 4) in [tuple(e) for e in tri_edges]
    # SVI: every SF / CE vertex and every vertex without a neighbour, ascending
    assert list(m.SVI) == list(range(12))
    # vNeighbor: tet edges, triangle edges, segments
    lo, hi = m.neighbor_pairs()
    assert set(zip(lo.tolist(), hi.tolist())) == {(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3), (4, 5), (4, 6), (5, 6), (7, 8), (8, 9)}


def test_masses_closed_forms():
    rho = 2.0
    m, _ = small_scene(rho)
    tet = rho * (1.0 / 6.0) / 4.0
    assert np.allclose(m.mass[:4], tet, rtol=1e-15)
    # segment ends: l^3 pi / 12 per segment end
    assert np.isclose(m.mass[7], rho * 8 * np.pi / 12, rtol=1e-14) and np.isclose(m.mass[9], rho * np.pi / 12, rtol=1e-14)
    assert np.isclose(m.mass[8], rho * 9 * np.pi / 12, rtol=1e-14)
    # triangle (2,0,0) (3,0,0) (2,2,0): right angle at vertex 4; Voronoi areas times mean edge length / 3
    l = np.array([np.sqrt(5.0), 2.0, 1.0])
    A = 1.0
    got = m.mass[4:7] / (rho * l.mean() / 3.0)
    assert np.isclose(got.sum(), A, rtol=1e-14)
    assert np.allclose(got, codim._voronoi_tri_mass(m.V_rest, np.array([[4, 5, 6]]))[0] / (l.mean() / 3.0), rtol=1e-15)
    # points: the mean mass of the tet component's vertices
    assert np.allclose(m.mass[10:], tet, rtol=1e-15)


def test_voronoi_acute_and_obtuse():
    # equilateral: a third of the area each
    V = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.5, np.sqrt(3) / 2, 0.0]])
    q = codim._voronoi_tri_mass(V, np.array([[0, 1, 2]]))[0]
    A = np.sqrt(3) / 4
    assert np.allclose(q, A / 3 * 1.0 / 3.0, rtol=1e-12)
    # obtuse at vertex 0: half of the area to the obtuse corner (0.25 dblA), a quarter to each other
    V = np.array([[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [-1.0, 0.1, 0.0]])
    q = codim._voronoi_tri_mass(V, np.array([[0, 1, 2]]))[0]
    A = 0.1
    l = np.array([2.0, np.hypot(1, 0.1), np.hypot(1, 0.1)])
    assert np.allclose(q / (l.mean() / 3.0), [A / 2, A / 4, A / 4], rtol=1e-12)


def test_readers_and_seg_fallback(tmp_path):
    V, E = codim.read_seg(os.path.join(oc.MESHES, "edge.seg"))
    assert V.tolist() == [[0, 0, 0], [1, 0, 0]] and E.tolist() == [[0, 1]]
    # .seg missing: the same-stem .obj's edges, (a, b) kept unless (b, a) came first, in set order
    (tmp_path / "quad.obj").write_text("v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nf 1 2 3\nf 1 3 4\n")
    V, E = codim.read_seg(str(tmp_path / "quad.seg"))
    assert len(V) == 4 and E.tolist() == [[0, 1], [1, 2], [2, 0], [2, 3], [3, 0]]
    # .pt missing: the .obj's vertices
    Vc = codim.read_pt(os.path.join(oc.MESHES, "cylinder.pt"))
    assert Vc.shape == (152, 3)
    V, F = codim.read_obj(os.path.join(oc.MESHES, "cylinder.obj"))
    assert F.shape == (300, 3) and F.min() == 0 and F.max() == 151
    assert codim.read_shape(os.path.join(oc.MESHES, "point.pt"))[0] == 0
    with pytest.raises(ValueError):
        codim.read_shape("x.msh")


def test_shape_transform_semantics():
    """x' = R (x * scale) + t, R = Rx(a) Ry(b) Rz(c) (Config.cpp:218-224): edge.seg rotated 90 degrees about z stands up along +y"""
    V = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])
    W = shape_transform(V, translate=(1, 1, 1), rotate_deg=(0, 0, 90), scale=(2, 2, 2))
    assert np.allclose(W, [[1, 1, 1], [1, 3, 1]], atol=1e-15)
    # order: first z, then y, then x on the column vector
    W = shape_transform(np.array([[1.0, 0.0, 0.0]]), rotate_deg=(90, 0, 90))
    assert np.allclose(W, [[0, 0, 1]], atol=1e-15)


def test_scenes_build():
    for f in (oc.pin_cushion, oc.point_roller, lambda: oc.plane_drop("point"), lambda: oc.plane_drop("seg")):
        m = f()
        assert m.nV == m.componentNodeRange[-1] and np.all(m.mass > 0) and np.all(np.diff(m.SVI) > 0)
        assert orc.Surf(m).intersection_free(nthreads=2)[0] and oc.points_in_tets(m.V, m.T, np.flatnonzero(m.vCoDim == 0)) == 0


def test_orient3d_signature_and_sign_convention():
    """the host count calls orc_orient3d through ctypes (int return, four double pointers); its sign is that of det [a - d; b - d; c - d],
    positive for the centroid in each of pointInsideTetrahedron's four calls on a positively oriented tet"""
    f = orc.lib().orc_orient3d
    assert f.restype == C.c_int
    x = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    q = x.mean(0)
    for i, j, k in ((0, 2, 1), (0, 3, 2), (0, 1, 3), (1, 2, 3)):
        assert orc.orient3d(x[i], x[j], x[k], q) == 1 == oc.orient3d_exact(x[i], x[j], x[k], q)
    assert oc.points_in_tets(x, np.zeros((0, 4), np.int32), [0]) == 0 and oc.points_in_tets(x, [[0, 1, 2, 3]], []) == 0


def _filter_undecided(a, b, c, d):
    """the floating-point filter of orc_orient3d (16 eps * permanent) cannot decide"""
    ad, bd, cd = a - d, b - d, c - d
    det = ad[2] * (bd[0] * cd[1] - cd[0] * bd[1]) + bd[2] * (cd[0] * ad[1] - ad[0] * cd[1]) + cd[2] * (ad[0] * bd[1] - bd[0] * ad[1])
    perm = ((abs(bd[0] * cd[1]) + abs(cd[0] * bd[1])) * abs(ad[2]) + (abs(cd[0] * ad[1]) + abs(ad[0] * cd[1])) * abs(bd[2])
            + (abs(ad[0] * bd[1]) + abs(bd[0] * ad[1])) * abs(cd[2]))
    return abs(det) <= 1.7763568394002505e-15 * perm


def test_points_in_tets_exact_on_crafted_cases():
    V, T, pts = oc.crafted_soup()
    # case by case, each (point, tet) against the rational evaluation
    for t in range(len(T)):
        for p in pts:
            assert oc.points_in_tets(V, T[t:t + 1], [p]) == oc.points_in_tets_exact(V, T[t:t + 1], [p]), (t, p)
    assert oc.points_in_tets(V, T, pts, nthreads=4) == oc.points_in_tets_exact(V, T, pts)
    # the expected verdicts of the named cases (tets 0-11 hold one point each, in order)
    want = [1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0]
    assert [oc.points_in_tets(V, T[k:k + 1], [pts[k]]) for k in range(12)] == want
    # some orientation of the last tet is left to the exact stage
    x = V[T[-1]]
    assert any(_filter_undecided(x[i], x[j], x[k], V[p]) for p in pts[12:] for i, j, k in ((0, 2, 1), (0, 3, 2), (0, 1, 3), (1, 2, 3)))


def test_points_in_tets_random_against_exact():
    rng = np.random.default_rng(7)
    V, T = M.grid_tets(2, 2, 2, h=0.5)
    V = V + 0.05 * rng.standard_normal(V.shape)
    P = np.concatenate([rng.uniform(-0.1, 1.1, (60, 3)), V[rng.integers(0, len(V), 10)], (V[T[:10, 0]] + V[T[:10, 1]]) / 2])
    Vall = np.concatenate([V, P])
    pts = np.arange(len(V), len(Vall))
    assert oc.points_in_tets(Vall, T, pts, 2) == oc.points_in_tets_exact(Vall, T, pts)
