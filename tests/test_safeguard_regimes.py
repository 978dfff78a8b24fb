"""The line-search safeguards where their decisions flip: tests/golden/safeguard_regimes_golden.npz (written by
tests/golden/gen_safeguard_regimes_golden.py) holds orientation, segment-triangle, point-in-tetrahedron and inversion stencils with every
decision evaluated from the stored doubles alone.

Pinned exactly: every orient3d sign, both exits of segTriIntersect, every pointInsideTetrahedron outcome.  Pinned to the restated rounding:
the FullPivLU solve of segTriIntersect (Eigen's order, bit for bit) and the determinant of checkInversion.  Recorded only: the row-order
solve's decisions and the double-vs-exact disagreements."""
import importlib.util
import os
import struct

import numpy as np
import pytest

import oracle as orc
from ipc_b200 import mesh as M

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "safeguard_regimes_golden.npz")
GEN = os.path.join(HERE, "golden", "gen_safeguard_regimes_golden.py")
# the device's expansion buffers (safeguard.cu: orient3d_exact): cda/dab/abc/bcd and the pairwise sums 12, the scaled terms 24, the sum 96
DEVICE_BOUNDS = dict(cda=12, dab=12, abc=12, bcd=12, pair_sum=12, adet=24, bdet=24, cdet=24, ddet=24, running_sum=96, det=96)


def gold():
    return dict(np.load(GOLD))


def gen_module():
    spec = importlib.util.spec_from_file_location("gen_safeguard_regimes_golden", GEN)
    g = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(g)
    return g


def bits(x):
    return struct.pack("<d", float(x))


# ---- CPU --------------------------------------------------------------------------------------------------------------------------------
def test_generator_reproduces_the_fixture():
    z = gold()
    g = gen_module()
    out = g.evaluate(*g.build())
    assert set(out) == set(z)
    for k, v in out.items():
        v = np.asarray(v)
        assert z[k].shape == v.shape and z[k].dtype == v.dtype and z[k].tobytes() == v.tobytes(), k


def test_oracle_orientation_and_filter_meet_the_fixture():
    z = gold()
    for p, s, f in zip(z["orient_pts"], z["orient_sign"], z["orient_filter"]):
        sign, decided, _ = orc.orient3d_trace(*p[:4])
        assert sign == s and orc.orient3d(*p[:4]) == s and orc.orient3d(*p[:4], exact=True) == s
        assert decided == (f != 2) and (not decided or f == s)


def test_oracle_point_in_tet_meets_the_fixture():
    z = gold()

    def pit(q, t):
        if np.any(q < t.min(0)) or np.any(q > t.max(0)):
            return 0
        return int(orc.orient3d(t[0], t[2], t[1], q) >= 0 and orc.orient3d(t[0], t[3], t[2], q) >= 0 and orc.orient3d(t[0], t[1], t[3], q) >= 0
                   and orc.orient3d(t[1], t[2], t[3], q) >= 0)

    for q, o, r in zip(z["pit_pts"], z["pit_owner"], z["pit_in"]):
        assert pit(q, z["pit_tets"][o]) == r
    for p, r in zip(z["orient_pts"], z["orient_pit"]):
        assert pit(p[3], np.array([p[0], p[2], p[1], p[4]])) == r[0] and pit(p[3], np.array([p[0], p[1], p[2], p[5]])) == r[1]


def test_oracle_segment_triangle_meets_the_fixture_bit_for_bit():
    z = gold()
    for k, p in enumerate(z["segtri_pts"]):
        dec, ex, rank, uvt = orc.seg_tri_trace(*p)
        assert ex == z["segtri_exit"][k] and dec == z["segtri_dec"][k], k
        if ex == 2:
            assert rank == z["segtri_rank"][k] and all(bits(a) == bits(b) for a, b in zip(uvt, z["segtri_uvt"][k])), (k, uvt, z["segtri_uvt"][k])


def test_oracle_inversion_count_meets_the_fixture():
    z = gold()
    T = z["inv_tets"]
    n = len(T)
    unit = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]])
    m = M.Mesh(np.tile(unit, (n, 1)), np.arange(4 * n, dtype=np.int32).reshape(n, 4), energy=0)
    m.V = np.ascontiguousarray(T.reshape(-1, 3))
    assert orc.Elastic(m).count_inverted() == int((z["inv_det"] < 0).sum())


def test_branch_and_family_coverage():
    z = gold()
    g = gen_module()
    # orientation: all three signs, the filter deciding and not, undecided inputs in every family but the generic one
    assert set(np.unique(z["orient_sign"])) == {-1, 0, 1}
    und = {name: int(((z["orient_family"] == k) & (z["orient_filter"] == 2)).sum()) for k, name in enumerate(g.FAMILIES["orient"])}
    print("\nfilter-undecided orientations per family:", und)
    assert und["generic"] == 0 and int((z["orient_filter"] != 2).sum()) > 0
    for name in ("coplanar_dyadic", "near_coplanar", "scale"):
        assert und[name] >= 24, name
    assert und["ulp_off"] >= 12 and und["long_expansion"] >= 12 and und["degenerate"] == 12 and und["offset"] >= 3
    # the exact stage's longest expansions stay within the device's buffers
    longest = dict.fromkeys(DEVICE_BOUNDS, 0)
    n_exact = 0
    for p in z["orient_pts"]:
        _, decided, lens = orc.orient3d_trace(*p[:4])
        n_exact += not decided
        for k, v in lens.items():
            longest[k] = max(longest[k], v)
    print("longest expansions reached:", longest, "device bounds:", DEVICE_BOUNDS, "exact-stage inputs:", n_exact)
    assert all(longest[k] <= DEVICE_BOUNDS[k] for k in DEVICE_BOUNDS)
    # segTriIntersect: both orientation exits, the solve at rank 2 and rank 3, hits and misses of the solve
    ex, rk, dec = z["segtri_exit"], z["segtri_rank"], z["segtri_dec"]
    assert set(np.unique(ex)) == {0, 1, 2} and {2, 3} <= set(np.unique(rk[ex == 2]))
    assert set(np.unique(dec[ex == 2])) == {0, 1}
    for k, name in enumerate(g.FAMILIES["segtri"]):
        assert (z["segtri_family"] == k).any(), name
    # the row-oriented back substitution decides otherwise on some boundary stencils (recorded; the device follows Eigen's columns)
    n_order = int((z["segtri_dec"] != z["segtri_dec_row"]).sum())
    print("row-order decisions that differ:", n_order, "double vs exact decisions that differ:", int((z["segtri_dec"] != z["segtri_dec_exact"]).sum()))
    assert n_order >= 1
    # point in tet: inside and outside in every family; the inversion signs
    for k, name in enumerate(g.FAMILIES["pit"]):
        sel = z["pit_family"][z["pit_owner"]] == k
        assert sel.any() and z["pit_in"][sel].any(), name
    assert (z["pit_in"] == 0).any()
    d = z["inv_det"]
    assert (d == 0).any() and (np.signbit(d) & (d == 0)).any() and (~np.signbit(d) & (d == 0)).any() and (d < 0).any() and (d > 0).any()


def test_solve_decision_meets_the_exact_one_outside_the_rounding_band():
    z = gold()
    sel = (z["segtri_exit"] == 2) & (np.abs(z["segtri_margin"]) > z["segtri_band"])
    assert sel.sum() > 100
    assert np.array_equal(z["segtri_dec"][sel], z["segtri_dec_exact"][sel])
    # the exits before the solve are exact: an endpoint in the plane or both on one side is never a hit
    assert not z["segtri_dec"][z["segtri_exit"] != 2].any() and not z["segtri_dec_exact"][z["segtri_exit"] != 2].any()


# ---- GPU --------------------------------------------------------------------------------------------------------------------------------
class Soup:
    """the fixture's orientation, segment-triangle and point-in-tet stencils as one scene, in the stencil order `perm` (per kind)"""

    def __init__(self, z, perm=None, pit_families=None):
        no, ns = len(z["orient_pts"]), len(z["segtri_pts"])
        pit_sel = np.arange(len(z["pit_tets"])) if pit_families is None else np.flatnonzero(np.isin(z["pit_family"], pit_families))
        if pit_families is not None:
            no = ns = 0
        self.o_ord = perm.permutation(no) if perm is not None else np.arange(no)
        self.s_ord = perm.permutation(ns) if perm is not None else np.arange(ns)
        self.p_ord = perm.permutation(pit_sel) if perm is not None else pit_sel
        V, T, pts, SF, SE = [], [], [], [], []

        def add(x):
            V.append(np.asarray(x, dtype=np.float64))
            return len(V) - 1
        for k in self.o_ord:
            a, b, c, d, pp, pm = (add(x) for x in z["orient_pts"][k])
            T += [[a, c, b, pp], [a, b, c, pm]]
            pts.append(d)
        self.n_orient_tets = len(T)
        for k in self.s_ord:
            e0, e1, t0, t1, t2 = (add(x) for x in z["segtri_pts"][k])
            SF.append([t0, t1, t2])
            SE.append([e0, e1])
        for k in self.p_ord:
            T.append([add(x) for x in z["pit_tets"][k]])
            pts += [add(q) for q in z["pit_pts"][z["pit_owner"] == k]]
        self.V = np.array(V)
        self.T = np.array(T, dtype=np.int32).reshape(-1, 4)
        self.SF = np.array(SF, dtype=np.int32).reshape(-1, 3)
        self.SE = np.array(SE, dtype=np.int32).reshape(-1, 2)
        self.pts = np.array(pts, dtype=np.int32)
        # expected, in this order
        self.tri = z["segtri_dec"][self.s_ord]
        self.tet = np.concatenate([z["orient_pit"][self.o_ord].reshape(-1), [int(z["pit_in"][z["pit_owner"] == k].sum()) for k in self.p_ord]]).astype(int)

    def upload(self, ctx):
        n = len(self.T)
        unit = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]])
        Vr = self.V.copy()
        for k, t in enumerate(self.T):
            Vr[t] = unit + np.array([3.0 * k, 0.0, 0.0])   # a positive rest shape per tet (the checks read the current positions only)
        m = M.Mesh(Vr, self.T, energy=0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        vcod = np.full(len(self.V), 3, np.int32)
        vcod[self.pts] = 0
        svi = np.unique(np.concatenate([self.SF.ravel(), self.SE.ravel()])).astype(np.int32)
        ctx.set_surface(svi, self.SE, np.ascontiguousarray(self.SF.T).ravel(), vcod)
        ctx.set_state(np.ascontiguousarray(self.V.T).ravel())
        assert n == len(self.tet)


def run_check(ctx, soup):
    """(total of the deferred check, per-triangle flags, per-tet counts)"""
    soup.upload(ctx)
    ctx.safeguard_debug_flags(1)
    ctx.intersection_free(want=False)
    total = ctx.fetch_iteration().n_intersected_triangles
    tri, tet = ctx.safeguard_debug_flags(0, read=True)
    return total, tri, tet


def assert_matches(soup, total, tri, tet):
    bad_t = np.flatnonzero(tri != soup.tri)
    bad_p = np.flatnonzero(tet != soup.tet)
    assert not len(bad_t), f"{len(bad_t)} segment-triangle stencils off Eigen's solve, e.g. {soup.s_ord[bad_t[:8]].tolist()}"
    assert not len(bad_p), f"{len(bad_p)} tets off the exact point-in-tet count, e.g. {bad_p[:8].tolist()}"
    assert total == int(soup.tri.sum()) + int(soup.tet.sum())


@pytest.mark.gpu
def test_device_decisions_per_stencil(gpu_ctx):
    z = gold()
    soup = Soup(z)
    total, tri, tet = run_check(gpu_ctx, soup)
    assert_matches(soup, total, tri, tet)
    # the eager form agrees with the deferred one
    assert gpu_ctx.intersection_free() == (total == 0)


@pytest.mark.gpu
def test_device_stencil_order_changes_no_decision(gpu_ctx):
    z = gold()
    for seed in (1, 2):
        soup = Soup(z, perm=np.random.default_rng(seed))
        assert_matches(soup, *run_check(gpu_ctx, soup))


@pytest.mark.gpu
def test_device_point_grid_scenes_alone(gpu_ctx):
    """families whose points alone make a degenerate point grid: one z for all points, a single point, duplicate points"""
    z = gold()
    g = gen_module()
    for name in g.ALONE:
        soup = Soup(z, pit_families=[g.FAMILIES["pit"].index(name)])
        assert_matches(soup, *run_check(gpu_ctx, soup))


@pytest.mark.gpu
def test_debug_buffers_off_keep_the_launch_count(gpu_ctx):
    z = gold()
    soup = Soup(z)
    soup.upload(gpu_ctx)
    counts = []
    for on in (0, 1, 0):
        gpu_ctx.safeguard_debug_flags(on)
        n0 = gpu_ctx.launch_count()
        gpu_ctx.intersection_free(want=False)
        counts.append((gpu_ctx.launch_count() - n0, gpu_ctx.fetch_iteration().n_intersected_triangles))
    assert counts[0] == counts[1] == counts[2]


@pytest.mark.gpu
def test_device_inversion_count_per_tet(gpu_ctx):
    """checkInversion's determinant in doubles, bit for bit: det == +0.0 and -0.0 are not inverted, one ulp either way decides"""
    z = gold()
    unit = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]])
    bad = []
    for k, t in enumerate(z["inv_tets"]):
        m = M.Mesh(unit, np.arange(4, dtype=np.int32).reshape(1, 4), energy=0)
        gpu_ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        gpu_ctx.set_state(np.ascontiguousarray(t.T).ravel())
        if gpu_ctx.check_inversion() != int(z["inv_det"][k] < 0):
            bad.append(k)
    assert not bad, bad
    n = len(z["inv_tets"])
    m = M.Mesh(np.tile(unit, (n, 1)), np.arange(4 * n, dtype=np.int32).reshape(n, 4), energy=0)
    gpu_ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
    gpu_ctx.set_state(np.ascontiguousarray(z["inv_tets"].reshape(-1, 3).T).ravel())
    assert gpu_ctx.check_inversion() == int((z["inv_det"] < 0).sum())
