"""Codimensional scenes on the device: every stage against the oracle on scenes modelled on the reference's codimensional examples, the
point-in-tetrahedron half of the intersection check against exact arithmetic, the line search with a point entering a tet, and a tet-only
scene with vCoDim given against one without."""

import numpy as np
import pytest

import oracle as orc
import oracle_codim as oc
from gpu_common import load_scene, scalar_bits, shared_ctx, soa
from ipc_b200 import codim
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from stagecheck import check_every_stage

pytestmark = pytest.mark.gpu
NTH = 8


def deformed(m, seed, amp):
    """a deformed state: free vertices jittered by amp (halved until no tet is inverted), scripted (Dirichlet) components shifted as a whole
    toward +y"""
    rng = np.random.default_rng(seed)
    noise = rng.standard_normal(m.V_rest.shape) * (m.dbc == 0)[:, None]
    while True:
        m.V = m.V_rest + amp * noise
        m.V[m.dbc != 0, 1] += 0.5 * amp
        if orc.Elastic(m).count_inverted() == 0:
            return m
        amp *= 0.5


def pts_of(m):
    return np.flatnonzero(m.vCoDim == 0).astype(np.int32)


def device_count(ctx):
    ctx.intersection_free(want=False)
    return ctx.fetch_iteration().n_intersected_triangles


SCENES = {"pin_cushion": oc.pin_cushion, "point_roller": oc.point_roller, "point_plane": lambda: oc.plane_drop("point"),
          "seg_plane": lambda: oc.plane_drop("seg")}


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("name", list(SCENES))
def test_codim_scene_every_stage(shared_ctx, name, seed):
    m = deformed(SCENES[name](), seed, 2e-3)
    dHat = 0.03 ** 2
    rng = np.random.default_rng(seed + 10)
    P = np.zeros_like(m.V)
    P[m.vCoDim == 3, 1] = -0.05
    P[m.dbc != 0, 1] = 0.03
    P += 0.005 * rng.standard_normal(P.shape)
    load_scene(shared_ctx, m)
    # (the summed CSR Hessian is compared in test_codim_scene_hessian: stagecheck's oracle writes the Dirichlet identity only on rows of
    # vertices that have a tet, as Energy::computeHessian does; the codimensional Dirichlet vertices have none)
    r = check_every_stage(shared_ctx, m, dict(dHat=dHat, p=np.ascontiguousarray(P).ravel()), kappa=1e4, min_active=1, h_tol=np.inf)
    assert r["n_active"] > 0
    s = orc.Surf(m)
    mm_r, pa_r, pe_r, _ = s.constraint_set(dHat)
    # codimensional pairs are in the set: a PP / PE / EE pair with a vertex of codimension < 3 (with multiplicities for PP / PE)
    vs = lambda q: [(-q[0] - 1) if q[0] < 0 else q[0]] + [x for x in q[1:] if x >= 0]
    assert any(min(m.vCoDim[v] for v in vs(q)) < 3 for q in mm_r)
    # lagged friction: the same pairs and the same energy
    Vt = m.V - 1e-3 * P
    shared_ctx.set_prev_state(soa(Vt))
    shared_ctx.constraint_set(dHat, 0)
    nfr = shared_ctx.friction_lag(dHat, 1e4)
    lam, co, ba = s.friction_lag(mm_r, dHat, 1e4)
    eps2 = (1e-3 * m.avgEdgeLen) ** 2
    Ef, Ef_r = shared_ctx.friction_energy(eps2, 0.3), s.friction_energy(Vt, mm_r, lam, co, ba, eps2, 0.3)
    assert nfr == len(mm_r) and abs(Ef - Ef_r) <= 1e-10 * abs(Ef_r)
    # device-built pattern: vNeighbor with the CE / codimension-2 triangle edges, plus the contact pairs
    import bench
    ia_r, ja_r = m.csr_pattern(1, extra_pairs=bench.contact_pattern_pairs(m, mm_r, pa_r, pe_r))
    shared_ctx.enable_device_pattern(1, 2 * ja_r.size)
    shared_ctx.constraint_set(dHat, 0)
    shared_ctx.update_pattern()
    ia, ja = shared_ctx.get_pattern()
    assert np.array_equal(ia, ia_r) and np.array_equal(ja, ja_r)
    shared_ctx.set_csr(ia_r, ja_r, 1)  # (back to host mode for the next test)
    # intersection check (both halves) and inversion check (tets only)
    ok_r, hits_r = s.intersection_free(nthreads=NTH)
    n_pit = oc.points_in_tets(m.V, m.T, pts_of(m), NTH)
    assert device_count(shared_ctx) == hits_r + n_pit
    assert shared_ctx.intersection_free() == (ok_r and n_pit == 0)
    assert shared_ctx.check_inversion() == orc.Elastic(m).count_inverted()


@pytest.mark.parametrize("name", list(SCENES))
def test_codim_scene_hessian(shared_ctx, name):
    m = deformed(SCENES[name](), 1, 2e-3)
    dHat, kappa, dt2 = 0.03 ** 2, 1e4, 0.025 ** 2
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    mm_r, pa_r, pe_r, _ = s.constraint_set(dHat)
    shared_ctx.constraint_set(dHat, 0)
    import bench
    ia, ja = m.csr_pattern(1, extra_pairs=bench.contact_pattern_pairs(m, mm_r, pa_r, pe_r))
    shared_ctx.set_csr(ia, ja, 1)
    a = np.zeros(ja.size)
    shared_ctx.elastic_hessian(dt2, 1, 1, 1, a)
    shared_ctx.barrier_hessian(dHat, kappa, 1, a)
    a_r = orc.Elastic(m).hessian_csr(dt2, ia, ja, 1, 1, 1, nthreads=NTH)
    s.barrier_hessian_csr(mm_r, pa_r, pe_r, dHat, kappa, ia, ja, 1, 1, a=a_r, nthreads=NTH)
    # Optimizer::computePrecondMtr (Optimizer.cpp:3634-3660) sets the identity on the diagonal of EVERY projected Dirichlet vertex, also of
    # the codimensional ones, which no tet touches (the oracle's per-tet assembly reaches only vertices with a tet).  The diagonal entry of
    # row r is the first entry of the row in the upper-triangular pattern.
    dbc_rows = 3 * np.repeat(np.flatnonzero(m.dbc == 1), 3) + np.tile(np.arange(3), int((m.dbc == 1).sum()))
    no_tet = np.ones(m.nV, dtype=bool)
    no_tet[m.T.ravel()] = False
    assert np.any(no_tet & (m.dbc == 1))  # the case this test is about
    a_r[ia[dbc_rows] - 1] = 1.0
    assert np.linalg.norm(a - a_r) <= 1e-9 * np.linalg.norm(a_r), np.linalg.norm(a - a_r) / np.linalg.norm(a_r)
    # the device writes that identity itself (k_diag_mass_dbc runs over every vertex)
    rows_nt = 3 * np.repeat(np.flatnonzero(no_tet & (m.dbc == 1)), 3) + np.tile(np.arange(3), int((no_tet & (m.dbc == 1)).sum()))
    assert np.all(a[ia[rows_nt] - 1] == 1.0)


def soup_mesh(V, T, pts):
    """tets of V[T] (current) with a positive rest shape per tet, and the points as a codimension-0 component"""
    base = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    Vr = np.asarray(V, dtype=np.float64).copy()
    for k, t in enumerate(T):
        Vr[t] = base + np.array([3.0 * k, 0.0, 0.0])
    m = M.Mesh(Vr, T, energy=0)
    m.V = np.asarray(V, dtype=np.float64).copy()
    m.vCoDim = np.full(m.nV, 3, dtype=np.int32)
    m.vCoDim[pts] = 0
    return m


def sheet_under_ball(n=60, span=3.0):
    """a scripted codimension-2 sheet of 2 n^2 triangles 0.01 under a tet ball.  The sheet comes first, so its edges hold the low edge
    indices: the EE candidates of the ball against it have first components (sheet edges) up to nSE, which is about three times nV.
    (Cells of 0.05, wider than the contact distance: the sheet's own box pairs stay within the broad phase's capacity.)"""
    g = np.linspace(-span / 2, span / 2, n + 1)
    X, Z = np.meshgrid(g, g, indexing="ij")
    V = np.stack([X.ravel(), np.zeros(X.size), Z.ravel()], 1)
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    a, b, c, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel(), idx[:-1, 1:].ravel()
    F = np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)])
    ball = oc._ball(6, 0.45, (0.0, 0.0, 0.0))
    ball["V"][:, 1] += 0.01 - ball["V"][:, 1].min()
    m = codim.codim_scene([dict(codim=2, V=V, F=F, dbc=True), ball], density=1000.0, YM=1e4, PR=0.4)
    m.V = m.V_rest.copy()
    return m


@pytest.mark.parametrize("level", [1, 2])
def test_candidates_beyond_nv_in_canonical_order(shared_ctx, level):
    """the candidate list sorted on a scene with more surface edges than vertices: its first components reach past nV"""
    m = sheet_under_ball()
    dHat = 0.03 ** 2
    load_scene(shared_ctx, m)
    shared_ctx.set_canonical_order(level)
    try:
        got = shared_ctx.constraint_set(dHat, 1)
    finally:
        shared_ctx.set_canonical_order(1)
    ref = orc.Surf(m).constraint_set(dHat)
    cand = ref[3]
    assert len(m.SFEdges) > m.nV and cand[:, 0].max() >= m.nV and cand[:, 0].min() < 0
    assert all(np.array_equal(x, y) for x, y in zip(got, ref))


def test_point_in_tet_crafted_soup(shared_ctx):
    V, T, pts = oc.crafted_soup()
    m = soup_mesh(V, T, pts)
    n_exact = oc.points_in_tets_exact(V, T, pts)
    assert n_exact == oc.points_in_tets(V, T, pts) and n_exact > 0
    load_scene(shared_ctx, m)
    _, hits_r = orc.Surf(m).intersection_free()
    assert hits_r == 0
    assert device_count(shared_ctx) == n_exact
    assert shared_ctx.intersection_free() is False


def test_point_in_tet_one_point_per_tet(shared_ctx):
    """every tet of a grid holds its own point (centroid), every point in another slot of the grid, plus points on shared faces"""
    V, T = M.grid_tets(7, 6, 5, h=0.1)
    C = V[T].mean(1)
    F = (V[T[:, 0]] + V[T[:, 1]] + V[T[:, 2]]) / 3.0  # on a face: counted by every tet that has it
    P = np.concatenate([C, F[::5]])
    Vall = np.concatenate([V, P])
    m = M.Mesh(np.concatenate([V, P]), T, energy=0)
    m.V = Vall.copy()
    m.vCoDim = np.full(m.nV, 3, dtype=np.int32)
    m.vCoDim[len(V):] = 0
    pts = pts_of(m)
    n_ref = oc.points_in_tets(Vall, T, pts, NTH)
    assert n_ref >= len(T) + len(F[::5])
    load_scene(shared_ctx, m)
    assert device_count(shared_ctx) == n_ref + orc.Surf(m).intersection_free()[1]


def test_tet_only_vcodim_bit_identical(shared_ctx):
    """a tet-only scene with vCoDim (all 3) equals vCoDim = NULL bit for bit with the same launch count"""
    V1, T1 = M.grid_tets(4, 4, 4, h=0.25)
    V2, T2 = M.grid_tets(4, 4, 4, h=0.25, origin=(0.1, 0.05, 1.01))
    m = M.merge_meshes([(V1, T1), (V2, T2)])
    rng = np.random.default_rng(4)
    m.V = m.V_rest + 1e-3 * rng.standard_normal(m.V.shape)
    P = np.zeros_like(m.V)
    P[len(V1):, 2] = -0.05
    p = np.ascontiguousarray(P).ravel()
    dHat = 0.02 ** 2
    out = []
    for codim in (True, False):
        load_scene(shared_ctx, m, vcodim=codim)
        n0 = shared_ctx.launch_count()
        mm, pa, pe, cand = shared_ctx.constraint_set(dHat, 1)
        evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
        a1 = shared_ctx.ccd_partial(p, 1e-6, evf, eee, 1.0)
        ag = shared_ctx.hash_build_swept(p, a1, m.avgEdgeLen / 3)
        a2, nc = shared_ctx.ccd_full(1e-6, evf, eee, ag)
        ok = shared_ctx.intersection_free()
        Eb = shared_ctx.barrier_energy(dHat, 1e4)
        out.append((mm.tobytes(), pa.tobytes(), cand.tobytes(), scalar_bits(a1), scalar_bits(a2), nc, ok, scalar_bits(Eb), shared_ctx.launch_count() - n0))
    assert out[0] == out[1]


# ---- line search with a point entering a tet ---------------------------------------------------------------------------------------
class _OrcWithPoints:
    """the oracle module with Surf.intersection_free extended by the point-in-tetrahedron half, for the line-search driver"""

    def __init__(self, pts):
        self.pts = pts

    def __getattr__(self, k):
        return getattr(orc, k)

    def Surf(self, m, V=None):
        s = orc.Surf(m, V=V)
        pts, Vc = self.pts, (m.V if V is None else V)
        base = s.intersection_free

        def intersection_free(*a, **kw):
            ok, hits = base(*a, **kw)
            n = oc.points_in_tets(Vc, m.T, pts)
            return ok and n == 0, hits + n

        s.intersection_free = intersection_free
        return s


def test_line_search_point_enters_tet(shared_ctx):
    import test_gpu_step_control as SC
    # a block falls onto a bed of points; at alpha = 1 the points are 0.3 deep inside it
    Vb, Tb = M.grid_tets(3, 3, 3, h=1.0 / 3, origin=(0.0, 0.0, 0.1))
    xs = np.linspace(0.1, 0.9, 5)
    Vp = np.array([[x, y, 0.05] for x in xs for y in xs])
    from ipc_b200 import codim
    m = codim.codim_scene([dict(codim=3, V=Vb, T=Tb), dict(codim=0, V=Vp, dbc=True)], density=1.0, YM=1e5, PR=0.4, energy=1)
    P = np.zeros_like(m.V)
    P[: len(Vb), 2] = -0.4
    xt = m.V.copy()
    xt[: len(Vb), 2] -= 0.2
    sc = SC.Scene("codim", m, P, 0.025 ** 2, 0.01 ** 2, 1e-2, xtilde=xt)
    real = SC.orc
    SC.orc = _OrcWithPoints(pts_of(m))
    try:
        ref = SC.oracle_line_search(sc, 1.0)
    finally:
        SC.orc = real
    assert ref["status"] == 0 and ref["counts"][1] > 0  # the point-in-tet half halved the step
    SC.load_step_scene(shared_ctx, sc)
    rc, alpha = shared_ctx.line_search(**sc.terms(), alpha=1.0)
    info = shared_ctx.step_control_info()
    assert rc == 0 and scalar_bits(alpha) == scalar_bits(ref["alpha"]) and SC.counts(info) == ref["counts"]
    # captured: the same step and counters from a replay (a captured line search keeps the device's list order)
    shared_ctx.set_canonical_order(0)
    SC.prepare(shared_ctx, sc, m.V, sc.p)
    shared_ctx.fetch_iteration()
    shared_ctx.capture_begin()
    shared_ctx.step_bound_set(1.0)
    shared_ctx.line_search(**sc.terms())
    gid = shared_ctx.capture_end()
    SC.prepare(shared_ctx, sc, m.V, sc.p)
    shared_ctx.graph_launch(gid)
    info = shared_ctx.step_control_info()
    assert info.status == 0 and scalar_bits(info.alpha) == scalar_bits(ref["alpha"]) and SC.counts(info) == ref["counts"]
    shared_ctx.graph_destroy(gid)
