"""Half-space collision objects (ipcgpu_set_halfspaces and the ipcgpu_halfspace_* stages, HalfSpace<3>) against the CPU oracle
(oracle/halfspace.cpp): sets, counts and step bounds bit for bit, energies and gradients to 1e-10, Hessians to 1e-9 -- eagerly, deferred and
replayed from a graph; the planes inside the line search; and a context with no planes launching exactly what it launched before."""

import numpy as np
import pytest

import oracle as orc
import oracle_halfspace as OH
from gpu_common import load_scene, own_context, rel, scalar_bits, soa
from ipc_b200 import lib as L
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu


class Small:
    """a few ball_pile balls over a floor and a tilted wall, some Dirichlet vertices and a codimension-2 vertex; p points down"""

    def __init__(self):
        m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
        self.m, self.dHat, self.kappa = m, info["dHat"], 1e6
        sq = np.sqrt(self.dHat)
        lo = m.V.min(axis=0)
        rng = np.random.default_rng(11)
        m.dbc[m.SVI[rng.choice(m.SVI.size, 6, replace=False)]] = 1
        low = m.SVI[np.argsort(m.V[m.SVI, 1])]
        m.vCoDim[low[0]] = 2  # the lowest surface vertex is codimension 2: no plane entry
        m.dbc[low[1]] = 1     # the next one is Dirichlet
        wall_n = np.array([1.0, 0.4, 0.2])
        wall_n /= np.linalg.norm(wall_n)
        wall_o = m.V[np.argmin(m.V @ wall_n)] - 0.3 * sq * wall_n
        self.origin = np.array([[0.0, lo[1] - 0.5 * sq, 0.0], wall_o])
        self.normal = np.array([[0.0, 1.0, 0.0], wall_n])
        self.vdt = np.array([[0.02 * sq, 0.0, 0.0], [0.0, 0.0, 0.01 * sq]])
        self.friction = np.array([0.3, 0.5])
        self.par = OH.planes(self.origin, self.normal, self.vdt, self.friction)
        P = 0.5 * rng.standard_normal(m.V.shape) * sq
        P[:, 1] -= 3.0 * sq
        P -= 2.0 * sq * wall_n
        self.P = P
        self.p = np.ascontiguousarray(P).ravel()
        # previous positions: even vertices slide (|u| > eps), odd ones stick (|u| < 0.04 sqrt(dHat) with velocitydt)
        self.eps2 = (0.05 * sq) ** 2
        T = rng.standard_normal(m.V.shape) * (0.01 * sq)
        T[::2] *= 100.0
        self.Vprev = m.V - T


def upload_with_csr(ctx, sc, V=None):
    m = sc.m
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(1)
    ia, ja = m.csr_pattern(1)
    ctx.set_csr(ia, ja, 1)
    ctx.set_state(soa(m.V if V is None else V))
    ctx.set_search_dir(sc.p)
    ctx.set_prev_state(soa(sc.Vprev))
    return ia, ja


def oracle_all(sc, V, ia, ja):
    m = sc.m
    s = orc.Surf(m, V=V)
    hs = OH.HalfSpaces(s, sc.par)
    act = hs.constraint_set(sc.dHat)
    E, bad = hs.energy(act, sc.dHat, sc.kappa)
    g = hs.gradient(act, sc.dHat, sc.kappa)
    a = hs.hessian_csr(act, sc.dHat, sc.kappa, ia, ja, 1)
    alpha = hs.step(sc.p, 0.9, 1.0)
    lag, lam = hs.lag(act, sc.dHat, sc.kappa)
    Vt = soa(sc.Vprev)
    Ef = hs.friction_energy(Vt, lag, lam, sc.eps2)
    gf = hs.friction_gradient(Vt, lag, lam, sc.eps2)
    af = hs.friction_hessian_csr(Vt, lag, lam, sc.eps2, ia, ja, 1)
    return dict(act=act, E=E, bad=bad, g=g, a=a, alpha=alpha, lag=lag, lam=lam, Ef=Ef, gf=gf, af=af, cross=hs.crossings())


@pytest.fixture(scope="module")
def ctx():
    with own_context() as c:
        yield c


def test_small_scene_eager_matches_oracle(ctx):
    sc = Small()
    ia, ja = upload_with_csr(ctx, sc)
    ctx.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
    ref = oracle_all(sc, sc.m.V, ia, ja)
    assert len(ref["act"]) >= 4 and {0, 1} <= set(ref["act"][:, 0]) and ref["bad"] == 0
    n = ctx.halfspace_constraint_set(sc.dHat)
    act, _, _ = ctx.get_halfspace_sets()
    assert n == len(ref["act"]) and np.array_equal(act, ref["act"])
    assert rel(ctx.halfspace_energy(sc.dHat, sc.kappa), ref["E"]) <= 1e-10
    g = ctx.halfspace_gradient(sc.dHat, sc.kappa, np.zeros(3 * sc.m.nV))
    assert rel(g, ref["g"]) <= 1e-10
    a = ctx.halfspace_hessian(sc.dHat, sc.kappa, 1, np.zeros(ja.size))
    assert rel(a, ref["a"]) <= 1e-9 and np.linalg.norm(ref["a"]) > 0
    alpha, rc = ctx.halfspace_step(None, 0.9, 1.0)
    assert rc == 0 and scalar_bits(alpha) == scalar_bits(ref["alpha"]) and 0.0 < alpha < 1.0
    assert ctx.halfspace_crossings() == ref["cross"] == 0
    assert ctx.halfspace_friction_lag(sc.dHat, sc.kappa) == len(ref["lag"])
    _, lag, lam = ctx.get_halfspace_sets()
    assert np.array_equal(lag, ref["lag"]) and rel(lam, ref["lam"]) <= 1e-13
    # both friction branches occur
    u = (sc.m.V - sc.Vprev)[lag[:, 1]] - sc.vdt[lag[:, 0]]
    nn = sc.par[lag[:, 0], :3]
    u -= (u * nn).sum(1)[:, None] * nn
    slide = (u * u).sum(1) > sc.eps2
    assert slide.any() and (~slide).any()
    assert rel(ctx.halfspace_friction_energy(sc.eps2), ref["Ef"]) <= 1e-10
    gf = ctx.halfspace_friction_gradient(sc.eps2, np.zeros(3 * sc.m.nV))
    assert rel(gf, ref["gf"]) <= 1e-10
    af = ctx.halfspace_friction_hessian(sc.eps2, 1, np.zeros(ja.size))
    assert rel(af, ref["af"]) <= 1e-9
    # the plane blocks sit in the vertices' diagonal blocks only
    rows = np.repeat(np.arange(ia.size - 1), np.diff(ia))
    cols = ja - 1
    assert not (a[rows // 3 != cols // 3]).any() and not (af[rows // 3 != cols // 3]).any()


def test_crossing_and_zero_step(ctx):
    sc = Small()
    V = sc.m.V.copy()
    ia, ja = upload_with_csr(ctx, sc, V)
    v = int(sc.m.SVI[np.argsort(sc.m.V[sc.m.SVI, 1])][2])  # not Dirichlet, codimension 3
    V[v, 1] = sc.origin[0, 1]                               # exactly on the floor
    ctx.set_state(soa(V))
    ctx.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
    s = OH.HalfSpaces(orc.Surf(sc.m, V=V), sc.par)
    assert ctx.halfspace_crossings() == s.crossings() == 1
    alpha, rc = ctx.halfspace_step(None, 0.9, 1.0)
    assert rc == L.ERR_LINE_SEARCH and alpha == 0.0 and s.step(sc.p, 0.9, 1.0) == 0.0
    ctx.step_bound_set(1.0)
    ctx.halfspace_step(None, 0.9, None)
    assert ctx.lib.ipcgpu_fetch_iteration(ctx.h, L.C.byref(L.Iteration())) == L.ERR_LINE_SEARCH
    assert ctx.fetch_iteration().status == 0  # reported once


def deferred_sequence(ctx, sc):
    ctx.halfspace_constraint_set(sc.dHat, want=False)
    ctx.halfspace_crossings(want=False)
    ctx.halfspace_energy(sc.dHat, sc.kappa, want=False)
    ctx.halfspace_friction_energy(sc.eps2, want=False)
    ctx.csr_set_zero()
    ctx.step_bound_set(1.0)
    ctx.halfspace_step(None, 0.9, None)
    ctx.halfspace_gradient(sc.dHat, sc.kappa)
    ctx.halfspace_hessian(sc.dHat, sc.kappa, 1)
    ctx.halfspace_friction_gradient(sc.eps2)
    ctx.halfspace_friction_hessian(sc.eps2, 1)


def run_eager_reference(ctx, sc, ia, ja):
    """every stage in its host-output form at the current state"""
    n = ctx.halfspace_constraint_set(sc.dHat)
    E = ctx.halfspace_energy(sc.dHat, sc.kappa)
    Ef = ctx.halfspace_friction_energy(sc.eps2)
    alpha, _ = ctx.halfspace_step(None, 0.9, 1.0)
    g = ctx.halfspace_gradient(sc.dHat, sc.kappa, np.zeros(3 * sc.m.nV))
    g = ctx.halfspace_friction_gradient(sc.eps2, g)
    a = ctx.halfspace_hessian(sc.dHat, sc.kappa, 1, np.zeros(ja.size))
    a = ctx.halfspace_friction_hessian(sc.eps2, 1, a)
    return n, E, Ef, alpha, g, a, ctx.get_halfspace_sets()[0]


@pytest.mark.parametrize("captured", [False, True])
def test_deferred_and_captured_equal_eager(ctx, captured):
    sc = Small()
    ia, ja = upload_with_csr(ctx, sc)
    ctx.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
    ctx.set_canonical_order(0)
    ctx.halfspace_constraint_set(sc.dHat)
    ctx.halfspace_friction_lag(sc.dHat, sc.kappa)  # lagged once, at the first state (held through the time step)
    g_dev = np.zeros(3 * sc.m.nV)
    deferred_sequence(ctx, sc)  # eager run first: lazy allocations
    ctx.fetch_iteration()
    gid = None
    if captured:
        ctx.capture_begin()
        deferred_sequence(ctx, sc)
        gid = ctx.capture_end()
    rng = np.random.default_rng(3)
    states = [sc.m.V, sc.m.V + 0.2 * np.sqrt(sc.dHat) * rng.standard_normal(sc.m.V.shape)]
    for V in states:
        ctx.set_state(soa(V))
        n, E, Ef, alpha, g, a, act = run_eager_reference(ctx, sc, ia, ja)
        ref = oracle_all(sc, V, ia, ja)
        assert n == len(ref["act"]) and scalar_bits(alpha) == scalar_bits(ref["alpha"]) and rel(E, ref["E"]) <= 1e-10
        ctx.set_state(soa(V))
        ctx.fetch_iteration()
        ctx.set_search_dir(sc.p)
        ctx.elastic_gradient(0.0, want=False)  # a zero device gradient: the derivative calls accumulate into it
        if captured:
            ctx.graph_launch(gid)
        else:
            deferred_sequence(ctx, sc)
        it = ctx.fetch_iteration()
        assert it.status == 0 and it.n_halfspace_active == n and it.n_halfspace_crossings == 0
        assert scalar_bits(it.alpha_halfspace) == scalar_bits(alpha) and scalar_bits(it.alpha) == scalar_bits(alpha)
        assert rel(it.energy_halfspace, E) <= 1e-12 and rel(it.energy_halfspace_friction, Ef) <= 1e-12
        act2, _, _ = ctx.get_halfspace_sets()
        assert np.array_equal(act2, act)
        ctx.download_into(L.BUF_GRADIENT, g_dev)
        assert rel(g_dev, g) <= 1e-12
        a_dev = ctx.download(L.BUF_CSR_VALUES, ja.size)
        assert rel(a_dev, a) <= 1e-12
    if gid is not None:
        ctx.graph_destroy(gid)


def test_device_pattern_holds_the_plane_blocks(ctx):
    sc = Small()
    ia, ja = upload_with_csr(ctx, sc)
    ctx.enable_device_pattern(1)
    ctx.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0)
    ctx.halfspace_constraint_set(sc.dHat)
    changed, nnz = ctx.update_pattern(0)  # the planes add no off-diagonal block
    assert changed == 0
    ia2, ja2 = ctx.get_pattern()
    ref = oracle_all(sc, sc.m.V, ia2, ja2)
    a = ctx.halfspace_hessian(sc.dHat, sc.kappa, 1, np.zeros(ja2.size))
    assert rel(a, ref["a"]) <= 1e-9
    ctx.set_csr(ia, ja, 1)


def iteration_calls(ctx, sc, planes):
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    ctx.halfspace_constraint_set(sc.dHat, want=False)
    ctx.barrier_energy(sc.dHat, sc.kappa, want=False)
    ctx.halfspace_energy(sc.dHat, sc.kappa, want=False)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.halfspace_step(None, 0.9, None)
    ctx.halfspace_crossings(want=False)
    ctx.barrier_gradient(sc.dHat, sc.kappa)
    ctx.halfspace_gradient(sc.dHat, sc.kappa)
    ctx.halfspace_hessian(sc.dHat, sc.kappa, 1)
    return ctx.fetch_iteration()


def test_no_planes_launch_nothing(ctx):
    sc = Small()
    counts, alphas = [], []
    for setting in ("never", "removed"):
        with own_context() as c:
            upload_with_csr(c, sc)
            if setting == "removed":
                c.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
                c.set_halfspaces([], [])
            n0 = c.launch_count()
            it = iteration_calls(c, sc, False)
            counts.append(c.launch_count() - n0)
            alphas.append(scalar_bits(it.alpha))
            assert it.n_halfspace_active == 0 and it.energy_halfspace == 0.0
    assert counts[0] == counts[1] and alphas[0] == alphas[1]


# ---- the line search with planes against an oracle driver ---------------------------------------------------------------------------
def ls_scene(scale, drop, gap, plane_fric):
    """test_gpu_step_control's Armijo scene (FCR, inertia, self friction, two cubes in contact), its direction scaled by `scale` and pushed down
    `drop` along y towards a floor `gap` sqrt(dHat) below its lowest vertex, the plane friction `plane_fric`"""
    import test_gpu_step_control as SC
    sc = SC.scene_armijo()
    m = sc.m
    sq = np.sqrt(sc.dHat)
    sc.P = scale * sc.P
    sc.P[:, 1] -= drop
    sc.p = np.ascontiguousarray(sc.P).ravel()
    sc.fric = (sc.fric[0], sc.fric[1], m.V - 1e-3 * sc.P)
    sc.plane = ([[0.0, m.V[:, 1].min() - gap * sq, 0.0]], [[0.0, 1.0, 0.0]], [[1e-4, 0.0, 0.0]], [plane_fric])
    sc.par = OH.planes(*sc.plane)
    return sc


def _energy_parts(sc, V, sets):
    """E_el + E_in, E_b, E_f of Optimizer::computeEnergyVal at V (the self-contact sets `sets`)"""
    import oracle as orc_
    m = sc.m
    e, _ = orc_.Elastic(m, V=V).energy(sc.coef)
    if sc.xtilde is not None:
        e += float(np.sum(np.sum((V - sc.xtilde) ** 2, axis=1) * m.mass / 2.0))
    s = orc_.Surf(m, V=V)
    eb, bad = s.barrier_energy(sets[0], sets[1], sets[2], sc.dHat, sc.kappa)
    assert bad == 0
    ef = s.friction_energy(sc.fric[2], *sc.lag, sc.fric[0], sc.fric[1]) if sc.fric is not None else 0.0
    return e, eb, ef


def oracle_line_search_planes(sc, planes):
    """Optimizer::lineSearch (:2662-2916, armijoParam = 0) as test_gpu_step_control.oracle_line_search restates it, with the planes' parts:
    every trial rebuilds the plane set next to the contact set, its energy is orc_hs_trial_energy's, and isIntersected (:2627-2642) adds
    the planes' crossing check to both intersection loops.  The entry step is the planes' bound (slackness 0.9) when planes is True, else
    the same number."""
    import test_gpu_step_control as SC
    m, V0 = sc.m, sc.m.V.copy()
    SC.orc_lag(sc)
    Vt = soa(sc.fric[2])
    hs0 = OH.HalfSpaces(orc.Surf(m, V=V0), sc.par)
    act0 = hs0.constraint_set(sc.dHat)
    lagged = hs0.lag(act0, sc.dHat, sc.kappa) if sc.fric[0] > 0.0 else None
    alpha = hs0.step(sc.p, 0.9, 1.0)
    r = dict(counts=[0, 0, 0, 0], stopped=False, rebuilt=False, status=0, margins=[], alpha0=alpha, n_act=len(act0))

    def energy(V, sets, act):
        parts = _energy_parts(sc, V, sets)
        if not planes:
            return (parts[0] + parts[1]) + parts[2]
        E, bad = OH.trial_energy(OH.HalfSpaces(orc.Surf(m, V=V), sc.par), Vt, act, sc.dHat, sc.kappa, lagged, sc.fric[0], *parts)
        assert bad == 0
        return E

    def sets_at(V):
        return SC.orc_sets(sc, V), (OH.HalfSpaces(orc.Surf(m, V=V), sc.par).constraint_set(sc.dHat) if planes else None)

    def intersected(V):
        bad = not orc.Surf(m, V=V).intersection_free()[0]
        return bad or (planes and OH.HalfSpaces(orc.Surf(m, V=V), sc.par).crossings() > 0)

    E0 = energy(V0, SC.orc_sets(sc, V0), act0)
    step = lambda a: V0 + a * sc.P
    a = alpha
    while intersected(step(a)):
        if a == 0.0:
            return dict(r, alpha=0.0, status=L.ERR_LINE_SEARCH)
        a /= 2.0
        r["counts"][1] += 1
    V = step(a)
    sets, act = sets_at(V)
    Et, LF = energy(V, sets, act), a
    while True:
        r["margins"].append(abs(Et - E0) / abs(E0))
        if not Et > E0:
            break
        a /= 2.0
        r["counts"][2] += 1
        if a == 0.0:
            r["stopped"] = True
            break
        V = step(a)
        sets, act = sets_at(V)
        Et = energy(V, sets, act)
    if a < LF:
        ran = False
        while intersected(V):
            a /= 2.0
            r["counts"][3] += 1
            V, ran = step(a), True
        if ran:
            r["rebuilt"] = True
    return dict(r, alpha=a, E0=E0, Et=Et, LF=LF)


# (scale, drop, gap, plane friction): the Armijo loop halves twice with the planes and not at all without them (asserted on the oracle below)
LS_CASE = (0.1, 0.5, 0.3, 0.4)


def ls_upload(ctx, sc, canonical):
    import test_gpu_step_control as SC
    SC.load_step_scene(ctx, sc, canonical=canonical)  # mesh, surface, state, p, xTilta, contact sets, prev state, self-friction lag
    ctx.set_halfspaces(*sc.plane)
    ctx.halfspace_constraint_set(sc.dHat)
    ctx.halfspace_friction_lag(sc.dHat, sc.kappa)


def ls_entry(ctx, sc, planes, alpha0):
    """the entry state of the search: positions, the sets held on entry, the step (the planes' bound, or the same number without planes)"""
    ctx.set_state(sc.m.V_soa)
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    ctx.step_bound_set(1.0 if planes else alpha0)
    if planes:
        ctx.halfspace_constraint_set(sc.dHat, want=False)
        ctx.halfspace_step(None, 0.9, None)


def test_line_search_with_planes_matches_oracle(ctx):
    import test_gpu_step_control as SC
    sc = ls_scene(*LS_CASE)
    ref = oracle_line_search_planes(sc, True)
    ref0 = oracle_line_search_planes(sc, False)
    assert ref["status"] == 0 and min(ref["margins"]) > SC.MARGIN and min(ref0["margins"]) > SC.MARGIN and ref["n_act"] > 0
    assert ref["counts"][2] > 0 == ref0["counts"][2], (ref["counts"], ref0["counts"])  # the plane terms make the Armijo loop halve
    t = sc.terms()
    for canonical in (1, 0):
        ls_upload(ctx, sc, canonical)
        for planes, want in ((True, ref), (False, ref0)):
            if not planes:
                ctx.set_halfspaces([], [])
            ls_entry(ctx, sc, planes, ref["alpha0"])
            assert ctx.line_search(**t, check=False) == 0
            e = ctx.step_control_info()
            assert e.status == 0
            assert scalar_bits(e.alpha) == scalar_bits(want["alpha"]) and SC.counts(e) == want["counts"], (planes, e.alpha, want["alpha"], SC.counts(e), want["counts"])
            assert bool(e.stopped) == want["stopped"] and bool(e.post_check_rebuilt) == want["rebuilt"] and scalar_bits(e.alpha_feasible) == scalar_bits(want["LF"])
            assert rel(e.energy_start, want["E0"]) <= 1e-10 and rel(e.energy, want["Et"]) <= 1e-10
            if canonical:
                continue
            # captured (lists in arbitrary order), replayed from the same entry state
            ls_entry(ctx, sc, planes, ref["alpha0"])
            ctx.fetch_iteration()
            ctx.capture_begin()
            ctx.line_search(**t)
            gid = ctx.capture_end()
            ls_entry(ctx, sc, planes, ref["alpha0"])
            ctx.graph_launch(gid)
            g = ctx.step_control_info()
            assert g.status == 0 and scalar_bits(g.alpha) == scalar_bits(want["alpha"]) and SC.counts(g) == want["counts"]
            assert rel(g.energy, want["Et"]) <= 1e-10 and rel(g.energy_start, want["E0"]) <= 1e-10
            ctx.graph_destroy(gid)


def test_two_ranks_match_the_oracle():
    """tests/mp/halfspace_check.py on two GPUs (skipped with fewer)"""
    import os
    import subprocess
    import sys
    try:
        n = int(subprocess.check_output(["nvidia-smi", "-L"], text=True).count("GPU "))
    except Exception:
        n = 0
    if n < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29617",
           os.path.join(root, "tests", "mp", "halfspace_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "HALFSPACE_CHECK world=2 OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_larger_surface_on_the_same_context(ctx):
    """planes on a small surface, then a larger surface on the same context: the scan's temporary storage follows the surface"""
    small = Small()
    upload_with_csr(ctx, small)
    ctx.set_halfspaces(small.origin, small.normal, small.vdt, small.friction)
    assert ctx.halfspace_constraint_set(small.dHat) == len(oracle_all(small, small.m.V, *small.m.csr_pattern(1))["act"])
    m, info = scenes.ball_pile(64, res=10, seed=7, height=8)
    assert m.SVI.size > 8 * small.m.SVI.size
    load_scene(ctx, m)
    sq = np.sqrt(info["dHat"])
    origin, normal = [[0.0, m.V[:, 1].min() - 0.5 * sq, 0.0], [m.V[:, 0].max() + 0.5 * sq, 0.0, 0.0]], [[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]]
    ctx.set_halfspaces(origin, normal, None, [0.0, 0.0])
    par = OH.planes(origin, normal, None, [0.0, 0.0])
    ref = OH.HalfSpaces(orc.Surf(m), par).constraint_set(info["dHat"])
    assert len(ref) > 0
    assert ctx.halfspace_constraint_set(info["dHat"]) == len(ref)
    assert np.array_equal(ctx.get_halfspace_sets()[0], ref)


def test_c5_captured_iteration_with_a_ground_plane():
    """C5 (146 x sphere1K.msh, 1M tets) with a ground plane 0.5 sqrt(dHat) below the lowest vertex and a downward component in p: the captured
    iteration with the plane stages against the oracle -- plane set, energy, gradient and Hessian, and the step after the inversion filter,
    the plane bound (binding: below the inversion step) and the partial CCD, bit for bit"""
    import bench

    class Args:
        tets, res, scene = 1_000_000, 10, "c5"
    m, info = bench.build_scene(Args())
    dHat, kappa, tol, h = info["dHat"], bench.KAPPA, bench.TI_TOL, m.avgEdgeLen / 3
    sq = np.sqrt(dHat)
    P = np.array(info["p"], dtype=np.float64).reshape(-1, 3)
    P[:, 1] -= 6.0 * sq
    p = np.ascontiguousarray(P).ravel()
    origin, normal = [[0.0, m.V[:, 1].min() - 0.5 * sq, 0.0]], [[0.0, 1.0, 0.0]]
    with own_context() as ctx:
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_canonical_order(0)
        ctx.set_state(m.V_soa)
        ctx.set_search_dir(p)
        ctx.set_halfspaces(origin, normal, None, [0.0])
        evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)

        def iteration():
            ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
            ctx.halfspace_constraint_set(dHat, want=False)
            ctx.halfspace_energy(dHat, kappa, want=False)
            ctx.halfspace_crossings(want=False)
            ctx.csr_set_zero()
            ctx.elastic_gradient(0.0, want=False)
            ctx.halfspace_gradient(dHat, kappa)
            ctx.halfspace_hessian(dHat, kappa, 1)
            ctx.step_bound_set(1.0)
            ctx.inversion_step(None, 0.2, None)
            ctx.halfspace_step(None, 0.9, None)
            ctx.ccd_partial(None, tol, evf, eee, None)
            ctx.hash_build_swept(None, None, h)
            ctx.ccd_full(tol, evf, eee, None)

        iteration()  # eager first: lazy allocations
        ctx.fetch_iteration()
        ctx.capture_begin()
        iteration()
        gid = ctx.capture_end()
        ctx.graph_launch(gid)
        it = ctx.fetch_iteration()
        assert it.status == 0
        s = orc.Surf(m)
        hs = OH.HalfSpaces(s, OH.planes(origin, normal, None, [0.0]))
        act = hs.constraint_set(dHat)
        assert len(act) > 0 and it.n_halfspace_active == len(act) and np.array_equal(ctx.get_halfspace_sets()[0], act)
        E_ref, bad = hs.energy(act, dHat, kappa)
        assert bad == 0 and rel(it.energy_halfspace, E_ref) <= 1e-10 and it.n_halfspace_crossings == hs.crossings() == 0
        g = np.empty(3 * m.nV)
        ctx.download_into(L.BUF_GRADIENT, g)
        assert rel(g, hs.gradient(act, dHat, kappa)) <= 1e-10
        a = ctx.download(L.BUF_CSR_VALUES, ja.size)
        assert rel(a, hs.hessian_csr(act, dHat, kappa, ia, ja, 1)) <= 1e-9
        a_inv, _ = orc.Elastic(m).inversion_step(p, 0.2, 1.0)
        assert rel(it.alpha_inversion, a_inv) <= 1e-9  # (the inversion filter's own tolerance)
        a_hs = hs.step(p, 0.9, it.alpha_inversion)       # the plane bound of the step that entered it
        assert scalar_bits(it.alpha_halfspace) == scalar_bits(a_hs) and a_hs < it.alpha_inversion  # ... binding
        nC, nP, nK = ctx.constraint_set_sizes()
        mm, pa, pe, cand = np.empty((nC, 4), np.int32), np.empty((nP, 4), np.int32), np.empty((nP, 2), np.int32), np.empty((nK, 2), np.int32)
        ctx._ck(ctx.lib.ipcgpu_get_constraint_set(ctx.h, L._i(mm), L._i(pa), L._i(pe), L._i(cand)))
        a_part, _ = orc.ccd_partial(s, p, cand, tol, evf, eee, a_hs, nthreads=8)
        assert scalar_bits(it.alpha_partial_ccd) == scalar_bits(a_part) and it.alpha_full_ccd <= a_part
        ctx.graph_destroy(gid)
