"""Rayleigh damping, Neumann forces and the augmented-Lagrangian Dirichlet penalty on the device against the restatements of
tests/oracle_damping.py: D added into the CSR (host pattern and device-built pattern), energies and gradients for projectDBC = 0 and 1, the
penalty's lambda update and completed step, the line search with each term against an oracle driver, and a captured iteration replayed after
rho doubles and lambda updates."""

import numpy as np
import pytest

import oracle as orc
import oracle_damping as OD
import test_gpu_step_control as SC
from gpu_common import own_context, rel, scalar_bits, soa
from ipc_b200 import lib as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    with own_context() as c:
        yield c


def scene(energy):
    """two cubes in contact (test_gpu_step_control's Armijo scene, Neo-Hookean or FCR), a ZERO and a NONZERO Dirichlet vertex at the bottom (the
    ZERO one does not move), V_prev = V - 1e-3 p, Dirichlet targets on every third vertex"""
    sc = SC.scene_armijo()
    m = sc.m
    if energy != m.energy:
        m.energy = energy
    lo = np.argsort(m.V[:, 2])[:2]
    m.dbc[lo[0]], m.dbc[lo[1]] = 1, 2
    sc.P[lo[0]] = 0.0
    sc.p = np.ascontiguousarray(sc.P).ravel()
    sc.Vprev = sc.fric[2]
    rng = np.random.default_rng(11)
    sc.vid = np.arange(0, m.nV, 3).astype(np.int32)
    sc.tgt = m.V[sc.vid] + 0.01 * rng.standard_normal((sc.vid.size, 3))
    sc.lam = rng.standard_normal((sc.vid.size, 3))
    sc.f = rng.standard_normal((m.nV, 3))
    return sc


def load_step_scene_csr(ctx, sc, canonical=1):
    SC.load_step_scene(ctx, sc, canonical=canonical)  # mesh, surface, state, p, xTilta, contact sets, V_prev, friction lag
    ia, ja = sc.m.csr_pattern(1)
    ctx.set_csr(ia, ja, 1)
    return ia, ja


# ---- D in the CSR -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("energy", [0, 1])
def test_damping_matrix_host_and_device_pattern(ctx, energy):
    sc = scene(energy)
    m, coef = sc.m, 0.3
    ia, ja = load_step_scene_csr(ctx, sc)
    D = OD.damping_matrix(m, m.V, coef)
    assert np.array_equal(D[0], ia) and np.array_equal(D[1], ja)
    ctx.damping_update(coef)
    a = ctx.damping_hessian(np.zeros(ja.size))
    assert rel(a, D[2]) <= 1e-9
    for v in np.flatnonzero(m.dbc):  # the identity of the reference's setCoeff
        for r in range(3):
            assert a[ia[3 * v + r] - 1] == 1.0
    # the device-built pattern, augmented by the contact blocks
    ctx.enable_device_pattern(1)
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    changed, nnz = ctx.update_pattern(0)
    ia2, ja2 = ctx.get_pattern()
    assert changed and nnz > ja.size
    ctx.csr_set_zero()
    ctx.damping_hessian(None)
    a2 = ctx.download(L.BUF_CSR_VALUES, nnz)
    assert rel(a2, OD.scatter(ia, ja, D[2], ia2, ja2)) <= 1e-9


# ---- energies and gradients ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("energy", [0, 1])
@pytest.mark.parametrize("projectDBC", [0, 1])
def test_energies_and_gradients(ctx, energy, projectDBC):
    sc = scene(energy)
    m, coef, dt2, rho = sc.m, 0.3, 1e-2, 1e3
    ia, ja = load_step_scene_csr(ctx, sc)
    V = m.V
    D = OD.damping_matrix(m, V, coef)
    ctx.damping_update(coef)
    assert rel(ctx.damping_energy(), OD.damping_energy(D, V, sc.Vprev, m.dbc)) <= 1e-10
    g = ctx.damping_gradient(projectDBC, np.zeros(3 * m.nV))
    assert rel(g, OD.damping_gradient(D, V, sc.Vprev, m.dbc, projectDBC)) <= 1e-10
    ctx.set_neumann_forces(dt2, sc.f)
    assert rel(ctx.neumann_energy(), OD.neumann_energy(V, sc.f, m.mass, m.dbc, dt2)) <= 1e-10
    g = ctx.neumann_gradient(np.zeros(3 * m.nV))
    assert rel(g, OD.neumann_gradient(sc.f, m.mass, m.dbc, dt2)) <= 1e-10
    ctx.set_dirichlet_targets(sc.vid, sc.tgt, sc.lam, 1e-6)
    ctx.set_dirichlet_penalty(rho)
    assert rel(ctx.dirichlet_energy(), OD.mdbc_energy(V, sc.vid, sc.tgt, sc.lam, m.mass, rho)) <= 1e-10
    g = ctx.dirichlet_gradient(projectDBC, np.zeros(3 * m.nV))
    want = OD.mdbc_gradient(V, sc.vid, sc.tgt, sc.lam, m.mass, rho, m.nV) if not projectDBC else np.zeros(3 * m.nV)
    assert rel(g, want) <= 1e-10 if not projectDBC else not g.any()
    a = ctx.dirichlet_hessian(projectDBC, np.zeros(ja.size))
    want = np.zeros(ja.size)
    if not projectDBC:
        want[ia[:-1] - 1] = OD.mdbc_hessian_diag(sc.vid, m.mass, rho, m.nV)
    assert rel(a, want) <= 1e-12 if not projectDBC else not a.any()
    # the deferred forms: the fetch reports the same energies
    for f in (ctx.damping_energy, ctx.neumann_energy, ctx.dirichlet_energy):
        f(want=False)
    it = ctx.fetch_iteration()
    assert it.energy_damping == ctx.damping_energy() and it.energy_neumann == ctx.neumann_energy() and it.energy_dirichlet == ctx.dirichlet_energy()
    # rho = 0: nothing at all
    ctx.set_dirichlet_penalty(0.0)
    assert ctx.dirichlet_energy() == 0.0
    g0 = np.arange(3 * m.nV, dtype=np.float64)
    assert np.array_equal(ctx.dirichlet_gradient(0, g0.copy()), g0)
    ctx.set_dirichlet_targets([], [])
    ctx.set_neumann_forces(0.0, None)
    ctx.damping_update(0.0)


def test_lambda_update_and_completed_step(ctx):
    sc = scene(1)
    m, rho, tol = sc.m, 2e3, 1e-5
    load_step_scene_csr(ctx, sc)
    ctx.set_dirichlet_targets(sc.vid, sc.tgt, sc.lam, tol)
    ctx.set_dirichlet_penalty(rho)
    s = ctx.dirichlet_completed_step()
    assert rel(s, OD.mdbc_completed_step(m.V, sc.vid, sc.tgt, tol)) <= 1e-12
    ctx.dirichlet_completed_step(want=False)
    assert rel(ctx.fetch_iteration().dirichlet_completed_step, s) <= 1e-15
    ctx.dirichlet_update_lambda()
    lam1 = OD.mdbc_update_lambda(m.V, sc.vid, sc.tgt, sc.lam, m.mass, rho)
    assert rel(ctx.get_dirichlet_lambda(), lam1) <= 1e-14
    ctx.set_dirichlet_targets(sc.vid, sc.tgt, None, 0.0)
    assert ctx.dirichlet_completed_step() == 1.0 and not ctx.get_dirichlet_lambda().any()
    ctx.set_dirichlet_targets([], [])


def test_refusals_and_a_new_mesh(ctx):
    """repeated target vertices are refused (targetPos is a map); a new mesh removes the three terms and their energies read 0"""
    sc = scene(1)
    m = sc.m
    load_step_scene_csr(ctx, sc)
    with pytest.raises(L.IpcGpuError, match="ARG"):
        ctx.set_dirichlet_targets([3, 5, 3], np.zeros((3, 3)))
    ctx.damping_update(0.3)
    ctx.set_neumann_forces(1e-2, sc.f)
    ctx.set_dirichlet_targets(sc.vid, sc.tgt, sc.lam, 1e-6)
    ctx.set_dirichlet_penalty(1e3)
    for f in (ctx.damping_energy, ctx.neumann_energy, ctx.dirichlet_energy):
        f(want=False)
    it = ctx.fetch_iteration()
    assert it.energy_damping != 0.0 and it.energy_neumann != 0.0 and it.energy_dirichlet != 0.0
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    it = ctx.fetch_iteration()
    assert it.energy_damping == it.energy_neumann == it.energy_dirichlet == 0.0
    with pytest.raises(L.IpcGpuError, match="STATE"):
        ctx.damping_energy()
    with pytest.raises(L.IpcGpuError, match="STATE"):
        ctx.neumann_energy()
    assert ctx.dirichlet_energy() == 0.0  # (no targets: nothing)
    ctx.set_dirichlet_penalty(0.0)


# ---- the line search with each term against an oracle driver -------------------------------------------------------------------------
def oracle_line_search(sc, extra):
    """test_gpu_step_control.oracle_line_search (FCR: no inversion guard) with the trial energy
    ((((((E_el + E_in) + E_nbc) + E_b) + E_f) + E_damp) + E_dbc, the terms of `extra` only"""
    m, V0 = sc.m, sc.m.V.copy()
    SC.orc_lag(sc)

    def energy(V, sets):
        e, _ = orc.Elastic(m, V=V).energy(sc.coef)
        e += float(np.sum(np.sum((V - sc.xtilde) ** 2, axis=1) * m.mass / 2.0))
        if "nbc" in extra:
            e += extra["nbc"](V)
        s = orc.Surf(m, V=V)
        eb, bad = s.barrier_energy(sets[0], sets[1], sets[2], sc.dHat, sc.kappa)
        assert bad == 0
        e += eb
        e += s.friction_energy(sc.fric[2], *sc.lag, sc.fric[0], sc.fric[1])
        if "damp" in extra:
            e += extra["damp"](V)
        if "dbc" in extra:
            e += extra["dbc"](V)
        return e

    r = dict(counts=[0, 0, 0, 0], margins=[])
    E0 = energy(V0, SC.orc_sets(sc, V0))
    step = lambda a: V0 + a * sc.P
    a = 1.0
    while not orc.Surf(m, V=step(a)).intersection_free()[0]:
        a /= 2.0
        r["counts"][1] += 1
    V = step(a)
    Et, LF = energy(V, SC.orc_sets(sc, V)), a
    while True:
        r["margins"].append(abs(Et - E0) / abs(E0))
        if not Et > E0:
            break
        a /= 2.0
        r["counts"][2] += 1
        V = step(a)
        Et = energy(V, SC.orc_sets(sc, V))
    assert a == LF or orc.Surf(m, V=V).intersection_free()[0]  # (no post-check halving in these scenes)
    return dict(r, alpha=a, E0=E0, Et=Et)


# term -> (switch on, switch off, oracle energy) with the parameters that make the Armijo loop halve more often than without the term
def _terms(sc):
    m = sc.m
    coef, k, rho = 0.003, -10.0, 1e3
    D = OD.damping_matrix(m, m.V, coef)
    f = k * sc.P / np.linalg.norm(sc.P, axis=1).max()
    vid, tgt = sc.vid, m.V[sc.vid].copy()
    lam = np.zeros((vid.size, 3))

    def on_dbc(c):
        c.set_dirichlet_targets(vid, tgt, lam, 1e-6)
        c.set_dirichlet_penalty(rho)
    return {
        "damp": (lambda c: c.damping_update(coef), lambda c: c.damping_update(0.0), lambda V: OD.damping_energy(D, V, sc.Vprev, m.dbc)),
        "nbc": (lambda c: c.set_neumann_forces(1.0, f), lambda c: c.set_neumann_forces(0.0, None), lambda V: OD.neumann_energy(V, f, m.mass, m.dbc, 1.0)),
        "dbc": (on_dbc, lambda c: c.set_dirichlet_targets([], []), lambda V: OD.mdbc_energy(V, vid, tgt, lam, m.mass, rho)),
    }


@pytest.mark.parametrize("term", ["damp", "nbc", "dbc"])
def test_line_search_with_each_term_matches_oracle(ctx, term):
    sc = scene(1)
    on, off, e_ref = _terms(sc)[term]
    ref = oracle_line_search(sc, {term: e_ref})
    ref0 = oracle_line_search(sc, {})
    assert min(ref["margins"]) > SC.MARGIN and min(ref0["margins"]) > SC.MARGIN
    assert ref["alpha"] <= ref0["alpha"] / 2.0 and ref["counts"][2] > ref0["counts"][2], (ref["counts"], ref0["counts"])
    load_step_scene_csr(ctx, sc)
    for with_term, want in ((True, ref), (False, ref0)):
        (on if with_term else off)(ctx)
        ctx.set_state(sc.m.V_soa)
        ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
        rc, alpha = ctx.line_search(**sc.terms(), alpha=1.0)
        e = ctx.step_control_info()
        assert rc == 0 and e.status == 0
        assert scalar_bits(alpha) == scalar_bits(want["alpha"]) and SC.counts(e) == want["counts"], (term, with_term, alpha, want["alpha"], SC.counts(e), want["counts"])
        assert rel(e.energy_start, want["E0"]) <= 1e-10 and rel(e.energy, want["Et"]) <= 1e-10


def test_zero_rho_leaves_the_line_search_bit_identical(ctx):
    sc = scene(1)
    load_step_scene_csr(ctx, sc)
    out = []
    for targets in (False, True):
        if targets:
            ctx.set_dirichlet_targets(sc.vid, sc.tgt, sc.lam, 1e-6)
            ctx.set_dirichlet_penalty(0.0)
        ctx.set_state(sc.m.V_soa)
        ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
        ctx.line_search(**sc.terms(), alpha=1.0)
        e = ctx.step_control_info()
        out.append((scalar_bits(e.alpha), scalar_bits(e.energy_start), scalar_bits(e.energy), tuple(SC.counts(e))))
    assert out[0] == out[1]
    ctx.set_dirichlet_targets([], [])


# ---- a captured iteration replayed after rho doubles and lambda updates ----------------------------------------------------------------
def test_captured_penalty_iteration_equals_eager(ctx):
    sc = scene(1)
    sc.fric = (sc.fric[0], 0.0, sc.fric[2])  # (friction off in the search: the captured line search needs no lag refresh)
    m = sc.m
    ia, ja = load_step_scene_csr(ctx, sc, canonical=0)
    ctx.enable_device_pattern(1)
    ctx.damping_update(0.003)
    ctx.set_neumann_forces(1e-2, sc.f)
    ctx.set_dirichlet_targets(sc.vid, sc.tgt, sc.lam, 1e-6)
    rho = 1e3
    ctx.set_dirichlet_penalty(rho)
    t = sc.terms()
    t.update(fric_eps2=0.0, fric_coef=0.0)

    def iteration():
        ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(0, want=False)
        ctx.elastic_energy_grad_hess(sc.coef, 1, 0, 1)
        ctx.barrier_gradient(sc.dHat, sc.kappa, None)
        ctx.barrier_hessian(sc.dHat, sc.kappa, 0, None)
        ctx.damping_gradient(0)
        ctx.damping_hessian()
        ctx.neumann_gradient()
        ctx.dirichlet_gradient(0)
        ctx.dirichlet_hessian(0)
        ctx.step_bound_set(1.0)
        ctx.line_search(**t)
        ctx.dirichlet_completed_step(want=False)

    def results():
        it, e = ctx.fetch_iteration(), ctx.step_control_info()
        g = np.empty(3 * m.nV)
        ctx.download_into(L.BUF_GRADIENT, g)
        nnz = ctx.pattern_info()[1]
        return it, e, g, ctx.download(L.BUF_CSR_VALUES, nnz)

    def entry():
        ctx.set_state(m.V_soa)
        ctx.set_search_dir(sc.p)

    entry()
    iteration()  # eager first: lazy allocations
    ctx.fetch_iteration()
    ctx.capture_begin()
    iteration()
    gid = ctx.capture_end()
    seen, steps = set(), set()
    for rep in range(4):
        if rep in (1, 2):
            rho *= 2.0
            ctx.set_dirichlet_penalty(rho)
            ctx.dirichlet_update_lambda()
        if rep == 3:  # the next time step's targets: the same number, new positions, the current multipliers and a new dist2Tol
            ctx.set_dirichlet_targets(sc.vid, sc.tgt + 0.005, ctx.get_dirichlet_lambda(), 4e-6)
        entry()
        iteration()
        ie, ee, ge, ae = results()
        entry()
        ctx.graph_launch(gid)  # (the same graph: refused if anything had required a new capture)
        ig, eg, gg, ag = results()
        assert ig.status == ie.status == 0 and eg.status == ee.status == 0
        assert scalar_bits(eg.alpha) == scalar_bits(ee.alpha) and SC.counts(eg) == SC.counts(ee)
        assert rel(eg.energy, ee.energy) <= 1e-12 and rel(eg.energy_start, ee.energy_start) <= 1e-12  # (contact lists in arbitrary order)
        assert scalar_bits(ig.dirichlet_completed_step) == scalar_bits(ie.dirichlet_completed_step)
        assert rel(gg, ge) <= 1e-12 and rel(ag, ae) <= 1e-12
        seen.add(scalar_bits(ee.energy_start))
        steps.add(scalar_bits(ie.dirichlet_completed_step))
    assert len(seen) == 4 and len(steps) == 4  # rho, lambda and the new targets reached the objective and the completed step
    ctx.graph_destroy(gid)
    ctx.set_canonical_order(1)
    ctx.damping_update(0.0)
    ctx.set_neumann_forces(0.0, None)
    ctx.set_dirichlet_targets([], [])


# ---- C5 size ------------------------------------------------------------------------------------------------------------------------
def test_c5_damping_matches_oracle():
    """C5 (146 x sphere1K.msh, 1M tets): D, its energy and its gradient against the oracle"""
    import bench

    class Args:
        tets, res, scene = 1_000_000, 10, "c5"
    m, info = bench.build_scene(Args())
    with own_context() as ctx:
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        P = np.array(info["p"], dtype=np.float64).reshape(-1, 3)
        Vprev = m.V - 1e-2 * P
        ctx.set_prev_state(soa(Vprev))
        coef = 0.1
        ctx.damping_update(coef)
        a = ctx.damping_hessian(np.zeros(ja.size))
        a_ref = orc.Elastic(m).hessian_csr(coef, ia, ja, 1, 1, 1, nthreads=8)
        assert rel(a, a_ref) <= 1e-9
        D = (ia, ja, a_ref)
        assert rel(ctx.damping_energy(), OD.damping_energy(D, m.V, Vprev, m.dbc)) <= 1e-10
        g = ctx.damping_gradient(1, np.zeros(3 * m.nV))
        assert rel(g, OD.damping_gradient(D, m.V, Vprev, m.dbc, 1)) <= 1e-10
