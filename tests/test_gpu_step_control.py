"""The CFL branch of the step bound (ipcgpu_ccd_cfl_ti) and the line search (ipcgpu_line_search) against oracle drivers restated from
Optimizer.cpp:1947-2027 and Optimizer::lineSearch (Optimizer.cpp:2662-2916, armijoParam = 0, lowerBound = 0), eagerly and replayed from a
graph with conditional nodes."""

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, own_context, rel, scalar_bits, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

pytestmark = pytest.mark.gpu

TOL = 1e-6
MARGIN = 1e-9  # every energy comparison of the oracle driver must be decided by more than this (relative)


# ---- scenes -------------------------------------------------------------------------------------------------------------------
class Scene:
    def __init__(self, name, m, P, coef, dHat, kappa, xtilde=None, fric=None):
        self.name, self.m, self.P, self.coef, self.dHat, self.kappa, self.xtilde = name, m, np.asarray(P, dtype=np.float64), coef, dHat, kappa, xtilde
        self.p = np.ascontiguousarray(self.P).ravel()  # interleaved search direction
        self.fric = fric  # (eps2, coef, Vprev) or None
        self.lag = None   # lagged friction data at the entry state (oracle)

    def terms(self):
        fr = self.fric or (0.0, 0.0, None)
        return dict(elastic_coef=self.coef, dHat=self.dHat, kappa=self.kappa, inertia=self.xtilde is not None, fric_eps2=fr[0], fric_coef=fr[1])


def two_cubes(gap, n=3, shift=(0.1, 0.05), energy=1, density=1.0):
    V1, T1 = M.grid_tets(n, n, n, h=1.0 / n)
    V2, T2 = M.grid_tets(n, n, n, h=1.0 / n, origin=(shift[0], shift[1], 1.0 + gap))
    return M.merge_meshes([(V1, T1), (V2, T2)], energy=energy, density=density), len(V1)


def scene_armijo():
    """FCR, inertia on, friction on: a direction that overshoots the rest shape five times, two bodies in contact"""
    m, n1 = two_cubes(0.02)
    M.deform(m, 3, twist=0.2, amp=0.01, noise=0.01)
    P = 5.0 * (m.V_rest - m.V)
    Vprev = m.V - 1e-3 * P
    return Scene("armijo", m, P, 0.025 ** 2, 0.05 ** 2, 1e3, xtilde=m.V.copy(), fric=((1e-3 * m.avgEdgeLen) ** 2, 0.3, Vprev))


def scene_inversion():
    """Neo-Hookean cube squashed through itself along z at alpha = 1"""
    V, T = M.grid_tets(3, 3, 3, h=1.0 / 3)
    m = M.Mesh(V, T, energy=0, density=1.0)
    M.deform(m, 5, twist=0.1, amp=0.005, noise=0.005)
    P = np.zeros_like(m.V)
    P[:, 2] = -2.5 * (m.V[:, 2] - m.V[:, 2].mean())
    return Scene("inversion", m, P, 0.025 ** 2, 1e-3 ** 2, 1e3)


def scene_intersection():
    """the upper cube is pushed 0.4 into the lower one at alpha = 1; inertia pulls it down"""
    m, n1 = two_cubes(0.2)
    P = np.zeros_like(m.V)
    P[n1:, 2] = -0.6
    xt = m.V.copy()
    xt[n1:, 2] -= 0.2
    return Scene("intersection", m, P, 0.025 ** 2, 0.05 ** 2, 1e-2, xtilde=xt)


def scene_tunnel():
    """a small cube passes right through a slab at alpha = 1; inertia pulls it into the slab"""
    V1, T1 = M.grid_tets(4, 4, 1, h=0.25)
    V2, T2 = M.grid_tets(2, 2, 2, h=0.15, origin=(0.35, 0.35, 0.35))
    m = M.merge_meshes([(V1, T1), (V2, T2)], energy=1, density=1.0)
    n1 = len(V1)
    P = np.zeros_like(m.V)
    P[n1:, 2] = -0.75
    xt = m.V.copy()
    xt[n1:, 2] -= 0.3
    return Scene("tunnel", m, P, 0.025 ** 2, 1e-3 ** 2, 1.0, xtilde=xt)


SCENES = {f.__name__[6:]: f for f in (scene_armijo, scene_inversion, scene_intersection, scene_tunnel)}


# ---- oracle drivers -----------------------------------------------------------------------------------------------------------
def orc_sets(sc, V):
    return orc.Surf(sc.m, V=V).constraint_set(sc.dHat)


def orc_energy(sc, V, sets):
    """Optimizer::computeEnergyVal: ((E_el + E_in) + E_b) + E_f"""
    m = sc.m
    e, _ = orc.Elastic(m, V=V).energy(sc.coef)
    if sc.xtilde is not None:
        e += float(np.sum(np.sum((V - sc.xtilde) ** 2, axis=1) * m.mass / 2.0))
    s = orc.Surf(m, V=V)
    eb, bad = s.barrier_energy(sets[0], sets[1], sets[2], sc.dHat, sc.kappa)
    assert bad == 0
    e += eb
    if sc.fric is not None:
        e += s.friction_energy(sc.fric[2], *sc.lag, sc.fric[0], sc.fric[1])
    return e


def orc_lag(sc):
    """friction_lag at the entry state (Optimizer.cpp:1582-1600)"""
    if sc.fric is not None:
        mm = orc_sets(sc, sc.m.V)[0]
        sc.lag = (mm, *orc.Surf(sc.m, V=sc.m.V).friction_lag(mm, sc.dHat, sc.kappa))


def oracle_line_search(sc, alpha):
    """Optimizer::lineSearch (:2662-2916) with armijoParam = 0, lowerBound = 0, the loops ending at alpha == 0 as ipcgpu_line_search does"""
    m, V0 = sc.m, sc.m.V.copy()
    r = dict(counts=[0, 0, 0, 0], stopped=False, rebuilt=False, status=0, margins=[])
    if alpha == 0.0:
        return dict(r, alpha=0.0, status=L.ERR_LINE_SEARCH, V=V0)
    E0 = orc_energy(sc, V0, orc_sets(sc, V0))  # (the sets held on entry are the ones at V0)
    step = lambda a: V0 + a * sc.P

    def halve(a, k, bad):
        while bad(step(a)):
            if a == 0.0:
                return None
            a /= 2.0
            r["counts"][k] += 1
        return a

    a = alpha
    if m.energy == 0:  # getNeedElemInvSafeGuard: Neo-Hookean
        a = halve(a, 0, lambda V: orc.Elastic(m, V=V).count_inverted() > 0)
        if a is None:
            return dict(r, alpha=0.0, status=L.ERR_LINE_SEARCH, V=V0)
    a = halve(a, 1, lambda V: not orc.Surf(m, V=V).intersection_free()[0])
    if a is None:
        return dict(r, alpha=0.0, status=L.ERR_LINE_SEARCH, V=V0)
    V = step(a)
    sets = orc_sets(sc, V)
    Et, LF = orc_energy(sc, V, sets), a
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
        sets = orc_sets(sc, V)
        Et = orc_energy(sc, V, sets)
    if a < LF:
        ran = False
        while not orc.Surf(m, V=V).intersection_free()[0]:
            a /= 2.0
            r["counts"][3] += 1
            V, ran = step(a), True
        if ran:
            sets, r["rebuilt"] = orc_sets(sc, V), True
    return dict(r, alpha=a, E0=E0, Et=Et, LF=LF, V=V, sets=sets)


def oracle_cfl(sc, first, alpha_partial, evf, eee, voxel):
    """Optimizer.cpp:1947-2027 (CFL_FOR_CCD == 2) after the partial CCD"""
    s = orc.Surf(sc.m)
    pmag = np.sqrt((sc.P[s.SVI, 0] * sc.P[s.SVI, 0] + sc.P[s.SVI, 1] * sc.P[s.SVI, 1]) + sc.P[s.SVI, 2] * sc.P[s.SVI, 2])
    with np.errstate(divide="ignore"):
        cfl = np.sqrt(sc.dHat) / (pmag.max() * 2.0)
    a = alpha_partial
    full = bool((first and a > cfl) or a > 2.0 * cfl)
    if full:
        a, _, _ = orc.ccd_full_hashed(s, sc.p, a, voxel, TOL, evf, eee, nthreads=8)
        if a < cfl:
            a = cfl
    else:
        a = min(a, cfl)
    return a, float(cfl), full


# ---- device side --------------------------------------------------------------------------------------------------------------
def load_step_scene(ctx, sc, canonical=1):
    load_scene(ctx, sc.m)
    ctx.set_canonical_order(canonical)
    ctx.set_search_dir(sc.p)
    if sc.xtilde is not None:
        ctx.set_xtilde(soa(sc.xtilde))
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)  # the sets held on entry
    if sc.fric is not None:
        ctx.set_prev_state(soa(sc.fric[2]))
        ctx.friction_lag(sc.dHat, sc.kappa)


@pytest.fixture(scope="module")
def ctx():
    with own_context() as c:
        yield c


def fingerprint(ctx, sc):
    """positions, bit for bit, without a download of V: the per-tet elastic energies (shape) and two inertia sums (placement)"""
    m = sc.m
    ctx.elastic_energy(1.0)
    fp = [ctx.download(L.BUF_ENERGY_PER_TET, m.nT).tobytes()]
    for k in range(2):
        ctx.set_xtilde(soa(m.V_rest + 0.37 * (k + 1)))
        fp.append(scalar_bits(ctx.inertia_energy()))
    if sc.xtilde is not None:
        ctx.set_xtilde(soa(sc.xtilde))
    return fp


def stepped_fingerprint(ctx, sc, V0, alpha):
    """fingerprint of ipcgpu_step_forward(alpha) from V0"""
    ctx.set_state(soa(V0))
    ctx.save_state()
    ctx.step_forward(None, alpha)
    return fingerprint(ctx, sc)


def counts(info):
    return [info.halvings_inversion, info.halvings_intersection, info.halvings_armijo, info.halvings_post_check]


# ---- 1. the CFL branch ------------------------------------------------------------------------------------------------------------
def approaching_cubes(gap, speed):
    m, n1 = two_cubes(gap, energy=1)
    P = np.zeros_like(m.V)
    P[:n1, 2], P[n1:, 2] = speed, -speed
    return Scene("cfl", m, P, 0.025 ** 2, 0.05 ** 2, 1e3)


# (gap, speed, k == 0, dHat of the candidate set): the full CCD (k = 0) / not taken (k > 0, alpha_CFL < alpha <= 2 alpha_CFL) / unchanged /
# full CCD below alpha_CFL, clamped (the candidates of a smaller dHat miss the pair that the full CCD finds)
CFL_CASES = {"full": (0.2, 1.0, 1, 0.05 ** 2, True, False), "not_taken": (0.2, 0.0357, 0, 0.05 ** 2, False, False),
             "unchanged": (0.2, 0.01, 1, 0.05 ** 2, False, False), "clamped": (0.02, 1.0, 1, 0.01 ** 2, True, True)}


@pytest.mark.parametrize("case", list(CFL_CASES))
def test_cfl_branch_matches_oracle(ctx, case):
    gap, speed, first, dhat_cs, want_full, want_clamp = CFL_CASES[case]
    sc = approaching_cubes(gap, speed)
    m, voxel = sc.m, sc.m.avgEdgeLen / 3.0
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    cand = s.constraint_set(dhat_cs)[3]
    a_part, _ = orc.ccd_partial(s, sc.p, cand, TOL, evf, eee, 1.0, nthreads=8)
    a_ref, cfl, full = oracle_cfl(sc, first, a_part, evf, eee, voxel)
    assert full == want_full and (full and a_ref == cfl) == want_clamp, (case, a_part, cfl, a_ref)
    if case == "not_taken":
        assert not first and cfl < a_part <= 2.0 * cfl and a_ref == cfl
    if case == "unchanged":
        assert a_part <= cfl and a_ref == a_part
    load_step_scene(ctx, sc)
    ctx.constraint_set(dhat_cs, 1, fetch=False, sizes=False)
    a = ctx.ccd_partial(None, TOL, evf, eee, 1.0)
    assert scalar_bits(a) == scalar_bits(a_part)
    assert scalar_bits(ctx.ccd_cfl(sc.dHat, first, voxel, TOL, evf, eee, a)) == scalar_bits(a_ref)
    info = ctx.step_control_info()
    assert info.status == 0 and bool(info.full_ccd) == full and scalar_bits(info.alpha_cfl) == scalar_bits(cfl)
    # the device-resident form: the same step in ipcgpu_fetch_iteration, the stages of a skipped branch report it
    ctx.step_bound_set(1.0)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    ctx.ccd_cfl(sc.dHat, first, voxel, TOL, evf, eee, None)
    it = ctx.fetch_iteration()
    assert it.status == 0 and scalar_bits(it.alpha) == scalar_bits(a_ref)
    if not full:
        assert scalar_bits(it.alpha_swept_grid) == scalar_bits(it.alpha_full_ccd) == scalar_bits(a_ref)
    assert bool(ctx.step_control_info().full_ccd) == full


# ---- 2. the line search against the oracle driver -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_line_search_matches_oracle(ctx, name):
    sc = SCENES[name]()
    orc_lag(sc)
    ref = oracle_line_search(sc, 1.0)
    assert ref["status"] == 0 and min(ref["margins"]) > MARGIN
    load_step_scene(ctx, sc)
    rc, alpha = ctx.line_search(**sc.terms(), alpha=1.0)
    info = ctx.step_control_info()
    assert rc == 0 and info.status == 0
    assert scalar_bits(alpha) == scalar_bits(ref["alpha"]) == scalar_bits(info.alpha)
    assert counts(info) == ref["counts"] and bool(info.stopped) == ref["stopped"] and bool(info.post_check_rebuilt) == ref["rebuilt"]
    assert scalar_bits(info.alpha_feasible) == scalar_bits(ref["LF"])
    assert rel(info.energy_start, ref["E0"]) <= 1e-10 and rel(info.energy, ref["Et"]) <= 1e-10
    mm, pa, pe, cand = held_sets(ctx)
    for got, want in zip((mm, pa, pe, cand), ref["sets"]):
        assert np.array_equal(got, want)
    assert scalar_bits(ctx.fetch_iteration().alpha) == scalar_bits(ref["alpha"])
    fp = fingerprint(ctx, sc)
    assert fp == stepped_fingerprint(ctx, sc, sc.m.V, alpha)


def held_sets(ctx):
    nC, nP, nK = ctx.constraint_set_sizes()
    mm, pa = np.empty((nC, 4), np.int32), np.empty((nP, 4), np.int32)
    pe, cand = np.empty((nP, 2), np.int32), np.empty((nK, 2), np.int32)
    ctx._ck(ctx.lib.ipcgpu_get_constraint_set(ctx.h, L._i(mm), L._i(pa), L._i(pe), L._i(cand)))
    return mm, pa, pe, cand


# ---- 3. captured against eager ------------------------------------------------------------------------------------------------------
def step_control_sequence(ctx, sc, evf, eee, first=1):
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    ctx.ccd_cfl(sc.dHat, first, sc.m.avgEdgeLen / 3.0, TOL, evf, eee, None)
    t = sc.terms()
    t.update(fric_eps2=0.0, fric_coef=0.0)
    ctx.line_search(**t)


def prepare(ctx, sc, V, p):
    ctx.set_state(soa(V))
    ctx.set_search_dir(p)
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)


def test_captured_line_search_equals_eager(ctx):
    sc = scene_armijo()
    sc.fric = None
    load_step_scene(ctx, sc, canonical=0)
    evf, eee = L.Context.ti_error(sc.m.V_soa, sc.m.nV, None)
    # halvings of the Armijo loop on the oracle: 1, 0 and 2
    pairs = [(sc.m.V, sc.p), (sc.m.V, 0.05 * sc.p), (sc.m.V + 0.1 * sc.P, 2.0 * sc.p)]
    prepare(ctx, sc, *pairs[0])
    step_control_sequence(ctx, sc, evf, eee)  # eager run first: lazy allocations
    ctx.fetch_iteration()
    ctx.capture_begin()
    step_control_sequence(ctx, sc, evf, eee)
    gid = ctx.capture_end()
    seen = []
    for V, p in pairs:
        prepare(ctx, sc, V, p)
        step_control_sequence(ctx, sc, evf, eee)
        e = ctx.step_control_info()
        fe = fingerprint(ctx, sc)
        prepare(ctx, sc, V, p)
        n0 = ctx.launch_count()
        ctx.graph_launch(gid)
        g = ctx.step_control_info()
        assert ctx.launch_count() > n0
        assert g.status == e.status == 0
        assert scalar_bits(g.alpha) == scalar_bits(e.alpha) and scalar_bits(g.alpha_cfl) == scalar_bits(e.alpha_cfl) and g.full_ccd == e.full_ccd
        assert counts(g) == counts(e) and g.stopped == e.stopped and g.post_check_rebuilt == e.post_check_rebuilt
        assert rel(g.energy, e.energy) <= 1e-12 and rel(g.energy_start, e.energy_start) <= 1e-12
        assert fingerprint(ctx, sc) == fe
        seen.append(tuple(counts(e)))
    assert len(set(seen)) >= 3 and any(c[2] == 0 for c in seen), seen
    ctx.graph_destroy(gid)


def whole_iteration(ctx, sc, evf, eee):
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0, want=False)
    ctx.elastic_energy_grad_hess(sc.coef, 1, 1, 1)
    ctx.barrier_gradient(sc.dHat, sc.kappa, None)
    ctx.barrier_hessian(sc.dHat, sc.kappa, 1, None)
    step_control_sequence(ctx, sc, evf, eee)


def test_whole_iteration_graph(ctx):
    sc = scene_armijo()
    sc.fric = None
    load_step_scene(ctx, sc, canonical=0)
    ctx.enable_device_pattern(1)
    evf, eee = L.Context.ti_error(sc.m.V_soa, sc.m.nV, None)
    prepare(ctx, sc, sc.m.V, sc.p)
    whole_iteration(ctx, sc, evf, eee)
    ctx.fetch_iteration()
    # the same iteration without the line search: the body kernels of the conditional nodes must be counted as well
    ctx.capture_begin()
    ctx.constraint_set(sc.dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0, want=False)
    ctx.elastic_energy_grad_hess(sc.coef, 1, 1, 1)
    ctx.barrier_gradient(sc.dHat, sc.kappa, None)
    ctx.barrier_hessian(sc.dHat, sc.kappa, 1, None)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    gid0 = ctx.capture_end()
    hi0, lo0 = ctx.graph_kernel_priorities(gid0)
    ctx.capture_begin()
    whole_iteration(ctx, sc, evf, eee)
    gid = ctx.capture_end()
    hi, lo = ctx.graph_kernel_priorities(gid)
    assert lo == lo0 > 0 and hi > hi0 + 30, (hi0, lo0, hi, lo)
    for rep in range(2):
        prepare(ctx, sc, sc.m.V, sc.p)
        whole_iteration(ctx, sc, evf, eee)
        e, ie = ctx.step_control_info(), ctx.fetch_iteration()
        fe = fingerprint(ctx, sc)
        prepare(ctx, sc, sc.m.V, sc.p)
        ctx.graph_launch(gid)
        g, ig = ctx.step_control_info(), ctx.fetch_iteration()
        assert ig.status == ie.status == 0 and g.status == e.status == 0
        assert scalar_bits(g.alpha) == scalar_bits(e.alpha) == scalar_bits(ig.alpha) == scalar_bits(ie.alpha) and counts(g) == counts(e)
        assert rel(ig.energy_elastic, ie.energy_elastic) <= 1e-12 and rel(g.energy, e.energy) <= 1e-12
        assert fingerprint(ctx, sc) == fe
    ctx.graph_destroy(gid)
    ctx.graph_destroy(gid0)


# ---- 4. termination and refusals (eager) ------------------------------------------------------------------------------------------
def test_intersecting_entry_state_returns_zero_step(ctx):
    sc = scene_intersection()
    sc.m.V[sc.m.nV // 2:, 2] -= 0.4
    V0 = sc.m.V.copy()
    load_step_scene(ctx, sc)
    rc, alpha = ctx.line_search(**sc.terms(), alpha=1.0, check=False)
    info = ctx.step_control_info()
    assert rc == info.status == L.ERR_LINE_SEARCH and alpha == 0.0 and info.alpha == 0.0
    assert fingerprint(ctx, sc) == stepped_fingerprint(ctx, sc, V0, 0.0)
    ctx.fetch_iteration()


def test_zero_entry_step_runs_nothing(ctx):
    sc = scene_tunnel()
    load_step_scene(ctx, sc)
    fp0 = fingerprint(ctx, sc)
    n0 = ctx.launch_count()
    rc, alpha = ctx.line_search(**sc.terms(), alpha=0.0, check=False)
    assert rc == L.ERR_LINE_SEARCH and alpha == 0.0
    assert ctx.launch_count() - n0 == 2  # the step set and the entry decision
    assert fingerprint(ctx, sc) == fp0


def test_line_search_refused_without_a_search_direction(ctx):
    sc = scene_tunnel()
    load_step_scene(ctx, sc, canonical=1)
    m = sc.m
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)  # forgets the search direction
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_state(m.V_soa)
    with pytest.raises(L.IpcGpuError, match="STATE"):
        ctx.line_search(**sc.terms(), alpha=1.0)
