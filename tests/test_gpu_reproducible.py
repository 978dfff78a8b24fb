"""The reproducible mode (ipcgpu_set_canonical_order(ctx, 2)): every contact sum in an order fixed by the lists alone.
The same sets handed in two random orders give bit-identical E, g and CSR values; level 2 stays within the parity bars of level 0; a
captured Newton iteration replays to the bits of the eager calls; two fresh contexts follow one trajectory; and the switch's contract."""
import numpy as np
import pytest

import oracle as orc
import oracle_codim as oc
import oracle_kappa as ok
from gpu_common import load_scene, own_context, rel, same_bits, scalar_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import scenes
from stagecheck import sort_rows

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2
TOL = 1e-6
KAPPA = 1e6
EPS2 = 1e-6
FRIC = 0.3


def mat_scene():
    """ball_on_mat with the ball lowered to half a contact distance over the mat, two planes under the mat (a vertex near the bottom is
    active for both) and a sliding previous state for the friction terms"""
    m, info = scenes.ball_on_mat(nx=24, res=5, seed=3)
    sq = np.sqrt(info["dHat"])
    nm = info["n_mat_verts"]
    m.V[nm:, 2] -= info["gap"] - 0.5 * sq
    z0 = m.V[:nm, 2].min() - 0.4 * sq
    planes = dict(origin=np.array([[0.0, 0.0, z0], [0.0, 0.0, z0]]), normal=np.array([[0.0, 0.0, 1.0], [0.05, 0.0, 1.0]]),
                  friction=np.array([0.2, 0.1]))
    Vprev = m.V.copy()
    Vprev[:, 0] -= 0.3 * sq
    return m, info, planes, Vprev


def pile_scene():
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    V = m.V.copy()
    return m, info, None, V - 0.2 * np.sqrt(info["dHat"]) * np.array([1.0, 0.0, 0.0])


def codim_scene():
    """pin_cushion (points, segments and triangles against a tet body): negative first components and codimensional stencils"""
    m = oc.pin_cushion()
    rng = np.random.default_rng(1)
    m.V = m.V_rest + 2e-3 * rng.standard_normal(m.V_rest.shape) * (m.dbc == 0)[:, None]
    m.V[m.dbc != 0, 1] += 0.01  # the scripted segments move toward the ball
    Vprev = m.V.copy()
    Vprev[:, 0] -= 0.01
    return m, dict(dHat=0.03 ** 2), None, Vprev


SCENES = {"ball_on_mat_planes": mat_scene, "ball_pile": pile_scene, "codim_pin_cushion": codim_scene}


def load_at_level(ctx, m, planes, Vprev, level):
    load_scene(ctx, m)
    ctx.set_prev_state(soa(Vprev))
    if planes is not None:
        ctx.set_halfspaces(planes["origin"], planes["normal"], friction=planes["friction"])
    else:  # (plane definitions outlive set_mesh)
        ctx.set_halfspaces([], [])
    ctx.set_canonical_order(level)


def terms(ctx, m, info, planes, nnz):
    """E, g and CSR values of every contact term at the lists the context holds (host-output forms)"""
    dHat, n = info["dHat"], 3 * m.nV
    E = [ctx.barrier_energy(dHat, KAPPA), ctx.friction_energy(EPS2, FRIC)]
    g = ctx.barrier_gradient(dHat, KAPPA, np.zeros(n))
    g = ctx.friction_gradient(EPS2, FRIC, g)
    a = ctx.barrier_hessian(dHat, KAPPA, 1, np.zeros(nnz))
    a = ctx.friction_hessian(EPS2, FRIC, 1, a)
    if planes is not None:
        E += [ctx.halfspace_energy(dHat, KAPPA), ctx.halfspace_friction_energy(EPS2)]
        g = ctx.halfspace_friction_gradient(EPS2, ctx.halfspace_gradient(dHat, KAPPA, g))
        a = ctx.halfspace_friction_hessian(EPS2, 1, ctx.halfspace_hessian(dHat, KAPPA, 1, a))
    return np.array(E), g, a


def build_sets(ctx, info, planes):
    dHat = info["dHat"]
    lists = ctx.constraint_set(dHat, 1)
    ctx.friction_lag(dHat, KAPPA)
    if planes is not None:
        ctx.halfspace_constraint_set(dHat)
        ctx.halfspace_friction_lag(dHat, KAPPA)
    ctx.update_pattern(1, want=False)
    return lists


# ---- 1. order independence ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_order_independence(shared_ctx, name):
    ctx = shared_ctx
    m, info, planes, Vprev = SCENES[name]()
    load_at_level(ctx, m, planes, Vprev, 2)
    ctx.enable_device_pattern(1)
    mm, pa, pe, _ = build_sets(ctx, info, planes)
    fr = ctx.get_friction_data()
    assert len(mm) >= (1 if name.startswith("codim") else 20) and len(fr[0]) == len(mm)
    _, ja = ctx.get_pattern()
    ref = terms(ctx, m, info, planes, len(ja))
    rng = np.random.default_rng(11)
    for trial in range(2):
        q, r, f = rng.permutation(len(mm)), rng.permutation(len(pa)), rng.permutation(len(fr[0]))
        ctx.set_constraint_set(mm[q], pa[r], pe[r])
        ctx.set_friction_data(*(x[f] for x in fr))
        got = ctx.constraint_set_sizes()
        assert got[:2] == (len(mm), len(pa))
        E, g, a = terms(ctx, m, info, planes, len(ja))
        assert same_bits(E, ref[0]) and same_bits(g, ref[1]) and same_bits(a, ref[2]), (name, trial)
        fr2 = ctx.get_friction_data()
        assert all(np.array_equal(x, y) for x, y in zip(fr2, fr))  # the uploaded list comes back in canonical order


# ---- 2. parity with level 0 ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SCENES))
def test_level2_matches_level0(shared_ctx, name):
    ctx = shared_ctx
    m, info, planes, Vprev = SCENES[name]()
    out = {}
    for level in (0, 2, 1):
        load_at_level(ctx, m, planes, Vprev, level)
        ctx.enable_device_pattern(1)
        mm, pa, pe, _ = build_sets(ctx, info, planes)
        ia, ja = ctx.get_pattern()
        out[level] = (mm, pa, pe, ia, ja) + terms(ctx, m, info, planes, len(ja))
    s0, s1, s2 = out[0], out[1], out[2]
    for k in range(3):  # level 2's lists are level 1's, bit for bit; level 0's are the same multiset
        assert np.array_equal(s2[k], s1[k])
    mm_r, pa_r, pe_r, _ = orc.Surf(m).constraint_set(info["dHat"])  # ... and the oracle's sets
    assert all(np.array_equal(x, y) for x, y in zip(sort_rows(s2[0]) + sort_rows(s2[1], s2[2]), sort_rows(mm_r) + sort_rows(pa_r, pe_r)))
    assert np.array_equal(s2[3], s0[3]) and np.array_equal(s2[4], s0[4])
    E0, g0, a0 = s0[5:]
    E2, g2, a2 = s2[5:]
    assert np.all(np.abs(E2 - E0) <= 1e-10 * np.maximum(np.abs(E0), 1e-300))
    assert rel(g2, g0) <= 1e-10 and rel(a2, a0) <= 1e-9


# ---- 3. captured equals eager, 4. two contexts, one trajectory -----------------------------------------------------------------------
def newton_iteration(ctx, m, info, evf, eee):
    """INTEGRATION.md section 4 with friction and planes: every call in its NULL-output form"""
    dHat = info["dHat"]
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.halfspace_constraint_set(dHat, want=False)
    ctx.update_pattern(1, want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, KAPPA, None)
    ctx.barrier_hessian(dHat, KAPPA, 1, None)
    ctx.friction_gradient(EPS2, FRIC, None)
    ctx.friction_hessian(EPS2, FRIC, 1, None)
    ctx.halfspace_gradient(dHat, KAPPA, None)
    ctx.halfspace_hessian(dHat, KAPPA, 1, None)
    ctx.halfspace_friction_gradient(EPS2, None)
    ctx.halfspace_friction_hessian(EPS2, 1, None)
    ctx.solve_pcg_multilevel(rel_tol=1e-8, max_iter=5000, want_x=False, adopt=True, deferred=True)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    ctx.ccd_cfl(dHat, 1, m.avgEdgeLen / 3.0, TOL, evf, eee, None)
    ctx.line_search(DT2, dHat, KAPPA, fric_eps2=EPS2, fric_coef=FRIC)


def snapshot(ctx, m):
    n = 3 * m.nV
    s, v = ctx.step_control_info(), ctx.solve_info()
    it = ctx.fetch_iteration()
    assert it.status == 0 and s.status == 0 and v.status == 0
    _, ja = ctx.get_pattern()
    return dict(V=ctx.download(L.BUF_POSITIONS, n), g=ctx.download(L.BUF_GRADIENT, n), a=ctx.download(L.BUF_CSR_VALUES, len(ja)),
                scalars=np.array([s.alpha, s.energy_start, s.energy]), counts=tuple(getattr(s, f) for f, _ in s._fields_ if f.startswith("halvings")) + (v.iterations,))


def start(ctx, m, info, planes, Vprev):
    load_at_level(ctx, m, planes, Vprev, 2)
    ctx.enable_device_pattern(1)
    ctx.constraint_set(info["dHat"], 1, fetch=False, sizes=False)
    ctx.friction_lag(info["dHat"], KAPPA, want=False)
    ctx.halfspace_constraint_set(info["dHat"], want=False)
    ctx.halfspace_friction_lag(info["dHat"], KAPPA, want=False)


def test_captured_iteration_equals_eager(shared_ctx):
    m, info, planes, Vprev = mat_scene()
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    g_ctx = shared_ctx
    with own_context() as e_ctx:
        for c in (g_ctx, e_ctx):
            start(c, m, info, planes, Vprev)
        newton_iteration(g_ctx, m, info, evf, eee)  # the eager run: lazy allocations
        g_ctx.fetch_iteration()
        g_ctx.set_state(soa(m.V))
        g_ctx.capture_begin()
        newton_iteration(g_ctx, m, info, evf, eee)
        gid = g_ctx.capture_end()
        for k in range(3):
            newton_iteration(e_ctx, m, info, evf, eee)
            e = snapshot(e_ctx, m)
            g_ctx.graph_launch(gid)
            g = snapshot(g_ctx, m)
            assert e["scalars"][0] > 0.0
            for key in ("V", "g", "a", "scalars"):
                assert same_bits(g[key], e[key]), (k, key)
            assert g["counts"] == e["counts"], k
        g_ctx.graph_destroy(gid)


def test_two_contexts_one_trajectory():
    m, info, planes, Vprev = mat_scene()
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    runs = []
    for _ in range(2):
        with own_context() as ctx:
            start(ctx, m, info, planes, Vprev)
            newton_iteration(ctx, m, info, evf, eee)  # eager first (lazy allocations), then replays from the same start
            ctx.fetch_iteration()
            ctx.set_state(soa(m.V))
            ctx.capture_begin()
            newton_iteration(ctx, m, info, evf, eee)
            gid = ctx.capture_end()
            traj = []
            for _ in range(4):
                ctx.graph_launch(gid)
                traj.append(snapshot(ctx, m))
            ctx.graph_destroy(gid)
            runs.append(traj)
    for k, (x, y) in enumerate(zip(*runs)):
        for key in ("V", "g", "a", "scalars"):
            assert same_bits(x[key], y[key]), (k, key)
        assert x["counts"] == y["counts"], k


# ---- 5. contract ---------------------------------------------------------------------------------------------------------------------
def test_contract(shared_ctx):
    ctx = shared_ctx
    m, info, planes, Vprev = mat_scene()
    with pytest.raises(L.IpcGpuError):
        ctx.set_canonical_order(3)
    start(ctx, m, info, planes, Vprev)
    ctx.capture_begin()
    ctx.constraint_set(info["dHat"], 1, fetch=False, sizes=False)  # level 2 inside a capture: accepted
    gid = ctx.capture_end()
    ctx.graph_launch(gid)
    ctx.set_canonical_order(2)  # a level change refuses the older graph
    with pytest.raises(L.IpcGpuError):
        ctx.graph_launch(gid)
    ctx.graph_destroy(gid)
    with own_context() as other:  # level 2 and several ranks: refused (before any collective is set up)
        other.set_canonical_order(2)
        with pytest.raises(L.IpcGpuError, match="STATE"):
            other.comm_init(0, 2, bytes(128))


def held_lists(ctx):
    """the lists the context holds, without a rebuild"""
    nC, nP, nK = ctx.constraint_set_sizes()
    mm, pa, pe, cand = (np.empty((n, k), dtype=np.int32) for n, k in ((nC, 4), (nP, 4), (nP, 2), (nK, 2)))
    ctx._ck(ctx.lib.ipcgpu_get_constraint_set(ctx.h, L._i(mm), L._i(pa), L._i(pe), L._i(cand)))
    return mm, pa, pe, cand


def test_level1_inside_a_capture(shared_ctx):
    """level 1 sorts sized on the device: a captured constraint set and line search replay to the eager calls' lists, which are the
    oracle's at the accepted step"""
    ctx = shared_ctx
    m, info, _, Vprev = pile_scene()
    dHat = info["dHat"]
    load_at_level(ctx, m, None, Vprev, 1)
    g = ctx.elastic_gradient(DT2) + ctx.barrier_gradient(dHat, KAPPA, np.zeros(3 * m.nV))
    p = -g / np.abs(g).max() * 0.5 * np.sqrt(dHat)  # a descent direction, at most half a contact distance per coordinate
    ctx.set_search_dir(p)

    def sequence():
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.step_bound_set(1.0)
        ctx.line_search(DT2, dHat, KAPPA)

    runs = []
    for captured in (False, True):
        ctx.set_state(soa(m.V))
        if captured:
            ctx.capture_begin()
            sequence()
            gid = ctx.capture_end()
            ctx.set_state(soa(m.V))
            ctx.graph_launch(gid)
            ctx.graph_destroy(gid)
        else:
            sequence()  # (also the eager run before the capture)
        s = ctx.step_control_info()
        assert s.status == 0 and s.alpha > 0.0
        runs.append((ctx.download(L.BUF_POSITIONS, 3 * m.nV), held_lists(ctx)))
    (V_e, eager), (V_g, replay) = runs
    assert same_bits(V_g, V_e) and all(np.array_equal(x, y) for x, y in zip(replay, eager))
    assert all(np.array_equal(x, y) for x, y in zip(eager, orc.Surf(m, V_e.reshape(3, -1).T).constraint_set(dHat)))
    assert len(eager[0]) > 0 and len(eager[3]) > 0


# ---- 4. five time steps: the time-integration frame, kappa on the device, a host-driven Newton loop over the captured iteration ----
KD = L.KAPPA_DEVICE
N_STEPS, N_ITERS = 5, 3


def step_start(ctx, info, s, mx, first):
    """the frame of a time step: end of the last step and warm start (x~ from compute_xtilde at the first), the lagged friction sets, and
    initKappa on the device"""
    dHat = info["dHat"]
    if not first:
        ctx.end_time_step()
        ctx.warm_start(2, info["voxel"], TOL, info["evf"], info["eee"], want=False)
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.halfspace_constraint_set(dHat, want=False)
    ctx.friction_lag(dHat, KD, want=False)
    ctx.halfspace_friction_lag(dHat, KD, want=False)
    ctx.set_kappa(s, s, mx)
    ctx.elastic_gradient(DT2, 1, 1, want=False)
    ctx.inertia_gradient(1, None)
    ctx.kappa_init(dHat)
    ctx.kappa_clear_close_set()


def kappa_iteration(ctx, m, info):
    dHat = info["dHat"]
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.halfspace_constraint_set(dHat, want=False)
    ctx.update_pattern(1, want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.inertia_gradient(1, None)
    ctx.barrier_gradient(dHat, KD, None)
    ctx.barrier_hessian(dHat, KD, 1, None)
    ctx.friction_gradient(EPS2, FRIC, None)
    ctx.friction_hessian(EPS2, FRIC, 1, None)
    ctx.halfspace_gradient(dHat, KD, None)
    ctx.halfspace_hessian(dHat, KD, 1, None)
    ctx.halfspace_friction_gradient(EPS2, None)
    ctx.halfspace_friction_hessian(EPS2, 1, None)
    ctx.solve_pcg_multilevel(rel_tol=1e-8, max_iter=5000, want_x=False, adopt=True, deferred=True)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, info["evf"], info["eee"], None)
    ctx.ccd_cfl(dHat, 1, m.avgEdgeLen / 3.0, TOL, info["evf"], info["eee"], None)
    ctx.line_search(DT2, dHat, KD, inertia=True, fric_eps2=EPS2, fric_coef=FRIC)
    ctx.kappa_post_line_search(dHat)


def test_five_time_steps_two_contexts():
    m, info, planes, Vprev = mat_scene()
    vel0 = np.zeros((m.nV, 3))
    vel0[info["n_mat_verts"]:, 2] = -0.05  # the ball moves down onto the mat, which lies on the two planes
    info = dict(info, voxel=m.avgEdgeLen / 3.0)
    info["evf"], info["eee"] = L.Context.ti_error(m.V_soa, m.nV, None)
    s, mx = ok.bounds(info["dHat"], 1e-11, float(np.mean(m.mass)), float(np.sum((m.V_rest.max(0) - m.V_rest.min(0)) ** 2)))
    runs = []
    for _ in range(2):
        with own_context() as ctx:  # a fresh context per run
            def reset():  # (nothing here refuses the graphs)
                ctx.set_state(soa(m.V))
                ctx.set_prev_state(soa(m.V))
                ctx.set_dynamics(vel0.ravel(), None, None)
                ctx.compute_xtilde()

            load_at_level(ctx, m, planes, m.V, 2)
            ctx.enable_device_pattern(1)
            ctx.set_time_integration(0, 0.025, gravity=(0.0, 0.0, -9.81))
            reset()
            for first in (True, False):  # the eager runs: lazy allocations (the warm start's streams too)
                step_start(ctx, info, s, mx, first)
                kappa_iteration(ctx, m, info)
                ctx.fetch_iteration()
            ctx.capture_begin()
            step_start(ctx, info, s, mx, False)
            gid_step = ctx.capture_end()
            ctx.capture_begin()
            kappa_iteration(ctx, m, info)
            gid_it = ctx.capture_end()
            reset()
            traj = []
            for k in range(N_STEPS):
                if k == 0:
                    step_start(ctx, info, s, mx, True)
                else:
                    ctx.graph_launch(gid_step)
                counts = []
                for _ in range(N_ITERS):  # the host-driven Newton loop: replay, read the iteration back
                    ctx.graph_launch(gid_it)
                    sc, sv, it = ctx.step_control_info(), ctx.solve_info(), ctx.fetch_iteration()
                    counts.append((sc.status, sv.status, it.status, sv.iterations, *(getattr(sc, f) for f, _ in sc._fields_ if f.startswith("halvings")),
                                   scalar_bits(sc.alpha), ctx.kappa_info().doublings))
                # (the mollified pairs' term alone, host form: augmentParaEEGradient with the device kappa)
                gp = ctx.para_ee_gradient(info["dHat"], KD, np.zeros(3 * m.nV))
                traj.append(dict(V=ctx.download(L.BUF_POSITIONS, 3 * m.nV), gp=gp, kappa=scalar_bits(ctx.kappa_info().kappa), counts=counts))
            ctx.graph_destroy(gid_step)
            ctx.graph_destroy(gid_it)
            runs.append(traj)
    a, b = runs
    for k in range(N_STEPS):
        assert same_bits(a[k]["V"], b[k]["V"]) and same_bits(a[k]["gp"], b[k]["gp"]), k
        assert a[k]["kappa"] == b[k]["kappa"] and a[k]["counts"] == b[k]["counts"], (k, a[k]["counts"], b[k]["counts"])
        assert all(c[0] == 0 and c[1] == 0 and c[2] == 0 and c[3] > 0 for c in a[k]["counts"]), a[k]["counts"]
    assert len({a[k]["V"].tobytes() for k in range(N_STEPS)}) == N_STEPS  # the bodies moved at every step
