"""ipcgpu_precondition_diag and ipcgpu_warm_start option 5 (initX's Jacobi predictor) on the device-resident gradient and matrix, against the
float64 restatement of tests/oracle_jacobi.py over the downloaded g and a, bit for bit: both signs, host and device-built patterns,
projected and penalty-mode Dirichlet rows; the adopted direction against the same vector uploaded; the warm start against the oracle driver;
captured against eager; the refusals and the non-finite status."""
import numpy as np
import pytest

import oracle_codim as oc
import oracle_halfspace as OH
import oracle_jacobi as OJ
import oracle_timestep as OT
from gpu_common import load_scene, own_context, same_bits, scalar_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2
TOL = 1e-6
KAPPA = 1e6
EPS2 = 1e-6
FRIC = 0.3


def mat_scene():
    """ball_on_mat lowered to half a contact distance over the mat, two friction planes under it, a sliding previous state, and a fixed
    mat corner (Dirichlet)"""
    m, info = scenes.ball_on_mat(nx=24, res=5, seed=3)
    sq = np.sqrt(info["dHat"])
    nm = info["n_mat_verts"]
    m.V[nm:, 2] -= info["gap"] - 0.5 * sq
    z0 = m.V[:nm, 2].min() - 0.4 * sq
    planes = dict(origin=np.array([[0.0, 0.0, z0], [0.0, 0.0, z0]]), normal=np.array([[0.0, 0.0, 1.0], [0.05, 0.0, 1.0]]),
                  friction=np.array([0.2, 0.1]))
    m.dbc[np.argsort(m.V[:nm, 0] + m.V[:nm, 1])[:6]] = 1
    Vprev = m.V.copy()
    Vprev[:, 0] -= 0.3 * sq
    return m, info, planes, Vprev


def codim_scene():
    """pin_cushion: points, segments and triangles against a tet body, with scripted (Dirichlet) segments; barrier terms only (the
    friction terms are exercised on ball_on_mat)"""
    m = oc.pin_cushion()
    m.V = m.V_rest.copy()
    m.V[m.dbc != 0, 1] += 0.01  # the scripted segments move toward the ball (the body stays at rest: no inverted tet)
    Vprev = m.V.copy()
    Vprev[:, 0] -= 0.01
    return m, dict(dHat=0.03 ** 2, friction=False), None, Vprev


SCENES = {"ball_on_mat_planes": mat_scene, "codim_pin_cushion": codim_scene}


def start(ctx, m, info, planes, Vprev, level=1):
    """scene, contact sets at V, the lagged friction, the device-built pattern (index base 1)"""
    dHat = info["dHat"]
    load_scene(ctx, m)
    ctx.set_prev_state(soa(Vprev))
    ctx.set_halfspaces(planes["origin"], planes["normal"], friction=planes["friction"]) if planes is not None else ctx.set_halfspaces([], [])
    ctx.set_canonical_order(level)
    ctx.enable_device_pattern(1)
    ctx.constraint_set(dHat, 1)
    if info.get("friction", True):
        ctx.friction_lag(dHat, KAPPA)
    if planes is not None:
        ctx.halfspace_constraint_set(dHat)
        ctx.halfspace_friction_lag(dHat, KAPPA)
    ctx.update_pattern(1 if info.get("friction", True) else 0, want=False)


def assemble(ctx, info, planes, projectDBC=1):
    """computeGradient + computePrecondMtr of the incremental potential's terms, every call in its NULL-output form"""
    dHat = info["dHat"]
    ctx.elastic_energy_grad_hess(DT2, 1, projectDBC, 1)
    ctx.barrier_gradient(dHat, KAPPA, None)
    ctx.barrier_hessian(dHat, KAPPA, projectDBC, None)
    if info.get("friction", True):
        ctx.friction_gradient(EPS2, FRIC, None)
        ctx.friction_hessian(EPS2, FRIC, projectDBC, None)
    if planes is not None:
        ctx.halfspace_gradient(dHat, KAPPA, None)
        ctx.halfspace_hessian(dHat, KAPPA, projectDBC, None)
        ctx.halfspace_friction_gradient(EPS2, None)
        ctx.halfspace_friction_hessian(EPS2, projectDBC, None)


def resident(ctx, m, pattern):
    """g, the CSR values and (ia, base) as the device holds them"""
    ia = pattern[0]
    return ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, len(pattern[1])), ia, pattern[2]


# ---- 1. the direction, bit for bit ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("projectDBC", [1, 0])
@pytest.mark.parametrize("pattern", ["device", "host"])
@pytest.mark.parametrize("name", list(SCENES))
def test_direction_bit_identical(shared_ctx, name, pattern, projectDBC):
    ctx = shared_ctx
    m, info, planes, Vprev = SCENES[name]()
    start(ctx, m, info, planes, Vprev)
    ia, ja = ctx.get_pattern()
    pat = (ia, ja, 1)
    if pattern == "host":  # the same structure handed in from the host, index base 0
        pat = (ia - 1, ja - 1, 0)
        ctx.set_csr(pat[0], pat[1], 0)
    assemble(ctx, info, planes, projectDBC)
    g, a, ia, base = resident(ctx, m, pat)
    assert np.abs(g).max() > 0.0
    fixed = np.repeat(m.dbc != 0, 3)
    for sign in (-1, 1):
        ref = OJ.precondition_diag(g, ia, a, base, sign)
        assert np.isfinite(ref).all()
        x = ctx.precondition_diag(sign)
        s = ctx.solve_info()
        assert same_bits(x, ref), (name, pattern, projectDBC, sign)
        assert s.status == 0 and s.iterations == 0 and s.rel_residual == 0.0
        assert same_bits(s.max_abs_x, np.abs(ref).max())
        if fixed.any() and projectDBC:  # identity rows: divided by 1, no special case (0 where the terms leave the row's gradient at 0)
            assert (a[ia[:-1][fixed] - base] == 1.0).all() and same_bits(ref[fixed], sign * g[fixed])
        # the deferred form, adopted: the search direction holds the same bits
        assert ctx.precondition_diag(sign, want_x=False, adopt=True) is None
        assert same_bits(ctx.download(L.BUF_SEARCH_DIR, 3 * m.nV), ref)
        assert same_bits(ctx.solve_info().max_abs_x, np.abs(ref).max())


# ---- 2. adopted against uploaded ----------------------------------------------------------------------------------------------------
def stages(ctx, m, info, evf, eee):
    """inversion filter, swept build, full CCD, then the line search from the full CCD's step"""
    a_inv = ctx.inversion_step(None, 0.2, 1.0)
    a_grid = ctx.hash_build_swept(None, a_inv, m.avgEdgeLen / 3.0)
    a_full, _ = ctx.ccd_full(TOL, evf, eee, a_grid)
    rc, a = ctx.line_search(DT2, info["dHat"], KAPPA, fric_eps2=EPS2, fric_coef=FRIC, alpha=a_full, check=False)
    s = ctx.step_control_info()
    out = dict(a_inv=a_inv, a_grid=a_grid, a_full=a_full, a=a, rc=rc,
               counts=(s.halvings_inversion, s.halvings_intersection, s.halvings_armijo, s.halvings_post_check),
               V=ctx.download(L.BUF_POSITIONS, 3 * m.nV))
    ctx.fetch_iteration()
    return out


def test_adopted_equals_uploaded(shared_ctx):
    ctx = shared_ctx
    m, info, planes, Vprev = mat_scene()
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    runs = []
    for adopt in (True, False):
        start(ctx, m, info, planes, Vprev, level=2)  # (fixed-order contact sums: both runs assemble the same g)
        assemble(ctx, info, planes)
        x = ctx.precondition_diag(-1, adopt=adopt)
        if not adopt:
            ctx.set_search_dir(x)
        runs.append(stages(ctx, m, info, evf, eee))
    d, u = runs
    assert d["rc"] == u["rc"] == 0 and d["a"] > 0.0
    for k in ("a_inv", "a_grid", "a_full", "a", "V"):
        assert same_bits(d[k], u[k]), k
    assert d["counts"] == u["counts"]


# ---- 3. warm start option 5 against the oracle driver ------------------------------------------------------------------------------
def test_warm_start_jacobi_matches_oracle(shared_ctx):
    ctx = shared_ctx
    m, info, planes, Vprev = mat_scene()
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    voxel = m.avgEdgeLen / 3.0
    start(ctx, m, info, planes, Vprev)
    ia, ja = ctx.get_pattern()
    assemble(ctx, info, planes)
    g, a, ia, base = resident(ctx, m, (ia, ja, 1))
    rc, alpha = ctx.warm_start(5, voxel, TOL, evf, eee, check=False)
    sc, it = ctx.step_control_info(), ctx.fetch_iteration()
    p = OJ.jacobi_predictor(g, ia, a, base, m.dbc)
    assert same_bits(ctx.download(L.BUF_SEARCH_DIR, 3 * m.nV), p)
    par = OH.planes(planes["origin"], planes["normal"])
    ref = OJ.warm_start(m, p, voxel, TOL, evf, eee, lambda s: OH.HalfSpaces(s, par), alpha_inversion=it.alpha_inversion)
    assert rc == ref["status"] == sc.status == 0
    for got, key in ((it.alpha_halfspace, "alpha_halfspace"), (it.alpha_swept_grid, "alpha_swept_grid"), (it.alpha_full_ccd, "alpha_full_ccd"),
                     (alpha, "alpha"), (sc.alpha, "alpha")):
        assert same_bits(got, ref[key]), key
    assert [sc.halvings_inversion, sc.halvings_intersection] == ref["counts"]
    V = ctx.download(L.BUF_POSITIONS, 3 * m.nV).reshape(3, m.nV).T
    assert same_bits(V, ref["V"])
    assert 0.0 < alpha and np.array_equal(V[m.dbc != 0], m.V[m.dbc != 0]) and not np.array_equal(V, m.V)


# ---- 4. captured against eager ------------------------------------------------------------------------------------------------------
def fallback_iteration(ctx, info, planes):
    """assemble -> the diagonally preconditioned direction, adopted -> line search"""
    assemble(ctx, info, planes)
    ctx.precondition_diag(-1, want_x=False, adopt=True)
    ctx.step_bound_set(1.0)
    ctx.line_search(DT2, info["dHat"], KAPPA, fric_eps2=EPS2, fric_coef=FRIC)


def frame(ctx, info, planes, evf, eee, voxel):
    """end of step -> assemble at the new state -> warm start 5"""
    ctx.end_time_step()
    assemble(ctx, info, planes)
    ctx.warm_start(5, voxel, TOL, evf, eee, want=False)


def test_captured_equals_eager(shared_ctx):
    ctx = shared_ctx
    m, info, planes, Vprev = mat_scene()
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    voxel, n = m.avgEdgeLen / 3.0, 3 * m.nV
    vel = np.zeros((m.nV, 3))
    vel[info["n_mat_verts"]:, 2] = -0.5

    def reset():
        ctx.set_state(soa(m.V))
        ctx.set_prev_state(soa(Vprev))
        ctx.set_dynamics(vel.ravel(), None, None)
        ctx.compute_xtilde()
        ctx.constraint_set(info["dHat"], 1, fetch=False, sizes=False)
        ctx.halfspace_constraint_set(info["dHat"], want=False)

    def snapshot():
        s, v = ctx.step_control_info(), ctx.solve_info()
        it = ctx.fetch_iteration()
        return (ctx.download(L.BUF_POSITIONS, n).tobytes(), ctx.download(L.BUF_SEARCH_DIR, n).tobytes(), scalar_bits(s.alpha),
                scalar_bits(v.max_abs_x), s.halvings_inversion, s.halvings_intersection, s.halvings_armijo, s.halvings_post_check,
                s.status, v.status, it.status)

    start(ctx, m, info, planes, Vprev, level=2)
    ctx.set_time_integration(OT.BE, 0.01)
    for seq in (lambda: fallback_iteration(ctx, info, planes), lambda: frame(ctx, info, planes, evf, eee, voxel)):
        reset()
        seq()  # eager: lazy allocations, streams of the conditional nodes
        eager = snapshot()
        assert eager[-3:] == (0, 0, 0) and eager[0] != soa(m.V).tobytes()
        reset()
        ctx.capture_begin()
        seq()
        gid = ctx.capture_end()
        for _ in range(2):
            reset()
            ctx.graph_launch(gid)
            assert snapshot() == eager
        ctx.graph_destroy(gid)


# ---- 5. refusals and the non-finite status ------------------------------------------------------------------------------------------
def test_refusals_and_non_finite():
    with own_context() as ctx:
        m, info, planes, Vprev = mat_scene()
        evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
        voxel = m.avgEdgeLen / 3.0
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
        with pytest.raises(L.IpcGpuError, match="ARG"):  # no sparsity pattern: no linear system, option 5 is no option of this context
            ctx.warm_start(5, voxel, TOL, evf, eee)
        start(ctx, m, info, planes, Vprev)
        for call in (lambda: ctx.warm_start(5, voxel, TOL, evf, eee), lambda: ctx.precondition_diag(-1)):
            with pytest.raises(L.IpcGpuError, match="STATE"):  # nothing assembled yet
                call()
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.warm_start(6, voxel, TOL, evf, eee)
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.precondition_diag(2)
        assemble(ctx, info, planes)
        ctx.precondition_diag(1)
        ctx.set_state(soa(m.V))  # a new state: the resident system is stale
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.precondition_diag(-1)
        assemble(ctx, info, planes)
        # a zero diagonal under a nonzero gradient entry, planted through the value array (the host Hessian form uploads it, adds 0 H)
        ia, ja = ctx.get_pattern()
        g, a = ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, len(ja))
        r = int(np.flatnonzero((g != 0) & ~np.repeat(m.dbc != 0, 3))[0])
        a[ia[r] - 1] = 0.0
        ctx.elastic_hessian(0.0, 1, 1, 1, a)
        assert ctx.download(L.BUF_CSR_VALUES, len(ja))[ia[r] - 1] == 0.0
        ctx.precondition_diag(-1, want_x=False)
        s = ctx.solve_info()
        assert s.status == L.ERR_SOLVE and np.isinf(s.max_abs_x)
        with pytest.raises(L.IpcGpuError, match="SOLVE"):
            ctx.precondition_diag(-1)

