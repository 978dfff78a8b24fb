"""The time-integration frame of a time step on the device -- ipcgpu_compute_xtilde, ipcgpu_end_time_step, ipcgpu_warm_start -- against the
float64 restatement of tests/oracle_timestep.py, bit for bit; captured against eager; a multi-step run against the same frame driven from the
host through the existing entry points; the refusals."""

import numpy as np
import pytest

import oracle as orc
import oracle_halfspace as OH
import oracle_timestep as OT
from gpu_common import load_scene, own_context, same_bits, scalar_bits, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

pytestmark = pytest.mark.gpu

TOL = 1e-6
G = (0.2, -9.81, -0.4)
PARAMS = {"BE": (OT.BE, 0.25, 0.5), "NM": (OT.NM, 0.25, 0.5), "NM_nondefault": (OT.NM, 0.3, 0.6)}


@pytest.fixture(scope="module")
def ctx():
    with own_context() as c:
        yield c


def upload_mesh(ctx, Vr, m, mass, dbc):
    ctx.set_mesh(soa(Vr), m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, mass, dbc, m.energy)


def positions(ctx, nV):
    return ctx.download(L.BUF_POSITIONS, 3 * nV).reshape(3, nV).T


def dynamics(ctx, nV):
    v, a, dx = ctx.get_dynamics()
    return v.reshape(nV, 3), a.reshape(3, nV).T, dx.reshape(3, nV).T


# ---- 1. the per-vertex kernels ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PARAMS))
def test_xtilde_and_end_of_step_bit_identical(ctx, name):
    typ, beta, gamma = PARAMS[name]
    P = OT.Params(typ, 0.01, beta, gamma, G)
    V, T = M.grid_tets(3, 3, 3, h=1.0 / 3)
    m = M.Mesh(V, T, energy=1, density=1.0)
    rng = np.random.default_rng(11 + typ)
    n_tail = 7  # an obstacle tail: no tets, Dirichlet flag, mass 0
    Vr = np.vstack([m.V_rest, rng.standard_normal((n_tail, 3))])
    nV = len(Vr)
    dbc = np.concatenate([rng.choice([0, 0, 0, 1, 2], m.nV), np.ones(n_tail)]).astype(np.uint8)
    mass = np.concatenate([m.mass, np.zeros(n_tail)])
    upload_mesh(ctx, Vr, m, mass, dbc)
    ctx.set_time_integration(typ, P.dt, beta, gamma, G)
    V1, Vp, vel, acc, dxe = (Vr + rng.standard_normal((nV, 3)) * s for s in (0.05, 0.05, 3.0, 50.0, 1e-3))
    ctx.set_state(soa(V1))
    ctx.set_prev_state(soa(Vp))
    ctx.set_dynamics(vel.ravel(), soa(acc), soa(dxe))
    assert all(same_bits(a, b) for a, b in zip(dynamics(ctx, nV), (vel, acc, dxe)))
    ctx.compute_xtilde()
    xt = OT.xtilde(P, Vp, vel, acc, dbc)
    assert same_bits(ctx.download(L.BUF_XTILDE, 3 * nV).reshape(3, nV).T, xt)
    assert np.array_equal(xt[dbc != 0], Vp[dbc != 0])
    # two ends of a time step: the second one reads what the first one left (V_prev, x~, velocity, acceleration)
    for k in range(2):
        ref = OT.end_time_step(P, V1, Vp, xt, vel, acc, dbc)
        ctx.end_time_step()
        got = dynamics(ctx, nV)
        for g, r in zip(got, ref[:3]):
            assert same_bits(g, r), (name, k)
        assert same_bits(ctx.download(L.BUF_XTILDE, 3 * nV).reshape(3, nV).T, ref[4])
        vel, acc, _, Vp, xt = ref
        V1 = V1 + rng.standard_normal((nV, 3)) * 0.01
        ctx.set_state(soa(V1))
    ctx.set_prev_state(soa(Vp))  # (V_prev is what the last end of step left: set it again from the host, the result must not change)
    ctx.compute_xtilde()
    assert same_bits(ctx.download(L.BUF_XTILDE, 3 * nV).reshape(3, nV).T, xt)


# ---- 2. the warm start against the oracle driver ------------------------------------------------------------------------------------------
class WScene:
    def __init__(self, m, vel, dxe, acc, voxel, plane=None):
        self.m, self.vel, self.dxe, self.acc, self.voxel, self.plane = m, vel, dxe, acc, voxel, plane

    def planes(self):
        if self.plane is None:
            return None
        par = OH.planes(*self.plane)
        return lambda s: OH.HalfSpaces(s, par)


def two_cubes(gap, energy=1):
    V1, T1 = M.grid_tets(3, 3, 3, h=1.0 / 3)
    V2, T2 = M.grid_tets(3, 3, 3, h=1.0 / 3, origin=(0.1, 0.05, 1.0 + gap))
    return M.merge_meshes([(V1, T1), (V2, T2)], energy=energy, density=1.0), len(V1)


def wscene_ccd():
    """two bodies closing fast: each moves 0.04 toward the other across a gap of 0.02, the full CCD binds"""
    m, n1 = two_cubes(0.02)
    rng = np.random.default_rng(2)
    vel = np.zeros((m.nV, 3))
    vel[:n1, 2], vel[n1:, 2] = 4.0, -4.0
    return WScene(m, vel, rng.standard_normal((m.nV, 3)) * 1e-4, rng.standard_normal((m.nV, 3)), m.avgEdgeLen / 3.0)


def wscene_plane():
    """a body falling onto a plane 0.03 below it at 5 per unit time: the plane's step binds"""
    V, T = M.grid_tets(3, 3, 3, h=1.0 / 3)
    m = M.Mesh(V, T, energy=1, density=1.0)
    vel = np.zeros((m.nV, 3))
    vel[:, 2] = -5.0
    rng = np.random.default_rng(3)
    return WScene(m, vel, rng.standard_normal((m.nV, 3)) * 1e-4, rng.standard_normal((m.nV, 3)), m.avgEdgeLen / 3.0,
                  plane=([[0.0, 0.0, -0.03]], [[0.0, 0.0, 1.0]]))


def wscene_inversion():
    """a Neo-Hookean body whose predicted motion squashes it through itself along z at step 1: the inversion filter binds"""
    V, T = M.grid_tets(3, 3, 3, h=1.0 / 3)
    m = M.Mesh(V, T, energy=0, density=1.0)
    M.deform(m, 5, twist=0.1, amp=0.005, noise=0.005)
    vel = np.zeros((m.nV, 3))
    vel[:, 2] = -120.0 * (m.V[:, 2] - m.V[:, 2].mean())
    rng = np.random.default_rng(4)
    return WScene(m, vel, rng.standard_normal((m.nV, 3)) * 1e-4, rng.standard_normal((m.nV, 3)), 1.0)


def wscene_zero():
    """a surface vertex already 1e-3 behind the plane moves further into it: the plane's bound is 0, which is not an error (the squared
    distance of isIntersected does not see the vertex)"""
    sc = wscene_plane()
    v = int(np.argmin(sc.m.V[:, 2]))
    sc.m.V[v, 2] = -0.031
    return sc


WSCENES = {f.__name__[7:]: f for f in (wscene_ccd, wscene_plane, wscene_inversion, wscene_zero)}


def setup_warm(ctx, sc, P):
    m = sc.m
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_halfspaces(*sc.plane) if sc.plane is not None else ctx.set_halfspaces([], [])
    ctx.set_state(m.V_soa)
    ctx.set_prev_state(m.V_soa)
    ctx.set_time_integration(P.type, P.dt, P.beta, P.gamma, P.gravity)
    ctx.set_dynamics(sc.vel.ravel(), soa(sc.acc), soa(sc.dxe))


@pytest.mark.parametrize("typ", ["BE", "NM"])
@pytest.mark.parametrize("option", range(5))
@pytest.mark.parametrize("scene", list(WSCENES))
def test_warm_start_matches_oracle(ctx, scene, option, typ):
    sc = WSCENES[scene]()
    m = sc.m
    P = OT.Params(PARAMS[typ][0], 0.01, 0.25, 0.5, G)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    setup_warm(ctx, sc, P)
    rc, a = ctx.warm_start(option, sc.voxel, TOL, evf, eee, check=False)
    info = ctx.step_control_info()
    it = ctx.fetch_iteration()
    ref = OT.warm_start(m, P, option, sc.vel, sc.dxe, sc.voxel, TOL, evf, eee, sc.planes(), alpha_inversion=it.alpha_inversion if option else None)
    assert rc == ref["status"] == info.status == 0
    assert same_bits(ctx.download(L.BUF_SEARCH_DIR, 3 * m.nV), ref["p"])
    assert scalar_bits(a) == scalar_bits(ref["alpha"]) == scalar_bits(info.alpha) == scalar_bits(info.alpha_feasible) == scalar_bits(it.alpha)
    assert [info.halvings_inversion, info.halvings_intersection] == ref["counts"]
    assert same_bits(positions(ctx, m.nV), ref["V"])
    if option:
        assert scalar_bits(it.alpha_inversion) == scalar_bits(ref["alpha_inversion"])
        if sc.plane is not None:
            assert scalar_bits(it.alpha_halfspace) == scalar_bits(ref["alpha_halfspace"])
        assert scalar_bits(it.alpha_swept_grid) == scalar_bits(ref["alpha_swept_grid"]) and scalar_bits(it.alpha_full_ccd) == scalar_bits(ref["alpha_full_ccd"])
        binding = {"ccd": ref["alpha_full_ccd"] < ref["alpha_swept_grid"], "plane": 0.0 < ref.get("alpha_halfspace", 1.0) < ref["alpha_inversion"],
                   "inversion": ref["alpha_inversion"] < 1.0, "zero": ref["alpha"] == 0.0}
        assert binding[scene], (scene, ref)
    else:
        assert a == 0.0 and not ref["p"].any()


@pytest.mark.parametrize("entry", ["intersecting", "inverted"])
def test_failing_entry_state_keeps_v0(ctx, entry):
    """the only way into the two loops' fail-safe: the entry state fails the check, so they halve to step 0 and stop with V = V0"""
    if entry == "intersecting":
        sc = wscene_ccd()
        n1 = sc.m.nV // 2
        sc.m.V[n1:, 2] -= 0.3
    else:
        sc = wscene_inversion()
        top = sc.m.V[:, 2] > sc.m.V[:, 2].mean() + 0.2
        sc.m.V[top, 2] -= 0.9  # the top layer pushed below the middle one: tets inverted at V0
        assert orc.Elastic(sc.m).count_inverted() > 0
    m = sc.m
    P = OT.Params(OT.BE, 0.01, 0.25, 0.5, G)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    setup_warm(ctx, sc, P)
    rc, a = ctx.warm_start(1, sc.voxel, TOL, evf, eee, check=False)
    info = ctx.step_control_info()
    ref = OT.warm_start(m, P, 1, sc.vel, sc.dxe, sc.voxel, TOL, evf, eee, alpha_inversion=ctx.fetch_iteration().alpha_inversion)
    assert rc == info.status == ref["status"] == L.ERR_LINE_SEARCH and a == 0.0
    assert [info.halvings_inversion, info.halvings_intersection] == ref["counts"]
    assert same_bits(positions(ctx, m.nV), m.V)


# ---- 3. captured against eager ------------------------------------------------------------------------------------------------------------
def frame(ctx, sc, evf, eee, dHat):
    ctx.end_time_step()
    ctx.warm_start(2, sc.voxel, TOL, evf, eee, want=False)
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)


def test_captured_frame_equals_eager(ctx):
    sc = wscene_ccd()
    m = sc.m
    P = OT.Params(OT.NM, 0.01, 0.3, 0.6, G)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    dHat = 1e-3 ** 2

    setup_warm(ctx, sc, P)
    ctx.set_canonical_order(0)

    def start():  # (nothing here refuses the graph: same mesh, same number of planes)
        ctx.set_state(m.V_soa)
        ctx.set_prev_state(m.V_soa)
        ctx.set_dynamics(sc.vel.ravel(), soa(sc.acc), soa(sc.dxe))
        ctx.compute_xtilde()

    start()
    frame(ctx, sc, evf, eee, dHat)  # eager run first: lazy allocations, streams of the conditional nodes
    ctx.fetch_iteration()
    ctx.capture_begin()
    frame(ctx, sc, evf, eee, dHat)
    gid = ctx.capture_end()
    runs = []
    for replay in (False, True):
        start()
        out = []
        for step in range(4):
            if replay:
                ctx.graph_launch(gid)
            else:
                frame(ctx, sc, evf, eee, dHat)
            info, it = ctx.step_control_info(), ctx.fetch_iteration()
            out.append((positions(ctx, m.nV).tobytes(), ctx.download(L.BUF_XTILDE, 3 * m.nV).tobytes(), *[x.tobytes() for x in ctx.get_dynamics()],
                        scalar_bits(info.alpha), info.halvings_intersection, scalar_bits(it.alpha_full_ccd), ctx.constraint_set_sizes()))
        runs.append(out)
    assert runs[0] == runs[1]
    assert len({r[0] for r in runs[0]}) == 4  # the bodies moved at every step
    ctx.graph_destroy(gid)


# ---- 4. a multi-step run: the device frame against the host-driven frame --------------------------------------------------------------------
def newton(ctx, m, coef, dHat, iters=2):
    """gradient-descent "Newton" iterations on deterministic device calls (no contact pairs, no atomics): the same in both runs"""
    for _ in range(iters):
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        g = np.zeros(3 * m.nV)
        ctx.elastic_gradient(coef, 1, 1, g)
        ctx.inertia_gradient(1, g)
        p = -g / np.repeat(m.mass, 3) * 0.5
        ctx.set_search_dir(p)
        ctx.line_search(coef, dHat, 1e3, inertia=True, alpha=1.0)


def host_frame(ctx, m, P, state, option, voxel, evf, eee):
    """the same frame through the existing entry points: x~, V_prev and p computed on the host, bound and loops driven from the host"""
    V = positions(ctx, m.nV)
    vel, acc, dxe, Vp, xt = OT.end_time_step(P, V, state["Vp"], state["xt"], state["vel"], state["acc"], m.dbc)
    state.update(vel=vel, acc=acc, dxe=dxe, Vp=Vp, xt=xt)
    ctx.set_xtilde(soa(xt))
    ctx.set_prev_state(soa(Vp))
    p = np.ascontiguousarray(OT.predictor(P, option, vel, dxe, m.dbc)).ravel()
    ctx.set_search_dir(p)
    a = ctx.inversion_step(None, 0.2, 1.0) if m.energy == 0 else 1.0
    a = ctx.hash_build_swept(None, a, voxel)
    a, _ = ctx.ccd_full(TOL, evf, eee, a)
    ctx.save_state()
    ctx.step_forward(None, a)
    while m.energy == 0 and ctx.check_inversion() > 0:
        a /= 2.0
        ctx.step_forward(None, a)
    while not ctx.intersection_free():
        a /= 2.0
        ctx.step_forward(None, a)
    return a


def test_multi_step_run_equals_host_driven(ctx):
    ctx.set_canonical_order(1)  # (the module's context: the captured-frame test above runs at 0)
    V1, T1 = M.grid_tets(3, 3, 3, h=1.0 / 3)
    V2, T2 = M.grid_tets(2, 2, 2, h=0.25, origin=(0.3, 0.3, 1.3))  # (K steps of at most 0.06 leave the bodies apart: no contact pairs)
    m = M.merge_meshes([(V1, T1), (V2, T2)], energy=0, density=1.0)
    m.dbc[:16] = 1  # the bottom layer of the lower body is fixed
    P = OT.Params(OT.BE, 0.01, 0.25, 0.5, (0.0, 0.0, -9.81))
    vel0 = np.zeros((m.nV, 3))
    vel0[len(V1):, 2] = -6.0
    voxel, coef, dHat, K = m.avgEdgeLen / 3.0, 0.01 ** 2, 1e-4 ** 2, 4
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    trajectories, alphas = [], []
    for device in (True, False):
        load_scene(ctx, m)
        ctx.set_prev_state(m.V_soa)
        ctx.set_time_integration(P.type, P.dt, P.beta, P.gamma, P.gravity)
        ctx.set_dynamics(vel0.ravel(), None, None)
        ctx.compute_xtilde()
        state = dict(Vp=m.V.copy(), vel=vel0.copy(), acc=np.zeros_like(vel0), xt=OT.xtilde(P, m.V, vel0, np.zeros_like(vel0), m.dbc))
        traj, al = [], []
        newton(ctx, m, coef, dHat)
        for k in range(K):
            if device:
                ctx.end_time_step()
                _, a = ctx.warm_start(1, voxel, TOL, evf, eee)
            else:
                a = host_frame(ctx, m, P, state, 1, voxel, evf, eee)
            al.append(a)
            newton(ctx, m, coef, dHat)
            traj.append(positions(ctx, m.nV).tobytes())
        trajectories.append(traj)
        alphas.append(al)
    assert alphas[0] == alphas[1], alphas
    assert trajectories[0] == trajectories[1] and len(set(trajectories[0])) == K


# ---- 5. refusals ----------------------------------------------------------------------------------------------------------------------------
def test_refusals():
    with own_context() as ctx:  # (a fresh context: no time integration set yet)
        sc = wscene_plane()
        m = sc.m
        evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
        load_scene(ctx, m)
        ctx.set_prev_state(m.V_soa)
        ctx.set_dynamics(sc.vel.ravel(), None, None)
        with pytest.raises(L.IpcGpuError, match="STATE"):  # no set_time_integration on this context yet
            ctx.warm_start(1, sc.voxel, TOL, evf, eee)
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.set_time_integration(2, 0.01)
        ctx.set_time_integration(OT.BE, 0.01)
        for option in (5, -1, 6):
            with pytest.raises(L.IpcGpuError, match="ARG"):
                ctx.warm_start(option, sc.voxel, TOL, evf, eee)
        ctx.warm_start(1, sc.voxel, TOL, evf, eee)
        # a new mesh forgets nothing of the time integration, but its V_prev must be set again when it has more vertices
        V, T = M.grid_tets(4, 4, 4, h=0.25)
        m2 = M.Mesh(V, T, energy=1, density=1.0)
        ctx.set_mesh(m2.V_rest_soa, m2.T_soa, m2.restTriInv, m2.vol, m2.mu, m2.lam, m2.mass, m2.dbc, m2.energy)
        ctx.set_surface(m2.SVI, m2.SFEdges, m2.SF_soa, m2.vCoDim)
        for call in (ctx.compute_xtilde, lambda: ctx.warm_start(1, sc.voxel, TOL, evf, eee)):
            with pytest.raises(L.IpcGpuError, match="STATE"):
                call()
