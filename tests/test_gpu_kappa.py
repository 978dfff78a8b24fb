"""The barrier stiffness held on the device (IPCGPU_KAPPA_DEVICE, ipcgpu_set_kappa) and its adaptation: the sentinel gives the host-kappa
results; ipcgpu_kappa_init (initKappa) and ipcgpu_kappa_post_line_search (postLineSearch's close-pair doubling) against the float64
restatement of tests/oracle_kappa.py; a few time steps of Newton iterations with kappa on the device, eagerly, replayed from one graph and
driven from the host with the restatement's kappa, take the same doubling decisions."""

import contextlib

import numpy as np
import pytest

import oracle_kappa as ok
from gpu_common import load_scene, own_context, rel, scalar_bits, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import obstacle as OB
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu
KD = L.KAPPA_DEVICE
DT2 = 0.025 ** 2
TOL = 1e-6


@contextlib.contextmanager
def context(m, nV_dof=None):
    with own_context() as ctx:
        load_scene(ctx, m)
        if nV_dof is not None:
            ctx.set_obstacle_tail(nV_dof)
        yield ctx


def mat_scene(**kw):
    """a ball just over a mat (self contact) and a ground plane just under the mat"""
    m, info = scenes.ball_on_mat(nx=10, res=4, gap_lo=0.2, gap_hi=0.5, **kw)
    dHat = info["dHat"]
    z0 = m.V[:, 2].min() - 0.5 * np.sqrt(dHat)
    return m, info, dHat, dict(origin=[[0.0, 0.0, z0]], normal=[[0.0, 0.0, 1.0]], friction=[0.3])


def host_sets(ctx, dHat, planes):
    mm, _, _, _ = ctx.constraint_set(dHat, 1)
    act = ctx.get_halfspace_sets()[0] if planes else np.empty((0, 2), np.int32)
    return mm, act


# ---- 1. the sentinel gives the host-kappa results -----------------------------------------------------------------------------------
def test_sentinel_equivalence():
    m, info, dHat, pl = mat_scene()
    K, n = 3.7e5, 3 * m.nV
    with context(m) as ctx:
        ctx.set_halfspaces(**pl)
        ctx.set_prev_state(soa(m.V - 1e-3 * info["p"].reshape(-1, 3)))
        ctx.enable_device_pattern(1)
        ctx.constraint_set(dHat, 1)
        assert ctx.halfspace_constraint_set(dHat) > 0 and ctx.nC > 0
        ctx.update_pattern()
        ctx.set_kappa(K, 0.0, 1e300)
        for f in (ctx.barrier_energy, ctx.halfspace_energy):
            assert scalar_bits(f(dHat, KD)) == scalar_bits(f(dHat, K))

        def spread_check(call, size):
            h1, h2, d = (call(k, np.zeros(size)) for k in (K, K, KD))
            tol = max(np.linalg.norm(h1 - h2), 1e-14 * np.linalg.norm(h1))
            assert np.linalg.norm(d - h1) <= 2 * tol
            return np.linalg.norm(h1)

        assert spread_check(lambda k, g: ctx.barrier_gradient(dHat, k, g), n) > 0
        spread_check(lambda k, g: ctx.para_ee_gradient(dHat, k, g), n)  # (no mollified pair in this scene: test_sentinel_mollified_pairs)
        assert spread_check(lambda k, g: ctx.halfspace_gradient(dHat, k, g), n) > 0
        assert spread_check(lambda k, a: ctx.barrier_hessian(dHat, k, 1, a), ctx.nnz) > 0
        assert spread_check(lambda k, a: ctx.halfspace_hessian(dHat, k, 1, a), ctx.nnz) > 0
        lam = []
        for k in (K, KD):
            ctx.friction_lag(dHat, k)
            ctx.halfspace_friction_lag(dHat, k)
            lam.append((ctx.get_friction_data()[1].copy(), ctx.get_halfspace_sets()[2].copy()))
        assert len(lam[0][0]) > 0 and len(lam[0][1]) > 0
        for a, b in zip(lam[0], lam[1]):
            assert a.tobytes() == b.tobytes()
        # the line search: the same trials, to the bit
        res = []
        for k in (K, KD):
            ctx.set_state(m.V_soa)
            ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
            ctx.halfspace_constraint_set(dHat, want=False)
            ctx.set_search_dir(info["p"])
            rc, a = ctx.line_search(DT2, dHat, k, alpha=1.0, check=False)
            s = ctx.step_control_info()
            res.append((rc, scalar_bits(a), scalar_bits(s.energy_start), scalar_bits(s.energy), s.halvings_inversion, s.halvings_intersection, s.halvings_armijo,
                        s.halvings_post_check, ctx.download(L.BUF_POSITIONS, n).tobytes()))
        assert res[0] == res[1]
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.line_search(DT2, dHat, -2.0, alpha=1.0)


def spread(h1, h2, d):
    """d (device kappa) within the spread of two host-kappa runs h1, h2 (the barrier terms add with atomics); returns |h1|"""
    tol = max(np.linalg.norm(h1 - h2), 1e-14 * np.linalg.norm(h1))
    assert np.linalg.norm(d - h1) <= 2 * tol, (np.linalg.norm(d - h1), tol)
    return np.linalg.norm(h1)


def test_sentinel_mollified_pairs():
    """nearly parallel mesh-obstacle edges: the mollified branches of the gradient and Hessian kernels with the device kappa"""
    m0, inf0 = scenes.balls_on_obstacle(plate_angle=0.0, res=4, plate=12)
    ob = inf0["obstacle"]
    m = OB.with_obstacle(m0, ob["V"], ob["E"], ob["F"])
    dHat, K, n = inf0["dHat"], 2.9e7, 3 * m.nV
    with context(m, m.nV_dof) as ctx:
        ctx.enable_device_pattern(1)
        ctx.constraint_set(dHat, 1)
        assert ctx.nP > 0
        ctx.update_pattern()
        ctx.set_kappa(K, 0.0, 1e300)
        assert scalar_bits(ctx.barrier_energy(dHat, KD)) == scalar_bits(ctx.barrier_energy(dHat, K))
        for call, size in [(lambda k, g: ctx.para_ee_gradient(dHat, k, g), n), (lambda k, g: ctx.barrier_gradient(dHat, k, g), n),
                           (lambda k, a: ctx.barrier_hessian(dHat, k, 1, a), ctx.nnz)]:
            assert spread(*(call(k, np.zeros(size)) for k in (K, K, KD))) > 0


def test_hessian_right_after_a_kappa_write():
    """the reference's order: initKappa, then the Hessian at the same positions and sets; postLineSearch's doubling, then the next
    iteration's Hessian with no set rebuild in between.  The device-kappa Hessian must be the one at the kappa that was just written."""
    m, info, dHat, pl = mat_scene()
    with context(m) as ctx:
        ctx.enable_device_pattern(1)
        ctx.constraint_set(dHat, 1)
        ctx.update_pattern()
        nnz = ctx.nnz

        def hessian_matches():
            d = ctx.barrier_hessian(dHat, KD, 1, np.zeros(nnz))  # the first call after the write
            k = ctx.kappa_info().kappa
            assert spread(*(ctx.barrier_hessian(dHat, k, 1, np.zeros(nnz)) for _ in range(2)), d) > 0
            return k

        ctx.elastic_gradient(DT2, 1, 1, want=False)
        ctx.set_kappa(0.0, 1.0, 1e30)
        ctx.kappa_init(dHat)
        k1 = hessian_matches()
        assert k1 >= 1.0
        ctx.kappa_clear_close_set()
        ctx.kappa_post_line_search(dHat)  # the snapshot
        ctx.kappa_post_line_search(dHat)  # the same positions: every saved d is equal, kappa doubles
        k2 = hessian_matches()
        assert scalar_bits(k2) == scalar_bits(2.0 * k1) and ctx.kappa_info().doublings == 1


# ---- 2. initKappa ----------------------------------------------------------------------------------------------------------------
def g_E_into(ctx, gE):
    """leave gE as the device gradient (a host-form barrier gradient with kappa 0 adds nothing)"""
    ctx.barrier_gradient(1e-30, 0.0, np.array(gE, dtype=np.float64))


def init_case(ctx, m, dHat, k0, s, mx, gE, planes=None, nV_dof=None):
    V = ctx.download(L.BUF_POSITIONS, 3 * m.nV).reshape(3, -1).T.copy()
    mm, act = host_sets(ctx, dHat, planes is not None)
    par = None
    if planes is not None:
        import oracle_halfspace as ohs
        par = ohs.planes(planes["origin"], planes["normal"], None, planes["friction"])
    g_E_into(ctx, gE)
    gE_dev = ctx.download(L.BUF_GRADIENT, 3 * m.nV)
    ctx.set_kappa(k0, s, mx)
    ctx.kappa_init(dHat)
    info = ctx.kappa_info()
    gc = ok.constraint_gradient(V, m.dbc, mm, dHat, par, act)
    kappa, minK = ok.init(k0, s, mx, gE_dev, gc, len(mm) + len(act))
    return info, kappa, minK, gc


@pytest.mark.parametrize("which", ["self", "obstacle", "plane"])
def test_kappa_init_scenes(which):
    if which == "obstacle":
        m0, inf0 = scenes.balls_on_obstacle(res=4)
        ob = inf0["obstacle"]
        m = OB.with_obstacle(m0, ob["V"], ob["E"], ob["F"])
        dHat, planes, nV_dof = inf0["dHat"], None, m.nV_dof
    else:
        m, info, dHat, pl = mat_scene()
        planes, nV_dof = (pl if which == "plane" else None), None
    with context(m, nV_dof) as ctx:
        if planes:
            ctx.set_halfspaces(**planes)
            ctx.halfspace_constraint_set(dHat)
        ctx.elastic_gradient(DT2, 1, 1, want=False)
        gE = ctx.download(L.BUF_GRADIENT, 3 * m.nV)
        s, mx = 1.0, 1e30
        info, kappa, minK, gc = init_case(ctx, m, dHat, 0.0, s, mx, gE, planes)
        assert np.linalg.norm(gc) > 0 and minK is not None
        assert abs(info.kappa - kappa) <= 1e-12 * abs(kappa), (info.kappa, kappa)
        assert abs(info.min_kappa - minK) <= 1e-12 * abs(minK)
        assert info.needs_init == 0


def test_kappa_init_branches():
    m, info, dHat, pl = mat_scene()
    with context(m) as ctx:
        n = 3 * m.nV
        V = m.V
        mm, act = host_sets(ctx, dHat, False)
        gc = ok.constraint_gradient(V, m.dbc, mm, dHat)
        s, mx, k0 = 1e3, 1e7, 5e4
        for K, expect in [(-1.0, k0), (1e9, mx), (10.0, s), (2e5, None)]:  # minK <= 0, above max, below suggest, in between
            got, kappa, minK, _ = init_case(ctx, m, dHat, k0, s, mx, -K * gc)
            exp = kappa if expect is None else expect
            assert scalar_bits(kappa) == scalar_bits(exp) or expect is None
            if expect is None:
                assert abs(got.kappa - kappa) <= 1e-12 * kappa
            else:
                assert scalar_bits(got.kappa) == scalar_bits(expect), (K, got.kappa, expect)
        # no active entries: nothing changes (not even minKappa)
        before = ctx.kappa_info().min_kappa
        ctx.constraint_set(1e-30, 1)
        assert ctx.nC == 0
        ctx.set_kappa(k0, s, mx)
        ctx.kappa_init(dHat)
        got = ctx.kappa_info()
        assert scalar_bits(got.kappa) == scalar_bits(k0) and scalar_bits(got.min_kappa) == scalar_bits(before)
    # contact only on Dirichlet vertices against the obstacle (pairs between two Dirichlet mesh vertices are not built, obstacle pairs are):
    # g_c = 0, minKappa = NaN, kappa stays, then the floor
    m0, inf0 = scenes.balls_on_obstacle(res=4)
    m0.dbc = np.ones(m0.nV, dtype=np.uint8)
    ob = inf0["obstacle"]
    m = OB.with_obstacle(m0, ob["V"], ob["E"], ob["F"])
    dHat = inf0["dHat"]
    with context(m, m.nV_dof) as ctx:
        ctx.elastic_gradient(DT2, 1, 1, want=False)
        for k0, expect in [(5e4, 5e4), (10.0, 1e3)]:
            got, kappa, minK, gc = init_case(ctx, m, dHat, k0, 1e3, 1e7, ctx.download(L.BUF_GRADIENT, 3 * m.nV))
            assert ctx.nC > 0 and not np.any(gc) and minK is not None and np.isnan(minK) and np.isnan(got.min_kappa)
            assert scalar_bits(got.kappa) == scalar_bits(expect) == scalar_bits(kappa)


# ---- 3. postLineSearch -----------------------------------------------------------------------------------------------------------
def cubes(gap):
    V1, T1 = M.grid_tets(2, 2, 2, h=0.5)
    V2, T2 = M.grid_tets(2, 2, 2, h=0.5, origin=(0.13, 0.07, 1.0 + gap))
    return M.merge_meshes([(V1, T1), (V2, T2)], energy=1, density=1.0), len(V1)


def run_post(ctx, m, ref, V, dHat, dTol, planes=None, par=None):
    ctx.set_state(soa(V))
    mm, act = (np.empty((0, 4), np.int32), np.empty((0, 2), np.int32))
    mm, _, _, _ = ctx.constraint_set(dHat, 1)
    if planes:
        ctx.halfspace_constraint_set(dHat)
        act = ctx.get_halfspace_sets()[0]
    ctx.kappa_post_line_search(dTol)
    ref.post_line_search(V, mm, act, dTol, par)
    got = ctx.kappa_info()
    assert scalar_bits(got.kappa) == scalar_bits(ref.kappa), (got.kappa, ref.kappa)
    assert got.n_close == len(ref.saved) and got.doublings == ref.doublings and bool(got.needs_init) == ref.needs_init
    return got


@pytest.mark.parametrize("case", ["approach", "recede", "equal", "left_set", "new_pair", "at_dTol", "capped", "zero"])
def test_post_line_search(case):
    gap = 0.02
    m, n1 = cubes(gap)
    m.V[n1:, 2] += 0.3 * gap * (m.V[n1:, 0] - 0.13)  # tilted: the pairs' distances differ
    dHat = (1.5 * gap) ** 2
    dTol = dHat if case != "new_pair" else (0.5 * gap) ** 2
    k0, mx = 1e4, (1.5e4 if case == "capped" else 1e9)
    with context(m) as ctx:
        ctx.set_kappa(0.0 if case == "zero" else k0, 1.0, mx)
        ctx.kappa_clear_close_set()
        ref = ok.CloseSet(0.0 if case == "zero" else k0, mx)
        V = m.V.copy()
        if case == "at_dTol":  # dTol equal to a distance the device evaluates: that entry is not saved
            mm0, _, _, _ = ctx.constraint_set(dHat, 1)
            dev = ctx.evaluate_constraints(ctx.nC)
            dTol = float(np.max(dev))
            # (the restatement takes the device's distances here: the oracle's may differ from them in the last bits, and d == dTol is
            # decided on the exact value)
            table = {tuple(int(v) for v in e): float(x) for e, x in zip(mm0, dev)}
            ref.d2 = lambda V_, par, key: table[key[1]]
        run_post(ctx, m, ref, V, dHat, dTol)
        assert ref.saved or case in ("new_pair", "zero")
        V2 = V.copy()
        shift = {"approach": -0.2, "recede": 0.2, "new_pair": -0.6, "capped": -0.2}.get(case, 0.0) * gap
        V2[n1:, 2] += shift
        got = run_post(ctx, m, ref, V2, dHat if case != "left_set" else (0.5 * gap) ** 2, dTol)
        expect = {"approach": 1, "recede": 0, "equal": 1, "left_set": 1, "new_pair": 0, "at_dTol": 1, "capped": 1, "zero": 0}[case]
        assert got.doublings == expect
        if case == "capped":
            assert scalar_bits(got.kappa) == scalar_bits(mx)
        if case == "zero":
            assert got.needs_init == 1 and got.kappa == 0.0
        if case == "new_pair":
            assert got.n_close > 0
        if case == "at_dTol":
            assert 0 < got.n_close < ctx.nC


def test_post_line_search_plane_and_obstacle():
    # a plane: the cube approaches the ground
    V, T = M.grid_tets(2, 2, 2, h=0.5)
    m = M.Mesh(V, T, energy=1, density=1.0)
    gap = 0.02
    dHat = (1.5 * gap) ** 2
    planes = dict(origin=[[0.0, 0.0, -gap]], normal=[[0.0, 0.0, 1.0]], friction=[0.0])
    import oracle_halfspace as ohs
    par = ohs.planes(planes["origin"], planes["normal"], None, planes["friction"])
    with context(m) as ctx:
        ctx.set_halfspaces(**planes)
        ctx.set_kappa(1e4, 1.0, 1e9)
        ref = ok.CloseSet(1e4, 1e9)
        got = run_post(ctx, m, ref, m.V, dHat, dHat, True, par)
        assert got.n_close > 0 and np.isfinite(got.close_min_dist2)
        V2 = m.V.copy()
        V2[:, 2] -= 0.2 * gap
        assert run_post(ctx, m, ref, V2, dHat, dHat, True, par).doublings == 1
    # an obstacle: the balls approach the plate
    m0, inf0 = scenes.balls_on_obstacle(res=4)
    ob = inf0["obstacle"]
    m = OB.with_obstacle(m0, ob["V"], ob["E"], ob["F"])
    dHat = inf0["dHat"]
    with context(m, m.nV_dof) as ctx:
        ctx.set_kappa(1e4, 1.0, 1e9)
        ref = ok.CloseSet(1e4, 1e9)
        got = run_post(ctx, m, ref, m.V, dHat, dHat)
        assert got.n_close > 0
        V2 = m.V.copy()
        V2[: m.nV_dof, 2] -= 0.1 * np.sqrt(dHat)
        assert run_post(ctx, m, ref, V2, dHat, dHat).doublings == 1


def test_capture_contract():
    V, T = M.grid_tets(2, 2, 2)
    m = M.Mesh(V, T, energy=0)
    with context(m) as ctx:
        ctx.set_kappa(1.0, 1.0, 2.0)
        ctx.capture_begin()
        ctx.set_kappa(2.0, 1.0, 2.0)
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.kappa_info()
        gid = ctx.capture_end()
        assert ctx.kappa_info().kappa == 1.0
        ctx.graph_launch(gid)
        assert ctx.kappa_info().kappa == 2.0
        ctx.graph_destroy(gid)


# ---- 4. Newton iterations with kappa on the device ---------------------------------------------------------------------------------
def newton_scene():
    m, info = scenes.ball_on_mat(nx=10, res=4, gap_lo=0.3, gap_hi=0.4)
    dHat = info["dHat"]
    xt = m.V.copy()
    xt[info["n_mat_verts"]:, 2] -= 3.0 * np.sqrt(dHat)  # inertia pulls the ball into the mat: the close pairs approach
    return m, info, dHat, xt


def prepare(ctx, m, xt):
    ctx.set_canonical_order(0)
    ctx.enable_device_pattern(1)
    ctx.set_xtilde(soa(xt))


def iteration(ctx, m, dHat, kappa, evf, eee, dTol):
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0, want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.inertia_gradient(1, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.solve_pcg_multilevel(rel_tol=1e-12, max_iter=5000, want_x=False, adopt=True, deferred=True)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    ctx.ccd_cfl(dHat, 1, m.avgEdgeLen / 3.0, TOL, evf, eee, None)
    ctx.line_search(DT2, dHat, kappa, inertia=True)
    if kappa == KD:
        ctx.kappa_post_line_search(dTol)


def time_step_start(ctx, dHat, s, mx):
    ctx.set_kappa(s, s, mx)
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.elastic_gradient(DT2, 1, 1, want=False)
    ctx.inertia_gradient(1, None)
    ctx.kappa_init(dHat)
    ctx.kappa_clear_close_set()


def test_newton_driver_eager_graph_host():
    m, info, dHat, xt = newton_scene()
    n, n_it, n_steps = 3 * m.nV, 2, 3
    dTol = dHat
    s, mx = ok.bounds(dHat, 1e-11, float(np.mean(m.mass)), float(np.sum((m.V_rest.max(0) - m.V_rest.min(0)) ** 2)))
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    with context(m) as e, context(m) as g, context(m) as h:
        for c in (e, g, h):
            prepare(c, m, xt)

        def step(c):
            time_step_start(c, dHat, s, mx)
            for _ in range(n_it):
                iteration(c, m, dHat, KD, evf, eee, dTol)

        step(g)  # the eager run: lazy allocations
        g.set_state(m.V_soa)
        g.kappa_info()
        g.capture_begin()
        step(g)
        gid = g.capture_end()
        # host-driven: the restatement's kappa handed to the host-kappa calls
        ref = ok.CloseSet(s, mx)
        log = {"e": [], "g": [], "h": []}
        for k in range(n_steps):
            step(e)
            ie = e.kappa_info()
            n0 = g.launch_count()
            g.graph_launch(gid)
            assert g.launch_count() > n0
            ig = g.kappa_info()
            # host loop
            h.constraint_set(dHat, 1, fetch=False, sizes=False)
            h.elastic_gradient(DT2, 1, 1, want=False)
            h.inertia_gradient(1, None)
            gE = h.download(L.BUF_GRADIENT, n)
            V = h.download(L.BUF_POSITIONS, n).reshape(3, -1).T.copy()
            mm, _, _, _ = h.constraint_set(dHat, 1)
            kappa, _ = ok.init(s, s, mx, gE, ok.constraint_gradient(V, m.dbc, mm, dHat), len(mm))
            ref.kappa, ref.saved, ref.doublings = kappa, [], 0
            for _ in range(n_it):
                iteration(h, m, dHat, ref.kappa, evf, eee, dTol)
                h.fetch_iteration()
                V = h.download(L.BUF_POSITIONS, n).reshape(3, -1).T.copy()
                mm, _, _, _ = h.constraint_set(dHat, 1)
                ref.post_line_search(V, mm, (), dTol)
            for key, c, i in (("e", e, ie), ("g", g, ig)):
                sc = c.step_control_info()
                assert sc.status == 0
                log[key].append((i.doublings, i.kappa, sc.alpha))
            log["h"].append((ref.doublings, ref.kappa, h.step_control_info().alpha))
        for k in range(n_steps):
            (de, ke, ae), (dg, kg, ag), (dh, kh, ah) = log["e"][k], log["g"][k], log["h"][k]
            assert de == dg == dh, log
            assert rel(kg, ke) <= 1e-9 and rel(kh, ke) <= 1e-9, log
            assert rel(ag, ae) <= 1e-6 and rel(ah, ae) <= 1e-6, log
        assert sum(x[0] for x in log["e"]) >= 1, log  # the scene doubles at least once
        g.graph_destroy(gid)
