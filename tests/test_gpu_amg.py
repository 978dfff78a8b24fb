"""ipcgpu_solve_pcg_amg: PCG on the device-resident Hessian with the smoothed-aggregation multigrid preconditioner.  The aggregates equal
the host mirror's (tests/amg_mirror.py) exactly, the level matrices, spectral radii, dampings, the application and the residuals along the
way equal it to rounding, two calls give identical bits, an iteration makes 67 * 2^(L-1) - 32 launches, Dirichlet and obstacle rows stay
exactly 0 (adopted too), the device-built pattern is covered, and a non-positive-definite matrix, a capture and bad arguments are errors."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import amg_mirror as am
import multilevel_mirror as mlm
from gpu_common import own_context, rel, same_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes
from test_gpu_multilevel import DT2, assemble, launches_of_25_more_iterations, load_sorted, resident_system, states

pytestmark = pytest.mark.gpu


def compare_hierarchy(ctx, A):
    """the device hierarchy against the mirror's A (am.AMG)"""
    h = ctx.amg_info()
    assert h["rows"] == [lv.n for lv in A.lv] and h["blocks"] == [lv.A.ja.size for lv in A.lv], h
    for l, lv in enumerate(A.lv):
        agg, ia, ja, blk = ctx.amg_debug_level(l)
        assert np.array_equal(ia, lv.A.ia) and np.array_equal(ja, lv.A.ja), l
        assert np.array_equal(agg, lv.agg if lv.agg is not None else np.full(lv.n, -1)), l
        scale = np.zeros(lv.n)
        np.maximum.at(scale, lv.A.rows, np.abs(lv.A.blk).max(axis=(1, 2)))
        assert (np.abs(blk - lv.A.blk).max(axis=(1, 2)) <= 1e-12 * scale[lv.A.rows]).all(), (l, np.abs(blk - lv.A.blk).max())
        assert abs(h["rho"][l] - lv.rho) <= 1e-12 * lv.rho, (l, h["rho"][l], lv.rho)
        om = lv.omega if l + 1 < A.levels else 0.0
        assert abs(h["omega"][l] - om) <= 1e-12 * max(om, 1e-300), (l, h["omega"][l], om)


def test_hierarchy_application_and_iterations_equal_the_mirror(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    ia, ja = assemble(ctx, m, info["dHat"], 1e6)
    n = 3 * m.nV
    H, g = resident_system(ctx, ia, ja, n)
    A = am.AMG(H)
    x, iters, res = ctx.solve_pcg_amg(None, rel_tol=1e-10, max_iter=5000)
    assert res <= 1e-10 and 0 < iters < 5000 and rel(x, spla.spsolve(H.tocsc(), -g)) <= 1e-7
    assert A.levels >= 2
    compare_hierarchy(ctx, A)
    # z = M^-1 r for a random r: the first iterate of a solve with right-hand side r is alpha z, alpha = r.z / z.Hz
    r = np.random.default_rng(1).standard_normal(n)
    z = A.apply(r)
    x1, it1, _ = ctx.solve_pcg_amg(r, rel_tol=1e-10, max_iter=1)
    cond = np.linalg.cond(H.toarray())
    assert it1 == 1 and rel(x1, (r @ z) / (z @ (H @ z)) * z) <= 1e-12 * cond, (rel(x1, (r @ z) / (z @ (H @ z)) * z), cond)
    for k in (5, 12):
        _, it_k, res_k = ctx.solve_pcg_amg(None, rel_tol=1e-30, max_iter=k)
        res_m = mlm.pcg(H, -g, A.apply, 1e-30, k)[2]
        assert it_k == k and abs(res_k - res_m) <= 1e-6 * res_m, (k, res_k, res_m)
    xm, it_m, _ = mlm.pcg(H, -g, A.apply, 1e-10, 5000)
    assert abs(iters - it_m) <= 25 and rel(x, xm) <= 1e-8


def test_two_solves_give_identical_bits_and_the_launches_of_the_cycle(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    assemble(ctx, m, info["dHat"], 1e8)
    x1, it1, res1 = ctx.solve_pcg_amg(None, rel_tol=1e-8, max_iter=5000)
    h1 = ctx.amg_info()
    blk1 = [ctx.amg_debug_level(l)[3] for l in range(len(h1["rows"]))]
    ctx.solve_pcg_multilevel(None, rel_tol=1e-3, max_iter=50)  # (other solvers in between share the workspace)
    ctx.solve_pcg(None, rel_tol=1e-3, max_iter=50)
    x2, it2, res2 = ctx.solve_pcg_amg(None, rel_tol=1e-8, max_iter=5000)
    h2 = ctx.amg_info()
    assert res1 <= 1e-8 and it1 == it2 and same_bits(res1, res2) and same_bits(x1, x2) and h1 == h2
    assert all(same_bits(b, ctx.amg_debug_level(l)[3]) for l, b in enumerate(blk1))
    # per iteration: SpMV, roll, direction and the W-cycle: 16 per Chebyshev application, 3 transfers per coarse visit
    Lv = len(h1["rows"])
    assert launches_of_25_more_iterations(ctx, ctx.solve_pcg_amg) == 25 * (67 * 2 ** (Lv - 1) - 32) + 1


def test_device_built_pattern_after_a_pattern_change(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    dHat, kappa = info["dHat"], 1e6
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(1)
    for name in ("A", "B"):
        ctx.set_state(soa(S[name]))
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        x, iters, res = ctx.solve_pcg_amg(None, rel_tol=1e-10, max_iter=5000)
        assert res <= 1e-10 and 0 < iters < 5000
    ia, ja = ctx.get_pattern()
    H, g = resident_system(ctx, ia, ja, 3 * m.nV)
    assert rel(x, spla.spsolve(H.tocsc(), -g)) <= 1e-7
    # the device-built pattern stores zero blocks: they are not kept, and the hierarchy is the mirror's
    A = am.AMG(H)
    compare_hierarchy(ctx, A)
    assert abs(mlm.pcg(H, -g, A.apply, 1e-10, 5000)[1] - iters) <= 25


def test_obstacle_tail_and_dirichlet_vertices(shared_ctx):
    from ipc_b200 import obstacle as OB
    ctx = shared_ctx
    m, info = scenes.balls_on_obstacle(plate_angle=0.0, res=4, plate=12)
    ob = info["obstacle"]
    M2 = OB.with_obstacle(m, ob["V"], ob["E"], ob["F"])
    M2.dbc = M2.dbc.copy()
    M2.dbc[:5] = 1
    load_sorted(ctx, M2)
    ctx.set_obstacle_tail(M2.nV_dof, 1)
    try:
        ctx.enable_device_pattern(1)
        ctx.constraint_set(info["dHat"], 1)
        ctx.update_pattern()
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(info["dHat"], 1e8, None)
        ctx.barrier_hessian(info["dHat"], 1e8, 1, None)
        ia, ja = ctx.get_pattern()
        n = 3 * M2.nV
        H, g = resident_system(ctx, ia, ja, n)
        fixed_v = np.zeros(M2.nV, dtype=bool)
        fixed_v[:5] = True
        fixed_v[M2.nV_dof:] = True
        fixed = np.flatnonzero(np.repeat(fixed_v, 3))
        b = np.random.default_rng(2).standard_normal(n)
        b[fixed] = 0.0
        x, iters, res = ctx.solve_pcg_amg(b, rel_tol=1e-10, max_iter=5000)
        assert res <= 1e-10 and 0 < iters < 5000 and rel(x, spla.spsolve(H.tocsc(), b)) <= 1e-7
        assert (x[fixed] == 0.0).all()
        A = am.AMG(H)
        assert A.levels == 1 or (A.lv[0].agg[fixed_v] == -1).all()
        compare_hierarchy(ctx, A)
        bn = -g
        bn[fixed] = 0.0
        xn, _, resn = ctx.solve_pcg_amg(bn, rel_tol=1e-6, max_iter=5000, adopt=True)
        p = ctx.download(L.BUF_SEARCH_DIR, n)
        assert resn <= 1e-6 and np.array_equal(p, xn) and (p[fixed] == 0.0).all() and np.abs(p).max() > 0.0
        assert ctx.solve_info().max_abs_x == np.abs(xn).max()
    finally:
        ctx.set_obstacle_tail(-1)


def test_not_positive_definite_is_an_error_and_not_a_hang():
    with own_context() as ctx:
        V, T = M.grid_tets(2, 2, 2)
        m = M.Mesh(V, T, energy=0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        ctx.csr_set_zero()  # an all-zero matrix: no diagonal block is positive definite
        with pytest.raises(L.IpcGpuError, match="SOLVE"):
            ctx.solve_pcg_amg(np.ones(3 * m.nV), rel_tol=1e-8, max_iter=100)
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.amg_info()
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        x, iters, res = ctx.solve_pcg_amg(np.ones(3 * m.nV), rel_tol=1e-10, max_iter=1000)
        assert res <= 1e-10 and np.isfinite(x).all()


def test_capture_and_arguments_are_rejected():
    with own_context() as ctx:
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.solve_pcg_amg(None)  # no matrix yet
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.amg_info()
        V, T = M.grid_tets(3, 3, 3)
        m = M.Mesh(V, T, energy=0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.solve_pcg_amg(None, rel_tol=0.0)
        with pytest.raises(L.IpcGpuError, match="ARG"):
            ctx.solve_pcg_amg(None, max_iter=0)
        ctx.solve_pcg_amg(None, rel_tol=1e-8)
        assert ctx.lib.ipcgpu_amg_debug_level(ctx.h, len(ctx.amg_info()["rows"]), None, None, None, None) == 2  # IPCGPU_ERR_ARG
        ctx.capture_begin()
        rc = ctx.lib.ipcgpu_solve_pcg_amg(ctx.h, None, 1e-8, 100, None, 0, None, None)  # (the deferred form)
        ctx.capture_end()
        assert rc == L.ERR_STATE
