"""The deferred form of both built-in solvers (ipcgpu_solve_pcg / _multilevel with rhs, x, iters and rel_residual NULL) inside CUDA graphs:
a captured solve replays to the bits and the iteration count of a synchronous one, the full-row structure follows a
pattern change at replay with nothing on the host, a whole Newton iteration with the solve is one graph, a failed solve is reported by
ipcgpu_fetch_iteration / ipcgpu_solve_info and leaves V = V0, and the capture contract (deferred form only, an eager run first) holds."""
import contextlib

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import multilevel_mirror as mlm
from gpu_common import load_scene, own_context, rel, same_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2
TOL = 1e-6


def load_unsorted(ctx, m):
    load_scene(ctx, m)
    ctx.set_canonical_order(0)  # (inside a capture the contact lists stay in build order)


def pile():
    """ball_pile and two states: A (the scene) and B (half of the feasible step along the scene's direction: more contacts, another pattern)"""
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    with own_context() as ctx:
        load_unsorted(ctx, m)
        p = info["p"]
        evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
        ctx.constraint_set(info["dHat"], 1, fetch=False)
        a = ctx.inversion_step(p, 0.2, 1.0)
        a = ctx.ccd_partial(None, 1e-6, evf, eee, a)
        a = ctx.hash_build_swept(None, a, m.avgEdgeLen / 3)
        a, _ = ctx.ccd_full(1e-6, evf, eee, a)
    return m, info, {"A": m.V.copy(), "B": m.V + 0.5 * a * p.reshape(-1, 3)}


def assemble_at(ctx, V, dHat, kappa):
    """constraint set, device-built pattern, g and H at V: nothing synchronises"""
    ctx.set_state(soa(V))
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)


def resident_system(ctx, n):
    ia, ja = ctx.get_pattern()
    a = ctx.download(L.BUF_CSR_VALUES, len(ja))
    return mlm.full_matrix(ia, ja, a, n, 1), ctx.download(L.BUF_GRADIENT, n)


@pytest.fixture(scope="module")
def scene():
    return pile()


# ---- 1, 2. a graph that holds the solve alone ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("multilevel", [True, False], ids=["multilevel", "block_jacobi"])
def test_solve_only_graph(shared_ctx, scene, multilevel):
    ctx = shared_ctx
    m, info, S = scene
    dHat, kappa, n, tol = info["dHat"], 1e6, 3 * m.nV, 1e-10
    solve = ctx.solve_pcg_multilevel if multilevel else ctx.solve_pcg
    load_unsorted(ctx, m)
    ctx.enable_device_pattern(1)
    assemble_at(ctx, S["A"], dHat, kappa)
    solve(None, rel_tol=tol, max_iter=5000, want_x=False, adopt=True)  # the eager run: lazy allocations
    ctx.capture_begin()
    assert solve(rel_tol=tol, max_iter=5000, want_x=False, adopt=True, deferred=True) is None
    gid = ctx.capture_end()
    for name in ("A", "B"):
        assemble_at(ctx, S[name], dHat, kappa)
        x, iters, res = solve(None, rel_tol=tol, max_iter=5000)
        ctx.graph_launch(gid)
        r = ctx.solve_info()
        p = ctx.download(L.BUF_SEARCH_DIR, n)
        assert r.status == 0 and res <= tol and r.rel_residual <= tol and 0 < r.iterations < 5000
        assert r.max_abs_x == np.abs(p).max()
        assert same_bits(p, x) and r.iterations == iters and same_bits(r.rel_residual, res)
    ctx.graph_destroy(gid)


# ---- 3. the pattern changes between replays ------------------------------------------------------------------------------------------
def test_pattern_change_between_replays(shared_ctx, scene):
    ctx = shared_ctx
    m, info, S = scene
    dHat, kappa, n, tol = info["dHat"], 1e6, 3 * m.nV, 1e-10

    def sequence(V):
        assemble_at(ctx, V, dHat, kappa)
        ctx.solve_pcg_multilevel(rel_tol=tol, max_iter=5000, want_x=False, adopt=True, deferred=True)

    load_unsorted(ctx, m)
    ctx.enable_device_pattern(1)
    sequence(S["A"])
    assert ctx.solve_info().status == 0 and ctx.fetch_iteration().status == 0
    ctx.capture_begin()
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.solve_pcg_multilevel(rel_tol=tol, max_iter=5000, want_x=False, adopt=True, deferred=True)
    gid = ctx.capture_end()
    ctx.set_state(soa(S["A"]))
    ctx.graph_launch(gid)
    assert ctx.fetch_iteration().status == 0
    _, nnz_a, version_a = ctx.pattern_info()
    ctx.set_state(soa(S["B"]))
    ctx.graph_launch(gid)
    r = ctx.solve_info()
    changed, nnz_b, version_b = ctx.pattern_info()
    assert changed == 1 and version_b > version_a and nnz_b != nnz_a and r.status == 0
    p = ctx.download(L.BUF_SEARCH_DIR, n)
    H, g = resident_system(ctx, n)
    assert rel(p, spla.spsolve(H.tocsc(), -g)) <= 1e-7
    x, iters, res = ctx.solve_pcg_multilevel(None, rel_tol=tol, max_iter=5000)  # eager, on the system the replay left
    assert same_bits(p, x) and iters == r.iterations and same_bits(res, r.rel_residual)
    # the same state again: the pattern does not change and the full rows are not rebuilt; the direction is again the eager solve's bits
    # (the barrier terms' atomics make the reassembled system differ from the first one in its last bits)
    ctx.set_state(soa(S["B"]))
    ctx.graph_launch(gid)
    assert ctx.pattern_info() == (0, nnz_b, version_b)
    p2, r2 = ctx.download(L.BUF_SEARCH_DIR, n), ctx.solve_info()
    x2, iters2, _ = ctx.solve_pcg_multilevel(None, rel_tol=tol, max_iter=5000)
    assert same_bits(p2, x2) and r2.iterations == iters2 and rel(p2, p) <= 1e-9
    ctx.graph_destroy(gid)


# ---- 4. a whole Newton iteration in one graph ----------------------------------------------------------------------------------------
def newton_iteration(ctx, m, dHat, kappa, evf, eee):
    """INTEGRATION.md section 4 with the multilevel solve: every call in its NULL-output form"""
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0, want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    # (a tight tolerance: the two contexts' systems differ in their last bits, and the directions agree to about rel_tol)
    ctx.solve_pcg_multilevel(rel_tol=1e-12, max_iter=5000, want_x=False, adopt=True, deferred=True)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, TOL, evf, eee, None)
    ctx.ccd_cfl(dHat, 1, m.avgEdgeLen / 3.0, TOL, evf, eee, None)
    ctx.line_search(DT2, dHat, kappa)


def test_whole_newton_iteration_graph(shared_ctx, scene):
    m, info, _ = scene
    dHat, kappa, n = info["dHat"], 1e6, 3 * m.nV
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    g_ctx = shared_ctx
    with own_context() as e_ctx:
        for c in (g_ctx, e_ctx):
            load_unsorted(c, m)
            c.enable_device_pattern(1)
        newton_iteration(g_ctx, m, dHat, kappa, evf, eee)  # the eager run: lazy allocations
        g_ctx.fetch_iteration()
        g_ctx.set_state(m.V_soa)
        g_ctx.capture_begin()
        newton_iteration(g_ctx, m, dHat, kappa, evf, eee)
        gid = g_ctx.capture_end()
        for k in range(3):
            newton_iteration(e_ctx, m, dHat, kappa, evf, eee)
            e, es, ie = e_ctx.step_control_info(), e_ctx.solve_info(), e_ctx.fetch_iteration()
            n0 = g_ctx.launch_count()
            g_ctx.graph_launch(gid)  # (one cudaGraphLaunch: the whole iteration, solve included)
            assert g_ctx.launch_count() > n0
            g, gs, ig = g_ctx.step_control_info(), g_ctx.solve_info(), g_ctx.fetch_iteration()
            assert ig.status == ie.status == 0 and g.status == e.status == 0 and gs.status == es.status == 0
            assert abs(gs.iterations - es.iterations) <= 25 and gs.iterations > 0
            assert rel(g.alpha, e.alpha) <= 1e-9 and g.alpha > 0.0, (k, g.alpha, e.alpha)
            assert rel(g.energy_start, e.energy_start) <= 1e-9 and rel(g.energy, e.energy) <= 1e-9
            Vg, Ve = g_ctx.download(L.BUF_POSITIONS, n), e_ctx.download(L.BUF_POSITIONS, n)
            assert rel(Vg, Ve) <= 1e-9 and not np.array_equal(Vg, soa(m.V))
        g_ctx.graph_destroy(gid)


# ---- 5. a failed solve -------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def small_context():
    with own_context() as ctx:  # (a context of its own: the error must not leak into the shared one)
        V, T = M.grid_tets(2, 2, 2)
        m = M.Mesh(V, T, energy=0)
        load_unsorted(ctx, m)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(soa(m.V * 1.05))  # stretched: a nonzero elastic gradient, no inverted tet
        yield ctx, m, len(ja)


@pytest.mark.parametrize("multilevel", [True, False], ids=["multilevel_pivot", "block_jacobi_nan"])
def test_failed_deferred_solve(multilevel):
    with small_context() as (ctx, m, nnz):
        n, dHat = 3 * m.nV, 1e-8
        solve = ctx.solve_pcg_multilevel if multilevel else ctx.solve_pcg

        def sequence():
            solve(rel_tol=1e-8, max_iter=100, want_x=False, adopt=True, deferred=True)
            ctx.line_search(DT2, dHat, 1.0)

        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        sequence()  # the eager run on a positive definite system: lazy allocations of the solve and of the line search
        assert ctx.fetch_iteration().status == 0 and ctx.solve_info().status == 0
        ctx.capture_begin()
        sequence()
        gid = ctx.capture_end()
        if multilevel:
            ctx.csr_set_zero()  # the first pivot of every domain is 0
        else:
            ctx.elastic_hessian(DT2, a_inout=np.full(nnz, np.nan))  # a non-finite residual
        V0 = ctx.download(L.BUF_POSITIONS, n)
        ctx.graph_launch(gid)  # (returns: no hang)
        r = ctx.solve_info()
        assert r.status == L.ERR_SOLVE and ctx.step_control_info().status == L.ERR_SOLVE
        with pytest.raises(L.IpcGpuError, match="SOLVE"):
            ctx.fetch_iteration()
        assert same_bits(ctx.download(L.BUF_POSITIONS, n), V0)
        ctx.fetch_iteration()  # (the flag is per fetch)
        # outside a capture the host-output forms return what they always did
        if multilevel:
            with pytest.raises(L.IpcGpuError, match="SOLVE"):
                ctx.solve_pcg_multilevel(np.ones(n), rel_tol=1e-8, max_iter=100)
        else:
            _, iters, res = ctx.solve_pcg(np.ones(n), rel_tol=1e-8, max_iter=100)
            assert np.isnan(res) and iters == 25
        assert ctx.fetch_iteration().status == 0  # (they raise no deferred flag)
        # the context solves a positive definite system afterwards
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        x, iters, res = solve(np.ones(n), rel_tol=1e-10, max_iter=1000)
        assert res <= 1e-10 and np.isfinite(x).all()
        ctx.graph_destroy(gid)


# ---- 6. the capture contract -------------------------------------------------------------------------------------------------------
def test_capture_contract():
    with small_context() as (ctx, m, _):
        n = 3 * m.nV
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        for solve in (ctx.solve_pcg, ctx.solve_pcg_multilevel):  # a capture before any eager run
            ctx.capture_begin()
            with pytest.raises(L.IpcGpuError, match="STATE.*outside a capture first"):
                solve(rel_tol=1e-8, max_iter=100, want_x=False, deferred=True)
            ctx.graph_destroy(ctx.capture_end())
        for solve, raw in ((ctx.solve_pcg, ctx.lib.ipcgpu_solve_pcg), (ctx.solve_pcg_multilevel, ctx.lib.ipcgpu_solve_pcg_multilevel)):
            x, iters, res = solve(None, rel_tol=1e-10, max_iter=1000)  # outside a capture: as before
            assert res <= 1e-10 and iters > 0
            r = ctx.solve_info()
            assert r.status == 0 and r.iterations == iters and same_bits(r.rel_residual, res) and r.max_abs_x == np.abs(x).max()
            ctx.capture_begin()
            with pytest.raises(L.IpcGpuError, match="STATE"):  # a host right-hand side
                ctx._ck(raw(ctx.h, L._d(np.ones(n)), 1e-8, 100, None, 0, None, None))
            with pytest.raises(L.IpcGpuError, match="STATE"):  # a host output
                solve(None, rel_tol=1e-8, max_iter=100, want_x=True)
            with pytest.raises(L.IpcGpuError, match="STATE"):
                solve(None, rel_tol=1e-8, max_iter=100, want_x=False)  # (iters / rel_residual are host outputs too)
            solve(rel_tol=1e-8, max_iter=100, want_x=False, deferred=True)
            gid = ctx.capture_end()
            ctx.graph_launch(gid)
            r = ctx.solve_info()
            assert r.status == 0 and 0 < r.iterations <= 100 and r.rel_residual <= 1e-8
            ctx.graph_destroy(gid)
        with pytest.raises(ValueError):
            ctx.solve_pcg(np.ones(n), deferred=True)
