"""ipcgpu_solve_pcg_amg after ipcgpu_amg_reserve: the set-up reads its sizes from device memory, so the deferred solve runs inside a CUDA
graph.  Every comparison is against an UNRESERVED eager solve in a second context driven through the same states in the reproducible mode
(ipcgpu_set_canonical_order(ctx, 2): the two contexts hold the same system bit for bit).  A reserved eager solve and a replayed graph give the
unreserved bits, iteration count, residual, hierarchy and level matrices on ball_pile and ball_on_mat, with the device-built and the host
pattern, also after contacts changed the device-built pattern; a whole captured Newton iteration with the AMG solve replays to the eager
iterations; the level count moves inside one graph with the coarse-enough hook; a set-up deeper than reserved, or one that outgrows a count,
is cut short, reported and still converges, and new reservations restore the unreserved bits; a failed solve inside a graph is reported at
the fetch and leaves V = V0; and the reservation's refusals hold."""
import contextlib

import numpy as np
import pytest

from gpu_common import load_scene, own_context, same_bits, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs
from test_gpu_reproducible import snapshot
from test_gpu_solve_capture import DT2, pile, small_context

pytestmark = pytest.mark.gpu
TOL = 1e-8
KAPPA = 1e6


def mat():
    """ball_on_mat with the ball at half a contact distance over the mat (A), then lowered by a fifth of it (B: more contacts)"""
    m, info = scenes.ball_on_mat(nx=24, res=5, seed=3)
    sq, nm = np.sqrt(info["dHat"]), info["n_mat_verts"]
    A = m.V.copy()
    A[nm:, 2] -= info["gap"] - 0.5 * sq
    B = A.copy()
    B[nm:, 2] -= 0.2 * sq
    return m, info, {"A": A, "B": B}


SCENES = {"ball_pile": pile, "ball_on_mat": mat}


def start(ctx, m, device_pattern):
    load_scene(ctx, m)
    ctx.set_canonical_order(2)
    if device_pattern:
        ctx.enable_device_pattern(1)


def assemble(ctx, m, V, dHat, device_pattern=True):
    """g and H at V; the host pattern is built from the fetched contact lists (a new pattern: a new epoch)"""
    ctx.set_state(soa(V))
    if device_pattern:
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
    else:
        mm, pa, pe, _ = ctx.constraint_set(dHat, 1)
        ctx.set_csr(*m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe)), 1)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, KAPPA, None)
    ctx.barrier_hessian(dHat, KAPPA, 1, None)


def hierarchy(ctx):
    h = ctx.amg_info()
    h.pop("bytes")
    return h, [ctx.amg_debug_level(l) for l in range(len(h["rows"]))]


def same_hierarchy(a, b):
    (ha, la), (hb, lb) = a, b
    return ha == hb and all(all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(p, q)) for p, q in zip(la, lb))


def eager(ctx, tol=TOL):
    """the synchronous solve; it adopts its solution as the captured solves do"""
    return ctx.solve_pcg_amg(None, rel_tol=tol, max_iter=5000, adopt=True)


def capture_solve(ctx, tol=TOL, **kw):
    """a graph that holds the deferred solve alone (the capture is ended even when the call is refused)"""
    ctx.capture_begin()
    try:
        ctx.solve_pcg_amg(rel_tol=tol, max_iter=5000, want_x=False, deferred=True, **kw)
    finally:
        gid = ctx.capture_end()
    return gid


def replay_equals_unreserved(r, gid, u, n):
    """replay the graph in r, solve eagerly in the never-reserved u: the same bits, iterations, residual and hierarchy"""
    r.graph_launch(gid)
    res = r.solve_info()
    p = r.download(L.BUF_SEARCH_DIR, n)
    x, iters, rr = eager(u)
    assert res.status == 0 and res.rel_residual <= TOL and np.isfinite(p).all()
    assert same_bits(p, x) and res.iterations == iters and same_bits(res.rel_residual, rr)
    assert same_hierarchy(hierarchy(r), hierarchy(u))
    return res


def reserve_until_it_fits(r, headroom):
    """reserve, solve eagerly, until the set-up is not cut (a cut set-up counts nothing past the count that cut it)"""
    for _ in range(24):
        r.amg_reserve(headroom)
        eager(r)
        if r.amg_capacity_info()[0] == -1:
            return
    raise AssertionError("the set-up is still cut after 24 reservations")


@contextlib.contextmanager
def contexts(m, device_pattern):
    with own_context() as r, own_context() as u:
        for c in (r, u):
            start(c, m, device_pattern)
        yield r, u


# ---- 1, 2. reserved eager and replays equal unreserved eager ---------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", ["device", "host"])
@pytest.mark.parametrize("name", list(SCENES))
def test_reserved_and_replayed_equal_unreserved(name, pattern):
    m, info, S = SCENES[name]()
    dHat, n, dev = info["dHat"], 3 * m.nV, pattern == "device"
    with contexts(m, dev) as (r, u):
        for c in (r, u):
            assemble(c, m, S["A"], dHat, dev)
        x0, it0, res0 = eager(r)  # (unreserved in both: the two contexts hold one system)
        xu, itu, resu = eager(u)
        assert res0 <= TOL and same_bits(x0, xu) and it0 == itu and same_bits(res0, resu) and same_hierarchy(hierarchy(r), hierarchy(u))
        assert name != "ball_pile" or len(r.amg_info()["rows"]) >= 2
        r.amg_reserve(1.5)
        x1, it1, res1 = eager(r)
        assert same_bits(x1, xu) and it1 == itu and same_bits(res1, resu) and same_hierarchy(hierarchy(r), hierarchy(u))
        assert r.amg_capacity_info()[0] == -1
        gid = capture_solve(r, adopt=True)
        # device pattern: at A, after a step towards B and at B (contacts change the device-built pattern and so level 0); host pattern: a
        # new pattern is a new epoch, so the replays stay at A
        Vs = (S["A"], 0.5 * (S["A"] + S["B"]), S["B"]) if dev else (S["A"], S["A"])
        for V in Vs:
            if dev:
                for c in (r, u):
                    assemble(c, m, V, dHat)
            replay_equals_unreserved(r, gid, u, n)
            assert r.amg_capacity_info()[0] == -1
        r.graph_destroy(gid)


# ---- 3. the whole Newton iteration in one graph --------------------------------------------------------------------------------------
def newton_iteration(ctx, m, dHat, evf, eee):
    """INTEGRATION.md section 4 with the AMG solve: every call in its NULL-output form"""
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, KAPPA, None)
    ctx.barrier_hessian(dHat, KAPPA, 1, None)
    ctx.solve_pcg_amg(rel_tol=TOL, max_iter=5000, want_x=False, adopt=True, deferred=True)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, 1e-6, evf, eee, None)
    ctx.ccd_cfl(dHat, 1, m.avgEdgeLen / 3.0, 1e-6, evf, eee, None)
    ctx.line_search(DT2, dHat, KAPPA)


def test_captured_newton_iteration_equals_unreserved_eager():
    m, info, _ = pile()
    dHat = info["dHat"]
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    with contexts(m, True) as (g, e):
        newton_iteration(g, m, dHat, evf, eee)  # unreserved: the hierarchy the reservation is sized from
        g.fetch_iteration()
        g.amg_reserve(1.5)
        g.set_state(soa(m.V))
        newton_iteration(g, m, dHat, evf, eee)  # the eager run after the reservation
        g.fetch_iteration()
        g.set_state(soa(m.V))
        g.capture_begin()
        try:
            newton_iteration(g, m, dHat, evf, eee)
        finally:
            gid = g.capture_end()
        for k in range(3):
            newton_iteration(e, m, dHat, evf, eee)
            se = snapshot(e, m)
            g.graph_launch(gid)
            sg = snapshot(g, m)
            assert se["scalars"][0] > 0.0 and se["counts"][-1] > 0
            for key in ("V", "g", "a", "scalars"):
                assert same_bits(sg[key], se[key]), (k, key)
            assert sg["counts"] == se["counts"], k  # (halvings and Krylov iterations)
        g.graph_destroy(gid)


# ---- 4. the level count moves inside one graph ---------------------------------------------------------------------------------------
def test_level_count_moves_inside_one_graph():
    m, info, S = pile()
    dHat, n = info["dHat"], 3 * m.nV
    with contexts(m, True) as (r, u), own_context() as d:
        start(d, m, True)
        for c in (r, u, d):
            assemble(c, m, S["A"], dHat)
        eager(u)
        rows = u.amg_info()["rows"]
        assert len(rows) >= 2 and rows[0] > 1000
        eager(r)
        r.amg_reserve(2.0)
        eager(r)
        gid = capture_solve(r, adopt=True)
        # fewer levels than reserved: level 0 is coarse enough.  The replay is the unreserved solve at that threshold
        for c in (r, u):
            c.amg_debug_coarse_enough(rows[0])
        replay_equals_unreserved(r, gid, u, n)
        assert len(r.amg_info()["rows"]) == 1 and r.amg_capacity_info()[0] == -1
        for c in (r, u):
            c.amg_debug_coarse_enough(1000)
        replay_equals_unreserved(r, gid, u, n)
        r.graph_destroy(gid)
        # more levels than reserved: a reservation of one level, replayed at the default threshold, is cut at level 0 by its depth
        d.amg_debug_coarse_enough(rows[0])
        eager(d)
        d.amg_reserve(1.5)
        eager(d)
        gid = capture_solve(d, adopt=True)
        d.amg_debug_coarse_enough(1000)
        d.graph_launch(gid)
        res = d.solve_info()
        p = d.download(L.BUF_SEARCH_DIR, n)
        cut, need, reserved = d.amg_capacity_info()
        assert cut == 0 and len(d.amg_info()["rows"]) == 1
        assert res.status == 0 and res.rel_residual <= TOL and np.isfinite(p).all()
        d.graph_destroy(gid)
        # reserving again adds the level the set-up wanted; once nothing is cut, a new graph gives the unreserved bits
        reserve_until_it_fits(d, 1.5)
        gid = capture_solve(d, adopt=True)
        replay_equals_unreserved(d, gid, u, n)
        d.graph_destroy(gid)


# ---- 5. a set-up that outgrows its reservation ---------------------------------------------------------------------------------------
def test_overflow_is_cut_short_and_new_reservations_restore_the_bits():
    m, info, S = pile()
    dHat, n = info["dHat"], 3 * m.nV
    with contexts(m, True) as (r, u):
        assemble(r, m, S["A"], 1e-8 * dHat)  # (a contact distance of 1e-4 of the scene's: no contact)
        eager(r)
        r.amg_reserve(1.0)  # exactly what the contact-free set-up needed
        eager(r)
        gid = capture_solve(r, adopt=True)
        for c in (r, u):
            assemble(c, m, S["B"], dHat)  # contacts add blocks to level 0, and so to its products
        r.graph_launch(gid)
        res = r.solve_info()
        p = r.download(L.BUF_SEARCH_DIR, n)
        cut, need, reserved = r.amg_capacity_info()
        assert cut >= 0, "contacts at B add blocks to level 0: a reservation of exactly A's counts must be cut"
        assert (need[cut] > reserved[cut]).any(), (cut, need[cut], reserved[cut])
        assert len(r.amg_info()["rows"]) == cut + 1
        assert res.status == 0 and res.rel_residual <= TOL and np.isfinite(p).all()
        r.graph_destroy(gid)
        reserve_until_it_fits(r, 1.0)
        gid = capture_solve(r, adopt=True)
        replay_equals_unreserved(r, gid, u, n)
        r.graph_destroy(gid)


# ---- 6. failure, 7. refusals -----------------------------------------------------------------------------------------------------------
def test_failed_solve_inside_a_graph():
    with small_context() as (ctx, m, nnz):
        n, dHat = 3 * m.nV, 1e-8

        def sequence():
            ctx.solve_pcg_amg(rel_tol=1e-8, max_iter=100, want_x=False, adopt=True, deferred=True)
            ctx.line_search(DT2, dHat, 1.0)

        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.solve_pcg_amg(None, rel_tol=1e-8)
        ctx.amg_reserve(1.5)
        sequence()  # the eager run after the reservation
        assert ctx.fetch_iteration().status == 0 and ctx.solve_info().status == 0
        ctx.capture_begin()
        try:
            sequence()
        finally:
            gid = ctx.capture_end()
        ctx.csr_set_zero()  # no diagonal block is positive definite
        V0 = ctx.download(L.BUF_POSITIONS, n)
        ctx.graph_launch(gid)  # (returns: no hang)
        r = ctx.solve_info()
        assert r.status == L.ERR_SOLVE and ctx.step_control_info().status == L.ERR_SOLVE
        with pytest.raises(L.IpcGpuError, match="SOLVE"):
            ctx.fetch_iteration()
        assert same_bits(ctx.download(L.BUF_POSITIONS, n), V0)
        ctx.graph_destroy(gid)


def test_refusals():
    with own_context() as ctx:
        V, T = M.grid_tets(4, 4, 4)
        m = M.Mesh(V, T, energy=0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.amg_reserve(1.5)  # no hierarchy yet
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.solve_pcg_amg(None, rel_tol=1e-8)
        for bad in (0.5, float("nan"), float("inf")):
            with pytest.raises(L.IpcGpuError, match="ARG"):
                ctx.amg_reserve(bad)
        ctx.amg_reserve(1.5)
        ctx.solve_pcg_amg(None, rel_tol=1e-8, want_x=False)
        gid = capture_solve(ctx, tol=1e-8)
        ctx.graph_launch(gid)
        assert ctx.solve_info().status == 0
        ctx.amg_reserve(2.0)  # a later reservation refuses the older graph
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.graph_launch(gid)
        ctx.graph_destroy(gid)
