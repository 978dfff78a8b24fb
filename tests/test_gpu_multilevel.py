"""ipcgpu_solve_pcg_multilevel: PCG on the device-resident Hessian with the multilevel additive Schwarz preconditioner.  The solution equals
a host direct solve, the stored inverses, the application and the iteration count equal the host mirror's (tests/multilevel_mirror.py),
two calls of either solver give identical bits and make 6 + L (multilevel) or 4 (block-Jacobi) launches per iteration, the device-built
pattern, an obstacle tail and Dirichlet vertices are covered, a non-positive pivot is an error and not a hang, and the iterations are at most
half of block-Jacobi's on ball_on_mat."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import multilevel_mirror as mlm
import oracle as orc
from gpu_common import load_scene, own_context, rel, same_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2


def load_sorted(ctx, m):
    load_scene(ctx, m)
    ctx.set_canonical_order(1)


def assemble(ctx, m, dHat, kappa):
    """g and H on the device (elastic + mass + barrier) on the host-built contact pattern; returns the pattern and the sets"""
    load_sorted(ctx, m)
    mm, pa, pe, _ = ctx.constraint_set(dHat, 1)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    ctx.set_csr(ia, ja, 1)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    return ia, ja


def resident_system(ctx, ia, ja, n, base=1):
    """the matrix and gradient the device holds, on the host"""
    a = ctx.download(L.BUF_CSR_VALUES, len(ja))
    return mlm.full_matrix(ia, ja, a, n, base), ctx.download(L.BUF_GRADIENT, n)


def states(ctx, m, info):
    """A (the scene) and B (half of the feasible step along the scene's direction: more contacts, another pattern)"""
    p = info["p"]
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    ctx.constraint_set(info["dHat"], 1, fetch=False)
    a = ctx.inversion_step(p, 0.2, 1.0)
    a = ctx.ccd_partial(None, 1e-6, evf, eee, a)
    a = ctx.hash_build_swept(None, a, m.avgEdgeLen / 3)
    a, _ = ctx.ccd_full(1e-6, evf, eee, a)
    return {"A": m.V.copy(), "B": m.V + 0.5 * a * p.reshape(-1, 3)}


def test_multilevel_pcg_on_the_device_resident_hessian(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    dHat, kappa = info["dHat"], 1e6
    ia, ja = assemble(ctx, m, dHat, kappa)
    x, iters, res = ctx.solve_pcg_multilevel(None, rel_tol=1e-10, max_iter=5000)
    assert res <= 1e-10 and 0 < iters < 5000
    # host reference: oracle matrix and gradient, direct solve
    _, ja_ref, a_ref, g_ref, H_ref, _ = mlm.newton_system(m, dHat, kappa, DT2)
    assert np.array_equal(ja_ref, ja)
    x_ref = spla.spsolve(H_ref.tocsc(), -g_ref)
    assert rel(x, x_ref) <= 1e-7
    b = np.linspace(-1.0, 1.0, 3 * m.nV)
    xb, _, resb = ctx.solve_pcg_multilevel(b, rel_tol=1e-10, max_iter=5000)
    assert resb <= 1e-10 and rel(xb, spla.spsolve(H_ref.tocsc(), b)) <= 1e-7
    # adoption as the search direction: the same inversion step as from the block-Jacobi solve and from the oracle
    ctx.solve_pcg_multilevel(None, rel_tol=1e-10, max_iter=5000, want_x=False, adopt=True)
    al = ctx.inversion_step(None, 0.2, 1.0)
    ctx.solve_pcg(None, rel_tol=1e-10, max_iter=5000, want_x=False, adopt=True)
    al_bj = ctx.inversion_step(None, 0.2, 1.0)
    al_ref, _ = orc.Elastic(m).inversion_step(x, 0.2, 1.0)
    assert abs(al - al_ref) <= 1e-9 * al_ref and abs(al - al_bj) <= 1e-9 * al_ref
    # fewer iterations than block-Jacobi at the same tolerance
    assert iters <= ctx.solve_pcg(None, rel_tol=1e-10, max_iter=5000)[1]


def test_hierarchy_application_and_iterations_equal_the_mirror(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    ia, ja = assemble(ctx, m, info["dHat"], 1e6)
    n = 3 * m.nV
    H, g = resident_system(ctx, ia, ja, n)
    ML = mlm.Multilevel(H, m.V)
    x, iters, res = ctx.solve_pcg_multilevel(None, rel_tol=1e-10, max_iter=5000)
    domains, nbytes = ctx.multilevel_info()
    assert domains == ML.domains and nbytes == ML.stored_bytes() == 73728 * sum(domains)
    inv = ctx.download(L.BUF_MULTILEVEL_INVERSES, 9216 * sum(domains))
    o = 0
    for l, nD in enumerate(domains):
        X = inv[o: o + 9216 * nD].reshape(nD, 96, 96)
        o += 9216 * nD
        assert np.array_equal(X, X.transpose(0, 2, 1))  # stored exactly symmetric
        cond = np.linalg.cond(ML.A[l]).max()
        # the stored inverses: an inverse is determined to rounding times the conditioning of what is inverted, by any algorithm
        assert rel(X, ML.Ainv[l]) <= 1e-12 * cond, (l, rel(X, ML.Ainv[l]), cond)
    # z = M^-1 r for a random r: the first iterate of a solve with right-hand side r is alpha z, alpha = r.z / z.Hz
    r = np.random.default_rng(1).standard_normal(n)
    z = ML.apply(r)
    x1, it1, _ = ctx.solve_pcg_multilevel(r, rel_tol=1e-10, max_iter=1)
    assert it1 == 1 and rel(x1, (r @ z) / (z @ (H @ z)) * z) <= 1e-12 * np.linalg.cond(ML.A[0]).max()
    # the same recurrences: residuals along the way, and the iteration count
    # (over the first iterations only: rounding differences grow along the recurrence, and the residual norm of CG is not monotone)
    for k in (5, 12):
        _, it_k, res_k = ctx.solve_pcg_multilevel(None, rel_tol=1e-30, max_iter=k)
        res_m = mlm.pcg(H, -g, ML.apply, 1e-30, k)[2]
        assert it_k == k and abs(res_k - res_m) <= 1e-6 * res_m, (k, res_k, res_m)
    xm, it_m, _ = mlm.pcg(H, -g, ML.apply, 1e-10, 5000)
    assert abs(iters - it_m) <= 2 and rel(x, xm) <= 1e-8
    # the level matrices as assembled, before any inversion: sums of the same entries in another order, entry by entry
    A_dev = ctx.multilevel_debug_matrices()
    for l, A in enumerate(A_dev):
        scale = np.abs(ML.A[l]).max(axis=(1, 2), keepdims=True)
        # (an entry and its transpose are sums in different orders: symmetric to rounding; the stored inverse mirrors one triangle)
        assert A.shape == ML.A[l].shape and (np.abs(A - A.transpose(0, 2, 1)) <= 1e-14 * scale).all()
        assert (np.abs(A - ML.A[l]) <= 1e-12 * scale).all(), (l, np.abs(A - ML.A[l]).max())
    with pytest.raises(L.IpcGpuError, match="STATE"):  # the hook leaves no inverses behind
        ctx.multilevel_info()


def launches_of_25_more_iterations(ctx, solve):
    """launches of a solve to max_iter 50 minus those of one to 25, at an unreachable tolerance: 25 iterations and one burst decision"""
    counts = []
    for max_iter in (25, 50):
        n0 = ctx.launch_count()
        assert solve(None, rel_tol=1e-30, max_iter=max_iter, want_x=False)[1] == max_iter
        counts.append(ctx.launch_count() - n0)
    return counts[1] - counts[0]


def test_two_solves_give_identical_bits(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    assemble(ctx, m, info["dHat"], 1e8)
    x1, it1, res1 = ctx.solve_pcg_multilevel(None, rel_tol=1e-8, max_iter=5000)
    inv1 = ctx.download(L.BUF_MULTILEVEL_INVERSES, 9216 * sum(ctx.multilevel_info()[0]))
    ctx.solve_pcg(None, rel_tol=1e-3, max_iter=50)  # (another solver in between shares the workspace)
    x2, it2, res2 = ctx.solve_pcg_multilevel(None, rel_tol=1e-8, max_iter=5000)
    inv2 = ctx.download(L.BUF_MULTILEVEL_INVERSES, 9216 * sum(ctx.multilevel_info()[0]))
    assert res1 <= 1e-8 and it1 == it2 and same_bits(res1, res2) and same_bits(x1, x2) and same_bits(inv1, inv2)
    # 6 + L launches per iteration: SpMV, reduce, update, L levels, prolongation, roll, direction
    assert launches_of_25_more_iterations(ctx, ctx.solve_pcg_multilevel) == 25 * (6 + len(ctx.multilevel_info()[0])) + 1


def test_two_block_jacobi_solves_give_identical_bits(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    assemble(ctx, m, info["dHat"], 1e8)
    x1, it1, res1 = ctx.solve_pcg(None, rel_tol=1e-8, max_iter=5000)
    ctx.solve_pcg_multilevel(None, rel_tol=1e-3, max_iter=50)  # (another solver in between shares the workspace)
    x2, it2, res2 = ctx.solve_pcg(None, rel_tol=1e-8, max_iter=5000)
    assert res1 <= 1e-8 and it1 == it2 and same_bits(res1, res2) and same_bits(x1, x2)
    # 4 launches per iteration: SpMV, block-Jacobi step (alpha summed inside), roll, direction
    assert launches_of_25_more_iterations(ctx, ctx.solve_pcg) == 25 * 4 + 1


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
        x, iters, res = ctx.solve_pcg_multilevel(None, rel_tol=1e-10, max_iter=5000)
        assert res <= 1e-10 and 0 < iters < 5000
        assert ctx.pattern_info()[0] == 1
    x2, iters2, _ = ctx.solve_pcg_multilevel(None, rel_tol=1e-10, max_iter=5000)
    assert iters2 == iters and same_bits(x, x2)
    _, _, _, g_ref, H_ref, _ = mlm.newton_system(m, dHat, kappa, DT2, V=S["B"])
    assert rel(x, spla.spsolve(H_ref.tocsc(), -g_ref)) <= 1e-7
    # the hierarchy follows the positions: the mirror at B gives the same count
    ia, ja = ctx.get_pattern()
    H, g = resident_system(ctx, ia, ja, 3 * m.nV)
    assert abs(mlm.pcg(H, -g, mlm.Multilevel(H, S["B"]).apply, 1e-10, 5000)[1] - iters) <= 2


def test_obstacle_tail_and_dirichlet_vertices(shared_ctx):
    from ipc_b200 import obstacle as OB
    ctx = shared_ctx
    m, info = scenes.balls_on_obstacle(plate_angle=0.0, res=4, plate=12)
    ob = info["obstacle"]
    M2 = OB.with_obstacle(m, ob["V"], ob["E"], ob["F"])
    M2.dbc = M2.dbc.copy()
    M2.dbc[:5] = 1  # Dirichlet vertices of the mesh besides the tail
    load_sorted(ctx, M2)
    ctx.set_obstacle_tail(M2.nV_dof, 1)
    try:
        ctx.enable_device_pattern(1)
        mm, _, _, _ = ctx.constraint_set(info["dHat"], 1)
        assert len(mm) > 0
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
        Hnz = H.copy()
        Hnz.eliminate_zeros()
        assert Hnz[fixed].nnz == fixed.size and (Hnz.diagonal()[fixed] > 0).all()  # decoupled rows
        b = np.random.default_rng(2).standard_normal(n)
        b[fixed] = 0.0
        x, iters, res = ctx.solve_pcg_multilevel(b, rel_tol=1e-10, max_iter=5000)
        x_ref = spla.spsolve(H.tocsc(), b)
        assert res <= 1e-10 and 0 < iters < 5000 and rel(x, x_ref) <= 1e-7
        # vertices without degrees of freedom are in no coarse aggregate: exactly zero, at any tolerance
        assert (x[fixed] == 0.0).all()
        assert ctx.multilevel_info()[0] == mlm.level_sizes(M2.nV)  # the tail is part of the order
        ML = mlm.Multilevel(H, M2.V, fixed=fixed_v)
        assert abs(mlm.pcg(H, b, ML.apply, 1e-10, 5000)[1] - iters) <= 2
        for l, A in enumerate(ctx.multilevel_debug_matrices()):
            scale = np.abs(ML.A[l]).max(axis=(1, 2), keepdims=True)
            assert (np.abs(A - ML.A[l]) <= 1e-12 * scale).all(), l
        # the Newton direction at the working tolerance, adopted: the step-bound stages must not move these vertices
        # (the right-hand side a caller with such vertices solves for: the gradient with their rows projected out)
        bn = -g
        bn[fixed] = 0.0
        xn, _, resn = ctx.solve_pcg_multilevel(bn, rel_tol=1e-6, max_iter=5000, adopt=True)
        p = ctx.download(L.BUF_SEARCH_DIR, n)
        assert resn <= 1e-6 and np.array_equal(p, xn) and (p[fixed] == 0.0).all() and np.abs(p).max() > 0.0
        assert rel(xn, spla.spsolve(H.tocsc(), bn)) <= 1e-3
    finally:
        ctx.set_obstacle_tail(-1)


def test_nonpositive_pivot_is_an_error_and_not_a_hang():
    with own_context() as ctx:  # (a context of its own: the error must not leak into the shared one)
        V, T = M.grid_tets(2, 2, 2)
        m = M.Mesh(V, T, energy=0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, 0)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        ctx.csr_set_zero()  # an all-zero matrix: the first pivot of every domain is 0
        with pytest.raises(L.IpcGpuError, match="SOLVE"):
            ctx.solve_pcg_multilevel(np.ones(3 * m.nV), rel_tol=1e-8, max_iter=100)
        with pytest.raises(L.IpcGpuError, match="STATE"):  # a failed call leaves no hierarchy to report
            ctx.multilevel_info()
        # the context stays usable: a positive definite matrix solves
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        x, iters, res = ctx.solve_pcg_multilevel(np.ones(3 * m.nV), rel_tol=1e-10, max_iter=1000)
        assert res <= 1e-10 and np.isfinite(x).all()


def test_single_rank_contract_and_arguments(shared_ctx):
    with own_context() as ctx:
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.solve_pcg_multilevel(None)  # no matrix yet
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.multilevel_info()
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    assemble(shared_ctx, m, info["dHat"], 1e6)
    with pytest.raises(L.IpcGpuError, match="ARG"):
        shared_ctx.solve_pcg_multilevel(None, rel_tol=0.0)


def first_iteration_below(solve, tol):
    """the solvers test the residual every 25 iterations; the first iteration at which it is below tol, by re-solving with that many"""
    x, hi, res = solve(None, rel_tol=tol, max_iter=20000)
    assert res <= tol
    for k in range(max(hi - 24, 1), hi):
        if solve(None, rel_tol=tol, max_iter=k, want_x=False)[2] <= tol:
            return x, k
    return x, hi


def test_half_the_iterations_of_block_jacobi_on_ball_on_mat(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_on_mat()
    assemble(ctx, m, info["dHat"], 1e8)
    for tol in (1e-6, 1e-10):
        x_bj, it_bj = first_iteration_below(ctx.solve_pcg, tol)
        x_ml, it_ml = first_iteration_below(ctx.solve_pcg_multilevel, tol)
        assert rel(x_ml, x_bj) <= 1e3 * tol
        assert 2 * it_ml <= it_bj, (tol, it_ml, it_bj)
