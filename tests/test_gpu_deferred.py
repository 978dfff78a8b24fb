"""The device-resident iteration (every stage enqueued with NULL outputs, one ipcgpu_fetch_iteration) must give exactly what the
synchronous calls give: same energies, same gradient / CSR values, bit-identical step after every bound -- and both match the oracle."""

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, rel, scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("canonical", [1, 0])
def test_deferred_iteration_equals_synchronous_calls(shared_ctx, canonical):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat, p, kappa, dt2, tol = info["dHat"], info["p"], 1e8, 0.025 ** 2, 1e-6
    h = m.avgEdgeLen / 3
    load_scene(ctx, m)
    ctx.set_canonical_order(canonical)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    mm, pa, pe, cand = ctx.constraint_set(dHat, 1)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    ctx.set_csr(ia, ja, 1)
    # synchronous reference run
    E_el, E_b = ctx.elastic_energy(dt2), ctx.barrier_energy(dHat, kappa)
    g, a = np.empty(3 * m.nV), np.empty(ja.size)
    ctx.elastic_grad_hess(dt2, 1, 1, 1, g, a)
    ctx.barrier_gradient(dHat, kappa, g)
    ctx.barrier_hessian(dHat, kappa, 1, a)
    a0 = ctx.inversion_step(p, 0.2, 1.0)
    a1 = ctx.ccd_partial(None, tol, evf, eee, a0)
    a2 = ctx.hash_build_swept(None, a1, h)
    a3, ncand = ctx.ccd_full(tol, evf, eee, a2)
    # the same through the device-resident chain
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.elastic_energy(dt2, 1, want=False)
    ctx.barrier_energy(dHat, kappa, want=False)
    ctx.elastic_grad_hess(dt2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.step_bound_set(1.0)
    ctx.inversion_step(None, 0.2, None)
    ctx.ccd_partial(None, tol, evf, eee, None)
    ctx.hash_build_swept(None, None, h)
    ctx.ccd_full(tol, evf, eee, None)
    it = ctx.fetch_iteration()
    assert it.status == 0 and it.ti_warnings == 0
    assert (it.n_active, it.n_mollified, it.n_candidates) == (len(mm), len(pa), len(cand)) == ctx.constraint_set_sizes()
    assert abs(it.energy_elastic - E_el) <= 1e-14 * abs(E_el) and abs(it.energy_barrier - E_b) <= 1e-12 * abs(E_b)
    assert [scalar_bits(x) for x in (it.alpha_inversion, it.alpha_partial_ccd, it.alpha_swept_grid, it.alpha_full_ccd, it.alpha)] == [scalar_bits(x) for x in (a0, a1, a2, a3, a3)]
    assert it.n_full_ccd_candidates == ncand
    g2, a_2 = ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, ja.size)
    assert rel(g2, g) <= 1e-13 and rel(a_2, a) <= 1e-13  # (atomics: summation order differs run to run)
    # and the oracle
    s, o = orc.Surf(m), orc.Elastic(m)
    al, _ = o.inversion_step(p, 0.2, 1.0)
    al, _ = orc.ccd_partial(s, p, cand, tol, evf, eee, al, 8)
    gr, ag = orc.grid_swept(s, p, al, h)
    al, _, _ = orc.ccd_full(s, p, gr, ag, tol, evf, eee, ag, 8)
    assert scalar_bits(it.alpha) == scalar_bits(al)


def test_deferred_errors_surface_at_fetch(shared_ctx):
    """d <= 0 in the barrier energy (the reference exits there) is reported by the fetch when nothing was read back in between"""
    ctx = shared_ctx
    m, info = scenes.ball_pile(2, res=4, seed=1, height=2)
    load_scene(ctx, m)
    ctx.set_canonical_order(1)
    bad = np.array([[-1, 0, -1, -1]], dtype=np.int32)  # a vertex against itself: d = 0
    ctx.set_constraint_set(bad, bad[:0], np.empty((0, 2), dtype=np.int32))
    ctx.barrier_energy(info["dHat"], 1e3, want=False)
    with pytest.raises(L.IpcGpuError, match="NONPOSITIVE"):
        ctx.fetch_iteration()
    assert ctx.fetch_iteration().status == 0  # flags are per fetch


def test_captured_graph_replays_the_iteration_at_new_states(shared_ctx):
    """ipcgpu_capture_begin/_end: the device-resident iteration captured ONCE into a CUDA graph and replayed at other positions and another
    search direction gives bit-identical step bounds and the same energies / gradient / CSR values as the eager calls at that state.
    A graph is refused after a call that may reallocate or re-partition."""
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat, p, kappa, dt2, tol = info["dHat"], info["p"], 1e8, 0.025 ** 2, 1e-6
    h = m.avgEdgeLen / 3
    load_scene(ctx, m)
    ctx.set_canonical_order(0)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    mm, pa, pe, cand = ctx.constraint_set(dHat, 1)
    # second state: half of the feasible step along p (closer contact, another active set); pattern wide enough for both states
    s1, o1 = orc.Surf(m), orc.Elastic(m)
    al1, _ = o1.inversion_step(p, 0.2, 1.0)
    al1, _ = orc.ccd_partial(s1, p, cand, tol, evf, eee, al1, 8)
    gr1, ag1 = orc.grid_swept(s1, p, al1, h)
    al1, _, _ = orc.ccd_full(s1, p, gr1, ag1, tol, evf, eee, ag1, 8)
    V2 = m.V + 0.5 * al1 * p.reshape(-1, 3)
    s2 = orc.Surf(m, V=V2)
    mm2, pa2, pe2, _ = s2.constraint_set(dHat, nthreads=8)
    pairs = np.concatenate([contact_pattern_pairs(m, mm, pa, pe), contact_pattern_pairs(m, mm2, pa2, pe2)])
    ia, ja = m.csr_pattern(1, extra_pairs=pairs)
    ctx.set_csr(ia, ja, 1)
    ctx.set_search_dir(p)

    def enqueue():
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.elastic_energy(dt2, 1, want=False)
        ctx.barrier_energy(dHat, kappa, want=False)
        ctx.elastic_grad_hess(dt2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(tol, evf, eee, None)

    def result():
        it = ctx.fetch_iteration()
        return it, ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, ja.size)

    enqueue()  # eager warm-up (lazy allocations)
    it0, g0, a0 = result()
    n_before = ctx.launch_count()
    ctx.capture_begin()
    enqueue()
    gid = ctx.capture_end()
    assert ctx.launch_count() == n_before  # nothing ran during the capture
    ctx.graph_launch(gid)
    it1, g1, a1 = result()
    assert ctx.launch_count() - n_before >= 40
    assert [scalar_bits(x) for x in (it1.alpha_inversion, it1.alpha_partial_ccd, it1.alpha_swept_grid, it1.alpha_full_ccd)] == \
        [scalar_bits(x) for x in (it0.alpha_inversion, it0.alpha_partial_ccd, it0.alpha_swept_grid, it0.alpha_full_ccd)]
    assert (it1.n_active, it1.n_mollified, it1.n_candidates) == (it0.n_active, it0.n_mollified, it0.n_candidates)
    assert rel(g1, g0) <= 1e-13 and rel(a1, a0) <= 1e-13 and abs(it1.energy_barrier - it0.energy_barrier) <= 1e-12 * abs(it0.energy_barrier)
    # another state and another search direction through the SAME graph
    p2 = 0.5 * p
    ctx.set_state(np.ascontiguousarray(V2.T).ravel())
    ctx.set_search_dir(p2)
    ctx.graph_launch(gid)
    it2, g2, a2 = result()
    enqueue()
    it3, g3, a3 = result()
    assert it2.n_active == len(mm2) == it3.n_active and len(mm2) != len(mm)
    assert [scalar_bits(x) for x in (it2.alpha_inversion, it2.alpha_partial_ccd, it2.alpha_swept_grid, it2.alpha_full_ccd, it2.alpha)] == \
        [scalar_bits(x) for x in (it3.alpha_inversion, it3.alpha_partial_ccd, it3.alpha_swept_grid, it3.alpha_full_ccd, it3.alpha)]
    assert rel(g2, g3) <= 1e-13 and rel(a2, a3) <= 1e-13
    assert abs(it2.energy_elastic - it3.energy_elastic) <= 1e-14 * abs(it3.energy_elastic)
    # ... and the oracle at that state
    o2 = orc.Elastic(m, V=V2)
    al, _ = o2.inversion_step(p2, 0.2, 1.0)
    _, _, _, cand2 = s2.constraint_set(dHat, nthreads=8)
    al, _ = orc.ccd_partial(s2, p2, cand2, tol, evf, eee, al, 8)
    gr, ag = orc.grid_swept(s2, p2, al, h)
    al, _, _ = orc.ccd_full(s2, p2, gr, ag, tol, evf, eee, ag, 8)
    assert scalar_bits(it2.alpha) == scalar_bits(al)
    # a call that may reallocate invalidates the graph
    ctx.set_csr(ia, ja, 1)
    with pytest.raises(L.IpcGpuError, match="capture it again"):
        ctx.graph_launch(gid)
    ctx.graph_destroy(gid)
    ctx.set_state(m.V_soa)


def test_async_download_on_the_copy_stream_eager_and_captured(shared_ctx):
    """ipcgpu_download_range_async: the copy is forked behind what produced the buffer and joined by the fetch -- also as part of a graph"""
    ctx = shared_ctx
    m, info = scenes.ball_pile(2, res=6, seed=1, height=2)
    dt2 = 0.025 ** 2
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ia, ja = m.csr_pattern(1)
    ctx.set_csr(ia, ja, 1)
    ctx.set_state(m.V_soa)
    hg, ha = L.PinnedArray(3 * m.nV), L.PinnedArray(ja.size)
    g_ref, a_ref = np.empty(3 * m.nV), np.empty(ja.size)
    ctx.elastic_grad_hess(dt2, 1, 1, 1, g_ref, a_ref)

    def enqueue():
        ctx.elastic_energy_grad_hess(dt2, 1, 1, 1, None, None)
        ctx.download_range_async(L.BUF_GRADIENT, 0, hg.array)
        ctx.download_range_async(L.BUF_CSR_VALUES, 100, ha.array[100:])
        ctx.elastic_energy(dt2, 1, want=False)  # later work on the main stream next to the copies

    hg.array[:] = 0; ha.array[:] = 0
    enqueue()
    ctx.fetch_iteration()
    assert np.array_equal(hg.array, g_ref) and np.array_equal(ha.array[100:], a_ref[100:]) and not ha.array[:100].any()
    ctx.capture_begin()
    enqueue()
    gid = ctx.capture_end()
    V2 = m.V * 1.01
    ctx.set_state(np.ascontiguousarray(V2.T).ravel())
    hg.array[:] = 0; ha.array[:] = 0
    ctx.graph_launch(gid)
    ctx.fetch_iteration()
    g2, a2 = np.empty(3 * m.nV), np.empty(ja.size)
    ctx.elastic_grad_hess(dt2, 1, 1, 1, g2, a2)
    assert np.array_equal(hg.array, g2) and np.array_equal(ha.array[100:], a2[100:]) and not np.array_equal(g2, g_ref)
    ctx.graph_destroy(gid)
    hg.free(); ha.free()
