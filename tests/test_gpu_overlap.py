"""The derivative chain of the device-resident iteration (elastic gradient/Hessian and its CSR assembly, barrier gradient, barrier Hessian
scatter) runs on a low-priority stream next to the step-bound chain; with the stage timers on, both run one after the other on one stream.
Either way the iteration gives a bit-identical elastic energy and step bounds, and gradient / CSR values that differ from a serial run by
no more than two serial runs differ (the atomic sums of the barrier terms).  A call outside both chains waits for the derivative chain."""

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, rel, scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs

pytestmark = pytest.mark.gpu

KAPPA, DT2, TOL = 1e8, 0.025 ** 2, 1e-6


def pile_with_contacts(ctx):
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    load_scene(ctx, m)
    mm, pa, pe, _ = ctx.constraint_set(info["dHat"], 1)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    ctx.set_csr(ia, ja, 1)
    ctx.set_canonical_order(0)
    ctx.set_search_dir(info["p"])
    return m, info, ia, ja


def test_concurrent_chains_equal_the_serial_order(shared_ctx):
    ctx = shared_ctx
    m, info, ia, ja = pile_with_contacts(ctx)
    dHat, h = info["dHat"], m.avgEdgeLen / 3
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)

    def enqueue():  # bench.py's iteration, in its order
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.barrier_energy(dHat, KAPPA, want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, KAPPA, None)
        ctx.barrier_hessian(dHat, KAPPA, 1, None)
        ctx.allreduce_grad_hess(1, 0)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, TOL, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(TOL, evf, eee, None)

    def result():
        it = ctx.fetch_iteration()
        assert it.status == 0 and it.ti_warnings == 0
        return it, ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, ja.size)

    def serial():
        ctx.profile(1)  # stage timers on: one stream
        enqueue()
        r = result()
        ctx.profile(0)
        return r

    enqueue()  # eager warm-up (lazy allocations)
    result()
    s1, s2 = serial(), serial()
    enqueue()
    eager = result()
    ctx.capture_begin()
    enqueue()
    gid = ctx.capture_end()
    n_high, n_low = ctx.graph_kernel_priorities(gid)
    # low: per-tet kernel, energy reduce + store, gather, assembly, diagonal, barrier gradient, pair-Hessian build + projection, scatter
    assert n_high > 0 and n_low >= 10, (n_high, n_low)
    ctx.graph_launch(gid)
    replay = result()
    ctx.graph_destroy(gid)
    # the same iteration handing its gradient and CSR values to the host: the derivative chain takes the high priority
    hg, ha = L.PinnedArray(3 * m.nV), L.PinnedArray(ja.size)
    ctx.download_range_async(L.BUF_GRADIENT, 0, hg.array)  # (outside a capture first: creates the copy stream)
    ctx.sync()
    ctx.capture_begin()
    enqueue()
    ctx.download_range_async(L.BUF_GRADIENT, 0, hg.array)
    ctx.download_range_async(L.BUF_CSR_VALUES, 0, ha.array)
    gid = ctx.capture_end()
    assert ctx.graph_kernel_priorities(gid) == (n_low, n_high)
    ctx.graph_launch(gid)
    copied = result()
    assert np.array_equal(hg.array, copied[1]) and np.array_equal(ha.array, copied[2])
    ctx.graph_destroy(gid)
    hg.free(); ha.free()

    def scalars(it):  # (the barrier energy sums the contact lists in the order the atomic appends left them: compared below)
        return [scalar_bits(x) for x in (it.energy_elastic, it.alpha_inversion, it.alpha_partial_ccd, it.alpha_swept_grid, it.alpha_full_ccd, it.alpha)] + \
            [it.n_active, it.n_mollified, it.n_candidates, it.n_full_ccd_candidates]

    g_noise, a_noise = rel(s2[1], s1[1]), rel(s2[2], s1[2])
    assert scalars(s2[0]) == scalars(s1[0])
    for it, g, a in (eager, replay, copied):
        assert scalars(it) == scalars(s1[0])
        assert abs(it.energy_barrier - s1[0].energy_barrier) <= 1e-12 * abs(s1[0].energy_barrier)
        # (the floor: two serial runs can happen to add in the same order; 1e-14 is far below any ordering or race error)
        assert rel(g, s1[1]) <= max(g_noise, 1e-14) and rel(a, s1[2]) <= max(a_noise, 1e-14), (rel(g, s1[1]), g_noise, rel(a, s1[2]), a_noise)


def test_setter_after_the_derivative_chain_waits_for_it(shared_ctx):
    """ipcgpu_set_state right behind ipcgpu_elastic_energy_grad_hess (NULL outputs, no fetch in between) must not move the positions
    under the derivative chain still running on its own stream: E / g / H are those of the old positions, the next call sees the new ones"""
    ctx = shared_ctx
    m, info, ia, ja = pile_with_contacts(ctx)
    V2 = m.V * 1.01
    diag = np.asarray(ia[:-1], dtype=np.int64)[: 3 * m.nV] - 1

    def reference(o):
        a = o.hessian_csr(DT2, ia, ja, 1, 1, 1, nthreads=8)
        a[diag] += np.repeat(m.mass, 3)
        return o.energy(DT2, 8)[0], o.gradient(DT2, 1, 8), a

    for o in (orc.Elastic(m), orc.Elastic(m, V=V2)):
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.set_state(np.ascontiguousarray(V2.T).ravel())
        it = ctx.fetch_iteration()
        g, a = ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, ja.size)
        E_r, g_r, a_r = reference(o)
        assert abs(it.energy_elastic - E_r) <= 1e-10 * abs(E_r) and rel(g, g_r) <= 1e-10 and rel(a, a_r) <= 1e-9, \
            (it.energy_elastic, E_r, rel(g, g_r), rel(a, a_r))
    ctx.set_state(m.V_soa)
