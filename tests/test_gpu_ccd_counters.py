"""GPU: the box counters of the Tight-Inclusion passes (ipcgpu_ccd_stats_ex: boxes_thread_pass, boxes_warp_pass) are sums the passes
keep per lane / per warp and add to the context's counters when a warp leaves.  Pruning against the running minimum makes the counts depend
on the order in which pairs report, so the running minimum is seeded with the iteration's own step bound (ipcgpu_ccd_debug_seed_bound):
every search then prunes against the same value, and the counts are a property of the inputs.  Two eager iterations and a replay of the
captured iteration must count the same boxes, at the default thread budget and at budget 0 (every search that goes past its root box is
handed to the warp pass)."""
import os
import sys

import pytest

from gpu_common import load_scene, scalar_bits, shared_ctx
from ipc_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


class _Args:
    tets, res = 1_000_000, 10

    def __init__(self, scene):
        self.scene = scene


@pytest.mark.parametrize("budget", [-1, 0], ids=["default_budget", "budget0"])
@pytest.mark.parametrize("scene", ["c5", "pile"])
def test_box_counts_are_identical_eager_and_replayed(shared_ctx, scene, budget):
    import bench
    ctx = shared_ctx
    m, info = bench.build_scene(_Args(scene))
    dHat, p, tol = info["dHat"], info["p"], bench.TI_TOL
    h = m.avgEdgeLen / 3.0
    load_scene(ctx, m)
    ctx.set_canonical_order(0)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    ctx.constraint_set(dHat, 1)
    ctx.set_search_dir(p)

    def iteration():  # the step-bound chain of bench.py's iteration, device-resident
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(tol, evf, eee, None)

    def counts():
        it = ctx.fetch_iteration()
        _, survivors, warnings = ctx.ccd_stats()
        deferred, boxes_thread, boxes_warp = ctx.ccd_stats_ex()
        return dict(alpha=scalar_bits(it.alpha), survivors=survivors, warnings=warnings, deferred=deferred, boxes_thread=boxes_thread, boxes_warp=boxes_warp)

    ctx.ccd_debug_thread_budget(budget)
    try:
        iteration()
        alpha = ctx.fetch_iteration().alpha
        ctx.ccd_debug_seed_bound(alpha)
        runs = []
        for _ in range(2):
            iteration()
            runs.append(counts())
        ctx.capture_begin()
        iteration()
        gid = ctx.capture_end()
        ctx.graph_launch(gid)
        runs.append(counts())
        ctx.graph_destroy(gid)
    finally:
        ctx.ccd_debug_seed_bound(-1.0)
        ctx.ccd_debug_thread_budget(-1)
        ctx.set_canonical_order(1)
    print("COUNTS", scene, budget, runs[0])
    assert runs[0]["alpha"] == scalar_bits(alpha), runs
    assert runs[0] == runs[1] == runs[2], runs
    # a handed-on search was counted by the thread pass at its first level (at least its root box) before the warp pass took it
    assert runs[0]["survivors"] > 0 and runs[0]["boxes_thread"] >= runs[0]["deferred"] > 0 and runs[0]["boxes_warp"] > 0, runs
