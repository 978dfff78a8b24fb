"""GPU: the hand-off from the thread-level pass (a thread per pair) to the warp-level pass (a warp per pair) does not change the step
bound.  The box budget of the thread pass decides which searches are handed on; ipcgpu_ccd_debug_thread_budget sets it per context.
At budget 0 every search that does not end at its root box is handed on; at a huge budget only searches that outgrow their level buffer."""
import os

import pytest

import oracle as orc
from gpu_common import load_scene, scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import scenes
from test_gpu_ccd import test_ms0_retry_is_not_pruned_by_a_competing_impact as _ms0_retry_check

pytestmark = pytest.mark.gpu

TOL = 1e-6
BIG = 1 << 40  # no search is handed on for its budget (only for an overflowing level buffer)


def test_c3_step_bounds_do_not_depend_on_the_thread_budget(shared_ctx):
    m, info = scenes.ball_on_mat_c3(nx=200)
    nth = os.cpu_count() or 8
    dHat, p = info["dHat"], info["p"]
    hvox = m.avgEdgeLen / 3.0
    load_scene(shared_ctx, m)
    _, _, _, cand = shared_ctx.constraint_set(dHat, 1)  # (equal to the oracle's set: test_gpu_fullsize)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    a_part_ref, _ = orc.ccd_partial(s, p, cand, TOL, evf, eee, 1.0, nth)
    a_full_ref, _, _ = orc.ccd_full_hashed(s, p, a_part_ref, hvox, TOL, evf, eee, nth)
    runs = {}
    try:
        for budget in (-1, 0, BIG):  # -1: the default
            shared_ctx.ccd_debug_thread_budget(budget)
            r = {}
            for name in ("partial", "full"):
                if name == "partial":
                    a = shared_ctx.ccd_partial(p, TOL, evf, eee, 1.0)
                    ag = shared_ctx.hash_build_swept(p, a, hvox)
                else:
                    a, _ = shared_ctx.ccd_full(TOL, evf, eee, ag)
                _, survivors, warnings = shared_ctx.ccd_stats()
                deferred, _, boxes_warp = shared_ctx.ccd_stats_ex()
                r[name] = dict(alpha=a, survivors=survivors, warnings=warnings, deferred=deferred, boxes_warp=boxes_warp)
            runs[budget] = r
    finally:
        shared_ctx.ccd_debug_thread_budget(-1)
    for budget, r in runs.items():
        for name, ref in (("partial", a_part_ref), ("full", a_full_ref)):
            x = r[name]
            assert scalar_bits(x["alpha"]) == scalar_bits(ref), (budget, name, x, ref)
            assert x["warnings"] == 0, (budget, name, x)
            assert x["survivors"] > 0, (budget, name, x)
    for name in ("partial", "full"):
        x = runs[0][name]
        assert x["deferred"] == x["survivors"] and x["boxes_warp"] > 0, x  # everything went through the hand-off


def test_ms0_retry_is_not_pruned_at_budget_zero(shared_ctx):
    """The rerun with ms = 0 of a handed-on pair runs in the warp-level pass (pair_ccd<32>), unpruned as in the thread pass."""
    shared_ctx.ccd_debug_thread_budget(0)
    try:
        _ms0_retry_check(shared_ctx)
        assert shared_ctx.ccd_stats_ex()[0] == shared_ctx.ccd_stats()[1] > 0
    finally:
        shared_ctx.ccd_debug_thread_budget(-1)
