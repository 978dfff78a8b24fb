"""The AMG solve inside a graph at BASELINE.json's full size: C5, the 1M-tet pile bench.py times, at the state and right-hand side of
tests/test_gpu_amg_fullsize.py.  An unreserved eager solve, a reserved eager solve and a replayed solve-only graph give the same bits,
iterations, residual and hierarchy, and the reservation's set-up is not cut."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gpu_common import load_scene, own_context, same_bits
from ipc_b200 import lib as L  # noqa: E402

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2


class _Args:
    tets, res, scene = 1_000_000, 10, "c5"


def test_c5_captured_amg_solve_equals_the_unreserved_one():
    import bench
    m, info = bench.build_scene(_Args())
    dHat, kappa, n = info["dHat"], bench.KAPPA, 3 * m.nV
    with own_context() as ctx:  # (a context of its own: the reservation does not reach the shared one)
        load_scene(ctx, m)
        ctx.set_canonical_order(0)
        ctx.enable_device_pattern(1)
        xt = m.V.copy()
        xt[:, 2] -= 9.81 * DT2
        ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        ctx.inertia_gradient(1, None)
        x0, it0, res0 = ctx.solve_pcg_amg(None, 1e-6, 10000, adopt=True)
        h0 = ctx.amg_info()
        h0.pop("bytes")
        assert res0 <= 1e-6 and len(h0["rows"]) >= 3
        ctx.amg_reserve(1.5)
        x1, it1, res1 = ctx.solve_pcg_amg(None, 1e-6, 10000, adopt=True)
        h1 = ctx.amg_info()
        h1.pop("bytes")
        assert same_bits(x1, x0) and it1 == it0 and same_bits(res1, res0) and h1 == h0
        ctx.capture_begin()
        try:
            ctx.solve_pcg_amg(None, 1e-6, 10000, want_x=False, adopt=True, deferred=True)
        finally:
            gid = ctx.capture_end()
        ctx.graph_launch(gid)
        r = ctx.solve_info()
        p = ctx.download(L.BUF_SEARCH_DIR, n)
        h2 = ctx.amg_info()
        h2.pop("bytes")
        assert r.status == 0 and same_bits(p, x0) and r.iterations == it0 and same_bits(r.rel_residual, res0) and h2 == h0
        assert ctx.amg_capacity_info()[0] == -1
        ctx.graph_destroy(gid)
