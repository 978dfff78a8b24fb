"""The swept grid of the full CCD registers every primitive in each cell of K x K x K reference voxels its range touches, with K chosen on
the device from the longest range and from the size of the cell table.  These scenes push K up and make many ranges straddle cell borders:
the candidate set must still be the reference hash's, every pair exactly once, and the step bound bit-equal to the oracle's."""

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu


def fast_vertices():
    """4-ball pile where a few surface vertices move ~100x faster than the rest: after the span rescale they sweep tens of voxels, so the
    longest range (and K) is large and the slow majority straddles the borders of the large cells"""
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    p = info["p"].reshape(-1, 3).copy()
    rng = np.random.default_rng(11)
    fast = rng.choice(np.asarray(m.SVI), 6, replace=False)
    p[fast] = 100.0 * np.abs(p).max() * rng.standard_normal((6, 3))
    return m, p.ravel()


def far_apart():
    """two bodies about to touch and a third one further out on the diagonal: at K = 2 the grid would need ~10^7 cells, so K grows until
    the dense cell table holds it"""
    n, h = 3, 1.0 / 3
    V1, T1 = M.grid_tets(n, n, n, h=h)
    V2, T2 = M.grid_tets(n, n, n, h=h, origin=(0.11, 0.07, 1.01))
    V3, T3 = M.grid_tets(n, n, n, h=h, origin=(60.0, 60.0, 60.0))
    m = M.merge_meshes([(V1, T1), (V2, T2), (V3, T3)])
    rng = np.random.default_rng(3)
    m.V = m.V_rest + 1e-3 * rng.standard_normal(m.V_rest.shape)
    p = np.zeros((m.nV, 3))
    upper = (m.V_rest[:, 2] > 1.0) & (m.V_rest[:, 0] < 30.0)
    p[upper, 2] = -0.05
    p[~upper, 2] = 0.015
    p += 1e-3 * rng.standard_normal(p.shape)
    return m, p.ravel()


@pytest.mark.parametrize("scene", [fast_vertices, far_apart])
def test_swept_grid_candidates_and_step_match_oracle(shared_ctx, scene):
    m, p = scene()
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, p)
    h = m.avgEdgeLen / 3
    g, ag_ref = orc.grid_swept(s, p, 1.0, h)
    ag = shared_ctx.hash_build_swept(p, 1.0, h)
    assert scalar_bits(ag) == scalar_bits(ag_ref)
    a_ref, _, npairs = orc.ccd_full(s, p, g, ag_ref, 1e-6, evf, eee, ag_ref, nthreads=8)
    a, ncand = shared_ctx.ccd_full(1e-6, evf, eee, ag)
    assert npairs > 0
    assert ncand == npairs  # no pair found twice, none missed
    assert scalar_bits(a) == scalar_bits(a_ref), (a, a_ref)
    assert shared_ctx.ccd_stats()[2] == 0
