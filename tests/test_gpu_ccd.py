"""GPU parity of the CCD step bound (through the C ABI): BIT-EXACT against the oracle (BASELINE.json north_star)."""

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu


def two_body(seed, n=4, gap=0.01, speed=0.05):
    V1, T1 = M.grid_tets(n, n, n, h=1.0 / n)
    V2, T2 = M.grid_tets(n, n, n, h=1.0 / n, origin=(0.11, 0.07, 1.0 + gap))
    m = M.merge_meshes([(V1, T1), (V2, T2)])
    rng = np.random.default_rng(seed)
    m.V = m.V_rest + 0.1 * gap * rng.standard_normal(m.V_rest.shape)
    p = np.zeros((m.nV, 3))
    upper = m.V_rest[:, 2] > 1.0
    p[upper, 2] = -speed
    p[~upper, 2] = 0.3 * speed
    p += 0.02 * speed * rng.standard_normal(p.shape)
    return m, p.ravel()


def test_ti_error_matches_oracle():
    rng = np.random.default_rng(0)
    V = rng.standard_normal((50, 3)) * 3 + 1
    p = rng.standard_normal(150)
    Vs = np.ascontiguousarray(V.T).ravel()
    for pp in (None, p):
        a, b = L.Context.ti_error(Vs, 50, pp)
        c, d = orc.ti_error(Vs, 50, pp)
        assert np.array_equal(a, c) and np.array_equal(b, d)


@pytest.mark.parametrize("seed,speed", [(1, 0.05), (2, 0.5), (3, 0.004)])
def test_partial_ccd_bit_exact(shared_ctx, seed, speed):
    m, p = two_body(seed, speed=speed)
    dHat = 0.02 ** 2
    load_scene(shared_ctx, m)
    mm, pa, pe, cand = shared_ctx.constraint_set(dHat, 1)
    s = orc.Surf(m)
    _, _, _, cand_r = s.constraint_set(dHat)
    assert np.array_equal(cand, cand_r) and len(cand) > 0
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, p)
    for alpha0 in (1.0, 0.37):
        a_ref, z = orc.ccd_partial(s, p, cand_r, 1e-6, evf, eee, alpha0, nthreads=8)
        a = shared_ctx.ccd_partial(p, 1e-6, evf, eee, alpha0)
        assert scalar_bits(a) == scalar_bits(a_ref), (a, a_ref)
        assert shared_ctx.ccd_stats()[2] == 0  # no conservative early-outs were taken
    a_sep = shared_ctx.ccd_partial(-p, 1e-6, evf, eee, 1.0)  # separating motion: step unchanged
    assert a_sep == 1.0 == orc.ccd_partial(s, -p, cand_r, 1e-6, evf, eee, 1.0)[0]


@pytest.mark.parametrize("seed,speed", [(4, 0.05), (5, 0.6)])
def test_full_ccd_bit_exact(shared_ctx, seed, speed):
    m, p = two_body(seed, n=3, speed=speed)
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, p)
    h = m.avgEdgeLen / 3
    g, a_grid_ref = orc.grid_swept(s, p, 1.0, h)
    a_grid = shared_ctx.hash_build_swept(p, 1.0, h)
    assert scalar_bits(a_grid) == scalar_bits(a_grid_ref)
    a_ref, z, npairs = orc.ccd_full(s, p, g, a_grid_ref, 1e-6, evf, eee, a_grid_ref, nthreads=8)
    a, ncand = shared_ctx.ccd_full(1e-6, evf, eee, a_grid)
    assert ncand == npairs  # the candidate SET is the reference hash's (voxel-range overlap + swept bbox test)
    assert scalar_bits(a) == scalar_bits(a_ref), (a, a_ref)
    assert 0 < a < a_grid
    assert shared_ctx.ccd_stats()[2] == 0


def test_zero_distance_returns_zero_step(shared_ctx):
    m, p = two_body(7, n=2)
    # put a vertex of the upper body exactly onto a face of the lower one
    up = np.nonzero(m.V_rest[:, 2] > 1.0)[0]
    v = up[np.argmin(m.V[up, 2])]
    m.V[v] = [0.3, 0.2, 1.0]  # inside a lower triangle, away from its edges (on an edge, pairs at distance ~1e-17 make the
    # no_zero_toi refinement of Tight-Inclusion spin forever -- in the library as well)
    m.V[m.V_rest[:, 2] <= 1.0] = m.V_rest[m.V_rest[:, 2] <= 1.0]
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, p)
    h = m.avgEdgeLen / 3
    g, ag = orc.grid_swept(s, p, 1.0, h)
    a_ref, z, _ = orc.ccd_full(s, p, g, ag, 1e-6, evf, eee, ag, nthreads=8)
    assert z == 1 and a_ref == 0.0
    shared_ctx.hash_build_swept(p, 1.0, h)
    a, _ = shared_ctx.ccd_full(1e-6, evf, eee, ag)
    assert a == 0.0


def test_ball_pile_ccd_bit_exact(shared_ctx):
    """BASELINE ball-pile workload at a size the brute-force oracle can sweep (4 balls)."""
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    p = info["p"]
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, p)
    mm, pa, pe, cand = shared_ctx.constraint_set(info["dHat"], 1)
    a_part_ref, _ = orc.ccd_partial(s, p, cand, 1e-6, evf, eee, 1.0, nthreads=8)
    a_part = shared_ctx.ccd_partial(p, 1e-6, evf, eee, 1.0)
    assert scalar_bits(a_part) == scalar_bits(a_part_ref)
    h = m.avgEdgeLen / 3
    g, ag_ref = orc.grid_swept(s, p, a_part_ref, h)
    ag = shared_ctx.hash_build_swept(p, a_part, h)
    assert scalar_bits(ag) == scalar_bits(ag_ref)
    a_ref, z, npairs = orc.ccd_full(s, p, g, ag_ref, 1e-6, evf, eee, ag_ref, nthreads=8)
    a, ncand = shared_ctx.ccd_full(1e-6, evf, eee, ag)
    assert ncand == npairs and scalar_bits(a) == scalar_bits(a_ref)
    assert shared_ctx.ccd_stats()[2] == 0
    # property: the step is intersection free for the active stencils
    V2 = m.V + 0.999 * a * p.reshape(-1, 3)
    for c in cand[:200]:
        if c[0] < 0:
            assert orc.point_tri_d(V2[[m.SVI[-c[0] - 1]] + list(m.SF[c[1]])]) > 0
        else:
            assert orc.edge_edge_d(V2[list(m.SFEdges[c[0]]) + list(m.SFEdges[c[1]])]) > 0


def _retry_scene():
    """Two point-triangle pairs built so that the `toi < 1e-6 -> rerun with ms = 0, toi *= 0.8` rule of SelfCollisionHandler.cpp:759-781
    matters: pair A (gap 1e-3, fast) hits at 1.0198e-6 (no rerun); pair B (gap 4e-6) first reports 2^-20 < 1e-6, its rerun with ms = 0
    finds 1.25 * 2^-20 = 1.19e-6 and reports 0.8 x that = 2^-20 = 9.54e-7 -- BELOW A's impact although the rerun's box starts ABOVE it."""
    def tri_tet(o):
        return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.3, 0.3, -1.0]]) + o, np.array([[0, 2, 1, 3]])

    def pt_tet(o, h):
        return np.array([[0.3, 0.3, h], [1.3, 0.3, h + 1], [0.3, 1.3, h + 1], [-0.7, -0.7, h + 1.2]]) + o, np.array([[0, 1, 2, 3]])

    d = 4e-6
    m = M.merge_meshes([tri_tet(np.zeros(3)), pt_tet(np.zeros(3), 1e-3), tri_tet(np.array([5.0, 0, 0])), pt_tet(np.array([5.0, 0, 0]), d)])
    p = np.zeros((m.nV, 3))
    p[4:8, 2] = -(1e-3 - 1e-6) / 1.02e-6
    p[12:16, 2] = -d / 1.3e-6
    sv = lambda v: int(np.nonzero(m.SVI == v)[0][0])
    sf = lambda vs: next(k for k, f in enumerate(m.SF) if set(f) == set(vs))
    candA = (-sv(4) - 1, sf([0, 1, 2]))
    candB = (-sv(12) - 1, sf([8, 9, 10]))
    return m, p.ravel(), np.array([candA], dtype=np.int32), np.array([candB], dtype=np.int32)


def test_ms0_retry_is_not_pruned_by_a_competing_impact(shared_ctx):
    """ADVICE r1: the running-minimum pruning must not cut the ms = 0 rerun, whose result is rescaled by 0.8 afterwards.  Which pair reports
    first is a race on the device, so the test seeds the running minimum with pair A's impact (ipcgpu_ccd_debug_seed_bound) and runs pair B
    alone: with the rerun pruned B would report nothing and the step would stay at A's 1.0198e-6; the oracle (no pruning) says 2^-20."""
    m, p, candA, candB = _retry_scene()
    load_scene(shared_ctx, m)
    s = orc.Surf(m)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    mm0 = np.empty((0, 4), dtype=np.int32)
    pe0 = np.empty((0, 2), dtype=np.int32)
    a_A, _ = orc.ccd_partial(s, p, candA, 1e-6, evf, eee, 1.0, 1)
    a_B, _ = orc.ccd_partial(s, p, candB, 1e-6, evf, eee, 1.0, 1)
    a_AB, _ = orc.ccd_partial(s, p, np.concatenate([candA, candB]), 1e-6, evf, eee, 1.0, 1)
    assert a_B == 2.0 ** -20 and a_A > a_B and a_AB == a_B and 1.25 * a_B > a_A  # the scenario is the intended one
    shared_ctx.set_constraint_set(mm0, mm0, pe0, candB)
    try:
        shared_ctx.ccd_debug_seed_bound(a_A)  # "pair A has already reported"
        a = shared_ctx.ccd_partial(p, 1e-6, evf, eee, 1.0)
    finally:
        shared_ctx.ccd_debug_seed_bound(-1.0)
    assert scalar_bits(a) == scalar_bits(a_AB), (a, a_AB)
    # and without the hook, both pairs in one list, whatever the race
    shared_ctx.set_constraint_set(mm0, mm0, pe0, np.concatenate([candA, candB]))
    assert scalar_bits(shared_ctx.ccd_partial(p, 1e-6, evf, eee, 1.0)) == scalar_bits(a_AB)
