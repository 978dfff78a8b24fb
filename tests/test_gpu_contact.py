"""GPU parity (through the C ABI) of the contact stage: constraint-set build and per-pair barrier E / g / H.
Integer outputs (the sets) must be IDENTICAL to the oracle's canonical sets; reals to 1e-10 relative."""
import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, rel, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import scenes
from stagecheck import sort_rows

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def contact_pairs_for_pattern(m, mm, pa, pe):
    pairs = []
    for r in list(mm) + list(pa):
        vs = [(-r[0] - 1) if r[0] < 0 else r[0]] + [x for x in r[1:] if x >= 0]
        pairs += [(a, b) for a in vs for b in vs if a < b]
    for e in pe:
        if e[0] >= 0:
            vs = list(m.SFEdges[e[0]]) + list(m.SFEdges[e[1]])
            pairs += [(a, b) for a in vs for b in vs if a != b]
    return pairs


def stacked_cubes(gap, n=3, seed=0, jitter=0.1, shift=(0.13, 0.07)):
    V1, T1 = M.grid_tets(n, n, n, h=1.0 / n)
    V2, T2 = M.grid_tets(n, n, n, h=1.0 / n, origin=(shift[0], shift[1], 1.0 + gap))
    m = M.merge_meshes([(V1, T1), (V2, T2)])
    rng = np.random.default_rng(seed)
    m.V = m.V_rest + jitter * gap * rng.standard_normal(m.V_rest.shape)
    return m


@pytest.mark.parametrize("case", ["offset", "aligned_parallel", "dbc"])
def test_constraint_set_identical_to_oracle(shared_ctx, case):
    if case == "offset":
        m = stacked_cubes(0.01, n=3, seed=1)
    elif case == "aligned_parallel":  # exactly parallel facing edges -> mollified set (sentinel encodings)
        m = stacked_cubes(0.01, n=2, seed=2, jitter=0.0, shift=(0.0, 0.0))
    else:
        m = stacked_cubes(0.012, n=3, seed=3)
        m.dbc[m.V_rest[:, 2] > 1.0] = 1  # the whole upper cube is Dirichlet: pairs inside it are skipped (:2185, :2295)
        m.dbc[:4] = 2
    dHat = 0.02 ** 2
    load_scene(shared_ctx, m)
    mm, pa, pe, cand = shared_ctx.constraint_set(dHat, 1)
    mm_r, pa_r, pe_r, cand_r = orc.Surf(m).constraint_set(dHat)
    assert len(mm_r) > 0
    if case == "aligned_parallel":
        assert len(pa_r) > 0
    assert np.array_equal(mm, mm_r)
    assert np.array_equal(pa, pa_r) and np.array_equal(pe, pe_r)
    assert np.array_equal(cand, cand_r)
    # getPTEE = 0 leaves the candidate list empty, sets unchanged
    mm2, pa2, pe2, cand2 = shared_ctx.constraint_set(dHat, 0)
    assert np.array_equal(mm2, mm_r) and len(cand2) == 0


@pytest.mark.parametrize("case", ["offset", "aligned_parallel"])
def test_barrier_energy_gradient_hessian_parity(shared_ctx, case):
    m = stacked_cubes(0.01, n=3, seed=5) if case == "offset" else stacked_cubes(0.01, n=2, seed=6, jitter=0.02, shift=(0.0, 0.0))
    if case == "offset":
        m.dbc[[1, 7]] = 1
    dHat, kappa = 0.02 ** 2, 1e4
    load_scene(shared_ctx, m)
    mm, pa, pe, _ = shared_ctx.constraint_set(dHat, 0)
    s = orc.Surf(m)
    E_ref, bad = s.barrier_energy(mm, pa, pe, dHat, kappa)
    assert bad == 0
    E = shared_ctx.barrier_energy(dHat, kappa)
    assert abs(E - E_ref) <= RTOL * abs(E_ref)
    g0 = np.linspace(-1, 1, 3 * m.nV)
    g = g0.copy()
    shared_ctx.barrier_gradient(dHat, kappa, g)
    g_ref = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=g0.copy())
    assert rel(g - g0, g_ref - g0) <= RTOL
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pairs_for_pattern(m, mm, pa, pe))
    shared_ctx.set_csr(ia, ja, 1)
    for projectDBC in (1, 0):
        a = np.zeros(ja.size)
        shared_ctx.barrier_hessian(dHat, kappa, projectDBC, a)
        a_ref = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, projectDBC)
        assert np.abs(a - a_ref).max() <= 1e-9 * np.abs(a_ref).max()
        assert rel(a, a_ref) <= 1e-9
    # a pattern without the contact blocks is reported, not silently dropped
    ia0, ja0 = m.csr_pattern(1)
    shared_ctx.set_csr(ia0, ja0, 1)
    with pytest.raises(L.IpcGpuError, match="PATTERN"):
        shared_ctx.barrier_hessian(dHat, kappa, 1, np.zeros(ja0.size))


def test_uploaded_sets_and_nonpositive_distance(shared_ctx):
    m = stacked_cubes(0.01, n=2, seed=8)
    dHat, kappa = 0.02 ** 2, 1e3
    load_scene(shared_ctx, m)
    mm, pa, pe, _ = orc.Surf(m).constraint_set(dHat)
    shared_ctx.set_constraint_set(mm, pa, pe)
    E_ref, _ = orc.Surf(m).barrier_energy(mm, pa, pe, dHat, kappa)
    assert abs(shared_ctx.barrier_energy(dHat, kappa) - E_ref) <= RTOL * abs(E_ref)
    # degenerate pair (a vertex against itself) -> d = 0 -> error code instead of the reference's exit(0)
    bad = np.array([[-1, 0, -1, -1]], dtype=np.int32)
    shared_ctx.set_constraint_set(bad, pa[:0], pe[:0])
    with pytest.raises(L.IpcGpuError, match="NONPOSITIVE"):
        shared_ctx.barrier_energy(dHat, kappa)


def test_ball_pile_sets_match_oracle(shared_ctx):
    """BASELINE 'ball pile' at a size the brute-force oracle finishes in seconds (8 balls, 48K tets)."""
    m, info = scenes.ball_pile(8, res=10, seed=5)
    load_scene(shared_ctx, m)
    mm, pa, pe, cand = shared_ctx.constraint_set(info["dHat"], 1)
    mm_r, pa_r, pe_r, cand_r = orc.Surf(m).constraint_set(info["dHat"], nthreads=8)
    assert len(mm_r) > 0
    assert np.array_equal(mm, mm_r) and np.array_equal(pa, pa_r) and np.array_equal(pe, pe_r) and np.array_equal(cand, cand_r)
    kappa = 1e9
    E_ref, bad = orc.Surf(m).barrier_energy(mm_r, pa_r, pe_r, info["dHat"], kappa)
    assert bad == 0 and abs(shared_ctx.barrier_energy(info["dHat"], kappa) - E_ref) <= RTOL * abs(E_ref)


def padded(m, nV):
    """m with unreferenced vertices appended up to nV: the surface arrays and the tets keep their indices"""
    k = nV - m.nV
    p = M.Mesh.__new__(M.Mesh)
    p.__dict__.update(m.__dict__)
    pad = lambda a, v: np.concatenate([np.asarray(a), np.full((k,) + np.shape(a)[1:], v, dtype=np.asarray(a).dtype)])
    p.V_rest, p.V, p.mass, p.dbc, p.vCoDim = pad(m.V_rest, 0.0), pad(m.V, 0.0), pad(m.mass, 1.0), pad(m.dbc, 0), pad(m.vCoDim, 3)
    p.nV = nV
    return p


def test_duplicate_merge_on_a_huge_mesh(shared_ctx):
    """from nV = 2^21 - 2 on, the PP/PE multiplicities are merged in canonical order instead of through the 64-bit key table: the same
    lists as the small mesh's, bit for bit at levels 1 and 2, as sorted multisets at level 0"""
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    dHat = info["dHat"]
    big = padded(m, (1 << 21) - 2)
    out = {}
    try:
        for level in (1, 2, 0):
            for name, mesh in (("small", m), ("huge", big)):
                load_scene(shared_ctx, mesh)
                shared_ctx.set_canonical_order(level)
                out[name, level] = shared_ctx.constraint_set(dHat, 1)
    finally:
        shared_ctx.set_canonical_order(1)
    mm = out["small", 1][0]
    assert (mm[:, 3] <= -2).any()  # PP / PE entries counted more than once
    for level in (1, 2):
        assert all(np.array_equal(x, y) for x, y in zip(out["huge", level], out["small", level])), level
    s, h = out["small", 0], out["huge", 0]
    assert all(np.array_equal(x, y) for x, y in zip(sort_rows(h[0]) + sort_rows(h[1], h[2]) + sort_rows(h[3]),
                                                    sort_rows(s[0]) + sort_rows(s[1], s[2]) + sort_rows(s[3])))


def test_reference_two_step_gradient_form(shared_ctx):
    """evaluateConstraints (:64-81) -> host maps through b'(d) -> leftMultiplyConstraintJacobianT (:84-148) + augmentParaEEGradient (:2990-3045):
    the reference's own call sequence (Optimizer.cpp:3492-3502) must give what the fused ipcgpu_barrier_gradient and the oracle give."""
    m = stacked_cubes(0.01, n=2, seed=6, jitter=0.02, shift=(0.0, 0.0))  # has mollified (nearly parallel) pairs too
    dHat, kappa = 0.02 ** 2, 1e4
    load_scene(shared_ctx, m)
    mm, pa, pe, _ = shared_ctx.constraint_set(dHat, 0)
    assert len(mm) > 0 and len(pa) > 0
    s = orc.Surf(m)
    val = shared_ctx.evaluate_constraints(len(mm))
    assert np.all(val > 0) and np.all(val < dHat)
    bvals = np.array([orc.barrier(d, dHat) for d in val])  # (b, b', b'')
    mult = np.where((mm[:, 0] < 0) & (mm[:, 3] < 0), -mm[:, 3], 1)
    E_ref, _ = s.barrier_energy(mm, pa[:0], pe[:0], dHat, kappa)
    assert abs(kappa * float((mult * bvals[:, 0]).sum()) - E_ref) <= RTOL * abs(E_ref)
    g0 = np.linspace(-1, 1, 3 * m.nV)
    g = g0.copy()
    shared_ctx.constraint_jacobian_t(bvals[:, 1], kappa, g)
    g_act = s.barrier_gradient(mm, pa[:0], pe[:0], dHat, kappa, g=g0.copy())
    assert rel(g - g0, g_act - g0) <= RTOL
    shared_ctx.para_ee_gradient(dHat, kappa, g)
    g_all = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=g0.copy())
    assert rel(g - g0, g_all - g0) <= RTOL
    fused = g0.copy()
    shared_ctx.barrier_gradient(dHat, kappa, fused)
    assert rel(fused - g0, g_all - g0) <= RTOL
