"""GPU parity (through the C ABI) of the elastic path against the CPU oracle.
Bars (BASELINE.json north_star): energy / gradient within 1e-10 relative; Hessian held to the same bar."""
import json
import os

import numpy as np
import pytest

import oracle as orc
from gpu_common import rel, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

pytestmark = pytest.mark.gpu
RTOL = 1e-10


def make(et, n=(6, 6, 5), seed=1, inverted=False, dbc=False):
    V, T = M.grid_tets(*n)
    m = M.Mesh(V, T, energy=et)
    M.deform(m, seed, twist=0.7, amp=0.03, noise=0.04, require_positive=True)
    rng = np.random.default_rng(seed)
    if inverted:  # FCR tolerates inverted elements (FixedCoRotEnergy.cpp:173-176)
        m.V[rng.integers(0, m.nV, max(2, m.nV // 100))] += 0.6 * m.avgEdgeLen * rng.standard_normal((max(2, m.nV // 100), 3))
    if dbc:
        m.dbc[rng.integers(0, m.nV, 6)] = 1
        m.dbc[rng.integers(0, m.nV, 4)] = 2
    return m


def load_with_csr(ctx, m, base=1):
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ia, ja = m.csr_pattern(index_base=base)
    ctx.set_csr(ia, ja, base)
    ctx.set_state(m.V_soa)
    return ia, ja


@pytest.mark.parametrize("et", [0, 1])
@pytest.mark.parametrize("inverted", [False, True])
def test_energy_gradient_hessian_parity(shared_ctx, et, inverted):
    if et == 0 and inverted:
        pytest.skip("NeoHookean is undefined for inverted tets (needElemInvSafeGuard, NeoHookeanEnergy.cpp:173-176)")
    m = make(et, inverted=inverted, dbc=True)
    ia, ja = load_with_csr(shared_ctx, m)
    coef = 0.025 ** 2
    o = orc.Elastic(m)
    E_ref, per_ref = o.energy(coef)
    E = shared_ctx.elastic_energy(coef)
    assert abs(E - E_ref) <= RTOL * abs(E_ref)
    per = shared_ctx.download(L.BUF_ENERGY_PER_TET, m.nT)
    assert np.allclose(per, per_ref, rtol=RTOL, atol=RTOL * abs(per_ref).max())
    for projectDBC in (0, 1):
        g = shared_ctx.elastic_gradient(coef, 1, projectDBC)
        assert rel(g, o.gradient(coef, projectDBC)) <= RTOL
    for projectSPD in (1, 0):
        H_ref = o.hessian_blocks(coef, projectSPD)
        a = np.zeros(ja.size)
        shared_ctx.elastic_hessian(coef, 1, projectSPD, 1, a)
        h78 = L.untile_hessians(shared_ctx.download(L.BUF_TET_HESSIANS, 78 * 64 * ((m.nT + 63) // 64)), m.nT)
        worst = 0.0
        for t in range(m.nT):
            worst = max(worst, np.abs(orc.blocks78_to_dense(h78[t], m.T[t]) - H_ref[t]).max() / np.abs(H_ref[t]).max())
        assert worst <= 1e-9, worst
        a_ref = o.hessian_csr(coef, ia, ja, 1, projectSPD, 1)
        assert rel(a, a_ref) <= RTOL
        assert np.abs(a - a_ref).max() <= 1e-9 * np.abs(a_ref).max()


def test_hessian_accumulates_and_index_base0(shared_ctx):
    m = make(0, n=(4, 3, 3), seed=4)
    ia, ja = load_with_csr(shared_ctx, m, base=0)
    coef = 1.0
    a0 = np.full(ja.size, 0.25)  # addCoeff semantics: prior content is kept (LinSysSolver.hpp:402-410)
    a = a0.copy()
    shared_ctx.elastic_hessian(coef, 1, 1, 0, a)
    a_ref = orc.Elastic(m).hessian_csr(coef, ia, ja, 0, 1, 0, a=a0.copy())
    assert rel(a, a_ref) <= RTOL


def test_fused_grad_hess_with_mass(shared_ctx):
    m = make(1, n=(5, 4, 4), seed=7, dbc=True)
    ia, ja = load_with_csr(shared_ctx, m)
    coef = 0.025 ** 2
    g, a = np.empty(3 * m.nV), np.empty(ja.size)
    shared_ctx.elastic_grad_hess(coef, 1, 1, 1, g, a)
    o = orc.Elastic(m)
    assert rel(g, o.gradient(coef, 1)) <= RTOL
    a_ref = o.hessian_csr(coef, ia, ja, 1, 1, 1)
    fixed = (m.dbc == 1) | (m.dbc == 2)
    for v in range(m.nV):  # mass on the diagonal of free vertices (Optimizer.cpp:3638-3668)
        if not fixed[v]:
            for r in range(3):
                a_ref[ia[3 * v + r] - 1] += m.mass[v]
    assert rel(a, a_ref) <= RTOL
    # device-resident variant: NULL outputs, then download
    shared_ctx.elastic_grad_hess(coef, 1, 1, 1, None, None)
    assert np.array_equal(shared_ctx.download(L.BUF_CSR_VALUES, ja.size), a)
    assert np.array_equal(shared_ctx.download(L.BUF_GRADIENT, 3 * m.nV), g)


def test_golden_single_tets(shared_ctx):
    """mpmath golden vectors (tests/golden/elastic_golden.json) through the kernels: one tet with F prescribed."""
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "elastic_golden.json")))
    X = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1.0]])
    T = np.array([[0, 1, 2, 3]], dtype=np.int32)
    for case in gold["cases"]:
        et, F = case["energy"], np.array(case["F"])
        m = M.Mesh(X, T, YM=100.0, PR=0.4, energy=et)
        m.V = X @ F.T
        shared_ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, None, None, et)
        shared_ctx.set_state(m.V_soa)
        E = shared_ctx.elastic_energy(1.0)
        assert abs(E - case["psi"] / 6.0) <= 1e-12 * max(1.0, abs(case["psi"]))
        g = shared_ctx.elastic_gradient(1.0, 1, 0).reshape(4, 3)
        P = np.array(case["P"]) / 6.0  # g_{a} = P * grad N_a, grad N_{i+1} = e_i for the unit tet
        g_ref = np.vstack([-P.sum(1), P[:, 0], P[:, 1], P[:, 2]])
        assert np.allclose(g, g_ref, atol=1e-12 * max(1.0, abs(P).max()))


def test_inversion_step_parity(shared_ctx):
    m = make(0, n=(6, 5, 5), seed=9)
    load_with_csr(shared_ctx, m)
    rng = np.random.default_rng(10)
    p = rng.standard_normal(3 * m.nV) * m.avgEdgeLen
    a_ref, per_ref = orc.Elastic(m).inversion_step(p, 0.2, 1.0)
    a = shared_ctx.inversion_step(p, 0.2, 1.0)
    per = shared_ctx.download(L.BUF_INVERSION_STEPS, m.nT)
    assert np.allclose(per, per_ref, rtol=1e-9)
    assert abs(a - a_ref) <= 1e-9 * a_ref
    assert shared_ctx.inversion_step(p * 1e-6, 0.2, 1.0) == 1.0  # no root below the incoming step: unchanged


def test_large_mesh_properties(shared_ctx):
    """Size-independent properties at 100K tets (BASELINE config C2): sum of forces = 0, E(rigid motion) = E, PSD blocks."""
    V, T = M.grid_tets(26, 26, 25)
    m = M.Mesh(V, T, energy=1)
    M.deform(m, 2, twist=1.0, amp=0.02, noise=0.02)
    ia, ja = load_with_csr(shared_ctx, m)
    coef = 0.025 ** 2
    E = shared_ctx.elastic_energy(coef)
    g = shared_ctx.elastic_gradient(coef, 1, 0).reshape(-1, 3)
    assert np.abs(g.sum(0)).max() <= 1e-9 * np.abs(g).max()
    th = 0.7
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1.0]])
    shared_ctx.set_state(np.ascontiguousarray((m.V @ R.T + [0.3, -0.2, 0.5]).T).ravel())
    E2 = shared_ctx.elastic_energy(coef)
    assert abs(E2 - E) <= 1e-10 * abs(E)
    shared_ctx.set_state(m.V_soa)
    a = np.zeros(ja.size)
    shared_ctx.elastic_hessian(coef, 1, 1, 0, a)
    h78 = L.untile_hessians(shared_ctx.download(L.BUF_TET_HESSIANS, 78 * 64 * ((m.nT + 63) // 64)), m.nT)
    rng = np.random.default_rng(0)
    for t in rng.integers(0, m.nT, 200):
        H = orc.blocks78_to_dense(h78[t], m.T[t])
        assert np.linalg.eigvalsh(H).min() >= -1e-9 * np.abs(H).max()
    # oracle spot check on a sample of tets + full CSR parity (the oracle does 100K tets in seconds)
    a_ref = orc.Elastic(m).hessian_csr(coef, ia, ja, 1, 1, 0, nthreads=8)
    assert rel(a, a_ref) <= RTOL


@pytest.mark.parametrize("drop", [1, 2, 3])
def test_partial_tile_odd_tet_count(shared_ctx, drop):
    """The per-tet blocks leave the kernel through TMA bulk stores of (tets in the tile) x 72 bytes; bulk copies move multiples of 16 bytes,
    so a last tile with an ODD tet count needs its size rounded up (round 1 dropped the last entry of the last tet: found on C3, nT % 64 = 3)."""
    V, T = M.grid_tets(3, 3, 3)
    m = M.Mesh(V, T[:-drop], energy=0)
    M.deform(m, 5, twist=0.5, amp=0.03, noise=0.03)
    assert (m.nT % 64) % 2 == drop % 2
    load_with_csr(shared_ctx, m)
    coef = 0.025 ** 2
    shared_ctx.elastic_hessian(coef, 1, 1, 1, None)
    h78 = L.untile_hessians(shared_ctx.download(L.BUF_TET_HESSIANS, 78 * 64 * ((m.nT + 63) // 64)), m.nT)
    H_ref = orc.Elastic(m).hessian_blocks(coef, 1)
    for t in range(m.nT):
        assert np.abs(orc.blocks78_to_dense(h78[t], m.T[t]) - H_ref[t]).max() <= 1e-10 * np.abs(H_ref[t]).max(), t


def test_fused_energy_gradient_hessian_equals_the_separate_calls(shared_ctx):
    """ipcgpu_elastic_energy_grad_hess: the energy as a by-product of the gradient/Hessian kernel (one SVD per tet) equals
    ipcgpu_elastic_energy and the oracle; gradient and CSR values are those of ipcgpu_elastic_grad_hess."""
    for et in (0, 1):
        V, T = M.grid_tets(9, 8, 7)
        m = M.Mesh(V, T, energy=et)
        M.deform(m, 3)
        ctx = shared_ctx
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ia, ja = m.csr_pattern(1)
        ctx.set_csr(ia, ja, 1)
        ctx.set_state(m.V_soa)
        coef = 0.025 ** 2
        E_sep = ctx.elastic_energy(coef)
        g0, a0 = np.empty(3 * m.nV), np.empty(ja.size)
        ctx.elastic_grad_hess(coef, 1, 1, 1, g0, a0)
        g1, a1 = np.empty(3 * m.nV), np.empty(ja.size)
        E_fused = ctx.elastic_energy_grad_hess(coef, 1, 1, 1, g1, a1, want_energy=True)
        E_ref, _ = orc.Elastic(m).energy(coef)
        assert abs(E_fused - E_sep) <= 1e-13 * abs(E_sep) and abs(E_fused - E_ref) <= 1e-10 * abs(E_ref)
        assert np.array_equal(g0, g1) and np.array_equal(a0, a1)
        # deferred form: the energy arrives with the fetch
        ctx.elastic_energy_grad_hess(coef, 1, 1, 1, None, None)
        assert abs(ctx.fetch_iteration().energy_elastic - E_fused) <= 1e-15 * abs(E_fused)
