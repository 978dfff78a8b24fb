"""The float64 restatement of the end-of-step diagnostics (tests/oracle_diagnostics.py) against closed forms: momentum M v of a rigid
translation, angular momentum I w of a rigid rotation in the discrete V x p form, -sum m g.V at rest, and the Fischer-Burmeister limits at
d = 0 and d = dHat."""
import math

import numpy as np

import oracle_diagnostics as od
import oracle_timestep as ot


def cloud(n=200, seed=3):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1.0, 1.0, (n, 3)), rng.uniform(0.5, 2.0, n)


def test_rigid_translation_momentum():
    P = ot.Params(ot.BE, 0.01, gravity=(0.0, 0.0, 0.0))
    X, m = cloud()
    v = np.array([0.3, -1.25, 2.0])
    e, p, _ = od.vertex_terms(X + P.dt * v, X, m, P)
    M = m.sum()
    assert np.allclose(p.sum(0), M * v, rtol=1e-13, atol=0)
    # kinetic energy 1/2 M |v|^2 (no gravity)
    assert math.isclose(math.fsum(e), 0.5 * M * (v @ v), rel_tol=1e-12)


def test_rigid_rotation_angular_momentum():
    """V = R(theta) X about the z axis through the origin, V_prev = X: sum V x p = I_zz omega_eff about z (the discrete form:
    p = m / dt (R X - X), and (R X) x (R X - X) = (R X) x (-X) has z component sin(theta) (x^2 + y^2))"""
    P = ot.Params(ot.BE, 0.02, gravity=(0.0, 0.0, 0.0))
    X, m = cloud(seed=4)
    th = 0.05
    R = np.array([[math.cos(th), -math.sin(th), 0.0], [math.sin(th), math.cos(th), 0.0], [0.0, 0.0, 1.0]])
    V = X @ R.T
    _, p, L = od.vertex_terms(V, X, m, P)
    Izz = float((m * (X[:, 0] ** 2 + X[:, 1] ** 2)).sum())
    Lz = Izz * math.sin(th) / P.dt
    assert math.isclose(L[:, 2].sum(), Lz, rel_tol=1e-12)
    # x and y components of -(m / dt) (R X) x X for a rotation about z
    c, s = math.cos(th), math.sin(th)
    x, y, z = X.T
    Lx = -(m * z * (s * x - (1.0 - c) * y)).sum() / P.dt
    Ly = -(m * z * ((1.0 - c) * x + s * y)).sum() / P.dt
    assert np.allclose(L[:, :2].sum(0), [Lx, Ly], rtol=1e-10, atol=1e-12 * abs(Lz))
    # a rigid rotation carries no net momentum when the cloud's mass centre sits on the axis
    Xc = X - (m[:, None] * X).sum(0) / m.sum()
    _, p0, _ = od.vertex_terms(Xc @ R.T, Xc, m, P)
    assert np.allclose(p0.sum(0), 0.0, atol=1e-12 * np.abs(p0).sum())


def test_state_at_rest_is_potential_energy():
    P = ot.Params(ot.NM, 0.025, gravity=(0.1, -9.81, 0.4))
    X, m = cloud(seed=5)
    e, p, L = od.vertex_terms(X, X, m, P)
    assert not p.any() and not L.any()
    ref = -(m * (X @ P.gravity))
    assert np.allclose(e, ref, rtol=1e-15, atol=1e-15 * np.abs(ref).max())
    out = od.system_energy(np.zeros(0), X, X, m, P, [len(X)], [0])
    assert math.isclose(out["E_v"][0], math.fsum(ref), rel_tol=1e-14)


def test_system_energy_components_partition_the_sums():
    P = ot.Params(ot.BE, 0.01)
    X, m = cloud(seed=6)
    V = X + 0.01 * np.random.default_rng(1).standard_normal(X.shape)
    et = np.random.default_rng(2).uniform(0.0, 1.0, 50)
    ve, te = [1, 1, 120, 200], [0, 10, 10, 50]
    out = od.system_energy(et, V, X, m, P, ve, te)
    whole = od.system_energy(et, V, X, m, P, [200], [50])
    assert out["E_el"][1] == math.fsum(et[:10]) and out["E_el"][2] == 0.0 and out["E_v"][1] == 0.0
    assert math.isclose(math.fsum(out["E_v"]), whole["E_v"][0], rel_tol=1e-14)
    assert np.allclose(out["M"].sum(0), whole["M"][0], rtol=1e-13)


def test_fischer_burmeister_limits():
    dHat, kappa = 1e-4, 1e5
    # d = dHat: g_b = 0, dual = 0, fb = d - |d| = 0
    f, _ = od.fb(np.array([dHat]), dHat, kappa)
    assert f[0] == 0.0
    # d -> 0: dual = -kappa g_b -> +inf and fb = dual + d - sqrt(dual^2 + d^2) -> d
    d = np.array([1e-14, 1e-12])
    f, _ = od.fb(d, dHat, kappa)
    assert np.allclose(f, d, rtol=1e-3)
    # kappa = 0: fb = d - |d| = 0 for every d > 0
    f, _ = od.fb(np.array([1e-8, 5e-5, 2e-4]), dHat, 0.0)
    assert not f.any()
    n, lo, hi, norm, _ = od.summary(np.array([3e-5, 1e-5, 7e-5]), dHat, kappa)
    assert (n, lo, hi) == (3, 1e-5, 7e-5) and norm > 0.0
    assert od.summary(np.zeros(0), dHat, kappa)[:4] == (0, 0.0, 0.0, 0.0)


def test_plane_distance_matches_halfspace_order():
    par = np.zeros((1, 8))
    par[0, :4] = [0.0, 0.0, 1.0, -0.25]
    V = np.array([[0.1, 0.2, 0.75], [0.0, 0.0, 0.25]])
    assert np.array_equal(od.plane_d2(par, V, [[0, 0], [0, 1]]), [0.25, 0.0])
