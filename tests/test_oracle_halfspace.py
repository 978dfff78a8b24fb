"""CPU checks of the half-space oracle (oracle/halfspace.cpp, HalfSpace<3>): finite differences E -> g -> H of the barrier and of both friction
branches, the closed forms of the blocks, the step bound against an independent numpy evaluation, the crossing quirk of isIntersected."""

import numpy as np
import pytest

import oracle as orc
import oracle_halfspace as OH
from ipc_b200 import mesh as M

def _block(nV=40, seed=0):
    V, T = M.grid_tets(3, 3, 3)
    m = M.Mesh(V, T, energy=0)
    rng = np.random.default_rng(seed)
    m.V = m.V + 0.01 * rng.standard_normal(m.V.shape)
    return m


def _single_vertex_plane(n, dist, seed=0, velocitydt=None, friction=0.4):
    """one plane with unit-normalised normal n through the origin; a point at signed distance `dist`"""
    par = OH.planes([[0.0, 0.0, 0.0]], [n], velocitydt, [friction])[0]
    rng = np.random.default_rng(seed)
    t = rng.standard_normal(3)
    t -= t.dot(par[:3]) * par[:3]
    x = dist * par[:3] + t
    return par, x


def _barrier_energy(par, x, dHat, kappa):
    dist = ((par[0] * x[0] + par[1] * x[1]) + par[2] * x[2]) + par[3]
    b, _, _ = orc_barrier(dist * dist, dHat)
    return kappa * b


def orc_barrier(d, dHat):
    import ctypes as C
    b, db, d2b = C.c_double(), C.c_double(), C.c_double()
    orc.lib().orc_barrier(C.c_double(d), C.c_double(dHat), C.byref(b), C.byref(db), C.byref(d2b))
    return b.value, db.value, d2b.value


@pytest.mark.parametrize("normal", [[0, 1, 0], [1, 0.3, -0.2], [-0.4, 0.9, 0.7]])
def test_barrier_fd_and_rank_one_block(normal):
    dHat, kappa = 1e-2, 3.0
    par, x = _single_vertex_plane(normal, 0.05)
    dist = x.dot(par[:3]) + par[3]
    _, db, d2b = orc_barrier(dist * dist, dHat)
    g = kappa * db * 2.0 * dist * par[:3]
    h = 1e-6
    g_fd = np.array([(_barrier_energy(par, x + h * e, dHat, kappa) - _barrier_energy(par, x - h * e, dHat, kappa)) / (2 * h) for e in np.eye(3)])
    assert np.allclose(g, g_fd, rtol=1e-6, atol=1e-9)
    H = OH.barrier_block(par, dist, dHat, kappa, project=0)

    def grad(y):
        dd = y.dot(par[:3]) + par[3]
        return kappa * orc_barrier(dd * dd, dHat)[1] * 2.0 * dd * par[:3]
    H_fd = np.array([(grad(x + h * e) - grad(x - h * e)) / (2 * h) for e in np.eye(3)]).T
    assert np.allclose(H, H_fd, rtol=1e-5, atol=1e-6 * np.abs(H).max())
    # closed form: rank one along n, kappa (4 b'' d + 2 b') n n^T; the projection keeps it iff that coefficient is positive
    param = 4.0 * d2b * dist * dist + 2.0 * db
    assert np.allclose(H, kappa * param * np.outer(par[:3], par[:3]), rtol=1e-14, atol=0)
    assert np.linalg.matrix_rank(H, tol=1e-10 * np.abs(H).max()) == 1
    Hp = OH.barrier_block(par, dist, dHat, kappa, project=1)
    assert np.array_equal(Hp, H) if param > 0 else not Hp.any()


def _fric_E(par, x, xt, lam, eps2):
    eps = np.sqrt(eps2)
    u = (x - xt) - par[4:7]
    u = u - u.dot(par[:3]) * par[:3]
    m2 = u.dot(u)
    m = par[7] * lam
    return m * (np.sqrt(m2) - eps * 0.5) if m2 > eps2 else m * m2 / eps * 0.5


@pytest.mark.parametrize("slide", [True, False])
def test_friction_fd_both_branches_and_spectrum(slide):
    eps2 = 1e-4
    par, x = _single_vertex_plane([0.2, 1.0, 0.1], 0.01, seed=3, velocitydt=[[1e-3, 0.0, 2e-3]])
    rng = np.random.default_rng(7)
    step = (0.3 if slide else 2e-3) * rng.standard_normal(3)
    xt = x - step
    lam = 2.5
    import ctypes as C
    from oracle import d
    # the gradient of the oracle: a one-vertex surface around orc_hs_friction_gradient
    V = np.ascontiguousarray(x.reshape(3, 1)).ravel()
    Vt = np.ascontiguousarray(xt.reshape(3, 1)).ravel()
    s = orc.OrcSurf(1, d(V), d(V), None, 0, None, 0, None, 0, None, None)
    g = np.zeros(3)
    lag = np.zeros((1, 2), np.int32)
    orc.lib().orc_hs_friction_gradient(C.byref(s), d(Vt), d(np.ascontiguousarray(par)), orc.i(lag), d(np.array([lam])), 1, C.c_double(eps2), d(g))
    E = C.c_double()
    orc.lib().orc_hs_friction_energy(C.byref(s), d(Vt), d(np.ascontiguousarray(par)), orc.i(lag), d(np.array([lam])), 1, C.c_double(eps2), C.byref(E))
    assert np.isclose(E.value, _fric_E(par, x, xt, lam, eps2), rtol=1e-14)
    h = 1e-7
    g_fd = np.array([(_fric_E(par, x + h * e, xt, lam, eps2) - _fric_E(par, x - h * e, xt, lam, eps2)) / (2 * h) for e in np.eye(3)])
    assert np.allclose(g, g_fd, rtol=1e-5, atol=1e-8 * max(1.0, np.abs(g).max()))

    def grad(y):
        out = np.zeros(3)
        Vy = np.ascontiguousarray(y.reshape(3, 1)).ravel()
        sy = orc.OrcSurf(1, d(Vy), d(Vy), None, 0, None, 0, None, 0, None, None)
        orc.lib().orc_hs_friction_gradient(C.byref(sy), d(Vt), d(np.ascontiguousarray(par)), orc.i(lag), d(np.array([lam])), 1, C.c_double(eps2), d(out))
        return out
    H = OH.friction_block(par, x, xt, lam, eps2, project=0)
    H_fd = np.array([(grad(x + h * e) - grad(x - h * e)) / (2 * h) for e in np.eye(3)]).T
    assert np.allclose(H, H_fd, rtol=1e-4, atol=1e-6 * np.abs(H).max())
    u = (x - xt) - par[4:7]
    u = u - u.dot(par[:3]) * par[:3]
    m = par[7] * lam
    ev = np.sort(np.linalg.eigvalsh(H))
    if slide:  # spectrum {0, 0, m/|u|}: the projection only moves entries at rounding level
        assert np.allclose(ev, [0.0, 0.0, m / np.linalg.norm(u)], atol=1e-12 * m / np.linalg.norm(u))
        Hp = OH.friction_block(par, x, xt, lam, eps2, project=1)
        assert np.allclose(Hp, H, atol=1e-13 * np.abs(H).max())
    else:  # m/eps (I - n n^T)
        assert np.allclose(H, m / np.sqrt(eps2) * (np.eye(3) - np.outer(par[:3], par[:3])), rtol=1e-14, atol=1e-14 * m / np.sqrt(eps2))


def _numpy_step(m, par, p, slack, alpha):
    out = alpha
    for pl in par:
        best = 1.0
        for v in m.SVI:
            if m.dbc[v]:
                continue
            c = (pl[0] * p[3 * v] + pl[1] * p[3 * v + 1]) + pl[2] * p[3 * v + 2]
            if c < 0:
                dist = ((pl[0] * m.V[v, 0] + pl[1] * m.V[v, 1]) + pl[2] * m.V[v, 2]) + pl[3]
                best = min(best, -dist / c * slack)
        out = min(out, best)
    return max(out, 0.0)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_step_bound_against_numpy(seed):
    m = _block(seed=seed)
    rng = np.random.default_rng(seed)
    m.dbc[rng.choice(m.nV, 5, replace=False)] = 1
    normals = [np.array([0.0, 1.0, 0.0]), rng.standard_normal(3), rng.standard_normal(3)]
    # every vertex in front of every plane (tilted normals included), at a gap of 0.05-0.3 from the nearest one
    origins = [m.V[np.argmin(m.V @ n)] - (0.05 + 0.1 * k) * n / np.linalg.norm(n) for k, n in enumerate(normals)]
    par = OH.planes(origins, normals, None, [0.0, 0.1, 0.2])
    p = rng.standard_normal(3 * m.nV)
    p.reshape(-1, 3)[:, 1] -= 2.0
    s = orc.Surf(m)
    hs = OH.HalfSpaces(s, par)
    a = hs.step(p, 0.9, 1.0)
    assert a == _numpy_step(m, par, p, 0.9, 1.0)
    assert 0.0 < a < 1.0


def test_step_bound_behind_the_plane_is_zero():
    m = _block()
    par = OH.planes([m.V[m.SVI[0]] + [0, 0.01, 0]], [[0, 1, 0]], None, [0.0])
    p = np.zeros(3 * m.nV)
    p[1::3] = -1.0
    hs = OH.HalfSpaces(orc.Surf(m), par)
    assert hs.step(p, 0.9, 1.0) == 0.0


def test_crossing_quirk_exactly_on_and_behind():
    m = _block()
    y0 = 0.25
    par = OH.planes([[0.0, y0, 0.0]], [[0, 1, 0]], None, [0.0])
    V = m.V.copy()
    V[:, 1] = np.maximum(V[:, 1], y0 + 0.1)
    v_on, v_behind, v_dbc = m.SVI[0], m.SVI[1], m.SVI[2]
    V[v_on, 1] = y0          # dist == 0: d <= 0, counted
    V[v_behind, 1] = y0 - 0.2  # behind the plane: d > 0, NOT counted (the reference tests the squared distance)
    V[v_dbc, 1] = y0
    m.dbc[v_dbc] = 1          # Dirichlet: skipped
    hs = OH.HalfSpaces(orc.Surf(m, V=V), par)
    assert hs.crossings() == 1
    m.vCoDim[v_on] = 2        # codimension != 3: skipped
    assert OH.HalfSpaces(orc.Surf(m, V=V), par).crossings() == 0


def test_active_set_order_and_filters():
    m = _block()
    lo = m.V[:, 1].min()
    par = OH.planes([[0, lo - 0.01, 0], [0, lo - 0.02, 0]], [[0, 1, 0], [0, 1, 0]], None, [0.5, 0.0])
    m.dbc[m.SVI[3]] = 2
    m.vCoDim[m.SVI[4]] = 1
    hs = OH.HalfSpaces(orc.Surf(m), par)
    dHat = 0.04
    act = hs.constraint_set(dHat)
    ref = [(k, v) for k in range(2) for v in m.SVI
           if not m.dbc[v] and m.vCoDim[v] == 3 and (m.V[v, 1] - (lo - 0.01 * (k + 1))) ** 2 < dHat]
    assert [tuple(e) for e in act] == ref and len(ref) > 0
    lag, lam = hs.lag(act, dHat, 2.0)
    assert all(e[0] == 0 for e in lag) and len(lag) == sum(1 for e in ref if e[0] == 0)
    assert (lam > 0).all()


def test_halfspace_adapter_compiles_against_the_restated_interface():
    """adapters/IpcGpuHalfSpace.hpp (HalfSpace<3> with the IP-path virtuals on the device) against tests/stubs/CollisionObject.h"""
    import os
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = ["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Wno-unused-parameter", "-I", os.path.join(root, "tests", "stubs"),
           "-I", os.path.join(root, "adapters"), "-I", root, os.path.join(root, "tests", "stubs", "halfspace_adapter_check.cpp")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
