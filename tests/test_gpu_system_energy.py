"""The end-of-step diagnostics on the device: ipcgpu_system_energy (computeSystemEnergy per component) against the float64 restatement of
tests/oracle_diagnostics.py on multi-body piles (NH and FCR), a codimensional scene with triangle, segment and point components and a scene
with an obstacle tail; identical bits for repeated, captured and replayed calls; a few time steps through ipcgpu_end_time_step; the
component table's edge cases and refusals; and ipcgpu_constraint_summary against numpy over ipcgpu_evaluate_constraints and the plane
distances of the downloaded positions."""
import contextlib

import numpy as np
import pytest

import oracle as orc
import oracle_diagnostics as od
import oracle_halfspace as ohs
import oracle_kappa as ok
import oracle_timestep as ot
from gpu_common import load_scene, own_context, same_bits, scalar_bits, soa
from ipc_b200 import codim
from ipc_b200 import lib as L
from ipc_b200 import mesh as M
from ipc_b200 import obstacle as OB
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu
KD = L.KAPPA_DEVICE
DT = 0.025
GRAVITY = (0.0, 0.0, -9.81)
EPS = np.finfo(np.float64).eps


@contextlib.contextmanager
def context(m, nV_dof=None, time=True):
    with own_context() as ctx:
        load_scene(ctx, m)
        if nV_dof is not None:
            ctx.set_obstacle_tail(nV_dof)
        if time:
            ctx.set_time_integration(L.TIT_BE, DT, gravity=GRAVITY)
        yield ctx


def moved(V, seed, amp):
    """V_prev: every vertex displaced by up to amp (a state with momentum)"""
    return V - amp * np.random.default_rng(seed).standard_normal(V.shape)


def check_energy(ctx, m_own, V, Vprev, mass, ve, te, got=None):
    """sysE, sysM, sysL of the device against the restatement per component: the vertex sums within 1e-14 of the sum of |terms|, the
    elastic part within 1e-10 relative of the oracle's per-tet energies summed with fsum"""
    E, Mo, Lo = ctx.system_energy() if got is None else got
    m_own.V = V[: m_own.nV]
    _, per = orc.Elastic(m_own).energy(1.0)
    ref = od.system_energy(per, V[: ve[-1]], Vprev[: ve[-1]], mass[: ve[-1]], ot.Params(ot.BE, DT, gravity=GRAVITY), ve, te)
    tolE = 1e-10 * np.abs(ref["E_el"]) + 1e-14 * ref["E_v_abs"] + 4 * EPS * np.abs(ref["E_el"] + ref["E_v"])
    assert np.all(np.abs(E - (ref["E_el"] + ref["E_v"])) <= tolE), np.max(np.abs(E - (ref["E_el"] + ref["E_v"])) / np.maximum(tolE, 1e-300))
    assert np.all(np.abs(Mo - ref["M"]) <= 1e-14 * ref["M_abs"])
    assert np.all(np.abs(Lo - ref["L"]) <= 1e-14 * ref["L_abs"])
    return E, Mo, Lo


def pile(energy):
    m, info = scenes.ball_pile(5, res=10, seed=3, energy=energy)
    nb = info["n_balls"]
    nv, nt = m.nV // nb, m.nT // nb
    return m, np.arange(1, nb + 1, dtype=np.int32) * nv, np.arange(1, nb + 1, dtype=np.int32) * nt


def codim_mix():
    """a ball, a triangle sheet, a segment polyline and five one-point components, in the order of a `shapes` list"""
    Vb, Tb = M.ball_tets(4, 0.5)
    g = np.linspace(-0.5, 0.5, 4)
    X, Y = np.meshgrid(g, g, indexing="ij")
    Vs = np.stack([X.ravel(), Y.ravel(), np.full(16, 0.55)], axis=1)
    F = np.array([[4 * i + j, 4 * i + j + 1, 4 * i + j + 4] for i in range(3) for j in range(3)]
                 + [[4 * i + j + 1, 4 * i + j + 5, 4 * i + j + 4] for i in range(3) for j in range(3)])
    Vseg = np.stack([np.linspace(-0.5, 0.5, 6), np.zeros(6), np.full(6, -0.55)], axis=1)
    comps = [dict(codim=3, V=Vb, T=Tb), dict(codim=2, V=Vs, F=F), dict(codim=1, V=Vseg, E=np.array([[i, i + 1] for i in range(5)]))]
    comps += [dict(codim=0, V=[[0.55 + 0.02 * k, 0.0, 0.05 * k]]) for k in range(5)]
    return codim.codim_scene(comps, density=1000.0, YM=1e4, PR=0.4)


@pytest.mark.parametrize("energy", [0, 1])
def test_pile_components(energy):
    m, ve, te = pile(energy)
    Vp = moved(m.V, 1, 1e-3)
    with context(m) as ctx:
        ctx.set_prev_state(soa(Vp))
        ctx.set_components(ve, te)
        check_energy(ctx, m, m.V, Vp, m.mass, ve, te)


def test_codim_components():
    m = codim_mix()
    ve, te = codim.component_ends(m)
    assert len(ve) == 8 and np.all(np.diff(ve)[-5:] == 1) and np.all(te[1:] == te[0])
    V = m.V_rest + 1e-3 * np.random.default_rng(4).standard_normal(m.V_rest.shape)
    m.V = V
    Vp = moved(V, 5, 1e-3)
    with context(m) as ctx:
        ctx.set_prev_state(soa(Vp))
        ctx.set_components(ve, te)
        check_energy(ctx, m, V, Vp, m.mass, ve, te)


def test_obstacle_tail_excluded():
    m, info = scenes.balls_on_obstacle(3, res=4)
    mm = OB.with_obstacle(m, info["obstacle"]["V"], info["obstacle"]["E"], info["obstacle"]["F"])
    nb = 3
    ve = np.arange(1, nb + 1, dtype=np.int32) * (m.nV // nb)
    te = np.arange(1, nb + 1, dtype=np.int32) * (m.nT // nb)
    Vp = moved(mm.V, 6, 1e-3)
    with context(mm, nV_dof=mm.nV_dof) as ctx:
        ctx.set_prev_state(soa(Vp))
        with pytest.raises(L.IpcGpuError, match="ARG"):  # the tail belongs to no component
            ctx.set_components(np.append(ve[:-1], mm.nV), te)
        ctx.set_components(ve, te)
        check_energy(ctx, m, mm.V, Vp, mm.mass, ve, te)


def test_bits_repeat_capture_and_edge_ranges():
    m, _, _ = pile(0)
    Vp = moved(m.V, 7, 1e-3)
    with context(m) as ctx:
        ctx.set_prev_state(soa(Vp))
        assert m.nV > 4200 and m.nT > 4200
        layouts = [
            ([1, 2047, 2049, 4100, m.nV], [0, 2048, 2048, 4097, m.nT]),  # a one-vertex component, ranges straddling the 2048-chunk grid
            ([m.nV], [m.nT]),                                            # one component covering everything
            (list(range(1, 301)) + [m.nV], [0] * 300 + [m.nT]),          # many one-vertex components
        ]
        for ve, te in layouts:
            ctx.set_components(ve, te)
            a = check_energy(ctx, m, m.V, Vp, m.mass, np.asarray(ve), np.asarray(te))
            b = ctx.system_energy()
            assert all(same_bits(x, y) for x, y in zip(a, b))
            n0 = ctx.launch_count()
            ctx.capture_begin()
            ctx.system_energy(want=False)
            gid = ctx.capture_end()
            ctx.graph_launch(gid)
            c = ctx.get_system_energy()
            assert all(same_bits(x, y) for x, y in zip(a, c))
            assert ctx.launch_count() - n0 == 3
        # a new component table refuses the graphs captured before it
        ctx.set_components([m.nV], [m.nT])
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.graph_launch(gid)


def test_time_steps_through_end_time_step():
    m, ve, te = pile(1)
    with context(m) as ctx:
        Vprev = m.V_rest.copy()
        ctx.set_prev_state(soa(Vprev))
        ctx.compute_xtilde()  # (the x~ that ipcgpu_end_time_step reads)
        ctx.set_components(ve, te)
        rng = np.random.default_rng(8)
        V = m.V.copy()
        for step in range(3):
            ctx.set_state(soa(V))
            check_energy(ctx, m, V, Vprev, m.mass, ve, te)
            ctx.end_time_step()  # V_prev := V on the device
            Vprev = V.copy()
            V = V + 1e-3 * rng.standard_normal(V.shape)


def test_refusals():
    m, ve, te = pile(0)
    with context(m, time=False) as ctx:
        ctx.set_prev_state(m.V_soa)
        with pytest.raises(L.IpcGpuError, match="STATE"):  # no components yet
            ctx.system_energy()
        for bad_v, bad_t in [(ve[::-1], te), (ve, te[::-1]), (np.append(-1, ve), np.append(0, te)), (ve - 1, te), (ve, te + 1),
                             (np.zeros(0), np.zeros(0))]:
            with pytest.raises(L.IpcGpuError, match="ARG"):
                ctx.set_components(bad_v, bad_t)
        ctx.set_components(ve, te)
        with pytest.raises(L.IpcGpuError, match="STATE"):  # no time integration
            ctx.system_energy()
        ctx.set_time_integration(L.TIT_BE, DT)
        ctx.system_energy()
        # a new mesh removes the components
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        with pytest.raises(L.IpcGpuError, match="STATE"):
            ctx.system_energy()


# ---- the constraint summary --------------------------------------------------------------------------------------------------------
def summary_check(ctx, m, dHat, kappa, par=None):
    """n, d_min and d_max bit-equal to numpy over ipcgpu_evaluate_constraints and the plane distances of the downloaded V; fb_norm within
    1e-13 relative (or within the rounding of its cancellation: fb = dual + d - sqrt(dual^2 + d^2) loses the scale of dual where dual >> d)"""
    got = ctx.constraint_summary(dHat, kappa)
    nC = ctx.constraint_set_sizes()[0]
    vals = ctx.evaluate_constraints(nC)
    V = ctx.download(L.BUF_POSITIONS, 3 * m.nV).reshape(3, -1).T
    d = vals
    if par is not None:
        act = ctx.get_halfspace_sets()[0]
        d = np.concatenate([od.plane_d2(par, V, act), vals])
    n, lo, hi, fbn, scale = od.summary(d, dHat, kappa)
    assert (got.n, scalar_bits(got.d_min), scalar_bits(got.d_max)) == (n, scalar_bits(lo), scalar_bits(hi))
    assert abs(got.fb_norm - fbn) <= max(1e-13 * fbn, 8 * EPS * scale), (got.fb_norm, fbn, scale)
    return got


def mat_with_plane():
    m, info = scenes.ball_on_mat(nx=10, res=4, gap_lo=0.2, gap_hi=0.5)
    dHat = info["dHat"]
    z0 = m.V[:, 2].min() - 0.5 * np.sqrt(dHat)
    return m, dHat, dict(origin=[[0.0, 0.0, z0]], normal=[[0.0, 0.0, 1.0]], friction=[0.0])


def planes_par(pl):
    return ohs.planes(np.asarray(pl["origin"], float), np.asarray(pl["normal"], float), None, np.asarray(pl["friction"], float))


def test_summary_self_and_planes_host_and_device_kappa():
    m, dHat, pl = mat_with_plane()
    with context(m, time=False) as ctx:
        ctx.set_halfspaces(**pl)
        ctx.constraint_set(dHat, 1)
        assert ctx.halfspace_constraint_set(dHat) > 0 and ctx.nC > 0
        K = 3.7e5
        a = summary_check(ctx, m, dHat, K, planes_par(pl))
        # deferred and captured: the same bits
        ctx.capture_begin()
        ctx.constraint_summary(dHat, K, want=False)
        gid = ctx.capture_end()
        ctx.graph_launch(gid)
        b = ctx.get_constraint_summary()
        assert (a.n, scalar_bits(a.d_min), scalar_bits(a.d_max), scalar_bits(a.fb_norm)) == (b.n, scalar_bits(b.d_min), scalar_bits(b.d_max), scalar_bits(b.fb_norm))
        # kappa on the device after initKappa: the host-kappa call at the kappa read back
        ctx.barrier_gradient(1e-30, 0.0, np.zeros(3 * m.nV))  # (a defined device gradient g_E for initKappa)
        ctx.set_kappa(1.0, 1e3, 1e12)
        ctx.kappa_init(dHat)
        k = ctx.kappa_info().kappa
        dev, host = ctx.constraint_summary(dHat, KD), ctx.constraint_summary(dHat, k)
        assert (dev.n, scalar_bits(dev.d_min), scalar_bits(dev.d_max), scalar_bits(dev.fb_norm)) == (host.n, scalar_bits(host.d_min), scalar_bits(host.d_max), scalar_bits(host.fb_norm))


def test_summary_planes_only_and_empty():
    V, T = M.grid_tets(4, 4, 4, h=0.25)
    m = M.Mesh(V, T, energy=0)
    dHat = 1e-4
    with context(m, time=False) as ctx:
        ctx.constraint_set(dHat, 1)
        assert ctx.nC == 0
        e = ctx.constraint_summary(dHat, 1e4)  # no plane, no pair: "no collision in this time step"
        assert (e.n, e.d_min, e.d_max, e.fb_norm) == (0, 0.0, 0.0, 0.0)
        pl = dict(origin=[[0.0, 0.0, -0.5 * np.sqrt(dHat)]], normal=[[0.0, 0.0, 1.0]], friction=[0.0])
        ctx.set_halfspaces(**pl)
        assert ctx.halfspace_constraint_set(dHat) > 0
        assert summary_check(ctx, m, dHat, 1e4, planes_par(pl)).n > 0


def test_summary_obstacle_pairs():
    m, info = scenes.balls_on_obstacle(3, res=4)
    mm = OB.with_obstacle(m, info["obstacle"]["V"], info["obstacle"]["E"], info["obstacle"]["F"])
    dHat = info["dHat"]
    with context(mm, nV_dof=mm.nV_dof, time=False) as ctx:
        mm_set = ctx.constraint_set(dHat, 1)[0]
        assert any(OB.involves_obstacle(q, mm.nV_dof) for q in mm_set)
        summary_check(ctx, mm, dHat, 2e5)


def test_summary_codim_pairs():
    m = codim_mix()
    m.V = m.V_rest.copy()
    dHat = 0.1 ** 2
    with context(m, time=False) as ctx:
        mm_set = ctx.constraint_set(dHat, 1)[0]
        codim_v = set(np.flatnonzero(m.vCoDim < 3).tolist())
        assert any(codim_v & set(ok.stencil(q)[1]) for q in mm_set)
        assert summary_check(ctx, m, dHat, 1e3).n == len(mm_set)
