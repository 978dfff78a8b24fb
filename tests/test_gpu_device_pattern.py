"""The contact-augmented sparsity pattern built on the device (ipcgpu_enable_device_pattern / ipcgpu_update_pattern): exactly the host
mirror's set_pattern(vNeighbor + augmentConnectivity(sets)) at every state, `changed` tracking, values equal to the oracle and to host-pattern
mode, one captured graph across changing contacts, the capacity error, the obstacle tail, the PCG solve after a change, and two ranks."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import oracle as orc
from gpu_common import rel, scalar_bits, shared_ctx, soa
from ipc_b200 import lib as L
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs
from test_gpu_multilevel import load_sorted
from test_oracle_meshco import contact_pairs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KAPPA, DT2, TOL = 1e8, 0.025 ** 2, 1e-6


def states(ctx, m, info):
    """A (the scene), B (half of the feasible step along p: more contacts), C (every body ten times farther apart: no contact)"""
    p = info["p"]
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    ctx.constraint_set(info["dHat"], 1, fetch=False)
    a = ctx.inversion_step(p, 0.2, 1.0)
    a = ctx.ccd_partial(None, TOL, evf, eee, a)
    a = ctx.hash_build_swept(None, a, m.avgEdgeLen / 3)
    a, _ = ctx.ccd_full(TOL, evf, eee, a)
    return {"A": m.V.copy(), "B": m.V + 0.5 * a * p.reshape(-1, 3), "C": 10.0 * m.V}


def host_pattern(m, sets, base=1, extra=None):
    pairs = [contact_pattern_pairs(m, *s) for s in sets]
    pairs = [x for x in pairs if x is not None] + ([extra] if extra is not None else [])
    return m.csr_pattern(base, extra_pairs=np.concatenate(pairs) if pairs else None)


def at(ctx, V, dHat):
    ctx.set_state(soa(V))
    mm, pa, pe, _ = ctx.constraint_set(dHat, 1)
    return mm, pa, pe


@pytest.mark.parametrize("base", [0, 1])
def test_exact_pattern_with_and_without_friction(shared_ctx, base):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat = info["dHat"]
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(base)
    ia, ja = ctx.get_pattern()
    ia0, ja0 = m.csr_pattern(base)
    assert np.array_equal(ia, ia0) and np.array_equal(ja, ja0)  # enable: the mesh pattern
    mm, pa, pe = at(ctx, S["A"], dHat)
    assert len(mm) > 0
    changed, nnz = ctx.update_pattern()
    ia, ja = ctx.get_pattern()
    ia_h, ja_h = host_pattern(m, [(mm, pa, pe)], base)
    assert changed == 1 and nnz == ja_h.size and np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h)
    # lagged friction set taken at B, active set of A: the update with friction holds both
    mmB, _, _ = at(ctx, S["B"], dHat)
    ctx.set_prev_state(soa(S["A"]))
    ctx.friction_lag(dHat, KAPPA)
    lagged = ctx.get_friction_data()[0]
    assert len(lagged) == len(mmB) > len(mm)
    mm, pa, pe = at(ctx, S["A"], dHat)
    changed, nnz = ctx.update_pattern(with_friction=1)
    ia, ja = ctx.get_pattern()
    ia_h, ja_h = host_pattern(m, [(mm, pa, pe), (lagged, np.zeros((0, 4), np.int32), np.zeros((0, 2), np.int32))], base)
    assert changed == 1 and np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h)
    assert ctx.update_pattern(with_friction=0)[0] == 1  # the lagged-only blocks leave again
    assert np.array_equal(ctx.get_pattern()[1], host_pattern(m, [(mm, pa, pe)], base)[1])


def test_c5_full_size_pattern(shared_ctx):
    sys.path.insert(0, ROOT)
    import bench

    class Args:
        tets, res, scene = 1_000_000, 10, "c5"

    ctx = shared_ctx
    m, info = bench.build_scene(Args())
    load_sorted(ctx, m)
    mm, pa, pe, _ = ctx.constraint_set(info["dHat"], 1)
    assert len(mm) > 1000
    ctx.enable_device_pattern(1)
    changed, nnz = ctx.update_pattern()
    ia, ja = ctx.get_pattern()
    ia_h, ja_h = host_pattern(m, [(mm, pa, pe)])
    assert changed == 1 and nnz == ja_h.size and np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h)
    assert ctx.update_pattern() == (0, nnz)


def test_change_tracking(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat = info["dHat"]
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(1)
    seen = []
    for name, want_changed in (("A", 1), ("B", 1), ("A", 1), ("A", 0), ("C", 1), ("C", 0)):
        sets = at(ctx, S[name], dHat)
        if name == "C":
            assert len(sets[0]) == 0 and len(sets[1]) == 0
        ctx.update_pattern(want=False)  # deferred form, read back by the fetch
        it = ctx.fetch_iteration()
        assert it.status == 0
        changed, nnz, version = ctx.pattern_info()
        ia, ja = ctx.get_pattern()
        ia_h, ja_h = host_pattern(m, [sets])
        assert (changed, nnz) == (want_changed, ja_h.size), name
        assert np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h), name
        seen.append((name, nnz, version))
    assert seen[1][1] > seen[0][1] and seen[2][1] == seen[0][1]
    assert [v for _, _, v in seen] == [1, 2, 3, 3, 4, 4]
    assert seen[-1][1] == m.csr_pattern(1)[1].size  # no contact: back to the mesh pattern


def test_values_match_oracle_and_host_mode(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat = info["dHat"]
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(1)
    at(ctx, S["A"], dHat)
    ctx.update_pattern()
    mm, pa, pe = at(ctx, S["B"], dHat)
    assert ctx.update_pattern()[0] == 1
    ia, ja = ctx.get_pattern()
    s, o = orc.Surf(m, V=S["B"]), orc.Elastic(m, V=S["B"])
    E, Er = ctx.elastic_energy(DT2), o.energy(DT2)[0]
    assert abs(E - Er) <= 1e-10 * abs(Er)
    Eb, (Ebr, bad) = ctx.barrier_energy(dHat, KAPPA), s.barrier_energy(mm, pa, pe, dHat, KAPPA)
    assert bad == 0 and abs(Eb - Ebr) <= 1e-10 * abs(Ebr)
    g = ctx.elastic_gradient(DT2, 1, 1)
    ctx.barrier_gradient(dHat, KAPPA, g)
    g_r = s.barrier_gradient(mm, pa, pe, dHat, KAPPA, g=o.gradient(DT2, 1))
    assert rel(g, g_r) <= 1e-10
    a = np.zeros(ja.size)
    ctx.elastic_hessian(DT2, 1, 1, 1, a)
    ctx.barrier_hessian(dHat, KAPPA, 1, a)
    a_r = s.barrier_hessian_csr(mm, pa, pe, dHat, KAPPA, ia, ja, 1, 1, a=o.hessian_csr(DT2, ia, ja, 1, 1, 1))
    assert rel(a, a_r) <= 1e-9
    # no barrier term: the elastic values are bit-identical to host-pattern mode on the same pattern
    g1, a1 = np.empty(3 * m.nV), np.empty(ja.size)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, g1, a1)
    ctx.set_csr(ia, ja, 1)
    g2, a2 = np.empty(3 * m.nV), np.empty(ja.size)
    ctx.elastic_grad_hess(DT2, 1, 1, 1, g2, a2)
    assert np.array_equal(a1, a2) and np.array_equal(g1, g2)


def test_one_graph_across_changing_contacts(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat, p, h = info["dHat"], info["p"], m.avgEdgeLen / 3
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    ctx.enable_device_pattern(1)
    ctx.set_canonical_order(0)
    ctx.set_search_dir(p)

    def enqueue():
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.barrier_energy(dHat, KAPPA, want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, KAPPA, None)
        ctx.barrier_hessian(dHat, KAPPA, 1, None)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, TOL, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(TOL, evf, eee, None)

    def result():
        it = ctx.fetch_iteration()
        assert it.status == 0 and it.ti_warnings == 0
        ia, ja = ctx.get_pattern()
        part = ctx.partition_info()
        assert part["value_begin"] == 0 and part["value_end"] == ja.size
        steps = [scalar_bits(x) for x in (it.alpha_inversion, it.alpha_partial_ccd, it.alpha_swept_grid, it.alpha_full_ccd, it.alpha)]
        return it, ia, ja, steps, ctx.download(L.BUF_GRADIENT, 3 * m.nV), ctx.download(L.BUF_CSR_VALUES, ja.size)

    ctx.set_state(soa(S["A"]))
    enqueue()  # eager warm-up (lazy allocations)
    result()
    hg = L.PinnedArray(16)
    ctx.download_range_async(L.BUF_GRADIENT, 0, hg.array)  # (creates the copy stream outside the capture)
    ctx.sync()
    ctx.capture_begin()
    enqueue()
    with pytest.raises(L.IpcGpuError, match="STATE"):
        ctx.download_range_async(L.BUF_CSR_VALUES, 0, hg.array)
    ctx.download_range_async(L.BUF_GRADIENT, 0, hg.array)  # the gradient copy stays allowed
    gid = ctx.capture_end()
    for name in ("A", "B", "C", "B"):
        ctx.set_state(soa(S[name]))
        ctx.graph_launch(gid)
        it1, ia1, ja1, st1, g1, a1 = result()
        assert np.array_equal(hg.array, g1[:16])
        enqueue()
        it2, ia2, ja2, st2, g2, a2 = result()
        assert np.array_equal(ia1, ia2) and np.array_equal(ja1, ja2) and st1 == st2, name
        assert rel(g1, g2) <= 1e-13 and rel(a1, a2) <= 1e-13 and abs(it1.energy_barrier - it2.energy_barrier) <= 1e-12 * max(abs(it2.energy_barrier), 1e-300)
        mm, pa, pe, _ = ctx.constraint_set(dHat, 1)
        ia_h, ja_h = host_pattern(m, [(mm, pa, pe)])
        assert np.array_equal(ia1, ia_h) and np.array_equal(ja1, ja_h), name
        if name == "C":
            assert it1.n_active == 0 and ja1.size == m.csr_pattern(1)[1].size
    ctx.graph_destroy(gid)
    hg.free()


def test_capacity_error_and_raise(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat = info["dHat"]
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(1)
    at(ctx, S["A"], dHat)
    nnzA = ctx.update_pattern()[1]
    mmB, paB, peB = at(ctx, S["B"], dHat)
    nnzB = ctx.update_pattern()[1]
    assert nnzB > nnzA
    ctx.enable_device_pattern(1, nnzA)
    at(ctx, S["A"], dHat)
    ctx.update_pattern(want=False)
    assert ctx.fetch_iteration().status == 0
    at(ctx, S["B"], dHat)
    ctx.update_pattern(want=False)
    with pytest.raises(L.IpcGpuError, match="CAPACITY"):
        ctx.fetch_iteration()
    assert ctx.pattern_info()[:2] == (0, nnzA)  # the previous pattern is kept, nothing written past it
    with pytest.raises(L.IpcGpuError, match="CAPACITY"):
        ctx.update_pattern()
    ctx.enable_device_pattern(1, nnzB)
    assert ctx.update_pattern() == (1, nnzB)
    assert ctx.fetch_iteration().status == 0
    assert np.array_equal(ctx.get_pattern()[1], host_pattern(m, [(mmB, paB, peB)])[1])


def test_obstacle_tail_rows_stay_diagonal(shared_ctx):
    from ipc_b200 import obstacle as OB
    ctx = shared_ctx
    m, info = scenes.balls_on_obstacle(plate_angle=0.0, res=4, plate=12)
    ob = info["obstacle"]
    M2 = OB.with_obstacle(m, ob["V"], ob["E"], ob["F"])
    load_sorted(ctx, M2)
    ctx.set_obstacle_tail(M2.nV_dof, 1)
    ctx.enable_device_pattern(1)
    mm, pa, pe, _ = ctx.constraint_set(info["dHat"], 1)
    assert any((r[1:] >= M2.nV_dof).any() or (r[0] < 0 and -r[0] - 1 >= M2.nV_dof) for r in mm)  # mesh-obstacle pairs are active
    assert ctx.update_pattern()[0] == 1
    ia, ja = ctx.get_pattern()
    ia_h, ja_h = M2.csr_pattern(1, extra_pairs=contact_pairs(mm, pa, pe, M2.SFEdges, M2.nV_dof))
    assert np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h)
    rows = np.arange(3 * M2.nV_dof, 3 * M2.nV)
    assert np.array_equal(np.diff(ia)[rows], 3 - rows % 3)  # the tail's rows: the diagonal block only
    assert (ja[: ia[3 * M2.nV_dof] - 1] <= 3 * M2.nV_dof).all()  # no mesh row reaches into the tail's columns


def full_matrix(ia, ja, a, n):
    U = sp.csr_matrix((a, np.asarray(ja) - 1, np.asarray(ia) - 1), shape=(n, n))
    return (U + sp.triu(U, 1).T).tocsc()


def test_pcg_after_a_pattern_change(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    dHat, kappa = info["dHat"], 1e6
    load_sorted(ctx, m)
    S = states(ctx, m, info)
    ctx.enable_device_pattern(1)
    for name in ("A", "B"):
        ctx.set_state(soa(S[name]))
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.elastic_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        x, iters, res = ctx.solve_pcg(None, rel_tol=1e-10, max_iter=5000)
        assert res <= 1e-10 and 0 < iters < 5000
        assert ctx.pattern_info()[0] == 1
    mm, pa, pe = at(ctx, S["B"], dHat)
    ia, ja = ctx.get_pattern()
    assert np.array_equal(ja, host_pattern(m, [(mm, pa, pe)])[1])
    s, o = orc.Surf(m, V=S["B"]), orc.Elastic(m, V=S["B"])
    g_ref = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=o.gradient(DT2, 1))
    a_ref = o.hessian_csr(DT2, ia, ja, 1, 1, 1)
    a_ref[np.asarray(ia[:-1], dtype=np.int64) - 1] += np.repeat(m.mass, 3)
    a_ref = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, 1, a=a_ref)
    x_ref = spla.spsolve(full_matrix(ia, ja, a_ref, 3 * m.nV), -g_ref)
    assert rel(x, x_ref) <= 1e-7


def test_two_ranks_build_the_same_pattern():
    try:
        n = int(subprocess.check_output(["nvidia-smi", "-L"], text=True).count("GPU "))
    except Exception:
        n = 0
    if n < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29613",
           os.path.join(ROOT, "tests", "mp", "device_pattern_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "DEVICE_PATTERN_CHECK world=2 OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
