"""Shared body of the full-size GPU parity tests: EVERY stage of the Newton hot path through the C ABI against the oracle's
reference-style (hashed) drivers on all host cores.  Integer sets identical (as sorted multisets when the device order is not canonical),
E / g <= 1e-10 relative, CSR values <= 1e-9, step bounds bit-exact.  Size-independent properties ride along."""
import os

import numpy as np

import oracle as orc
from gpu_common import load_scene, rel, scalar_bits
from ipc_b200 import lib as L

RTOL = 1e-10


def sort_rows(a, *companions):
    """lexicographic row sort of an integer array (with companion arrays as less significant keys, permuted alongside)"""
    a = np.asarray(a)
    if len(a) == 0:
        return (a,) + tuple(np.asarray(c) for c in companions)
    keys = []
    for c in reversed(companions):
        keys += [np.asarray(c)[:, k] for k in range(np.asarray(c).shape[1] - 1, -1, -1)]
    keys += [a[:, k] for k in range(a.shape[1] - 1, -1, -1)]
    order = np.lexsort(keys)
    return (a[order],) + tuple(np.asarray(c)[order] for c in companions)


def contact_pattern_pairs(m, mm, pa, pe):
    import bench
    return bench.contact_pattern_pairs(m, mm, pa, pe)


def check_every_stage(ctx, m, info, kappa=1e8, dt2=0.025 ** 2, tol=1e-6, canonical=True, min_active=1, n_prop=300, h_tol=1e-9):
    nth = os.cpu_count() or 8
    dHat, p = info["dHat"], info["p"]
    hvox = m.avgEdgeLen / 3.0
    load_scene(ctx, m)
    ctx.set_canonical_order(1 if canonical else 0)
    ctx.set_contact_partition(0 if canonical else 1)  # (a no-op on one rank; this is the exact mode bench.py times)
    o, s = orc.Elastic(m), orc.Surf(m)
    out = {}

    # constraint set: identical integer sets
    mm, pa, pe, cand = ctx.constraint_set(dHat, 1)
    mm_r, pa_r, pe_r, cand_r = s.constraint_set_hashed(dHat, hvox, nth)
    assert len(mm_r) >= min_active, len(mm_r)
    if canonical:
        assert np.array_equal(mm, mm_r) and np.array_equal(pa, pa_r) and np.array_equal(pe, pe_r) and np.array_equal(cand, cand_r)
    else:  # the device order is whatever the atomic appends produced (the reference's own order is scheduling dependent too)
        assert np.array_equal(sort_rows(mm)[0], sort_rows(mm_r)[0])
        a1, b1 = sort_rows(pa, pe)
        a2, b2 = sort_rows(pa_r, pe_r)
        assert np.array_equal(a1, a2) and np.array_equal(b1, b2)
        assert np.array_equal(sort_rows(cand)[0], sort_rows(cand_r)[0])
    out["n_active"], out["n_para"], out["n_cand"] = len(mm_r), len(pa_r), len(cand_r)

    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm_r, pa_r, pe_r))
    ctx.set_csr(ia, ja, 1)

    # energies
    E, Er = ctx.elastic_energy(dt2), o.energy(dt2, nth)[0]
    assert abs(E - Er) <= RTOL * abs(Er), (E, Er)
    Eb = ctx.barrier_energy(dHat, kappa)
    Ebr, bad = s.barrier_energy(mm_r, pa_r, pe_r, dHat, kappa)
    assert bad == 0 and abs(Eb - Ebr) <= RTOL * abs(Ebr), (Eb, Ebr)

    # gradients (+ property: internal forces of each kind sum to zero)
    g = ctx.elastic_gradient(dt2, 1, 1)
    g_r = o.gradient(dt2, 1, nth)
    assert rel(g, g_r) <= RTOL
    assert np.abs(g.reshape(-1, 3).sum(0)).max() <= 1e-9 * np.abs(g).max()
    gb = np.zeros(3 * m.nV)
    ctx.barrier_gradient(dHat, kappa, gb)
    gb_r = np.zeros(3 * m.nV)
    s.barrier_gradient(mm_r, pa_r, pe_r, dHat, kappa, g=gb_r)
    assert rel(gb, gb_r) <= RTOL
    assert np.abs(gb.reshape(-1, 3).sum(0)).max() <= 1e-9 * np.abs(gb).max()

    # Hessian: elastic + barrier in the solver's CSR
    a = np.zeros(ja.size)
    ctx.elastic_hessian(dt2, 1, 1, 1, a)
    ctx.barrier_hessian(dHat, kappa, 1, a)
    a_r = o.hessian_csr(dt2, ia, ja, 1, 1, 1, nthreads=nth)
    s.barrier_hessian_csr(mm_r, pa_r, pe_r, dHat, kappa, ia, ja, 1, 1, a=a_r, nthreads=nth)
    assert rel(a, a_r) <= h_tol, rel(a, a_r)

    # step bounds: inversion filter, partial CCD, swept hash, full CCD -- the step is bit-exact
    al = ctx.inversion_step(p, 0.2, 1.0)
    al_r, _ = o.inversion_step(p, 0.2, 1.0)
    assert abs(al - al_r) <= 1e-9 * al_r
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)  # computeTightInclusionError uses mesh.V only (CCDUtils.cpp:29-46)
    al = ctx.ccd_partial(p, tol, evf, eee, al_r)
    al_r, _ = orc.ccd_partial(s, p, cand_r, tol, evf, eee, al_r, nth)
    assert scalar_bits(al) == scalar_bits(al_r), (al, al_r)
    ag = ctx.hash_build_swept(p, al, hvox)
    al2, ncand = ctx.ccd_full(tol, evf, eee, ag)
    al2_r, _, npairs = orc.ccd_full_hashed(s, p, al_r, hvox, tol, evf, eee, nth)
    assert ncand == npairs and scalar_bits(al2) == scalar_bits(al2_r), (ncand, npairs, al2, al2_r)
    assert ctx.ccd_stats()[2] == 0  # no conservative early-out was needed
    assert 0.0 < al2 <= 1.0
    out["alpha"], out["n_full_cand"] = al2, int(ncand)

    # property: at 0.999 * step every sampled candidate stencil still has positive distance
    if len(cand_r):
        V2 = m.V + 0.999 * al2 * p.reshape(-1, 3)
        rng = np.random.default_rng(1)
        for c in cand_r[rng.integers(0, len(cand_r), n_prop)]:
            if c[0] < 0:
                assert orc.point_tri_d(V2[[m.SVI[-c[0] - 1]] + list(m.SF[c[1]])]) > 0
            else:
                assert orc.edge_edge_d(V2[list(m.SFEdges[c[0]]) + list(m.SFEdges[c[1]])]) > 0
    ctx.set_canonical_order(1)
    ctx.set_contact_partition(0)
    return out
