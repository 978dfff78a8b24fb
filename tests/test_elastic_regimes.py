"""The per-tet elastic path (k_elastic_energy, k_elastic_grad_hess: svd3.cuh, elastic.cuh) and the CPU oracle against
tests/golden/elastic_regimes_golden.npz: an mpmath evaluation (tests/golden/gen_elastic_regimes_golden.py) on a soup of tets whose deformation
gradients reach every exit of the 3x3 SVD, both of its sorts, repeated and nearly repeated singular values, near-singular, singular and inverted
F, large stretch, the Jacobi path of the A-block projection and the indefinite branch of the B-block projection.

The fixture is evaluated independently of any SVD code for the unprojected quantities (closed-form P, central differences); the projected Hessian
is the reference's sigma-space formula restated in mpmath.  Bars, per tet (eps = 2^-52):

* Unprojected E, g, H: 1e-12 of the per-tet scale while kappa <= 1e3.  The SVD's singular values carry an absolute error ~eps sigma_max, and
  forming F = Ds Dm^-1 in doubles an error ~eps sigma_max cond(Dm); so sigma_min (NH) or the smallest sigma_i + sigma_j (FCR, whose B blocks
  divide by it) is known to a relative eps kappa, kappa = cond(Dm) sigma_max / that quantity.  NH: P carries F^-T = cof F / J with J from the
  singular values, and dP/dF is dominated by the 1/sigma_min^2 terms of the A block whose relative error is 2 eps kappa, while E sees the same
  error in ln J; FCR: the B blocks carry (dpsi_i + dpsi_j) / (sigma_i + sigma_j).  Every quantity is therefore off by a relative c eps kappa^k with
  k = 1 (not fitted: one division by the ill-known quantity per term, and its square enters only through the 1/sigma^2 terms whose own relative
  error is again first order).  c = 512 bounds the roundings of the 3x3 chain, which reach the result both through the singular values and
  through U and V (the oracle needs c ~ 150 on an inverted tet with sigma_2 + sigma_3 = 7e-5).
* Projected H, neither near_branch nor basis-dependent: 1e-10 of the block maximum, plus the same c eps kappa, plus c eps / delta with delta the
  smallest relative gap between singular values when delta > 1e-6: the singular vectors of a pair delta apart are known to eps / delta, and
  the projection of a block that is clamped rotates with them.  Closer pairs are the fixture's basis-dependent case below.
* Basis-dependent tets (basis_spread > 0: two singular values within 1e-6 sigma_max): the projected Hessian is not a function of F there
  (DESIGN 3.4).  Checked: symmetric, smallest eigenvalue >= -1e-12 ||H||, and within basis_spread plus the bar above of the fixture.  The same
  for H and g where the 1e-6 floor makes them basis-dependent (basis_spread_H, basis_spread_g).
* near_branch tets (a projection switches branches within 1e-9 of the switch): PSD and symmetric only.
"""
import importlib.util
import os

import numpy as np
import pytest

import oracle as orc
from gpu_common import shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "elastic_regimes_golden.npz")
EPS = np.finfo(float).eps
C_ROUND = 512.0  # roundings in the 3x3 chain (see the module docstring)
TIGHT = 1e-12    # unprojected E, g, H while kappa <= KAPPA_TIGHT
KAPPA_TIGHT = 1e3
PROJ = 1e-10     # projected H, away from branches and basis dependence
PSD = 1e-12      # smallest eigenvalue of a projected H, relative to ||H||
DEGENERATE = 1e-6  # relative gap below which the fixture evaluates other SVD bases


def gold():
    return dict(np.load(GOLD))


def gen_module():
    spec = importlib.util.spec_from_file_location("gen_elastic_regimes_golden", os.path.join(HERE, "golden", "gen_elastic_regimes_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def subset(z, et, order=None):
    """the soup's tets of one energy type (optionally reordered) as a Mesh with the stored inputs; vertex ids follow the tets"""
    idx = np.flatnonzero(z["energy"] == et)
    if order is not None:
        idx = idx[order]
    n = idx.size
    T0 = z["T"][idx]
    T = (4 * np.arange(n)[:, None] + (T0 - 4 * idx[:, None])).astype(np.int32)  # keep each tet's internal vertex permutation
    V, Vr = np.empty((4 * n, 3)), np.empty((4 * n, 3))
    V[T.ravel()] = z["V"][T0.ravel()]
    Vr[T.ravel()] = z["V_rest"][T0.ravel()]
    m = M.Mesh(Vr, T, energy=et)
    m.V = V
    m.restTriInv, m.vol, m.mu, m.lam = (np.ascontiguousarray(z[k][idx]) for k in ("restTriInv", "vol", "mu", "lam"))
    return idx, m


def bars(z, idx):
    """per-tet scales and bars (module docstring)"""
    S = np.abs(z["sigma"][idx])
    sig = z["sigma"][idx]
    et = z["energy"][idx]
    A = z["restTriInv"][idx].reshape(-1, 3, 3)  # (column-major storage: A[t] is Dm^-T, same 2-norm condition)
    cond = np.linalg.cond(A)
    smax = S.max(1)
    pair = np.minimum.reduce([sig[:, 0] + sig[:, 1], sig[:, 1] + sig[:, 2], sig[:, 0] + sig[:, 2]])
    ill = np.where(et == 0, S.min(1), np.maximum(pair, 1e-6))
    with np.errstate(divide="ignore"):
        kappa = np.where(smax > 0, cond * smax / np.maximum(ill, 1e-300), 1.0)
        gaps = np.array([min(abs(s[0] - s[1]), abs(s[1] - s[2]), abs(s[0] - s[2])) for s in sig]) / np.maximum(smax, 1e-300)
    unit = z["vol"][idx] * (z["mu"][idx] + z["lam"][idx])
    gmax = np.abs(np.concatenate([-A.sum(1, keepdims=True), A], 1)).max((1, 2))
    sc = {"E": np.maximum(np.abs(z["E"][idx]), unit), "g": np.maximum(np.abs(z["g"][idx]).max(1), unit * gmax),
          "H": np.maximum(np.abs(z["H"][idx]).max((1, 2)), unit * gmax ** 2), "Hp": np.abs(z["Hp"][idx]).max((1, 2))}
    unproj = np.where(kappa <= KAPPA_TIGHT, TIGHT, np.maximum(TIGHT, C_ROUND * EPS * kappa))
    # the eps / delta term where the pair is resolved; below the fixture's degeneracy threshold basis_spread measures the dependence itself
    with np.errstate(divide="ignore"):
        proj = PROJ + C_ROUND * EPS * kappa + np.where(gaps > DEGENERATE, C_ROUND * EPS / np.maximum(gaps, DEGENERATE), 0.0)
    return sc, unproj, proj, kappa


def check(z, idx, E, g, H, Hp, who):
    """E (n,), g (n,12), H and Hp (n,12,12) of the tets idx against the fixture; returns the worst error / bar per family and kind"""
    sc, unproj, proj, kappa = bars(z, idx)
    fam = z["families"][z["family"][idx]]
    worst = {}

    def note(kind, t, err, bar):
        key = (str(fam[t]), kind)
        r = err / bar if bar > 0 else (0.0 if err == 0 else np.inf)
        worst[key] = max(worst.get(key, 0.0), r)
        assert err <= bar, f"{who}: tet {idx[t]} ({fam[t]}, energy {z['energy'][idx[t]]}, sigma {z['sigma'][idx[t]]}, kappa {kappa[t]:.2e}) {kind}: " \
                           f"error {err:.3e} > bar {bar:.3e}"

    for t, k in enumerate(idx):
        note("E", t, abs(E[t] - z["E"][k]), unproj[t] * sc["E"][t])
        note("g", t, np.abs(g[t] - z["g"][k]).max(), z["basis_spread_g"][k] + unproj[t] * sc["g"][t])
        note("H", t, np.abs(H[t] - z["H"][k]).max(), z["basis_spread_H"][k] + unproj[t] * sc["H"][t])
        h = Hp[t]
        hn = np.linalg.norm(h, 2)
        note("Hp symmetric", t, np.abs(h - h.T).max(), 1e-15 * max(hn, 1e-300))
        note("Hp PSD", t, max(0.0, -np.linalg.eigvalsh(0.5 * (h + h.T)).min()), PSD * hn)
        if not z["near_branch"][k]:
            note("Hp", t, np.abs(h - z["Hp"][k]).max(), z["basis_spread"][k] + proj[t] * sc["Hp"][t])
    return worst


def fixture_counts(z):
    return {"tets": int(z["E"].size), "NH": int((z["energy"] == 0).sum()), "FCR": int((z["energy"] == 1).sum()),
            "basis_spread": int((z["basis_spread"] > 0).sum()), "near_branch": int(z["near_branch"].sum()),
            "floor_active": int(z["floor_active"].sum()), "a_indef": int(z["a_indef"].sum())}


# ---------------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------------
def test_fixture_shape():
    """both soups span several 64-tet tiles and end in a partial one; every family sits at more than one tile position"""
    z = gold()
    c = fixture_counts(z)
    for et in (0, 1):
        n = int((z["energy"] == et).sum())
        assert n > 64 and n % 64 != 0, n
        idx = np.flatnonzero(z["energy"] == et)
        for f in np.unique(z["family"][idx]):
            pos = np.flatnonzero(z["family"][idx] == f)
            assert len(pos) < 2 or len(np.unique(pos // 64)) > 1 or len(np.unique(pos % 64)) > 1
    # the regimes the fixture exists for are present
    assert c["basis_spread"] > 0 and c["near_branch"] > 0 and c["floor_active"] > 0
    assert z["a_indef"][z["energy"] == 0].sum() > 0 and z["a_indef"][z["energy"] == 1].sum() > 0  # the Jacobi path, both energies
    assert (z["mu"][z["energy"] == 0] == 0).any()


@pytest.mark.parametrize("et", [0, 1])
def test_oracle_matches_fixture(et):
    z = gold()
    idx, m = subset(z, et)
    o = orc.Elastic(m)
    _, E = o.energy(1.0)
    g = o.gradient(1.0, 0).reshape(-1, 3)[m.T].reshape(-1, 12)  # a soup: every vertex belongs to one tet
    H = o.hessian_blocks(1.0, 0)
    Hp = o.hessian_blocks(1.0, 1)
    check(z, idx, E, g, H, Hp, "oracle")


def test_svd_branch_coverage():
    """the restated SVD leaves through all five exits and takes both branches of both sorts on the fixture's deformation gradients (formed the
    way the oracle forms them); the kernels follow the same statements"""
    z = gold()
    seen = {}
    for t in range(z["E"].size):
        x = z["V"][z["T"][t]]
        A = z["restTriInv"][t].reshape(3, 3).T
        Ds = (x[1:] - x[0]).T
        F = Ds @ A
        seen.setdefault(orc.svd3_branch(F), []).append(t)
    exits = {k[0] for k in seen}
    sorts = {(k[1], k[2]) for k in seen}
    table = "\n".join(f"  exit {k[0]:8s} sort{k[1]} {'reordered' if k[2] else 'early return':12s}: {len(v)} tets" for k, v in sorted(seen.items()))
    print("svd3 branches taken by the fixture:\n" + table)
    assert exits == set(orc.SVD3_EXITS), table
    assert sorts == {(0, False), (0, True), (1, False), (1, True)}, table


def test_generator_reproduces_the_fixture():
    """the script rebuilds the stored inputs bit for bit and, re-run on the first tets, the stored reference values"""
    pytest.importorskip("mpmath")
    z = gold()
    gen = gen_module()
    V, Vr, T, Ainv, vol, mu, lam, et, fam = gen.soup(gen.cases())
    for k, a in dict(V=V, V_rest=Vr, T=T, restTriInv=Ainv, vol=vol, mu=mu, lam=lam, energy=et, family=fam).items():
        assert np.array_equal(z[k], a), k
    picks = list(range(4)) + [int(np.flatnonzero(z["floor_active"])[0]), int(np.flatnonzero(z["basis_spread"] > 0)[0])]
    for t in picks:
        r = gen.evaluate(et[t], mu[t], lam[t], V[T[t]], Ainv[t], vol[t])
        for k, v in r.items():
            np.testing.assert_allclose(np.asarray(v, dtype=float), z[k][t], rtol=1e-14, atol=0, err_msg=f"tet {t} {k}")


# ---------------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------------
def run_gpu(ctx, m):
    """per-tet E (k_elastic_energy), g, H and projected H (k_elastic_grad_hess) of a soup, the CSR values, and the fused energy"""
    n = m.nT
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, None, None, m.energy)
    ia, ja = m.csr_pattern(1)
    ctx.set_csr(ia, ja, 1)
    ctx.set_state(m.V_soa)
    out = {"E_sum": ctx.elastic_energy(1.0), "E": ctx.download(L.BUF_ENERGY_PER_TET, n)}
    ctx.elastic_gradient(1.0, 1, 0)
    out["g"] = ctx.download(L.BUF_TET_GRADIENTS, 12 * n).reshape(n, 12)
    for key, spd in (("H", 0), ("Hp", 1)):
        a = np.zeros(ja.size)
        ctx.elastic_hessian(1.0, 1, spd, 0, a)
        out[key + "78"] = L.untile_hessians(ctx.download(L.BUF_TET_HESSIANS, 78 * 64 * ((n + 63) // 64)), n)
        out[key] = np.array([orc.blocks78_to_dense(out[key + "78"][t], m.T[t]) for t in range(n)])
        out[key + "_csr"] = a
    g1, a1 = np.empty(3 * m.nV), np.empty(ja.size)
    out["E_fused"] = ctx.elastic_energy_grad_hess(1.0, 1, 0, 0, g1, a1, want_energy=True)
    out["ia"], out["ja"] = ia, ja
    return out


def csr_of_blocks(m, H, ia, ja):
    """upper-triangular CSR values (index base 1) of the sum of per-tet 12x12 blocks"""
    a = np.zeros(ja.size)
    for t in range(m.nT):
        for p in range(4):
            for q in range(4):
                vp, vq = m.T[t, p], m.T[t, q]
                for r in range(3):
                    row = 3 * vp + r
                    cols = ja[ia[row] - 1:ia[row + 1] - 1] - 1
                    for c in range(3):
                        col = 3 * vq + c
                        if row <= col:
                            a[ia[row] - 1 + np.searchsorted(cols, col)] += H[t, 3 * p + r, 3 * q + c]
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("et", [0, 1])
def test_kernels_match_fixture(shared_ctx, et):
    z = gold()
    idx, m = subset(z, et)
    out = run_gpu(shared_ctx, m)
    worst = check(z, idx, out["E"], out["g"], out["H"], out["Hp"], "gpu")
    print(f"energy {et}: {fixture_counts(z)}; worst error / bar per family:")
    for (f, kind), r in sorted(worst.items()):
        print(f"  {f:14s} {kind:13s} {r:.3e}")
    # the energy kernel (svd3<false>) and the energy fused into the gradient/Hessian kernel (svd3<true>) agree; their sums differ only in order
    sc, _, _, _ = bars(z, idx)
    assert abs(out["E_fused"] - out["E_sum"]) <= 1e-14 * np.abs(out["E"]).sum() + TIGHT * sc["E"].max()
    assert abs(out["E_sum"] - z["E"][idx].sum()) <= 1e-14 * np.abs(z["E"][idx]).sum() + (bars(z, idx)[1] * sc["E"]).sum()
    # one contribution per CSR entry (the tets share no vertex): the assembly is exact, and the unprojected one is the fixture's sum within
    # the per-tet bars
    for key in ("H", "Hp"):
        assert np.array_equal(out[key + "_csr"], csr_of_blocks(m, out[key], out["ia"], out["ja"])), key
    _, unproj, _, _ = bars(z, idx)
    bar = np.broadcast_to((z["basis_spread_H"][idx] + unproj * sc["H"])[:, None, None], (m.nT, 12, 12))
    a_ref = csr_of_blocks(m, z["H"][idx], out["ia"], out["ja"])
    assert np.all(np.abs(out["H_csr"] - a_ref) <= csr_of_blocks(m, bar, out["ia"], out["ja"]))


@pytest.mark.gpu
@pytest.mark.parametrize("et", [0, 1])
def test_tile_slot_does_not_change_a_tet(shared_ctx, et):
    """the same soup uploaded in an order that moves every tet to another slot of its 64-tet tile gives bit-identical per-tet results"""
    z = gold()
    n = int((z["energy"] == et).sum())
    order = None
    j = np.arange(n)
    for cand in [(s - j) % n for s in range(n)] + [(j + s) % n for s in range(1, n)]:  # reversed or rotated, shifted
        if np.all(cand % 64 != j % 64):
            order = cand
            break
    assert order is not None and np.array_equal(np.sort(order), np.arange(n))
    _, m0 = subset(z, et)
    a = run_gpu(shared_ctx, m0)
    _, m1 = subset(z, et, order)
    b = run_gpu(shared_ctx, m1)
    for k in ("E", "g", "H78", "Hp78"):
        assert np.array_equal(a[k][order], b[k]), k
