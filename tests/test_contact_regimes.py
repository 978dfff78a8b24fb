"""The per-pair contact math (contact.cuh, barrier.cu, friction.cu) and the CPU oracle (oracle/contact.cpp, oracle/friction.cpp) against
tests/golden/contact_regimes_golden.npz: an mpmath evaluation (tests/golden/gen_contact_regimes_golden.py) on a soup of disjoint stencils at
d/dHat from 1e-12 to 1 - 1e-10 over four dHat decades, multiplicities, sizes 1e-4 .. 1e2 at offsets up to 1e3, slivers, near-parallel and
exactly parallel edges on both sides of the mollifier switch and the PP friction-basis tie.  The fixture's derivatives come from the
definitions of the distances (sympy), not from the difference-space derivation the kernels and the oracle share.

Error model (eps = 2^-52).  Every quantity Q of a pair (d, E, g, H; friction lambda, coordinates, basis, E, g, H) is held to

    |Q - Q_ref| <= C eps S_Q + TAU scale_Q         (componentwise)

S_Q = sum_i |dQ/dx_i| |x_i| is the fixture's first-order sensitivity to the stored inputs (coordinates, dHat, kappa, rest coordinates of a
mollified pair; friction: also V_prev, the lagged data and eps2), plus its sensitivity to the roundings of the cross products (of d, of c
and of the lag's basis) and of the lag's 2x2 Gram system, each at the size of that rounding: a rounded cross-product component tilts the
normal of a sliver triangle or of nearly parallel edges in a direction no input perturbation reaches (without these terms the oracle misses
the bar by 3.5x on the 1e-4 sliver PT pair).  A rounding of relative size u in any other intermediate that the arithmetic
computes from the inputs moves Q by at most the same amount as a relative input perturbation u applied to every input it depends on, to
first order and times the path's amplification; the longest chains (the Hessian of the line-line distance: difference vectors, a cross
product, s = m.n, N = s^2, L = |n|^2, N/L, its gradient and Hessian, b'' and b', their products) have about 30 roundings on any path and
amplify by at most two, so C = 64 with a factor of two to spare.  TAU = 1e-13 of the pair's own largest entry (scale_Q, not the matrix
maximum) covers roundings the input sensitivity does not see: sums of terms that cancel for every input (translation invariance, the zero
rows of H) and the structure of b'' grad d grad d^T + b' H_d, whose two terms are each rounded before they are added.

Projected Hessians.  The PSD projection is 1-Lipschitz in the Frobenius norm, so ||Hp - Hp_ref||_F <= ||bar_H||_F + TAU_J ||H_ref||_F, with
bar_H the componentwise bar of H above and TAU_J = 1e-12 the Jacobi stopping rule (off^2 <= 2e-26 diag^2) and its rotations.  No exclusion
near a branch is needed; a mollified pair within 1e-8 of c = eps_x, or within the rounding of c / eps_x in doubles (64 eps times its
sensitivity, up to 1e-6 on edges 1e-9 rad from parallel), accepts either side of the switch.  Every projected block is PSD (smallest
eigenvalue >= -1e-12 ||H||); the oracle's blocks, which hold both triangles, are also symmetric (a block read back from the CSR's upper
triangle is symmetric by construction).  Blocks that are exactly zero (d == dHat, family early_return) take makePD's early return in any
rounding and must come back exactly zero; the e = 0 blocks of exactly parallel edges are PSD only in exact arithmetic, and are held to
the same Frobenius bar whichever path the rounding sends them down.

Friction: the lag (lambda, coordinates, basis) is checked with the bars above against the exact lag, except the basis of a near_branch PP
pair (within 1e-9 of the tie, where the basis is discontinuous).  E, g, H are checked on the fixture's lagged data (S_f*) and on the
device-lagged data (S_f* + S_f*_lag, the sensitivity with the lag recomputed from V).
"""
import importlib.util
import os

import numpy as np
import pytest
import scipy.sparse as sps

import oracle as orc
import refpairs
from gpu_common import load_scene, shared_ctx
from ipc_b200 import mesh as M
from test_elastic_regimes import csr_of_blocks

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "contact_regimes_golden.npz")
EPS = np.finfo(float).eps
C_ROUND = 64.0   # roundings on a path through the pair arithmetic (module docstring)
TAU = 1e-13      # of the pair's own largest entry
TAU_J = 1e-12    # Jacobi stopping rule, relative to ||H||_F
PSD = 1e-12      # smallest eigenvalue of a projected block, relative to ||H||_2
KINDS = ("PT", "EE", "PE", "PP")
C_REF = 64.0     # the reference's own codegen (refpairs) against the fixture, same form of bar (test_reference_codegen_matches_fixture)


def gold():
    return dict(np.load(GOLD))


def gen_module():
    spec = importlib.util.spec_from_file_location("gen_contact_regimes_golden", os.path.join(HERE, "golden", "gen_contact_regimes_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def soup_mesh(z):
    m = M.Mesh(z["V_rest"], z["T"])
    m.mu[:] = 0.0
    m.lam[:] = 0.0
    m.V = z["V"].copy()
    return m


def groups(z, idx):
    """pairs of idx by (dHat, kappa): one kernel call each"""
    key = {}
    for k in idx:
        key.setdefault((float(z["dHat"][k]), float(z["kappa"][k])), []).append(int(k))
    return key


def lists(z, ks):
    ks = np.asarray(ks, dtype=int)
    a, p = ks[~z["moll"][ks]], ks[z["moll"][ks]]
    return a, p, z["mm"][a], z["mm"][p], z["pe"][p]


def blocks_of_csr(a, ia, ja, nV, T):
    """per-tet 12x12 blocks (tet vertex order) of the symmetric matrix whose upper triangle a holds"""
    U = sps.csr_matrix((a, ja - 1, ia - 1), shape=(3 * nV, 3 * nV))
    S = (U + sps.triu(U, 1).T).tocsr()
    out = np.empty((len(T), 12, 12))
    for k, t in enumerate(T):
        r = (3 * t[:, None] + np.arange(3)[None, :]).ravel()
        out[k] = S[r][:, r].toarray()
    return out


def bar(S, scale):
    return C_ROUND * EPS * np.asarray(S, dtype=float) + TAU * scale


class Report:
    """worst error / bar per (family, quantity); assert on every check"""

    def __init__(self, z, who):
        self.z, self.who, self.worst = z, who, {}

    def note(self, k, q, err, b):
        err, b = np.asarray(err, dtype=float), np.asarray(b, dtype=float)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(b > 0, err / b, np.where(err == 0, 0.0, np.inf))
        key = (str(self.z["families"][self.z["family"][k]]), q)
        self.worst[key] = max(self.worst.get(key, 0.0), float(r.max()))
        assert np.all(err <= b), f"{self.who}: pair {k} ({key[0]}, {KINDS[self.z['kind'][k]]}, moll {self.z['moll'][k]}, dHat {self.z['dHat'][k]:.1e}, " \
                                 f"kappa {self.z['kappa'][k]:.0e}) {q}: error {err.max():.3e} vs bar {b.ravel()[np.argmax(r)]:.3e}, ratio {r.max():.3e}"

    def scalar(self, k, q, val, ref, S):
        self.note(k, q, abs(val - ref), bar(S, abs(ref)))

    def array(self, k, q, val, ref, S):
        self.note(k, q, np.abs(val - ref), bar(S, np.abs(ref).max()))

    def projected(self, k, q, Hp, refs, H_ref, S_H, full=True):
        """Frobenius bar of the projection; refs: the admissible projected references (both sides at a mollifier switch).  full: Hp holds
        both triangles as computed (the oracle's pair blocks); a block rebuilt from the CSR's upper triangle is symmetric by construction"""
        hb = np.linalg.norm(bar(S_H, np.abs(H_ref).max())) + TAU_J * np.linalg.norm(H_ref)
        self.note(k, q, min(np.linalg.norm(Hp - r) for r in refs), hb)
        hn = max(np.linalg.norm(H_ref, 2), np.linalg.norm(Hp, 2))
        if full:
            self.note(k, q + " symmetric", np.abs(Hp - Hp.T).max(), 1e-15 * hn)
        self.note(k, q + " PSD", max(0.0, -np.linalg.eigvalsh(0.5 * (Hp + Hp.T)).min()), PSD * hn)

    def table(self, title):
        print(f"{title}; worst error / bar per family:")
        for (f, q), r in sorted(self.worst.items()):
            print(f"  {f:14s} {q:22s} {r:.3e}")


def check_barrier(rep, z, k, d, E, g, Hp, full=False):
    if d is not None:
        rep.scalar(k, "d", d, z["d"][k], z["S_d"][k])
    if E is not None:
        rep.scalar(k, "E", E, z["E"][k], z["S_E"][k])
    if g is not None:
        rep.array(k, "g", g, z["g"][k], z["S_g"][k])
    refs = [z["Hp"][k]] + ([z["Hp_alt"][k]] if z["switch"][k] else [])
    H_ref = z["H"][k] if not z["switch"][k] else np.where(np.abs(z["H"][k]) >= np.abs(z["H_alt"][k]), z["H"][k], z["H_alt"][k])
    rep.projected(k, "Hp", Hp, refs, H_ref, z["S_H"][k], full)


def check_lag(rep, z, k, lam, co, ba):
    rep.scalar(k, "lambda", lam, z["lam_ref"][k], z["S_lam"][k])
    rep.array(k, "coord", co, z["coord_ref"][k], z["S_coord"][k])
    if not z["near_branch"][k]:
        rep.note(k, "basis", np.abs(ba - z["basis_ref"][k]), bar(z["S_basis"][k], 1.0))
    else:  # the tie: any orthonormal pair in the tangent plane, i.e. across the contact normal v01
        B = ba.reshape(2, 3)
        x = z["V"][z["T"][k]]
        v01 = x[1] - x[0]
        rep.note(k, "basis (near_branch)", np.abs(B @ B.T - np.eye(2)), np.full((2, 2), 1e-15))
        rep.note(k, "basis (near_branch) tangent", np.abs(B @ v01), np.full(2, C_ROUND * EPS * np.linalg.norm(v01)))


def check_friction(rep, z, k, E, g, H, lagged_on_device, full=False):
    S = {q: z["S_f" + q][k] + (z["S_f" + q + "_lag"][k] if lagged_on_device else 0) for q in ("E", "g", "H")}
    tag = " (device lag)" if lagged_on_device else ""
    rep.scalar(k, "fE" + tag, E, z["fE"][k], S["E"])
    rep.array(k, "fg" + tag, g, z["fg"][k], S["g"])
    rep.projected(k, "fHp" + tag, H, [z["fHp"][k]], z["fH"][k], S["H"], full)


def fixture_counts(z):
    fr = z["fric"]
    c = {"pairs": int(z["E"].size), "mollified": int(z["moll"].sum()), "friction": int(fr.sum())}
    for i, kn in enumerate(KINDS):
        c[kn] = int(((z["kind"] == i) & ~z["moll"]).sum())
        c[kn + " mollified"] = int(((z["kind"] == i) & z["moll"]).sum())
    c.update({"mollifier below": int((z["moll"] & (z["c_ratio"] < 1)).sum()), "mollifier above": int((z["moll"] & (z["c_ratio"] >= 1)).sum()),
              "switch": int(z["switch"].sum()), "early return": int(z["psd"].sum()), "clamped": int((~z["psd"]).sum()),
              "sticking": int((fr & (z["u_ratio"] <= 1)).sum()), "sliding": int((fr & (z["u_ratio"] > 1)).sum()),
              "u = 0": int((fr & (z["u_ratio"] == 0)).sum()), "near_branch": int(z["near_branch"].sum())})
    return c


# ---------------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------------
def test_fixture_coverage():
    z = gold()
    c = fixture_counts(z)
    print(c)
    fam = z["families"]
    need = {"sweep": (0, 1, 2, 3), "multiplicity": (2, 3), "scale": (0, 1, 2, 3), "sliver": (0, 1, 2), "near_parallel": (1,),
            "parallel": (2, 3), "pp_tie": (3,)}
    for f, kinds in need.items():
        fi = list(fam).index(f)
        for kd in kinds:
            assert ((z["family"] == fi) & (z["kind"] == kd)).any(), (f, KINDS[kd])
    # multiplicities 1, 2 and >= 3 of PP and PE
    w = -z["mm"][:, 3]
    for kd in (2, 3):
        sel = (z["kind"] == kd) & ~z["moll"]
        assert {1, 2} <= set(w[sel]) and (w[sel] >= 3).any()
    # both sides of the mollifier switch, pairs at it, exactly parallel edges (e = 0), sentinel encodings of both kinds
    cr = z["c_ratio"][z["moll"]]
    assert (cr < 1).any() and (cr >= 1).any() and z["switch"].any() and (cr == 0).any()
    assert ((z["pe"][:, 0] >= 0) & (z["kind"] == 3)).any() and ((z["pe"][:, 0] >= 0) & (z["kind"] == 2)).any()
    # both makePD outcomes.  The early return is deterministic in doubles only on an exactly zero block (d == dHat: b = b' = b'' = 0 for
    # every evaluation order), which every stencil kind provides; the oracle's makePD hands those blocks back untouched
    assert c["early return"] > 0 and c["clamped"] > 0
    er = np.flatnonzero(z["family"] == list(fam).index("early_return"))
    assert set(z["kind"][er]) == {0, 1, 2, 3}
    for k in er:
        assert z["psd"][k] and not np.any(z["H"][k]) and z["d"][k] == z["dHat"][k]
        assert np.array_equal(orc.makePD(z["H"][k]), z["H"][k])
    # friction: both clamp branches, |u| = 0, both PP basis branches and a near tie
    assert c["sticking"] > 0 and c["sliding"] > 0 and c["u = 0"] > 0
    assert {0, 1} <= set(z["pp_branch"][z["fric"] & (z["kind"] == 3)]) and c["near_branch"] > 0
    # the near-parallel EE stencils span 1e-2 .. 1e-18 and stay above the classification guard
    x = z["V"][z["T"]]
    sel = z["family"] == list(fam).index("near_parallel")
    a, b = x[sel, 1] - x[sel, 0], x[sel, 3] - x[sel, 2]
    par = np.sum(np.cross(a, b) ** 2, 1) / (np.sum(a * a, 1) * np.sum(b * b, 1))
    assert par.min() < 1e-17 and par.max() > 1e-3 and par.min() > 1e-20
    assert 250 <= c["pairs"] <= 400 and os.path.getsize(GOLD) < 1.5e6


def test_generator_reproduces_the_fixture():
    """the script rebuilds the stored inputs bit for bit and, re-run on a handful of pairs (a mollified one and friction pairs
    among them), the stored reference values"""
    pytest.importorskip("mpmath")
    pytest.importorskip("sympy")
    z = gold()
    gen = gen_module()
    cs = gen.cases()
    s = gen.soup(cs)
    for k, a in s.items():
        assert np.array_equal(z[k], a), k
    lam, co, ba, Vp, eps2 = gen.friction_inputs(cs, s)
    for k, a in dict(lam=lam, coord=co, basis=ba, V_prev=Vp, eps2=eps2).items():
        assert np.array_equal(z[k], a), k
    kinds = z["kind"]
    picks = [int(np.flatnonzero(z["fric"] & (kinds == 3))[0]), int(np.flatnonzero(z["fric"] & (kinds == 2))[0]),
             int(np.flatnonzero(z["moll"] & (kinds == 3))[-1]), int(np.flatnonzero(z["pp_branch"] == 0)[0])]
    for k in picks:
        c = cs[k]
        fr = bool(z["fric"][k])
        r = gen.evaluate(c, z["V"][4 * k:4 * k + 4], z["V_rest"][4 * k:4 * k + 4], z["dHat"][k], z["kappa"][k],
                         z["V_prev"][4 * k:4 * k + 4] if fr else None, z["eps2"][k], (z["lam"][k], z["coord"][k], z["basis"][k]) if fr else None,
                         sens=False)
        for q, v in r.items():
            np.testing.assert_allclose(np.asarray(v, dtype=float), z[q][k], rtol=1e-14, atol=0, err_msg=f"pair {k} {q}")


def test_oracle_matches_fixture():
    z = gold()
    m = soup_mesh(z)
    s = orc.Surf(m)
    rep = Report(z, "oracle")
    ia, ja = m.csr_pattern(1)
    x = z["V"][z["T"]]
    for (dHat, kappa), ks in groups(z, range(z["E"].size)).items():
        a_idx, p_idx, mm, pa, pe = lists(z, ks)
        g = s.barrier_gradient(mm, pa, pe, dHat, kappa)
        Hb = blocks_of_csr(s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1), ia, ja, m.nV, m.T[ks])
        for j, k in enumerate(ks):
            sv = z["mm"][k]
            one = (sv[None], pa[:0], pe[:0]) if not z["moll"][k] else (mm[:0], sv[None], z["pe"][k][None])
            E, bad = s.barrier_energy(*one, dHat, kappa)
            assert bad == 0
            kd = z["kind"][k]
            nv = (4, 4, 3, 2)[kd]
            loc = [0, 1, 2, 3][:nv] if not (z["moll"][k] and z["pe"][k][0] >= 0) else None
            d = orc.d_pair(KINDS[kd], x[k][loc].ravel()) if loc is not None else None
            check_barrier(rep, z, k, d, E, g.reshape(-1, 3)[m.T[k]].ravel(), Hb[j])
            if z["family"][k] == list(z["families"]).index("early_return"):
                assert not np.any(Hb[j]) and E == 0 and not np.any(g.reshape(-1, 3)[m.T[k]])
    fr = np.flatnonzero(z["fric"])
    Vt = z["V_prev"]
    for (dHat, kappa), ks in groups(z, fr).items():
        mm = z["mm"][ks]
        lam, co, ba = s.friction_lag(mm, dHat, kappa)
        for j, k in enumerate(ks):
            check_lag(rep, z, k, lam[j], co[j], ba[j])
            for dev, data in ((False, (z["lam"][k], z["coord"][k], z["basis"][k])), (True, (lam[j], co[j], ba[j]))):
                if dev and z["near_branch"][k]:
                    continue
                args = (Vt, mm[j:j + 1], np.atleast_1d(data[0]), data[1][None], data[2][None], z["eps2"][k], float(z["coef"]))
                E = s.friction_energy(*args)
                g = s.friction_gradient(*args).reshape(-1, 3)[m.T[k]].ravel()
                H, nv = s.friction_pair_hessian(Vt, mm[j], data[0], data[1], data[2], z["eps2"][k], float(z["coef"]))
                check_friction(rep, z, k, E, g, H, dev, full=True)
    rep.table(f"oracle: {fixture_counts(z)}")


@pytest.mark.skipif(not refpairs.available(), reason="oracle/_ref/libref_pairs.so is not built (no reference checkout)")
def test_reference_codegen_matches_fixture():
    """the reference's own codegen (MeshCollisionUtils.hpp g/H of PT, EE, PE and of the EE cross norm, BarrierFunctions b_C2, compute_q),
    composed by the chain rule, against the fixture's E, g and unprojected H with bars C_REF eps S_Q + TAU scale_Q: how far the reference
    itself is from exact in these regimes.  The squared distance comes from the oracle (which matches the reference's to the last bit)."""
    z = gold()
    rep = Report(z, "reference codegen")
    x = z["V"][z["T"]]
    X = z["V_rest"][z["T"]]
    fn = {0: (refpairs.g_PT, refpairs.H_PT), 1: (refpairs.g_EE, refpairs.H_EE), 2: (refpairs.g_PE, refpairs.H_PE)}
    global C_ROUND
    saved, C_ROUND = C_ROUND, C_REF
    try:
        for k in range(z["E"].size):
            kd = int(z["kind"][k])
            if kd == 3 or (z["moll"][k] and z["pe"][k][0] >= 0):
                continue  # PP has no codegen; the sentinel encodings embed PP / PE stencils in the edge stencil
            nv = (4, 4, 3)[kd]
            v = x[k][:nv].ravel()
            dist = orc.d_pair(KINDS[kd], v)
            b, db, d2b = refpairs.barrier(dist, z["dHat"][k])
            gd = np.zeros(12)
            Hd = np.zeros((12, 12))
            gd[:3 * nv] = fn[kd][0](v)
            Hd[:3 * nv, :3 * nv] = fn[kd][1](v)
            kap = z["kappa"][k]
            if not z["moll"][k]:
                mult = float(-z["mm"][k][3]) if kd == 2 else 1.0
                E, g, H = kap * mult * b, kap * mult * db * gd, kap * mult * (d2b * np.outer(gd, gd) + db * Hd)
            else:
                c = float(np.sum(np.cross(x[k][1] - x[k][0], x[k][3] - x[k][2]) ** 2))
                eps_x = 1.0e-3 * np.sum((X[k][1] - X[k][0]) ** 2) * np.sum((X[k][3] - X[k][2]) ** 2)
                e, de, d2e = refpairs.q(c, eps_x)
                if not c < eps_x:
                    e, de, d2e = 1.0, 0.0, 0.0
                gc, Hc = refpairs.EEcross_g(x[k].ravel()), refpairs.EEcross_H(x[k].ravel())
                E = kap * e * b
                g = kap * (b * de * gc + e * db * gd)
                H = kap * (b * (d2e * np.outer(gc, gc) + de * Hc) + db * de * (np.outer(gd, gc) + np.outer(gc, gd)) + e * (d2b * np.outer(gd, gd) + db * Hd))
            rep.scalar(k, "E", E, z["E"][k], z["S_E"][k])
            rep.array(k, "g", g, z["g"][k], z["S_g"][k])
            H_ref = z["H"][k] if not z["switch"][k] else None
            if H_ref is not None:
                rep.array(k, "H", H, H_ref, z["S_H"][k])
    finally:
        C_ROUND = saved
    rep.table("reference codegen")


# ---------------------------------------------------------------------------------------------------------------------------------------
# GPU (through the C ABI only)
# ---------------------------------------------------------------------------------------------------------------------------------------
def gpu_hessian(ctx, m, ia, ja, mm, pa, pe, dHat, kappa):
    ctx.set_constraint_set(mm, pa, pe)
    a = np.zeros(ja.size)
    ctx.barrier_hessian(dHat, kappa, 1, a)
    return a


@pytest.mark.gpu
def test_barrier_kernels_match_fixture(shared_ctx):
    z = gold()
    m = soup_mesh(z)
    load_scene(shared_ctx, m, mass=False, dbc=False)
    ia, ja = m.csr_pattern(1)
    shared_ctx.set_csr(ia, ja, 1)
    rep = Report(z, "gpu")
    n = z["E"].size
    for (dHat, kappa), ks in groups(z, range(n)).items():
        a_idx, p_idx, mm, pa, pe = lists(z, ks)
        # d of every pair (the mollified pairs' encodings are valid active encodings of the same distance)
        shared_ctx.set_constraint_set(np.concatenate([mm, pa]), pa[:0], pe[:0])
        d = dict(zip(np.concatenate([a_idx, p_idx]), shared_ctx.evaluate_constraints(len(ks))))
        # energy one pair at a time, and of the whole group
        E = {}
        for k in ks:
            one = (z["mm"][k][None], pa[:0], pe[:0]) if not z["moll"][k] else (mm[:0], z["mm"][k][None], z["pe"][k][None])
            shared_ctx.set_constraint_set(*one)
            E[k] = shared_ctx.barrier_energy(dHat, kappa)
        shared_ctx.set_constraint_set(mm, pa, pe)
        E_sum = shared_ctx.barrier_energy(dHat, kappa)
        tot = sum(abs(v) for v in E.values())
        assert abs(E_sum - sum(E.values())) <= 4 * len(ks) * EPS * tot, (dHat, kappa)
        g = shared_ctx.barrier_gradient(dHat, kappa, np.zeros(3 * m.nV)).reshape(-1, 3)
        a = gpu_hessian(shared_ctx, m, ia, ja, mm, pa, pe, dHat, kappa)
        Hb = blocks_of_csr(a, ia, ja, m.nV, m.T)
        # one contribution per CSR entry: the group's blocks rebuild the CSR exactly, nothing lands outside them
        only = np.zeros((n, 12, 12))
        only[ks] = Hb[ks]
        assert np.array_equal(a, csr_of_blocks(m, only, ia, ja)), (dHat, kappa)
        for k in ks:
            check_barrier(rep, z, k, d[k], E[k], g[m.T[k]].ravel(), Hb[k])
            if z["family"][k] == list(z["families"]).index("early_return"):  # makePD returned the (zero) raw block
                assert not np.any(Hb[k]) and E[k] == 0 and not np.any(g[m.T[k]])
    rep.table(f"gpu barrier: {fixture_counts(z)}")


def rotations(n):
    """list orders that move every pair through each of the six group positions of a projection warp and into other warps"""
    return [np.roll(np.arange(n), r) for r in (0, 1, 2, 3, 4, 5, 37, 101)]


@pytest.mark.gpu
def test_projection_does_not_depend_on_the_slot(shared_ctx):
    """the whole soup under one dHat and kappa.  dHat is the d of the early_return stencils, so their blocks are exactly zero and take
    makePD's early return whatever the rounding (their projection groups leave the shuffles early); they share warps with clamped blocks
    of widely spread spectra (d / dHat down to 1e-23) and slow-converging ones, and with pairs beyond dHat.  The CSR values are
    bit-identical for every list order, and the active and mollified lists uploaded together give exactly the sum of each alone (the
    stencils are disjoint)."""
    z = gold()
    m = soup_mesh(z)
    load_scene(shared_ctx, m, mass=False, dbc=False)
    ia, ja = m.csr_pattern(1)
    shared_ctx.set_csr(ia, ja, 1)
    n = z["E"].size
    er = np.flatnonzero(z["family"] == list(z["families"]).index("early_return"))
    dHat, kappa = float(z["dHat"][er[0]]), 1.0
    assert np.all(z["d"][er] == dHat)
    a_idx, p_idx, mm, pa, pe = lists(z, range(n))
    ref = gpu_hessian(shared_ctx, m, ia, ja, mm, pa, pe, dHat, kappa)
    assert np.count_nonzero(ref) > 0 and np.all(np.isfinite(ref))
    assert not np.any(blocks_of_csr(ref, ia, ja, m.nV, m.T[er]))
    for oa, op in zip(rotations(len(mm)), rotations(len(pa))[::-1]):
        a = gpu_hessian(shared_ctx, m, ia, ja, mm[oa], pa[op], pe[op], dHat, kappa)
        assert np.array_equal(a, ref)
    act = gpu_hessian(shared_ctx, m, ia, ja, mm, pa[:0], pe[:0], dHat, kappa)
    par = gpu_hessian(shared_ctx, m, ia, ja, mm[:0], pa, pe, dHat, kappa)
    assert not np.any((act != 0) & (par != 0))
    assert np.array_equal(act + par, ref)


@pytest.mark.gpu
def test_friction_kernels_match_fixture(shared_ctx):
    z = gold()
    m = soup_mesh(z)
    load_scene(shared_ctx, m, mass=False, dbc=False)
    ia, ja = m.csr_pattern(1)
    shared_ctx.set_csr(ia, ja, 1)
    shared_ctx.set_prev_state(np.ascontiguousarray(z["V_prev"].T).ravel())
    rep = Report(z, "gpu")
    coef = float(z["coef"])
    for (dHat, kappa), ks in groups(z, np.flatnonzero(z["fric"])).items():
        mm = z["mm"][ks]
        shared_ctx.set_constraint_set(mm, np.zeros((0, 4), np.int32), np.zeros((0, 2), np.int32))
        assert shared_ctx.friction_lag(dHat, kappa) == len(ks)
        mm_l, lam, co, ba = shared_ctx.get_friction_data()
        assert np.array_equal(mm_l, mm)
        for j, k in enumerate(ks):
            check_lag(rep, z, k, lam[j], co[j], ba[j])
            for dev, data in ((True, (lam[j], co[j], ba[j])), (False, (z["lam"][k], z["coord"][k], z["basis"][k]))):
                if dev and z["near_branch"][k]:
                    continue
                shared_ctx.set_friction_data(mm[j:j + 1], np.atleast_1d(data[0]), data[1][None], data[2][None])
                eps2 = float(z["eps2"][k])
                E = shared_ctx.friction_energy(eps2, coef)
                g = shared_ctx.friction_gradient(eps2, coef, np.zeros(3 * m.nV)).reshape(-1, 3)
                a = shared_ctx.friction_hessian(eps2, coef, 1, np.zeros(ja.size))
                H = blocks_of_csr(a, ia, ja, m.nV, m.T[k:k + 1])[0]
                assert np.count_nonzero(g) == np.count_nonzero(g[m.T[k]])
                check_friction(rep, z, k, E, g[m.T[k]].ravel(), H, dev)
    rep.table(f"gpu friction: {fixture_counts(z)}")
