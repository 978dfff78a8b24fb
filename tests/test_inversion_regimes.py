"""The inversion filter's root finder (k_inversion_step / k_inversion_apply in elastic.cu), the CPU oracle (orc_inversion_step) and the
reference's own getSmallestPositiveRealCubicRoot against tests/golden/inversion_regimes_golden.npz: an mpmath evaluation
(tests/golden/gen_inversion_regimes_golden.py) of the formula and of the true roots on a soup of disjoint tets that reaches every exit
of the formula and every decision within its rounding margin -- the linear exit (c > 0, c < 0, c = 0, d = +-0, the mm scale), the
quadratic exit (a root of each sign, two positive roots, desc == 0 exactly, desc < 0, |a| on both sides of 1e-6 and within rounding of
it), Cardano with one real root (both signs of the real radicand) and three, nearly equal roots (|Im t| around 1e-6), the |C| == 0
fallback and the triple root, a root just above 0, uniform contractions, rotations, slivers, inverted and flat tets, edges 1e-3 .. 1e2 at
offsets up to 1e3.

Error model (eps = 2^-52, C = C_ROUND = 32).  The coefficients a, b, c, d are sums of products of edge differences (det3v); each is
within C eps S_k of its exact value, S_k the sum of |products| that forms it (three factors with a rounded difference each, the products,
at most eleven additions: 16 roundings, with a factor of two to spare; fused multiply-adds round less, not more).  Delta0, Delta1, the
radicand R = Delta1^2 - 4 Delta0^3 and Delta1 + sqrt(R) are each within C eps of the sum of |terms| that forms them (the last sum cancels
where Delta1 < 0 and Delta0 is small: without that term the oracle misses the bar by 20x on three nearly equal roots shifted by the slack).  The fixture evaluates the formula exactly at the corners of that box, and with every
value threshold (|Im t| < 1e-6, Re t > 0, desc > 0, the quadratic's t < 0) moved by C eps times the scale of the value it tests:
  - where every evaluation takes the same exit and keeps the same root, a tet's bound r is held to
        |r - root| <= C eps cscale + spread
    with cscale the scale of the formula's last combination ((|b| + |C| + |Delta0/C|) / |3a| for Cardano, (|B| + sqrt|desc|) / |2A|
    for the quadratic, |d/c| for the linear exit) and spread the largest distance of a corner's value from the center's;
  - elsewhere (`ambiguous`) any outcome the evaluations met is admissible: r lies in one of the intervals of values met, widened by C eps
    times that outcome's largest cscale, or r = 1e20 where an evaluation kept no root;
  - where the double arithmetic is exact (`exact`: no root, a zero d or c formed only of zero products), r is held bit for bit: 1e20,
    +-0 with its sign, +inf.
The bars hold for the oracle (no fused operations), the device (elastic.cu is compiled with fused multiply-adds and CUDA's own libm) and
the reference's code given the round-to-nearest coefficients, which differ from exact by at most eps/2 |coef|.

The step (Energy.cpp:576-579): alpha_out = m if 0 < m < alpha_in else alpha_in, with m the minimum of the per-tet bounds taken left to
right with `<` (Eigen's minCoeff) -- a zero bound of either sign is that minimum wherever it lies and leaves alpha unchanged.  The device's
alpha is held bit for bit to that rule applied to its own per-tet bounds, whatever CTA and lane each tet lands in.
"""
import importlib.util
import os

import numpy as np
import pytest

import oracle as orc
import refcubic
from gpu_common import scalar_bits, shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "inversion_regimes_golden.npz")
GEN = os.path.join(HERE, "golden", "gen_inversion_regimes_golden.py")
EPS = np.finfo(float).eps
C_ROUND = 32.0
NONE = 1e20
TOL = 1e-6


def gold():
    return dict(np.load(GOLD))


def gen_module():
    spec = importlib.util.spec_from_file_location("gen_inversion_regimes_golden", GEN)
    g = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(g)
    return g


def check(z, idx, got, who):
    """per-tet bounds `got` of tets idx against the fixture's bars; returns the worst error/bar ratio of the value checks"""
    worst, bad = 0.0, []
    for t, r in zip(idx, got):
        if z["exact"][t] and not z["ambiguous"][t]:
            if scalar_bits(r) != scalar_bits(z["root"][t]):
                bad.append((t, "exact", r, z["root"][t]))
            continue
        if not z["ambiguous"][t]:
            bar = C_ROUND * EPS * z["cscale"][t] + z["spread"][t]
            err = abs(r - z["root"][t])
            if r == NONE or not err <= bar:
                bad.append((t, "value", r, z["root"][t], err, bar))
            elif bar > 0:
                worst = max(worst, err / bar)
            continue
        ok = False
        for lo, hi, tol in z["adm"][t]:
            if np.isnan(lo):
                continue
            if lo == NONE:
                ok |= r == NONE
            else:
                ok |= lo - tol <= r <= hi + tol
        if not ok:
            bad.append((t, "admissible", r, z["adm"][t]))
    assert not bad, f"{who}: {len(bad)} tets off the fixture, e.g. {bad[:4]}"
    return worst


def soup_mesh(X, P):
    """disjoint tets with unit rest shapes (the filter reads only the current positions and the direction)"""
    n = len(X)
    unit = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]])
    m = M.Mesh(np.tile(unit, (n, 1)), np.arange(4 * n, dtype=np.int32).reshape(n, 4), energy=0)
    m.V = np.ascontiguousarray(np.asarray(X, dtype=np.float64).reshape(-1, 3))
    return m, np.ascontiguousarray(np.asarray(P, dtype=np.float64).reshape(-1))


def groups(z):
    return {s: np.flatnonzero(z["slack"] == s) for s in np.unique(z["slack"])}


def ref_rule(per, alpha):
    """Energy.cpp:576-579 with Eigen's minCoeff: a left-to-right `<` minimum, then 0 < m < alpha"""
    m = per[0]
    for v in per[1:]:
        if v < m:
            m = v
    return m if (0.0 < m < alpha) else alpha


def double_coefs(z, t):
    """a, b, c, d as the oracle forms them (det3v sums, no fused operations)"""
    return gen_module().coefficients(z["X"][t], z["P"][t], z["slack"][t], exact=False)[0]


# ---- CPU --------------------------------------------------------------------------------------------------------------------------------
def test_fixture_shape():
    z = gold()
    g = gen_module()
    n = len(z["family"])
    assert n >= 150 and set(np.unique(z["family"])) == set(range(len(g.FAMILIES)))
    assert set(np.unique(z["exit"])) == set(range(len(g.EXITS)))
    assert set(np.unique(z["category"])) == set(range(len(g.CATEGORIES)))
    assert z["ambiguous"].sum() < n // 4
    print("\ncategories:", {c: int((z["category"] == k).sum()) for k, c in enumerate(g.CATEGORIES)},
          "ambiguous:", int(z["ambiguous"].sum()), "of", n)


def test_oracle_matches_fixture():
    z = gold()
    worst = 0.0
    for s, idx in groups(z).items():
        m, p = soup_mesh(z["X"][idx], z["P"][idx])
        _, per = orc.Elastic(m).inversion_step(p, s, 1.0)
        worst = max(worst, check(z, idx, per, "oracle"))
    print(f"\noracle: worst error/bar {worst:.3g}")


def test_cubic_branch_coverage():
    """every exit and every decision of the formula is reached by the oracle's own doubles"""
    z = gold()
    seen = set()
    per_all = np.empty(len(z["family"]))
    for s, idx in groups(z).items():
        m, p = soup_mesh(z["X"][idx], z["P"][idx])
        per_all[idx] = orc.Elastic(m).inversion_step(p, s, 1.0)[1]
    for t in range(len(z["family"])):
        a, b, c, d = double_coefs(z, t)
        r, ex, fb, passed, kept = orc.cubic_branch(a, b, c, d)
        assert scalar_bits(r if r >= 0 else NONE) == scalar_bits(per_all[t])   # the branch report is the filter's own computation
        seen.add(ex)
        if ex == "linear":
            seen.add("linear c>0" if c > 0 else "linear c<0" if c < 0 else "linear c=0")
            if d == 0:
                seen.add("linear d=0 -> " + ("-0" if np.signbit(r) else "+0"))
        if ex == "quad_second" and r > 0:
            seen.add("quad first root negative, second positive")
        if ex == "quad_first" and b * d > 0 and c * b < 0:
            seen.add("quad two positive roots")
        if ex == "quad_none":
            seen.add("quad desc == 0" if c * c - 4 * b * d == 0 else "quad desc < 0")
        if abs(abs(a) - TOL) <= C_ROUND * EPS * z["S"][t, 0]:
            seen.add("|a| within rounding of tol, " + ("cubic" if abs(a) > TOL else "quadratic"))
        if ex.startswith("cardano"):
            D0 = b * b - 3 * a * c
            D1 = 2 * b * b * b - 9 * a * b * c + 27 * a * a * d
            R = D1 * D1 - 4 * D0 * D0 * D0
            seen.add(f"{ex}, " + ("three real roots" if R < 0 else "one real root"))
            if fb:
                seen.add("fallback |C| == 0" + (", triple root: no root" if kept == 0 else ""))
            seen.add(f"kept t{kept}" if kept else "cardano none kept")
            if 0 < r < 1e-12:
                seen.add("Re t just above 0")
        if z["ambiguous"][t] and z["family"][t] == gen_module().FAMILIES.index("near_double"):
            seen.add("|Im t| within rounding of tol")
        if r == 0 and np.signbit(r) and ex in ("quad_first", "quad_second"):
            seen.add("quad d=0 -> -0")
    want = {"linear", "quad_first", "quad_second", "quad_none", "cardano_real", "cardano_complex", "linear c>0", "linear c<0", "linear c=0",
            "linear d=0 -> -0", "linear d=0 -> +0", "quad first root negative, second positive", "quad two positive roots", "quad desc == 0",
            "quad desc < 0", "|a| within rounding of tol, cubic", "|a| within rounding of tol, quadratic", "cardano_real, one real root",
            "cardano_complex, one real root", "cardano_complex, three real roots", "fallback |C| == 0", "fallback |C| == 0, triple root: no root",
            "kept t1", "kept t2", "kept t3", "cardano none kept", "Re t just above 0", "|Im t| within rounding of tol", "quad d=0 -> -0"}
    assert want <= seen, sorted(want - seen)
    print("\nreached:", sorted(seen))


def test_generator_reproduces_the_fixture():
    z = gold()
    g = gen_module()
    fam, X, P, slack = g.build()
    for k, v in (("family", fam), ("X", X), ("P", P), ("slack", slack)):
        assert z[k].shape == v.shape and z[k].tobytes() == v.tobytes(), k
    for t in range(0, len(fam), 13):
        r = g.evaluate(X[t], P[t], slack[t])
        for k in ("exit", "kept", "exact", "ambiguous", "category"):
            assert r[k] == z[k][t], (t, k)
        for k in ("root", "cscale", "spread", "true_root", "coef", "S"):
            assert np.array_equal(np.asarray(r[k]), z[k][t]), (t, k)


@pytest.mark.skipif(not refcubic.available(), reason="oracle/_ref/libref_cubic.so not built (needs the reference sources)")
def test_reference_root_finder_meets_the_fixture():
    """the reference's own getSmallestPositiveRealCubicRoot, given the round-to-nearest coefficients"""
    z = gold()
    n = len(z["family"])
    per = np.empty(n)
    for t in range(n):
        r = refcubic.cubic_root(*z["coef"][t])
        per[t] = r if r >= 0 else NONE
        a, b, c, d = z["coef"][t]
        if abs(a) <= TOL and abs(b) > TOL:
            assert scalar_bits(refcubic.quad_root(b, c, d)) == scalar_bits(r)
    # a coefficient that the fixture holds exactly as a signed zero (a flat tet's d, a zero direction's c) is +0.0 in coef: the sign
    # the double arithmetic gives it is not in the rounded value, so those tets are compared by value
    sz = z["exact"] & ~z["ambiguous"] & ((z["root"] == 0) | np.isinf(z["root"]))
    worst = check(z, np.flatnonzero(~sz), per[~sz], "reference")
    assert np.all((per[sz] == z["root"][sz]) | (np.isinf(z["root"][sz]) & (per[sz] >= NONE)))
    print(f"\nreference root finder: worst error/bar {worst:.3g}")


@pytest.mark.skipif(not refcubic.available(), reason="oracle/_ref/libref_cubic.so not built (needs the reference sources)")
def test_reference_coefficients_lose_digits_at_an_offset():
    """The reference expands a, b, c, d in absolute coordinates.  Near the origin that is as accurate as the edge-difference form; at an
    offset of 1e3 with 1e-3 .. 1e-2 edges it loses the leading digits of c and d (recorded, DESIGN 3): the device is pinned to exact
    coefficients instead."""
    z = gold()
    near, far = [], []
    for t in range(len(z["family"])):
        X = z["X"][t]
        edge = np.abs(X[1:] - X[0]).max()
        rc = refcubic.coefs(X, z["P"][t], z["slack"][t])
        exact = np.array([float(s) for s in z["coef_str"][t]])
        err = np.abs(rc - exact) / np.maximum(z["S"][t], 1e-300)
        (near if np.abs(X).max() <= 4 * edge else far).append(err[2:].max() if z["S"][t, 3] > 0 else 0.0)
    near, far = np.array(near), np.array(far)
    assert near.max() <= 64 * C_ROUND * EPS, near.max()   # the absolute expansion's products reach 4^3 S_k at coordinates of 4 edges
    assert far.max() > 1e6 * C_ROUND * EPS, far.max()
    print(f"\nreference coefficients: c, d error / S near the origin {near.max():.3g}, at an offset up to {far.max():.3g}")


# ---- GPU --------------------------------------------------------------------------------------------------------------------------------
def run_gpu(ctx, X, P, slack, alpha=1.0):
    m, p = soup_mesh(X, P)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, None, None, 0)
    ctx.set_state(m.V_soa)
    a = ctx.inversion_step(p, slack, alpha)
    return a, ctx.download(L.BUF_INVERSION_STEPS, m.nT)


@pytest.mark.gpu
def test_device_matches_fixture(shared_ctx):
    z = gold()
    worst = 0.0
    for s, idx in groups(z).items():
        _, per = run_gpu(shared_ctx, z["X"][idx], z["P"][idx], s)
        worst = max(worst, check(z, idx, per, "device"))
    print(f"\ndevice: worst error/bar {worst:.3g}")


def _pad_tet(k):
    """a unit tet with a zero direction: a = b = c = 0, no bound"""
    X = np.array([[0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]]) + 3.0 * k
    return X, np.zeros((4, 3))


def _soup(z, picks, n=3 * 256 + 40):
    """tets picks[i] = (position, fixture tet) placed at their positions, padding elsewhere"""
    X = np.empty((n, 4, 3)); P = np.empty((n, 4, 3))
    for k in range(n):
        X[k], P[k] = _pad_tet(k)
    for pos, t in picks:
        X[pos], P[pos] = z["X"][t], z["P"][t]
    return X, P


@pytest.mark.gpu
def test_device_step_follows_the_reference_rule(shared_ctx):
    """alpha_out == the reference's rule on the device's own per-tet bounds, with zero bounds of either sign in the CTA of the smallest
    positive bound and in another one, and with no bound at all"""
    z = gold()
    s2 = z["slack"] == 0.2
    exact_fin = s2 & z["exact"] & ~z["ambiguous"]
    neg0 = [t for t in np.flatnonzero(exact_fin) if z["root"][t] == 0 and np.signbit(z["root"][t])]
    pos0 = [t for t in np.flatnonzero(exact_fin) if z["root"][t] == 0 and not np.signbit(z["root"][t])]
    plain = np.flatnonzero(s2 & ~z["ambiguous"] & ~z["exact"] & (z["root"] > 1e-3) & (z["root"] < 10))
    assert neg0 and pos0 and len(plain) >= 3
    small, mid, big = plain[np.argsort(z["root"][plain])][[0, len(plain) // 2, -1]]
    roots = sorted(z["root"][[small, mid, big]])
    alphas = [roots[0] / 2, (roots[0] + roots[1]) / 2, roots[2] * 2, 1.0]
    soups = {"positive only": [(5, small), (300, mid), (700, big)]}
    for name, zs in (("-0.0", neg0[0]), ("+0.0", pos0[0])):
        soups[f"{name} in the CTA of the smallest root"] = [(5, small), (300, mid), (700, big), (40, zs)]
        soups[f"{name} in another CTA"] = [(5, small), (300, mid), (700, big), (600, zs)]
        soups[f"{name} before the smallest root"] = [(0, zs), (5, small), (300, mid), (700, big)]
    soups["no root"] = []
    for name, picks in soups.items():
        X, P = _soup(z, picks)
        for alpha in alphas:
            a, per = run_gpu(shared_ctx, X, P, 0.2, alpha)
            want = ref_rule(per, alpha)
            assert scalar_bits(a) == scalar_bits(want), (name, alpha, a, want)
            for pos, t in picks:
                assert scalar_bits(per[pos]) == scalar_bits(z["root"][t]) or not z["exact"][t], (name, pos, per[pos], z["root"][t])
            if "0.0" in name:
                assert a == alpha, (name, alpha, a)   # a zero bound leaves the step unchanged
            if name == "no root":
                assert np.all(per >= NONE) and a == alpha


@pytest.mark.gpu
def test_device_placement_does_not_change_a_tet(shared_ctx):
    """the slack-0.2 soup padded past three CTAs, and the same tets shifted by 257 places (cyclically): every tet changes CTA and lane, its
    bound's bits and the step do not"""
    z = gold()
    idx = np.flatnonzero(z["slack"] == 0.2)
    n = max(3 * 256 + 40, len(idx))
    X, P = _soup(z, list(enumerate(idx)), n)
    perm = (np.arange(n) + 257) % n   # tet k goes to place perm[k]
    assert np.all(perm // 256 != np.arange(n) // 256) and np.all(perm % 256 != np.arange(n) % 256)
    X2, P2 = np.empty_like(X), np.empty_like(P)
    X2[perm], P2[perm] = X, P
    for alpha in (1.0, 0.01):
        a1, per1 = run_gpu(shared_ctx, X, P, 0.2, alpha)
        a2, per2 = run_gpu(shared_ctx, X2, P2, 0.2, alpha)
        assert per1.view(np.uint64).tolist() == per2[perm].view(np.uint64).tolist()
        assert scalar_bits(a1) == scalar_bits(a2) == scalar_bits(ref_rule(per1, alpha))
