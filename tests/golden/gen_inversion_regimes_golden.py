"""Generates tests/golden/inversion_regimes_golden.npz: a soup of disjoint tets (four own vertices and four own directions each) at the
places where the inversion filter's root finder (getSmallestPositiveRealCubicRoot, get_feasible_steps.cpp:75-108) changes exit or
degenerates, with the formula and the true roots evaluated in mpmath (DPS digits) from the stored doubles alone.

Coefficients.  det(e + t f) - slack' det(e) = a t^3 + b t^2 + c t + d with e_i = x_{i+1} - x_0, f_i = p_{i+1} - p_0 (the edge-difference
form the kernels use), slack' = 1 - slack rounded once to a double (as the kernels form it), all exact rationals of the stored doubles.
S_k is the rounding scale of coefficient k: the sum of |products| of the det3v expansions that form it (times slack' for d).

The formula's result.  The formula is evaluated in mpmath with every decision taken on exact values: at the exact coefficients (the
"center"), at the 256 corners of the rounding box (a, b, c, d each moved by C_ROUND eps S_k; Delta0, Delta1, the radicand
R = Delta1^2 - 4 Delta0^3 and the real part of Delta1 + sqrt(R) each by C_ROUND eps times the sum of |terms| that forms it), and at the center with the value thresholds (|Im t| < tol, Re t > 0, desc > 0, the quadratic's t < 0)
moved by C_ROUND eps times the scale of the rounded value they test, both ways.  An outcome is the exit with the root it kept; a tet whose
evaluations do not all take the center's outcome is `ambiguous`, and every outcome met is admissible, as an interval [lo, hi] of the
values met, widened by adm_tol = C_ROUND eps times the largest rounding scale among them.  For the center:
  root     the value (1e20 for no root, as the kernels store it; +-inf and +-0 with the sign the double arithmetic gives them, see `exact`)
  cscale   the rounding scale of the final combination: (|b| + |C| + |Delta0/C|) / |3a| for Cardano, (|B| + sqrt|desc|) / |2A| for the
           quadratic, |d / c| for the linear exit
  spread   the largest distance of a corner value of the center's outcome from the center value
  exact    the double arithmetic gives root exactly: 1e20, a signed zero (a zero d formed only of zero products), +-inf (c formed only of
           zero products); the sign of a zero coefficient is that of its det3v sums in IEEE double (a zero product makes the sum exact, so
           fused multiply-adds give the same sign)
True roots (mpmath.polyroots of the exact polynomial, its degree lowered past exactly zero leading coefficients): true_root is the
smallest positive real one (+inf for none), and category says what the formula does about it: CATEGORIES.
Run:  python tests/golden/gen_inversion_regimes_golden.py
"""
import os
from fractions import Fraction as Fr
from itertools import product

import mpmath as mp
import numpy as np

DPS = 60
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "inversion_regimes_golden.npz")
EPS = 2.0 ** -52
C_ROUND = 32.0
TOL = 1.0e-6
NONE = 1e20
K_ADM = 8
EXITS = ("linear", "quad_first", "quad_second", "quad_none", "cardano_real", "cardano_complex")
CATEGORIES = ("finds", "larger", "none", "smaller")
FAMILIES = ("linear", "quadratic", "a_at_tol", "cardano_one_real", "cardano_three_real", "near_double", "fallback", "near_zero",
            "contraction", "rotation", "sliver", "random")


# ---- exact coefficients ----------------------------------------------------------------------------------------------------------------
def _det(u, v, w):
    return u[0] * (v[1] * w[2] - v[2] * w[1]) - u[1] * (v[0] * w[2] - v[2] * w[0]) + u[2] * (v[0] * w[1] - v[1] * w[0])


def _dets(u, v, w):
    """sum of |products| of the det3v expansion"""
    a = [abs(x) for x in u]; b = [abs(x) for x in v]; c = [abs(x) for x in w]
    return a[0] * (b[1] * c[2] + b[2] * c[1]) + a[1] * (b[0] * c[2] + b[2] * c[0]) + a[2] * (b[0] * c[1] + b[1] * c[0])


def coefficients(X, P, slack, exact=True):
    """(a, b, c, d) and (S_a, S_b, S_c, S_d): exact rationals, or the kernels' det3v sums in IEEE double (exact=False, no fused ops)"""
    cv = Fr if exact else float
    X = [[cv(float(v)) for v in r] for r in X]
    P = [[cv(float(v)) for v in r] for r in P]
    e = [[X[k + 1][j] - X[0][j] for j in range(3)] for k in range(3)]
    f = [[P[k + 1][j] - P[0][j] for j in range(3)] for k in range(3)]
    s1 = cv(1.0 - float(slack))
    a = _det(f[0], f[1], f[2])
    b = _det(e[0], f[1], f[2]) + _det(f[0], e[1], f[2]) + _det(f[0], f[1], e[2])
    c = _det(f[0], e[1], e[2]) + _det(e[0], f[1], e[2]) + _det(e[0], e[1], f[2])
    d = s1 * _det(e[0], e[1], e[2])
    S = (_dets(f[0], f[1], f[2]), _dets(e[0], f[1], f[2]) + _dets(f[0], e[1], f[2]) + _dets(f[0], f[1], e[2]),
         _dets(f[0], e[1], e[2]) + _dets(e[0], f[1], e[2]) + _dets(e[0], e[1], f[2]), abs(s1) * _dets(e[0], e[1], e[2]))
    return (a, b, c, d), S


# ---- the formula in mpmath ---------------------------------------------------------------------------------------------------------------
def _cbrt(z):
    """std::pow(complex, 1/3): the real pow of a positive real radicand, the principal branch otherwise"""
    if z == 0:
        return mp.mpc(0)
    if mp.im(z) == 0 and mp.re(z) > 0:
        return mp.mpc(mp.cbrt(mp.re(z)))
    return mp.exp(mp.log(z) / 3)


def formula(a, b, c, d, d0=0, d1=0, dr=0, dq=0, shift=0, m=None):
    """getSmallestPositiveRealCubicRoot with exact decisions.  d0, d1: offsets added to Delta0, Delta1; shift (+-1): the value thresholds
    moved by m[name] in the direction that makes the test pass (shift = 1) or fail (shift = -1).  Returns (outcome, value, scale):
    outcome = (exit, kept), value None for no root (or a NaN root)."""
    mv = (lambda k: shift * m[k]) if shift else (lambda k: 0)
    tolv = mp.mpf(TOL)
    if abs(a) <= tolv:
        A, B, Cq = b, c, d
        if abs(A) <= tolv:
            if B == 0:
                return (0, 0), (None if Cq == 0 else mp.inf * (-mp.sign(Cq))), mp.inf
            t = -Cq / B
            return (0, 0), (None if t != 0 and t < mv("qt") else t), abs(Cq / B)   # a negative root: none
        desc = B * B - 4 * A * Cq
        if desc > -mv("desc"):
            sq = mp.sqrt(max(desc, mp.mpf(0)))
            t = (-B - sq) / (2 * A)
            sc = (abs(B) + sq) / abs(2 * A)
            if t != 0 and t < mv("qt"):
                t = (-B + sq) / (2 * A)
                return (2, 0), (None if t != 0 and t < mv("qt") else t), sc
            return (1, 0), t, sc
        return (3, 0), None, mp.mpf(0)
    D0 = b * b - 3 * a * c + d0
    D1 = 2 * b ** 3 - 9 * a * b * c + 27 * a * a * d + d1
    R = D1 * D1 - 4 * D0 ** 3
    R += dr * (D1 * D1 + 4 * abs(D0) ** 3)
    sR = mp.sqrt(mp.mpc(R))
    rad = (D1 + sR) / 2
    if rad != 0:   # the rounding of the sum, which cancels where Delta1 < 0 and |Delta0| is small
        rad += dq * (abs(D1) + abs(sR)) / 2
    C = _cbrt(rad)
    fb = 0
    if C == 0:
        rad = (D1 - sR) / 2
        C = _cbrt(rad)
        fb = 1
    ex = 4 if (mp.im(rad) == 0 and mp.re(rad) > 0) else 5
    if C == 0:
        return (ex, 0), None, mp.inf   # 0/0: NaN roots, none kept
    u2 = mp.mpc(-0.5, mp.sqrt(3) / 2)
    u3 = mp.mpc(-0.5, -mp.sqrt(3) / 2)
    ts = [(b + Ck + D0 / Ck) / (-3 * a) for Ck in (C, u2 * C, u3 * C)]
    sc = (abs(b) + abs(C) + abs(D0 / C)) / abs(3 * a)
    t, k = None, 0
    for j, tj in enumerate(ts):
        if abs(mp.im(tj)) < tolv + mv("im") and mp.re(tj) > -mv("re") and (t is None or mp.re(tj) < t):
            t, k = mp.re(tj), j + 1
    return (ex, k), t, sc


def _delta_scales(a, b, c, d):
    return abs(b) ** 2 + 3 * abs(a * c), 2 * abs(b) ** 3 + 9 * abs(a * b * c) + 27 * a * a * abs(d)


def evaluate(X, P, slack):
    """every fixture field of one tet (module docstring)"""
    mp.mp.dps = DPS
    (a, b, c, d), S = coefficients(X, P, slack)
    (fa, fb_, fc, fd), _ = coefficients(X, P, slack, exact=False)
    co = [mp.mpf(x.numerator) / x.denominator for x in (a, b, c, d)]
    Sm = [mp.mpf(x.numerator) / x.denominator for x in S]
    u = C_ROUND * EPS
    out, val, sc = formula(*co)
    # value-threshold margins at the center: the rounding of the tested values
    m = {"desc": u * (co[2] ** 2 + 4 * abs(co[1] * co[3])), "qt": u * sc if sc != mp.inf else 0, "im": u * sc, "re": u * sc}
    evals = [(out, val, sc)]
    for sh in (1, -1):
        evals.append(formula(*co, shift=sh, m=m))
    S0, S1 = _delta_scales(*co)
    for sg in product((-1, 1), repeat=8):
        cc = [co[k] + sg[k] * u * Sm[k] for k in range(4)]
        evals.append(formula(*cc, d0=sg[4] * u * S0, d1=sg[5] * u * S1, dr=sg[6] * u, dq=sg[7] * u))
    groups = {}
    for o, v, s in evals:
        g = groups.setdefault(o, [[], []])
        g[0].append(v)
        g[1].append(s)
    ambiguous = len(groups) > 1
    adm = np.full((K_ADM, 3), np.nan)
    for j, (o, (vs, ss)) in enumerate(sorted(groups.items())):
        if any(v is None for v in vs):
            adm[j] = (NONE, NONE, 0.0)
        else:
            adm[j] = (float(min(vs)), float(max(vs)), float(u * max(ss)) if all(s != mp.inf for s in ss) else 0.0)
    center_vals = groups[out][0]
    spread = 0.0 if val is None or abs(val) == mp.inf else float(max(abs(v - val) for v in center_vals))
    # the stored root and whether the double arithmetic gives it exactly
    exact = False
    if val is None:
        root, exact = NONE, True
    elif abs(val) == mp.inf:   # linear exit with c of zero products: -d / (+-0)
        assert S[2] == 0
        with np.errstate(divide="ignore"):
            root = float(-np.float64(fd) / np.float64(fc))
        root, exact = (root if root >= 0 else NONE), True
    elif val == 0 and out[0] <= 2 and S[3] == 0:   # a zero d of zero products: -(+-0)/c, or +0/(2A)
        root = float(-np.float64(fd) / np.float64(fc)) if out[0] == 0 else float(np.float64(0.0) / (2.0 * np.float64(fb_)))
        exact = True
    else:
        root = float(val)
        if root < 0:   # (cannot happen: a kept root is >= 0 or the exit returns none)
            root = NONE
    # true roots
    poly = list(co)
    while poly and poly[0] == 0:
        poly.pop(0)
    real_pos = []
    if len(poly) >= 2:
        try:
            rts = mp.polyroots(poly, maxsteps=400, extraprec=400)
        except mp.NoConvergence:   # a triple root: the companion matrix's eigenvalues (accurate to a cube root of the working precision)
            n = len(poly) - 1
            Cm = mp.zeros(n, n)
            for k in range(n):
                Cm[0, k] = -poly[k + 1] / poly[0]
                if k + 1 < n:
                    Cm[k + 1, k] = 1
            rts = list(mp.eig(Cm, left=False, right=False))
        scale = max(abs(r) for r in rts)
        for r in rts:
            r = mp.mpc(r)
            if abs(mp.im(r)) <= mp.mpf(10) ** -18 * (1 + scale) and mp.re(r) > 0:
                real_pos.append(mp.re(r))
    true_root = float(min(real_pos)) if real_pos else np.inf
    # category: the formula's value v (+inf for no root) against the true smallest positive root tr (+inf for none)
    v = mp.inf if (val is None or root == NONE) else mp.mpf(root)
    tr = min(real_pos) if real_pos else mp.inf
    if v == tr:
        cat = 0
    elif v == mp.inf:
        cat = 2
    else:
        bar = u * (sc if sc != mp.inf else 0) + spread + mp.mpf(10) ** -18 * (1 + abs(v))
        cat = 0 if abs(v - tr) <= bar else (1 if v > tr else 3)
    return dict(coef=np.array([float(x) for x in co]), coef_str=np.array([mp.nstr(x, 40) for x in co]), S=np.array([float(x) for x in Sm]),
                exit=out[0], kept=out[1], root=root, exact=exact, cscale=float(sc) if sc != mp.inf else 0.0, spread=spread,
                ambiguous=ambiguous, adm=adm, true_root=true_root, category=cat)


# ---- the soup ---------------------------------------------------------------------------------------------------------------------------
def _rot(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def cases():
    """[(family, X (4,3), P (4,3), slack)] in fixture order; deterministic"""
    out = []
    rng = np.random.default_rng(20261017)

    def add(fam, e, f, slack=0.2, h=1.0, off=(0.0, 0.0, 0.0), p0=(0.0, 0.0, 0.0), mirror=True):
        """a tet x0 = off, x_{k+1} = off + h e[k] with directions p0, p0 + h f[k]; mirror: also the reflected tet (x -> -x), whose
        polynomial is the negated one (Delta1 changes sign, Delta0 does not)"""
        e, f = np.asarray(e, float), np.asarray(f, float)
        X = np.vstack([np.zeros(3), h * e]) + np.asarray(off, float)
        P = np.vstack([np.zeros(3), h * f]) + np.asarray(p0, float)
        out.append((FAMILIES.index(fam), X, P, float(slack)))
        if mirror:
            out.append((FAMILIES.index(fam), -X, -P, float(slack)))

    I = np.eye(3)
    D = np.diag
    # linear exit (|a|, |b| <= tol): rank-1 directions f = u v^T at unit and mm scale, positive / negative / zero c, inverted tets
    for h in (1.0, 1e-3):
        for uv in (-0.5, 0.5, -2.0):
            f = np.outer([1.0, 0.0, 0.0], [uv, 0.0, 0.0])
            add("linear", I, f, h=h)
    add("linear", I, np.zeros((3, 3)), mirror=True)                 # c = 0 of zero products: -d/(+-0) -> -inf (1e20) or +inf
    add("linear", I * [1, 1, -1], np.zeros((3, 3)), mirror=False)   # inverted tet, c = +-0
    flat = np.array([[1.0, 0, 0], [0, 1.0, 0], [0.5, 0.5, 0]])      # zero volume: d of zero products
    for cz in (1e-4, -1e-4):
        add("linear", flat, cz * np.array([[0, 0, 1.0], [0, 0, 0], [0, 0, 0]]))  # d = +-0, c = +-1e-4: roots -0/c
    for s in (1e-3, 2e-3):                                          # mm-scale compression: the linearised root is not the cubic's
        add("linear", I, -0.9 * I, h=s, off=(1e3, -1e3, 1e3))
        add("linear", I, _rot([1, 2, 3], 2.0) - I, h=s)
    # quadratic exit (a = 0 exactly: f of rank 2)
    def f2(f00, f01, f10, f11):
        return np.array([[f00, f01, 0], [f10, f11, 0], [0, 0, 0.0]])
    add("quadratic", I * [1, 1, -1], f2(1.0, 0, 0, -2.0), slack=0.2)  # inverted, A > 0: first root negative, second positive
    add("quadratic", I, f2(-1.0, 0, 0, -2.0), slack=0.2)             # both positive
    add("quadratic", I, f2(-1.0, 0, 0, -2.0), slack=0.0)
    add("quadratic", I, f2(-1.0, 0, 0, -1.0), slack=0.0)             # desc == 0 exactly: a double root at 1 the formula drops
    add("quadratic", I, f2(0.0, -1.0, 1.0, 0.0), slack=0.2)          # desc < 0
    add("quadratic", I, f2(-1e-3, 0, 0, -2e-3), slack=0.2, h=10.0)   # |B| > tol at h = 10
    add("quadratic", flat, np.array([[0, 0, 0.3], [0, 0, 0], [0, 0, -0.2]]), slack=0.2)  # d = +-0 with A, B of both signs
    add("quadratic", flat, np.array([[0, 0, 0.3], [0, 0, 0], [0.5, 0, -0.2]]), slack=0.2)
    # |a| at the 1e-6 threshold, on both sides and within rounding of it (a = f22 exactly with f = diag(-1, -1, f22))
    t = TOL
    for f22 in (t, np.nextafter(t, 1), np.nextafter(t, 0), t * (1 + 1e-9), t * (1 - 1e-9), t * (1 + 1e-13), t * (1 - 1e-13)):
        add("a_at_tol", I, D([-1.0, -1.0, f22]), slack=0.2)
        add("a_at_tol", I, D([-1.0, -1.0, -f22]), slack=0.2, mirror=False)
    # Cardano, one real root (a complex pair): both radicand signs through the mirror
    for al, be, ga in ((-1.0, 1.0, -0.5), (0.5, 2.0, -3.0), (-2.0, 0.3, 1.0), (-0.25, 4.0, -0.7)):
        add("cardano_one_real", I, np.array([[al, -be, 0], [be, al, 0], [0, 0, ga]]), slack=0.2)
        add("cardano_one_real", I, np.array([[al, -be, 0], [be, al, 0], [0, 0, ga]]), slack=0.0)
    # Cardano, three distinct real roots
    for diag, s in (([-1.0, -2.0, -4.0], 0.0), ([-1.0, -2.0, -4.0], 0.2), ([1.0, -2.0, -3.0], 0.2), ([-0.5, 3.0, -7.0], 0.0),
                    ([2.0, 3.0, -5.0], 0.2), ([-1.0, -1.1, -1.2], 0.2)):
        add("cardano_three_real", I, D(diag), slack=s)
    # two nearly equal real roots: a complex pair (1 +- i beta) / (1 + beta^2) with |Im| around tol, and an exact double root
    for be in (0.0, 1e-7, 5e-7, 1e-6, 1e-6 * (1 + 1e-6), 1e-6 * (1 - 1e-6), 2e-6, 1e-5):
        add("near_double", I, np.array([[-1.0, -be, 0], [be, -1.0, 0], [0, 0, -0.5]]), slack=0.0)
    add("near_double", I, D([-1.0, -1.0, -3.0]), slack=0.0)
    add("near_double", I, D([-1.0, -1.0 - 1e-9, -3.0]), slack=0.0)
    # |C| == 0: Delta0 = 0 and Delta1 < 0 (the contraction f = -e at slack > 0), the triple root at slack 0 (C = 0 on both branches)
    add("fallback", I, -I, slack=0.2)
    add("fallback", I, -I, slack=0.5)
    add("fallback", I, -I, slack=0.0)
    add("fallback", 2.0 * I, -2.0 * I, slack=0.0, h=0.5)
    # a root just above 0
    for r in (1e-8, 1e-13, 1e-15, 1e-17):
        add("near_zero", I, D([-1.0 / r, -1.0, -2.0]), slack=0.0)
    # uniform contraction P = -(X - centroid) at slack 0.2 (Delta0 at rounding level), on tets of every scale and offset
    for h, off in ((1.0, 0.0), (1e-3, 1e3), (1e-2, 1.0), (1e2, -1e3), (3e-3, 0.0)):
        E = I + 0.3 * rng.standard_normal((3, 3))
        X = np.vstack([np.zeros(3), h * E]) + off
        P = -(X - X.mean(0))
        out.append((FAMILIES.index("contraction"), X, P, 0.2))
    # rigid rotations: p = (R - I)(x - c)
    for ang in (0.3, 1.5, 3.0):
        for h, off in ((1.0, 0.0), (1e-2, 1e3)):
            E = I + 0.2 * rng.standard_normal((3, 3))
            X = np.vstack([np.zeros(3), h * E]) + off
            R = _rot(rng.standard_normal(3), ang)
            P = (X - X.mean(0)) @ (R - I).T
            out.append((FAMILIES.index("rotation"), X, P, 0.2))
    # slivers (height 1e-6 .. 1e-3 of the edge), random directions at the edge length
    for ht in (1e-3, 1e-6):
        for h in (1.0, 1e-3):
            E = np.array([[1.0, 0, 0], [0, 1.0, 0], [0.3, 0.4, ht]])
            for _ in range(2):
                X = np.vstack([np.zeros(3), h * E]) + rng.uniform(-1e3, 1e3, 3) * (h < 1)
                out.append((FAMILIES.index("sliver"), X, h * rng.standard_normal((4, 3)), 0.2))
    # random tets, inverted or not, edges 1e-3 .. 1e2, offsets up to 1e3, directions at 0.1 .. 3 edge lengths
    for k in range(48):
        h = 10.0 ** rng.uniform(-3, 2)
        X = h * rng.standard_normal((4, 3)) + rng.uniform(-1e3, 1e3, 3) * (k % 2)
        P = h * 10.0 ** rng.uniform(-1, 0.5) * rng.standard_normal((4, 3))
        out.append((FAMILIES.index("random"), X, P, 0.2))
    return out


def build():
    cs = cases()
    fam = np.array([c[0] for c in cs], dtype=np.int32)
    X = np.array([c[1] for c in cs])
    P = np.array([c[2] for c in cs])
    slack = np.array([c[3] for c in cs])
    return fam, X, P, slack


def main():
    fam, X, P, slack = build()
    rows = [evaluate(X[t], P[t], slack[t]) for t in range(len(fam))]
    out = dict(family=fam, X=X, P=P, slack=slack)
    for k in rows[0]:
        out[k] = np.array([r[k] for r in rows])
    np.savez_compressed(OUT, **out)
    print(f"{len(fam)} tets -> {OUT}")


if __name__ == "__main__":
    main()
