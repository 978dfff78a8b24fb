"""Generates tests/golden/contact_regimes_golden.npz: a soup of disjoint contact stencils (four own vertices each, one tet with mu = lam = 0
per stencil) placed where the per-pair barrier, mollifier and friction math degrades -- d/dHat from 1e-12 to 1 - 1e-10 over four dHat decades,
multiplicities, stencil sizes 1e-4 .. 1e2 at offsets up to 1e3, sliver triangles and edges, near-parallel and exactly parallel edges on both
sides of the mollifier switch, the PP friction basis tie -- with reference values evaluated in mpmath (50 digits) from the stored doubles
alone.  Nothing here reuses the kernels' difference-space derivation: the squared distances are written from their definitions
(point-point, point-line, point-plane, line-line) and differentiated by sympy, the barrier and mollifier are differentiated by hand in
closed form, and the chain rule is applied in 12 vertex coordinates.

Inputs stored (exactly what the kernels read): V, V_rest (4n,3); T (n,4) = 4k + (0,1,2,3); mm (n,4) the MMCVID encoding of pair k (global
vertex ids); moll (n,) the pair is on the mollified list, with pe (n,2) its two surface edges (indices into M.Mesh(V_rest, T).SFEdges) for
the sentinel PP / PE encodings and (-1,-1) otherwise; dHat, kappa (n,).  Friction (fric, the non-mollified pairs): V_prev (4n,3), eps2 (n,),
COEF; the lagged data lam (n,), coord (n,2), basis (n,6) are the exact lag of the stored V rounded to doubles.  kind (n,) 0 PT 1 EE 2 PE 3 PP
(of the distance stencil), family (index into FAMILIES), coef (the friction coefficient).

Outputs per pair, all in the tet's vertex order (12 coordinates; unused vertices are zero rows):
  d          the squared distance of the pair's stencil
  E, g, H    kappa mult b(d) (active) or kappa e(c) b(d) (mollified, c = |e1 x e2|^2 of the edge stencil, e the reference's
             q(c, eps_x) = (2 - c/eps_x) c/eps_x below eps_x and 1 above, eps_x = 1.0e-3 |a|^2 |b|^2 of the rest edges), and its exact
             gradient and Hessian (the chain rule on sympy's exact derivatives of d and c)
  Hp         the PSD projection of H (mp.eigsy, negative eigenvalues clamped to 0), what IglUtils::makePD computes
  psd        H has no negative eigenvalue in exact arithmetic (makePD returns its input).  In doubles that decision is deterministic only
             where H is exactly zero (family early_return, d == dHat); the e = 0 blocks of exactly parallel edges are PSD with exact zero
             eigenvalues, which any double evaluation turns into rounding noise of either sign, so they may take either path
  c_ratio    c / eps_x (mollified pairs; 0 elsewhere); switch: |c_ratio - 1| < 1e-8 + 64 eps (S_c / c + S_eps_x / eps_x), the rounding
             of c / eps_x in doubles (switch_width); there H_alt, Hp_alt hold the other branch's H, Hp
  S_d, S_E, S_g, S_H   componentwise first-order sensitivities sum_i |dQ/dx_i| |x_i| over V, dHat, kappa (and V_rest for mollified
             pairs), plus sum_j |dQ/dp_j| w_j over the components p_j of the cross products of d and c, w_j = |a_i b_k| + |a_k b_i| the size of
             their rounding (a rounding there tilts the normal in directions no input perturbation reaches: slivers, nearly parallel edges);
             forward differences at 50 digits with relative steps 1e-20 (a few digits are all the bars need; float32).  The lag's and the
             device-lagged friction terms' sensitivities add, the same way, the lag's cross products and its 2x2 Gram system (entries and
             right-hand sides, w = |u| |v|)
  friction lag: lam_ref, coord_ref, basis_ref (exact), S_lam, S_coord, S_basis; near_branch (PP: |x v01|^2 and |y v01|^2 within 1e-9
             relative of each other but not equal; an exact tie in small dyadic coordinates is deterministic and checked)
  friction terms from the stored lagged data: fE, fg, fH (= coef lam times f0, f1, f2 of the reference's C1 clamping, SFCLAMPING_ORDER 1),
             fHp (projected), u_ratio = |u|^2 / eps2, S_fE, S_fg, S_fH over V, V_prev, lam, coord, basis, eps2; S_fE_lag, S_fg_lag, S_fH_lag
             the same with the lag recomputed from V (the bar of the device-lagged run)
Run:  python tests/golden/gen_contact_regimes_golden.py   (about two minutes on eight cores)
"""
import functools
import multiprocessing
import os
import sys
import time

import mpmath as mp
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from ipc_b200 import mesh as M  # noqa: E402

OUT = os.path.join(HERE, "contact_regimes_golden.npz")
DPS = 50
STEP = mp.mpf("1e-20")  # relative forward-difference step of the sensitivities
COEF = 0.3
FAMILIES = ("sweep", "multiplicity", "scale", "sliver", "near_parallel", "parallel", "pp_tie", "early_return")
SWEEP = (1e-12, 1e-8, 1e-4, 0.1, 0.5, 0.9, 1 - 1e-6, 1 - 1e-10)
DHATS = (1e-10, 1e-6, 1e-3, 1.0)
U_RATIOS = (0.0, 1e-20, 0.25, 1 - 1e-12, 1.0, 1 + 1e-12, 4.0, 1e6)
PARALLEL = (1e-2, 1e-6, 1e-10, 1e-14, 1e-18)  # |e1 x e2|^2 / (|e1|^2 |e2|^2)
C_RATIOS = (1e-12, 1e-6, 0.5, 0.99, 1 - 1e-10, 1 + 1e-10, 4.0)
EPS_X = 1.0e-3  # the reference's literal (a double)


# ---------------------------------------------------------------------------------------------------------------------------------------
# cases (doubles)
# ---------------------------------------------------------------------------------------------------------------------------------------
def _rand_rot(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    Q = Q * np.sign(np.diag(R))
    return Q if np.linalg.det(Q) > 0 else -Q


def _rest(sa=1.0, sb=1.0):
    """rest tet with edge (0,1) along x (length sa) and edge (2,3) along y (length sb), one apart: eps_x = 1e-3 sa^2 sb^2"""
    return np.array([[0, 0, 0], [sa, 0, 0], [0, 0, 1.0], [0, sb, 1.0]])


def _stencil(kind, L, h, rng=None):
    """canonical 4-vertex stencils at squared distance h^2 (size L); unused vertices are padding"""
    if kind == 0:  # PT: point above the interior of a generic triangle
        return np.array([[0.3 * L, 0.3 * L, h], [0, 0, 0], [L, 0, 0], [0.3 * L, 0.9 * L, 0]])
    if kind == 1:  # EE: crossing edges 60 degrees apart, one above the other
        c, s = 0.5, np.sqrt(3) / 2
        return np.array([[-L / 2, 0, 0], [L / 2, 0, 0], [-c * L / 2, -s * L / 2, h], [c * L / 2, s * L / 2, h]])
    if kind == 2:  # PE: point beside the middle of an edge
        return np.array([[0.1 * L, h * np.cos(0.7), h * np.sin(0.7)], [-L / 2, 0, 0], [L / 2, 0, 0], [0, L, -L]])
    u = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])  # PP
    return np.array([[0, 0, 0], h * u, [L, 0, -L], [0, L, -L]])


def cases():
    """[dict(family, kind, x (4,3), X rest (4,3), dHat, kappa, mult, moll, sentinel, fric, u_ratio)] in fixture order; deterministic."""
    rng = np.random.default_rng(20261016)
    out = []

    def add(fam, kind, x, dHat, kappa, mult=1, moll=None, X=None, rot=True, off=0.0, fric=True, target=None):
        x = np.asarray(x, float)
        if rot:
            R = _rand_rot(rng)
            x = x @ R.T
        if off:
            x = x + off * rng.uniform(0.5, 1.0, 3) * rng.choice([-1, 1], 3)
        out.append(dict(family=FAMILIES.index(fam), kind=kind, x=x, X=_rest() if X is None else X, dHat=float(dHat), kappa=float(kappa),
                        mult=mult, moll=moll, fric=fric and moll is None, target=target))

    # d/dHat sweep: every ratio x kind x dHat decade, kappa alternating
    n = 0
    for r in SWEEP:
        for kind in range(4):
            for dHat in DHATS:
                add("sweep", kind, _stencil(kind, 3 * np.sqrt(dHat), np.sqrt(r * dHat)), dHat, (1.0, 1e9)[n % 2], target=r)
                n += 1
            n += 1
    # multiplicities of PP and PE (the duplicated-pair encodings, mm.w < -1)
    for kind in (2, 3):
        for mult in (1, 2, 3, 5):
            for dHat in (1e-2, 1e-6):
                add("multiplicity", kind, _stencil(kind, 3 * np.sqrt(dHat), np.sqrt(0.2 * dHat)), dHat, 1e4, mult=mult)
    # scale and offset
    for L in (1e-4, 1e-2, 1.0, 1e2):
        for off in (0.0, 1.0, 1e3):
            for kind in range(4):
                dHat = (0.1 * L) ** 2
                add("scale", kind, _stencil(kind, L, np.sqrt(0.3 * dHat)), dHat, 1e9 if kind % 2 else 1.0, off=off)
    for off in (0.0, 1e3):  # a point just inside a triangle edge: |p - t0| >> sqrt(d)
        L, h = 1.0, 1e-4
        add("scale", 0, [[0.5 * L, 1e-6 * L, h], [0, 0, 0], [L, 0, 0], [0.3 * L, 0.9 * L, 0]], 2 * h * h, 1e4, off=off)
    # slivers: triangles with height/base down to 1e-4, short edges against long ones
    for a in (1e-1, 1e-2, 1e-3, 1e-4):
        L, h = 1.0, 1e-3
        add("sliver", 0, [[0.4 * L, 0.3 * a * L, h], [0, 0, 0], [L, 0, 0], [0.4 * L, a * L, 0]], h * h / 0.3, 1e4)
    for a in (1e-1, 1e-2, 1e-3, 1e-4):
        L, h = 1.0, 1e-3
        c, s = 0.5, np.sqrt(3) / 2
        add("sliver", 1, [[-L / 2, 0, 0], [L / 2, 0, 0], [-c * a * L / 2, -s * a * L / 2, h], [c * a * L / 2, s * a * L / 2, h]], h * h / 0.3, 1e4)
        add("sliver", 2, [[0.1 * a * L, h, 0], [-a * L / 2, 0, 0], [a * L / 2, 0, 0], [0, L, -L]], h * h / 0.3, 1e4)
    # near-parallel edges on the EE stencil: mollified on both sides of the switch, and active (c >= eps_x) for friction
    for p2 in PARALLEL:
        L, h = 1.0, 1e-2
        th = np.arcsin(np.sqrt(p2))
        x = np.array([[-L / 2, 0, 0], [L / 2, 0, 0], [-L / 2 * np.cos(th), -L / 2 * np.sin(th), h], [L / 2 * np.cos(th), L / 2 * np.sin(th), h]])
        x = x @ _rand_rot(rng).T
        c = sum(mp.mpf(float(v)) ** 2 for v in np.cross(x[1] - x[0], x[3] - x[2]))  # (a first guess; the stored c_ratio is exact)
        for cq in C_RATIOS:
            s = float(mp.root(c / (mp.mpf(cq) * mp.mpf(EPS_X)), 4))
            add("near_parallel", 1, x, h * h * 2, 1e4, moll="EE", X=_rest(s, s), rot=False)
        add("near_parallel", 1, x, h * h * 2, 1e4, rot=False, X=_rest(1e-4, 1e-4))  # eps_x tiny: an ordinary active EE pair
    # exactly parallel edges (sentinel PP / PE encodings, e = 0) and nearly parallel ones on the same encodings
    for dHat in (0.1, 1e-3):
        s = np.sqrt(dHat / 0.1)
        pp = s * np.array([[0, 0, 0], [1, 0, 0], [1.25, 0.0625, 0], [2.25, 0.0625, 0]])
        pe = s * np.array([[0, 0, 0], [1, 0, 0], [0.5, 0.0625, 0], [1.5, 0.0625, 0]])
        add("parallel", 3, pp, dHat, 1e4, moll=("PP", 1, 2), rot=False)
        add("parallel", 2, pe, dHat, 1e4, moll=("PE", 2, 0), rot=False)
    for kind, base in ((3, [[0, 0, 0], [1, 0, 0], [1.25, 0.0625, 0], [2.25, 0.0625, 0]]), (2, [[0, 0, 0], [1, 0, 0], [0.5, 0.0625, 0], [1.5, 0.0625, 0]])):
        x = np.array(base, float)
        x[3, 2] += 1e-4  # b tilted out of plane by 1e-4: c / (|a|^2 |b|^2) = 1e-8
        a, b = x[1] - x[0], x[3] - x[2]
        c = float(np.sum(np.cross(a, b) ** 2))
        s = (c / (0.5 * EPS_X)) ** 0.25
        add("parallel", kind, x, 0.1, 1e4, moll=("PP", 1, 2) if kind == 3 else ("PE", 2, 0), X=_rest(s, s), rot=False)
    # the PP friction basis tie |x v01|^2 == |y v01|^2 (dyadic: exact in any order of evaluation), both sides, and a near tie
    for v in ([0.25, 0.25, 0.125], [0.25 * (1 + 1e-6), 0.25, 0.125], [0.25, 0.25 * (1 + 1e-6), 0.125], [0.25 * (1 + 1e-12), 0.25, 0.125]):
        x = np.array([[0.5, 0.5, 0.5], [0.5 + v[0], 0.5 + v[1], 0.5 + v[2]], [1.5, 0.5, 0.5], [0.5, 1.5, 0.5]])
        add("pp_tie", 3, x, 0.2, 1e4, rot=False)
    # d == dHat exactly in doubles (dyadic coordinates: every evaluation order gives the same d), so b = b' = b'' = 0 and the pair Hessian
    # is exactly zero: makePD's early return (no negative eigenvalue) is deterministic in doubles, unlike on the e = 0 blocks above whose
    # exact zero eigenvalues come out of any double evaluation as rounding noise of either sign
    t = [[0, 0, 0], [1, 0, 0], [0, 1, 0]]
    for kind, x in ((0, [[0.25, 0.25, 0.5]] + t), (1, [[-0.5, 0, 0], [0.5, 0, 0], [0, -0.5, 0.5], [0, 0.5, 0.5]]),
                    (2, [[0.25, 0.5, 0], [0, 0, 0], [1, 0, 0], [0, 1, -1]]), (3, [[0, 0, 0], [0.5, 0, 0], [1, 0, -1], [0, 1, -1]])):
        add("early_return", kind, x, 0.25, 1e4, rot=False, fric=False)
    # friction slip targets, cycled over the friction pairs
    k = 0
    for c in out:
        if c["fric"]:
            c["u_ratio"] = U_RATIOS[k % len(U_RATIOS)]
            k += 1
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# exact derivatives of the squared distances and of |e1 x e2|^2 (sympy, from the definitions)
# ---------------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _fn(name):
    import sympy as sp
    n = {"PP": 2, "PE": 3, "PT": 4, "EE": 4, "C": 4}[name]
    X = sp.symbols(f"x0:{3 * n}")
    D = sp.Matrix(sp.symbols("D0:3"))  # added to the cross product: its rounding
    P = [sp.Matrix(X[3 * i:3 * i + 3]) for i in range(n)]
    sq = lambda v: v.dot(v)  # noqa: E731
    if name == "PP":
        f = sq(P[0] - P[1])
    elif name == "PE":  # point-line: |(e0 - p) x (e1 - p)|^2 / |e1 - e0|^2
        f = sq((P[1] - P[0]).cross(P[2] - P[0]) + D) / sq(P[2] - P[1])
    elif name == "PT":  # point-plane
        nn = (P[2] - P[1]).cross(P[3] - P[1]) + D
        f = (P[0] - P[1]).dot(nn) ** 2 / sq(nn)
    elif name == "EE":  # line-line
        nn = (P[1] - P[0]).cross(P[3] - P[2]) + D
        f = (P[2] - P[0]).dot(nn) ** 2 / sq(nn)
    else:
        f = sq((P[1] - P[0]).cross(P[3] - P[2]) + D)
    g = [sp.diff(f, x) for x in X]
    H = [[sp.diff(gi, x) for x in X] for gi in g]
    return sp.lambdify(list(X) + list(D), [f, g, H], modules="mpmath", cse=True), n


def _dgH(name, xs, dn=None):
    """value, gradient (3n), Hessian (3n x 3n) at the mp coordinates xs (n x 3, flattened); dn is added to the cross product"""
    f, n = _fn(name)
    v, g, H = f(*xs, *(dn or (0, 0, 0)))
    return v, g, H


def cross_weights(name, xs):
    """|a_i b_j| + |a_j b_i| per component of the cross product a x b the function forms: the size of its rounding"""
    P = [xs[3 * i:3 * i + 3] for i in range(len(xs) // 3)]
    if name == "PP":
        return None
    if name == "PE":
        return _cw(_sub(P[1], P[0]), _sub(P[2], P[0]))
    if name == "PT":
        return _cw(_sub(P[2], P[1]), _sub(P[3], P[1]))
    return _cw(_sub(P[1], P[0]), _sub(P[3], P[2]))


KIND_NAME = ("PT", "EE", "PE", "PP")


def b_all(d, dHat):
    """the reference's C2 log barrier and its exact first two derivatives"""
    t = d - dHat
    lg = mp.log(d / dHat)
    return -t * t * lg, -2 * t * lg - t * t / d, -2 * lg - 4 * t / d + t * t / (d * d)


def q_all(c, ex, above=None):
    """the reference's mollifier q(c, eps_x) and its exact derivatives; above forces a branch"""
    if above is None:
        above = not (c < ex)
    if above:
        return mp.mpf(1), mp.mpf(0), mp.mpf(0)
    r = c / ex
    return (2 - r) * r, 2 / ex * (1 - r), -2 / (ex * ex)


def stencil_local(case):
    """local vertex ids of the distance stencil and (mollified) of the edge stencil"""
    k = case["kind"]
    nv = (4, 4, 3, 2)[k]
    if case["moll"] is None or case["moll"] == "EE":
        return list(range(nv)), ([0, 1, 2, 3] if case["moll"] == "EE" else None)
    _, p, q = case["moll"]
    if k == 3:
        return [p, q], [0, 1, 2, 3]
    return [p] + ([2, 3] if p < 2 else [0, 1]), [0, 1, 2, 3]


def barrier_eval(x, X, dHat, kappa, case, above=None, dn=None, dc=None):
    """E, d, g (12), H (12x12) of one pair, tet order; x, X (4,3) mp; dn, dc perturb the cross products of d and c"""
    sv, ev = stencil_local(case)
    xs = [x[v][i] for v in sv for i in range(3)]
    d, gd0, Hd0 = _dgH(KIND_NAME[case["kind"]], xs, dn)
    gd = [mp.mpf(0)] * 12
    Hd = [[mp.mpf(0)] * 12 for _ in range(12)]
    for a, va in enumerate(sv):
        for i in range(3):
            gd[3 * va + i] = gd0[3 * a + i]
            for b_, vb in enumerate(sv):
                for j in range(3):
                    Hd[3 * va + i][3 * vb + j] = Hd0[3 * a + i][3 * b_ + j]
    b, db, d2b = b_all(d, dHat)
    if ev is None:
        k = kappa * case["mult"]
        g = [k * db * gi for gi in gd]
        H = [[k * (d2b * gd[i] * gd[j] + db * Hd[i][j]) for j in range(12)] for i in range(12)]
        return k * b, d, g, H, mp.mpf(0)
    xe = [x[v][i] for v in ev for i in range(3)]
    c, gc, Hc = _dgH("C", xe, dc)
    Xe = [X[v] for v in ev]
    n2 = lambda a: sum(t * t for t in a)  # noqa: E731
    ex = mp.mpf(EPS_X) * n2([Xe[1][i] - Xe[0][i] for i in range(3)]) * n2([Xe[3][i] - Xe[2][i] for i in range(3)])
    e, de, d2e = q_all(c, ex, above)
    ge = [de * t for t in gc]
    g = [kappa * (b * ge[i] + e * db * gd[i]) for i in range(12)]
    H = [[kappa * (b * (d2e * gc[i] * gc[j] + de * Hc[i][j]) + db * (gd[i] * ge[j] + ge[i] * gd[j]) + e * (d2b * gd[i] * gd[j] + db * Hd[i][j]))
          for j in range(12)] for i in range(12)]
    return kappa * e * b, d, g, H, c / ex


def project(H):
    """PSD projection (eigenvalue clamp) of a symmetric mp matrix; (Hp, has a negative eigenvalue)"""
    n = len(H)
    A = mp.matrix(H)
    w, Q = mp.eigsy(A)
    wmax = max(abs(w[i]) for i in range(n))
    neg = any(w[i] < -mp.mpf("1e-35") * wmax for i in range(n))  # (below that: the 50-digit roundoff of a PSD matrix's zero eigenvalues)
    Hp = [[sum(max(w[k], 0) * Q[i, k] * Q[j, k] for k in range(n)) for j in range(n)] for i in range(n)]
    return Hp, neg


# ---------------------------------------------------------------------------------------------------------------------------------------
# friction (FrictionUtils.hpp restated: closest points, tangent bases, C1 clamping SFCLAMPING_ORDER 1)
# ---------------------------------------------------------------------------------------------------------------------------------------
def _sub(a, b): return [a[i] - b[i] for i in range(3)]
def _dot(a, b): return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
def _cross(a, b): return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
def _unit(a):
    z = _dot(a, a)
    return [t / mp.sqrt(z) for t in a] if z > 0 else a


def _dist(kind, xs, dn=(0, 0, 0)):
    """the squared distance alone, from the same definitions as _fn"""
    if kind == 3:
        r = _sub(xs[0], xs[1])
        return _dot(r, r)
    if kind == 2:
        n, e = _cross(_sub(xs[1], xs[0]), _sub(xs[2], xs[0])), _sub(xs[2], xs[1])
        n = [n[i] + dn[i] for i in range(3)]
        return _dot(n, n) / _dot(e, e)
    n = _cross(_sub(xs[2], xs[1]), _sub(xs[3], xs[1])) if kind == 0 else _cross(_sub(xs[1], xs[0]), _sub(xs[3], xs[2]))
    n = [n[i] + dn[i] for i in range(3)]
    s = _dot(_sub(xs[0], xs[1]), n) if kind == 0 else _dot(_sub(xs[2], xs[0]), n)
    return s * s / _dot(n, n)


def _vadd(a, b): return [a[i] + b[i] for i in range(3)]


def _cw(a, b):
    return [abs(a[(i + 1) % 3] * b[(i + 2) % 3]) + abs(a[(i + 2) % 3] * b[(i + 1) % 3]) for i in range(3)]


def _nrm(a): return mp.sqrt(_dot(a, a))


def lag_weights(kind, xs):
    """rounding sizes of the lag's intermediates: cross products |a_i b_j| + |a_j b_i|, dot products |u| |v|"""
    if kind == 3:
        return [0] * LAG_INT
    if kind == 0:
        r0, r1, rel = _sub(xs[2], xs[1]), _sub(xs[3], xs[1]), _sub(xs[0], xs[1])
        return _cw(r0, r1) + [_dot(r0, r0), _nrm(r0) * _nrm(r1), _dot(r1, r1), _nrm(r0) * _nrm(rel), _nrm(r1) * _nrm(rel)] + _cw(r0, r1)
    if kind == 1:
        e20, e01, e23 = _sub(xs[0], xs[2]), _sub(xs[1], xs[0]), _sub(xs[3], xs[2])
        return _cw(e01, e23) + [_dot(e01, e01), _nrm(e01) * _nrm(e23), _dot(e23, e23), _nrm(e20) * _nrm(e01), _nrm(e20) * _nrm(e23)] + _cw(e01, e23)
    e12, r = _sub(xs[2], xs[1]), _sub(xs[0], xs[1])
    return _cw(_sub(xs[1], xs[0]), _sub(xs[2], xs[0])) + [_dot(e12, e12), 0, 0, _nrm(r) * _nrm(e12), 0] + _cw(e12, r)


def _solve2(a, b, c, r0, r1):
    D = a * c - b * b
    return (c * r0 - b * r1) / D, (a * r1 - b * r0) / D


LAG_INT = 11  # intermediates of the lag: 3 cross product of d, 5 Gram system (a, b, c, r0, r1), 3 inner cross product of the basis


def lag_eval(x, dHat, kappa, case, pert=None, branch=None):
    """lambda, (c0, c1), basis (b0 | b1), PP tie gap: the exact lag of the stencil at x (mp, 4x3).  pert (LAG_INT): additive perturbations
    of the intermediates whose rounding the input sensitivity does not see, in units of their rounding size (see lag_weights).  branch
    forces the PP basis branch (the sensitivities keep the base point's: the basis is discontinuous at the tie)"""
    kind = case["kind"]
    sv, _ = stencil_local(case)
    xs = [x[v] for v in sv]
    w = lag_weights(kind, xs) if pert is not None else None
    p = [pert[i] * w[i] for i in range(LAG_INT)] if pert is not None else [0] * LAG_INT
    d = _dist(kind, xs, p[0:3])
    _, db, _ = b_all(d, dHat)
    lam = -kappa * db * 2 * mp.sqrt(d) * case["mult"]
    c0 = c1 = mp.mpf(0)
    gap = None
    if kind == 0:  # closest point on the triangle's plane
        r0, r1, rel = _sub(xs[2], xs[1]), _sub(xs[3], xs[1]), _sub(xs[0], xs[1])
        c0, c1 = _solve2(_dot(r0, r0) + p[3], _dot(r0, r1) + p[4], _dot(r1, r1) + p[5], _dot(r0, rel) + p[6], _dot(r1, rel) + p[7])
        b0, b1 = _unit(r0), _unit(_cross(_vadd(_cross(r0, r1), p[8:11]), r0))
    elif kind == 1:  # closest points of the two lines
        e20, e01, e23 = _sub(xs[0], xs[2]), _sub(xs[1], xs[0]), _sub(xs[3], xs[2])
        c0, c1 = _solve2(_dot(e01, e01) + p[3], -_dot(e23, e01) + p[4], _dot(e23, e23) + p[5], -_dot(e20, e01) + p[6], _dot(e20, e23) + p[7])
        b0, b1 = _unit(e01), _unit(_cross(_vadd(_cross(e01, e23), p[8:11]), e01))
    elif kind == 2:
        e12 = _sub(xs[2], xs[1])
        c0 = (_dot(_sub(xs[0], xs[1]), e12) + p[6]) / (_dot(e12, e12) + p[3])
        b0, b1 = _unit(e12), _unit(_vadd(_cross(e12, _sub(xs[0], xs[1])), p[8:11]))
    else:
        v01 = _sub(xs[1], xs[0])
        xc, yc = _cross([1, 0, 0], v01), _cross([0, 1, 0], v01)
        nx, ny = _dot(xc, xc), _dot(yc, yc)
        gap = (nx - ny) / (nx + ny)
        if (nx > ny) if branch is None else branch:
            b0, b1 = _unit(xc), _unit(_cross(v01, xc))
        else:
            b0, b1 = _unit(yc), _unit(_cross(v01, yc))
    return lam, [c0, c1], b0 + b1, gap


def fweights(kind, c):
    if kind == 0: return [1, -1 + c[0] + c[1], -c[0], -c[1]]
    if kind == 1: return [1 - c[0], c[0], c[1] - 1, -c[1]]
    if kind == 2: return [1, c[0] - 1, -c[0], 0]
    return [1, -1, 0, 0]


def fric_eval(x, xt, lam, co, ba, eps2, coef, case):
    """E, g (12), H (12x12) of the lagged friction term, tet order, from the given lagged data (exact in those inputs)"""
    kind = case["kind"]
    sv, _ = stencil_local(case)
    w = fweights(kind, co)
    rel = [sum(w[k] * (x[sv[k]][i] - xt[sv[k]][i]) for k in range(len(sv))) for i in range(3)]
    B = [ba[0:3], ba[3:6]]
    u = [_dot(B[0], rel), _dot(B[1], rel)]
    x2 = u[0] * u[0] + u[1] * u[1]
    eps = mp.sqrt(eps2)
    xn = mp.sqrt(x2)
    if x2 > eps2:
        f0, f1d, f2 = xn, 1 / xn, mp.mpf(0)
    else:
        f0 = x2 * (-xn / 3 + eps) / eps2 + eps / 3
        f1d, f2 = (-xn + 2 * eps) / eps2, 2 * (eps - xn) / eps2
    cl = coef * lam
    gu = [cl * f1d * u[0], cl * f1d * u[1]]
    if x2 > 0:
        uh = [u[0] / xn, u[1] / xn]
        Su = [[cl * (f1d * ((1 if a == b else 0) - uh[a] * uh[b]) + f2 * uh[a] * uh[b]) for b in range(2)] for a in range(2)]
    else:
        Su = [[cl * f1d * (1 if a == b else 0) for b in range(2)] for a in range(2)]
    T = [[mp.mpf(0)] * 2 for _ in range(12)]  # d u / d x (12 x 2)
    for k, v in enumerate(sv):
        for i in range(3):
            T[3 * v + i] = [w[k] * B[0][i], w[k] * B[1][i]]
    g = [T[i][0] * gu[0] + T[i][1] * gu[1] for i in range(12)]
    H = [[sum(T[i][a] * Su[a][b] * T[j][b] for a in range(2) for b in range(2)) for j in range(12)] for i in range(12)]
    return cl * f0, g, H, x2 / eps2


# ---------------------------------------------------------------------------------------------------------------------------------------
# per-pair evaluation
# ---------------------------------------------------------------------------------------------------------------------------------------
def _mpv(a):
    return [[mp.mpf(float(t)) for t in row] for row in np.asarray(a, dtype=float)]


def _flat(q):
    return np.array([float(t) for t in q]) if isinstance(q, list) and not isinstance(q[0], list) else (
        np.array([[float(t) for t in r] for r in q]) if isinstance(q, list) else np.array(float(q)))


def _sens(f, inputs, base, above):
    """componentwise sum |dQ/dz| |z| over the listed scalar inputs (forward differences, relative step STEP); f(inputs) -> list of Q"""
    acc = [np.zeros_like(np.asarray(b, dtype=float)) for b in base]
    for k, z in enumerate(inputs):
        if z == 0:
            continue
        h = STEP * abs(z)
        zz = list(inputs)
        zz[k] = z + h
        q = f(zz)
        for j in range(len(base)):
            acc[j] += np.abs(_flat(_lsub(q[j], base[j])) / float(h)) * float(abs(z))
    return [a.astype(np.float32) for a in acc]


def _lsub(a, b):
    if isinstance(a, list):
        return [_lsub(p, q) for p, q in zip(a, b)]
    return a - b


def switch_width(xm, Xm, case):
    """64 eps times the relative sensitivity of c / eps_x to the inputs and to the rounding of the cross product: within that of the
    switch, a double evaluation of c may land on either side (on edges 1e-9 rad from parallel it is about 1e-6)"""
    _, ev = stencil_local(case)
    xe = [xm[v][i] for v in ev for i in range(3)]
    c, gc, _ = _dgH("C", xe)
    if c == 0:
        return mp.mpf(0)
    n = _cross(_sub(xe[3:6], xe[0:3]), _sub(xe[9:12], xe[6:9]))
    S_c = sum(abs(gc[i]) * abs(xe[i]) for i in range(12)) + sum(2 * abs(n[j]) * w for j, w in enumerate(cross_weights("C", xe)))
    X = [Xm[v] for v in ev]
    a, b = _sub(X[1], X[0]), _sub(X[3], X[2])
    S_ex = 4 * sum(abs(a[i]) * (abs(X[1][i]) + abs(X[0][i])) for i in range(3)) / _dot(a, a) \
        + 4 * sum(abs(b[i]) * (abs(X[3][i]) + abs(X[2][i])) for i in range(3)) / _dot(b, b)  # relative, of eps_x = 1e-3 |a|^2 |b|^2
    return 64 * mp.mpf(2) ** -52 * (S_c / c + S_ex + 4)


def _sens_int(f, m, base):
    """sum_j |dQ/dp_j| over m intermediates p_j, each in units of its rounding size (forward differences, step STEP)"""
    acc = [np.zeros_like(np.asarray(b, dtype=float)) for b in base]
    for j in range(m):
        q = f(j, STEP)
        for i in range(len(base)):
            acc[i] += np.abs(_flat(_lsub(q[i], base[i])) / float(STEP))
    return [a.astype(np.float32) for a in acc]


def _add(a, b):
    return [(p + q).astype(np.float32) for p, q in zip(a, b)]


def evaluate(case, x, X, dHat, kappa, xt=None, eps2=None, lagged=None, sens=True):
    """every stored output of one pair from its stored doubles (dict of numpy arrays)"""
    mp.mp.dps = DPS
    xm, Xm = _mpv(x), _mpv(X)
    dH, kp = mp.mpf(float(dHat)), mp.mpf(float(kappa))
    E, d, g, H, cr = barrier_eval(xm, Xm, dH, kp, case)
    Hp, neg = project(H)
    out = dict(E=_flat(E), d=_flat(d), g=_flat(g), H=_flat(H), Hp=_flat(Hp), psd=not neg, c_ratio=_flat(cr))
    switch = case["moll"] is not None and abs(cr - 1) < mp.mpf("1e-8") + switch_width(xm, Xm, case)
    above = None
    if case["moll"] is not None:
        above = not (cr < 1)
    if switch:
        _, _, _, Ha, _ = barrier_eval(xm, Xm, dH, kp, case, above=not above)
        out["H_alt"], out["Hp_alt"] = _flat(Ha), _flat(project(Ha)[0])
    out["switch"] = switch
    if sens:
        moll = case["moll"] is not None
        z0 = [t for r in xm for t in r] + [dH, kp] + ([t for r in Xm for t in r] if moll else [])

        def fb(z):
            xx = [z[3 * i:3 * i + 3] for i in range(4)]
            XX = [z[14 + 3 * i:17 + 3 * i] for i in range(4)] if moll else Xm
            e_, d_, g_, H_, _ = barrier_eval(xx, XX, z[12], z[13], case, above=above)
            return [e_, d_, g_, H_]
        S = _sens(fb, z0, [E, d, g, H], above)
        # the roundings of the cross products of d and c, which no relative input perturbation reproduces (sliver triangles, nearly
        # parallel edges: a rounding tilts the normal in any direction, an input perturbation only about the edges)
        sv, ev = stencil_local(case)
        wn = cross_weights(KIND_NAME[case["kind"]], [xm[v][i] for v in sv for i in range(3)]) or [0, 0, 0]
        wc = cross_weights("C", [xm[v][i] for v in ev for i in range(3)]) if moll else [0, 0, 0]

        def fi(j, h):
            dn, dc = [0, 0, 0], [0, 0, 0]
            if j < 3:
                dn[j] = h * wn[j]
            else:
                dc[j - 3] = h * wc[j - 3]
            e_, d_, g_, H_, _ = barrier_eval(xm, Xm, dH, kp, case, above=above, dn=dn, dc=dc)
            return [e_, d_, g_, H_]
        S = _add(S, _sens_int(fi, 6, [E, d, g, H]))
        out["S_E"], out["S_d"], out["S_g"], out["S_H"] = S
    if xt is None:
        return out
    # friction: the exact lag of x (rounded = the stored lagged data), then E, g, H from the stored lagged data
    lam, co, ba, gap = lag_eval(xm, dH, kp, case)
    out.update(lam_ref=_flat(lam), coord_ref=_flat(co), basis_ref=_flat(ba))
    out["near_branch"] = gap is not None and gap != 0 and abs(gap) < mp.mpf("1e-9")
    out["pp_branch"] = -1 if gap is None else int(gap > 0)
    if lagged is None:
        return out
    xtm = _mpv(xt)
    lam_s, co_s, ba_s = mp.mpf(float(lagged[0])), [mp.mpf(float(t)) for t in lagged[1]], [mp.mpf(float(t)) for t in lagged[2]]
    e2, cf = mp.mpf(float(eps2)), mp.mpf(COEF)
    fE, fg, fH, ur = fric_eval(xm, xtm, lam_s, co_s, ba_s, e2, cf, case)
    out.update(fE=_flat(fE), fg=_flat(fg), fH=_flat(fH), fHp=_flat(project(fH)[0]), u_ratio=_flat(ur))
    if sens:
        z0 = [t for r in xm for t in r]
        br = None if gap is None else bool(gap > 0)
        S = _sens(lambda z: list(lag_eval([z[3 * i:3 * i + 3] for i in range(4)], z[12], z[13], case, branch=br)[:3]), z0 + [dH, kp], [lam, co, ba], None)

        def li(j, h):
            pert = [0] * LAG_INT
            pert[j] = h
            return list(lag_eval(xm, dH, kp, case, pert, br)[:3])
        out["S_lam"], out["S_coord"], out["S_basis"] = _add(S, _sens_int(li, LAG_INT, [lam, co, ba]))
        z1 = z0 + [t for r in xtm for t in r] + [lam_s] + co_s + ba_s + [e2]

        def ff(z):  # (E, g and H are continuous across the clamp, so a step that crosses it costs nothing)
            xx, tt = [z[3 * i:3 * i + 3] for i in range(4)], [z[12 + 3 * i:15 + 3 * i] for i in range(4)]
            return list(fric_eval(xx, tt, z[24], z[25:27], z[27:33], z[33], cf, case)[:3])
        out["S_fE"], out["S_fg"], out["S_fH"] = _sens(ff, z1, [fE, fg, fH], None)
        z2 = z0 + [t for r in xtm for t in r] + [dH, kp, e2]

        def fl(z):
            xx, tt = [z[3 * i:3 * i + 3] for i in range(4)], [z[12 + 3 * i:15 + 3 * i] for i in range(4)]
            lm, c_, b_, _ = lag_eval(xx, z[24], z[25], case, branch=br)
            return list(fric_eval(xx, tt, lm, c_, b_, z[26], cf, case)[:3])
        S = _sens(fl, z2, [fE, fg, fH], None)

        def fli(j, h):
            pert = [0] * LAG_INT
            pert[j] = h
            lm, c_, b_, _ = lag_eval(xm, dH, kp, case, pert, br)
            return list(fric_eval(xm, xtm, lm, c_, b_, e2, cf, case)[:3])
        out["S_fE_lag"], out["S_fg_lag"], out["S_fH_lag"] = _add(S, _sens_int(fli, LAG_INT, [fE, fg, fH]))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# soup
# ---------------------------------------------------------------------------------------------------------------------------------------
def soup(cs):
    """stored inputs of the case list (everything but the reference values); deterministic"""
    n = len(cs)
    V = np.concatenate([c["x"] for c in cs])
    Vr = np.concatenate([c["X"] for c in cs])
    T = (4 * np.arange(n)[:, None] + np.arange(4)[None, :]).astype(np.int32)
    m = M.Mesh(Vr, T)
    edge_id = {tuple(sorted(map(int, e))): i for i, e in enumerate(m.SFEdges)}
    mm = np.full((n, 4), -1, np.int32)
    pe = np.full((n, 2), -1, np.int32)
    for k, c in enumerate(cs):
        sv, ev = stencil_local(c)
        g = [4 * k + v for v in sv]
        if c["kind"] == 1:
            mm[k] = g
        elif c["kind"] == 0:
            mm[k] = [-g[0] - 1, g[1], g[2], g[3]]
        elif c["kind"] == 2:
            mm[k] = [-g[0] - 1, g[1], g[2], -c["mult"]]
        else:
            mm[k] = [-g[0] - 1, g[1], -1, -c["mult"]]
        if c["moll"] is not None and c["moll"] != "EE":
            pe[k] = [edge_id[(4 * k, 4 * k + 1)], edge_id[(4 * k + 2, 4 * k + 3)]]
    fam = np.array([c["family"] for c in cs], np.int32)
    kind = np.array([c["kind"] for c in cs], np.int32)
    moll = np.array([c["moll"] is not None for c in cs])
    fric = np.array([c["fric"] for c in cs])
    return dict(V=V, V_rest=Vr, T=T, mm=mm, pe=pe, moll=moll, fric=fric, family=fam, kind=kind,
                dHat=np.array([c["dHat"] for c in cs]), kappa=np.array([c["kappa"] for c in cs]))


def friction_inputs(cs, z):
    """the lagged data (exact lag rounded), V_prev and eps2 per friction pair: relDX = Delta in the lagged tangent plane with
    |u|^2 / eps2 at the pair's target (eps2 chosen from the realized slip where the target is within 1e-12 of the clamp or is it)"""
    n = len(cs)
    lamd, cod, bad = np.zeros(n), np.zeros((n, 2)), np.zeros((n, 6))
    Vp = z["V"].copy()
    eps2 = np.zeros(n)
    mp.mp.dps = DPS
    for k, c in enumerate(cs):
        if not c["fric"]:
            continue
        lam, co, ba, _ = lag_eval(_mpv(c["x"]), mp.mpf(c["dHat"]), mp.mpf(c["kappa"]), c)
        lamd[k], cod[k], bad[k] = float(lam), [float(t) for t in co], [float(t) for t in ba]
        sv, _ = stencil_local(c)
        L = float(np.linalg.norm(c["x"][sv].max(0) - c["x"][sv].min(0)))
        eps = 1e-2 * L
        r = c["u_ratio"]
        phi = 0.3 + 0.7 * k
        D = np.sqrt(r) * eps * (np.cos(phi) * bad[k, :3] + np.sin(phi) * bad[k, 3:])
        moved = [0, 1] if c["kind"] == 1 else [0]  # relDX = Delta (EE: (1 - c0) + c0)
        for v in moved:
            Vp[4 * k + v] = c["x"][v] - D
        eps2[k] = eps * eps
        if r > 0.5 and r < 2:
            xt = _mpv(Vp[4 * k:4 * k + 4])
            _, _, _, ur = fric_eval(_mpv(c["x"]), xt, mp.mpf(lamd[k]), [mp.mpf(t) for t in cod[k]], [mp.mpf(t) for t in bad[k]],
                                    mp.mpf(eps2[k]), mp.mpf(COEF), c)
            eps2[k] = float(ur * mp.mpf(eps2[k]) / mp.mpf(r))
    return lamd, cod, bad, Vp, eps2


def _work(args):
    c, x, X, dHat, kappa, xt, eps2, lagged = args
    return evaluate(c, x, X, dHat, kappa, xt, eps2, lagged)


def main():
    t0 = time.time()
    cs = cases()
    z = soup(cs)
    lam, co, ba, Vp, eps2 = friction_inputs(cs, z)
    z.update(V_prev=Vp, eps2=eps2, lam=lam, coord=co, basis=ba)
    n = len(cs)
    jobs = []
    for k, c in enumerate(cs):
        fr = c["fric"]
        jobs.append((c, z["V"][4 * k:4 * k + 4], z["V_rest"][4 * k:4 * k + 4], z["dHat"][k], z["kappa"][k], Vp[4 * k:4 * k + 4] if fr else None,
                     eps2[k], (lam[k], co[k], ba[k]) if fr else None))
    with multiprocessing.Pool(os.cpu_count() or 1) as pool:
        res = pool.map(_work, jobs, chunksize=1)
    shapes = dict(E=(), d=(), g=(12,), H=(12, 12), Hp=(12, 12), psd=(), c_ratio=(), switch=(), H_alt=(12, 12), Hp_alt=(12, 12),
                  S_E=(), S_d=(), S_g=(12,), S_H=(12, 12), lam_ref=(), coord_ref=(2,), basis_ref=(6,), near_branch=(), pp_branch=(),
                  fE=(), fg=(12,), fH=(12, 12), fHp=(12, 12), u_ratio=(), S_lam=(), S_coord=(2,), S_basis=(6,), S_fE=(), S_fg=(12,),
                  S_fH=(12, 12), S_fE_lag=(), S_fg_lag=(12,), S_fH_lag=(12, 12))
    for key, shp in shapes.items():
        proto = next(r[key] for r in res if key in r)
        dt = np.float32 if key.startswith("S_") else (bool if key in ("psd", "switch", "near_branch") else
                                                      (np.int32 if key == "pp_branch" else np.float64))
        a = np.zeros((n,) + shp, dt)
        if key == "pp_branch":
            a[:] = -1
        for k, r in enumerate(res):
            if key in r:
                a[k] = np.asarray(r[key], dtype=dt).reshape(shp)
        z[key] = a
        del proto
    z["families"] = np.array(FAMILIES)
    z["coef"] = np.float64(COEF)
    np.savez_compressed(OUT, **z)
    print(f"{n} pairs ({int(z['moll'].sum())} mollified, {int(z['fric'].sum())} with friction) -> {OUT} "
          f"({os.path.getsize(OUT) / 1e6:.2f} MB) in {time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()
