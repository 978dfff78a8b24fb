"""Generates tests/golden/ccd_regimes_golden.npz: a soup of disjoint point-triangle and edge-edge stencils (four own vertices and one tet
with mu = lam = 0 each, as in the contact fixture) placed where the Tight-Inclusion narrow phase degenerates -- generic hits from toi 1e-9 to
1, impacts on a triangle's edge and vertex, coplanar and grazing motion, exactly and nearly parallel edges, zero-length edges and zero-area
triangles, zero relative motion (a static t axis, tol[0] = inf), sizes 1e-4 .. 1e2 at offsets up to 1e2, initial distances 0 and
1e-12 .. 1e-9, and searches whose levels outgrow 184 and 4,096 boxes or that end at the library's max_itr.

Inputs stored (exactly what the narrow phase reads): V, V_rest (4n,3); p (4n,3), the search direction; T (n,4) = 4k + (0,1,2,3);
kind (n,) 0 point-triangle (vertex 4k against face 4k+1..3) 1 edge-edge (edge 4k,4k+1 against edge 4k+2,4k+3); family (index into
FAMILIES).  The narrow phase forms x1 = fl(x0 + p) per vertex; so does everything here.

Reference values, in mpmath at 50 digits from the stored doubles only (nothing is shared with the oracle): the distance of two features
is written from its definition (point-triangle: the plane when the projection is inside, else the three edges; edge-edge: the four
endpoint-segment distances and the interior critical point of the two lines); class Ref turns it into first times and minima over time
(see there).  Stored for the record, at two levels s, 0 (column 0) and the pair's first ms = min(0.2 d0, 1e-6) (column 1):
  t_lo[k, j]   d > s on [0, t_lo)
  t_wit[k, j]  d(t_wit) <= s (inf: the distance stays above s on [0, 1])
  dmin[k, q]   a lower bound of the distance over [0, MAX_T[q]];  d0 the initial distance;  dev the bound of Ref's rigid model
tests/test_ccd_regimes.py evaluates Ref at the levels its bars need (the ms a search ended with, the tight bar's level).
Run:  python tests/golden/gen_ccd_regimes_golden.py   (about two minutes)
"""
import os

import mpmath as mp
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "ccd_regimes_golden.npz")
DPS = 50
MAX_T = (1.0, 0.37)
FAMILIES = ("generic", "boundary", "coplanar", "grazing", "parallel", "degenerate", "static", "scale", "initial", "wide")


def _rot(seed):
    rng = np.random.default_rng(seed)
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    Q = Q * np.sign(np.diag(R))
    return Q if np.linalg.det(Q) > 0 else -Q


def cases():
    """[(family, kind, x0 (4,3), p (4,3))] in fixture order; deterministic"""
    out = []

    def add(fam, kind, x, p, rot=None, off=None):
        x, p = np.asarray(x, float), np.asarray(p, float)
        if rot is not None:
            R = _rot(rot)
            x, p = x @ R.T, p @ R.T
        if off is not None:
            x = x + np.asarray(off, float)
        out.append((FAMILIES.index(fam), kind, x, p))

    tri = [[0, 0, 0], [1, 0, 0], [0.2, 0.9, 0]]
    down = lambda v: [[0, 0, -v], [0, 0, 0], [0, 0, 0], [0, 0, 0]]
    # generic hits: the point falls onto the triangle's interior with toi = 1e-9 .. 0.999 (toi < 1e-6: the ms = 0 retry runs)
    for toi in (1e-9, 3e-7, 1e-3, 0.25, 0.5, 0.999):
        h = 1e-3
        add("generic", 0, [[0.3, 0.3, h]] + tri, down(h / toi), rot=1)
    # a point 4e-7 above the face sinking by 1e-7: the first search returns toi = 0, one no_zero_toi trip (tolerance *= 0.1) follows and
    # the search ends with t_max
    add("generic", 0, [[0.3, 0.3, 4e-7]] + tri, down(1e-7), rot=2)
    # the ms = 0 retry with a hit: the first search (ms = 8e-7) reports 2^-20 < 1e-6, the retry finds 1.25 * 2^-20 and reports 0.8 x that
    add("generic", 0, [[0.3, 0.3, 4e-6], [0, 0, 0], [1, 0, 0], [0, 1, 0]], down(4e-6 / 1.3e-6))
    # contact exactly at max_t = 0.37
    add("generic", 0, [[0.3, 0.3, 1e-2]] + tri, down(1e-2 / 0.37))
    c, s = 0.5, np.sqrt(3) / 2
    for toi in (1e-8, 0.3, 0.75):
        h = 1e-2
        add("generic", 1, [[-0.5, 0, 0], [0.5, 0, 0], [-c / 2, -s / 2, h], [c / 2, s / 2, h]], [[0, 0, 0], [0, 0, 0], [0, 0, -h / toi], [0, 0, -h / toi]], rot=3)
    # impacts exactly on the triangle's boundary: an edge (u + v = 1: sum_le_1) and a vertex
    add("boundary", 0, [[0.6, 0.45, 1e-2]] + tri, down(2e-2))
    add("boundary", 0, [[0.5, 0.0, 1e-2]] + tri, down(2e-2))
    add("boundary", 0, [[1.0, 0.0, 1e-2]] + tri, down(2e-2))
    # coplanar motion: the point moves inside the triangle's plane, from outside into the face
    add("coplanar", 0, [[-0.5, 0.3, 0]] + tri, [[1.0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]])
    # grazing: the point slides parallel to the face, edges cross, at heights around ms = 1e-6 and err
    for h in (1e-6, 1e-6 + 1e-13, 1.5e-6, 1e-5):
        add("grazing", 0, [[-0.5, 0.3, h]] + tri, [[2.0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]])
    for h in (1e-6, 2e-6):
        add("grazing", 1, [[-0.5, 0, 0], [0.5, 0, 0], [0, -1, h], [0, 1, h]], [[0, 0, 0], [0, 0, 0], [-1, 0, 0], [-1, 0, 0]])
    # parallel edges at parallelism 0, 1e-12, 1e-6: approaching, sliding, both.  The first is the pair whose levels outgrow 4,096 boxes and
    # whose search ends at max_itr in the library
    h = 1e-3
    for tilt in (0.0, 1e-12, 1e-6):
        e = [[-1, 0, 0], [1, 0, 0], [-1, 0, h - tilt], [1, 0, h + tilt]]
        add("parallel", 1, e, [[0, 0, 0], [0, 0, 0], [0, 0, -2 * h], [0, 0, -2 * h]])
        add("parallel", 1, e, [[0, 0, 0], [0, 0, 0], [0.5, 0, 0], [0.5, 0, 0]])
        add("parallel", 1, e, [[0, 0, 0], [0, 0, 0], [0.5, 0, -2 * h], [0.5, 0, -2 * h]])
    # degenerate primitives: a zero-length edge, a zero-area triangle, a sliver triangle and edge
    add("degenerate", 1, [[-0.5, 0, 0], [0.5, 0, 0], [0, 0, 1e-2], [0, 0, 1e-2]], [[0, 0, 0], [0, 0, 0], [0, 0, -2e-2], [0, 0, -2e-2]])
    add("degenerate", 0, [[0.3, 0.1, 1e-2], [0, 0, 0], [1, 0, 0], [0.5, 0, 0]], down(2e-2))
    add("degenerate", 0, [[0.3, 0.1e-6, 1e-2], [0, 0, 0], [1, 0, 0], [0.5, 1e-6, 0]], down(2e-2))
    add("degenerate", 1, [[-0.5, 0, 0], [0.5, 0, 0], [0, -1e-6, 1e-2], [0, 1e-6, 1e-2]], [[0, 0, 0], [0, 0, 0], [0, 0, -2e-2], [0, 0, -2e-2]])
    # zero relative motion: dl = 0 gives tol[0] = inf; distance well above err, and 4e-8 against a per-pair err of about 2.5e-8 (with
    # ms = 8e-9 the root box just excludes the origin)
    for h in (1e-2, 4e-8):
        add("static", 0, [[0.3, 0.3, h]] + tri, [[0.1, 0.2, 0.3]] * 4)
        add("static", 1, [[-0.5, 0, 0], [0.5, 0, 0], [0, -0.5, h], [0, 0.5, h]], [[0.1, -0.2, 0.05]] * 4)
    # scale: sizes 1e-4 .. 1e2 at offsets up to 1e2
    for L, off in ((1e-4, 0.0), (1e-2, 10.0), (1.0, 100.0), (1e2, 0.0)):
        add("scale", 0, np.array([[0.3, 0.3, 0.05]] + tri) * L, np.array(down(0.1)) * L, rot=4, off=[off, -0.5 * off, 0.25 * off])
        add("scale", 1, np.array([[-0.5, 0, 0], [0.5, 0, 0], [-c / 2, -s / 2, 0.05], [c / 2, s / 2, 0.05]]) * L,
            np.array([[0, 0, 0], [0, 0, 0], [0, 0, -0.1], [0, 0, -0.1]]) * L, rot=5, off=[-off, off, 0.5 * off])
    # initial distance exactly 0 (the zero flag) and 1e-12 .. 1e-9 (ms = 0.2 d)
    add("initial", 0, [[0.3, 0.3, 0]] + tri, down(1e-3))
    for h in (1e-12, 1e-10, 1e-9):
        add("initial", 0, [[0.3, 0.3, h]] + tri, down(2 * h))
        add("initial", 1, [[-0.5, 0, 0], [0.5, 0, 0], [0, -0.5, h], [0, 0.5, h]], [[0, 0, 0], [0, 0, 0], [0, 0, -2 * h], [0, 0, -2 * h]])
    # wide searches: a point falling flat onto the triangle's plane from far, so that many boxes stay alive per level
    add("wide", 0, [[0.3, 0.3, 1e-4]] + tri, [[0.4, 0.3, -2e-4], [0, 0, 0], [0, 0, 0], [0, 0, 0]])
    add("wide", 1, [[-1, 0, 0], [1, 0, 0], [-1, 1e-4, 1e-4], [1, -1e-4, 1e-4]], [[0, 0, 0], [0, 0, 0], [0.3, 0, -2e-4], [0.3, 0, -2e-4]])
    return out


def soup(cs, spacing=4.0):
    """stencil k at x + (spacing * k, 0, 0) unless it carries its own offset; rest tets are regular"""
    n = len(cs)
    V = np.zeros((4 * n, 3)); P = np.zeros((4 * n, 3)); Vr = np.zeros((4 * n, 3))
    kind = np.zeros(n, np.int32); fam = np.zeros(n, np.int32)
    rest = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1.0]])
    for k, (f, kd, x, p) in enumerate(cs):
        shift = np.array([spacing * k, 0, 0]) if FAMILIES[f] != "scale" or np.abs(x).max() < 50 else np.zeros(3)
        if FAMILIES[f] == "scale" and np.abs(x).max() >= 50:
            shift = np.array([0, 0, 400.0 + 300.0 * (k % 2)])  # clear of the row of small stencils
        V[4 * k:4 * k + 4] = x + shift
        P[4 * k:4 * k + 4] = p
        Vr[4 * k:4 * k + 4] = rest + np.array([spacing * k, -10.0, 0])
        kind[k], fam[k] = kd, f
    T = (4 * np.arange(n)[:, None] + np.arange(4)[None, :]).astype(np.int32)
    return V, Vr, P, T, kind, fam


# ---- mpmath reference ------------------------------------------------------------------------------------------------------------------
def _sub(a, b): return [a[i] - b[i] for i in range(3)]
def _dot(a, b): return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
def _cross(a, b): return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _pt_seg(p, a, b):
    ab = _sub(b, a)
    L = _dot(ab, ab)
    t = mp.mpf(0) if L == 0 else min(max(_dot(_sub(p, a), ab) / L, mp.mpf(0)), mp.mpf(1))
    q = [a[i] + t * ab[i] for i in range(3)]
    return mp.sqrt(_dot(_sub(p, q), _sub(p, q)))


def dist(kind, x):
    """distance of the two features at the positions x (4 points, mpf)"""
    if kind == 0:
        p, a, b, c = x
        ds = [_pt_seg(p, a, b), _pt_seg(p, b, c), _pt_seg(p, c, a)]
        n = _cross(_sub(b, a), _sub(c, a))
        nn = _dot(n, n)
        if nn > 0:
            ap = _sub(p, a)
            # barycentric coordinates of the projection
            w1 = _dot(_cross(_sub(a, p), _sub(b, p)), n) / nn
            w2 = _dot(_cross(_sub(b, p), _sub(c, p)), n) / nn
            w3 = _dot(_cross(_sub(c, p), _sub(a, p)), n) / nn
            if w1 >= 0 and w2 >= 0 and w3 >= 0:
                ds.append(abs(_dot(ap, n)) / mp.sqrt(nn))
        return min(ds)
    a0, a1, b0, b1 = x
    ds = [_pt_seg(a0, b0, b1), _pt_seg(a1, b0, b1), _pt_seg(b0, a0, a1), _pt_seg(b1, a0, a1)]
    u, v, w = _sub(a1, a0), _sub(b1, b0), _sub(a0, b0)
    A, B, C, D, E = _dot(u, u), _dot(u, v), _dot(v, v), _dot(u, w), _dot(v, w)
    den = A * C - B * B
    if den > 0:
        s = (B * E - C * D) / den
        t = (A * E - B * D) / den
        if 0 < s < 1 and 0 < t < 1:
            q = [w[i] + s * u[i] - t * v[i] for i in range(3)]
            ds.append(mp.sqrt(_dot(q, q)))
    return min(ds)


def at(x0, x1, t):
    return [[x0[k][i] + t * (x1[k][i] - x0[k][i]) for i in range(3)] for k in range(4)]


class Ref:
    """Exact reference of one pair from its stored doubles.  In every stencil here one feature translates relative to the other: each
    side's vertices share a velocity up to the rounding of x1 = fl(x0 + p).  With the side's first vertex as its velocity, the distance of
    the rigidly translated pair is d_r(t) = dist(t w, A0 - B0), w the relative velocity and A0 - B0 the triangle (point-triangle) or the
    parallelogram (edge-edge) of differences: the distance of a point moving on a line to a convex set, a CONVEX function of t.  The true
    distance differs from it by at most dev * t, dev the largest deviation of a vertex's velocity from its side's (convexity of the
    features), so first times and minima of d_r, found by golden-section search and bisection to 1e-40, bound the true ones:
      first(s) -> (t_lo, t_wit): d > s on [0, t_lo) (first time of d_r at s + dev), d(t_wit) <= s (first time of d_r at s - dev, or of
                  d_r at s where the true distance there is checked to be <= s); inf where there is none on [0, 1]
      dmin(T)  -> a lower bound of the true distance over [0, T]"""

    def __init__(self, kind, x0d, x1d):
        self.kind = kind
        self.x0 = [[mp.mpf(float(v)) for v in r] for r in x0d]
        self.x1 = [[mp.mpf(float(v)) for v in r] for r in x1d]
        vel = [_sub(self.x1[k], self.x0[k]) for k in range(4)]
        A, B = ((1, 2, 3), (0,)) if kind == 0 else ((0, 1), (2, 3))
        self.dev = sum(max(mp.sqrt(_dot(_sub(vel[i], vel[S[0]]), _sub(vel[i], vel[S[0]]))) for i in S) for S in (A, B))
        self.w = _sub(vel[B[0]], vel[A[0]])
        x = self.x0
        if kind == 0:
            self.tris = [[_sub(x[i], x[0]) for i in (1, 2, 3)]]
        else:
            q = [_sub(x[0], x[2]), _sub(x[1], x[2]), _sub(x[1], x[3]), _sub(x[0], x[3])]
            self.tris = [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]

    def d_rigid(self, t):
        pt = [t * c for c in self.w]
        return min(dist(0, [pt] + tri) for tri in self.tris)

    def d_true(self, t):
        return dist(self.kind, at(self.x0, self.x1, t))

    def argmin(self, T):
        lo, hi = mp.mpf(0), mp.mpf(T)
        g = (mp.sqrt(5) - 1) / 2
        for _ in range(200):
            a, b = hi - g * (hi - lo), lo + g * (hi - lo)
            if self.d_rigid(a) <= self.d_rigid(b):
                hi = b
            else:
                lo = a
        return min((mp.mpf(0), lo, mp.mpf(T)), key=self.d_rigid)

    def _first(self, s, tm):
        """first time d_rigid <= s on [0, 1] as a bracket (lo: d_r > s, hi: d_r <= s); None where it stays above s"""
        if self.d_rigid(mp.mpf(0)) <= s:
            return mp.mpf(0), mp.mpf(0)
        if self.d_rigid(tm) > s:
            return None
        lo, hi = mp.mpf(0), tm
        for _ in range(160):
            mid = (lo + hi) / 2
            if self.d_rigid(mid) <= s:
                hi = mid
            else:
                lo = mid
        return lo, hi

    def first(self, s):
        s = mp.mpf(s)
        tm = self.argmin(1)
        lo = self._first(s + self.dev, tm)
        t_lo = lo[0] if lo else mp.inf
        wit = self._first(s - self.dev, tm) if s - self.dev >= 0 else None
        if wit:
            t_wit = wit[1]
        else:
            at_s = self._first(s, tm)
            t_wit = at_s[1] if at_s and self.d_true(at_s[1]) <= s else mp.inf
        return t_lo, t_wit

    def dmin(self, T):
        return self.d_rigid(self.argmin(T)) - self.dev * mp.mpf(T)


def reference(kind, x0d, x1d, max_ts):
    r = Ref(kind, x0d, x1d)
    d0 = r.d_true(mp.mpf(0))
    ms = min(0.2 * float(d0), 1e-6)
    rows = [r.first(lv) for lv in (0.0, ms)]
    dm = [r.dmin(mt) for mt in max_ts]
    return [float(x[0]) for x in rows], [float(x[1]) for x in rows], [float(x) for x in dm], float(d0), float(r.dev)


def build():
    mp.mp.dps = DPS
    cs = cases()
    V, Vr, P, T, kind, fam = soup(cs)
    X1 = V + P  # fl(x0 + p), as the narrow phase forms it
    n = len(cs)
    t_lo = np.zeros((n, 2)); t_wit = np.zeros((n, 2)); dmin = np.zeros((n, len(MAX_T))); d0 = np.zeros(n); dev = np.zeros(n)
    for k in range(n):
        a, b, c, d, v = reference(int(kind[k]), V[4 * k:4 * k + 4], X1[4 * k:4 * k + 4], MAX_T)
        t_lo[k], t_wit[k], dmin[k], d0[k], dev[k] = a, b, c, d, v
    return dict(V=V, V_rest=Vr, p=P, T=T, kind=kind, family=fam, t_lo=t_lo, t_wit=t_wit, dmin=dmin, d0=d0, dev=dev,
                max_t=np.array(MAX_T), families=np.array(FAMILIES))


if __name__ == "__main__":
    np.savez_compressed(OUT, **build())
    print("wrote", OUT)
