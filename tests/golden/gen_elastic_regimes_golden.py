"""Generates tests/golden/elastic_regimes_golden.npz: a tet soup (disjoint tets, four own vertices each) whose deformation gradients sit where
the per-tet elastic path branches -- every exit and both sorts of the 3x3 SVD, repeated and nearly repeated singular values, near-singular,
singular and inverted F, large stretch, sliver and scaled rest shapes -- with reference values evaluated in mpmath (70 digits) from the
stored doubles alone.

Inputs stored (exactly what the kernels read): V (deformed) and V_rest (nV,3), T (nT,4), restTriInv (nT,9, per-tet column-major as in
ipc_b200.mesh.Mesh), vol, mu, lam, energy (0 = NeoHookean, 1 = FixedCoRot).  F = Ds * restTriInv is formed in high precision from those
doubles; the structured families use the unit right tet (restTriInv = I), so F is exactly the matrix written below.

Outputs per tet (coef = 1):
  E        psi * vol
  g        the 12-gradient, vol * dF/dx^T P, with NH  P = mu (F - F^-T) + lam ln J F^-T  (no SVD)
                                                  FCR P = 2 mu (F - R) + lam (J - 1) cof F, R the polar factor in the rotation-variant
                                                          convention of the reference's SVD (det R = +1; for det F < 0 the smallest singular
                                                          direction is flipped, gen_elastic_golden.polar_R)
  H        the UNprojected 12x12 Hessian vol * G^T (dP/dF) G, dP/dF by central differences of P at two step sizes scaled to the smallest
           quantity P is differentiated through (sigma_min for NH, min sigma_i + sigma_j for FCR) that must agree to 1e-25.  Where the
           reference's 1e-6 floor on sigma_i + sigma_j is active (Energy.cpp:448-562) the reference does not compute the derivative; there H is
           the sigma-space formula as the reference states it, and floor_active is set.
  Hp       the projected Hessian: the sigma-space formula with makePD of the 3x3 A block (eigenvalue clamp, mp.eigsy) and the reference's
           makePD2d formula on the three 2x2 B blocks, as it stands (DESIGN 3.4: it is not the eigenvalue clamp).
  basis_spread, basis_spread_H, basis_spread_g
           where two singular values are within 1e-6 sigma_max of each other (or of each other's negative), the same quantities evaluated in
           further valid SVD bases, rotated within the (near-)degenerate plane; the largest max-abs difference to the stored value.  Zero
           elsewhere.  basis_spread is that of Hp; _H and _g are nonzero only where the floor makes H or the polar factor basis-dependent.
  near_branch
           an eigenvalue of the A block, or the smaller eigenvalue L2 of a B block, within 1e-9 (relative) of 0: the projection switches there.
  a_indef  the A block has a negative eigenvalue (the kernel's Jacobi path clamps).
  sigma    singular values in the rotation-variant convention (only the last may be negative); family (index into FAMILIES).
Run:  python tests/golden/gen_elastic_regimes_golden.py
"""
import os

import mpmath as mp
import numpy as np

DPS = 70
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "elastic_regimes_golden.npz")
FLOOR = mp.mpf("1e-6")  # Energy.cpp: eps on sigma_i + sigma_j
FAMILIES = ("generic", "repeated", "rotation", "near_repeated", "svd_exit", "near_singular", "singular", "inverted", "stretch", "det_only",
            "rest_shape", "zero_material")


# ---------------------------------------------------------------------------------------------------------------------------------------
# cases (doubles)
# ---------------------------------------------------------------------------------------------------------------------------------------
def _rot(axis, ang):
    a = np.asarray(axis, float)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _rand_rot(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    Q = Q * np.sign(np.diag(R))
    return Q if np.linalg.det(Q) > 0 else -Q


UNIT = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1.0]])
MAT0 = (100.0 / 2 / 1.4, 100.0 * 0.4 / 1.4 / 0.2)  # YM = 100, PR = 0.4: the reference's unit-test material (Energy.cpp:588)


def cases():
    """[(family, energy, mu, lam, X rest (4,3), x deformed (4,3))] in fixture order; deterministic."""
    rng = np.random.default_rng(20261016)
    out = []

    def mat():
        # half the tets on the reference material, the rest log-uniform mu in [0.1, 1e3], lam / mu in [0, 30]
        if rng.random() < 0.5:
            return MAT0
        mu = 10 ** rng.uniform(-1, 3)
        return mu, mu * (0.0 if rng.random() < 0.1 else rng.uniform(0.05, 30))

    def add(fam, F, ets=(0, 1), X=UNIT, material=None):
        F = np.asarray(F, dtype=np.float64)
        for et in ets:
            if et == 0 and not np.linalg.det(F) > 0:
                continue  # NH is undefined for det F <= 0
            mu, lam = material if material is not None else mat()
            x = X[0] + (X - X[0]) @ F.T if X is not UNIT else np.vstack([np.zeros(3), F.T])
            out.append((fam, et, float(mu), float(lam), np.array(X, float), x))

    def usv(s, Q1=None, Q2=None):
        Q1 = _rand_rot(rng) if Q1 is None else Q1
        Q2 = _rand_rot(rng) if Q2 is None else Q2
        return Q1 @ np.diag(s) @ Q2.T

    for _ in range(10):  # control
        add("generic", usv(rng.uniform(0.5, 2.0, 3)))
    # exactly repeated singular values: diagonal and permutation forms are exact; rotated forms repeat them to rounding
    for s in [(1.3, 1.3, 0.8), (1.3, 0.8, 0.8), (0.8, 0.8, 0.8), (1.5, 1.5, 1.2), (1.2, 1.0, 1.0), (0.7, 0.7, 0.5)]:
        add("repeated", np.diag(s))
        Q = _rand_rot(rng)
        add("repeated", usv(s, Q, Q))
        add("repeated", usv(s))
    add("repeated", 0.8 * np.eye(3))
    add("repeated", 1.25 * np.eye(3))
    for P in ([[0, 1, 0], [0, 0, 1], [1, 0, 0.0]], [[0, 0, 1], [1, 0, 0], [0, 1, 0.0]], [[0, 1, 0], [1, 0, 0], [0, 0, 1.0]],
              [[1, 0, 0], [0, 0, 1], [0, 1, 0.0]]):  # two even (det +1), two odd (det -1: FCR only)
        add("repeated", P)
        add("repeated", 1.1 * np.array(P))
    # pure rotations, 180 degrees included
    add("rotation", np.diag([-1.0, -1.0, 1.0]))
    add("rotation", np.diag([1.0, -1.0, -1.0]))
    add("rotation", _rot([1, 1, 0], np.pi))
    add("rotation", _rot([0.3, -0.5, 0.8], np.pi))
    for _ in range(3):
        add("rotation", _rand_rot(rng))
    add("rotation", np.eye(3))
    # nearly repeated: relative gaps 1e-4, 1e-8, 1e-12 between the top pair, the bottom pair, and all three
    for g in (1e-4, 1e-8, 1e-12):
        add("near_repeated", np.diag([1.2 * (1 + g), 1.2, 0.7]))
        add("near_repeated", np.diag([1.3, 0.9, 0.9 * (1 - g)]))
        add("near_repeated", usv([1.1 * (1 + g), 1.1, 0.6]))
        add("near_repeated", usv([1.4, 0.8 * (1 + g), 0.8]))
        add("near_repeated", usv([1.0 + g, 1.0, 1.0 - g]))
    # every exit of svd3 and both branches of both sorts
    add("svd_exit", np.diag([1.0, 2.0, 3.0]))                                 # beta_2 exit, sort0 reorders (s1 > s0 after the swap)
    add("svd_exit", np.diag([3.0, 1.0, 2.0]))                                 # beta_2 exit, sort0 reorders (else branch)
    add("svd_exit", np.diag([1.5, 1.2, 0.9]))                                 # beta_2 exit, sort0 early return
    add("svd_exit", [[1.0, 0, 0], [0, 3.0, 1.0], [0, 0, 2.0]])                # F(0,1) = 0: beta_1 exit, sort1 reorders
    add("svd_exit", [[3.0, 0, 0], [0, 1.0, 0.5], [0, 0, 0.8]])                # beta_1 exit, sort1 early return
    add("svd_exit", [[0.5, 0, 0], [0, 1.0, 2.0], [0, 0, 1.5]])                # beta_1 exit, sort1 reorders twice
    add("svd_exit", [[1.2, 0.4, 0], [0, 0.0, 0.7], [0, 0, 0.9]])              # zero second pivot: alpha_2 exit
    add("svd_exit", [[0.6, 0.4, 0], [0, 0.0, 1.7], [0, 0, 0.9]])
    add("svd_exit", [[1.2, 0.4, 0], [0, 0.9, 0.7], [0, 0, 0.0]])              # zero third pivot: alpha_3 exit
    add("svd_exit", [[0.3, 0.4, 0], [0, 1.9, 0.7], [0, 0, 0.0]])
    add("svd_exit", [[0.0, 0.4, 0], [0, 0.9, 0.7], [0, 0, 1.1]])              # zero first column: alpha_1 exit
    add("svd_exit", [[0.0, 0.4, 0.2], [0, 0.9, 0.7], [0, -0.3, 1.1]])
    add("svd_exit", [[0.0, 2.0, 0], [0, 0.5, 0.2], [0, 0, 0.4]])
    add("svd_exit", [[1.0, 0, 0], [0.3, 0.9, 0], [0.2, -0.1, 1.1]])           # lower triangular
    add("svd_exit", [[0.8, 0, 0], [-0.4, 1.3, 0], [0.5, 0.6, 0.7]])
    add("svd_exit", [[1.1, 0.2, -0.1], [0, 0.9, 0.3], [0, 0, 1.2]])           # upper triangular
    # near-singular
    for s3 in (1e-4, 1e-8, 1e-12):
        add("near_singular", np.diag([1.3, 0.9, s3]))
        add("near_singular", usv([1.2, 0.8, s3]))
        add("near_singular", usv([2.5, 1.5, s3]))
    # FCR only: exactly singular
    add("singular", np.diag([1.2, 0.8, 0.0]), ets=(1,))
    add("singular", [[1.0, 0.5, 0.0], [-0.25, 0.75, 0.0], [0.5, 0.125, 0.0]], ets=(1,))     # rank 2 (zero column)
    add("singular", [[0.5, 1.0, 0.0], [0.25, 0.5, 0.0], [-0.75, -1.5, 0.0]], ets=(1,))      # rank 1
    add("singular", np.diag([1.3, 0.0, 0.0]), ets=(1,))
    add("singular", np.zeros((3, 3)), ets=(1,))
    # FCR only: inverted, sigma_2 + sigma_3 on either side of the floor, and |sigma_3| ~ sigma_2
    for s in [(1.2, 5e-7, -2e-7), (1.2, 3e-6, -1e-6), (1.1, 0.6, -0.6), (1.1, 0.6, -0.6 * (1 - 1e-8)), (1.1, 0.8, -0.5), (0.9, 0.7, -0.7 * (1 - 1e-4))]:
        add("inverted", np.diag(s), ets=(1,))
        add("inverted", usv(s), ets=(1,))
    # large stretch (NH: A block indefinite; FCR: B blocks indefinite)
    for s in [(100.0, 1.0, 0.5), (100.0, 30.0, 2.0), (20.0, 5.0, 0.3), (3.0, 2.5, 2.0), (8.0, 8.0, 1.0)]:
        add("stretch", np.diag(s))
        add("stretch", usv(s))
    # FCR A block with non-negative diagonal and 2x2 minors but a negative determinant: only the det term of the early return sees it
    for s in [(0.72, 0.7, 0.68), (0.7, 0.69, 0.66), (0.74, 0.71, 0.7)]:
        add("det_only", usv(s), ets=(1,), material=(1.0, 20.0))
    # rest shapes: slivers, scaled by 1e-3 and 1e3
    for X in (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.3, 0.3, 1e-3]]), np.array([[0, 0, 0], [1, 0, 0], [0.5, 1e-3, 0], [0.5, 0, 1.0]]),
              1e-3 * UNIT + 0.25, 1e3 * UNIT - 7.0):
        add("rest_shape", usv(rng.uniform(0.6, 1.6, 3)), X=X)
        add("rest_shape", usv([1.3, 0.9, 1e-4]), X=X)
    # NH with mu = lam = 0 (the kernels return zeros), FCR with mu = 0 and with lam = 0
    add("zero_material", usv([1.2, 0.9, 0.8]), ets=(0,), material=(0.0, 0.0))
    add("zero_material", np.diag([2.0, 0.5, 0.1]), ets=(0,), material=(0.0, 0.0))
    add("zero_material", usv([1.2, 0.9, 0.8]), ets=(1,), material=(0.0, 40.0))
    add("zero_material", usv([1.2, 0.9, -0.8]), ets=(1,), material=(30.0, 0.0))
    # spread the families over tile positions
    order = rng.permutation(len(out))
    return [out[i] for i in order]


def soup(cs):
    """(V, V_rest, T, restTriInv, vol, mu, lam, energy, family) arrays of the soup; the vertex ids inside a tet are permuted so that the
    kernel's orientation of off-diagonal blocks (rows to the smaller global id) takes both ways"""
    n = len(cs)
    rng = np.random.default_rng(7)
    V, Vr, T = np.empty((4 * n, 3)), np.empty((4 * n, 3)), np.empty((n, 4), np.int32)
    Ainv, vol = np.empty((n, 9)), np.empty(n)
    for t, (_, _, _, _, X, x) in enumerate(cs):
        perm = rng.permutation(4)
        T[t] = 4 * t + perm
        V[T[t]] = x
        Vr[T[t]] = X
        Dm = np.stack([X[1] - X[0], X[2] - X[0], X[3] - X[0]], axis=1)
        Ainv[t] = np.linalg.inv(Dm).T.ravel()  # per-tet column-major
        vol[t] = np.linalg.det(Dm) / 6.0
    mu = np.array([c[2] for c in cs])
    lam = np.array([c[3] for c in cs])
    et = np.array([c[1] for c in cs], np.int32)
    fam = np.array([FAMILIES.index(c[0]) for c in cs], np.int32)
    return V, Vr, T, Ainv, vol, mu, lam, et, fam


# ---------------------------------------------------------------------------------------------------------------------------------------
# reference values (mpmath)
# ---------------------------------------------------------------------------------------------------------------------------------------
def cof(F):
    return mp.matrix([[F[1, 1] * F[2, 2] - F[1, 2] * F[2, 1], F[1, 2] * F[2, 0] - F[1, 0] * F[2, 2], F[1, 0] * F[2, 1] - F[1, 1] * F[2, 0]],
                      [F[0, 2] * F[2, 1] - F[0, 1] * F[2, 2], F[0, 0] * F[2, 2] - F[0, 2] * F[2, 0], F[0, 1] * F[2, 0] - F[0, 0] * F[2, 1]],
                      [F[0, 1] * F[1, 2] - F[0, 2] * F[1, 1], F[0, 2] * F[1, 0] - F[0, 0] * F[1, 2], F[0, 0] * F[1, 1] - F[0, 1] * F[1, 0]]])


def det3(F):
    C = cof(F)  # (mp.det pivots through LU and fails on exactly singular F)
    return F[0, 0] * C[0, 0] + F[0, 1] * C[0, 1] + F[0, 2] * C[0, 2]


def svd_rv(F):
    """F = U diag(S) V^T, det U = det V = +1, S descending in magnitude with only S[2] allowed negative (the reference's convention)"""
    U0, S0, Vt0 = mp.svd_r(F)
    idx = sorted(range(3), key=lambda k: -S0[k])
    U, V, S = mp.matrix(3, 3), mp.matrix(3, 3), [S0[k] for k in idx]
    for c, k in enumerate(idx):
        for r in range(3):
            U[r, c], V[r, c] = U0[r, k], Vt0[k, r]
    for M in (U, V):
        if det3(M) < 0:
            for r in range(3):
                M[r, 2] = -M[r, 2]
            S[2] = -S[2]
    return U, S, V


def P_closed(et, F, mu, lam, R=None):
    J = det3(F)
    C = cof(F)
    if et == 0:
        if mu == 0 and lam == 0:
            return mp.zeros(3, 3)
        FinvT = C / J
        return mu * (F - FinvT) + lam * mp.log(J) * FinvT
    if R is None:
        U, _, V = svd_rv(F)
        R = U * V.T
    return 2 * mu * (F - R) + lam * (J - 1) * C


def psi(et, F, S, mu, lam):
    if et == 0:
        if mu == 0 and lam == 0:
            return mp.mpf(0)
        J = det3(F)
        return mu / 2 * (sum(F[i, j] ** 2 for i in range(3) for j in range(3)) - 3) - mu * mp.log(J) + lam / 2 * mp.log(J) ** 2
    return mu * sum((s - 1) ** 2 for s in S) + lam / 2 * (S[0] * S[1] * S[2] - 1) ** 2


def dPdF_fd(et, F, mu, lam, h):
    D = mp.matrix(9, 9)
    for r in range(3):
        for s in range(3):
            Fp, Fm = F.copy(), F.copy()
            Fp[r, s] += h
            Fm[r, s] -= h
            dP = (P_closed(et, Fp, mu, lam) - P_closed(et, Fm, mu, lam)) / (2 * h)
            for i in range(3):
                for j in range(3):
                    D[3 * i + j, 3 * r + s] = dP[i, j]
    return D


def sigma_blocks(et, S, mu, lam):
    """dpsi/dsigma, d2psi/dsigma2 and the B-block 'left' coefficients (NeoHookeanEnergy.cpp:71-136, FixedCoRotEnergy.cpp:72-143)"""
    if et == 0:
        if mu == 0 and lam == 0:
            return [mp.mpf(0)] * 3, mp.zeros(3, 3), [mp.mpf(0)] * 3
        lJ = mp.log(S[0] * S[1] * S[2])
        dE = [mu * (s - 1 / s) + lam / s * lJ for s in S]
        A = mp.matrix(3, 3)
        for i in range(3):
            A[i, i] = mu * (1 + 1 / S[i] ** 2) - lam * (lJ - 1) / S[i] ** 2
            for j in range(3):
                if i != j:
                    A[i, j] = lam / (S[i] * S[j])
        mid = mu - lam * lJ
        BL = [(mu + mid / (S[c] * S[(c + 1) % 3])) / 2 for c in range(3)]
        return dE, A, BL
    J = S[0] * S[1] * S[2]
    n = [S[1] * S[2], S[2] * S[0], S[0] * S[1]]
    dE = [2 * mu * (S[i] - 1) + n[i] * lam * (J - 1) for i in range(3)]
    A = mp.matrix(3, 3)
    for i in range(3):
        A[i, i] = 2 * mu + lam * n[i] ** 2
        for j in range(3):
            if i != j:
                k = 3 - i - j
                A[i, j] = lam * (S[k] * (J - 1) + n[i] * n[j])
    BL = [mu - lam / 2 * S[(c + 2) % 3] * (J - 1) for c in range(3)]
    return dE, A, BL


def make_pd(A):
    E, Q = mp.eigsy(A)
    if min(E) >= 0:
        return A
    Ec = [max(e, 0) for e in E]
    return Q * mp.diag(Ec) * Q.T


def make_pd2d(a, b, d):
    """IglUtils.hpp:138-177 as it stands, on the symmetric block [[a, b], [b, d]]"""
    D = a * d - b * b
    Th = (a + d) / 2
    sq = mp.sqrt(Th * Th - D)
    L2 = Th - sq
    if L2 < 0:
        L1 = Th + sq
        if L1 <= 0:
            return mp.mpf(0), mp.mpf(0), mp.mpf(0)
        if b == 0:
            return L1, mp.mpf(0), mp.mpf(0)
        L1md = L1 - d
        r = L1md / L1
        return r * L1md, b * r, b * b / L1
    return a, b, d


def dPdF_sigma(et, U, S, V, mu, lam, project):
    """compute_dP_div_dF (Energy.cpp:448-562): sigma-space 9x9 M, rotated by U, V (row-major vec(F) index 3i+j)"""
    dE, A, BL = sigma_blocks(et, S, mu, lam)
    if project:
        A = make_pd(A)
    M = mp.matrix(9, 9)
    for i in range(3):
        for j in range(3):
            M[4 * i, 4 * j] = A[i, j]
    for c in range(3):
        cp = (c + 1) % 3
        ssum = S[c] + S[cp]
        right = (dE[c] + dE[cp]) / (2 * (FLOOR if ssum < FLOOR else ssum))
        p, q, r = BL[c] + right, BL[c] - right, BL[c] + right
        if project:
            p, q, r = make_pd2d(p, q, r)
        # pair (c, cp): M(c cp, c cp) = p, M(cp c, cp c) = r, M(c cp, cp c) = M(cp c, c cp) = q
        a, b = 3 * c + cp, 3 * cp + c
        M[a, a], M[b, b], M[a, b], M[b, a] = p, r, q, q
    nz = [(a, b) for a in range(9) for b in range(9) if M[a, b] != 0]
    D = mp.matrix(9, 9)
    for i in range(3):
        for j in range(3):
            for r in range(3):
                for s in range(3):
                    D[3 * i + j, 3 * r + s] = mp.fsum(M[kl, mn] * U[i, kl // 3] * V[j, kl % 3] * U[r, mn // 3] * V[s, mn % 3] for kl, mn in nz)
    return D


def near_branch(et, S, mu, lam):
    dE, A, BL = sigma_blocks(et, S, mu, lam)
    tol = mp.mpf("1e-9")
    E = mp.eigsy(A)[0]
    amax = max(abs(e) for e in E)
    if min(abs(e) for e in E) <= tol * amax:
        return True
    for c in range(3):
        cp = (c + 1) % 3
        ssum = S[c] + S[cp]
        right = (dE[c] + dE[cp]) / (2 * (FLOOR if ssum < FLOOR else ssum))
        L1, L2 = max(2 * BL[c], 2 * right), min(2 * BL[c], 2 * right)  # eigenvalues of [[BL+r, BL-r],[BL-r, BL+r]]
        if abs(L2) <= tol * max(abs(L1), abs(L2)):
            return True
    return False


def _plane_rot(i, j, th):
    Q = mp.eye(3)
    c, s = mp.cos(th), mp.sin(th)
    Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
    return Q


def other_bases(S):
    """(QU, QV) with U QU, V QV another valid SVD basis of F when singular values are (nearly) repeated (same rotation of U and V), (nearly)
    opposite (opposite rotations) or both (nearly) zero (independent rotations).  The turns sample each family finely, up to a relative turn
    of pi and a common turn of pi/2 (the projected blocks depend on double angles); three equal values rotate freely in 3D."""
    smax = max(abs(s) for s in S)
    tol = mp.mpf("1e-6") * smax
    q = mp.pi / 16
    out = []
    same = [abs(S[i] - S[j]) <= tol for i, j in ((0, 1), (1, 2), (0, 2))]
    for (i, j), sm in zip(((0, 1), (1, 2), (0, 2)), same):
        opp = abs(S[i] + S[j]) <= tol
        if sm and opp:  # both (nearly) zero: independent turns
            out += [(_plane_rot(i, j, a), _plane_rot(i, j, a + k * q)) for a in (0, 4 * q) for k in range(1, 32)]
        elif sm:
            out += [(_plane_rot(i, j, k * q), _plane_rot(i, j, k * q)) for k in range(1, 16)]
        elif opp:
            out += [(_plane_rot(i, j, k * q), _plane_rot(i, j, -k * q)) for k in range(1, 16)]
    if all(same):
        for a in range(3):
            for b in range(1, 4):
                for c in range(3):
                    Q = _plane_rot(0, 1, 2 * a * mp.pi / 3) * _plane_rot(0, 2, b * mp.pi / 6) * _plane_rot(0, 1, 2 * c * mp.pi / 3)
                    out.append((Q, Q if smax > 0 else _plane_rot(1, 2, b * mp.pi / 3) * Q))
    return out


def polar_turns(S):
    """relative turns QU QV^T of U and V that keep F (and change R = U V^T): a fine circle in every plane where that is free, because the
    largest entry-wise change of an affine function of (cos, sin) need not sit at a turn of pi"""
    smax = max(abs(s) for s in S)
    tol = mp.mpf("1e-6") * smax
    planes = [(i, j) for i, j in ((0, 1), (1, 2), (0, 2)) if abs(S[i] + S[j]) <= tol or smax == 0]
    return [_plane_rot(i, j, k * mp.pi / 32) for i, j in planes for k in range(1, 64)]


def evaluate(et, mu, lam, x, Ainv_cm, vol):
    """reference values of one tet from its stored doubles"""
    mp.mp.dps = DPS
    mu, lam, vol = mp.mpf(float(mu)), mp.mpf(float(lam)), mp.mpf(float(vol))
    A = mp.matrix(3, 3)
    for i in range(3):
        for j in range(3):
            A[i, j] = mp.mpf(float(Ainv_cm[i + 3 * j]))
    X = [[mp.mpf(float(v)) for v in row] for row in x]
    Ds = mp.matrix(3, 3)
    for c in range(3):
        for r in range(3):
            Ds[r, c] = X[c + 1][r] - X[0][r]
    F = Ds * A
    U, S, V = svd_rv(F)
    Gv = [[-(A[0, j] + A[1, j] + A[2, j]) for j in range(3)]] + [[A[c, j] for j in range(3)] for c in range(3)]
    G = mp.matrix(9, 12)
    for a in range(4):
        for k in range(3):
            for j in range(3):
                G[3 * k + j, 3 * a + k] = Gv[a][j]

    def grad(P):
        return [vol * mp.fsum(P[k, j] * Gv[a][j] for j in range(3)) for a in range(4) for k in range(3)]

    def hess(D):
        return vol * (G.T * D * G)

    floor_active = et == 1 and min(S[0] + S[1], S[1] + S[2], S[0] + S[2]) < FLOOR
    E = vol * psi(et, F, S, mu, lam)
    g = grad(P_closed(et, F, mu, lam, R=U * V.T))
    if floor_active:
        D = dPdF_sigma(et, U, S, V, mu, lam, 0)
    else:
        scale = abs(S[2]) if et == 0 else min(S[0] + S[1], S[1] + S[2], S[0] + S[2])
        h = mp.mpf("1e-18") * min(scale, 1)
        D = dPdF_fd(et, F, mu, lam, h)
        D2 = dPdF_fd(et, F, mu, lam, h / 3)
        dmax = max(abs(v) for v in D)
        assert max(abs(a - b) for a, b in zip(D, D2)) <= mp.mpf("1e-25") * max(dmax, mp.mpf("1e-300")), "central differences disagree"
    H = hess(D)
    Hp = hess(dPdF_sigma(et, U, S, V, mu, lam, 1))
    spread = [mp.mpf(0)] * 3  # Hp, H, g
    nb = near_branch(et, S, mu, lam)
    for QU, QV in ([] if nb else other_bases(S)):  # (near_branch tets are checked for properties only)
        U2, V2 = U * QU, V * QV
        Hp2 = hess(dPdF_sigma(et, U2, S, V2, mu, lam, 1))
        spread[0] = max(spread[0], max(abs(a - b) for a, b in zip(Hp, Hp2)))
        if floor_active:
            H2 = hess(dPdF_sigma(et, U2, S, V2, mu, lam, 0))
            spread[1] = max(spread[1], max(abs(a - b) for a, b in zip(H, H2)))
    if et == 1:
        for Q in polar_turns(S):
            g2 = grad(P_closed(et, F, mu, lam, R=U * Q * V.T))
            spread[2] = max(spread[2], max(abs(a - b) for a, b in zip(g, g2)))
    # differences at the working precision's noise level (dps 70) are no basis dependence
    for k, M in ((0, Hp), (1, H)):
        if spread[k] <= mp.mpf("1e-40") * max(abs(v) for v in M):
            spread[k] = mp.mpf(0)
    if spread[2] <= mp.mpf("1e-40") * max(abs(v) for v in g):
        spread[2] = mp.mpf(0)
    _, Ablk, _ = sigma_blocks(et, S, mu, lam)
    a_indef = min(mp.eigsy(Ablk)[0]) < 0
    f = lambda M: np.array([float(v) for v in M], dtype=np.float64)
    return {"E": float(E), "g": f(g), "H": f(H).reshape(12, 12), "Hp": f(Hp).reshape(12, 12), "sigma": f(S),
            "floor_active": bool(floor_active), "near_branch": bool(nb), "a_indef": bool(a_indef),
            "basis_spread": float(spread[0]), "basis_spread_H": float(spread[1]), "basis_spread_g": float(spread[2])}


def main():
    cs = cases()
    V, Vr, T, Ainv, vol, mu, lam, et, fam = soup(cs)
    n = len(cs)
    res = [evaluate(et[t], mu[t], lam[t], V[T[t]], Ainv[t], vol[t]) for t in range(n)]
    out = {"V": V, "V_rest": Vr, "T": T, "restTriInv": Ainv, "vol": vol, "mu": mu, "lam": lam, "energy": et, "family": fam,
           "families": np.array(FAMILIES)}
    for k in res[0]:
        out[k] = np.array([r[k] for r in res])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, n, "tets:", int((et == 0).sum()), "NH,", int((et == 1).sum()), "FCR;",
          int(out["floor_active"].sum()), "floor_active,", int((out["basis_spread"] > 0).sum()), "basis-dependent,",
          int(out["near_branch"].sum()), "near_branch,", int(out["a_indef"].sum()), "with an indefinite A block")


if __name__ == "__main__":
    main()
