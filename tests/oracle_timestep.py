"""Float64 restatement of the time-integration frame of Optimizer (the oracle of csrc/timestep.cu and ipcgpu_warm_start). TEST INFRASTRUCTURE ONLY.

Every expression keeps the evaluation order of the reference's Eigen expressions (numpy rounds each elementwise operation once, with no fused
multiply-add), so the device results must match bit for bit:
  - computeXTilta (Optimizer.cpp:1236-1278), setTime (:421-428);
  - the end of a time step in Optimizer::solve for TIT_BE / TIT_NM (:572-590);
  - the predictors of initX, options 0-4 (:930-1080), and its step bound and backtracking loops (:1120-1215), composed from the existing
    oracle pieces (oracle.Elastic, oracle_halfspace, oracle.ccd_full_hashed, oracle.Surf.intersection_free).
Arrays are (nV, 3): positions, acceleration and dx_Elastic as the rows of their nV x 3 matrices, velocity as the interleaved 3 nV vector
reshaped, so that row v, column d is velocity component 3v + d (the reference's RowMatrixXd maps pair it with acceleration(v, d)).
"""
from fractions import Fraction as Fr

import numpy as np

BE, NM = 0, 1


class Params:
    """Optimizer::setTime: dtSq = dt * dt, gravityDtSq = dtSq * gravity"""

    def __init__(self, type, dt, beta=0.25, gamma=0.5, gravity=(0.0, -9.81, 0.0)):
        self.type, self.dt, self.beta, self.gamma = type, float(dt), float(beta), float(gamma)
        self.gravity = np.asarray(gravity, dtype=np.float64)
        self.dtSq = self.dt * self.dt
        self.gDtSq = self.dtSq * self.gravity


def fixed(dbc, nV):
    """Mesh::isDBCVertex: dbc != NOT_DBC"""
    return np.zeros(nV, bool) if dbc is None else np.asarray(dbc) != 0


def xtilde(P, Vprev, vel, acc, dbc=None):
    if P.type == BE:
        xt = Vprev + (vel * P.dt + P.gDtSq)
    else:
        xt = Vprev + ((vel * P.dt + P.beta * P.gDtSq) + (0.5 - P.beta) * (P.dtSq * acc))
    f = fixed(dbc, len(Vprev))
    xt[f] = Vprev[f]
    return xt


def end_time_step(P, V, Vprev, xt, vel, acc, dbc=None):
    """-> (velocity, acceleration, dx_Elastic, V_prev, xTilta) after Optimizer::solve's switch; xt is the x~ of the step that ends"""
    dxe = V - xt
    if P.type == BE:
        vel_new = (V - Vprev) / P.dt
        acc_new = (vel_new - vel) / P.dt
    else:
        v = vel + (P.dt * (1 - P.gamma)) * acc
        acc_new = (V - xt) / (P.dtSq * P.beta) + P.gravity
        vel_new = v + (P.dt * P.gamma) * acc_new
    Vprev_new = V.copy()
    return vel_new, acc_new, dxe, Vprev_new, xtilde(P, Vprev_new, vel_new, acc_new, dbc)


def predictor(P, option, vel, dxe, dbc=None):
    """initX's searchDir, (nV, 3); 0 on Dirichlet vertices and for option 0"""
    dv = P.dt * vel
    be = P.type == BE
    if option == 0:
        p = np.zeros_like(vel)
    elif option == 1:
        p = dv
    elif option == 2:
        p = dv + P.gDtSq if be else dv + P.gDtSq / 2.0
    elif option == 3:
        p = (dv + P.gDtSq) + dxe if be else (dv + P.gDtSq / 2.0) + dxe * 2.0
    elif option == 4:
        p = dv + (P.gDtSq + 0.5 * dxe) if be else (dv + P.gDtSq / 2.0) + dxe
    else:
        raise ValueError(option)
    p = p.copy()
    p[fixed(dbc, len(vel))] = 0.0
    return p


def step_forward(V0, t, p3):
    """V0 + t p as the device's stepForward computes it (csrc/misc.cu is compiled with contraction): one fused multiply-add per entry, rounded
    once (exact rational arithmetic, then one correctly rounded conversion)"""
    ft = Fr(t)
    return np.array([float(Fr(x) + ft * Fr(q)) for x, q in zip(V0.ravel(), p3.ravel())]).reshape(V0.shape)


def warm_start(m, P, option, vel, dxe, voxel, tol, evf, eee, planes=None, alpha_inversion=None):
    """initX(option) with solveIP: the predictor, its step bound (filterStepSize on Neo-Hookean meshes, the planes with slackness 0.9, the swept
    hash + full CCD) and the two backtracking loops; each loop ends at step 0 with an error, as ipcgpu_warm_start does.  `planes`: an
    oracle_halfspace.HalfSpaces factory taking an oracle.Surf.  The inversion filter's step agrees with the device's to 1e-9 only (elastic.cu
    rounds with fused multiply-adds, DESIGN §0 row (a) 8): given the device's `alpha_inversion`, the driver checks it to that bar and goes on
    from it, so that every later stage is compared bit for bit.  Returns a dict of p, the stage steps, alpha, V, the halvings and the status."""
    import oracle as orc
    V0 = m.V.copy()
    p3 = predictor(P, option, vel, dxe, m.dbc)
    p = np.ascontiguousarray(p3).ravel()
    r = dict(p=p, counts=[0, 0], status=0)
    if option == 0:
        return dict(r, alpha=0.0, V=V0)
    a = 1.0
    if m.energy == 0:  # getNeedElemInvSafeGuard: Neo-Hookean only
        a, _ = orc.Elastic(m).inversion_step(p, 0.2, a)
        if alpha_inversion is not None:
            assert abs(alpha_inversion - a) <= 1e-9 * a, (alpha_inversion, a)
            a = alpha_inversion
    r["alpha_inversion"] = a
    s = orc.Surf(m)
    if planes is not None:
        a = planes(s).step(p, 0.9, a)
        r["alpha_halfspace"] = a
    _, ag = orc.grid_swept(s, p, a, voxel)
    r["alpha_swept_grid"] = ag
    a, _, _ = orc.ccd_full_hashed(s, p, a, voxel, tol, evf, eee, nthreads=8)
    r["alpha_full_ccd"] = a
    step = lambda t: step_forward(V0, t, p3)

    def halve(t, k, bad):
        while bad(step(t)):
            if t == 0.0:
                return None
            t /= 2.0
            r["counts"][k] += 1
        return t

    if m.energy == 0:
        a = halve(a, 0, lambda V: orc.Elastic(m, V=V).count_inverted() > 0)
    if a is not None:
        def intersected(V):
            s2 = orc.Surf(m, V=V)
            return not s2.intersection_free()[0] or (planes is not None and planes(s2).crossings() > 0)
        a = halve(a, 1, intersected)
    if a is None:
        return dict(r, alpha=0.0, V=V0, status=8)
    return dict(r, alpha=a, V=step(a))
