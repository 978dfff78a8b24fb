// halfspace.cpp -- CPU ORACLE (test infrastructure) of the analytic half-space collision objects, HalfSpace<3>
// (src/CollisionObject/HalfSpace.cpp, CollisionObject.h, Optimizer.cpp).  Compiled with -ffp-contract=off: n.x is summed as
// (n0 x0 + n1 x1) + n2 x2, the order the device kernels (ipc_b200/csrc/halfspace.cu, --fmad=false) use, so sets, counts and step bounds are
// bit-identical.  Planes: 8 doubles each [n0 n1 n2 D v0 v1 v2 mu]; entries (plane, vertex) interleaved.
#include "oracle.h"
#include <algorithm>
#include <cmath>

namespace {

double dist_of(const double* pl, const orc_surf* s, int v)
{
    const int n = s->nV;
    return ((pl[0] * s->V[v] + pl[1] * s->V[n + v]) + pl[2] * s->V[2 * n + v]) + pl[3];
}
bool dbc_of(const orc_surf* s, int v) { return s->dbc && s->dbc[v] != 0; }
bool codim3(const orc_surf* s, int v) { return !s->vCoDim || s->vCoDim[v] == 3; }
bool proj(const orc_surf* s, int v, int projectDBC) { return s->dbc && (s->dbc[v] == 1 || (s->dbc[v] == 2 && projectDBC)); }

// upper triangle of a 3x3 block (row-major M) into the vertex's diagonal block (LinSysSolver::addCoeff on the upper-triangular CSR)
void add_block(const int* ia, const int* ja, int base, int v, const double* M, double* a)
{
    for (int r = 0; r < 3; ++r)
        for (int q = r; q < 3; ++q) {
            const int row = 3 * v + r, col = 3 * v + q;
            for (int k = ia[row] - base; k < ia[row + 1] - base; ++k)
                if (ja[k] - base == col) { a[k] += M[3 * r + q]; break; }
        }
}

struct Slip {
    double u[3], mag2;
};
// HalfSpace.cpp:285-288: VDiff = (x - x_prev) - velocitydt, VProj = VDiff - (VDiff.n) n
Slip slip_of(const double* pl, const double* x, const double* xt)
{
    double vd[3];
    for (int r = 0; r < 3; ++r) vd[r] = (x[r] - xt[r]) - pl[4 + r];
    const double un = (vd[0] * pl[0] + vd[1] * pl[1]) + vd[2] * pl[2];
    Slip s;
    for (int r = 0; r < 3; ++r) s.u[r] = vd[r] - un * pl[r];
    s.mag2 = (s.u[0] * s.u[0] + s.u[1] * s.u[1]) + s.u[2] * s.u[2];
    return s;
}
void pos(const orc_surf* s, const double* V, int v, double* x)
{
    for (int r = 0; r < 3; ++r) x[r] = V[(size_t)r * s->nV + v];
}

} // namespace

extern "C" {

/* HalfSpace::init (HalfSpace.cpp:42-52): normal.normalize(), D = -normal.dot(origin) */
void orc_hs_planes(int n, const double* origin, const double* normal, const double* velocitydt, const double* friction, double* par)
{
    for (int k = 0; k < n; ++k) {
        const double* nr = normal + 3 * k;
        const double* o = origin + 3 * k;
        const double z = (nr[0] * nr[0] + nr[1] * nr[1]) + nr[2] * nr[2];
        const double sq = std::sqrt(z);
        double* q = par + 8 * k;
        for (int r = 0; r < 3; ++r) q[r] = nr[r] / sq;
        q[3] = -((q[0] * o[0] + q[1] * o[1]) + q[2] * o[2]);
        for (int r = 0; r < 3; ++r) q[4 + r] = velocitydt ? velocitydt[3 * k + r] : 0.0;
        q[7] = friction[k];
    }
}

/* CollisionObject::computeConstraintSet (CollisionObject.h:323-352) per plane, concatenated over the planes */
int orc_hs_constraint_set(const orc_surf* s, int nP, const double* par, double dHat, int* act2)
{
    int n = 0;
    for (int k = 0; k < nP; ++k)
        for (int sv = 0; sv < s->nSV; ++sv) {
            const int v = s->SVI[sv];
            if (dbc_of(s, v) || !codim3(s, v)) continue;
            const double dist = dist_of(par + 8 * k, s, v);
            if (dist * dist < dHat) { act2[2 * n] = k; act2[2 * n + 1] = v; ++n; }
        }
    return n;
}

/* kappa * sum b(d) (Optimizer.cpp:3254-3267, serial sum); returns 1 where the reference would exit (d <= 0) */
int orc_hs_energy(const orc_surf* s, const double* par, const int* act2, int n, double dHat, double kappa, double* E)
{
    double sum = 0.0;
    int bad = 0;
    for (int c = 0; c < n; ++c) {
        const double dist = dist_of(par + 8 * act2[2 * c], s, act2[2 * c + 1]), d = dist * dist;
        if (d <= 0.0) { bad = 1; continue; }
        double b, db, d2b;
        orc_barrier(d, dHat, &b, &db, &d2b);
        sum += b;
    }
    *E = kappa * sum;
    return bad;
}

/* HalfSpace::leftMultiplyConstraintJacobianT (:121-143) with input b'(d): g += coef input 2 dist n */
void orc_hs_gradient(const orc_surf* s, const double* par, const int* act2, int n, double dHat, double kappa, double* g)
{
    for (int c = 0; c < n; ++c) {
        const double* pl = par + 8 * act2[2 * c];
        const int v = act2[2 * c + 1];
        const double dist = dist_of(pl, s, v), d = dist * dist;
        double b, db, d2b;
        orc_barrier(d, dHat, &b, &db, &d2b);
        const double f = kappa * db * 2.0 * dist;
        for (int r = 0; r < 3; ++r) g[3 * v + r] += f * pl[r];
    }
}

/* one entry's block, row-major: project = 1 the reference's (param > 0 ? kappa param nn^T : 0, HalfSpace.cpp:169-213), 0 the unprojected
 * kappa (b'' (2 dist)^2 + 2 b') nn^T = kappa (4 b'' d + 2 b') nn^T */
void orc_hs_barrier_block(const double* pl, double dist, double dHat, double kappa, int project, double* H9)
{
    const double d = dist * dist;
    double b, db, d2b;
    orc_barrier(d, dHat, &b, &db, &d2b);
    const double param = 4.0 * d2b * d + 2.0 * db;
    const double s = (project && !(param > 0.0)) ? 0.0 : kappa * param;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) H9[3 * i + j] = s * (pl[i] * pl[j]);
}

void orc_hs_hessian_csr(const orc_surf* s, const double* par, const int* act2, int n, double dHat, double kappa, int projectDBC, const int* ia, const int* ja,
    int base, double* a)
{
    for (int c = 0; c < n; ++c) {
        const double* pl = par + 8 * act2[2 * c];
        const int v = act2[2 * c + 1];
        if (proj(s, v, projectDBC)) continue;
        double H[9];
        orc_hs_barrier_block(pl, dist_of(pl, s, v), dHat, kappa, 1, H);
        add_block(ia, ja, base, v, H, a);
    }
}

/* HalfSpace::largestFeasibleStepSize (:242-269) of every plane in turn; a bound <= 0 is returned as 0 */
void orc_hs_step(const orc_surf* s, int nP, const double* par, const double* p, double slackness, double* alpha)
{
    for (int k = 0; k < nP; ++k) {
        const double* pl = par + 8 * k;
        double m = 1.0;
        for (int sv = 0; sv < s->nSV; ++sv) {
            const int v = s->SVI[sv];
            if (dbc_of(s, v)) continue;
            const double c = (pl[0] * p[3 * v] + pl[1] * p[3 * v + 1]) + pl[2] * p[3 * v + 2];
            if (c < 0.0) m = std::min(m, -dist_of(pl, s, v) / c * slackness);
        }
        *alpha = std::min(*alpha, m);
    }
    if (!(*alpha > 0.0)) *alpha = 0.0;
}

/* CollisionObject::isIntersected (:386-401), counted: (plane, vertex) with codim 3, not Dirichlet, dist^2 <= 0 */
int orc_hs_crossings(const orc_surf* s, int nP, const double* par)
{
    int n = 0;
    for (int v = 0; v < s->nV; ++v) {
        if (!codim3(s, v) || dbc_of(s, v)) continue;
        for (int k = 0; k < nP; ++k) {
            const double dist = dist_of(par + 8 * k, s, v);
            n += dist * dist <= 0.0;
        }
    }
    return n;
}

/* Optimizer.cpp:1555-1572: planes with friction > 0 are lagged, lambda = -kappa 2 sqrt(d) b'(d) */
int orc_hs_lag(const orc_surf* s, const double* par, const int* act2, int n, double dHat, double kappa, int* lag2, double* lam)
{
    int m = 0;
    for (int c = 0; c < n; ++c) {
        const double* pl = par + 8 * act2[2 * c];
        if (!(pl[7] > 0.0)) continue;
        const double dist = dist_of(pl, s, act2[2 * c + 1]), d = dist * dist;
        double b, db, d2b;
        orc_barrier(d, dHat, &b, &db, &d2b);
        double l = db;
        l *= -kappa * 2.0 * std::sqrt(d);
        lag2[2 * m] = act2[2 * c];
        lag2[2 * m + 1] = act2[2 * c + 1];
        lam[m] = l;
        ++m;
    }
    return m;
}

/* HalfSpace::computeFrictionEnergy (:272-299), summed plane by plane as Optimizer.cpp:3355-3365 adds them */
void orc_hs_friction_energy(const orc_surf* s, const double* Vt, const double* par, const int* lag2, const double* lam, int n, double eps2, double* E)
{
    const double eps = std::sqrt(eps2);
    double total = 0.0, Ef = 0.0;
    for (int c = 0; c < n; ++c) {
        if (c > 0 && lag2[2 * c] != lag2[2 * c - 2]) { total += Ef * 1.0; Ef = 0.0; }
        const double* pl = par + 8 * lag2[2 * c];
        const int v = lag2[2 * c + 1];
        double x[3], xt[3];
        pos(s, s->V, v, x);
        pos(s, Vt, v, xt);
        const Slip u = slip_of(pl, x, xt);
        if (u.mag2 > eps2) Ef += pl[7] * lam[c] * (std::sqrt(u.mag2) - eps * 0.5);
        else Ef += pl[7] * lam[c] * u.mag2 / eps * 0.5;
    }
    *E = total + Ef * 1.0;
}

/* HalfSpace::augmentFrictionGradient (:300-326) */
void orc_hs_friction_gradient(const orc_surf* s, const double* Vt, const double* par, const int* lag2, const double* lam, int n, double eps2, double* g)
{
    const double eps = std::sqrt(eps2);
    for (int c = 0; c < n; ++c) {
        const double* pl = par + 8 * lag2[2 * c];
        const int v = lag2[2 * c + 1];
        double x[3], xt[3];
        pos(s, s->V, v, x);
        pos(s, Vt, v, xt);
        const Slip u = slip_of(pl, x, xt);
        const double f = (u.mag2 > eps2) ? 1.0 * pl[7] * lam[c] / std::sqrt(u.mag2) : 1.0 * pl[7] * lam[c] / eps;
        for (int r = 0; r < 3; ++r) g[3 * v + r] += f * u.u[r];
    }
}

/* one entry's friction block (:339-362), row-major; project = 0 skips the makePD of the sliding branch (finite-difference tests).
 * x, xt: the vertex now and at the start of the step */
void orc_hs_friction_block(const double* pl, const double* x, const double* xt, double lam, double eps2, int project, double* H9)
{
    const double eps = std::sqrt(eps2);
    const double m = 1.0 * pl[7] * lam;
    const Slip u = slip_of(pl, x, xt);
    if (u.mag2 > eps2) {
        const double mag = std::sqrt(u.mag2);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) H9[3 * i + j] = (u.u[i] * (-m / u.mag2 / mag)) * u.u[j] + ((i == j ? 1.0 : 0.0) - pl[i] * pl[j]) * (m / mag);
        if (project) orc_makePD(3, H9);
    }
    else {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) H9[3 * i + j] = ((i == j ? 1.0 : 0.0) - pl[i] * pl[j]) * (m / eps);
    }
}

/* HalfSpace::augmentFrictionHessian (:327-380) */
void orc_hs_friction_hessian_csr(const orc_surf* s, const double* Vt, const double* par, const int* lag2, const double* lam, int n, double eps2, int projectDBC,
    const int* ia, const int* ja, int base, double* a)
{
    for (int c = 0; c < n; ++c) {
        const double* pl = par + 8 * lag2[2 * c];
        const int v = lag2[2 * c + 1];
        if (proj(s, v, projectDBC)) continue;
        double x[3], xt[3], H[9];
        pos(s, s->V, v, x);
        pos(s, Vt, v, xt);
        orc_hs_friction_block(pl, x, xt, lam[c], eps2, 1, H);
        add_block(ia, ja, base, v, H, a);
    }
}

} // extern "C"

extern "C" {

/* The plane parts of a line-search trial's energy (Optimizer::computeEnergyVal, Optimizer.cpp:3252-3377) around the other terms:
 *   E = ((E_el_in) + (E_b + kappa sum_planes b(d))) + E_plane_f + E_f
 * where E_el_in = E_el + E_in, E_b = the self-contact barrier energy and E_f = the self friction, as the caller computed them: both barrier parts
 * are one kappa * bVals.sum() (:3352), the planes' friction (fricDHat > 0 and a lagged plane set, :3355-3365) comes before self friction.
 * act2 / n: the plane set the trial holds; with_friction = 0 leaves the planes' friction out.  Returns 1 where the reference would exit (d <= 0). */
int orc_hs_trial_energy(const orc_surf* s, const double* Vt, const double* par, const int* act2, int n, double dHat, double kappa, int with_friction,
    const int* lag2, const double* lam, int nlag, double eps2, double E_el_in, double E_b, double E_f, double* E)
{
    double Ehb = 0.0, Ehf = 0.0;
    const int bad = orc_hs_energy(s, par, act2, n, dHat, kappa, &Ehb);
    if (with_friction) orc_hs_friction_energy(s, Vt, par, lag2, lam, nlag, eps2, &Ehf);
    double e = E_el_in;
    e += E_b + Ehb;
    if (with_friction) e += Ehf;
    e += E_f;
    *E = e;
    return bad;
}

} // extern "C"
