/*
 * elastic.cpp -- CPU ORACLE (test infrastructure only; see oracle.h header).
 * Restates the per-tet elastic path of ipc-sim/IPC:
 *   src/Utils/SVD/ImplicitQRSVD.h, src/Utils/AutoFlipSVD.hpp,
 *   src/Energy/Energy.cpp, src/Energy/Physics_Elasticity/{NeoHookean,FixedCoRot}Energy.cpp,
 *   src/Utils/IglUtils.{hpp,cpp} (makePD, makePD2d, dF_div_dx_mult, cofactor, addBlockToMatrix),
 *   src/Utils/get_feasible_steps.cpp, src/LinSysSolver/LinSysSolver.hpp (CSR sink).
 */
#include "oracle.h"
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstring>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

inline double& at(double* M, int i, int j) { return M[3 * i + j]; }
inline double at(const double* M, int i, int j) { return M[3 * i + j]; }

/* ---- Givens rotation, ImplicitQRSVD.h:101-240 ------------------------------ */
struct Givens {
    int i, k;
    double c, s;
    Givens(int i_, int k_) : i(i_), k(k_), c(1.0), s(0.0) {}
    /* (c -s; s c)(a;b) = (*;0)   ImplicitQRSVD.h:137-150 ; rsqrt = 1/sqrt  Tools.h:143-147 */
    void compute(double a, double b)
    {
        double d = a * a + b * b;
        c = 1.0;
        s = 0.0;
        if (d != 0.0) {
            double t = 1.0 / std::sqrt(d);
            c = a * t;
            s = -b * t;
        }
    }
    /* (c -s; s c)(a;b) = (0;*)   ImplicitQRSVD.h:157-170 */
    void computeUnconventional(double a, double b)
    {
        double d = a * a + b * b;
        c = 0.0;
        s = 1.0;
        if (d != 0.0) {
            double t = 1.0 / std::sqrt(d);
            s = a * t;
            c = b * t;
        }
    }
    void rowRotation(double* A) const /* :193-201 */
    {
        for (int j = 0; j < 3; ++j) {
            double t1 = at(A, i, j), t2 = at(A, k, j);
            at(A, i, j) = c * t1 - s * t2;
            at(A, k, j) = s * t1 + c * t2;
        }
    }
    void columnRotation(double* A) const /* :211-219 */
    {
        for (int j = 0; j < 3; ++j) {
            double t1 = at(A, j, i), t2 = at(A, j, k);
            at(A, j, i) = c * t1 - s * t2;
            at(A, j, k) = s * t1 + c * t2;
        }
    }
    void mulAssign(const Givens& A) /* :224-230 */
    {
        double nc = c * A.c - s * A.s;
        double ns = s * A.c + c * A.s;
        c = nc;
        s = ns;
    }
};

/* ImplicitQRSVD.h:252-301 */
void zeroChase(double* H, double* U, double* V)
{
    Givens r1(0, 1);
    r1.compute(at(H, 0, 0), at(H, 1, 0));
    Givens r2(1, 2);
    if (at(H, 1, 0) != 0.0)
        r2.compute(at(H, 0, 0) * at(H, 0, 1) + at(H, 1, 0) * at(H, 1, 1),
            at(H, 0, 0) * at(H, 0, 2) + at(H, 1, 0) * at(H, 1, 2));
    else
        r2.compute(at(H, 0, 1), at(H, 0, 2));
    r1.rowRotation(H);
    r2.columnRotation(H);
    r2.columnRotation(V);
    Givens r3(1, 2);
    r3.compute(at(H, 1, 1), at(H, 2, 1));
    r3.rowRotation(H);
    r1.columnRotation(U);
    r3.columnRotation(U);
}

/* ImplicitQRSVD.h:314-328 */
void makeUpperBidiag(double* H, double* U, double* V)
{
    for (int q = 0; q < 9; ++q) U[q] = V[q] = (q % 4 == 0) ? 1.0 : 0.0;
    Givens r(1, 2);
    r.compute(at(H, 1, 0), at(H, 2, 0));
    r.rowRotation(H);
    r.columnRotation(U);
    zeroChase(H, U, V);
}

/* 2x2 polar (ImplicitQRSVD.h:398-418) + 2x2 SVD (:454-518). A row-major 2x2. */
void svd2x2(const double A[4], Givens& U, double sigma[2], Givens& V)
{
    double x0 = A[0] + A[3], x1 = A[2] - A[1];
    double den = std::sqrt(x0 * x0 + x1 * x1);
    U.c = 1.0;
    U.s = 0.0;
    if (den != 0.0) {
        U.c = x0 / den;
        U.s = -x1 / den;
    }
    /* S = R.rowRotation(A) with rowi=0,rowk=1 */
    double S[4];
    for (int j = 0; j < 2; ++j) {
        double t1 = A[j], t2 = A[2 + j];
        S[j] = U.c * t1 - U.s * t2;
        S[2 + j] = U.s * t1 + U.c * t2;
    }
    double cosine, sine;
    double x = S[0], y = S[1], z = S[3];
    if (y == 0.0) {
        cosine = 1.0;
        sine = 0.0;
        sigma[0] = x;
        sigma[1] = z;
    }
    else {
        double tau = 0.5 * (x - z);
        double w = std::sqrt(tau * tau + y * y);
        double t;
        if (tau > 0.0)
            t = y / (tau + w);
        else
            t = y / (tau - w);
        cosine = 1.0 / std::sqrt(t * t + 1.0);
        sine = -t * cosine;
        double c2 = cosine * cosine;
        double csy = 2.0 * cosine * sine * y;
        double s2 = sine * sine;
        sigma[0] = c2 * x - csy + s2 * z;
        sigma[1] = s2 * x + csy + c2 * z;
    }
    if (sigma[0] < sigma[1]) {
        std::swap(sigma[0], sigma[1]);
        V.c = -sine;
        V.s = cosine;
    }
    else {
        V.c = cosine;
        V.s = sine;
    }
    U.mulAssign(V);
}

/* ImplicitQRSVD.h:552-565 */
double wilkinsonShift(double a1, double b1, double a2)
{
    double d = 0.5 * (a1 - a2);
    double bs = b1 * b1;
    return a2 - std::copysign(bs / (std::fabs(d) + std::sqrt(d * d + bs)), d);
}

/* ImplicitQRSVD.h:570-585 */
void process(int t, double* B, double* U, double* sigma, double* V)
{
    int other = (t == 1) ? 0 : 2;
    Givens u(0, 1), v(0, 1);
    sigma[other] = at(B, other, other);
    double blk[4] = { at(B, t, t), at(B, t, t + 1), at(B, t + 1, t), at(B, t + 1, t + 1) };
    svd2x2(blk, u, sigma + t, v);
    u.i += t; u.k += t; v.i += t; v.k += t;
    u.columnRotation(U);
    v.columnRotation(V);
}

void flipSign(int i, double* U, double* sigma) /* :590-594 */
{
    sigma[i] = -sigma[i];
    for (int r = 0; r < 3; ++r) at(U, r, i) = -at(U, r, i);
}
void swapCol(double* M, int a, int b)
{
    for (int r = 0; r < 3; ++r) std::swap(at(M, r, a), at(M, r, b));
}
void negCol(double* M, int a)
{
    for (int r = 0; r < 3; ++r) at(M, r, a) = -at(M, r, a);
}

/* both sorts return 1 when they reorder (the swapping branch), 0 on the early return */
int sort0(double* U, double* sigma, double* V) /* :599-636 */
{
    if (std::fabs(sigma[1]) >= std::fabs(sigma[2])) {
        if (sigma[1] < 0) {
            flipSign(1, U, sigma);
            flipSign(2, U, sigma);
        }
        return 0;
    }
    if (sigma[2] < 0) {
        flipSign(1, U, sigma);
        flipSign(2, U, sigma);
    }
    std::swap(sigma[1], sigma[2]);
    swapCol(U, 1, 2);
    swapCol(V, 1, 2);
    if (sigma[1] > sigma[0]) {
        std::swap(sigma[0], sigma[1]);
        swapCol(U, 0, 1);
        swapCol(V, 0, 1);
    }
    else {
        negCol(U, 2);
        negCol(V, 2);
    }
    return 1;
}
int sort1(double* U, double* sigma, double* V) /* :641-678 */
{
    if (std::fabs(sigma[0]) >= sigma[1]) {
        if (sigma[0] < 0) {
            flipSign(0, U, sigma);
            flipSign(2, U, sigma);
        }
        return 0;
    }
    std::swap(sigma[0], sigma[1]);
    swapCol(U, 0, 1);
    swapCol(V, 0, 1);
    if (std::fabs(sigma[1]) < std::fabs(sigma[2])) {
        std::swap(sigma[1], sigma[2]);
        swapCol(U, 1, 2);
        swapCol(V, 1, 2);
    }
    else {
        negCol(U, 1);
        negCol(V, 1);
    }
    if (sigma[1] < 0) {
        flipSign(1, U, sigma);
        flipSign(2, U, sigma);
    }
    return 1;
}

/* ImplicitQRSVD.h:687-850; br (optional): exit, sort, reordered -- see orc_svd3_branch */
int svd3(const double A[9], double U[9], double sigma[3], double V[9], int* br = nullptr)
{
    int ex = -1, so = -1, re = -1; /* stay -1 only for a non-finite F */
    double B[9];
    std::memcpy(B, A, sizeof(B));
    makeUpperBidiag(B, U, V);
    int count = 0;
    double tol = 1024.0 * 2.220446049250313e-16;
    Givens r(0, 1);
    double alpha_1 = at(B, 0, 0), beta_1 = at(B, 0, 1), alpha_2 = at(B, 1, 1), alpha_3 = at(B, 2, 2), beta_2 = at(B, 1, 2);
    double gamma_1 = alpha_1 * beta_1, gamma_2 = alpha_2 * beta_2;
    tol *= std::max(0.5 * std::sqrt(alpha_1 * alpha_1 + alpha_2 * alpha_2 + alpha_3 * alpha_3 + beta_1 * beta_1 + beta_2 * beta_2), 1.0);
    while (std::fabs(beta_2) > tol && std::fabs(beta_1) > tol && std::fabs(alpha_1) > tol && std::fabs(alpha_2) > tol && std::fabs(alpha_3) > tol) {
        double mu = wilkinsonShift(alpha_2 * alpha_2 + beta_1 * beta_1, gamma_2, alpha_3 * alpha_3 + beta_2 * beta_2);
        r.compute(alpha_1 * alpha_1 - mu, gamma_1);
        r.columnRotation(B);
        r.columnRotation(V);
        zeroChase(B, U, V);
        alpha_1 = at(B, 0, 0); beta_1 = at(B, 0, 1); alpha_2 = at(B, 1, 1); alpha_3 = at(B, 2, 2); beta_2 = at(B, 1, 2);
        gamma_1 = alpha_1 * beta_1;
        gamma_2 = alpha_2 * beta_2;
        ++count;
    }
    if (std::fabs(beta_2) <= tol) {
        process(0, B, U, sigma, V);
        ex = 0, so = 0, re = sort0(U, sigma, V);
    }
    else if (std::fabs(beta_1) <= tol) {
        process(1, B, U, sigma, V);
        ex = 1, so = 1, re = sort1(U, sigma, V);
    }
    else if (std::fabs(alpha_2) <= tol) {
        Givens r1(1, 2);
        r1.computeUnconventional(at(B, 1, 2), at(B, 2, 2));
        r1.rowRotation(B);
        r1.columnRotation(U);
        process(0, B, U, sigma, V);
        ex = 2, so = 0, re = sort0(U, sigma, V);
    }
    else if (std::fabs(alpha_3) <= tol) {
        Givens r1(1, 2);
        r1.compute(at(B, 1, 1), at(B, 1, 2));
        r1.columnRotation(B);
        r1.columnRotation(V);
        Givens r2(0, 2);
        r2.compute(at(B, 0, 0), at(B, 0, 2));
        r2.columnRotation(B);
        r2.columnRotation(V);
        process(0, B, U, sigma, V);
        ex = 3, so = 0, re = sort0(U, sigma, V);
    }
    else if (std::fabs(alpha_1) <= tol) {
        Givens r1(0, 1);
        r1.computeUnconventional(at(B, 0, 1), at(B, 1, 1));
        r1.rowRotation(B);
        r1.columnRotation(U);
        Givens r2(0, 2);
        r2.computeUnconventional(at(B, 0, 2), at(B, 2, 2));
        r2.rowRotation(B);
        r2.columnRotation(U);
        process(1, B, U, sigma, V);
        ex = 4, so = 1, re = sort1(U, sigma, V);
    }
    if (br) br[0] = ex, br[1] = so, br[2] = re;
    return count;
}

/* ---- symmetric eigen-solver (stands in for Eigen::SelfAdjointEigenSolver, IglUtils.hpp:122):
 * cyclic Jacobi; eigenvalues ascending. ------------------------------------------------ */
void jacobi_eig(int n, const double* Min, double* evals, double* evecs /* columns = vectors, row-major n x n */)
{
    std::vector<double> A(Min, Min + n * n);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) evecs[i * n + j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 100; ++sweep) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < n; ++i) {
            diag += A[i * n + i] * A[i * n + i];
            for (int j = i + 1; j < n; ++j) off += A[i * n + j] * A[i * n + j];
        }
        if (off <= 1e-300 || off <= 1e-28 * diag) break; /* rounding floor of the off-diagonal mass is ~1e-30*diag */
        for (int p = 0; p < n; ++p)
            for (int q = p + 1; q < n; ++q) {
                double apq = A[p * n + q];
                if (apq == 0.0) continue;
                double app = A[p * n + p], aqq = A[q * n + q];
                double theta = (aqq - app) / (2.0 * apq);
                double t = ((theta >= 0) ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < n; ++k) {
                    double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; ++k) {
                    double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; ++k) {
                    double vkp = evecs[k * n + p], vkq = evecs[k * n + q];
                    evecs[k * n + p] = c * vkp - s * vkq;
                    evecs[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    std::vector<int> idx(n);
    for (int i = 0; i < n; ++i) idx[i] = i;
    std::sort(idx.begin(), idx.end(), [&](int a, int b) { return A[a * n + a] < A[b * n + b]; });
    std::vector<double> tmp(evecs, evecs + n * n);
    for (int c = 0; c < n; ++c) {
        evals[c] = A[idx[c] * n + idx[c]];
        for (int r = 0; r < n; ++r) evecs[r * n + c] = tmp[r * n + idx[c]];
    }
}

/* IglUtils.hpp:436-464 (3D branch) */
void cofactor3(const double* F, double* A)
{
    at(A, 0, 0) = at(F, 1, 1) * at(F, 2, 2) - at(F, 1, 2) * at(F, 2, 1);
    at(A, 0, 1) = at(F, 1, 2) * at(F, 2, 0) - at(F, 1, 0) * at(F, 2, 2);
    at(A, 0, 2) = at(F, 1, 0) * at(F, 2, 1) - at(F, 1, 1) * at(F, 2, 0);
    at(A, 1, 0) = at(F, 0, 2) * at(F, 2, 1) - at(F, 0, 1) * at(F, 2, 2);
    at(A, 1, 1) = at(F, 0, 0) * at(F, 2, 2) - at(F, 0, 2) * at(F, 2, 0);
    at(A, 1, 2) = at(F, 0, 1) * at(F, 2, 0) - at(F, 0, 0) * at(F, 2, 1);
    at(A, 2, 0) = at(F, 0, 1) * at(F, 1, 2) - at(F, 0, 2) * at(F, 1, 1);
    at(A, 2, 1) = at(F, 0, 2) * at(F, 1, 0) - at(F, 0, 0) * at(F, 1, 2);
    at(A, 2, 2) = at(F, 0, 0) * at(F, 1, 1) - at(F, 0, 1) * at(F, 1, 0);
}

/* gather tet t: x[4][3], A row-major from ref layout */
inline void tet_load(const orc_mesh* m, int t, int vi[4], double x[4][3], double A[9])
{
    for (int k = 0; k < 4; ++k) {
        vi[k] = m->T[(size_t)k * m->nT + t];
        for (int c = 0; c < 3; ++c) x[k][c] = m->V[(size_t)c * m->nV + vi[k]];
    }
    const double* a = m->Ainv + (size_t)9 * t;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) at(A, i, j) = a[i + 3 * j];
}

/* Energy.cpp:209-215: F = [x1-x0 | x2-x0 | x3-x0] * A */
inline void deformation_gradient(const double x[4][3], const double* A, double* F)
{
    double Xt[9];
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) at(Xt, r, c) = x[c + 1][r] - x[0][r];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += at(Xt, i, k) * at(A, k, j);
            at(F, i, j) = s;
        }
}

/* IglUtils.cpp:656-667 : 12-vector from 3x3 P and A */
inline void dFdx_mult_vec(const double* P, const double* A, double* g)
{
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) {
            double s = 0.0;
            for (int j = 0; j < 3; ++j) s += at(A, i, j) * at(P, k, j);
            g[3 + 3 * i + k] = s;
        }
    for (int k = 0; k < 3; ++k) g[k] = -g[3 + k] - g[6 + k] - g[9 + k];
}

/* IglUtils.hpp:417-430 : right is 9 x ncol (row-major, leading dim ld), result 12 x ncol */
inline void dFdx_mult_mat(const double* right, int ncol, const double* A, double* result)
{
    for (int col = 0; col < ncol; ++col) {
        for (int i = 0; i < 3; ++i)
            for (int k = 0; k < 3; ++k) {
                double s = 0.0;
                for (int j = 0; j < 3; ++j) s += at(A, i, j) * right[(3 * k + j) * ncol + col];
                result[(3 + 3 * i + k) * ncol + col] = s;
            }
        for (int k = 0; k < 3; ++k)
            result[k * ncol + col] = -result[(3 + k) * ncol + col] - result[(6 + k) * ncol + col] - result[(9 + k) * ncol + col];
    }
}

inline bool is_project_dbc(const orc_mesh* m, int v, int projectDBC) /* Mesh.hpp:135-144 */
{
    if (!m->dbc) return false;
    return m->dbc[v] == 1 || (m->dbc[v] == 2 && projectDBC);
}

void tet_hessian(const orc_mesh* m, int t, double coef, int projectSPD, double* H /*144*/)
{
    int vi[4];
    double x[4][3], A[9], F[9], U[9], S[3], V[9];
    tet_load(m, t, vi, x, A);
    deformation_gradient(x, A, F);
    svd3(F, U, S, V);
    double w = coef * m->vol[t];
    double dPdF[81];
    orc_dPdF(m->energy_type, U, S, V, m->mu[t], m->lam[t], w, projectSPD, dPdF);
    /* Energy.cpp:398-400: two chain-rule passes */
    double dPdFt[81];
    for (int i = 0; i < 9; ++i)
        for (int j = 0; j < 9; ++j) dPdFt[i * 9 + j] = dPdF[j * 9 + i];
    double wdPdx[12 * 9];
    dFdx_mult_mat(dPdFt, 9, A, wdPdx);
    double wdPdxT[9 * 12];
    for (int i = 0; i < 12; ++i)
        for (int j = 0; j < 9; ++j) wdPdxT[j * 12 + i] = wdPdx[i * 9 + j];
    dFdx_mult_mat(wdPdxT, 12, A, H);
}

struct CsrSink {
    const int* ia;
    const int* ja;
    int base;
    double* a;
    int find(int r, int c) const
    {
        int lo = ia[r] - base, hi = ia[r + 1] - base;
        const int* p = std::lower_bound(ja + lo, ja + hi, c + base);
        if (p == ja + hi || *p != c + base) return -1;
        return (int)(p - ja);
    }
    void add(int r, int c, double v) const /* LinSysSolver.hpp:402-410 */
    {
        if (r <= c) {
            int k = find(r, c);
            if (k >= 0) a[k] += v;
        }
    }
    void set(int r, int c, double v) const /* :331-339 */
    {
        if (r <= c) {
            int k = find(r, c);
            if (k >= 0) a[k] = v;
        }
    }
};

} // namespace

extern "C" {

int orc_svd3(const double F[9], double U[9], double S[3], double V[9]) { return svd3(F, U, S, V); }

int orc_svd3_branch(const double F[9], int* exit_id, int* sort_id, int* reordered)
{
    double U[9], S[3], V[9];
    int br[3];
    int n = svd3(F, U, S, V, br);
    *exit_id = br[0];
    *sort_id = br[1];
    *reordered = br[2];
    return n;
}

/* NeoHookeanEnergy.cpp:55-69 ; FixedCoRotEnergy.cpp:62-70 */
void orc_psi(int et, const double S[3], double mu, double lam, double* E)
{
    if (et == 0) {
        if (mu == 0.0 && lam == 0.0) { *E = 0.0; return; }
        double s2 = S[0] * S[0] + S[1] * S[1] + S[2] * S[2];
        double J = S[0] * S[1] * S[2];
        double lJ = std::log(J);
        *E = mu / 2.0 * (s2 - 3) - (mu - lam / 2.0 * lJ) * lJ;
    }
    else {
        double a = S[0] - 1.0, b = S[1] - 1.0, c = S[2] - 1.0;
        double Jm1 = S[0] * S[1] * S[2] - 1.0;
        *E = mu * (a * a + b * b + c * c) + lam / 2.0 * Jm1 * Jm1;
    }
}
/* NeoHookeanEnergy.cpp:71-90 ; FixedCoRotEnergy.cpp:72-94 */
void orc_dpsi(int et, const double S[3], double mu, double lam, double dE[3])
{
    if (et == 0) {
        if (mu == 0.0 && lam == 0.0) { dE[0] = dE[1] = dE[2] = 0.0; return; }
        double lJ = std::log(S[0] * S[1] * S[2]);
        for (int i = 0; i < 3; ++i) {
            double inv = 1.0 / S[i];
            dE[i] = mu * (S[i] - inv) + lam * inv * lJ;
        }
    }
    else {
        double k = lam * (S[0] * S[1] * S[2] - 1.0);
        double n0 = S[1] * S[2], n1 = S[2] * S[0], n2 = S[0] * S[1];
        double m2 = mu * 2;
        dE[0] = m2 * (S[0] - 1.0) + n0 * k;
        dE[1] = m2 * (S[1] - 1.0) + n1 * k;
        dE[2] = m2 * (S[2] - 1.0) + n2 * k;
    }
}
/* NeoHookeanEnergy.cpp:92-114 ; FixedCoRotEnergy.cpp:96-127 */
void orc_d2psi(int et, const double S[3], double mu, double lam, double H[9])
{
    if (et == 0) {
        if (mu == 0.0 && lam == 0.0) { for (int q = 0; q < 9; ++q) H[q] = 0.0; return; }
        double lJ = std::log(S[0] * S[1] * S[2]);
        for (int i = 0; i < 3; ++i) {
            double inv2 = 1.0 / S[i] / S[i];
            at(H, i, i) = mu * (1.0 + inv2) - lam * inv2 * (lJ - 1.0);
        }
        at(H, 0, 1) = at(H, 1, 0) = lam / S[0] / S[1];
        at(H, 1, 2) = at(H, 2, 1) = lam / S[1] / S[2];
        at(H, 2, 0) = at(H, 0, 2) = lam / S[2] / S[0];
    }
    else {
        double J = S[0] * S[1] * S[2];
        double n[3] = { S[1] * S[2], S[2] * S[0], S[0] * S[1] };
        double m2 = mu * 2;
        for (int i = 0; i < 3; ++i) at(H, i, i) = m2 + lam * n[i] * n[i];
        at(H, 0, 1) = at(H, 1, 0) = lam * (S[2] * (J - 1.0) + n[0] * n[1]);
        at(H, 0, 2) = at(H, 2, 0) = lam * (S[1] * (J - 1.0) + n[0] * n[2]);
        at(H, 2, 1) = at(H, 1, 2) = lam * (S[0] * (J - 1.0) + n[2] * n[1]);
    }
}
/* NeoHookeanEnergy.cpp:116-136 ; FixedCoRotEnergy.cpp:129-143 */
void orc_bleft(int et, const double S[3], double mu, double lam, double BL[3])
{
    double J = S[0] * S[1] * S[2];
    if (et == 0) {
        if (mu == 0.0 && lam == 0.0) { BL[0] = BL[1] = BL[2] = 0.0; return; }
        double middle = mu - lam * std::log(J);
        BL[0] = (mu + middle / S[0] / S[1]) / 2.0;
        BL[1] = (mu + middle / S[1] / S[2]) / 2.0;
        BL[2] = (mu + middle / S[2] / S[0]) / 2.0;
    }
    else {
        double hl = lam / 2.0;
        BL[0] = mu - hl * S[2] * (J - 1);
        BL[1] = mu - hl * S[0] * (J - 1);
        BL[2] = mu - hl * S[1] * (J - 1);
    }
}
/* NeoHookeanEnergy.cpp:138-153 ; FixedCoRotEnergy.cpp:145-153 */
void orc_pk1(int et, const double F[9], const double U[9], const double S[3], const double V[9], double mu, double lam, double P[9])
{
    double J = S[0] * S[1] * S[2];
    double C[9];
    cofactor3(F, C);
    if (et == 0) {
        if (mu == 0.0 && lam == 0.0) { for (int q = 0; q < 9; ++q) P[q] = 0.0; return; }
        double lJ = std::log(J);
        for (int q = 0; q < 9; ++q) {
            double FinvT = C[q] / J;
            P[q] = mu * (F[q] - FinvT) + lam * lJ * FinvT;
        }
    }
    else {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double R = 0.0;
                for (int k = 0; k < 3; ++k) R += at(U, i, k) * at(V, j, k);
                at(P, i, j) = mu * 2 * (at(F, i, j) - R) + lam * (J - 1) * at(C, i, j);
            }
    }
}

/* IglUtils.hpp:119-137 */
void orc_makePD(int n, double* M)
{
    std::vector<double> ev(n), evec((size_t)n * n);
    jacobi_eig(n, M, ev.data(), evec.data());
    if (ev[0] >= 0.0) return;
    for (int i = 0; i < n; ++i) {
        if (ev[i] < 0.0) ev[i] = 0.0;
        else break;
    }
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) {
            double s = 0.0;
            for (int k = 0; k < n; ++k) s += evec[i * n + k] * ev[k] * evec[j * n + k];
            M[i * n + j] = s;
        }
}
/* IglUtils.hpp:138-177 */
void orc_makePD2d(double M[4])
{
    const double a = M[0];
    const double b = (M[1] + M[2]) / 2.0;
    const double d = M[3];
    double b2 = b * b;
    const double D = a * d - b2;
    const double T_div_2 = (a + d) / 2.0;
    const double sqrtTT4D = std::sqrt(T_div_2 * T_div_2 - D);
    const double L2 = T_div_2 - sqrtTT4D;
    if (L2 < 0.0) {
        const double L1 = T_div_2 + sqrtTT4D;
        if (L1 <= 0.0) {
            M[0] = M[1] = M[2] = M[3] = 0.0;
        }
        else if (b2 == 0.0) {
            M[0] = L1; M[1] = M[2] = M[3] = 0.0;
        }
        else {
            const double L1md = L1 - d;
            const double r = L1md / L1;
            M[0] = r * L1md;
            M[1] = M[2] = b * r;
            M[3] = b2 / L1;
        }
    }
}

/* Energy.cpp:448-562 */
void orc_dPdF(int et, const double U[9], const double S[3], const double V[9], double mu, double lam, double w, int projectSPD, double dPdF[81])
{
    double dE[3], A[9], BL[3];
    orc_dpsi(et, S, mu, lam, dE);
    orc_d2psi(et, S, mu, lam, A);
    if (projectSPD) orc_makePD(3, A);
    orc_bleft(et, S, mu, lam, BL);
    double B[3][4];
    for (int c = 0; c < 3; ++c) {
        int cp = (c + 1) % 3;
        double right = dE[c] + dE[cp];
        double sum = S[c] + S[cp];
        const double eps = 1.0e-6;
        if (sum < eps) right /= 2.0 * eps;
        else right /= 2.0 * sum;
        double left = BL[c];
        B[c][0] = B[c][3] = left + right;
        B[c][1] = B[c][2] = left - right;
        if (projectSPD) orc_makePD2d(B[c]);
    }
    double M[81];
    for (int q = 0; q < 81; ++q) M[q] = 0.0;
#define MM(i, j) M[(i) * 9 + (j)]
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) MM(4 * i, 4 * j) = w * at(A, i, j);
    MM(1, 1) = w * B[0][0]; MM(1, 3) = w * B[0][1]; MM(3, 1) = w * B[0][2]; MM(3, 3) = w * B[0][3];
    MM(5, 5) = w * B[1][0]; MM(5, 7) = w * B[1][1]; MM(7, 5) = w * B[1][2]; MM(7, 7) = w * B[1][3];
    MM(2, 2) = w * B[2][3]; MM(2, 6) = w * B[2][2]; MM(6, 2) = w * B[2][1]; MM(6, 6) = w * B[2][0];
    /* non-zeros of M in the reference's summation order, Energy.cpp:551 */
    static const int nz[21][2] = { { 0, 0 }, { 0, 4 }, { 0, 8 }, { 4, 0 }, { 4, 4 }, { 4, 8 }, { 8, 0 }, { 8, 4 }, { 8, 8 },
        { 1, 1 }, { 1, 3 }, { 3, 1 }, { 3, 3 }, { 5, 5 }, { 5, 7 }, { 7, 5 }, { 7, 7 }, { 2, 2 }, { 2, 6 }, { 6, 2 }, { 6, 6 } };
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            int ij = 3 * i + j;
            for (int r = 0; r < 3; ++r)
                for (int s = 0; s < 3; ++s) {
                    int rs = 3 * r + s;
                    if (ij > rs) continue;
                    double acc = 0.0;
                    for (int q = 0; q < 21; ++q) {
                        int kl = nz[q][0], mn = nz[q][1];
                        int k = kl / 3, l = kl % 3, mm = mn / 3, n = mn % 3;
                        double term = MM(kl, mn) * at(U, i, k) * at(V, j, l) * at(U, r, mm) * at(V, s, n);
                        acc = (q == 0) ? term : acc + term;
                    }
                    dPdF[ij * 9 + rs] = acc;
                    if (ij < rs) dPdF[rs * 9 + ij] = acc;
                }
        }
#undef MM
}

void orc_elastic_energy(const orc_mesh* m, double coef, double* Eper, double* E, int nthreads)
{
    std::vector<double> tmp;
    if (!Eper) {
        tmp.resize(m->nT);
        Eper = tmp.data();
    }
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(static)
    for (int t = 0; t < m->nT; ++t) {
        int vi[4];
        double x[4][3], A[9], F[9], U[9], S[3], V[9];
        tet_load(m, t, vi, x, A);
        deformation_gradient(x, A, F);
        svd3(F, U, S, V);
        double e;
        orc_psi(m->energy_type, S, m->mu[t], m->lam[t], &e);
        Eper[t] = e * m->vol[t];
    }
    double s = 0.0;
    for (int t = 0; t < m->nT; ++t) s += Eper[t]; /* Eigen .sum(): order unspecified; sequential here */
    *E = coef * s;
}

void orc_elastic_gradient(const orc_mesh* m, double coef, int projectDBC, double* g, int nthreads)
{
    std::vector<double> gc((size_t)12 * m->nT);
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(static)
    for (int t = 0; t < m->nT; ++t) {
        int vi[4];
        double x[4][3], A[9], F[9], U[9], S[3], V[9], P[9];
        tet_load(m, t, vi, x, A);
        deformation_gradient(x, A, F);
        svd3(F, U, S, V);
        orc_pk1(m->energy_type, F, U, S, V, m->mu[t], m->lam[t], P);
        double w = coef * m->vol[t];
        for (int q = 0; q < 9; ++q) P[q] *= w;
        dFdx_mult_vec(P, A, &gc[(size_t)12 * t]);
    }
    for (size_t q = 0; q < (size_t)3 * m->nV; ++q) g[q] = 0.0;
    /* vFLoc order = ascending (tet, local) per vertex (Energy.cpp:276-278) == ascending tet sweep */
    for (int t = 0; t < m->nT; ++t)
        for (int k = 0; k < 4; ++k) {
            int v = m->T[(size_t)k * m->nT + t];
            for (int c = 0; c < 3; ++c) g[3 * (size_t)v + c] += gc[(size_t)12 * t + 3 * k + c];
        }
    if (projectDBC && m->dbc) /* Energy.cpp:284-288: all DBCVertexIds (type != NOT_DBC) */
        for (int v = 0; v < m->nV; ++v)
            if (m->dbc[v]) g[3 * (size_t)v] = g[3 * (size_t)v + 1] = g[3 * (size_t)v + 2] = 0.0;
}

void orc_elastic_hessian_blocks(const orc_mesh* m, double coef, int projectSPD, double* H_all, int nthreads)
{
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(static)
    for (int t = 0; t < m->nT; ++t) tet_hessian(m, t, coef, projectSPD, H_all + (size_t)144 * t);
}

void orc_elastic_hessian_csr(const orc_mesh* m, double coef, int projectSPD, int projectDBC,
    const int* ia, const int* ja, int index_base, double* a, int nthreads)
{
    std::vector<double> H((size_t)144 * m->nT);
    orc_elastic_hessian_blocks(m, coef, projectSPD, H.data(), nthreads);
    CsrSink sink{ ia, ja, index_base, a };
    /* Energy.cpp:317-330 + IglUtils.hpp:39-116; per vertex in ascending (tet, local) order == tet sweep per row */
    for (int t = 0; t < m->nT; ++t) {
        int vInd[4];
        for (int k = 0; k < 4; ++k) {
            int v = m->T[(size_t)k * m->nT + t];
            vInd[k] = is_project_dbc(m, v, projectDBC) ? (-v - 1) : v;
        }
        const double* Ht = &H[(size_t)144 * t];
        for (int rk = 0; rk < 4; ++rk) {
            int rowStart = vInd[rk] * 3;
            if (rowStart < 0) {
                rowStart = -rowStart - 3;
                for (int c = 0; c < 3; ++c) sink.set(rowStart + c, rowStart + c, 1.0);
                continue;
            }
            for (int ck = 0; ck < 4; ++ck) {
                if (vInd[ck] < 0) continue;
                int colStart = vInd[ck] * 3;
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) sink.add(rowStart + r, colStart + c, Ht[(3 * rk + r) * 12 + 3 * ck + c]);
            }
        }
    }
}

/* get_feasible_steps.cpp:9-28, :75-108 */
/* br (optional, see orc_cubic_branch): br[0] the exit, br[1] the |C| == 0 fallback, br[2] the mask of Cardano roots that pass the filter,
 * br[3] the root kept (1..3, 0 for none) */
static double quadRoot(double a, double b, double c, double tol, int* br = nullptr)
{
    double t;
    if (std::abs(a) <= tol) {
        t = -c / b;
        if (br) br[0] = 0;
    }
    else {
        double desc = b * b - 4 * a * c;
        if (desc > 0) {
            t = (-b - std::sqrt(desc)) / (2 * a);
            if (br) br[0] = 1;
            if (t < 0) {
                t = (-b + std::sqrt(desc)) / (2 * a);
                if (br) br[0] = 2;
            }
        }
        else {
            t = -1;
            if (br) br[0] = 3;
        }
    }
    return t;
}
static double cubicRoot(double a, double b, double c, double d, double tol, int* br = nullptr)
{
    double t = -1;
    if (br) br[0] = br[1] = br[2] = br[3] = 0;
    if (std::abs(a) <= tol) t = quadRoot(b, c, d, tol, br);
    else {
        typedef std::complex<double> cd;
        cd i(0, 1);
        cd delta0(b * b - 3 * a * c, 0);
        cd delta1(2 * b * b * b - 9 * a * b * c + 27 * a * a * d, 0);
        cd rad = (delta1 + std::sqrt(delta1 * delta1 - 4.0 * delta0 * delta0 * delta0)) / 2.0;
        cd C = std::pow(rad, 1.0 / 3.0);
        if (std::abs(C) == 0.0) {
            rad = (delta1 - std::sqrt(delta1 * delta1 - 4.0 * delta0 * delta0 * delta0)) / 2.0;
            C = std::pow(rad, 1.0 / 3.0);
            if (br) br[1] = 1;
        }
        if (br) br[0] = (std::imag(rad) == 0.0 && std::real(rad) > 0.0) ? 4 : 5; /* libstdc++'s real pow, or the complex log/polar path */
        cd u2 = (-1.0 + std::sqrt(3.0) * i) / 2.0;
        cd u3 = (-1.0 - std::sqrt(3.0) * i) / 2.0;
        cd t1 = (b + C + delta0 / C) / (-3.0 * a);
        cd t2 = (b + u2 * C + delta0 / (u2 * C)) / (-3.0 * a);
        cd t3 = (b + u3 * C + delta0 / (u3 * C)) / (-3.0 * a);
        const bool p1 = (std::abs(std::imag(t1)) < tol) && (std::real(t1) > 0);
        const bool p2 = (std::abs(std::imag(t2)) < tol) && (std::real(t2) > 0);
        const bool p3 = (std::abs(std::imag(t3)) < tol) && (std::real(t3) > 0);
        int k = 0;
        if (p1) t = std::real(t1), k = 1;
        if (p2 && ((std::real(t2) < t) || (t < 0))) t = std::real(t2), k = 2;
        if (p3 && ((std::real(t3) < t) || (t < 0))) t = std::real(t3), k = 3;
        if (br) br[2] = (int)p1 | (int)p2 << 1 | (int)p3 << 2, br[3] = k;
    }
    return t;
}

int orc_cubic_branch(double a, double b, double c, double d, double tol, double* t, int* fallback, int* passed, int* kept)
{
    int br[4];
    *t = cubicRoot(a, b, c, d, tol, br);
    *fallback = br[1];
    *passed = br[2];
    *kept = br[3];
    return br[0];
}
static inline double det3c(const double* a, const double* b, const double* c)
{
    return a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) + a[2] * (b[0] * c[1] - b[1] * c[0]);
}

void orc_inversion_step(const orc_mesh* m, const double* p, double slack, double* per_tet, double* alpha_inout)
{
    /* get_feasible_steps.cpp:110-172: a t^3 + b t^2 + c t + (1-slack) det(e) = 0 with
     * e_i = x_{i+1}-x_0, f_i = p_{i+1}-p_0; a = det(f), d = det(e), b and c the mixed terms
     * (multilinear expansion of det[e1+t f1, e2+t f2, e3+t f3]). */
    double best = 1e300;
    for (int t = 0; t < m->nT; ++t) {
        int vi[4];
        double x[4][3], A[9];
        tet_load(m, t, vi, x, A);
        double e[3][3], f[3][3];
        for (int k = 0; k < 3; ++k)
            for (int c = 0; c < 3; ++c) {
                e[k][c] = x[k + 1][c] - x[0][c];
                f[k][c] = p[3 * (size_t)vi[k + 1] + c] - p[3 * (size_t)vi[0] + c];
            }
        double a = det3c(f[0], f[1], f[2]);
        double b = det3c(e[0], f[1], f[2]) + det3c(f[0], e[1], f[2]) + det3c(f[0], f[1], e[2]);
        double c = det3c(f[0], e[1], e[2]) + det3c(e[0], f[1], e[2]) + det3c(e[0], e[1], f[2]);
        double d = (1.0 - slack) * det3c(e[0], e[1], e[2]);
        double r = cubicRoot(a, b, c, d, 1.0e-6);
        double out = (r >= 0) ? r : 1e20;
        if (per_tet) per_tet[t] = out;
        best = std::min(best, out);
    }
    if (m->nT > 0 && best > 0.0 && best < *alpha_inout) *alpha_inout = best; /* Energy.cpp:576-579 */
}

int orc_csr_pattern(int nV, const int* nbr_ptr, const int* nbr, int base, int* ia, int* ja)
{
    /* LinSysSolver.hpp:46-150: row 3v: [3v,3v+1,3v+2, 3n.. for n>v]; row 3v+1 drops first; row 3v+2 drops two */
    int nnz = 0;
    for (int v = 0; v < nV; ++v) {
        int up = 0;
        for (int q = nbr_ptr[v]; q < nbr_ptr[v + 1]; ++q)
            if (nbr[q] > v) ++up;
        for (int r = 0; r < 3; ++r) {
            if (ia) ia[3 * v + r] = nnz + base;
            if (ja) {
                int k = nnz;
                for (int c = r; c < 3; ++c) ja[k++] = 3 * v + c + base;
                for (int q = nbr_ptr[v]; q < nbr_ptr[v + 1]; ++q)
                    if (nbr[q] > v)
                        for (int c = 0; c < 3; ++c) ja[k++] = 3 * nbr[q] + c + base;
            }
            nnz += (3 - r) + 3 * up;
        }
    }
    if (ia) ia[3 * nV] = nnz + base;
    return nnz;
}

} // extern "C"
