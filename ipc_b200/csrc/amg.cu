// amg.cu -- conjugate gradients on the device-resident matrix, preconditioned by smoothed-aggregation algebraic multigrid: the
// reference's `linearSolver AMGCL` (src/LinSysSolver/AMGCLSolver.cpp:24-44: Chebyshev relaxation of degree 16, at most 6 levels, the
// coarsest level smoothed, W-cycle, every connection strong), rebuilt from the resident matrix at every call as AMGCLSolver::factorize
// rebuilds it at every Newton iteration (:173-191).  One deliberate difference: the reference aggregates x, y and z unknowns separately
// (scalar backend); here vertices are aggregated and every level is a block CSR matrix of 3 x 3 blocks, with the translations of each
// aggregate as the coarse space (DESIGN 3.23).  This file holds the hierarchy and its step of solve.cu's Krylov loop (solver_pcg).
//
// Set-up (eager: it reads sizes back).  Every sum is taken in a fixed order and no floating-point atomic is used, so two calls on one
// state give identical bits.  tests/amg_mirror.py restates every step.
//   1. Level 0: block row i covers the full rows 3i..3i+2 (fia / fja / fpos, LinSysSolver::set_pattern's block layout, checked); a block is
//      kept when one of its 9 entries is nonzero (the device-built pattern stores zero blocks).
//   2. Rows i != j are connected when block (i, j) is kept; a row without a connection (Dirichlet vertex, obstacle tail, a vertex with
//      nothing but mass) is in no aggregate: its row of P is zero.
//   3. Distance-2 maximal independent set, priority (splitmix64(row), row): per round two max-propagations of (state, priority) and one
//      update, until no row is undecided (a counter read back per round).  A root and its neighbours form an aggregate; every other
//      connected row joins the aggregate of its assigned neighbour of largest priority; aggregates are numbered by ascending root (a scan).
//   4. P = (I - omega D^-1 A) P_tent, omega = (4/3) / max_row sum_c |(D^-1 A)_rc|; a row of P is its neighbours' aggregates, walked in
//      ascending column, every block summed over the row's entries in storage order.
//   5. A_{l+1} = R (A_l P), R = P^T by a radix sort of (column, row): one block SpGEMM for both products.  Every output row is the list of
//      (column, entry pair) in enumeration order (the left row's blocks in storage order, each with the right row's blocks in storage
//      order), stably sorted by column (cub segmented sort), then summed run by run in that order.
//   6. D^-1 by a 3 x 3 Cholesky factorisation; a pivot <= 0 raises the word kSolveStart turns into IPCGPU_ERR_SOLVE (identity stored).
//   7. rho of D^-1 A by 100 power steps from splitmix64(i) mapped to [-1, 1) (fixed-order norms); Chebyshev over [2 rho / 120, 2 rho].
//   8. At most 6 levels; the first level with at most 1000 block rows is the last, and so is one whose coarsening keeps more than 4/5 of
//      its rows or makes no aggregate.
// Apply.  One W-cycle: at level l < L-1 a Chebyshev application, the residual, its restriction, two visits of level l+1 (the first from
//      x = 0), the prolongated correction, a Chebyshev application; the last level two Chebyshev applications.  A Chebyshev application is
//      one kernel for r = D^-1 (f - A x), d = r / theta and 15 fused kernels (SpMV, update, next direction; the 15th adds the 16th
//      direction too).  In an iteration the first kernel also finishes the CG update (alpha summed from the SpMV's partials in every CTA);
//      level 0's last kernel leaves the partials of r.z and r.r.  Launches per iteration, with solve.cu's SpMV, roll and direction:
//      67 * 2^(L-1) - 32.
// Rows outside the coarse space (identity rows with a zero right-hand side) stay exactly 0: a polynomial in D^-1 A keeps an uncoupled zero
// entry at zero, and their rows of P are empty.
#include "common.cuh"
#include "abi.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cub/cub.cuh>

namespace ipcgpu {

constexpr int kAmgDegree = 16;
constexpr int kAmgPowerSteps = 100;
constexpr int kAmgCoarseEnough = 1000; // block rows (3,000 unknowns)
constexpr int kAmgCycles = 2;          // W-cycle

DEV unsigned long long splitmix64(unsigned long long z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// ---- set-up ---------------------------------------------------------------------------------------------------------------
// step 1, one thread per block row: ia == NULL counts the kept blocks into cnt, otherwise writes them at ia[i]
__global__ void __launch_bounds__(256) k_amg_level0(int nb, const int* __restrict__ fia, const int* __restrict__ fja, const int* __restrict__ fpos,
    const double* __restrict__ a, const int* __restrict__ ia, int* __restrict__ cnt, int* __restrict__ ja, double* __restrict__ blk, int* __restrict__ flags)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nb) return;
    const int len = fia[3 * i + 1] - fia[3 * i];
    int kept = 0, out = ia ? ia[i] : 0;
    if (len % 3 || fia[3 * i + 2] - fia[3 * i + 1] != len || fia[3 * i + 3] - fia[3 * i + 2] != len) {
        flags[1] = 1;
        if (!ia) cnt[i] = 0;
        return;
    }
    for (int k = 0; k < len / 3; ++k) {
        const int j = fja[fia[3 * i] + 3 * k];
        double v[9];
        bool nz = false;
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int e = fia[3 * i + c] + 3 * k + d;
                if (fja[e] != j + d || j % 3) flags[1] = 1;
                v[3 * c + d] = a[fpos[e]];
                nz |= v[3 * c + d] != 0.0;
            }
        if (!nz) continue;
        if (ia) {
            ja[out + kept] = j / 3;
#pragma unroll
            for (int q = 0; q < 9; ++q) blk[9 * (size_t)(out + kept) + q] = v[q];
        }
        ++kept;
    }
    if (!ia) cnt[i] = kept;
}

// step 6 (and the Gershgorin bound of step 4, the connections of step 2): D_i^-1 by Cholesky (identity and flags[2] on a pivot <= 0 or a
// missing diagonal block), max absolute row sum of D^-1 A into *absrow, state 1 (undecided) for a connected row, 0 otherwise
__global__ void __launch_bounds__(256) k_amg_diag(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk, double* __restrict__ dinv,
    unsigned long long* __restrict__ absrow, unsigned char* __restrict__ state, int* __restrict__ flags)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* D = nullptr;
    bool connected = false;
    for (int e = ia[i]; e < ia[i + 1]; ++e) {
        if (ja[e] == i) D = blk + 9 * (size_t)e;
        else connected = true;
    }
    state[i] = connected ? 1 : 0;
    double m[9] = { 1, 0, 0, 0, 1, 0, 0, 0, 1 };
    bool ok = D != nullptr;
    if (ok) {
        const double p0 = D[0];
        ok = p0 > 0.0;
        if (ok) {
            const double l00 = sqrt(p0), l10 = D[3] / l00, l20 = D[6] / l00;
            const double p1 = D[4] - l10 * l10;
            ok = p1 > 0.0;
            if (ok) {
                const double l11 = sqrt(p1), l21 = (D[7] - l20 * l10) / l11;
                const double p2 = D[8] - l20 * l20 - l21 * l21;
                ok = p2 > 0.0;
                if (ok) {
                    const double l22 = sqrt(p2);
                    // L^-1 (lower), then D^-1 = L^-T L^-1
                    const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
                    const double i10 = -l10 * i00 / l11, i21 = -l21 * i11 / l22, i20 = -(l20 * i00 + l21 * i10) / l22;
                    m[0] = i00 * i00 + i10 * i10 + i20 * i20;
                    m[1] = m[3] = i10 * i11 + i20 * i21;
                    m[2] = m[6] = i20 * i22;
                    m[4] = i11 * i11 + i21 * i21;
                    m[5] = m[7] = i21 * i22;
                    m[8] = i22 * i22;
                }
            }
        }
    }
    if (!ok) {
        flags[2] = 1;
        m[0] = m[4] = m[8] = 1.0;
        m[1] = m[2] = m[3] = m[5] = m[6] = m[7] = 0.0;
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) dinv[9 * (size_t)i + q] = m[q];
    double s[3] = { 0.0, 0.0, 0.0 };
    for (int e = ia[i]; e < ia[i + 1]; ++e) {
        const double* B = blk + 9 * (size_t)e;
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int d = 0; d < 3; ++d) s[c] += fabs(m[3 * c] * B[d] + m[3 * c + 1] * B[3 + d] + m[3 * c + 2] * B[6 + d]);
    }
    const double mx = fmax(fmax(s[0], s[1]), s[2]);
    atomicMax(absrow, dbl_to_ord(isnan(mx) ? __longlong_as_double(0x7ff0000000000000ll) : mx)); // (NaN counts as infinite: a failure)
}

// step 3: does row a hold a larger (state, priority) than row b
DEV bool amg_above(int a, int b, const unsigned char* __restrict__ s)
{
    if (s[a] != s[b]) return s[a] > s[b];
    const unsigned long long ha = splitmix64((unsigned long long)a), hb = splitmix64((unsigned long long)b);
    return ha != hb ? ha > hb : a > b;
}
// out[i] = the row of largest key among src[j] for j in the closed neighbourhood of i (src NULL: j itself)
__global__ void __launch_bounds__(256) k_amg_mis_max(int n, const int* __restrict__ ia, const int* __restrict__ ja, const int* __restrict__ src,
    const unsigned char* __restrict__ state, int* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int best = src ? src[i] : i;
    for (int e = ia[i]; e < ia[i + 1]; ++e) {
        const int c = src ? src[ja[e]] : ja[e];
        if (amg_above(c, best, state)) best = c;
    }
    out[i] = best;
}
// an undecided row that is the largest of its distance-2 neighbourhood becomes a root (2); one whose largest is a root is out (0)
__global__ void __launch_bounds__(256) k_amg_mis_update(int n, const int* __restrict__ m2, const unsigned char* __restrict__ in, unsigned char* __restrict__ out,
    int* __restrict__ undecided)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned char s = in[i];
    if (s == 1) {
        const int w = m2[i];
        s = w == i ? 2 : in[w] == 2 ? 0 : 1;
        if (s == 1) atomicAdd(undecided, 1);
    }
    out[i] = s;
}
__global__ void __launch_bounds__(256) k_amg_roots(int n, const unsigned char* __restrict__ state, int* __restrict__ flag)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = state[i] == 2;
}
// a root: its aggregate; a neighbour of a root: that root's (unique: roots are at least 3 apart); otherwise -1
__global__ void __launch_bounds__(256) k_amg_assign1(int n, const int* __restrict__ ia, const int* __restrict__ ja, const unsigned char* __restrict__ state,
    const int* __restrict__ id, int* __restrict__ agg1)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int a = -1;
    if (state[i] == 2) a = id[i];
    else
        for (int e = ia[i]; e < ia[i + 1]; ++e)
            if (state[ja[e]] == 2) {
                a = id[ja[e]];
                break;
            }
    agg1[i] = a;
}
// the other connected rows: the aggregate of their assigned neighbour of largest priority
__global__ void __launch_bounds__(256) k_amg_assign2(int n, const int* __restrict__ ia, const int* __restrict__ ja, const int* __restrict__ agg1, int* __restrict__ agg)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int a = agg1[i];
    if (a < 0) {
        int best = -1;
        unsigned long long hb = 0;
        for (int e = ia[i]; e < ia[i + 1]; ++e) {
            const int j = ja[e];
            if (j == i || agg1[j] < 0) continue;
            const unsigned long long h = splitmix64((unsigned long long)j);
            if (best < 0 || h > hb || (h == hb && j > best)) {
                best = j;
                hb = h;
            }
        }
        a = best >= 0 ? agg1[best] : -1;
    }
    agg[i] = a;
}

// step 4, one thread per row: pia == NULL counts the row's distinct aggregates into cnt, otherwise writes the row of P at pia[i]
__global__ void __launch_bounds__(256) k_amg_prolongator(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ dinv, const int* __restrict__ agg, double omega, const int* __restrict__ pia, int* __restrict__ cnt, int* __restrict__ pja,
    double* __restrict__ pblk, int* __restrict__ prow)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* m = dinv + 9 * (size_t)i;
    int out = pia ? pia[i] : 0, last = -1;
    for (;;) {
        int col = INT_MAX;
        for (int e = ia[i]; e < ia[i + 1]; ++e) {
            const int c = agg[ja[e]];
            if (c > last && c < col) col = c;
        }
        if (col == INT_MAX) break;
        if (pia) {
            double acc[9];
            bool first = true;
            for (int e = ia[i]; e < ia[i + 1]; ++e) {
                if (agg[ja[e]] != col) continue;
                const double* B = blk + 9 * (size_t)e;
                const bool eye = ja[e] == i;
#pragma unroll
                for (int c = 0; c < 3; ++c)
#pragma unroll
                    for (int d = 0; d < 3; ++d) {
                        double v = -omega * (m[3 * c] * B[d] + m[3 * c + 1] * B[3 + d] + m[3 * c + 2] * B[6 + d]);
                        if (eye && c == d) v += 1.0;
                        acc[3 * c + d] = first ? v : acc[3 * c + d] + v;
                    }
                first = false;
            }
            pja[out] = col;
            prow[out] = i;
#pragma unroll
            for (int q = 0; q < 9; ++q) pblk[9 * (size_t)out + q] = acc[q];
        }
        ++out;
        last = col;
    }
    if (!pia) cnt[i] = out;
}

// R = P^T: keys (column, row) of P's entries
__global__ void __launch_bounds__(256) k_amg_tkeys(int np, int n, const int* __restrict__ pja, const int* __restrict__ prow, unsigned long long* __restrict__ key,
    int* __restrict__ pos)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= np) return;
    key[e] = (unsigned long long)pja[e] * (unsigned long long)n + (unsigned long long)prow[e];
    pos[e] = e;
}
__global__ void __launch_bounds__(256) k_amg_tfill(int np, int n, int nc, const unsigned long long* __restrict__ key, const int* __restrict__ pos,
    const double* __restrict__ pblk, int* __restrict__ ria, int* __restrict__ rja, double* __restrict__ rblk)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < np) {
        const unsigned long long k = key[e];
        const int c = (int)(k / (unsigned long long)n);
        rja[e] = (int)(k % (unsigned long long)n);
        const double* B = pblk + 9 * (size_t)pos[e];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) rblk[9 * (size_t)e + 3 * a + b] = B[3 * b + a];
        // row starts: the first entry of every column, and the columns without entries before it
        const int prev = e ? (int)(key[e - 1] / (unsigned long long)n) : -1;
        for (int q = prev + 1; q <= c; ++q) ria[q] = e;
        if (e == np - 1)
            for (int q = c + 1; q <= nc; ++q) ria[q] = np;
    }
}

// step 5: C = Lm Rm.  Entries of the products per row, then their enumeration, then the stable sort, then the sums
__global__ void __launch_bounds__(256) k_amg_gemm_count(int n, const int* __restrict__ lia, const int* __restrict__ lja, const int* __restrict__ ria, int* __restrict__ cnt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int s = 0;
    for (int e = lia[i]; e < lia[i + 1]; ++e) s += ria[lja[e] + 1] - ria[lja[e]];
    cnt[i] = s;
}
__global__ void __launch_bounds__(256) k_amg_gemm_expand(int n, const int* __restrict__ lia, const int* __restrict__ lja, const int* __restrict__ ria,
    const int* __restrict__ rja, const int* __restrict__ off, int* __restrict__ key, int* __restrict__ pos, int* __restrict__ lidx, int* __restrict__ ridx)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int p = off[i];
    for (int e = lia[i]; e < lia[i + 1]; ++e)
        for (int f = ria[lja[e]]; f < ria[lja[e] + 1]; ++f, ++p) {
            key[p] = rja[f];
            pos[p] = p;
            lidx[p] = e;
            ridx[p] = f;
        }
}
// cia == NULL: distinct columns per row into cnt; otherwise the row's blocks, each the sum of its run in sorted (stable) order
__global__ void __launch_bounds__(256) k_amg_gemm_fill(int n, const int* __restrict__ off, const int* __restrict__ skey, const int* __restrict__ spos,
    const int* __restrict__ lidx, const int* __restrict__ ridx, const double* __restrict__ lblk, const double* __restrict__ rblk, const int* __restrict__ cia,
    int* __restrict__ cnt, int* __restrict__ cja, double* __restrict__ cblk)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int p0 = off[i], p1 = off[i + 1];
    if (!cia) {
        int d = 0;
        for (int p = p0; p < p1; ++p) d += p == p0 || skey[p] != skey[p - 1];
        cnt[i] = d;
        return;
    }
    int out = cia[i];
    double acc[9];
    for (int p = p0; p < p1; ++p) {
        const double* A = lblk + 9 * (size_t)lidx[spos[p]];
        const double* B = rblk + 9 * (size_t)ridx[spos[p]];
        const bool first = p == p0 || skey[p] != skey[p - 1];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) {
                const double v = A[3 * a] * B[b] + A[3 * a + 1] * B[3 + b] + A[3 * a + 2] * B[6 + b];
                acc[3 * a + b] = first ? v : acc[3 * a + b] + v;
            }
        if (p + 1 == p1 || skey[p + 1] != skey[p]) {
            cja[out] = skey[p];
#pragma unroll
            for (int q = 0; q < 9; ++q) cblk[9 * (size_t)out + q] = acc[q];
            ++out;
        }
    }
}

// y_i = D_i^-1 sum_j A_ij b_j  (times s = 1 / sqrt(*sq) when sq != NULL, 1 otherwise); per-CTA partial of |y|^2.  start != 0: b_0 from splitmix64
__global__ void __launch_bounds__(256) k_amg_power(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ dinv, const double* __restrict__ b, const double* __restrict__ sq, double* __restrict__ y, double* __restrict__ part, int start)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double yy = 0.0;
    if (i < n) {
        const double s = sq ? 1.0 / sqrt(*sq) : 1.0;
        double q[3] = { 0.0, 0.0, 0.0 };
        for (int e = ia[i]; e < ia[i + 1]; ++e) {
            const int j = ja[e];
            double bj[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                if (start) bj[c] = (double)(splitmix64((unsigned long long)(3 * (long long)j + c)) >> 11) * 0x1p-52 - 1.0;
                else bj[c] = b[3 * (size_t)j + c] * s;
            }
            const double* B = blk + 9 * (size_t)e;
#pragma unroll
            for (int c = 0; c < 3; ++c) q[c] += B[3 * c] * bj[0] + B[3 * c + 1] * bj[1] + B[3 * c + 2] * bj[2];
        }
        const double* m = dinv + 9 * (size_t)i;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double v = m[3 * c] * q[0] + m[3 * c + 1] * q[1] + m[3 * c + 2] * q[2];
            y[3 * (size_t)i + c] = v;
            yy += v * v;
        }
    }
    cta_sum(&yy, part + blockIdx.x);
}

// ---- application ------------------------------------------------------------------------------------------------------------
DEV void amg_row_product(int i, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk, const double* __restrict__ v, double q[3])
{
    q[0] = q[1] = q[2] = 0.0;
    for (int e = ia[i]; e < ia[i + 1]; ++e) {
        const double* B = blk + 9 * (size_t)e;
        const double* x = v + 3 * (size_t)ja[e];
        const double x0 = x[0], x1 = x[1], x2 = x[2];
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c] += B[3 * c] * x0 + B[3 * c + 1] * x1 + B[3 * c + 2] * x2;
    }
}
DEV void amg_dinv(const double* __restrict__ dinv, int i, const double q[3], double out[3])
{
    const double* m = dinv + 9 * (size_t)i;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = m[3 * c] * q[0] + m[3 * c + 1] * q[1] + m[3 * c + 2] * q[2];
}

// first kernel of a Chebyshev application: r = D^-1 (f - A x) (zero: x = 0, no product), d = r / theta.  cg_p != NULL (level 0 in an
// iteration, zero): first the CG update x_s += alpha p, f -= alpha Ap (Ap in x's storage), alpha = scal[0] / (the n_dot SpMV partials)
__global__ void __launch_bounds__(256) k_amg_cheb_init(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ dinv, double* __restrict__ f, double* __restrict__ x, double* __restrict__ r, double* __restrict__ d, double inv_theta, int zero,
    const double* __restrict__ cg_p, double* __restrict__ cg_x, const double* __restrict__ scal, const double* __restrict__ dot, int n_dot)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    __shared__ double pAp;
    if (cg_p) {
        double s = 0.0;
        for (int k = threadIdx.x; k < n_dot; k += blockDim.x) s += dot[k];
        cta_sum(&s, &pAp);
        __syncthreads();
    }
    if (i >= n) return;
    double q[3] = { 0.0, 0.0, 0.0 };
    if (!zero) amg_row_product(i, ia, ja, blk, x, q);
    double fv[3];
    const double alpha = cg_p && pAp != 0.0 ? scal[0] / pAp : 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t k = 3 * (size_t)i + c;
        fv[c] = f[k];
        if (cg_p) {
            cg_x[k] += alpha * cg_p[k];
            fv[c] -= alpha * x[k];
            f[k] = fv[c];
        }
        q[c] = fv[c] - q[c];
    }
    double rv[3];
    amg_dinv(dinv, i, q, rv);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t k = 3 * (size_t)i + c;
        r[k] = rv[c];
        d[k] = rv[c] * inv_theta;
        if (zero) x[k] = 0.0;
    }
}

// step k of a Chebyshev application: x += d ; r -= D^-1 A d ; d' = c1 d + c2 r ; last (k = 15): x += d' too.  part != NULL: the per-CTA
// partials of f.x and f.f (level 0's last kernel: r.z and r.r of the Krylov loop)
__global__ void __launch_bounds__(256) k_amg_cheb_step(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ dinv, double* __restrict__ x, double* __restrict__ r, const double* __restrict__ d, double* __restrict__ dn, double c1, double c2,
    int last, const double* __restrict__ f, double* __restrict__ part)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double rz_rr[2] = { 0.0, 0.0 };
    if (i < n) {
        double q[3], u[3];
        amg_row_product(i, ia, ja, blk, d, q);
        amg_dinv(dinv, i, q, u);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t k = 3 * (size_t)i + c;
            const double dk = d[k];
            const double rk = r[k] - u[c];
            const double dnk = c1 * dk + c2 * rk;
            double xk = x[k] + dk;
            if (last) xk += dnk;
            else {
                r[k] = rk;
                dn[k] = dnk;
            }
            x[k] = xk;
            if (part) {
                const double fk = f[k];
                rz_rr[0] += fk * xk;
                rz_rr[1] += fk * fk;
            }
        }
    }
    if (part) cta_sum<2>(rz_rr, part + 2 * blockIdx.x);
}

// t = f - A x
__global__ void __launch_bounds__(256) k_amg_residual(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ f, const double* __restrict__ x, double* __restrict__ t)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double q[3];
    amg_row_product(i, ia, ja, blk, x, q);
#pragma unroll
    for (int c = 0; c < 3; ++c) t[3 * (size_t)i + c] = f[3 * (size_t)i + c] - q[c];
}
// y = M v (restriction with R), or y += M v (prolongation with P)
__global__ void __launch_bounds__(256) k_amg_transfer(int n, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk,
    const double* __restrict__ v, double* __restrict__ y, int add)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double q[3];
    amg_row_product(i, ia, ja, blk, v, q);
#pragma unroll
    for (int c = 0; c < 3; ++c) y[3 * (size_t)i + c] = add ? y[3 * (size_t)i + c] + q[c] : q[c];
}

} // namespace ipcgpu

using namespace ipcgpu;

// exclusive scan of cnt[0, n) into out[0, n] (cnt[n] is set to 0 first); returns the total, read back
static int amg_scan(ipcgpu_ctx* ctx, int* cnt, int* out, int n, long long* total)
{
    AmgWork& w = ctx->amg;
    cudaStream_t st = ctx->stream;
    size_t bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt, out, n + 1, st));
    REQUIRE(w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG scan workspace allocation failed");
    CK(cudaMemsetAsync(cnt + n, 0, sizeof(int), st));
    CK(cub::DeviceScan::ExclusiveSum(w.tmp.p, bytes, cnt, out, n + 1, st));
    int t = 0;
    CK(cudaMemcpyAsync(&t, out + n, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    ctx->launches += 2;
    *total = t;
    return IPCGPU_OK;
}

// C = Lm Rm (step 5): n rows of Lm; Lm's and Rm's block CSR.  C's arrays are reserved here
static int amg_gemm(ipcgpu_ctx* ctx, int n, const int* lia, const int* lja, const double* lblk, const int* ria, const int* rja, const double* rblk,
    DevBuf<int>& cia, DevBuf<int>& cja, DevBuf<double>& cblk, int* nnz_out)
{
    AmgWork& w = ctx->amg;
    cudaStream_t st = ctx->stream;
    const int g = nblk(n, 256);
    REQUIRE(w.cnt.reserve((size_t)n + 1) && w.scan_out.reserve((size_t)n + 1) && cia.reserve((size_t)n + 1), IPCGPU_ERR_CUDA, "AMG product allocation failed");
    k_amg_gemm_count<<<g, 256, 0, st>>>(n, lia, lja, ria, w.cnt.p);
    ++ctx->launches;
    long long T = 0;
    int rc = amg_scan(ctx, w.cnt.p, w.scan_out.p, n, &T);
    if (rc) return rc;
    REQUIRE(T < INT_MAX, IPCGPU_ERR_CUDA, "AMG product: too many entries for an int index");
    const size_t t = std::max<long long>(T, 1);
    REQUIRE(w.key.reserve(t) && w.pos.reserve(t) && w.lidx.reserve(t) && w.ridx.reserve(t) && w.skey.reserve(t) && w.spos.reserve(t), IPCGPU_ERR_CUDA,
        "AMG product allocation failed");
    k_amg_gemm_expand<<<g, 256, 0, st>>>(n, lia, lja, ria, rja, w.scan_out.p, w.key.p, w.pos.p, w.lidx.p, w.ridx.p);
    size_t bytes = 0;
    CK(cub::DeviceSegmentedSort::StableSortPairs(nullptr, bytes, w.key.p, w.skey.p, w.pos.p, w.spos.p, (int)T, n, w.scan_out.p, w.scan_out.p + 1, st));
    REQUIRE(w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG sort workspace allocation failed");
    CK(cub::DeviceSegmentedSort::StableSortPairs(w.tmp.p, bytes, w.key.p, w.skey.p, w.pos.p, w.spos.p, (int)T, n, w.scan_out.p, w.scan_out.p + 1, st));
    k_amg_gemm_fill<<<g, 256, 0, st>>>(n, w.scan_out.p, w.skey.p, w.spos.p, w.lidx.p, w.ridx.p, lblk, rblk, nullptr, w.cnt.p, nullptr, nullptr);
    ctx->launches += 3;
    long long nnz = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, cia.p, n, &nnz))) return rc;
    REQUIRE(cja.reserve(std::max<long long>(nnz, 1)) && cblk.reserve(9 * (size_t)std::max<long long>(nnz, 1)), IPCGPU_ERR_CUDA, "AMG level allocation failed");
    k_amg_gemm_fill<<<g, 256, 0, st>>>(n, w.scan_out.p, w.skey.p, w.spos.p, w.lidx.p, w.ridx.p, lblk, rblk, cia.p, nullptr, cja.p, cblk.p);
    ++ctx->launches;
    CK(cudaGetLastError());
    *nnz_out = (int)nnz;
    return IPCGPU_OK;
}

// the vectors, D^-1, the Gershgorin bound and rho of level l (its matrix built); *fail: a pivot <= 0 or a non-finite rho or omega bound
static int amg_level_setup(ipcgpu_ctx* ctx, int l, bool* fail, double* rho_g)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    cudaStream_t st = ctx->stream;
    const int n = L.n, g = nblk(n, 256);
    const size_t n3 = 3 * (size_t)n;
    bool ok = L.dinv.reserve(9 * (size_t)n) && L.r.reserve(n3) && L.d0.reserve(n3) && L.d1.reserve(n3) && L.t.reserve(n3) && w.state0.reserve(n)
        && w.state1.reserve(n) && w.part.reserve(g) && w.sq.reserve(kAmgPowerSteps) && w.absrow.reserve(1) && w.flags.reserve(4);
    if (l > 0) ok = ok && L.f.reserve(n3) && L.x.reserve(n3);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "AMG level allocation failed");
    CK(cudaMemsetAsync(w.absrow.p, 0, sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(w.flags.p + 2, 0, sizeof(int), st));
    k_amg_diag<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, w.absrow.p, w.state0.p, w.flags.p);
    ++ctx->launches;
    // power iteration (step 7): y_k = D^-1 A (y_{k-1} / |y_{k-1}|), |y_k|^2 in sq[k-1]; rho = |y_100| (|b_99| = 1)
    double* y[2] = { L.d0.p, L.d1.p };
    for (int k = 0; k < kAmgPowerSteps; ++k) {
        k_amg_power<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, k ? y[(k - 1) & 1] : nullptr, k ? w.sq.p + k - 1 : nullptr, y[k & 1], w.part.p, k == 0);
        reduce_sum(w.part.p, g, 1.0, w.sq.p + k, st);
    }
    ctx->launches += 2 * kAmgPowerSteps;
    CK(cudaGetLastError());
    int bad = 0;
    unsigned long long ord = 0;
    double sq = 0.0;
    CK(cudaMemcpyAsync(&bad, w.flags.p + 2, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ord, w.absrow.p, sizeof(ord), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&sq, w.sq.p + kAmgPowerSteps - 1, sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    std::memcpy(rho_g, &ord, sizeof(double));
    L.rho = std::sqrt(sq);
    *fail = bad != 0 || !std::isfinite(L.rho) || !(L.rho > 0.0) || !std::isfinite(*rho_g);
    if (*fail) L.rho = 1.0; // (coefficients that make no NaN: the solve stops before its first iteration)
    // Chebyshev coefficients, in the mirror's order
    const double hi = 2.0 * L.rho, lo = hi / 120.0;
    const double theta = 0.5 * (hi + lo), delta = 0.5 * (hi - lo), sigma = theta / delta;
    L.theta = theta;
    double rho_prev = 1.0 / sigma;
    for (int k = 1; k < kAmgDegree; ++k) {
        const double rho_k = 1.0 / (2.0 * sigma - rho_prev);
        L.c1[k] = rho_k * rho_prev;
        L.c2[k] = 2.0 * rho_k / delta;
        rho_prev = rho_k;
    }
    return IPCGPU_OK;
}

// aggregation and P, R of level l (steps 2-4); *nagg = 0 when the level makes no aggregate
static int amg_coarsen(ipcgpu_ctx* ctx, int l, double rho_g, int* nagg)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    cudaStream_t st = ctx->stream;
    const int n = L.n, g = nblk(n, 256);
    REQUIRE(w.m1.reserve(n) && w.m2.reserve(n) && w.cnt.reserve((size_t)n + 1) && w.scan_out.reserve((size_t)n + 1) && L.agg.reserve(n) && L.pia.reserve((size_t)n + 1),
        IPCGPU_ERR_CUDA, "AMG aggregation allocation failed");
    unsigned char* s_in = w.state0.p; // (k_amg_diag left the connected rows undecided there)
    unsigned char* s_out = w.state1.p;
    for (int round = 0;; ++round) {
        REQUIRE(round <= n, IPCGPU_ERR_CUDA, "AMG aggregation did not converge");
        CK(cudaMemsetAsync(w.flags.p, 0, sizeof(int), st));
        k_amg_mis_max<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, nullptr, s_in, w.m1.p);
        k_amg_mis_max<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, w.m1.p, s_in, w.m2.p);
        k_amg_mis_update<<<g, 256, 0, st>>>(n, w.m2.p, s_in, s_out, w.flags.p);
        ctx->launches += 3;
        int undecided = 0;
        CK(cudaMemcpyAsync(&undecided, w.flags.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        std::swap(s_in, s_out);
        if (undecided == 0) break;
    }
    k_amg_roots<<<g, 256, 0, st>>>(n, s_in, w.cnt.p);
    ++ctx->launches;
    long long na = 0;
    int rc = amg_scan(ctx, w.cnt.p, w.scan_out.p, n, &na);
    if (rc) return rc;
    *nagg = (int)na;
    if (na == 0 || 5 * na > 4 * (long long)n) return IPCGPU_OK;
    k_amg_assign1<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, s_in, w.scan_out.p, w.m1.p);
    k_amg_assign2<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, w.m1.p, L.agg.p);
    L.omega = (4.0 / 3.0) / rho_g;
    k_amg_prolongator<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, L.agg.p, L.omega, nullptr, w.cnt.p, nullptr, nullptr, nullptr);
    ctx->launches += 3;
    long long np = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, L.pia.p, n, &np))) return rc;
    L.np = (int)np;
    const size_t np1 = std::max<long long>(np, 1);
    REQUIRE(L.pja.reserve(np1) && L.pblk.reserve(9 * np1) && w.prow.reserve(np1) && L.ria.reserve((size_t)na + 1) && L.rja.reserve(np1) && L.rblk.reserve(9 * np1)
            && w.tkey.reserve(np1) && w.tkey_sorted.reserve(np1) && w.pos.reserve(np1) && w.spos.reserve(np1),
        IPCGPU_ERR_CUDA, "AMG prolongator allocation failed");
    k_amg_prolongator<<<g, 256, 0, st>>>(n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, L.agg.p, L.omega, L.pia.p, nullptr, L.pja.p, L.pblk.p, w.prow.p);
    // R = P^T: sort (column, row), then rows of R = runs of equal column
    k_amg_tkeys<<<nblk(np, 256), 256, 0, st>>>((int)np, n, L.pja.p, w.prow.p, w.tkey.p, w.pos.p);
    size_t bytes = 0;
    int bits = 1;
    while (bits < 64 && ((unsigned long long)na * (unsigned long long)n) >> bits) ++bits;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, w.tkey.p, w.tkey_sorted.p, w.pos.p, w.spos.p, (int)np, 0, bits, st));
    REQUIRE(w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG sort workspace allocation failed");
    CK(cub::DeviceRadixSort::SortPairs(w.tmp.p, bytes, w.tkey.p, w.tkey_sorted.p, w.pos.p, w.spos.p, (int)np, 0, bits, st));
    k_amg_tfill<<<nblk(np, 256), 256, 0, st>>>((int)np, n, (int)na, w.tkey_sorted.p, w.spos.p, L.pblk.p, L.ria.p, L.rja.p, L.rblk.p);
    ctx->launches += 4;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// the hierarchy of the resident matrix (steps 1-8).  A pivot <= 0 or a non-finite spectral radius leaves 1.0 in *bad_pivot and ends the
// hierarchy at that level
int solver_amg_build(ipcgpu_ctx* ctx, double* bad_pivot)
{
    AmgWork& w = ctx->amg;
    cudaStream_t st = ctx->stream;
    w.built = false;
    w.levels = 0;
    const int nb = ctx->nV;
    AmgLevel& L0 = w.lv[0];
    REQUIRE(w.flags.reserve(4) && w.cnt.reserve((size_t)nb + 1) && L0.ia.reserve((size_t)nb + 1), IPCGPU_ERR_CUDA, "AMG allocation failed");
    CK(cudaMemsetAsync(w.flags.p, 0, 4 * sizeof(int), st));
    k_amg_level0<<<nblk(nb, 256), 256, 0, st>>>(nb, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, nullptr, w.cnt.p, nullptr, nullptr, w.flags.p);
    ++ctx->launches;
    long long nnzb = 0;
    int rc = amg_scan(ctx, w.cnt.p, L0.ia.p, nb, &nnzb);
    if (rc) return rc;
    int layout = 0;
    CK(cudaMemcpyAsync(&layout, w.flags.p + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    REQUIRE(!layout, IPCGPU_ERR_ARG, "ipcgpu_solve_pcg_amg: the pattern is not LinSysSolver::set_pattern's 3 x 3 block layout");
    REQUIRE(L0.ja.reserve(std::max<long long>(nnzb, 1)) && L0.blk.reserve(9 * (size_t)std::max<long long>(nnzb, 1)), IPCGPU_ERR_CUDA, "AMG level allocation failed");
    k_amg_level0<<<nblk(nb, 256), 256, 0, st>>>(nb, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, L0.ia.p, nullptr, L0.ja.p, L0.blk.p, w.flags.p);
    ++ctx->launches;
    L0.n = nb;
    L0.nnzb = (int)nnzb;
    for (int l = 0;; ++l) {
        AmgLevel& L = w.lv[l];
        L.np = 0;
        L.omega = 0.0;
        w.levels = l + 1;
        bool fail = false;
        double rho_g = 0.0;
        if ((rc = amg_level_setup(ctx, l, &fail, &rho_g))) return rc;
        if (fail) {
            const double one = 1.0;
            CK(cudaMemcpyAsync(bad_pivot, &one, sizeof(double), cudaMemcpyHostToDevice, st));
            CK(cudaStreamSynchronize(st));
            return IPCGPU_OK;
        }
        if (l + 1 == kAmgMaxLevels || L.n <= kAmgCoarseEnough) break;
        int nagg = 0;
        if ((rc = amg_coarsen(ctx, l, rho_g, &nagg))) return rc;
        if (L.np == 0) { // (no aggregate, or less than a fifth fewer rows: this level is the last)
            L.omega = 0.0;
            break;
        }
        AmgLevel& C = w.lv[l + 1];
        // A_{l+1} = R (A_l P); A_l P lives only for this level's product
        DevBuf<int> api, apj;
        DevBuf<double> apb;
        int nap = 0, nc = 0;
        if ((rc = amg_gemm(ctx, L.n, L.ia.p, L.ja.p, L.blk.p, L.pia.p, L.pja.p, L.pblk.p, api, apj, apb, &nap))) return rc;
        if ((rc = amg_gemm(ctx, nagg, L.ria.p, L.rja.p, L.rblk.p, api.p, apj.p, apb.p, C.ia, C.ja, C.blk, &nc))) return rc;
        CK(cudaStreamSynchronize(st)); // (api / apj / apb are freed on return)
        C.n = nagg;
        C.nnzb = nc;
    }
    w.built = true;
    return IPCGPU_OK;
}

// one Chebyshev application at level l on (f, x); zero: from x = 0; cg: level 0's first in an iteration (the CG update); part: level 0's last
static void amg_chebyshev(ipcgpu_ctx* ctx, int l, double* f, double* x, bool zero, bool cg, double* part)
{
    AmgLevel& L = ctx->amg.lv[l];
    cudaStream_t st = ctx->stream;
    const int g = nblk(L.n, 256);
    k_amg_cheb_init<<<g, 256, 0, st>>>(L.n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, f, x, L.r.p, L.d0.p, 1.0 / L.theta, zero ? 1 : 0, cg ? ctx->pcg_p.p : nullptr,
        cg ? ctx->sol.p : nullptr, ctx->pcg_scal.p, ctx->pcg_part.p, kPcgSpmvBlocks);
    double* d[2] = { L.d0.p, L.d1.p };
    for (int k = 1; k < kAmgDegree; ++k) {
        const bool last = k == kAmgDegree - 1;
        k_amg_cheb_step<<<g, 256, 0, st>>>(L.n, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, x, L.r.p, d[(k - 1) & 1], d[k & 1], L.c1[k], L.c2[k], last ? 1 : 0, f,
            last ? part : nullptr);
    }
    ctx->launches += kAmgDegree;
}

// one visit of level l (W-cycle)
static void amg_cycle(ipcgpu_ctx* ctx, int l, double* f, double* x, bool zero, bool cg, double* part)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    cudaStream_t st = ctx->stream;
    if (l == w.levels - 1) {
        amg_chebyshev(ctx, l, f, x, zero, cg, nullptr);
        amg_chebyshev(ctx, l, f, x, false, false, part);
        return;
    }
    AmgLevel& C = w.lv[l + 1];
    amg_chebyshev(ctx, l, f, x, zero, cg, nullptr);
    k_amg_residual<<<nblk(L.n, 256), 256, 0, st>>>(L.n, L.ia.p, L.ja.p, L.blk.p, f, x, L.t.p);
    k_amg_transfer<<<nblk(C.n, 256), 256, 0, st>>>(C.n, L.ria.p, L.rja.p, L.rblk.p, L.t.p, C.f.p, 0);
    ctx->launches += 2;
    for (int v = 0; v < kAmgCycles; ++v) amg_cycle(ctx, l + 1, C.f.p, C.x.p, v == 0, false, nullptr);
    k_amg_transfer<<<nblk(L.n, 256), 256, 0, st>>>(L.n, L.pia.p, L.pja.p, L.pblk.p, C.x.p, x, 1);
    ++ctx->launches;
    amg_chebyshev(ctx, l, f, x, false, false, part);
}

// the AMG step of solver_pcg (solve.cu).  In an iteration: the CG update (inside the first kernel).  Then z = M^-1 r in pcg_q, and the
// partials of r.z and r.r behind the SpMV's
void solver_amg_step(ipcgpu_ctx* ctx, bool start)
{
    amg_cycle(ctx, 0, ctx->pcg_r.p, ctx->pcg_q.p, true, !start, ctx->pcg_part.p + kPcgSpmvBlocks);
}

size_t solver_amg_bytes(const ipcgpu_ctx* ctx)
{
    const AmgWork& w = ctx->amg;
    size_t b = (w.cnt.n + w.scan_out.n + w.m1.n + w.m2.n + w.key.n + w.pos.n + w.lidx.n + w.ridx.n + w.skey.n + w.spos.n + w.prow.n + w.flags.n) * sizeof(int)
        + (w.tkey.n + w.tkey_sorted.n + w.absrow.n) * 8 + w.state0.n + w.state1.n + w.tmp.n + (w.part.n + w.sq.n) * sizeof(double);
    for (const AmgLevel& L : w.lv)
        b += (L.ia.n + L.ja.n + L.agg.n + L.pia.n + L.pja.n + L.ria.n + L.rja.n) * sizeof(int)
            + (L.blk.n + L.dinv.n + L.pblk.n + L.rblk.n + L.f.n + L.x.n + L.r.n + L.d0.n + L.d1.n + L.t.n) * sizeof(double);
    return b;
}
