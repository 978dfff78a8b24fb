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
//      order), stably sorted by column (one radix sort of (row, column) keys), then summed run by run in that order.
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

constexpr int kAmgPowerSteps = 100;
constexpr int kAmgCoarseEnough = 1000; // block rows (3,000 unknowns); ipcgpu_amg_debug_coarse_enough moves it
constexpr int kAmgCycles = 2;          // W-cycle
constexpr int kAmgGridMax = kSMs * 8;  // CTAs of a coarse level's launches (grid-stride beyond)
enum { kFitLevel0 = -2, kFitAgg = -1 }; // k_amg_fit's other rules (the rest are kAmgQ*)

// rows i < n of a launch, grid-stride
#define AMG_ROWS(i, n) for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += gridDim.x * blockDim.x)

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

// a set-up starts: nothing built, level 0 has nb rows
__global__ void k_amg_begin(AmgDev* __restrict__ d, int nb)
{
    if (threadIdx.x) return;
    for (int l = 0; l < kAmgMaxLevels; ++l) {
        d->n[l] = d->nnzb[l] = d->np[l] = d->na[l] = d->go[l] = 0;
        d->rho[l] = d->rho_g[l] = d->omega[l] = d->inv_theta[l] = 0.0;
        for (int q = 0; q < kAmgQty; ++q) d->need[l][q] = 0;
    }
    d->n[0] = nb;
    d->levels = d->fail = d->cut_depth = 0;
    d->cut_level = -1;
}

// step 6 (and the Gershgorin bound of step 4, the connections of step 2): D_i^-1 by Cholesky (identity and flags[2] on a pivot <= 0 or a
// missing diagonal block), max absolute row sum of D^-1 A into *absrow, state 1 (undecided) for a connected row, 0 otherwise
__global__ void __launch_bounds__(256) k_amg_diag(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, double* __restrict__ dinv, unsigned long long* __restrict__ absrow, unsigned char* __restrict__ state, int* __restrict__ flags)
{
    AMG_ROWS(i, dv->n[l]) {
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
}

// step 3: does row a hold a larger (state, priority) than row b
DEV bool amg_above(int a, int b, const unsigned char* __restrict__ s)
{
    if (s[a] != s[b]) return s[a] > s[b];
    const unsigned long long ha = splitmix64((unsigned long long)a), hb = splitmix64((unsigned long long)b);
    return ha != hb ? ha > hb : a > b;
}
// out[i] = the row of largest key among src[j] for j in the closed neighbourhood of i (src NULL: j itself)
__global__ void __launch_bounds__(256) k_amg_mis_max(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const int* __restrict__ src, const unsigned char* __restrict__ state, int* __restrict__ out)
{
    AMG_ROWS(i, dv->n[l]) {
        int best = src ? src[i] : i;
        for (int e = ia[i]; e < ia[i + 1]; ++e) {
            const int c = src ? src[ja[e]] : ja[e];
            if (amg_above(c, best, state)) best = c;
        }
        out[i] = best;
    }
}
// an undecided row that is the largest of its distance-2 neighbourhood becomes a root (2); one whose largest is a root is out (0).
// undecided != NULL: the rows still undecided are counted there
__global__ void __launch_bounds__(256) k_amg_mis_update(const AmgDev* __restrict__ dv, int l, const int* __restrict__ m2, const unsigned char* __restrict__ in,
    unsigned char* __restrict__ out, int* __restrict__ undecided)
{
    AMG_ROWS(i, dv->n[l]) {
        unsigned char s = in[i];
        if (s == 1) {
            const int w = m2[i];
            s = w == i ? 2 : in[w] == 2 ? 0 : 1;
            if (s == 1 && undecided) atomicAdd(undecided, 1);
        }
        out[i] = s;
    }
}
// the aggregation rounds of level l start: their loop runs when the level is coarsened, at most (rows) passes
__global__ void k_amg_agg_begin(const AmgDev* __restrict__ d, int l, IterState* __restrict__ st)
{
    if (threadIdx.x) return;
    st->amg_round = st->amg_undecided = st->amg_stuck = 0;
    st->amg_limit = d->go[l] ? d->n[l] : 0;
}
// flag[i] = row i is a root, for i <= cap (0 from the level's rows on, and everywhere when the level is not coarsened)
__global__ void __launch_bounds__(256) k_amg_roots(const AmgDev* __restrict__ dv, int l, int cap, const unsigned char* __restrict__ state, int* __restrict__ flag)
{
    const int n = dv->go[l] ? dv->n[l] : 0;
    AMG_ROWS(i, cap + 1) flag[i] = i < n && state[i] == 2;
}
// a root: its aggregate; a neighbour of a root: that root's (unique: roots are at least 3 apart); otherwise -1
__global__ void __launch_bounds__(256) k_amg_assign1(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const unsigned char* __restrict__ state, const int* __restrict__ id, int* __restrict__ agg1)
{
    AMG_ROWS(i, dv->go[l] ? dv->n[l] : 0) {
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
}
// the other connected rows: the aggregate of their assigned neighbour of largest priority
__global__ void __launch_bounds__(256) k_amg_assign2(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const int* __restrict__ agg1, int* __restrict__ agg)
{
    AMG_ROWS(i, dv->go[l] ? dv->n[l] : 0) {
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
}

// step 4, row i of P: pia == NULL counts its distinct aggregates (returned), otherwise writes the row at pia[i]
DEV int amg_p_row(int i, const int* __restrict__ ia, const int* __restrict__ ja, const double* __restrict__ blk, const double* __restrict__ dinv,
    const int* __restrict__ agg, double omega, const int* __restrict__ pia, int* __restrict__ pja, double* __restrict__ pblk, int* __restrict__ prow)
{
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
    return out;
}
// pia == NULL: the counts into cnt[0, cap] (0 from the level's rows on); otherwise the rows of P
__global__ void __launch_bounds__(256) k_amg_prolongator(const AmgDev* __restrict__ dv, int l, int cap, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, const double* __restrict__ dinv, const int* __restrict__ agg, const int* __restrict__ pia, int* __restrict__ cnt,
    int* __restrict__ pja, double* __restrict__ pblk, int* __restrict__ prow)
{
    const int n = dv->go[l] ? dv->n[l] : 0;
    const double omega = dv->omega[l];
    if (!pia) {
        AMG_ROWS(i, cap + 1) cnt[i] = i < n ? amg_p_row(i, ia, ja, blk, dinv, agg, omega, nullptr, nullptr, nullptr, nullptr) : 0;
        return;
    }
    AMG_ROWS(i, n) amg_p_row(i, ia, ja, blk, dinv, agg, omega, pia, pja, pblk, prow);
}

// R = P^T: keys (column, row) of P's entries, then `pad` (above every key) up to the capacity
__global__ void __launch_bounds__(256) k_amg_tkeys(const AmgDev* __restrict__ dv, int l, int cap, unsigned long long pad, const int* __restrict__ pja,
    const int* __restrict__ prow, unsigned long long* __restrict__ key, int* __restrict__ pos)
{
    const int np = dv->go[l] ? dv->np[l] : 0;
    const unsigned long long n = (unsigned long long)dv->n[l];
    AMG_ROWS(e, cap) {
        key[e] = e < np ? (unsigned long long)pja[e] * n + (unsigned long long)prow[e] : pad;
        pos[e] = e;
    }
}
__global__ void __launch_bounds__(256) k_amg_tfill(const AmgDev* __restrict__ dv, int l, const unsigned long long* __restrict__ key, const int* __restrict__ pos,
    const double* __restrict__ pblk, int* __restrict__ ria, int* __restrict__ rja, double* __restrict__ rblk)
{
    const int np = dv->go[l] ? dv->np[l] : 0, nc = dv->na[l];
    const unsigned long long n = (unsigned long long)dv->n[l];
    AMG_ROWS(e, np) {
        const unsigned long long k = key[e];
        const int c = (int)(k / n);
        rja[e] = (int)(k % n);
        const double* B = pblk + 9 * (size_t)pos[e];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) rblk[9 * (size_t)e + 3 * a + b] = B[3 * b + a];
        // row starts: the first entry of every column, and the columns without entries before it
        const int prev = e ? (int)(key[e - 1] / n) : -1;
        for (int q = prev + 1; q <= c; ++q) ria[q] = e;
        if (e == np - 1)
            for (int q = c + 1; q <= nc; ++q) ria[q] = np;
    }
}

// step 5: C = Lm Rm over the *rows rows of Lm, when *go.  Entries of the products per row (cnt[0, cap], 0 from *rows on), then their
// enumeration, then the stable sort, then the sums
__global__ void __launch_bounds__(256) k_amg_gemm_count(const int* __restrict__ rows, const int* __restrict__ go, int cap, const int* __restrict__ lia,
    const int* __restrict__ lja, const int* __restrict__ ria, int* __restrict__ cnt)
{
    const int n = *go ? *rows : 0;
    AMG_ROWS(i, cap + 1) {
        int s = 0;
        if (i < n)
            for (int e = lia[i]; e < lia[i + 1]; ++e) s += ria[lja[e] + 1] - ria[lja[e]];
        cnt[i] = s;
    }
}
// key (row, column) = row << 32 | column of every entry, then `pad` (above every key) from the total up to the capacity `items`
__global__ void __launch_bounds__(256) k_amg_gemm_expand(const int* __restrict__ rows, const int* __restrict__ go, const int* __restrict__ lia,
    const int* __restrict__ lja, const int* __restrict__ ria, const int* __restrict__ rja, const int* __restrict__ off, const int* __restrict__ total,
    int items, unsigned long long pad, unsigned long long* __restrict__ key, int* __restrict__ pos, int* __restrict__ lidx, int* __restrict__ ridx)
{
    for (int p = *total + blockIdx.x * blockDim.x + threadIdx.x; p < items; p += gridDim.x * blockDim.x) key[p] = pad;
    AMG_ROWS(i, *go ? *rows : 0) {
        int p = off[i];
        for (int e = lia[i]; e < lia[i + 1]; ++e)
            for (int f = ria[lja[e]]; f < ria[lja[e] + 1]; ++f, ++p) {
                key[p] = (unsigned long long)i << 32 | (unsigned)rja[f];
                pos[p] = p;
                lidx[p] = e;
                ridx[p] = f;
            }
    }
}
// cia == NULL: distinct columns per row into cnt[0, cap] (0 from *rows on); otherwise the row's blocks, each the sum of its run in sorted
// (stable) order
__global__ void __launch_bounds__(256) k_amg_gemm_fill(const int* __restrict__ rows, const int* __restrict__ go, int cap, const int* __restrict__ off,
    const unsigned long long* __restrict__ skey, const int* __restrict__ spos, const int* __restrict__ lidx, const int* __restrict__ ridx, const double* __restrict__ lblk,
    const double* __restrict__ rblk, const int* __restrict__ cia, int* __restrict__ cnt, int* __restrict__ cja, double* __restrict__ cblk)
{
    const int n = *go ? *rows : 0;
    if (!cia) {
        AMG_ROWS(i, cap + 1) {
            int d = 0;
            if (i < n)
                for (int p = off[i]; p < off[i + 1]; ++p) d += p == off[i] || skey[p] != skey[p - 1];
            cnt[i] = d;
        }
        return;
    }
    AMG_ROWS(i, n) {
        const int p0 = off[i], p1 = off[i + 1];
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
                cja[out] = (int)(unsigned)skey[p];
#pragma unroll
                for (int q = 0; q < 9; ++q) cblk[9 * (size_t)out + q] = acc[q];
                ++out;
            }
        }
    }
}

// the rule of one size of the set-up (one thread), from a total a scan left in device memory:
//   kFitLevel0: the kept blocks of level 0;  kFitAgg: the aggregates -- none, or more than 4/5 of the rows, make the level the last (and a
//   pass limit reached fails the set-up), otherwise the damping omega;  kAmgQ*: a count the coarsening needs, recorded, and past `cap` it
//   ends the hierarchy at level l (cut_level).  kAmgQCoarse, the last, sizes level l + 1, or leaves level l the last (no P, omega 0).
__global__ void k_amg_fit(AmgDev* __restrict__ d, int l, int q, const int* __restrict__ total, long long cap, const IterState* __restrict__ st,
    double* __restrict__ bad_pivot)
{
    if (threadIdx.x) return;
    const int t = *total;
    if (q == kFitLevel0) {
        d->nnzb[0] = t;
        return;
    }
    if (q == kFitAgg) {
        if (!d->go[l]) return;
        if (st->amg_stuck) {
            d->fail = 1;
            d->go[l] = 0;
            *bad_pivot = 1.0;
        } else if (t == 0 || 5 * (long long)t > 4 * (long long)d->n[l]) d->go[l] = 0;
        else {
            d->na[l] = t;
            d->omega[l] = __ddiv_rn(4.0 / 3.0, d->rho_g[l]);
        }
        return;
    }
    d->need[l][q] = t;
    if (d->go[l] && t > cap) {
        d->go[l] = 0;
        if (d->cut_level < 0) d->cut_level = l;
    }
    if (q == kAmgQP && d->go[l]) d->np[l] = t;
    if (q == kAmgQCoarse) {
        if (d->go[l]) {
            d->n[l + 1] = d->na[l];
            d->nnzb[l + 1] = t;
        } else {
            d->np[l] = 0;
            d->omega[l] = 0.0;
        }
    }
}

// y_i = D_i^-1 sum_j A_ij b_j  (times s = 1 / sqrt(*sq) when sq != NULL, 1 otherwise); the partial of |y|^2 of every 256-row chunk.  start != 0:
// b_0 from splitmix64
__global__ void __launch_bounds__(256) k_amg_power(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, const double* __restrict__ dinv, const double* __restrict__ b, const double* __restrict__ sq, double* __restrict__ y,
    double* __restrict__ part, int start)
{
    const int n = dv->n[l];
    for (int ch = blockIdx.x; ch * (int)blockDim.x < n; ch += gridDim.x) {
        const int i = ch * blockDim.x + threadIdx.x;
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
        cta_sum(&yy, part + ch);
        __syncthreads(); // (cta_sum's shared words are written again by the next chunk)
    }
}
// *out = the sum of the level's chunk partials, in reduce_sum's order over as many partials as the level has chunks
__global__ void __launch_bounds__(1024) k_amg_norm(const AmgDev* __restrict__ dv, int l, const double* __restrict__ partials, double* __restrict__ out)
{
    __shared__ double sm[32];
    const int n = (dv->n[l] + 255) / 256;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
        v = warp_sum(v);
        if (threadIdx.x == 0) out[0] = v;
    }
}
// after the power steps of a built level (one thread): rho, the failure rule, the Chebyshev coefficients in the order of the mirror, each
// operation rounded as the host rounds it; then whether the level is coarsened (go): not the last of lmax levels, not coarse enough.  A level
// that would be coarsened but is the last of the reserved depth is a cut.
__global__ void k_amg_coef(AmgDev* __restrict__ d, int l, int lmax, const double* __restrict__ sq, const unsigned long long* __restrict__ absrow,
    const int* __restrict__ flags, double* __restrict__ bad_pivot)
{
    if (threadIdx.x || d->n[l] == 0) return;
    d->levels = l + 1;
    const double rho_g = __longlong_as_double((long long)*absrow);
    double rho = __dsqrt_rn(sq[kAmgPowerSteps - 1]);
    const bool fail = flags[1] || flags[2] || !isfinite(rho) || !(rho > 0.0) || !isfinite(rho_g);
    if (fail) { // (coefficients that make no NaN: the solve stops before its first iteration)
        rho = 1.0;
        d->fail = 1;
        *bad_pivot = 1.0;
    }
    d->rho[l] = rho;
    d->rho_g[l] = rho_g;
    const double hi = __dmul_rn(2.0, rho), lo = __ddiv_rn(hi, 120.0);
    const double theta = __dmul_rn(0.5, __dadd_rn(hi, lo)), delta = __dmul_rn(0.5, __dsub_rn(hi, lo)), sigma = __ddiv_rn(theta, delta);
    d->inv_theta[l] = __ddiv_rn(1.0, theta);
    double rho_prev = __ddiv_rn(1.0, sigma);
    for (int k = 1; k < kAmgDegree; ++k) {
        const double rho_k = __ddiv_rn(1.0, __dsub_rn(__dmul_rn(2.0, sigma), rho_prev));
        d->c[l][k][0] = __dmul_rn(rho_k, rho_prev);
        d->c[l][k][1] = __ddiv_rn(__dmul_rn(2.0, rho_k), delta);
        rho_prev = rho_k;
    }
    const bool deeper = !fail && l + 1 < kAmgMaxLevels && d->n[l] > d->coarse_enough;
    d->go[l] = deeper && l + 1 < lmax;
    if (deeper && l + 1 == lmax && d->cut_level < 0) {
        d->cut_level = l;
        d->cut_depth = 1;
    }
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

// first kernel of a Chebyshev application at level l: r = D^-1 (f - A x) (zero: x = 0, no product), d = r / theta.  cg_p != NULL (level 0
// in an iteration, zero): first the CG update x_s += alpha p, f -= alpha Ap (Ap in x's storage), alpha = scal[0] / (the n_dot SpMV partials)
__global__ void __launch_bounds__(256) k_amg_cheb_init(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, const double* __restrict__ dinv, double* __restrict__ f, double* __restrict__ x, double* __restrict__ r,
    double* __restrict__ d, int zero, const double* __restrict__ cg_p, double* __restrict__ cg_x, const double* __restrict__ scal,
    const double* __restrict__ dot, int n_dot)
{
    __shared__ double pAp;
    if (cg_p) {
        double s = 0.0;
        for (int k = threadIdx.x; k < n_dot; k += blockDim.x) s += dot[k];
        cta_sum(&s, &pAp);
        __syncthreads();
    }
    const double inv_theta = dv->inv_theta[l];
    AMG_ROWS(i, dv->n[l]) {
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
}

// step k of a Chebyshev application at level l: x += d ; r -= D^-1 A d ; d' = c1 d + c2 r ; last (k = 15): x += d' too.  part != NULL: the
// partials of f.x and f.f of every 256-row chunk (level 0's last kernel: r.z and r.r of the Krylov loop)
__global__ void __launch_bounds__(256) k_amg_cheb_step(const AmgDev* __restrict__ dv, int l, int k, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, const double* __restrict__ dinv, double* __restrict__ x, double* __restrict__ r, const double* __restrict__ d,
    double* __restrict__ dn, int last, const double* __restrict__ f, double* __restrict__ part)
{
    const int n = dv->n[l];
    const double c1 = dv->c[l][k][0], c2 = dv->c[l][k][1];
    for (int ch = blockIdx.x; ch * (int)blockDim.x < n; ch += gridDim.x) {
        const int i = ch * blockDim.x + threadIdx.x;
        double rz_rr[2] = { 0.0, 0.0 };
        if (i < n) {
            double q[3], u[3];
            amg_row_product(i, ia, ja, blk, d, q);
            amg_dinv(dinv, i, q, u);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const size_t kk = 3 * (size_t)i + c;
                const double dk = d[kk];
                const double rk = r[kk] - u[c];
                const double dnk = c1 * dk + c2 * rk;
                double xk = x[kk] + dk;
                if (last) xk += dnk;
                else {
                    r[kk] = rk;
                    dn[kk] = dnk;
                }
                x[kk] = xk;
                if (part) {
                    const double fk = f[kk];
                    rz_rr[0] += fk * xk;
                    rz_rr[1] += fk * fk;
                }
            }
        }
        if (part) {
            cta_sum<2>(rz_rr, part + 2 * ch);
            __syncthreads(); // (cta_sum's shared words are written again by the next chunk)
        }
    }
}

// t = f - A x at level l, when level l + 1 was built (its restriction reads t)
__global__ void __launch_bounds__(256) k_amg_residual(const AmgDev* __restrict__ dv, int l, const int* __restrict__ ia, const int* __restrict__ ja,
    const double* __restrict__ blk, const double* __restrict__ f, const double* __restrict__ x, double* __restrict__ t)
{
    AMG_ROWS(i, dv->n[l + 1] > 0 ? dv->n[l] : 0) {
        double q[3];
        amg_row_product(i, ia, ja, blk, x, q);
#pragma unroll
        for (int c = 0; c < 3; ++c) t[3 * (size_t)i + c] = f[3 * (size_t)i + c] - q[c];
    }
}
// over *rows rows when *coarse > 0 (the coarse level was built): y = M v (restriction with R), or y += M v (prolongation with P)
__global__ void __launch_bounds__(256) k_amg_transfer(const int* __restrict__ rows, const int* __restrict__ coarse, const int* __restrict__ ia,
    const int* __restrict__ ja, const double* __restrict__ blk, const double* __restrict__ v, double* __restrict__ y, int add)
{
    AMG_ROWS(i, *coarse > 0 ? *rows : 0) {
        double q[3];
        amg_row_product(i, ia, ja, blk, v, q);
#pragma unroll
        for (int c = 0; c < 3; ++c) y[3 * (size_t)i + c] = add ? y[3 * (size_t)i + c] + q[c] : q[c];
    }
}

} // namespace ipcgpu

using namespace ipcgpu;

// CTAs of a launch over `rows` rows: level 0 takes one thread per row as the Krylov loop's partials do, a coarse level at most kAmgGridMax
static int amg_grid(long long rows) { return std::max(1, std::min(nblk(rows, 256), kAmgGridMax)); }
static int amg_level_grid(const ipcgpu_ctx* ctx, int l) { return l == 0 ? nblk(ctx->nV, 256) : amg_grid(ctx->amg.lv[l].cap_n); }

// full-row entries of the pattern (solver_full_pattern's count), / 9: the blocks level 0 can hold
static long long amg_level0_blocks(const ipcgpu_ctx* ctx)
{
    const long long nf = ctx->device_pattern ? 2 * (long long)ctx->pw.nnz_cap - ctx->n_rows : 2 * (long long)ctx->nnz - ctx->n_rows;
    return (nf + 8) / 9;
}

// the device words and the per-level scalars' scratch, allocated once (coarse_enough at its default)
static int amg_alloc_dev(ipcgpu_ctx* ctx)
{
    AmgWork& w = ctx->amg;
    if (w.dev.n) return IPCGPU_OK;
    REQUIRE(w.dev.reserve(1) && w.flags.reserve(4) && w.absrow.reserve(1) && w.sq.reserve(kAmgPowerSteps), IPCGPU_ERR_CUDA, "AMG allocation failed");
    w.h = AmgDev{};
    w.h.coarse_enough = kAmgCoarseEnough;
    w.h.cut_level = -1;
    CK(cudaMemcpyAsync(w.dev.p, &w.h, sizeof(AmgDev), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// the buffers of level l for n rows (vectors, D^-1, P's row starts) and the set-up's row-sized scratch
static bool amg_level_buffers(AmgWork& w, int l, long long n)
{
    AmgLevel& L = w.lv[l];
    const size_t n1 = std::max<long long>(n, 1), n3 = 3 * n1;
    bool ok = L.ia.reserve(n1 + 1) && L.dinv.reserve(9 * n1) && L.r.reserve(n3) && L.d0.reserve(n3) && L.d1.reserve(n3) && L.t.reserve(n3) && L.agg.reserve(n1)
        && L.pia.reserve(n1 + 1) && w.state0.reserve(n1) && w.state1.reserve(n1) && w.m1.reserve(n1) && w.m2.reserve(n1) && w.cnt.reserve(n1 + 1)
        && w.scan_out.reserve(n1 + 1) && w.api.reserve(n1 + 1) && w.part.reserve(nblk(n1, 256));
    if (l > 0) ok = ok && L.f.reserve(n3) && L.x.reserve(n3);
    L.cap_n = n;
    return ok;
}
// the buffers of quantity q of level l's coarsening for c entries (R's row starts need level l + 1's rows first)
static bool amg_q_buffers(AmgWork& w, int l, int q, long long c)
{
    AmgLevel& L = w.lv[l];
    const size_t m = std::max<long long>(c, 1);
    L.cap[q] = c;
    switch (q) {
    case kAmgQP:
        return L.pja.reserve(m) && L.pblk.reserve(9 * m) && w.prow.reserve(m) && L.rja.reserve(m) && L.rblk.reserve(9 * m) && w.tkey.reserve(m)
            && w.tkey_sorted.reserve(m) && w.pos.reserve(m) && w.spos.reserve(m) && L.ria.reserve((size_t)w.lv[l + 1].cap_n + 1);
    case kAmgQApExp:
    case kAmgQRapExp:
        return w.key.reserve(m) && w.pos.reserve(m) && w.lidx.reserve(m) && w.ridx.reserve(m) && w.skey.reserve(m) && w.spos.reserve(m);
    case kAmgQAp: return w.apj.reserve(m) && w.apb.reserve(9 * m);
    default: w.lv[l + 1].cap_nnzb = c; return w.lv[l + 1].ja.reserve(m) && w.lv[l + 1].blk.reserve(9 * m);
    }
}
// the radix bits of R's keys (column * rows + row) for n rows and nc columns
static int amg_tbits(long long n, long long nc)
{
    int bits = 1;
    while (bits < 64 && ((unsigned long long)nc * (unsigned long long)n) >> bits) ++bits;
    return bits;
}
// the radix bits of a product's keys (row << 32 | column) for rows rows
static int amg_gemm_bits(long long rows) { return 32 + amg_tbits(rows, 1); }
// cub scratch of the sort of product q of level l's coarsening at its reserved size (rows rows)
static int amg_sort_bytes(ipcgpu_ctx* ctx, int q, int l, long long rows, size_t* bytes)
{
    const int items = (int)std::max<long long>(ctx->amg.lv[l].cap[q], 1);
    size_t s = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, s, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, items, 0,
        amg_gemm_bits(rows), ctx->stream));
    *bytes = std::max(*bytes, s);
    return IPCGPU_OK;
}

// exclusive scan of cnt[0, m] into out[0, m] (the count kernels leave cnt[m] = 0).  total != NULL (unreserved): the total, read back
static int amg_scan(ipcgpu_ctx* ctx, int* cnt, int* out, long long m, long long* total)
{
    AmgWork& w = ctx->amg;
    cudaStream_t st = ctx->stream;
    size_t bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt, out, (int)m + 1, st));
    REQUIRE(w.reserved ? w.tmp.n >= bytes : w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG scan workspace allocation failed");
    CK(cub::DeviceScan::ExclusiveSum(w.tmp.p, bytes, cnt, out, (int)m + 1, st));
    ++ctx->launches;
    if (total) {
        int t = 0;
        CK(cudaMemcpyAsync(&t, out + m, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        *total = t;
    }
    return IPCGPU_OK;
}

static int amg_read_word(ipcgpu_ctx* ctx, const int* word, int* out)
{
    CK(cudaMemcpyAsync(out, word, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// C = Lm Rm (step 5) of level l's coarsening: *rows rows of Lm (at most cap_rows), counts q_exp (the expansion) and q_out (C's blocks).
// Unreserved, C's arrays are grown here
static int amg_gemm(ipcgpu_ctx* ctx, int l, const int* rows, long long cap_rows, const int* lia, const int* lja, const double* lblk, const int* ria, const int* rja,
    const double* rblk, int q_exp, int* cia, DevBuf<int>& cja, DevBuf<double>& cblk, int q_out, double* bad_pivot)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    AmgDev* d = w.dev.p;
    cudaStream_t st = ctx->stream;
    const bool res = w.reserved > 0;
    const int g = amg_grid(cap_rows + 1), cr = (int)cap_rows;
    const int* go = &d->go[l];
    k_amg_gemm_count<<<g, 256, 0, st>>>(rows, go, cr, lia, lja, ria, w.cnt.p);
    ++ctx->launches;
    long long T = 0;
    int rc = amg_scan(ctx, w.cnt.p, w.scan_out.p, cap_rows, res ? nullptr : &T);
    if (rc) return rc;
    if (!res) {
        REQUIRE(T < INT_MAX, IPCGPU_ERR_CUDA, "AMG product: too many entries for an int index");
        REQUIRE(amg_q_buffers(w, l, q_exp, T), IPCGPU_ERR_CUDA, "AMG product allocation failed");
    }
    k_amg_fit<<<1, 32, 0, st>>>(d, l, q_exp, w.scan_out.p + cap_rows, L.cap[q_exp], ctx->iter.p, bad_pivot);
    // the enumeration in (row, column) order, stable: within a row the order of a stable sort by column (padding keys last)
    const int items = (int)std::max<long long>(L.cap[q_exp], 1), bits = amg_gemm_bits(cap_rows);
    const unsigned long long pad = bits == 64 ? ~0ull : (1ull << bits) - 1;
    k_amg_gemm_expand<<<g, 256, 0, st>>>(rows, go, lia, lja, ria, rja, w.scan_out.p, w.scan_out.p + cap_rows, items, pad, w.key.p, w.pos.p, w.lidx.p,
        w.ridx.p);
    size_t bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, w.key.p, w.skey.p, w.pos.p, w.spos.p, items, 0, bits, st));
    REQUIRE(res ? w.tmp.n >= bytes : w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG sort workspace allocation failed");
    CK(cub::DeviceRadixSort::SortPairs(w.tmp.p, bytes, w.key.p, w.skey.p, w.pos.p, w.spos.p, items, 0, bits, st));
    k_amg_gemm_fill<<<g, 256, 0, st>>>(rows, go, cr, w.scan_out.p, w.skey.p, w.spos.p, w.lidx.p, w.ridx.p, lblk, rblk, nullptr, w.cnt.p, nullptr, nullptr);
    ctx->launches += 4;
    long long nnz = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, cia, cap_rows, res ? nullptr : &nnz))) return rc;
    if (!res) REQUIRE(amg_q_buffers(w, l, q_out, nnz), IPCGPU_ERR_CUDA, "AMG level allocation failed");
    k_amg_fit<<<1, 32, 0, st>>>(d, l, q_out, cia + cap_rows, L.cap[q_out], ctx->iter.p, bad_pivot);
    k_amg_gemm_fill<<<g, 256, 0, st>>>(rows, go, cr, w.scan_out.p, w.skey.p, w.spos.p, w.lidx.p, w.ridx.p, lblk, rblk, cia, nullptr, cja.p, cblk.p);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// D^-1, the Gershgorin bound, rho, the Chebyshev coefficients of level l and whether it is coarsened (a level not built: nothing runs)
static int amg_level_setup(ipcgpu_ctx* ctx, int l, int lmax, double* bad_pivot)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    AmgDev* d = w.dev.p;
    cudaStream_t st = ctx->stream;
    const int g = amg_level_grid(ctx, l);
    CK(cudaMemsetAsync(w.absrow.p, 0, sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(w.flags.p + 2, 0, sizeof(int), st));
    k_amg_diag<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, w.absrow.p, w.state0.p, w.flags.p);
    // power iteration (step 7): y_k = D^-1 A (y_{k-1} / |y_{k-1}|), |y_k|^2 in sq[k-1]; rho = |y_100| (|b_99| = 1)
    double* y[2] = { L.d0.p, L.d1.p };
    for (int k = 0; k < kAmgPowerSteps; ++k) {
        k_amg_power<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, k ? y[(k - 1) & 1] : nullptr, k ? w.sq.p + k - 1 : nullptr, y[k & 1], w.part.p, k == 0);
        k_amg_norm<<<1, 1024, 0, st>>>(d, l, w.part.p, w.sq.p + k);
    }
    k_amg_coef<<<1, 32, 0, st>>>(d, l, lmax, w.sq.p, w.absrow.p, w.flags.p, bad_pivot);
    ctx->launches += 2 + 2 * kAmgPowerSteps;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// aggregation, P, R and A_{l+1} = R (A P) of level l (steps 2-5).  Unreserved: *stop when level l is the last (read back)
static int amg_coarsen(ipcgpu_ctx* ctx, int l, double* bad_pivot, bool* stop)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    AmgLevel& C = w.lv[l + 1];
    AmgDev* d = w.dev.p;
    IterState* it = ctx->iter.p;
    cudaStream_t st = ctx->stream;
    const bool res = w.reserved > 0;
    const long long capn = L.cap_n;
    const int g = amg_level_grid(ctx, l), gc = amg_grid(capn + 1);
    // step 3: passes of two rounds each (a round after the last changes nothing) as a WHILE of kAmgRound, states back in state0
    unsigned char *s0 = w.state0.p, *s1 = w.state1.p;
    k_amg_agg_begin<<<1, 32, 0, st>>>(d, l, it);
    ++ctx->launches;
    int rc = cond_node(ctx, true, kAmgRound, 0.0, 0, [&]() {
        cudaStream_t s = ctx->stream; // (the body's stream inside a capture)
        k_amg_mis_max<<<g, 256, 0, s>>>(d, l, L.ia.p, L.ja.p, nullptr, s0, w.m1.p);
        k_amg_mis_max<<<g, 256, 0, s>>>(d, l, L.ia.p, L.ja.p, w.m1.p, s0, w.m2.p);
        k_amg_mis_update<<<g, 256, 0, s>>>(d, l, w.m2.p, s0, s1, nullptr);
        k_amg_mis_max<<<g, 256, 0, s>>>(d, l, L.ia.p, L.ja.p, nullptr, s1, w.m1.p);
        k_amg_mis_max<<<g, 256, 0, s>>>(d, l, L.ia.p, L.ja.p, w.m1.p, s1, w.m2.p);
        k_amg_mis_update<<<g, 256, 0, s>>>(d, l, w.m2.p, s1, s0, &ctx->iter.p->amg_undecided);
        ctx->launches += 6;
        CK(cudaGetLastError());
        return IPCGPU_OK;
    });
    if (rc) return rc;
    k_amg_roots<<<gc, 256, 0, st>>>(d, l, (int)capn, s0, w.cnt.p);
    ++ctx->launches;
    long long na = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, w.scan_out.p, capn, res ? nullptr : &na))) return rc;
    k_amg_fit<<<1, 32, 0, st>>>(d, l, kFitAgg, w.scan_out.p + capn, 0, it, bad_pivot);
    ++ctx->launches;
    if (!res) {
        int go = 0;
        if ((rc = amg_read_word(ctx, &d->go[l], &go))) return rc;
        *stop = !go;
        if (!go) return IPCGPU_OK;
        REQUIRE(amg_level_buffers(w, l + 1, na), IPCGPU_ERR_CUDA, "AMG level allocation failed");
    }
    k_amg_assign1<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, s0, w.scan_out.p, w.m1.p);
    k_amg_assign2<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, w.m1.p, L.agg.p);
    k_amg_prolongator<<<gc, 256, 0, st>>>(d, l, (int)capn, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, L.agg.p, nullptr, w.cnt.p, nullptr, nullptr, nullptr);
    ctx->launches += 3;
    long long np = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, L.pia.p, capn, res ? nullptr : &np))) return rc;
    if (!res) REQUIRE(amg_q_buffers(w, l, kAmgQP, np), IPCGPU_ERR_CUDA, "AMG prolongator allocation failed");
    k_amg_fit<<<1, 32, 0, st>>>(d, l, kAmgQP, L.pia.p + capn, L.cap[kAmgQP], it, bad_pivot);
    k_amg_prolongator<<<g, 256, 0, st>>>(d, l, (int)capn, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, L.agg.p, L.pia.p, nullptr, L.pja.p, L.pblk.p, w.prow.p);
    // R = P^T: sort (column, row) over the capacity (padding keys last), then rows of R = runs of equal column
    const int capp = (int)std::max<long long>(L.cap[kAmgQP], 1), bits = amg_tbits(capn, C.cap_n);
    const unsigned long long pad = bits == 64 ? ~0ull : (1ull << bits) - 1;
    k_amg_tkeys<<<amg_grid(capp), 256, 0, st>>>(d, l, capp, pad, L.pja.p, w.prow.p, w.tkey.p, w.pos.p);
    size_t bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, w.tkey.p, w.tkey_sorted.p, w.pos.p, w.spos.p, capp, 0, bits, st));
    REQUIRE(res ? w.tmp.n >= bytes : w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG sort workspace allocation failed");
    CK(cub::DeviceRadixSort::SortPairs(w.tmp.p, bytes, w.tkey.p, w.tkey_sorted.p, w.pos.p, w.spos.p, capp, 0, bits, st));
    k_amg_tfill<<<amg_grid(capp), 256, 0, st>>>(d, l, w.tkey_sorted.p, w.spos.p, L.pblk.p, L.ria.p, L.rja.p, L.rblk.p);
    ctx->launches += 5;
    CK(cudaGetLastError());
    // A_{l+1} = R (A_l P)
    if ((rc = amg_gemm(ctx, l, &d->n[l], capn, L.ia.p, L.ja.p, L.blk.p, L.pia.p, L.pja.p, L.pblk.p, kAmgQApExp, w.api.p, w.apj, w.apb, kAmgQAp, bad_pivot)))
        return rc;
    return amg_gemm(ctx, l, &d->na[l], C.cap_n, L.ria.p, L.rja.p, L.rblk.p, w.api.p, w.apj.p, w.apb.p, kAmgQRapExp, C.ia.p, C.ja, C.blk, kAmgQCoarse, bad_pivot);
}

// a reservation holds while the mesh and the pattern it was sized for do; otherwise it is dropped (the set-up grows again)
bool solver_amg_reserved(ipcgpu_ctx* ctx)
{
    AmgWork& w = ctx->amg;
    if (w.reserved && (w.res_nV != ctx->nV || w.lv[0].cap_nnzb < amg_level0_blocks(ctx))) w.reserved = 0;
    return w.reserved > 0;
}

// the hierarchy of the resident matrix (steps 1-8).  A pivot <= 0 or a non-finite spectral radius leaves 1.0 in *bad_pivot and ends the
// hierarchy at that level.  Unreserved: the totals are read back to grow the buffers and to end the loop.  Reserved: nothing is allocated
// or read back; the reserved depth of levels is enqueued and a level the set-up does not build (AmgDev::n = 0) does nothing
int solver_amg_build(ipcgpu_ctx* ctx, double* bad_pivot)
{
    AmgWork& w = ctx->amg;
    cudaStream_t st = ctx->stream;
    const bool res = solver_amg_reserved(ctx);
    const int nb = ctx->nV, lmax = res ? w.reserved : kAmgMaxLevels;
    int rc = amg_alloc_dev(ctx);
    if (rc) return rc;
    if (!res) REQUIRE(amg_level_buffers(w, 0, nb), IPCGPU_ERR_CUDA, "AMG allocation failed");
    AmgDev* d = w.dev.p;
    w.ran = true;
    AmgLevel& L0 = w.lv[0];
    CK(cudaMemsetAsync(w.flags.p, 0, 4 * sizeof(int), st));
    CK(cudaMemsetAsync(w.cnt.p + nb, 0, sizeof(int), st));
    k_amg_begin<<<1, 32, 0, st>>>(d, nb);
    k_amg_level0<<<nblk(nb, 256), 256, 0, st>>>(nb, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, nullptr, w.cnt.p, nullptr, nullptr, w.flags.p);
    ctx->launches += 2;
    long long nnzb = 0;
    if ((rc = amg_scan(ctx, w.cnt.p, L0.ia.p, nb, res ? nullptr : &nnzb))) return rc;
    if (!res) {
        int layout = 0;
        if ((rc = amg_read_word(ctx, w.flags.p + 1, &layout))) return rc;
        REQUIRE(!layout, IPCGPU_ERR_ARG, "ipcgpu_solve_pcg_amg: the pattern is not LinSysSolver::set_pattern's 3 x 3 block layout");
        REQUIRE(L0.ja.reserve(std::max<long long>(nnzb, 1)) && L0.blk.reserve(9 * (size_t)std::max<long long>(nnzb, 1)), IPCGPU_ERR_CUDA,
            "AMG level allocation failed");
        L0.cap_nnzb = nnzb;
    }
    k_amg_level0<<<nblk(nb, 256), 256, 0, st>>>(nb, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, L0.ia.p, nullptr, L0.ja.p, L0.blk.p, w.flags.p);
    k_amg_fit<<<1, 32, 0, st>>>(d, 0, kFitLevel0, L0.ia.p + nb, 0, ctx->iter.p, bad_pivot);
    ctx->launches += 2;
    w.levels = 0;
    for (int l = 0; l < lmax; ++l) {
        w.levels = l + 1;
        if ((rc = amg_level_setup(ctx, l, lmax, bad_pivot))) return rc;
        if (!res) {
            int go = 0;
            if ((rc = amg_read_word(ctx, &d->go[l], &go))) return rc;
            if (!go) break; // (a failed level: the solve stops before its first iteration)
        }
        if (l + 1 == lmax) break;
        bool stop = false;
        if ((rc = amg_coarsen(ctx, l, bad_pivot, &stop))) return rc;
        if (stop) break;
    }
    return IPCGPU_OK;
}

// ipcgpu_amg_reserve: every buffer for the reserved depth -- the built levels of the last set-up (one more after a depth cut), or more --
// at the row bounds (level 0:
// nV rows and the blocks of the full pattern; level l: 4/5 of level l - 1's rows, floored) and headroom x what the last set-up needed of
// each count of a coarsening (never less than an earlier reservation), and the cub scratch of every scan and sort at those sizes
int solver_amg_reserve(ipcgpu_ctx* ctx, double headroom)
{
    AmgWork& w = ctx->amg;
    int rc = solver_amg_read(ctx);
    if (rc) return rc;
    REQUIRE(w.h.levels > 0 && !w.h.fail, IPCGPU_ERR_STATE, "ipcgpu_amg_reserve: an eager ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    const bool again = solver_amg_reserved(ctx);
    // (a depth cut adds the level the set-up wanted; its counts are unknown until a set-up reaches it: the next one may cut there)
    const int lr = std::min(kAmgMaxLevels, std::max(again ? w.reserved : 0, w.h.levels) + w.h.cut_depth);
    long long capn = ctx->nV;
    for (int l = 0; l < lr; ++l, capn = capn * 4 / 5) REQUIRE(amg_level_buffers(w, l, capn), IPCGPU_ERR_CUDA, "AMG reservation failed");
    const long long b0 = amg_level0_blocks(ctx);
    REQUIRE(w.lv[0].ja.reserve(b0) && w.lv[0].blk.reserve(9 * (size_t)b0), IPCGPU_ERR_CUDA, "AMG reservation failed");
    w.lv[0].cap_nnzb = b0;
    size_t bytes = 0;
    for (int l = 0; l < lr; ++l) {
        AmgLevel& L = w.lv[l];
        size_t s = 0;
        CK(cub::DeviceScan::ExclusiveSum(nullptr, s, (int*)nullptr, (int*)nullptr, (int)L.cap_n + 1, ctx->stream));
        bytes = std::max(bytes, s);
        if (l + 1 == lr) continue;
        for (int q = 0; q < kAmgQty; ++q) {
            const double need = std::ceil(headroom * (double)w.h.need[l][q]);
            REQUIRE(need < (double)INT_MAX, IPCGPU_ERR_ARG, "ipcgpu_amg_reserve: headroom x a count of the set-up exceeds an int index");
            const long long c = std::max<long long>({ again ? L.cap[q] : 0, (long long)need, 1 });
            REQUIRE(amg_q_buffers(w, l, q, c), IPCGPU_ERR_CUDA, "AMG reservation failed");
        }
        const int capp = (int)L.cap[kAmgQP];
        CK(cub::DeviceRadixSort::SortPairs(nullptr, s, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, capp, 0,
            amg_tbits(L.cap_n, w.lv[l + 1].cap_n), ctx->stream));
        bytes = std::max(bytes, s);
        if ((rc = amg_sort_bytes(ctx, kAmgQApExp, l, L.cap_n, &bytes)) || (rc = amg_sort_bytes(ctx, kAmgQRapExp, l, w.lv[l + 1].cap_n, &bytes))) return rc;
    }
    REQUIRE(w.tmp.reserve(std::max<size_t>(bytes, 1)), IPCGPU_ERR_CUDA, "AMG reservation failed");
    w.reserved = lr;
    w.res_nV = ctx->nV;
    ++ctx->epoch; // graphs captured before this call are refused (the buffers change)
    return IPCGPU_OK;
}

// AmgDev into the host copy (synchronises)
int solver_amg_read(ipcgpu_ctx* ctx)
{
    AmgWork& w = ctx->amg;
    REQUIRE(w.ran, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    CK(cudaMemcpyAsync(&w.h, w.dev.p, sizeof(AmgDev), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int solver_amg_coarse_enough(ipcgpu_ctx* ctx, int rows)
{
    int rc = amg_alloc_dev(ctx);
    if (rc) return rc;
    CK(cudaMemcpyAsync(&ctx->amg.dev.p->coarse_enough, &rows, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// one Chebyshev application at level l on (f, x); zero: from x = 0; cg: level 0's first in an iteration (the CG update); part: level 0's last
static void amg_chebyshev(ipcgpu_ctx* ctx, int l, double* f, double* x, bool zero, bool cg, double* part)
{
    AmgLevel& L = ctx->amg.lv[l];
    const AmgDev* d = ctx->amg.dev.p;
    cudaStream_t st = ctx->stream;
    const int g = amg_level_grid(ctx, l);
    k_amg_cheb_init<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, f, x, L.r.p, L.d0.p, zero ? 1 : 0, cg ? ctx->pcg_p.p : nullptr,
        cg ? ctx->sol.p : nullptr, ctx->pcg_scal.p, ctx->pcg_part.p, kPcgSpmvBlocks);
    double* dd[2] = { L.d0.p, L.d1.p };
    for (int k = 1; k < kAmgDegree; ++k) {
        const bool last = k == kAmgDegree - 1;
        k_amg_cheb_step<<<g, 256, 0, st>>>(d, l, k, L.ia.p, L.ja.p, L.blk.p, L.dinv.p, x, L.r.p, dd[(k - 1) & 1], dd[k & 1], last ? 1 : 0, f,
            last ? part : nullptr);
    }
    ctx->launches += kAmgDegree;
}

// one visit of level l (W-cycle).  Level l + 1 not built at this set-up: its residual, restriction, visits and prolongation do nothing, and
// the two Chebyshev applications of level l are what the last level does
static void amg_cycle(ipcgpu_ctx* ctx, int l, double* f, double* x, bool zero, bool cg, double* part)
{
    AmgWork& w = ctx->amg;
    AmgLevel& L = w.lv[l];
    AmgDev* d = w.dev.p;
    cudaStream_t st = ctx->stream;
    if (l == w.levels - 1) {
        amg_chebyshev(ctx, l, f, x, zero, cg, nullptr);
        amg_chebyshev(ctx, l, f, x, false, false, part);
        return;
    }
    AmgLevel& C = w.lv[l + 1];
    const int g = amg_level_grid(ctx, l);
    amg_chebyshev(ctx, l, f, x, zero, cg, nullptr);
    k_amg_residual<<<g, 256, 0, st>>>(d, l, L.ia.p, L.ja.p, L.blk.p, f, x, L.t.p);
    k_amg_transfer<<<amg_level_grid(ctx, l + 1), 256, 0, st>>>(&d->n[l + 1], &d->n[l + 1], L.ria.p, L.rja.p, L.rblk.p, L.t.p, C.f.p, 0);
    ctx->launches += 2;
    for (int v = 0; v < kAmgCycles; ++v) amg_cycle(ctx, l + 1, C.f.p, C.x.p, v == 0, false, nullptr);
    k_amg_transfer<<<g, 256, 0, st>>>(&d->n[l], &d->n[l + 1], L.pia.p, L.pja.p, L.pblk.p, C.x.p, x, 1);
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
    size_t b = (w.cnt.n + w.scan_out.n + w.m1.n + w.m2.n + w.pos.n + w.lidx.n + w.ridx.n + w.spos.n + w.prow.n + w.api.n + w.apj.n + w.flags.n)
            * sizeof(int)
        + (w.key.n + w.skey.n + w.tkey.n + w.tkey_sorted.n + w.absrow.n) * 8 + w.state0.n + w.state1.n + w.tmp.n + (w.part.n + w.sq.n + w.apb.n) * sizeof(double)
        + w.dev.n * sizeof(AmgDev);
    for (const AmgLevel& L : w.lv)
        b += (L.ia.n + L.ja.n + L.agg.n + L.pia.n + L.pja.n + L.ria.n + L.rja.n) * sizeof(int)
            + (L.blk.n + L.dinv.n + L.pblk.n + L.rblk.n + L.f.n + L.x.n + L.r.n + L.d0.n + L.d1.n + L.t.n) * sizeof(double);
    return b;
}
