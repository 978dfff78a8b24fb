// solve.cu -- device-resident linear-solve hand-off (SURVEY 8(f) rank 1): the Hessian never leaves HBM.
//
// Reference being stood in for: LinSysSolver::{factorize, solve} (src/LinSysSolver/LinSysSolver.hpp:230-236) as used by
// Optimizer::computeSearchDir (src/TimeStepper/Optimizer.cpp:2324-2355), i.e. CHOLMODSolver.cpp:123-154.  The north star keeps the sparse
// Cholesky a black box (CHOLMOD / cuDSS); cuDSS is not in this image, so the production binding is documented in INTEGRATION.md
// (ipcgpu_device_ptr hands cuDSS the device-resident ia / ja / a) and what is BUILT here is the hand-off itself plus a reference solver
// that runs entirely on the device: a preconditioned conjugate gradient on the upper-triangular CSR the assembly stages fill, with the
// block-Jacobi preconditioner (here), the multilevel one (multilevel.cu) or smoothed-aggregation multigrid (amg.cu).  It takes its right-hand side from the device-resident gradient
// and leaves the search direction where the step-bound stages read it, so that a whole Newton iteration (assembly -> solve -> CCD) needs no
// host transfer of any vertex- or matrix-sized array.
//
// One Krylov loop (solver_pcg) for the three preconditioners: init, SpMV with per-CTA partials, the preconditioner's step, roll, direction.
// Every dot product is a fixed-order two-level sum (per-CTA partials, then one order for every launch), so two solves of one system give
// identical bits with any preconditioner: an adopted direction feeds the Armijo and step-bound decisions (DESIGN 3.13 / 3.17).
//
// SpMV on a symmetric matrix stored by its upper triangle: the device builds the FULL row structure once per pattern (col index + position
// of the value inside the upper-triangular array for every entry of both triangles), so the product is a plain deterministic row-parallel
// CSR SpMV that gathers a[] through that position map -- no atomics, no transposed pass.
//
// Full-row build (solver_full_pattern).  Row i of the full matrix is its transposed (lower) entries in ascending source row, then its own
// upper entries in storage order: the order every SpMV and the multilevel set-up sum a row in.  Five launches of sizes fixed by n_rows,
// gated on the device by IterState::pat_version against the version the structure was built for (sv_fp_version), so that a captured solve
// rebuilds it exactly when a replayed ipcgpu_update_pattern rewrote the pattern, and otherwise nothing:
//   k_fp_gate (one thread) -> k_fp_count (own lengths, +1 per transposed entry: integer atomics) -> exclusive scan into fp_start ->
//   k_fp_scatter (own entries at their place, transposed ones behind per-row cursors: in any order) -> k_fp_sort (each row's transposed
//   part sorted by source row -- distinct within a column, so the result does not depend on the order of the scatter's atomics -- and
//   fia = fp_start).  The scan runs ungated into scratch; fia, fja and fpos are written only by gated kernels.
#include "common.cuh"
#include "abi.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cub/cub.cuh>

namespace ipcgpu {

// block-Jacobi preconditioner: inverse of the 3x3 diagonal block of every vertex (row 3v: [d00 d01 d02], row 3v+1: [d11 d12], row 3v+2: [d22])
__global__ void __launch_bounds__(256) k_block_jacobi(int nV, const int* __restrict__ ia, int base, const double* __restrict__ a, double* __restrict__ Minv /* 6 per vertex */)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    const int o0 = ia[3 * v] - base, o1 = ia[3 * v + 1] - base, o2 = ia[3 * v + 2] - base;
    const double d00 = a[o0], d01 = a[o0 + 1], d02 = a[o0 + 2], d11 = a[o1], d12 = a[o1 + 1], d22 = a[o2];
    const double c00 = d11 * d22 - d12 * d12, c01 = d02 * d12 - d01 * d22, c02 = d01 * d12 - d02 * d11;
    const double det = d00 * c00 + d01 * c01 + d02 * c02;
    double* m = Minv + 6 * (size_t)v;
    if (!(fabs(det) > 0.0)) { // singular block (should not happen for an SPD matrix): fall back to the scalar diagonal
        m[0] = d00 != 0.0 ? 1.0 / d00 : 1.0; m[3] = d11 != 0.0 ? 1.0 / d11 : 1.0; m[5] = d22 != 0.0 ? 1.0 / d22 : 1.0;
        m[1] = m[2] = m[4] = 0.0;
        return;
    }
    const double id = 1.0 / det;
    m[0] = c00 * id; m[1] = c01 * id; m[2] = c02 * id;
    m[3] = (d00 * d22 - d02 * d02) * id; m[4] = (d01 * d02 - d00 * d12) * id;
    m[5] = (d00 * d11 - d01 * d01) * id;
}

// block-Jacobi step, one thread per vertex.  In an iteration (dot != NULL): x += alpha p, r -= alpha Ap with alpha = r.z / p.Ap, p.Ap the
// sum of the SpMV's n_dot partials, added by every CTA in the same order (so every CTA has the same alpha, with no launch of its own).
// Then z = Minv r in Ap's storage, and the partials of r.z and r.r.
__global__ void __launch_bounds__(256) k_block_jacobi_step(int nV, const double* __restrict__ Minv, const double* __restrict__ p, double* __restrict__ Ap_z,
    double* __restrict__ x, double* __restrict__ r, const double* __restrict__ scal, const double* __restrict__ dot, int n_dot, double* __restrict__ part)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    __shared__ double pAp;
    if (dot) {
        double s = 0.0;
        for (int i = threadIdx.x; i < n_dot; i += blockDim.x) s += dot[i];
        cta_sum(&s, &pAp);
        __syncthreads();
    }
    double rz_rr[2] = { 0.0, 0.0 };
    if (v < nV) {
        const double alpha = dot && pAp != 0.0 ? scal[0] / pAp : 0.0;
        double rv[3];
        for (int c = 0; c < 3; ++c) {
            const size_t i = 3 * (size_t)v + c;
            rv[c] = r[i];
            if (dot) {
                x[i] += alpha * p[i];
                rv[c] -= alpha * Ap_z[i];
                r[i] = rv[c];
            }
        }
        const double* m = Minv + 6 * (size_t)v;
        const double z0 = m[0] * rv[0] + m[1] * rv[1] + m[2] * rv[2], z1 = m[1] * rv[0] + m[3] * rv[1] + m[4] * rv[2], z2 = m[2] * rv[0] + m[4] * rv[1] + m[5] * rv[2];
        Ap_z[3 * (size_t)v] = z0; Ap_z[3 * (size_t)v + 1] = z1; Ap_z[3 * (size_t)v + 2] = z2;
        rz_rr[0] = rv[0] * z0 + rv[1] * z1 + rv[2] * z2;
        rz_rr[1] = rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2];
    }
    cta_sum<2>(rz_rr, part + 2 * blockIdx.x);
}

// ---- the Krylov loop of both solvers ----------------------------------------------------------------------------------------
// scal: [0] r.z, [1] p.Ap (multilevel), [3] |r|^2, [4] |b|^2, [5] beta, [6] a domain of the multilevel set-up had a non-positive pivot
// x = 0, p = 0, r = sign * src
__global__ void __launch_bounds__(256) k_pcg_init(int n, const double* __restrict__ src, double sign, double* __restrict__ x, double* __restrict__ r, double* __restrict__ p)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    x[i] = 0.0;
    p[i] = 0.0;
    r[i] = sign * src[i];
}

// y = A x over full rows (one warp per row, rows dealt to the warps of a fixed grid), partial of x.y per CTA
__global__ void __launch_bounds__(256) k_pcg_spmv(int n, const int* __restrict__ fia, const int* __restrict__ fja, const int* __restrict__ fpos, const double* __restrict__ a,
    const double* __restrict__ x, double* __restrict__ y, double* __restrict__ part)
{
    const int lane = threadIdx.x & 31;
    const int row0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    double acc = 0.0; // (lane 0's; the other lanes add +0.0)
    for (int row = row0; row < n; row += (gridDim.x * blockDim.x) >> 5) {
        double s = 0.0;
        for (int k = fia[row] + lane; k < fia[row + 1]; k += 32) s += __ldg(a + fpos[k]) * __ldg(x + fja[k]);
        s = warp_sum(s);
        if (lane == 0) {
            y[row] = s;
            acc += x[row] * s;
        }
    }
    cta_sum(&acc, part + blockIdx.x);
}

// after a preconditioner step: r.z and |r|^2 from its partials, beta = r.z / (the previous r.z) (0 at the start), |r|^2 and the count of
// the solve in flight (start: |b|^2 instead)
__global__ void __launch_bounds__(1024) k_pcg_roll(const double* __restrict__ part, int n_part, double* __restrict__ scal, IterState* __restrict__ st, int start)
{
    __shared__ double sm[2][32];
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n_part; i += blockDim.x) {
        s0 += part[2 * i];
        s1 += part[2 * i + 1];
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    if ((threadIdx.x & 31) == 0) {
        sm[0][threadIdx.x >> 5] = s0;
        sm[1][threadIdx.x >> 5] = s1;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        s0 = warp_sum(sm[0][threadIdx.x]);
        s1 = warp_sum(sm[1][threadIdx.x]);
        if (threadIdx.x == 0) {
            const double rz_old = scal[0];
            scal[5] = rz_old != 0.0 ? s0 / rz_old : 0.0;
            scal[0] = s0;
            scal[3] = s1;
            if (start) scal[4] = s1; // r = b
            else {
                st->sv_rr = s1;
                ++st->sv_iters;
            }
        }
    }
}

// p = z + beta p
__global__ void __launch_bounds__(256) k_pcg_direction(int n, const double* __restrict__ z, double* __restrict__ p, const double* __restrict__ scal)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double beta = scal[5];
    if (i < n) p[i] = z[i] + beta * p[i];
}

// out_i = (sign g_i) / a(i,i) on every row (LinSysSolver::precondition_diag, LinSysSolver.hpp:411-420): the diagonal is the first stored
// entry of its row, read as k_block_jacobi reads it, and the quotient is one correctly rounded division, as the reference's.  Rows of
// vertices flagged in dbc (nullable) or from v_fixed on are 0 (initX option 5, Optimizer.cpp:1096-1097).  st != NULL: a non-finite entry
// fails the result as a solve fails (step_control.cu: solve_fail)
__global__ void __launch_bounds__(256) k_precondition_diag(int n, const int* __restrict__ ia, int base, const double* __restrict__ a,
    const double* __restrict__ g, double sign, const uint8_t* __restrict__ dbc, int v_fixed, double* __restrict__ out, IterState* __restrict__ st)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int v = i / 3;
    const double r = (v >= v_fixed || (dbc && dbc[v])) ? 0.0 : (sign * g[i]) / a[ia[i] - base];
    out[i] = r;
    if (st && !isfinite(r)) {
        st->sv_status = IPCGPU_ERR_SOLVE;
        st->flags[FLAG_SOLVE] = 1;
    }
}

// max |x_i| (exact, so the order does not matter; NaN entries are skipped)
__global__ void __launch_bounds__(256) k_abs_max(int n, const double* __restrict__ x, unsigned long long* __restrict__ out)
{
    double m = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmax(m, fabs(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(out, dbl_to_ord(m)); // (non-negative doubles order like their bit patterns)
}

// ---- full-row structure -------------------------------------------------------------------------------------------------------
__global__ void k_fp_gate(IterState* st)
{
    if (threadIdx.x == 0) st->sv_fp_build = st->pat_version != st->sv_fp_version;
}
// cnt[i] += entries of full row i (cnt zeroed by k_fp_zero); the scatter cursors zeroed
__global__ void __launch_bounds__(256) k_fp_count(int n, const int* __restrict__ ia, const int* __restrict__ ja, int base, int* __restrict__ cnt,
    int* __restrict__ cur, const IterState* __restrict__ st)
{
    if (!st->sv_fp_build) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int k0 = ia[i] - base, k1 = ia[i + 1] - base;
        int own = 0;
        for (int k = k0; k < k1; ++k) {
            const int j = ja[k] - base;
            ++own;
            if (j != i) atomicAdd(cnt + j, 1);
        }
        atomicAdd(cnt + i, own);
        cur[i] = 0;
    }
}
__global__ void __launch_bounds__(256) k_fp_zero(int n, int* __restrict__ cnt, const IterState* __restrict__ st)
{
    if (!st->sv_fp_build) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += gridDim.x * blockDim.x) cnt[i] = 0;
}
__global__ void __launch_bounds__(256) k_fp_scatter(int n, const int* __restrict__ ia, const int* __restrict__ ja, int base, const int* __restrict__ start,
    const int* __restrict__ cnt, int* __restrict__ cur, int* __restrict__ fja, int* __restrict__ fpos, const IterState* __restrict__ st)
{
    if (!st->sv_fp_build) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int k0 = ia[i] - base, k1 = ia[i + 1] - base;
        const int own0 = start[i] + cnt[i] - (k1 - k0); // the row's own entries come after its transposed ones
        for (int k = k0; k < k1; ++k) {
            const int j = ja[k] - base;
            fja[own0 + k - k0] = j;
            fpos[own0 + k - k0] = k;
            if (j != i) {
                const int e = start[j] + atomicAdd(cur + j, 1);
                fja[e] = i;
                fpos[e] = k;
            }
        }
    }
}
// each row's transposed part by source row (insertion sort: a few dozen entries), fia = start; the version the structure now holds
__global__ void __launch_bounds__(256) k_fp_sort(int n, const int* __restrict__ start, const int* __restrict__ cur, int* __restrict__ fja, int* __restrict__ fpos,
    int* __restrict__ fia, IterState* __restrict__ st)
{
    if (!st->sv_fp_build) return;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    for (int i = t; i < n; i += gridDim.x * blockDim.x) {
        int* c = fja + start[i];
        int* q = fpos + start[i];
        const int m = cur[i];
        for (int a = 1; a < m; ++a) {
            const int cj = c[a], qa = q[a];
            int b = a - 1;
            while (b >= 0 && c[b] > cj) {
                c[b + 1] = c[b];
                q[b + 1] = q[b];
                --b;
            }
            c[b + 1] = cj;
            q[b + 1] = qa;
        }
        fia[i] = start[i];
    }
    if (t == 0) {
        fia[n] = start[n];
        st->sv_fp_version = st->pat_version;
    }
}
// mean |p| over the surface vertices (SpatialHash.hpp:603-612) for a direction that was produced on the device: fixed-order two-level sum
__global__ void __launch_bounds__(256) k_psize(int nSV, const int* __restrict__ SVI, int nVdof, const double* __restrict__ p, double* __restrict__ partials)
{
    double s = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nSV; i += gridDim.x * blockDim.x) {
        const int v = SVI[i];
        if (v >= nVdof) continue; // the obstacle's surface vertices do not count (SpatialHash::build sees the mesh alone)
        s += fabs(p[3 * (size_t)v]) + fabs(p[3 * (size_t)v + 1]) + fabs(p[3 * (size_t)v + 2]);
    }
    cta_sum(&s, partials + blockIdx.x);
}
// ... then the partials in block order, over the 3 nMeshSV components (0 without mesh surface vertices)
__global__ void k_psize_mean(const double* __restrict__ partials, int n, long long n3, double* __restrict__ out)
{
    if (threadIdx.x != 0) return;
    double s = 0.0;
    for (int b = 0; b < n; ++b) s += partials[b];
    *out = n3 > 0 ? s / (double)n3 : 0.0;
}

} // namespace ipcgpu

using namespace ipcgpu;

// fia / fja / fpos of the pattern in ia / ja, rebuilt on the device when IterState::pat_version differs from the version they hold.  Nothing
// synchronises.  fja / fpos hold 2 nnz entries of the host pattern, 2 nnz_capacity - n_rows of the device-built one (every row has its diagonal).
int solver_full_pattern(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->stream;
    const int n = ctx->n_rows, base = ctx->index_base;
    const size_t nf = ctx->device_pattern ? (size_t)(2 * ctx->pw.nnz_cap - n) : (size_t)2 * ctx->nnz;
    size_t scan_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, n + 1, st));
    const size_t n1 = (size_t)n + 1;
    // (sizes fixed within an epoch: inside a capture, after an eager solve of the same epoch, nothing is allocated here)
    bool ok = ctx->fia.reserve(n1) && ctx->fja.reserve(nf) && ctx->fpos.reserve(nf) && ctx->fp_start.reserve(n1) && ctx->fp_cur.reserve(n1)
        && ctx->fp_tmp.reserve(std::max<size_t>(scan_bytes, 1));
    if (ctx->fp_cnt.n < n1) { // (the ungated scan reads it: defined contents from the start)
        ok = ok && ctx->fp_cnt.reserve(n1);
        if (ok) CK(cudaMemsetAsync(ctx->fp_cnt.p, 0, n1 * sizeof(int), st));
    }
    REQUIRE(ok, IPCGPU_ERR_CUDA, "allocation of the full-row pattern failed");
    IterState* it = ctx->iter.p;
    const int grid = std::min(nblk(n1, 256), kSMs * 8);
    k_fp_gate<<<1, 32, 0, st>>>(it);
    k_fp_zero<<<grid, 256, 0, st>>>(n, ctx->fp_cnt.p, it);
    k_fp_count<<<grid, 256, 0, st>>>(n, ctx->ia.p, ctx->ja.p, base, ctx->fp_cnt.p, ctx->fp_cur.p, it);
    CK(cub::DeviceScan::ExclusiveSum(ctx->fp_tmp.p, scan_bytes, ctx->fp_cnt.p, ctx->fp_start.p, n + 1, st));
    k_fp_scatter<<<grid, 256, 0, st>>>(n, ctx->ia.p, ctx->ja.p, base, ctx->fp_start.p, ctx->fp_cnt.p, ctx->fp_cur.p, ctx->fja.p, ctx->fpos.p, it);
    k_fp_sort<<<grid, 256, 0, st>>>(n, ctx->fp_start.p, ctx->fp_cur.p, ctx->fja.p, ctx->fpos.p, ctx->fia.p, it);
    ctx->launches += 6; // (the scan counts as one)
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int solver_forget_full_pattern(ipcgpu_ctx* ctx)
{
    CK(cudaMemsetAsync(&ctx->iter.p->sv_fp_version, 0xff, sizeof(unsigned long long), ctx->stream));
    return IPCGPU_OK;
}

int solver_finish(ipcgpu_ctx* ctx)
{
    const int n = ctx->n_rows;
    k_abs_max<<<std::min(nblk(n, 256), kSMs * 4), 256, 0, ctx->stream>>>(n, ctx->sol.p, &ctx->iter.p->sv_xmax_ord);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// the diagonally preconditioned gradient into `out` (3 nV), one thread per row.  jacobi: initX option 5's predictor (0 on Dirichlet vertices
// and the obstacle tail; no status); otherwise the result ipcgpu_precondition_diag reports, whose status words kSolveStart has reset
void solver_precondition_diag(ipcgpu_ctx* ctx, double sign, double* out, bool jacobi)
{
    const int n = ctx->n_rows;
    k_precondition_diag<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, ctx->ia.p, ctx->index_base, ctx->a.p, ctx->g.p, sign,
        jacobi && ctx->has_dbc ? ctx->dbc.p : nullptr, jacobi ? ctx->nVdof : INT_MAX, out, jacobi ? nullptr : ctx->iter.p);
    ++ctx->launches;
}

// block-Jacobi step (start: z = Minv r alone)
static void block_jacobi_step(ipcgpu_ctx* ctx, bool start)
{
    double* part = ctx->pcg_part.p;
    k_block_jacobi_step<<<nblk(ctx->nV, 256), 256, 0, ctx->stream>>>(ctx->nV, ctx->pcg_minv.p, ctx->pcg_p.p, ctx->pcg_q.p, ctx->sol.p, ctx->pcg_r.p,
        ctx->pcg_scal.p, start ? nullptr : part, kPcgSpmvBlocks, part + kPcgSpmvBlocks);
    ++ctx->launches;
}

static void preconditioner_step(ipcgpu_ctx* ctx, int precond, bool start)
{
    if (precond == kPrecondAmg) solver_amg_step(ctx, start);
    else if (precond == kPrecondMultilevel) solver_multilevel_step(ctx, start);
    else block_jacobi_step(ctx, start);
}

// PCG on the device-resident matrix, preconditioned by block-Jacobi, the multilevel hierarchy (multilevel.cu) or smoothed-aggregation
// multigrid (amg.cu).  rhs_dev: device vector
// (3 nV) scaled by `sign`.  The solution is left in ctx->sol, the result in IterState (sv_*); a pivot <= 0 of the multilevel or AMG set-up is
// the solve's failure (kSolveStart).  The workspace is reserved by the caller (solve_pcg in api_mesh.cu).  pcg_part holds the SpMV's partials
// of p.Ap, then the preconditioner step's partials of r.z and r.r (2 per CTA of one thread per vertex).  The step is all the three solvers
// differ in: in an iteration it finishes the CG update from the SpMV's partials, then it leaves z = M^-1 r in pcg_q.
int solver_pcg(ipcgpu_ctx* ctx, const double* rhs_dev, double sign, double rel_tol, int max_iter, int precond)
{
    cudaStream_t st = ctx->stream;
    const int n = ctx->n_rows, n_pre = nblk(ctx->nV, 256);
    double *x = ctx->sol.p, *r = ctx->pcg_r.p, *p = ctx->pcg_p.p, *q = ctx->pcg_q.p, *scal = ctx->pcg_scal.p, *pre = ctx->pcg_part.p + kPcgSpmvBlocks;
    CK(cudaMemsetAsync(scal, 0, 8 * sizeof(double), st));
    if (precond != kPrecondJacobi) {
        int rc = precond == kPrecondAmg ? solver_amg_build(ctx, scal + 6) : solver_multilevel_build(ctx, scal + 6);
        if (rc) return rc;
    } else {
        k_block_jacobi<<<n_pre, 256, 0, st>>>(ctx->nV, ctx->ia.p, ctx->index_base, ctx->a.p, ctx->pcg_minv.p);
        ++ctx->launches;
    }
    k_pcg_init<<<nblk(n, 256), 256, 0, st>>>(n, rhs_dev, sign, x, r, p);
    preconditioner_step(ctx, precond, true);
    k_pcg_roll<<<1, 1024, 0, st>>>(pre, n_pre, scal, ctx->iter.p, 1);
    k_pcg_direction<<<nblk(n, 256), 256, 0, st>>>(n, q, p, scal);
    ctx->launches += 3;
    int rc = decide(ctx, kSolveStart, rel_tol, max_iter, 0, nullptr, scal);
    if (rc) return rc;
    return krylov_loops(ctx, max_iter, [&]() {
        cudaStream_t s = ctx->stream; // (the body's stream inside a capture)
        k_pcg_spmv<<<kPcgSpmvBlocks, 256, 0, s>>>(n, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, p, q, ctx->pcg_part.p);
        preconditioner_step(ctx, precond, false);
        k_pcg_roll<<<1, 1024, 0, s>>>(pre, n_pre, scal, ctx->iter.p, 0);
        k_pcg_direction<<<nblk(n, 256), 256, 0, s>>>(n, q, p, scal);
        ctx->launches += 3;
    });
}

// a direction produced on the device (src, or `dir` itself when src is NULL) becomes the search direction of the step-bound stages: pSize
// by a fixed-order device sum into pSize_dev.  Nothing synchronises, so a captured sequence may adopt a direction (the warm start's predictor).
int solver_adopt_direction(ipcgpu_ctx* ctx, const double* src)
{
    cudaStream_t st = ctx->stream;
    if (src) CK(cudaMemcpyAsync(ctx->dir.p, src, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, st));
    const int nb = ctx->nSV > 0 ? 64 : 0;
    REQUIRE(!ctx->capturing || (ctx->partials.n >= (size_t)nb + 8 && ctx->pSize_dev.n >= 1), IPCGPU_ERR_STATE,
        "adopt a search direction once outside a capture first (it sizes its workspace)");
    REQUIRE(ctx->partials.reserve(nb + 8) && ctx->pSize_dev.reserve(1), IPCGPU_ERR_CUDA, "search-direction workspace allocation failed");
    long long nMeshSV = 0;
    for (int v : ctx->h_SVI) nMeshSV += v < ctx->nVdof ? 1 : 0;
    if (nb) k_psize<<<nb, 256, 0, st>>>(ctx->nSV, ctx->SVI.p, ctx->nVdof, ctx->dir.p, ctx->partials.p);
    k_psize_mean<<<1, 32, 0, st>>>(ctx->partials.p, nb, nMeshSV * 3, ctx->pSize_dev.p);
    ctx->launches += nb ? 2 : 1;
    CK(cudaGetLastError());
    ctx->pSize_surface = ctx->surface_ready;
    ctx->dir_valid = true;
    return 0;
}
