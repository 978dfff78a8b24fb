// multilevel.cu -- conjugate gradients on the device-resident matrix, preconditioned by a multilevel additive Schwarz hierarchy (MAS: Wu,
// Wang, Wang, "A GPU-based multilevel additive Schwarz preconditioner for cloth and deformable body simulation", 2022) that is rebuilt from
// the matrix and the current positions at every solve.  This file holds the hierarchy and its step of solve.cu's Krylov loop (solver_pcg),
// which it shares with the block-Jacobi preconditioner: same recurrences, same contract (right-hand side from the resident gradient,
// solution left where the step-bound stages read it).
//
// Order.   Vertices (obstacle tail included) are sorted by a 30-bit Morton code of their current position: 10 bits per axis of the cube
//          that spans the largest extent of their bounding box (one cell size on every axis, so that a thin body is not cut into layers),
//          stable radix sort of (code, vertex id): ties keep ascending ids, the order is a pure function of the positions.  rank[v] is the
//          vertex's place.  Contacts couple vertices that are close in space, hence close in rank.
// Levels.  At level l the aggregates are the runs of 32^l consecutive ranks (level 0: the vertices) and the domains the runs of 32
//          consecutive aggregates; the levels end with the first that has one domain.  A_l[D] (96 x 96) is the sum of the 3 x 3 blocks H_ij
//          over the vertices i, j of domain D, added at (aggregate of i, aggregate of j): the Galerkin matrix of piecewise-constant
//          translations.  Vertices without degrees of freedom (Dirichlet vertices, the obstacle tail) belong to their level-0 domain only
//          and to no aggregate of the levels >= 1: their rows of H are identity rows, and with a zero right-hand side there the residual,
//          the direction and the solution stay exactly 0 on them, as with block-Jacobi -- an adopted search direction must not move them.
//          Aggregates without a free vertex (among them those the last domain does not have) are identity rows.
// Set-up.  One warp per row aggregate at level 0, per chunk of 32 ranks above it, walks its vertices in rank order and their full rows
//          (fia / fja / fpos, both triangles) in storage order; lane c owns column aggregate c and adds the entries that land there one by
//          one; at the levels >= 1 a second kernel adds the chunks of every aggregate in chunk order.  No floating-point atomics: the
//          matrices are bit-identical from call to call.  One CTA per domain then inverts its tile in shared memory by
//          unpivoted Gauss-Jordan elimination (its pivots are the squares of the Cholesky pivots of the tile: the same positivity test) and
//          stores the inverse dense and exactly symmetric.  A pivot <= 0 raises a word the solve reports as IPCGPU_ERR_SOLVE; the domain
//          then stores the identity, so nothing downstream is NaN.
// Apply.   z = sum_l P_l^T A_l^-1 P_l r.  One kernel per level, one CTA per domain: restrict (level 0 reads r through the order, level l
//          sums the 32 children of each aggregate from level l-1's restricted vector: a fixed shuffle tree), multiply by the stored inverse
//          (coalesced rows, warp reductions).  One kernel per vertex then adds the levels' contributions in level order and leaves the
//          per-CTA partials of r.z and r.r.
// Step.    In an iteration: p.Ap = k_reduce_sum of the SpMV's partials, then x += alpha p, r -= alpha Ap (k_ml_update); then the levels
//          and k_ml_prolong.  6 + L launches per iteration with the SpMV, roll and direction of solve.cu; set-up and step never
//          synchronise.
//
// Memory: the stored inverses (73,728 bytes per domain, 0.61 GB at 257 k vertices) and the level vectors stay allocated for the life of the
// context after the first call, like every workspace of the context.
//
// Follow-ups this layout leaves open: a block-CSR SpMV, and single-precision storage of the inverses (the 0.6 GB read per application at
// 257 k vertices).
#include "common.cuh"
#include "abi.h"
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cub/cub.cuh>

namespace ipcgpu {

constexpr int kAgg = 32;               // aggregates per domain, children per aggregate
constexpr int kTile = 3 * kAgg;        // rows of a domain matrix
constexpr int kTile2 = kTile * kTile;
constexpr int kBoxBlocks = 64;
constexpr size_t kInvertSmem = (size_t)(kTile2 + 2 * kTile) * sizeof(double);

struct MlLevels {
    int n;
    long long off[kMultilevelMax]; // first entry of level l in the restricted / coarse-solved vectors (96 per domain)
};

// ---- order ------------------------------------------------------------------------------------------------------------------
// per-CTA bounding box of the positions (SoA), 6 doubles per CTA: min x y z, max x y z
__global__ void __launch_bounds__(256) k_ml_bbox(int nV, const double* __restrict__ V, double* __restrict__ box)
{
    double b[6] = { DBL_MAX, DBL_MAX, DBL_MAX, DBL_MAX, DBL_MAX, DBL_MAX }; // (maxima negated: one min-reduction for all six)
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nV; v += gridDim.x * blockDim.x)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double x = V[(size_t)c * nV + v];
            b[c] = fmin(b[c], x);
            b[3 + c] = fmin(b[3 + c], -x);
        }
    __shared__ double sm[8][6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const double m = warp_min(b[c]);
        if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5][c] = m;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        double m = sm[0][threadIdx.x];
        for (int w = 1; w < 8; ++w) m = fmin(m, sm[w][threadIdx.x]);
        box[6 * blockIdx.x + threadIdx.x] = threadIdx.x < 3 ? m : -m;
    }
}

DEV unsigned spread3(unsigned x) // 10 bits -> every third bit
{
    x = (x | (x << 16)) & 0x030000FFu;
    x = (x | (x << 8)) & 0x0300F00Fu;
    x = (x | (x << 4)) & 0x030C30C3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

__global__ void __launch_bounds__(256) k_ml_morton(int nV, const double* __restrict__ V, const double* __restrict__ box, unsigned* __restrict__ code, int* __restrict__ id)
{
    __shared__ double b[6];
    if (threadIdx.x < 6) {
        double m = box[threadIdx.x];
        for (int k = 1; k < kBoxBlocks; ++k) m = threadIdx.x < 3 ? fmin(m, box[6 * k + threadIdx.x]) : fmax(m, box[6 * k + threadIdx.x]);
        b[threadIdx.x] = m;
    }
    __syncthreads();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    const double ext = fmax(fmax(b[3] - b[0], b[4] - b[1]), b[5] - b[2]);
    const double scale = ext > 0.0 ? 1024.0 / ext : 0.0;
    unsigned q[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) q[c] = (unsigned)min(1023, (int)((V[(size_t)c * nV + v] - b[c]) * scale));
    code[v] = spread3(q[0]) | (spread3(q[1]) << 1) | (spread3(q[2]) << 2);
    id[v] = v;
}

// rank, and the mask of the vertices without degrees of freedom: Dirichlet vertices and the obstacle tail
__global__ void __launch_bounds__(256) k_ml_rank(int nV, const int* __restrict__ order, int* __restrict__ rank, const uint8_t* __restrict__ dbc, int nVdof,
    unsigned char* __restrict__ fixed)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nV) return;
    rank[order[k]] = k;
    fixed[k] = (dbc && dbc[k]) || k >= nVdof;
}

// ---- level matrices ---------------------------------------------------------------------------------------------------------
// Level `shift / 5`.  One warp per chunk of 2^cshift consecutive ranks of one row aggregate; lane c accumulates the 3 x 3 block at column
// aggregate c.  Level 0 (cshift = 0, part == NULL): a chunk is the aggregate, the rows go straight into the tile (identity rows past the
// last vertex).  Levels >= 1 (cshift = 5): an aggregate has 32^(l-1) chunks, so that the walk over its 32^l vertices is spread over as many
// warps; the chunk's share is left in part ([chunk][9][lane]) for k_ml_gather.  `fixed` (levels >= 1, NULL at level 0): rows and columns
// of these vertices are left out.
__global__ void __launch_bounds__(128, 2) k_ml_assemble(int nV, int shift, int cshift, long long n_warps, const int* __restrict__ order, const int* __restrict__ rank,
    const int* __restrict__ fia, const int* __restrict__ fja, const int* __restrict__ fpos, const double* __restrict__ a, const unsigned char* __restrict__ fixed, double* __restrict__ A, double* __restrict__ part)
{
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; // chunk
    if (w >= n_warps) return;
    const long long agg = w >> (shift - cshift), D = agg >> 5; // row aggregate (padding included), domain
    const int ra = (int)(agg & 31);
    const long long k0 = w << cshift, k1 = min((long long)nV, (w + 1) << cshift);
    double acc[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int d = 0; d < 3; ++d) acc[c][d] = (k0 >= nV && lane == ra && c == d) ? 1.0 : 0.0; // an aggregate without vertices: identity rows
    // one full row of the matrix: the chunk's entries of this domain in storage order, each added by the lane that owns its column aggregate
    auto add_row = [&](int row, double& a0, double& a1, double& a2) {
        const int end = fia[row + 1];
        for (int base = fia[row]; base < end; base += 32) {
            const int e = base + lane;
            int tgt = -1, comp = 0;
            double val = 0.0;
            if (e < end) {
                const int j = fja[e];
                const long long aj = ((long long)rank[j / 3] >> shift) - (D << 5);
                if (aj >= 0 && aj < kAgg && !(fixed && fixed[j / 3])) {
                    tgt = (int)aj;
                    comp = j % 3;
                    val = a[fpos[e]];
                }
            }
            unsigned m = __ballot_sync(0xffffffffu, tgt >= 0);
            while (m) {
                const int s = __ffs(m) - 1;
                m &= m - 1;
                const int t = __shfl_sync(0xffffffffu, tgt, s), d = __shfl_sync(0xffffffffu, comp, s);
                const double x = __shfl_sync(0xffffffffu, val, s);
                if (t == lane) {
                    if (d == 0) a0 += x;
                    else if (d == 1) a1 += x;
                    else a2 += x;
                }
            }
        }
    };
    for (long long k = k0; k < k1; ++k) {
        const int v = order[k];
        if (fixed && fixed[v]) continue; // (levels >= 1: a vertex without degrees of freedom is in no aggregate)
        add_row(3 * v, acc[0][0], acc[0][1], acc[0][2]);
        add_row(3 * v + 1, acc[1][0], acc[1][1], acc[1][2]);
        add_row(3 * v + 2, acc[2][0], acc[2][1], acc[2][2]);
    }
    if (part) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int d = 0; d < 3; ++d) part[((size_t)w * 9 + 3 * c + d) * 32 + lane] = acc[c][d];
        return;
    }
    double* tile = A + (size_t)D * kTile2;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int d = 0; d < 3; ++d) tile[(3 * ra + c) * kTile + 3 * lane + d] = acc[c][d];
}

// levels >= 1: one warp per row aggregate (padding included) adds its chunks' shares in chunk order; `per` = chunks per aggregate.  An
// aggregate without a free vertex (padding, or Dirichlet / obstacle vertices only) has a zero diagonal -- a free vertex of a positive
// definite matrix makes it positive -- and becomes identity rows.
__global__ void __launch_bounds__(128) k_ml_gather(long long n_warps, long long n_chunks, long long per, const double* __restrict__ part, double* __restrict__ A)
{
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n_warps) return;
    const int ra = (int)(w & 31);
    const long long c0 = w * per, c1 = min(n_chunks, c0 + per);
    double acc[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) acc[e] = 0.0;
    for (long long c = c0; c < c1; ++c)
#pragma unroll
        for (int e = 0; e < 9; ++e) acc[e] += part[((size_t)c * 9 + e) * 32 + lane];
    if (lane == ra) {
        if (acc[0] == 0.0) acc[0] = 1.0;
        if (acc[4] == 0.0) acc[4] = 1.0;
        if (acc[8] == 0.0) acc[8] = 1.0;
    }
    double* tile = A + (size_t)(w >> 5) * kTile2;
#pragma unroll
    for (int e = 0; e < 9; ++e) tile[(3 * ra + e / 3) * kTile + 3 * lane + e % 3] = acc[e];
}

// one CTA per domain: the tile is replaced by its inverse (in-place Gauss-Jordan without pivoting; the k-th pivot is the k-th Schur
// complement of an SPD tile, positive exactly when Cholesky's is)
__global__ void __launch_bounds__(256) k_ml_invert(double* __restrict__ A, double* __restrict__ bad_pivot)
{
    extern __shared__ double sm[];
    double* T = sm;
    double* col = sm + kTile2;
    double* row = col + kTile;
    double* G = A + (size_t)blockIdx.x * kTile2;
    for (int e = threadIdx.x; e < kTile2; e += blockDim.x) T[e] = G[e];
    __syncthreads();
    bool ok = true;
    for (int k = 0; k < kTile; ++k) {
        const double p = T[k * kTile + k]; // (the same word for every thread: the branch is uniform)
        if (!(p > 0.0)) {
            ok = false;
            break;
        }
        if (threadIdx.x < kTile) {
            col[threadIdx.x] = T[threadIdx.x * kTile + k];
            row[threadIdx.x] = T[k * kTile + threadIdx.x];
        }
        __syncthreads();
        const double ip = 1.0 / p;
        for (int e = threadIdx.x; e < kTile2; e += blockDim.x) {
            const int i = e / kTile, j = e - i * kTile;
            double v;
            if (i == k) v = j == k ? ip : row[j] * ip;
            else if (j == k) v = -col[i] * ip;
            else v = T[e] - col[i] * (row[j] * ip);
            T[e] = v;
        }
        __syncthreads();
    }
    if (!ok && threadIdx.x == 0) *bad_pivot = 1.0;
    for (int e = threadIdx.x; e < kTile2; e += blockDim.x) {
        const int i = e / kTile, j = e - i * kTile;
        G[e] = ok ? (i <= j ? T[e] : T[j * kTile + i]) : (i == j ? 1.0 : 0.0);
    }
}

// ---- application ------------------------------------------------------------------------------------------------------------
// level `level`, one CTA per domain: R = P r (3 per aggregate, kept for the next level), Y = A^-1 R.  What level 0 keeps for level 1 is 0
// at the vertices without degrees of freedom: they are in no aggregate of the levels >= 1.
__global__ void __launch_bounds__(256) k_ml_level(int nV, int level, long long n_prev, const int* __restrict__ order, const unsigned char* __restrict__ fixed,
    const double* __restrict__ r, const double* __restrict__ Rprev, double* __restrict__ R, const double* __restrict__ inv, double* __restrict__ Y)
{
    __shared__ double x[kTile];
    const long long D = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (level == 0) {
        if (threadIdx.x < kTile) {
            const long long k = D * kAgg + threadIdx.x / 3;
            const int v = k < nV ? order[k] : -1;
            const double s = v >= 0 ? r[3 * (size_t)v + threadIdx.x % 3] : 0.0;
            x[threadIdx.x] = s;
            R[D * kTile + threadIdx.x] = v >= 0 && fixed[v] ? 0.0 : s;
        }
    } else {
        for (int ag = warp; ag < kAgg; ag += 8) {
            const long long child = (D * kAgg + ag) * kAgg + lane;
            double s[3] = { 0.0, 0.0, 0.0 };
            if (child < n_prev)
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] = Rprev[3 * child + c];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                s[c] = warp_sum(s[c]);
                if (lane == 0) {
                    x[3 * ag + c] = s[c];
                    R[D * kTile + 3 * ag + c] = s[c];
                }
            }
        }
    }
    __syncthreads();
    const double x0 = x[lane], x1 = x[lane + 32], x2 = x[lane + 64];
    for (int i = warp; i < kTile; i += 8) {
        const double* row = inv + ((size_t)D * kTile + i) * kTile;
        double s = row[lane] * x0 + row[lane + 32] * x1 + row[lane + 64] * x2;
        s = warp_sum(s);
        if (lane == 0) Y[D * kTile + i] = s;
    }
}

// z = sum over the levels, in level order, of the coarse solution of the vertex's aggregate (level 0 alone for a vertex without degrees of
// freedom); partials of r.z and r.r (2 per CTA)
__global__ void __launch_bounds__(256) k_ml_prolong(int nV, MlLevels lv, const int* __restrict__ rank, const unsigned char* __restrict__ fixed, const double* __restrict__ Y,
    const double* __restrict__ r,
    double* __restrict__ z, double* __restrict__ part)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    double rz_rr[2] = { 0.0, 0.0 };
    if (v < nV) {
        const long long rk = rank[v];
        const int n_lv = fixed[v] ? 1 : lv.n;
        double s[3] = { 0.0, 0.0, 0.0 };
#pragma unroll
        for (int l = 0; l < kMultilevelMax; ++l)
            if (l < n_lv) {
                const double* y = Y + lv.off[l] + 3 * (rk >> (5 * l));
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] += y[c];
            }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double rc = r[3 * (size_t)v + c];
            z[3 * (size_t)v + c] = s[c];
            rz_rr[0] += rc * s[c];
            rz_rr[1] += rc * rc;
        }
    }
    cta_sum<2>(rz_rr, part + 2 * blockIdx.x);
}

// the CG update of an iteration: x += alpha p ; r -= alpha Ap       with alpha = r.z / p.Ap (scal: solve.cu's layout)
__global__ void __launch_bounds__(256) k_ml_update(int n, const double* __restrict__ p, const double* __restrict__ Ap, double* __restrict__ x, double* __restrict__ r,
    const double* __restrict__ scal)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double pAp = scal[1];
    const double alpha = pAp != 0.0 ? scal[0] / pAp : 0.0;
    if (i >= n) return;
    x[i] += alpha * p[i];
    r[i] -= alpha * Ap[i];
}

} // namespace ipcgpu

using namespace ipcgpu;

// order and level matrices of the resident matrix at the current positions (the matrices where the inverses will be).  Nothing synchronises.
// The hierarchy counts as built (ipcgpu_multilevel_info, IPCGPU_BUF_MULTILEVEL_INVERSES) only once a solve has seen every pivot positive.
static int multilevel_matrices(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->stream;
    MultilevelWork& w = ctx->ml;
    const int nV = ctx->nV;
    w.built = false;
    w.levels = 0;
    size_t tiles = 0;
    for (long long span = kAgg;; span *= kAgg) {
        REQUIRE(w.levels < kMultilevelMax, IPCGPU_ERR_ARG, "too many vertices for the multilevel hierarchy");
        w.domains[w.levels] = (nV + span - 1) / span;
        w.tile_off[w.levels] = tiles;
        tiles += (size_t)w.domains[w.levels];
        if (w.domains[w.levels++] == 1) break;
    }
    w.tiles = tiles;
    size_t sort_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, nV, 0, 30, st));
    bool ok = w.box.reserve(6 * kBoxBlocks) && w.code.reserve(nV) && w.code_sorted.reserve(nV) && w.id.reserve(nV) && w.order.reserve(nV) && w.rank.reserve(nV)
        && w.fixed.reserve(nV) && w.sort_tmp.reserve(sort_bytes) && w.chunk.reserve((size_t)w.domains[0] * 9 * 32) && w.inv.reserve(tiles * kTile2) && w.R.reserve(tiles * kTile) && w.Y.reserve(tiles * kTile);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "allocation of the multilevel hierarchy failed");
    k_ml_bbox<<<kBoxBlocks, 256, 0, st>>>(nV, ctx->V.p, w.box.p);
    k_ml_morton<<<nblk(nV, 256), 256, 0, st>>>(nV, ctx->V.p, w.box.p, w.code.p, w.id.p);
    CK(cub::DeviceRadixSort::SortPairs(w.sort_tmp.p, sort_bytes, w.code.p, w.code_sorted.p, w.id.p, w.order.p, nV, 0, 30, st));
    k_ml_rank<<<nblk(nV, 256), 256, 0, st>>>(nV, w.order.p, w.rank.p, ctx->has_dbc ? ctx->dbc.p : nullptr, ctx->nVdof, w.fixed.p);
    const long long n_chunks = w.domains[0]; // chunks of 32 ranks
    for (int l = 0; l < w.levels; ++l) {
        const long long n_aggs = w.domains[l] * kAgg;
        double* tiles_l = w.inv.p + w.tile_off[l] * kTile2;
        if (l == 0) {
            k_ml_assemble<<<nblk(n_aggs * 32, 128), 128, 0, st>>>(nV, 0, 0, n_aggs, w.order.p, w.rank.p, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, nullptr, tiles_l,
                nullptr);
            continue;
        }
        k_ml_assemble<<<nblk(n_chunks * 32, 128), 128, 0, st>>>(nV, 5 * l, 5, n_chunks, w.order.p, w.rank.p, ctx->fia.p, ctx->fja.p, ctx->fpos.p, ctx->a.p, w.fixed.p,
            nullptr, w.chunk.p);
        long long per = 1;
        for (int k = 1; k < l; ++k) per *= kAgg;
        k_ml_gather<<<nblk(n_aggs * 32, 128), 128, 0, st>>>(n_aggs, n_chunks, per, w.chunk.p, tiles_l);
    }
    ctx->launches += 3 + 2 * w.levels; // (the sort counts as one)
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// ... and their inverses in place: the set-up of a multilevel solve; a pivot <= 0 leaves 1.0 in *bad_pivot
int solver_multilevel_build(ipcgpu_ctx* ctx, double* bad_pivot)
{
    MultilevelWork& w = ctx->ml;
    int rc = multilevel_matrices(ctx);
    if (rc) return rc;
    if (!w.smem_opted) {
        CK(cudaFuncSetAttribute(k_ml_invert, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kInvertSmem));
        w.smem_opted = true;
    }
    k_ml_invert<<<(unsigned)w.tiles, 256, kInvertSmem, ctx->stream>>>(w.inv.p, bad_pivot);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

// TEST HOOK behind ipcgpu_multilevel_debug_matrices: the level matrices as assembled, before any inversion
int solver_multilevel_matrices(ipcgpu_ctx* ctx, double* dst, uint64_t count)
{
    int rc = multilevel_matrices(ctx);
    if (rc) return rc;
    REQUIRE(dst && count == (uint64_t)ctx->ml.tiles * kTile2, IPCGPU_ERR_ARG, "level matrices: 96*96 doubles per domain of every level");
    CK(cudaMemcpyAsync(dst, ctx->ml.inv.p, count * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// the multilevel step of solver_pcg (solve.cu).  In an iteration: p.Ap = the sum of the SpMV's partials, then the CG update.  Then
// z = M^-1 r in pcg_q, and the partials of r.z and r.r behind the SpMV's.
void solver_multilevel_step(ipcgpu_ctx* ctx, bool start)
{
    cudaStream_t st = ctx->stream;
    MultilevelWork& w = ctx->ml;
    const double* r = ctx->pcg_r.p;
    double *z = ctx->pcg_q.p, *part = ctx->pcg_part.p;
    if (!start) {
        reduce_sum(part, kPcgSpmvBlocks, 1.0, ctx->pcg_scal.p + 1, st);
        k_ml_update<<<nblk(ctx->n_rows, 256), 256, 0, st>>>(ctx->n_rows, ctx->pcg_p.p, z, ctx->sol.p, ctx->pcg_r.p, ctx->pcg_scal.p);
        ctx->launches += 2;
    }
    MlLevels lv;
    lv.n = w.levels;
    for (int l = 0; l < w.levels; ++l) {
        lv.off[l] = (long long)w.tile_off[l] * kTile;
        k_ml_level<<<(unsigned)w.domains[l], 256, 0, st>>>(ctx->nV, l, l ? w.domains[l - 1] * kAgg : 0, w.order.p, w.fixed.p, r, l ? w.R.p + lv.off[l - 1] : nullptr, w.R.p + lv.off[l],
            w.inv.p + w.tile_off[l] * kTile2, w.Y.p + lv.off[l]);
    }
    k_ml_prolong<<<nblk(ctx->nV, 256), 256, 0, st>>>(ctx->nV, lv, w.rank.p, w.fixed.p, w.Y.p, r, z, part + kPcgSpmvBlocks);
    ctx->launches += w.levels + 1;
}
