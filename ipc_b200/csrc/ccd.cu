// ccd.cu -- CCD line-search step bound: swept broad phase + Tight-Inclusion narrow phase + device-wide min (sm_90a).
//   *** this translation unit is compiled with --fmad=false ***  (bit-exact step bound: every product/sum is rounded
//   exactly like the CPU oracle built with -ffp-contract=off; see __graft_entry__.py NOFMA_FILES)
//
// Reference being replaced:
//   SpatialHash<3>::build(mesh, searchDir, curMaxStepSize, voxelSize)          src/Utils/SpatialHash.hpp:589-750
//   SpatialHash queries  queryPointForPrimitives / queryEdgeForEdgesWithBBoxCheck  :752-773, :803-832
//   SelfCollisionHandler::largestFeasibleStepSize_TightInclusion (partial)      src/CollisionObject/SelfCollisionHandler.cpp:690-866
//   SelfCollisionHandler::largestFeasibleStepSize_CCD_TightInclusion (full)     :1370-1630
//   inclusion_ccd::vertexFaceCCD_double / edgeEdgeCCD_double (un-vendored Tight-Inclusion; restated from the published algorithm, see DESIGN.md)
//
// Structure
//   broad phase : a grid on the reference's own voxel lattice (voxel = avgEdgeLen/3, origin = swept bbox corner), cells of K x K x K
//                 voxels; every primitive is registered in each cell its voxel range touches, and a pair becomes a candidate iff the
//                 two ranges overlap -- i.e. exactly the pairs the reference's hash query returns -- plus its swept-AABB test for edge
//                 pairs.  Pairs are found inside one cell (the one holding the per-axis max of the two range starts) and go straight
//                 through the reference's candidate rules into the candidate list.
//   narrow, stage 1 (thread per candidate, HBM-bound: 8 B pair + 4 x 48 B gather): current distance, ms, and the ROOT box
//                 of the interval search; a candidate whose root box excludes the origin cannot collide and dies here.
//   narrow, stage 2 (warp per surviving pair, persistent CTAs + atomic work counter): level-synchronous breadth-first
//                 interval bisection.  The library's (level, t_lo) priority order is realised without sorting: per level,
//                 two warp min-reductions over the lexicographic key (t_lo,u_lo,v_lo) give the first box containing the
//                 origin and the first "terminal" box, which is all the sequential semantics depend on.
//   reduction   : atomicMin on the order-preserving uint64 image of the (non-negative) time of impact.
#include "broadphase.cuh"
#include "abi.h"
#include <cub/cub.cuh>

namespace ipcgpu {

// ------------------------------------------------------------------------------------------------------------------
// reference voxel ranges of every surface vertex on the swept grid (SpatialHash.hpp:642-662, :841-845)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ref_ranges(SurfArgs s, const double* __restrict__ dir, const IterState* __restrict__ st, int* __restrict__ vmin, int* __restrict__ vmax)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.nSV) return;
    const double alpha = st->alpha_grid, inv_h = st->ref_inv_h;
    const int v = s.SVI[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double x = s.V[(size_t)c * s.nV + v];
        const double xt = x + alpha * dir[3 * (size_t)v + c];
        const int a = (int)floor((x - st->ref_lo[c]) * inv_h), b = (int)floor((xt - st->ref_lo[c]) * inv_h);
        vmin[3 * (size_t)v + c] = min(a, b);
        vmax[3 * (size_t)v + c] = max(a, b);
    }
}

// bbox of all vertices (V) and of the displaced surface vertices: bounds[0..2] min, [3..5] max (flipped-order uint64).  Grid-stride with
// one atomic per CTA and value: one per warp serialised ~48 K same-address atomics in the L2 (37 us on C5, against 7 us now)
__global__ void __launch_bounds__(256) k_swept_bounds(SurfArgs s, const double* __restrict__ dir, const IterState* __restrict__ st, unsigned long long* __restrict__ bounds)
{
    __shared__ double sm[6][8];
    const double alpha = st->alpha_grid;
    double r[6] = { 1e300, 1e300, 1e300, -1e300, -1e300, -1e300 }; // lo[3], hi[3]
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(s.nV, s.nSV); i += gridDim.x * blockDim.x) {
        if (i < s.nV) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double x = s.V[(size_t)c * s.nV + i];
                r[c] = fmin(r[c], x);
                r[3 + c] = fmax(r[3 + c], x);
            }
        }
        if (i < s.nSV) {
            const int v = s.SVI[i];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double xt = s.V[(size_t)c * s.nV + v] + alpha * dir[3 * (size_t)v + c];
                r[c] = fmin(r[c], xt);
                r[3 + c] = fmax(r[3 + c], xt);
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        double x = r[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double y = __shfl_xor_sync(0xffffffffu, x, o);
            x = q < 3 ? fmin(x, y) : fmax(x, y);
        }
        if ((threadIdx.x & 31) == 0) sm[q][threadIdx.x >> 5] = x;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        const int q = threadIdx.x;
        double x = sm[q][0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) x = q < 3 ? fmin(x, sm[q][w]) : fmax(x, sm[q][w]);
        if (q < 3) atomicMin(bounds + q, flip_ord(x));
        else atomicMax(bounds + q, flip_ord(x));
    }
}

// SpatialHash.hpp:603-618 on the device-resident step: spanSize = alpha * mean|p| / h ; if (spanSize > 1) alpha /= spanSize.
// (pSize is the reference's serial host sum over the surface vertices, computed when the search direction is uploaded.)
__global__ void k_swept_alpha(IterState* st, const double* __restrict__ pSize_ptr, double h, unsigned long long* __restrict__ bounds)
{
    if (threadIdx.x != 0) return;
    const double pSize = *pSize_ptr;
    double alpha = ord_to_dbl(st->step_ord);
    const double span = alpha * pSize / h;
    if (span > 1) alpha /= span;
    st->step_ord = dbl_to_ord(alpha);
    st->alpha_grid = alpha;
    st->alpha_stage[2] = alpha;
    for (int c = 0; c < 3; ++c) { bounds[c] = ~0ull; bounds[3 + c] = 0ull; }
}
// reference grid geometry from the swept bbox (SpatialHash.hpp:627-640), incl. the cast-overflow fallback (:632-636)
__global__ void k_refgrid_params(IterState* st, const unsigned long long* __restrict__ bounds, double h, SweptCells* __restrict__ sc)
{
    if (threadIdx.x != 0) return;
    sc->lmax = 0;
    sc->hmax[0] = sc->hmax[1] = sc->hmax[2] = 0;
    double lo[3], hi[3], rmax = 0.0;
    double inv_h = 1.0 / h;
    bool bad = false;
    for (int c = 0; c < 3; ++c) {
        lo[c] = unflip_ord(bounds[c]);
        hi[c] = unflip_ord(bounds[3 + c]);
        st->ref_lo[c] = lo[c];
        st->ref_count[c] = (int)ceil((hi[c] - lo[c]) * inv_h);
        rmax = fmax(rmax, hi[c] - lo[c]);
        if (st->ref_count[c] <= 0) bad = true;
    }
    if (bad) { // cast overflow due to a huge search direction
        inv_h = 1.0 / (rmax * 1.01);
        st->ref_count[0] = st->ref_count[1] = st->ref_count[2] = 1;
    }
    st->ref_inv_h = inv_h;
}

// ------------------------------------------------------------------------------------------------------------------
// swept grid on the reference voxel lattice, and the candidate pairs inside its cells
// ------------------------------------------------------------------------------------------------------------------
// A cell is K x K x K reference voxels with its origin at IterState::ref_lo; every primitive (triangle, edge, surface vertex) is registered
// in each cell its voxel range [lo, hi] touches.  The reference's hash pairs two primitives iff their ranges overlap, and then both are
// registered in the cell that holds the per-axis max(lo_a, lo_b): testing the entries of a cell against each other and keeping the pairs
// whose max(lo) lies in that cell finds every such pair exactly once, with no neighbourhood and no inflation.  K >= (longest range) - 1
// keeps a primitive in <= 2 cells per axis, so there are at most 8 entries per primitive.
// An entry (16 bytes) is the range relative to the voxel before its cell, rel = v - (K c - 1) saturated to [0, 65535] per axis, and the
// id: rel lo == 0 <=> the range starts in an earlier cell.  Up to K = kSweptExactK the relative values are exact.  Beyond it the saturated
// overlap test is a superset (saturation is monotone) while the cell condition max(rel lo) >= 1 stays exact, and each hit is checked again
// on the vertices' ranges.
constexpr int kSweptExactK = 65534;

DEV bool ranges_overlap(const int* alo, const int* ahi, const int* blo, const int* bhi)
{
    return !(blo[0] > ahi[0] || bhi[0] < alo[0] || blo[1] > ahi[1] || bhi[1] < alo[1] || blo[2] > ahi[2] || bhi[2] < alo[2]);
}
DEV void prim_range(const int* __restrict__ vmin, const int* __restrict__ vmax, const int* vs, int n, int* lo, int* hi)
{
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        lo[c] = vmin[3 * (size_t)vs[0] + c];
        hi[c] = vmax[3 * (size_t)vs[0] + c];
        for (int k = 1; k < n; ++k) {
            lo[c] = min(lo[c], vmin[3 * (size_t)vs[k] + c]);
            hi[c] = max(hi[c], vmax[3 * (size_t)vs[k] + c]);
        }
    }
}
DEV bool dbc_v(const SurfArgs& s, int v) { return s.dbc && s.dbc[v] != 0; }
DEV int cod_v(const SurfArgs& s, int v) { return s.vCoDim ? s.vCoDim[v] : 3; }

// primitive i of [0, nSF + nSE + nSV): triangles, then edges, then surface vertices.  Returns its vertex count (type = 3 - count) and id.
DEV int swept_prim(const SurfArgs& s, int i, int* vs, int& id)
{
    if (i < s.nSF) {
        id = i;
        vs[0] = s.SF[i]; vs[1] = s.SF[(size_t)s.nSF + i]; vs[2] = s.SF[(size_t)2 * s.nSF + i];
        return 3;
    }
    i -= s.nSF;
    if (i < s.nSE) {
        id = i;
        vs[0] = s.SE[2 * i]; vs[1] = s.SE[2 * i + 1];
        return 2;
    }
    id = i - s.nSE;
    vs[0] = s.SVI[id];
    return 1;
}

// longest voxel range of any primitive along any axis, and the largest voxel index per axis (both reset by k_refgrid_params).  Grid-stride
// with one atomic per CTA and value: one per warp serialised ~135 K same-address atomics in the L2 (~0.1 ms on C5)
__global__ void __launch_bounds__(256) k_swept_extent(SurfArgs s, const int* __restrict__ vmin, const int* __restrict__ vmax, SweptCells* __restrict__ sc)
{
    __shared__ int sm[4][8];
    int r[4] = { 0, 0, 0, 0 }; // lmax, hmax[3]
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.nSF + s.nSE + s.nSV; i += gridDim.x * blockDim.x) {
        int vs[3], id, lo[3], hi[3];
        const int nv = swept_prim(s, i, vs, id);
        prim_range(vmin, vmax, vs, nv, lo, hi);
        for (int c = 0; c < 3; ++c) {
            r[0] = max(r[0], hi[c] - lo[c] + 1);
            r[1 + c] = max(r[1 + c], hi[c]);
        }
    }
    for (int q = 0; q < 4; ++q) {
        r[q] = __reduce_max_sync(0xffffffffu, r[q]);
        if ((threadIdx.x & 31) == 0) sm[q][threadIdx.x >> 5] = r[q];
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        int x = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) x = max(x, sm[threadIdx.x][w]);
        atomicMax(threadIdx.x == 0 ? &sc->lmax : &sc->hmax[threadIdx.x - 1], x);
    }
}
// K = the smallest integer >= max(2, lmax - 1) whose grid fits the dense cell table (the cell count does not grow with K)
__global__ void k_swept_cells(SweptCells* sc)
{
    if (threadIdx.x != 0) return;
    auto fits = [&](long long K) {
        unsigned long long n = 1;
        for (int c = 0; c < 3; ++c) n *= (unsigned long long)(sc->hmax[c] / K + 1);
        return n <= (unsigned long long)kGridCells;
    };
    long long lo = max(2, sc->lmax - 1);
    if (!fits(lo)) {
        long long hi = (long long)max(sc->hmax[0], max(sc->hmax[1], sc->hmax[2])) + 1; // one cell
        while (hi - lo > 1) {
            const long long mid = (lo + hi) / 2;
            if (fits(mid)) hi = mid;
            else lo = mid;
        }
        lo = hi;
    }
    const int K = (int)min(lo, 0x7fffffffll);
    sc->K = K;
    for (int c = 0; c < 3; ++c) sc->n[c] = sc->hmax[c] / K + 1;
}
DEV unsigned swept_key(const SweptCells& g, int type, int x, int y, int z) { return ((unsigned)type << kGridCellsLog2) | (unsigned)((z * g.n[1] + y) * g.n[0] + x); }

// count -> exclusive scan -> scatter, one entry per covered cell
__global__ void __launch_bounds__(256) k_swept_count(SurfArgs s, const int* __restrict__ vmin, const int* __restrict__ vmax, const SweptCells* __restrict__ sc,
    int* __restrict__ cnt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.nSF + s.nSE + s.nSV) return;
    const SweptCells g = *sc;
    int vs[3], id, lo[3], hi[3];
    const int nv = swept_prim(s, i, vs, id);
    prim_range(vmin, vmax, vs, nv, lo, hi);
    for (int z = lo[2] / g.K; z <= hi[2] / g.K; ++z)
        for (int y = lo[1] / g.K; y <= hi[1] / g.K; ++y)
            for (int x = lo[0] / g.K; x <= hi[0] / g.K; ++x) atomicAdd(cnt + swept_key(g, 3 - nv, x, y, z), 1);
}
// the counters serve as the cursors of the scatter (each ends at zero); the order inside a cell is whatever the atomics produce
__global__ void __launch_bounds__(256) k_swept_scatter(SurfArgs s, const int* __restrict__ vmin, const int* __restrict__ vmax, const SweptCells* __restrict__ sc,
    int* __restrict__ cnt, const int* __restrict__ off, unsigned* __restrict__ keys, uint4* __restrict__ ent)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.nSF + s.nSE + s.nSV) return;
    const SweptCells g = *sc;
    int vs[3], id, lo[3], hi[3];
    const int nv = swept_prim(s, i, vs, id);
    prim_range(vmin, vmax, vs, nv, lo, hi);
    auto rel = [&](int v, int c) { return (unsigned)min(max((long long)v - ((long long)g.K * c - 1), 0ll), 65535ll); };
    for (int z = lo[2] / g.K; z <= hi[2] / g.K; ++z)
        for (int y = lo[1] / g.K; y <= hi[1] / g.K; ++y)
            for (int x = lo[0] / g.K; x <= hi[0] / g.K; ++x) {
                const unsigned key = swept_key(g, 3 - nv, x, y, z);
                const int pos = off[key] + atomicSub(cnt + key, 1) - 1;
                keys[pos] = key;
                ent[pos] = make_uint4(rel(lo[0], x) | (rel(lo[1], y) << 16), rel(lo[2], z) | (rel(hi[0], x) << 16), rel(hi[1], y) | (rel(hi[2], z) << 16), (unsigned)id);
            }
}

// two entries of one cell: their ranges overlap and the per-axis max of their starts lies in this cell (see above).  Entry layout as QEntry:
// {lo0 | lo1 << 16, lo2 | hi0 << 16, hi1 | hi2 << 16, id}
DEV bool swept_hit(const uint4& a, const uint4& b)
{
    const unsigned M01 = __vmaxu2(a.x, b.x), m01 = __vminu2(__funnelshift_r(a.y, a.z, 16), __funnelshift_r(b.y, b.z, 16));
    const unsigned M2 = max(a.y & 0xffffu, b.y & 0xffffu), m2 = min(a.z >> 16, b.z >> 16);
    return __vcmpleu2(M01, m01) == 0xffffffffu && (M01 & 0xffffu) != 0u && (M01 >> 16) != 0u && M2 != 0u && M2 <= m2;
}

struct CandOut {
    int2* cand;
    unsigned long long* n;
    unsigned long long cap;
    int* overflow;
};
DEV void push_cand(const CandOut& o, int2 c)
{
    // aggregated over the lanes that are active here: one atomic per warp
    const unsigned m = __activemask();
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(o.n, (unsigned long long)__popc(m));
    base = __shfl_sync(m, base, leader);
    const unsigned long long i = base + __popc(m & ((1u << lane) - 1u));
    if (i < o.cap) o.cand[i] = c;
    else atomicExch(o.overflow, 1);
}

struct SweptArgs {
    SurfArgs s;
    const double* dir;
    const IterState* st;
    const int *vmin, *vmax;
    const SweptCells* sc;
    const unsigned* keys;
    const uint4* ent;
    const int* off;
    int lo, hi; // this rank's share: surface vertices [lo, hi) for PT, smaller edge id in [lo, hi) for EE
    CandOut out;
};

// the rules of the reference's candidate loops applied to one pair of the grid (SelfCollisionHandler.cpp:1385-1630, MeshCO.cpp:1396-1660)
DEV void pt_candidate(const SweptArgs& a, bool wide, int svI, int sfI)
{
    const SurfArgs& s = a.s;
    const int vI = s.SVI[svI];
    const int tv[3] = { s.SF[sfI], s.SF[(size_t)s.nSF + sfI], s.SF[(size_t)2 * s.nSF + sfI] };
    if (wide) {
        int lo[3], hi[3];
        prim_range(a.vmin, a.vmax, tv, 3, lo, hi);
        if (!ranges_overlap(a.vmin + 3 * (size_t)vI, a.vmax + 3 * (size_t)vI, lo, hi)) return;
    }
    const bool oP = obstacle_vertex(s, vI), oT = obstacle_vertex(s, tv[0]); // mesh-obstacle pairs are not filtered (MeshCO.cpp:1396-1570)
    if (oP && oT) return;
    if (!oP && !oT && ((cod_v(s, vI) < 3 && cod_v(s, tv[0]) < 3) || (dbc_v(s, vI) && dbc_v(s, tv[0]) && dbc_v(s, tv[1]) && dbc_v(s, tv[2])))) return;
    push_cand(a.out, make_int2(-svI - 1, sfI));
}
DEV void ee_candidate(const SweptArgs& a, bool wide, int eI, int eJ)
{
    const SurfArgs& s = a.s;
    if (eI < a.lo || eI >= a.hi) return;
    const int v[4] = { s.SE[2 * eI], s.SE[2 * eI + 1], s.SE[2 * eJ], s.SE[2 * eJ + 1] };
    if (wide) {
        int qlo[3], qhi[3], lo[3], hi[3];
        prim_range(a.vmin, a.vmax, v, 2, qlo, qhi);
        prim_range(a.vmin, a.vmax, v + 2, 2, lo, hi);
        if (!ranges_overlap(qlo, qhi, lo, hi)) return;
    }
    {   // swept-AABB test of queryEdgeForEdgesWithBBoxCheck (SpatialHash.hpp:819-828) on the exact boxes {x, x + alpha p} of both edges,
        // rounded like k_boxes
        const double alpha = a.st->alpha_grid;
        double blo[2][3], bhi[2][3];
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                blo[e][c] = 1e300;
                bhi[e][c] = -1e300;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const int w = v[2 * e + k];
                    const double x = __ldg(s.V + (size_t)c * s.nV + w), xt = x + alpha * __ldg(a.dir + 3 * (size_t)w + c);
                    blo[e][c] = fmin(fmin(blo[e][c], x), xt);
                    bhi[e][c] = fmax(fmax(bhi[e][c], x), xt);
                }
            }
        bool sep = false;
#pragma unroll
        for (int c = 0; c < 3; ++c) sep = sep || (blo[1][c] - bhi[0][c] > 0.0) || (blo[0][c] - bhi[1][c] > 0.0);
        if (sep) return;
    }
    const bool oA = obstacle_vertex(s, v[0]), oB = obstacle_vertex(s, v[2]); // (MeshCO.cpp:1576-1660)
    if (oA && oB) return;
    if (!oA && !oB && ((cod_v(s, v[0]) < 3 && cod_v(s, v[2]) < 3) || (dbc_v(s, v[0]) && dbc_v(s, v[1]) && dbc_v(s, v[2]) && dbc_v(s, v[3])))) return;
    push_cand(a.out, make_int2(eI, eJ));
}

// Pair kernels: a warp takes 32 consecutive entries of the sorted array as queries (shared memory); consecutive entries share their cell,
// so the partners of a run of queries are the entries of one cell, read once, a lane per partner, each tested against every query of the
// run.  The grid-stride over runs of 32 queries spreads a crowded cell over as many warps as it has query chunks.  Hits are staged per
// warp and checked by the candidate rules lane-parallel once the stage is half full.
constexpr int kSweptWarps = 8;
constexpr int kHitCap = 256;
struct alignas(16) SweptQuery {
    uint4 e;
    int pos, v0, v1, pad;
};
struct HitStage {
    int2 buf[kHitCap];
    unsigned count;
};
template <typename F> DEV void stage_hit(HitStage& hs, int2 p, F rule)
{
    const unsigned i = atomicAdd(&hs.count, 1u);
    if (i < (unsigned)kHitCap) hs.buf[i] = p;
    else rule(p); // stage full: check it right here
}
// all 32 lanes
template <typename F> DEV void flush_hits(HitStage& hs, int lane, unsigned threshold, F rule)
{
    __syncwarp();
    const unsigned n = min(hs.count, (unsigned)kHitCap);
    if (n < threshold || n == 0u) return;
    for (unsigned i = lane; i < n; i += 32) rule(hs.buf[i]);
    __syncwarp();
    if (lane == 0) hs.count = 0;
    __syncwarp();
}

// edge-edge: every pair of edge entries of a cell once, from the entry with the smaller sorted position
__global__ void __launch_bounds__(32 * kSweptWarps) k_swept_pairs_ee(SweptArgs a)
{
    __shared__ HitStage sStage[kSweptWarps];
    __shared__ SweptQuery sQ[kSweptWarps][32];
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    HitStage& stage = sStage[wib];
    SweptQuery* Q = sQ[wib];
    if (lane == 0) stage.count = 0;
    const bool wide = a.sc->K > kSweptExactK;
    auto rule = [&](int2 p) { ee_candidate(a, wide, p.x, p.y); };
    const int first = a.off[1u << kGridCellsLog2], last = a.off[2u << kGridCellsLog2];
    const int2* __restrict__ SE2 = reinterpret_cast<const int2*>(a.s.SE);
    for (int base = first + (blockIdx.x * kSweptWarps + wib) * 32; base < last; base += gridDim.x * kSweptWarps * 32) {
        const int pos = base + lane;
        const bool valid = pos < last;
        unsigned key = 0xffffffffu;
        __syncwarp();
        if (valid) {
            const uint4 e = __ldg(a.ent + pos);
            key = a.keys[pos];
            const int2 v = __ldg(SE2 + (int)e.w);
            Q[lane] = SweptQuery{ e, pos, v.x, v.y, 0 };
        }
        __syncwarp();
        unsigned remaining = __ballot_sync(full, valid);
        while (remaining) {
            const int leader = __ffs(remaining) - 1;
            const unsigned k0 = __shfl_sync(full, key, leader);
            const unsigned m = __ballot_sync(full, valid && key == k0); // the run: consecutive lanes (the array is sorted by cell)
            remaining &= ~m;
            const int q_lo = leader, q_hi = 32 - __clz(m);
            const int cs = __shfl_sync(full, pos, leader) + 1, ce = __ldg(a.off + k0 + 1); // partners: the cell's entries behind the run's first query
            for (int j = cs + lane; j - lane < ce; j += 32) {
                if (j < ce) {
                    const uint4 e = __ldg(a.ent + j);
                    const int2 bv = __ldg(SE2 + (int)e.w);
                    for (int q = q_lo; q < q_hi; ++q) {
                        const SweptQuery& A = Q[q]; // same address on every lane: broadcast
                        // edges that share a vertex are no pair
                        if (j > A.pos && swept_hit(A.e, e) && A.v0 != bv.x && A.v0 != bv.y && A.v1 != bv.x && A.v1 != bv.y)
                            stage_hit(stage, make_int2(min((int)A.e.w, (int)e.w), max((int)A.e.w, (int)e.w)), rule);
                    }
                }
                flush_hits(stage, lane, kHitCap / 2, rule);
            }
        }
    }
    flush_hits(stage, lane, 1u, rule);
}

// point-triangle: every surface-vertex entry of a cell against every triangle entry of the cell
__global__ void __launch_bounds__(32 * kSweptWarps) k_swept_pairs_pt(SweptArgs a)
{
    __shared__ HitStage sStage[kSweptWarps];
    __shared__ SweptQuery sQ[kSweptWarps][32];
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    HitStage& stage = sStage[wib];
    SweptQuery* Q = sQ[wib];
    if (lane == 0) stage.count = 0;
    const bool wide = a.sc->K > kSweptExactK;
    auto rule = [&](int2 p) { pt_candidate(a, wide, p.x, p.y); };
    const int first = a.off[2u << kGridCellsLog2], last = a.off[3u << kGridCellsLog2];
    const int* __restrict__ SF = a.s.SF;
    const size_t nSF = (size_t)a.s.nSF;
    for (int base = first + (blockIdx.x * kSweptWarps + wib) * 32; base < last; base += gridDim.x * kSweptWarps * 32) {
        const int pos = base + lane;
        bool valid = pos < last;
        unsigned key = 0xffffffffu;
        __syncwarp();
        if (valid) {
            const uint4 e = __ldg(a.ent + pos);
            valid = (int)e.w >= a.lo && (int)e.w < a.hi; // this rank's surface vertices
            key = a.keys[pos] & (kGridCells - 1u);       // the cell; its triangles are entries of type 0
            Q[lane] = SweptQuery{ e, pos, __ldg(a.s.SVI + (int)e.w), 0, 0 };
        }
        __syncwarp();
        unsigned remaining = __ballot_sync(full, valid);
        while (remaining) {
            const int leader = __ffs(remaining) - 1;
            const unsigned k0 = __shfl_sync(full, key, leader);
            const unsigned m = __ballot_sync(full, valid && key == k0);
            remaining &= ~m;
            const int q_lo = leader, q_hi = 32 - __clz(m);
            const int cs = __ldg(a.off + k0), ce = __ldg(a.off + k0 + 1);
            for (int j = cs + lane; j - lane < ce; j += 32) {
                if (j < ce) {
                    const uint4 e = __ldg(a.ent + j);
                    const int t0 = __ldg(SF + (int)e.w), t1 = __ldg(SF + nSF + (int)e.w), t2 = __ldg(SF + 2 * nSF + (int)e.w);
                    for (int q = q_lo; q < q_hi; ++q) {
                        const SweptQuery& A = Q[q];
                        // a triangle that contains the vertex is no partner
                        if (((m >> q) & 1u) && swept_hit(A.e, e) && A.v0 != t0 && A.v0 != t1 && A.v0 != t2) stage_hit(stage, make_int2((int)A.e.w, (int)e.w), rule);
                    }
                }
                flush_hits(stage, lane, kHitCap / 2, rule);
            }
        }
    }
    flush_hits(stage, lane, 1u, rule);
}

// ------------------------------------------------------------------------------------------------------------------
// Tight-Inclusion pieces shared by both narrow-phase stages
// ------------------------------------------------------------------------------------------------------------------
struct TiPair {
    double x0[12], x1[12]; // 4 vertices at t=0 / t=1 ; VF: (p,t0,t1,t2)  EE: (a0,a1,b0,b1)
    // 1: an edge pair of the mesh and the obstacle that runs through the vertex-face ROUTINE on its four points in edge order (MeshCO.cpp:900-940,
    // :1609-1655 call vertexFaceCCD_double there) while its initial distance and its error bound stay the edge-edge ones
    int ee_metric;
};
// the routine flag `vf` says which inclusion function runs; distance and error bound follow the kind of the PAIR
DEV bool vf_metric(bool vf, const TiPair& P) { return vf && !P.ee_metric; }
struct DBox { // parameter box: [n/2^k, (n+1)/2^k] per axis; kk = tk | uk<<8 | vk<<16 | flags<<24
    unsigned long long tn, un, vn;
    unsigned kk;
    unsigned pad;
};
DEV double pow2neg(int k) { return __longlong_as_double((long long)(1023 - k) << 52); }
DEV double dy_lo(unsigned long long n, int k) { return (double)n * pow2neg(k); }
DEV double dy_hi(unsigned long long n, int k) { return (double)(n + 1) * pow2neg(k); }

// co-domain test of one box: returns zero_in; sets box_in and max/each true_tol   (oracle: origin_in_box)
DEV bool origin_in_box(bool VF, const TiPair& P, const DBox& b, const double* err, double ms, bool& box_in, double* true_tol)
{
    const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
    const double tv[2] = { dy_lo(b.tn, tk), dy_hi(b.tn, tk) }, uv[2] = { dy_lo(b.un, uk), dy_hi(b.un, uk) }, vv[2] = { dy_lo(b.vn, vk), dy_hi(b.vn, vk) };
    box_in = true;
    bool zero_in = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        double mn = 1e300, mx = -1e300;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            double p[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) p[k] = (P.x1[3 * k + c] - P.x0[3 * k + c]) * tv[i] + P.x0[3 * k + c];
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int l = 0; l < 2; ++l) {
                    double f;
                    if (VF) {
                        const double pt = ((p[2] - p[1]) * uv[j] + (p[3] - p[1]) * vv[l]) + p[1];
                        f = p[0] - pt;
                    }
                    else {
                        const double pa = (p[1] - p[0]) * uv[j] + p[0];
                        const double pb = (p[3] - p[2]) * vv[l] + p[2];
                        f = pa - pb;
                    }
                    mn = fmin(mn, f);
                    mx = fmax(mx, f);
                }
        }
        true_tol[c] = mx - mn;
        const double eps = err[c] + ms;
        if (mn > eps || mx < -eps) zero_in = false;
        if (!(mn >= -eps && mx <= eps)) box_in = false;
    }
    return zero_in;
}

DEV double linf3(const double* a, const double* b) { return fmax(fmax(fabs(a[0] - b[0]), fabs(a[1] - b[1])), fabs(a[2] - b[2])); }

DEV void width_tolerances(bool VF, const TiPair& P, double tolerance, double* tol)
{
    double ps[4][3], pe[4][3];
#pragma unroll
    for (int side = 0; side < 2; ++side) {
        const double* x = side ? P.x1 : P.x0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double q0, q1, q2, q3;
            if (VF) {
                q0 = x[c] - x[3 + c];
                q1 = x[c] - x[9 + c];
                q2 = x[c] - (x[6 + c] + x[9 + c] - x[3 + c]);
                q3 = x[c] - x[6 + c];
            }
            else {
                q0 = x[c] - x[6 + c];
                q1 = x[c] - x[9 + c];
                q2 = x[3 + c] - x[9 + c];
                q3 = x[3 + c] - x[6 + c];
            }
            if (side) { pe[0][c] = q0; pe[1][c] = q1; pe[2][c] = q2; pe[3][c] = q3; }
            else { ps[0][c] = q0; ps[1][c] = q1; ps[2][c] = q2; ps[3][c] = q3; }
        }
    }
    double dl = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) dl = fmax(dl, linf3(pe[q], ps[q]));
    const double e0 = fmax(fmax(linf3(ps[3], ps[0]), linf3(pe[3], pe[0])), fmax(linf3(pe[2], pe[1]), linf3(ps[2], ps[1])));
    const double e1 = fmax(fmax(linf3(ps[1], ps[0]), linf3(pe[1], pe[0])), fmax(linf3(pe[2], pe[3]), linf3(ps[2], ps[3])));
    tol[0] = tolerance / (3.0 * dl);
    tol[1] = tolerance / (3.0 * e0);
    tol[2] = tolerance / (3.0 * e1);
}

DEV void load_pair(const SurfArgs& s, const double* __restrict__ dir, int2 c, bool& vf, int* v, TiPair& P)
{
    vf = c.x < 0;
    if (vf) {
        const int svI = -c.x - 1, sfI = c.y;
        v[0] = s.SVI[svI]; v[1] = s.SF[sfI]; v[2] = s.SF[(size_t)s.nSF + sfI]; v[3] = s.SF[(size_t)2 * s.nSF + sfI];
    }
    else {
        v[0] = s.SE[2 * c.x]; v[1] = s.SE[2 * c.x + 1]; v[2] = s.SE[2 * c.y]; v[3] = s.SE[2 * c.y + 1];
    }
    P.ee_metric = 0;
    if (!vf && s.ee_as_vf && obstacle_vertex(s, v[0]) != obstacle_vertex(s, v[2])) { // (mesh edge first: its sorted index is the smaller one)
        vf = true;
        P.ee_metric = 1;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const double x = __ldg(s.V + (size_t)q * s.nV + v[k]);
            P.x0[3 * k + q] = x;
            P.x1[3 * k + q] = x + __ldg(dir + 3 * (size_t)v[k] + q);
        }
}

DEV double pair_distance_sqrt(bool vf, const TiPair& P)
{
    const V3 a = { P.x0[0], P.x0[1], P.x0[2] }, b = { P.x0[3], P.x0[4], P.x0[5] }, c = { P.x0[6], P.x0[7], P.x0[8] }, d = { P.x0[9], P.x0[10], P.x0[11] };
    return sqrt(vf_metric(vf, P) ? point_tri_d(a, b, c, d) : edge_edge_d(a, b, c, d));
}

// ------------------------------------------------------------------------------------------------------------------
// stage 1: one thread per candidate
// ------------------------------------------------------------------------------------------------------------------
struct NarrowArgs {
    SurfArgs s;
    const double* dir;
    const int2* cand;
    double err_vf[3], err_ee[3];
    double tol;
    int max_itr;
    // device-resident: cand_range = the slice of `cand` this rank walks, max_t = the step on entry (every pair's max_t), ccd_ord = the
    // running device-wide minimum (ordered-uint image): boxes starting at or after it cannot lower the result
    const IterState* st;
    DBox* arena;     // overflow arena of the warp-level pass (ti_root_finder_arena) and its lock
    int* arena_lock;
};

__global__ void __launch_bounds__(128) k_ti_stage1(NarrowArgs a, unsigned* __restrict__ survivors, unsigned* __restrict__ nSurv, int* __restrict__ zero_flag)
{
    const unsigned long long begin = a.st->cand_range[0], end = a.st->cand_range[1];
    // grid-stride over whole warps (the warp-aggregated append below needs all 32 lanes)
    for (unsigned long long base = begin + (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < end; base += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long i = base + (threadIdx.x & 31);
    bool alive = false;
    if (i < end) {
        bool vf;
        int v[4];
        TiPair P;
        load_pair(a.s, a.dir, a.cand[i], vf, v, P);
        const double d = pair_distance_sqrt(vf, P);
        if (d == 0.0) atomicExch(zero_flag, 1); // "Initial CCD distance is zero! Returning 0 stepSize." (:730-737)
        else {
            const double ms = fmin(0.2 * d, 1e-6);
            DBox root = { 0ull, 0ull, 0ull, 0u, 0u };
            bool box_in;
            double tt[3];
            alive = origin_in_box(vf, P, root, vf_metric(vf, P) ? a.err_vf : a.err_ee, ms, box_in, tt);
        }
    }
    // warp-aggregated append of the survivors
    const unsigned m = __ballot_sync(0xffffffffu, alive);
    if (m) {
        const int lane = threadIdx.x & 31;
        unsigned base = 0;
        if (lane == __ffs(m) - 1) base = atomicAdd(nSurv, __popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        if (alive) survivors[base + __popc(m & ((1u << lane) - 1))] = (unsigned)i;
    }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// stage 2: warp per surviving pair
// ------------------------------------------------------------------------------------------------------------------
struct Key3 {
    double t, u, v;
};
DEV bool key_less(const Key3& a, const Key3& b)
{
    if (a.t != b.t) return a.t < b.t;
    if (a.u != b.u) return a.u < b.u;
    return a.v < b.v;
}
// warp min of (key, payload)
DEV void warp_min_key(Key3& k, unsigned& pay, double& aux)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Key3 r;
        r.t = __shfl_xor_sync(0xffffffffu, k.t, o);
        r.u = __shfl_xor_sync(0xffffffffu, k.u, o);
        r.v = __shfl_xor_sync(0xffffffffu, k.v, o);
        const unsigned rp = __shfl_xor_sync(0xffffffffu, pay, o);
        const double ra = __shfl_xor_sync(0xffffffffu, aux, o);
        if (key_less(r, k)) {
            k = r;
            pay = rp;
            aux = ra;
        }
    }
}
DEV bool sum_le_1(unsigned long long an, int ak, unsigned long long bn, int bk)
{
    // lo(a) + lo(b) <= 1 exactly; k <= 60 so the aligned sum fits in 64 bits when the larger exponent is used carefully
    const int k = max(ak, bk);
    // n < 2^ak: n << (k-ak) < 2^k <= 2^60 -> the sum is < 2^61
    const unsigned long long s = (an << (k - ak)) + (bn << (k - bk));
    return s <= (1ull << k);
}

constexpr unsigned F_ZERO = 1u << 24; // zero_in flag stored in DBox::kk
constexpr unsigned F_VIS = 1u << 25;  // the box was evaluated at this level (the library counts it towards max_itr)

constexpr int kStage2WarpsPerCtaDev = 4;
constexpr int kSmemLevel = 184; // boxes per level buffer kept in shared memory by the warp-level pass
constexpr int kWideLevel = 10; // levels with at least this many boxes are evaluated box-parallel, narrower ones corner-parallel
// Boxes per level buffer of the overflow arena.  A level only splits boxes the library has counted, and it leaves before the count
// exceeds max_itr (1e6), so no level holds more than 2 max_itr boxes: a search in the arena never outgrows it.
constexpr int kArenaLevel = 2000000;

DEV Key3 box_key(const DBox& b)
{
    const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
    return Key3{ dy_lo(b.tn, tk), dy_lo(b.un, uk), dy_lo(b.vn, vk) };
}

// warp inclusive prefix sum of v
DEV int warp_incl_scan(int v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += y;
    }
    return v;
}

// Does the library leave this level through max_itr?  It walks the level in key order, counting every evaluated box, and leaves at the
// first box containing the origin whose count exceeds max_itr -- unless a terminal box comes first.  The last box it can leave at is the
// last one containing the origin before K2 when K2 is terminal, up to and including K2 when K2 only stops the level's splitting, or the
// last one of the level.  room = max_itr - (boxes counted at earlier levels).
DEV bool library_leaves_at_max_itr(const DBox* cur, int n, int lane, bool has_k2, bool k2_terminal, const Key3& k2, long long room)
{
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    Key3 nz = { INF, INF, INF }; // the last candidate box, as the minimum of the negated keys
    unsigned pay = 0;
    double aux = 0.0;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        Key3 mk = { INF, INF, INF };
        if (i < n && (cur[i].kk & F_ZERO)) {
            const Key3 key = box_key(cur[i]);
            if (!has_k2 || key_less(key, k2) || (!k2_terminal && !key_less(k2, key))) mk = Key3{ -key.t, -key.u, -key.v };
        }
        warp_min_key(mk, pay, aux);
        if (key_less(mk, nz)) nz = mk;
    }
    if (nz.t == INF) return false;
    const Key3 z = { -nz.t, -nz.u, -nz.v };
    long long count = 0; // the library's count when it reaches z
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        count += __popc(__ballot_sync(0xffffffffu, i < n && (cur[i].kk & F_VIS) && !key_less(z, box_key(cur[i]))));
    }
    return count > room;
}

// box-parallel root finder of the warp-level pass, one box per lane, level buffers in global memory: 0 no collision, 1 collision (toi set),
// -1 a level outgrew the buffers (toi / out_tol hold the conservative estimate of the level before)
__device__ int ti_root_finder(bool VF, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err, double ms, int max_itr, DBox* bufA,
    DBox* bufB, int cap, int lane, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes, const unsigned long long* best)
{
    const bool check_t = (max_t != 1.0);
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    DBox* cur = bufA;
    DBox* nxt = bufB;
    if (lane == 0) cur[0] = DBox{ 0ull, 0ull, 0ull, 0u, 0u };
    __syncwarp();
    int n = 1;
    double toi_skip = INF;
    bool use_skip = false;
    long long refine = 0;
    double temp_toi = INF, temp_out_tol = co_tol;
    out_tol = co_tol;
    toi = INF;
    unsigned long long bo_cur = best ? *reinterpret_cast<const volatile unsigned long long*>(best) : 0ull;
    while (n > 0) {
        // exact pruning against the running device-wide minimum: a box that starts at t_lo >= max(best, 1e-6) can only yield a time of
        // impact >= best (and no 0.8-rescaled retry, which needs toi < 1e-6), so dropping it cannot change the final min over pairs
        // The bound used here was requested one level ago (stale = prunes less, never wrong): its L2 round trip overlaps the level.
        double t_prune = INF;
        if (best) {
            t_prune = fmax(ord_to_dbl(bo_cur), 1e-6);
            bo_cur = *reinterpret_cast<const volatile unsigned long long*>(best); // same address on all lanes, one value
        }
        // ---- pass 1: evaluate, find K1 (first box containing the origin) and K2 (first terminal box) ----------
        Key3 k1 = { INF, INF, INF }, k2 = { INF, INF, INF };
        unsigned p1 = 0, p2 = 0; // payload bit0: flagged (K1) / cond1 (K2)
        double a1 = 0.0, a2 = 0.0;
        int visited = 0;
        for (int base = 0; base < n; base += 32) {
            const int i = base + lane;
            Key3 mk1 = { INF, INF, INF }, mk2 = { INF, INF, INF };
            unsigned mp1 = 0, mp2 = 0;
            double ma1 = 0.0, ma2 = 0.0;
            bool vis = false;
            if (i < n) {
                DBox b = cur[i];
                const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
                const double tlo = dy_lo(b.tn, tk);
                unsigned flags = 0;
                if (tlo < toi_skip && tlo < t_prune) {
                    vis = true;
                    flags = F_VIS;
                    bool box_in;
                    double tt[3];
                    if (origin_in_box(VF, P, b, err, ms, box_in, tt)) {
                        flags |= F_ZERO;
                        const bool tol_cond = tt[0] <= co_tol && tt[1] <= co_tol && tt[2] <= co_tol;
                        const bool cond1 = pow2neg(tk) <= tol[0] && pow2neg(uk) <= tol[1] && pow2neg(vk) <= tol[2];
                        const Key3 key = { tlo, dy_lo(b.un, uk), dy_lo(b.vn, vk) };
                        mk1 = key;
                        mp1 = (tol_cond || box_in || cond1) ? 1u : 0u;
                        ma1 = fmax(fmax(tt[0], tt[1]), tt[2]);
                        if (mp1) {
                            mk2 = key;
                            mp2 = cond1 ? 1u : 0u;
                        }
                    }
                }
                cur[i].kk = (b.kk & 0x00ffffffu) | flags;
            }
            visited += __popc(__ballot_sync(0xffffffffu, vis));
            warp_min_key(mk1, mp1, ma1);
            warp_min_key(mk2, mp2, ma2);
            if (key_less(mk1, k1)) { k1 = mk1; p1 = mp1; a1 = ma1; }
            if (key_less(mk2, k2)) { k2 = mk2; p2 = mp2; a2 = ma2; }
        }
        __syncwarp();
        const bool any_zero = k1.t != INF;
        if (!any_zero) { // nothing at this level contains the origin: the search space is exhausted
            n = 0;
            break;
        }
        if (p1 & 1u) { // the first box containing the origin is terminal: conditions 1/2/3 of the library
            toi = k1.t;
            return 1;
        }
        const bool has_k2 = k2.t != INF;
        boxes += (unsigned)visited; // diagnostics: boxes evaluated (the same on every lane)
        if (max_itr > 0) {
            temp_toi = k1.t;
            temp_out_tol = fmax(a1, co_tol);
            // the library's own early-out, at the box where its count crosses max_itr; it can only cross where the count of every
            // evaluated box does, which levels of the per-warp buffers never reach (181 levels x 4,096 boxes < 1e6)
            if (refine + visited > max_itr && library_leaves_at_max_itr(cur, n, lane, has_k2, (p2 & 1u) != 0, k2, max_itr - refine)) {
                if (lane == 0) atomicAdd(warn, 1);
                toi = temp_toi;
                out_tol = temp_out_tol;
                return 1;
            }
        }
        if (has_k2 && (p2 & 1u)) { // a later box already below the width tolerances (condition 1)
            // boxes between K1 and K2 do not matter: the library returns here
            toi = k2.t;
            return 1;
        }
        if (has_k2) {
            if (k2.t < toi_skip) toi_skip = k2.t;
            use_skip = true;
        }
        // ---- pass 2: split every box that contains the origin and precedes K2; count the boxes the library evaluated (up to K2) --
        int nn = 0;
        long long counted = 0;
        bool over = false, full = false;
        for (int base = 0; base < n; base += 32) {
            const int i = base + lane;
            int nchild = 0;
            DBox c0, c1;
            bool cnt = false;
            if (i < n) {
                const DBox b = cur[i];
                if (b.kk & F_VIS) cnt = !has_k2 || !key_less(k2, box_key(b));
                if (b.kk & F_ZERO) {
                    const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
                    const Key3 key = { dy_lo(b.tn, tk), dy_lo(b.un, uk), dy_lo(b.vn, vk) };
                    if (!has_k2 || key_less(key, k2)) {
                        const double w[3] = { pow2neg(tk), pow2neg(uk), pow2neg(vk) };
                        int split = -1;
                        double best = -1.0;
#pragma unroll
                        for (int d = 0; d < 3; ++d)
                            if (w[d] > tol[d]) {
                                const double r = inv_tol[d] * w[d]; // = w[d] / tol[d] bit for bit: w[d] is a power of two (see ti_ccd)
                                if (r > best) { best = r; split = d; }
                            }
                        const int pk = split == 0 ? tk : (split == 1 ? uk : vk);
                        if (split < 0 || pk >= 60) over = true; // bisection overflow: handled like the iteration overflow
                        else {
                            const unsigned long long pn = split == 0 ? b.tn : (split == 1 ? b.un : b.vn);
#pragma unroll
                            for (int half = 0; half < 2; ++half) {
                                const unsigned long long hn = 2 * pn + half;
                                const int hk = pk + 1;
                                bool keep = true;
                                if (split == 0) { if (check_t) keep = !(dy_hi(hn, hk) < 0.0 || dy_lo(hn, hk) > max_t); }
                                else if (VF) keep = (split == 1) ? sum_le_1(hn, hk, b.vn, vk) : sum_le_1(hn, hk, b.un, uk);
                                if (keep) {
                                    DBox c = b;
                                    c.kk &= 0x00ffffffu;
                                    if (split == 0) { c.tn = hn; c.kk = (c.kk & ~0xffu) | (unsigned)hk; }
                                    else if (split == 1) { c.un = hn; c.kk = (c.kk & ~0xff00u) | ((unsigned)hk << 8); }
                                    else { c.vn = hn; c.kk = (c.kk & ~0xff0000u) | ((unsigned)hk << 16); }
                                    if (nchild == 0) c0 = c;
                                    else c1 = c;
                                    ++nchild;
                                }
                            }
                        }
                    }
                }
            }
            counted += __popc(__ballot_sync(0xffffffffu, cnt));
            // warp exclusive scan of nchild
            const int incl = warp_incl_scan(nchild, lane), total = __shfl_sync(0xffffffffu, incl, 31);
            const int off = nn + incl - nchild;
            if (nn + total > cap) full = true;
            else {
                if (nchild > 0) nxt[off] = c0;
                if (nchild > 1) nxt[off + 1] = c1;
            }
            nn += total;
            if (__any_sync(0xffffffffu, over || full)) break;
        }
        if (__any_sync(0xffffffffu, over || full)) {
            // bisection depth exhausted: return the conservative per-level estimate (earliest box containing the origin); a level that
            // outgrew the buffers returns the same estimate as -1, and the caller runs the search again in larger ones
            toi = temp_toi;
            out_tol = temp_out_tol;
            if (__any_sync(0xffffffffu, over)) {
                if (lane == 0) atomicAdd(warn, 1);
                return 1;
            }
            return -1;
        }
        refine += counted;
        __syncwarp();
        DBox* t = cur; cur = nxt; nxt = t;
        n = nn;
    }
    if (use_skip) {
        toi = toi_skip;
        return 1;
    }
    return 0;
}

// ---- corner-parallel variant of the root finder for the warp-level pass ------------------------------------------------------
// Deep searches are narrow (a handful of boxes per level), so there is little parallelism over boxes; what can be parallelised is
// the box itself.  A narrow level is evaluated four boxes at a time: each 8-lane group takes one box, a lane is one of its 8 corners
// and evaluates the 3 coordinates of F in turn; the co-domain interval of a coordinate is a 3-step shuffle min/max inside the group,
// after which all 8 lanes know every inclusion flag of their box (no ballots).  Each group keeps its own K1/K2 candidates, merged by
// one 2-step exchange per level.  Levels of >= kWideLevel boxes switch to one box per lane.  The split pass is always one box per
// lane with a warp scan.  Level buffers live in shared memory.  Same arithmetic per corner, same decisions => same result as the
// box-parallel variant.  Returns -1 when a level outgrows the shared-memory buffer (the caller restarts with the box-parallel variant).
__device__ int ti_root_finder_cp(bool VF, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err, double ms, int max_itr, DBox* sA, DBox* sB,
    int lane, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes, const unsigned long long* best)
{
    const bool check_t = (max_t != 1.0);
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    const int corner = lane & 7;
    const int ci = corner >> 2, cj = (corner >> 1) & 1, cl = corner & 1;
    DBox* cur = sA;
    DBox* nxt = sB;
    if (lane == 0) cur[0] = DBox{ 0ull, 0ull, 0ull, 0u, 0u };
    __syncwarp();
    int n = 1;
    double toi_skip = INF;
    bool use_skip = false;
    long long refine = 0;
    double temp_toi = INF, temp_out_tol = co_tol;
    out_tol = co_tol;
    toi = INF;
    unsigned long long bo_cur = best ? *reinterpret_cast<const volatile unsigned long long*>(best) : 0ull;
    while (n > 0) {
        Key3 k1 = { INF, INF, INF }, k2 = { INF, INF, INF };
        unsigned p1 = 0, p2 = 0;
        double a1max = 0.0;
        int visited = 0;
        // exact pruning against the running device-wide minimum (see ti_root_finder).  The value used at this level was requested
        // one level ago (a stale bound only prunes less), so its L2 round trip is off the per-level critical path.
        double t_prune = INF;
        if (best) {
            t_prune = fmax(ord_to_dbl(bo_cur), 1e-6);
            bo_cur = *reinterpret_cast<const volatile unsigned long long*>(best); // same address on all lanes: one broadcast request
        }
        if (n >= kWideLevel) {
            // wide level: one box per lane (box-parallel), K1/K2 by warp min-reduction over the keys
            for (int base = 0; base < n; base += 32) {
                const int i = base + lane;
                Key3 mk1 = { INF, INF, INF }, mk2 = { INF, INF, INF };
                unsigned mp1 = 0, mp2 = 0;
                double ma1 = 0.0, ma2 = 0.0;
                bool vis = false;
                if (i < n) {
                    const DBox b = cur[i];
                    const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
                    const double tlo = dy_lo(b.tn, tk);
                    unsigned flags = 0;
                    if (tlo < toi_skip && tlo < t_prune) {
                        vis = true;
                        bool box_in;
                        double tt[3];
                        if (origin_in_box(VF, P, b, err, ms, box_in, tt)) {
                            flags = F_ZERO;
                            const bool tol_cond = tt[0] <= co_tol && tt[1] <= co_tol && tt[2] <= co_tol;
                            const bool cond1 = pow2neg(tk) <= tol[0] && pow2neg(uk) <= tol[1] && pow2neg(vk) <= tol[2];
                            const Key3 key = { tlo, dy_lo(b.un, uk), dy_lo(b.vn, vk) };
                            mk1 = key;
                            mp1 = (tol_cond || box_in || cond1) ? 1u : 0u;
                            ma1 = fmax(fmax(tt[0], tt[1]), tt[2]);
                            if (mp1) { mk2 = key; mp2 = cond1 ? 1u : 0u; }
                        }
                    }
                    cur[i].kk = (b.kk & 0x00ffffffu) | flags;
                }
                visited += __popc(__ballot_sync(0xffffffffu, vis));
                warp_min_key(mk1, mp1, ma1);
                warp_min_key(mk2, mp2, ma2);
                if (key_less(mk1, k1)) { k1 = mk1; p1 = mp1; a1max = ma1; }
                if (key_less(mk2, k2)) { k2 = mk2; p2 = mp2; }
            }
        }
        else {
            // narrow level: FOUR boxes at a time, one per 8-lane group; a lane is one corner and evaluates the three coordinates in
            // turn, so the co-domain interval of a coordinate is a 3-step shuffle min/max inside the group and every inclusion flag
            // is known to all 8 lanes without a ballot.  Each group tracks its own K1/K2; one 2-step exchange merges them.
            Key3 gk1 = { INF, INF, INF }, gk2 = { INF, INF, INF };
            unsigned gp1 = 0, gp2 = 0;
            double ga1 = 0.0, ga2 = 0.0;
            const int grp = lane >> 3;
            for (int base = 0; base < n; base += 4) {
                const int bI = base + grp;
                DBox b = DBox{ 0ull, 0ull, 0ull, 0u, 0u };
                if (bI < n) b = cur[bI];
                const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
                const double tlo = dy_lo(b.tn, tk);
                const bool act = bI < n && tlo < toi_skip && tlo < t_prune;
                const double tv = ci ? dy_hi(b.tn, tk) : tlo;
                const double uv = cj ? dy_hi(b.un, uk) : dy_lo(b.un, uk);
                const double vv = cl ? dy_hi(b.vn, vk) : dy_lo(b.vn, vk);
                bool excl = false, inside = true, tolc = true;
                double tmax = 0.0;
#pragma unroll
                for (int cc = 0; cc < 3; ++cc) {
                    double pp[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) pp[k] = (P.x1[3 * k + cc] - P.x0[3 * k + cc]) * tv + P.x0[3 * k + cc];
                    double f;
                    if (VF) {
                        const double pt = ((pp[2] - pp[1]) * uv + (pp[3] - pp[1]) * vv) + pp[1];
                        f = pp[0] - pt;
                    }
                    else {
                        const double pa = (pp[1] - pp[0]) * uv + pp[0];
                        const double pb = (pp[3] - pp[2]) * vv + pp[2];
                        f = pa - pb;
                    }
                    double mn = f, mx = f;
#pragma unroll
                    for (int o = 1; o < 8; o <<= 1) {
                        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                    }
                    const double e = err[cc] + ms;
                    const double tt = mx - mn;
                    excl = excl || (mn > e || mx < -e);
                    inside = inside && (mn >= -e && mx <= e);
                    tolc = tolc && !(tt > co_tol);
                    tmax = (cc == 0) ? tt : fmax(tmax, tt);
                }
                unsigned flags = 0;
                if (act && !excl) { // the co-domain box contains the origin
                    flags = F_ZERO;
                    const bool cond1 = pow2neg(tk) <= tol[0] && pow2neg(uk) <= tol[1] && pow2neg(vk) <= tol[2];
                    const Key3 key = { tlo, dy_lo(b.un, uk), dy_lo(b.vn, vk) };
                    const bool flagged = tolc || inside || cond1;
                    if (key_less(key, gk1)) { gk1 = key; gp1 = flagged ? 1u : 0u; ga1 = tmax; }
                    if (flagged && key_less(key, gk2)) { gk2 = key; gp2 = cond1 ? 1u : 0u; }
                }
                visited += __popc(__ballot_sync(0xffffffffu, act && corner == 0));
                if (bI < n && corner == 0) cur[bI].kk = (b.kk & 0x00ffffffu) | flags;
            }
#pragma unroll
            for (int o = 8; o <= 16; o <<= 1) { // merge the four groups (all lanes of a group hold the same candidates)
                Key3 r1, r2;
                r1.t = __shfl_xor_sync(0xffffffffu, gk1.t, o); r1.u = __shfl_xor_sync(0xffffffffu, gk1.u, o); r1.v = __shfl_xor_sync(0xffffffffu, gk1.v, o);
                r2.t = __shfl_xor_sync(0xffffffffu, gk2.t, o); r2.u = __shfl_xor_sync(0xffffffffu, gk2.u, o); r2.v = __shfl_xor_sync(0xffffffffu, gk2.v, o);
                const unsigned rp1 = __shfl_xor_sync(0xffffffffu, gp1, o), rp2 = __shfl_xor_sync(0xffffffffu, gp2, o);
                const double ra1 = __shfl_xor_sync(0xffffffffu, ga1, o);
                if (key_less(r1, gk1)) { gk1 = r1; gp1 = rp1; ga1 = ra1; }
                if (key_less(r2, gk2)) { gk2 = r2; gp2 = rp2; }
            }
            (void)ga2;
            k1 = gk1; p1 = gp1; a1max = ga1;
            k2 = gk2; p2 = gp2;
        }
        __syncwarp();
        if (k1.t == INF) break; // search space exhausted
        if (p1 & 1u) { toi = k1.t; return 1; }
        const bool has_k2 = k2.t != INF;
        if (has_k2 && (p2 & 1u)) { toi = k2.t; return 1; }
        boxes += (unsigned)visited;
        if (max_itr > 0) {
            temp_toi = k1.t;
            temp_out_tol = fmax(a1max, co_tol);
            refine += visited;
            if (refine > max_itr) {
                if (lane == 0) atomicAdd(warn, 1);
                toi = temp_toi;
                out_tol = temp_out_tol;
                return 1;
            }
        }
        if (has_k2) {
            if (k2.t < toi_skip) toi_skip = k2.t;
            use_skip = true;
        }
        int nn = 0;
        { // split pass, one box per lane (levels of the warp-level pass never exceed a few dozen boxes before the box-parallel switch)
            bool over = false, deep = false;
            for (int base = 0; base < n; base += 32) {
                const int i = base + lane;
                int nchild = 0;
                DBox c0, c1;
                if (i < n) {
                    const DBox b = cur[i];
                    if (b.kk & F_ZERO) {
                        const int tk = b.kk & 0xff, uk = (b.kk >> 8) & 0xff, vk = (b.kk >> 16) & 0xff;
                        const Key3 key = { dy_lo(b.tn, tk), dy_lo(b.un, uk), dy_lo(b.vn, vk) };
                        if (!has_k2 || key_less(key, k2)) {
                            const double w[3] = { pow2neg(tk), pow2neg(uk), pow2neg(vk) };
                            int split = -1;
                            double best = -1.0;
#pragma unroll
                            for (int d = 0; d < 3; ++d)
                                if (w[d] > tol[d]) {
                                    const double r = inv_tol[d] * w[d]; // = w[d] / tol[d] bit for bit: w[d] is a power of two (see ti_ccd)
                                    if (r > best) { best = r; split = d; }
                                }
                            const int pk = split == 0 ? tk : (split == 1 ? uk : vk);
                            if (split < 0 || pk >= 60) deep = true;
                            else {
                                const unsigned long long pn = split == 0 ? b.tn : (split == 1 ? b.un : b.vn);
#pragma unroll
                                for (int half = 0; half < 2; ++half) {
                                    const unsigned long long hn = 2 * pn + half;
                                    const int hk = pk + 1;
                                    bool keep = true;
                                    if (split == 0) { if (check_t) keep = !(dy_hi(hn, hk) < 0.0 || dy_lo(hn, hk) > max_t); }
                                    else if (VF) keep = (split == 1) ? sum_le_1(hn, hk, b.vn, vk) : sum_le_1(hn, hk, b.un, uk);
                                    if (keep) {
                                        DBox ch = b;
                                        ch.kk &= 0x00ffffffu;
                                        if (split == 0) { ch.tn = hn; ch.kk = (ch.kk & ~0xffu) | (unsigned)hk; }
                                        else if (split == 1) { ch.un = hn; ch.kk = (ch.kk & ~0xff00u) | ((unsigned)hk << 8); }
                                        else { ch.vn = hn; ch.kk = (ch.kk & ~0xff0000u) | ((unsigned)hk << 16); }
                                        if (nchild == 0) c0 = ch;
                                        else c1 = ch;
                                        ++nchild;
                                    }
                                }
                            }
                        }
                    }
                }
                const int incl = warp_incl_scan(nchild, lane), total = __shfl_sync(0xffffffffu, incl, 31);
                const int off = nn + incl - nchild;
                if (nn + total > kSmemLevel) over = true;
                else {
                    if (nchild > 0) nxt[off] = c0;
                    if (nchild > 1) nxt[off + 1] = c1;
                }
                nn += total;
                if (__any_sync(0xffffffffu, over || deep)) break;
            }
            if (__any_sync(0xffffffffu, deep)) {
                if (lane == 0) atomicAdd(warn, 1);
                toi = temp_toi;
                out_tol = temp_out_tol;
                return 1;
            }
            if (__any_sync(0xffffffffu, over)) return -1;
        }
        __syncwarp();
        DBox* t = cur; cur = nxt; nxt = t;
        n = nn;
    }
    if (use_skip) { toi = toi_skip; return 1; }
    return 0;
}

// out-of-line instances for the warp-level pass.  Round 2, second half: ncu on k_ti_stage2 showed "no instruction" as the largest stall
// (3.4 per issued instruction): 16 K SASS instructions -- VF and EE template copies of both root finders, each inlined at two call sites
// (first run and ms = 0 retry) -- with four warps per CTA at unrelated program counters.  VF / EE is now a run-time flag tested inside the
// corner evaluation (a few instructions differ), the retry is a second trip through ONE call site, and the split rule multiplies by exact
// reciprocals instead of dividing (below): one copy of each root finder.
__device__ __noinline__ int ti_root_finder_cp_call(bool vf, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err, double ms,
    int max_itr, DBox* sA, DBox* sB, int lane, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes, const unsigned long long* best)
{
    return ti_root_finder_cp(vf, P, tol, inv_tol, co_tol, max_t, err, ms, max_itr, sA, sB, lane, toi, out_tol, warn, boxes, best);
}
__device__ __noinline__ int ti_root_finder_warp_call(bool vf, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err, double ms,
    int max_itr, DBox* bufA, DBox* bufB, int cap, int lane, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes,
    const unsigned long long* best)
{
    return ti_root_finder(vf, P, tol, inv_tol, co_tol, max_t, err, ms, max_itr, bufA, bufB, cap, lane, toi, out_tol, warn, boxes, best);
}

// A search that outgrows the per-warp level buffers runs again in the context's overflow arena (two levels of kArenaLevel boxes), which one
// warp holds at a time: such searches are rare, and the library itself runs them to max_itr.  The arena run does not prune against the
// running minimum, so its count of evaluated boxes -- and with it the max_itr exit -- is the library's own.
__device__ __noinline__ int ti_root_finder_arena(bool vf, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err,
    double ms, int max_itr, DBox* arena, int* arena_lock, int lane, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes)
{
    if (lane == 0) {
        while (atomicCAS(arena_lock, 0, 1) != 0) __nanosleep(1000);
        __threadfence();
    }
    __syncwarp();
    int rc = ti_root_finder_warp_call(vf, P, tol, inv_tol, co_tol, max_t, err, ms, max_itr, arena, arena + kArenaLevel, kArenaLevel, lane, toi, out_tol, warn, boxes, nullptr);
    __syncwarp();
    if (lane == 0) {
        __threadfence();
        atomicExch(arena_lock, 0);
    }
    if (rc == -1) { // cannot happen (see kArenaLevel); keep the conservative estimate and report it
        if (lane == 0) atomicAdd(warn, 1);
        rc = 1;
    }
    return rc;
}

// vertexFaceCCD_double / edgeEdgeCCD_double including the no_zero_toi refinement loop; returns 0 / 1.  The corner-parallel root finder runs
// in the shared-memory level buffers sA / sB; a search that outgrows them restarts box-parallel in the global buffers bufA / bufB, and one
// that outgrows those in the overflow arena.
__device__ int ti_ccd(bool vf, const TiPair& P, const double* err, double ms, double tolerance, double t_max, int max_itr, DBox* bufA, DBox* bufB, int cap, int lane,
    double& toi, int* __restrict__ warn, unsigned long long& boxes, DBox* sA, DBox* sB, const unsigned long long* best, DBox* arena, int* arena_lock)
{
    double tolerance_in = tolerance, ms_in = ms, out_tol = tolerance;
    bool is_impacting = false, tmp = false;
    unsigned iter = 0;
    do {
        double tol[3], inv_tol[3];
        width_tolerances(vf, P, tolerance_in, tol);
        // The split rule compares width / tolerance per axis.  Every width is a power of two, and x -> x * 2^-k commutes with rounding
        // (no overflow / underflow here: tolerances are ~1e-9 .. 1e-3 or inf for a static axis), so 2^-k / tol == (1 / tol) * 2^-k bit
        // for bit: one division per axis and search instead of three per box.
#pragma unroll
        for (int d = 0; d < 3; ++d) inv_tol[d] = 1.0 / tol[d];
        int rc = ti_root_finder_cp_call(vf, P, tol, inv_tol, tolerance_in, t_max, err, ms_in, max_itr, sA, sB, lane, toi, out_tol, warn, boxes, best);
        if (rc == -1) rc = ti_root_finder_warp_call(vf, P, tol, inv_tol, tolerance_in, t_max, err, ms_in, max_itr, bufA, bufB, cap, lane, toi, out_tol, warn, boxes, best);
        if (rc == -1) rc = ti_root_finder_arena(vf, P, tol, inv_tol, tolerance_in, t_max, err, ms_in, max_itr, arena, arena_lock, lane, toi, out_tol, warn, boxes);
        tmp = rc == 1;
        if (iter == 0) is_impacting = tmp;
        else toi = tmp ? toi : t_max;
        if (tmp && toi == 0.0) {
            if (out_tol > tolerance_in) t_max *= 0.9;
            else if (10 * tolerance_in < ms_in) ms_in *= 0.5;
            else tolerance_in *= 0.1;
        }
        ++iter;
    } while (iter < 0x7fffffffu && tmp && toi == 0.0);
    return is_impacting ? 1 : 0;
}

// one candidate end to end (SelfCollisionHandler.cpp:740-790): 0 / 1 (toi set)
__device__ int pair_ccd(bool vf, const TiPair& P, const NarrowArgs& a, DBox* bufA, DBox* bufB, int cap, int lane, double& toi, int* __restrict__ warn, unsigned long long& boxes,
    DBox* sA, DBox* sB)
{
    const double d = pair_distance_sqrt(vf, P);
    const double max_t = a.st->max_t;                 // canonical semantics: every pair sees the step on entry (SURVEY 8a row 10)
    const double* err = vf_metric(vf, P) ? a.err_vf : a.err_ee;
    int hit = 0;
    // first trip: ms = min(0.2 d, 1e-6), pruned against the running device-wide minimum; second trip (:759-781, only after a hit with
    // toi < 1e-6): ms = 0, result scaled by 0.8 and NOT pruned -- a box starting in [best, 1.25 best) can still lower the global step
    // (the exactness argument of ti_root_finder only covers unscaled results).  One call site for both.
#pragma unroll 1
    for (int attempt = 0; attempt < 2; ++attempt) {
        const double ms = attempt ? 0.0 : fmin(0.2 * d, 1e-6);
        const unsigned long long* best = attempt ? nullptr : &a.st->ccd_ord;
        hit = ti_ccd(vf, P, err, ms, a.tol, max_t, a.max_itr, bufA, bufB, cap, lane, toi, warn, boxes, sA, sB, best, a.arena, a.arena_lock);
        if (attempt == 1) {
            if (hit) toi *= 0.8;
            break;
        }
        if (!(hit && toi < 1e-6)) break;
    }
    return hit;
}

// ------------------------------------------------------------------------------------------------------------------
// Thread pass with LANE-LEVEL REFILL (round 2, second half).  With one pair per lane and grid-stride round, ncu showed 7.4 of 32 lanes active per issued instruction -- a lane whose
// search ended after two boxes waited for the lane of its warp that used its whole 24-box budget.  Here the search is a resumable state
// machine: one loop iteration = ONE LEVEL of one lane's breadth-first search (the body of ti_root_finder's level loop, same arithmetic, same
// decisions); a lane whose pair is finished takes the next survivor from a work counter in the same iteration.  The no_zero_toi loop of
// ti_ccd and the ms = 0 retry of pair_ccd are states of the same machine.
// ------------------------------------------------------------------------------------------------------------------
struct Bfs1 {
    DBox* cur;
    DBox* nxt;
    int n;
    double toi_skip;
    bool use_skip;
    long long refine;
    double temp_toi, temp_out_tol;
    unsigned long long bo_cur;
};
DEV void bfs1_init(Bfs1& b, DBox* bufA, DBox* bufB, double co_tol, const unsigned long long* best)
{
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    b.cur = bufA; b.nxt = bufB;
    b.cur[0] = DBox{ 0ull, 0ull, 0ull, 0u, 0u };
    b.n = 1;
    b.toi_skip = INF; b.use_skip = false; b.refine = 0;
    b.temp_toi = INF; b.temp_out_tol = co_tol;
    b.bo_cur = best ? *reinterpret_cast<const volatile unsigned long long*>(best) : 0ull;
}
// one level of the thread pass (ti_root_finder's level loop run by one lane): 0 no collision, 1 collision (toi set), 2 deferred, 3 go on
// with the next level
DEV int bfs1_level(bool VF, const TiPair& P, const double* tol, const double* inv_tol, double co_tol, double max_t, const double* err, double ms, int max_itr,
    int cap, long long thread_budget, const unsigned long long* best, Bfs1& b, double& toi, double& out_tol, int* __restrict__ warn, unsigned long long& boxes)
{
    const bool check_t = (max_t != 1.0);
    const double INF = __longlong_as_double(0x7ff0000000000000ll);
    double t_prune = INF;
    if (best) {
        t_prune = fmax(ord_to_dbl(b.bo_cur), 1e-6);
        b.bo_cur = *reinterpret_cast<const volatile unsigned long long*>(best);
    }
    Key3 k1 = { INF, INF, INF }, k2 = { INF, INF, INF };
    unsigned p1 = 0, p2 = 0;
    double a1 = 0.0;
    int visited = 0;
    for (int i = 0; i < b.n; ++i) {
        DBox bx = b.cur[i];
        const int tk = bx.kk & 0xff, uk = (bx.kk >> 8) & 0xff, vk = (bx.kk >> 16) & 0xff;
        const double tlo = dy_lo(bx.tn, tk);
        unsigned flags = 0;
        if (tlo < b.toi_skip && tlo < t_prune) {
            ++visited;
            bool box_in;
            double tt[3];
            if (origin_in_box(VF, P, bx, err, ms, box_in, tt)) {
                flags = F_ZERO;
                const bool tol_cond = tt[0] <= co_tol && tt[1] <= co_tol && tt[2] <= co_tol;
                const bool cond1 = pow2neg(tk) <= tol[0] && pow2neg(uk) <= tol[1] && pow2neg(vk) <= tol[2];
                const Key3 key = { tlo, dy_lo(bx.un, uk), dy_lo(bx.vn, vk) };
                const unsigned mp1 = (tol_cond || box_in || cond1) ? 1u : 0u;
                if (key_less(key, k1)) { k1 = key; p1 = mp1; a1 = fmax(fmax(tt[0], tt[1]), tt[2]); }
                if (mp1 && key_less(key, k2)) { k2 = key; p2 = cond1 ? 1u : 0u; }
            }
        }
        b.cur[i].kk = (bx.kk & 0x00ffffffu) | flags;
    }
    if (k1.t == INF) { // nothing at this level contains the origin: the search space is exhausted
        if (b.use_skip) { toi = b.toi_skip; return 1; }
        return 0;
    }
    if (p1 & 1u) { toi = k1.t; return 1; }
    const bool has_k2 = k2.t != INF;
    if (has_k2 && (p2 & 1u)) { toi = k2.t; return 1; }
    boxes += (unsigned)visited; // diagnostics: boxes evaluated by the thread pass
    if (b.refine + visited > thread_budget) return 2; // over budget: handed to the warp pass
    if (max_itr > 0) {
        b.temp_toi = k1.t;
        b.temp_out_tol = fmax(a1, co_tol);
        b.refine += visited;
        if (b.refine > max_itr) {
            atomicAdd(warn, 1);
            toi = b.temp_toi;
            out_tol = b.temp_out_tol;
            return 1;
        }
    }
    if (has_k2) {
        if (k2.t < b.toi_skip) b.toi_skip = k2.t;
        b.use_skip = true;
    }
    int nn = 0;
    for (int i = 0; i < b.n; ++i) {
        const DBox bx = b.cur[i];
        if (!(bx.kk & F_ZERO)) continue;
        const int tk = bx.kk & 0xff, uk = (bx.kk >> 8) & 0xff, vk = (bx.kk >> 16) & 0xff;
        const Key3 key = { dy_lo(bx.tn, tk), dy_lo(bx.un, uk), dy_lo(bx.vn, vk) };
        if (has_k2 && !key_less(key, k2)) continue;
        const double w[3] = { pow2neg(tk), pow2neg(uk), pow2neg(vk) };
        int split = -1;
        double bestr = -1.0;
#pragma unroll
        for (int d = 0; d < 3; ++d)
            if (w[d] > tol[d]) {
                const double r = inv_tol[d] * w[d]; // = w[d] / tol[d] bit for bit (see ti_ccd)
                if (r > bestr) { bestr = r; split = d; }
            }
        const int pk = split == 0 ? tk : (split == 1 ? uk : vk);
        if (split < 0 || pk >= 60) return 2; // bisection overflow: the warp pass handles it like the iteration overflow
        const unsigned long long pn = split == 0 ? bx.tn : (split == 1 ? bx.un : bx.vn);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const unsigned long long hn = 2 * pn + half;
            const int hk = pk + 1;
            bool keep = true;
            if (split == 0) { if (check_t) keep = !(dy_hi(hn, hk) < 0.0 || dy_lo(hn, hk) > max_t); }
            else if (VF) keep = (split == 1) ? sum_le_1(hn, hk, bx.vn, vk) : sum_le_1(hn, hk, bx.un, uk);
            if (keep) {
                if (nn >= cap) return 2; // the level outgrew the buffer
                DBox c = bx;
                c.kk &= 0x00ffffffu;
                if (split == 0) { c.tn = hn; c.kk = (c.kk & ~0xffu) | (unsigned)hk; }
                else if (split == 1) { c.un = hn; c.kk = (c.kk & ~0xff00u) | ((unsigned)hk << 8); }
                else { c.vn = hn; c.kk = (c.kk & ~0xff0000u) | ((unsigned)hk << 16); }
                b.nxt[nn++] = c;
            }
        }
    }
    DBox* t = b.cur; b.cur = b.nxt; b.nxt = t;
    b.n = nn;
    if (nn == 0) {
        if (b.use_skip) { toi = b.toi_skip; return 1; }
        return 0;
    }
    return 3;
}

constexpr int kThreadLevel = 8;  // boxes per level buffer of a lane of the thread pass (2 buffers per lane, in shared memory)
// idle lanes of a warp refill together once this many are idle (H100 SXM, 400 W, C5: batch 1 / 8 / 16 / 32 -> 1.06 / 1.05 / 1.03 / 1.03 ms;
// again with the box counter in registers, 700 W, budget 64, iteration ms: 8 / 16 / 32 -> 2.54 / 2.52 / 2.53)
constexpr int kRefillBatch = 16;
__global__ void __launch_bounds__(128, 2) k_ti_stage15_refill(NarrowArgs a, const unsigned* __restrict__ survivors, const unsigned* __restrict__ nSurvPtr, unsigned* __restrict__ work,
    unsigned* __restrict__ deferred, unsigned* __restrict__ nDeferred, long long budget, unsigned long long* __restrict__ min_ord, int* __restrict__ warn)
{
    extern __shared__ __align__(16) unsigned char s_lvl[];
    constexpr int kSlab = kThreadLevel * (int)sizeof(DBox) + 8;
    DBox* bufA = reinterpret_cast<DBox*>(s_lvl + (size_t)threadIdx.x * kSlab);
    DBox* bufB = reinterpret_cast<DBox*>(s_lvl + (size_t)(blockDim.x + threadIdx.x) * kSlab);
    const unsigned nSurv = *nSurvPtr;
    const double max_t0 = a.st->max_t;
    const unsigned long long* best0 = &a.st->ccd_ord;
    const int lane = threadIdx.x & 31;
    // per-lane state of pair_ccd / ti_ccd / the root finder
    bool busy = false, vf = false;
    unsigned idx = 0;
    TiPair P;
    Bfs1 bf;
    int attempt = 0;
    unsigned iter = 0;
    bool is_impacting = false;
    double dist = 0.0, ms_in = 0.0, tolerance_in = 0.0, t_max = 0.0, out_tol = 0.0, toi = 0.0;
    double tol[3] = { 0, 0, 0 }, inv_tol[3] = { 0, 0, 0 };
    const double* err = a.err_vf;
    const unsigned long long* best = nullptr;
    bool drained = false;
    // diagnostics: the boxes this lane evaluated over all its searches.  A count per lane and one atomic per warp when it leaves: an add to
    // the pass's single counter at every level of every search was a serial chain of same-address reductions on one L2 slice.
    unsigned long long boxes = 0;
    for (;;) {
        // Refill in batches: fetching a pair is two dependent rounds of global loads (candidate -> vertex ids -> positions, directions), and the
        // whole warp waits for them -- refilling whenever any lane is idle made every iteration pay that latency (ncu: long scoreboard 3.0 per
        // issued instruction).  Lanes wait until kRefillBatch of them are idle (or nothing is running).
        __syncwarp();
        const unsigned idle_m = __ballot_sync(0xffffffffu, !busy && !drained);
        const bool refill_now = __popc(idle_m) >= kRefillBatch || __ballot_sync(0xffffffffu, busy) == 0u;
        if (!busy && !drained && refill_now) { // take the next survivor (one atomic per warp and round)
            const unsigned m = __activemask();
            const int leader = __ffs(m) - 1;
            unsigned base = 0;
            if (lane == leader) base = atomicAdd(work, (unsigned)__popc(m));
            base = __shfl_sync(m, base, leader);
            const unsigned w = base + __popc(m & ((1u << lane) - 1u));
            if (w < nSurv) {
                idx = survivors[w];
                int v[4];
                load_pair(a.s, a.dir, a.cand[idx], vf, v, P);
                err = vf_metric(vf, P) ? a.err_vf : a.err_ee;
                dist = pair_distance_sqrt(vf, P);
                attempt = 0;
                // ti_ccd entry state of the first trip (pair_ccd): ms = min(0.2 d, 1e-6), pruned against the running minimum
                ms_in = fmin(0.2 * dist, 1e-6); tolerance_in = a.tol; t_max = max_t0; out_tol = a.tol; iter = 0; is_impacting = false; best = best0;
                width_tolerances(vf, P, tolerance_in, tol);
#pragma unroll
                for (int d = 0; d < 3; ++d) inv_tol[d] = 1.0 / tol[d];
                bfs1_init(bf, bufA, bufB, tolerance_in, best);
                out_tol = tolerance_in;
                busy = true;
            }
            else drained = true;
        }
        __syncwarp();
        if (__all_sync(0xffffffffu, !busy)) { // the lanes of a warp leave together: all idle and the list exhausted
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) boxes += __shfl_xor_sync(0xffffffffu, boxes, o);
            if (lane == 0 && boxes) atomicAdd(reinterpret_cast<unsigned long long*>(warn + 5), boxes);
            break;
        }
        if (busy) {
            const int rc = bfs1_level(vf, P, tol, inv_tol, tolerance_in, t_max, err, ms_in, a.max_itr, kThreadLevel, budget, best, bf, toi, out_tol, warn, boxes);
            if (rc != 3) {
                bool restart = false, finished = false;
                int hit = 0;
                if (rc == 2) { deferred[atomicAdd(nDeferred, 1u)] = idx; finished = true; }
                else { // ti_ccd: the no_zero_toi refinement loop around the root finder
                    const bool tmp = rc == 1;
                    if (iter == 0) is_impacting = tmp;
                    else toi = tmp ? toi : t_max;
                    if (tmp && toi == 0.0) {
                        if (out_tol > tolerance_in) t_max *= 0.9;
                        else if (10 * tolerance_in < ms_in) ms_in *= 0.5;
                        else tolerance_in *= 0.1;
                        ++iter;
                        restart = true;
                    }
                    else {
                        hit = is_impacting ? 1 : 0;
                        // pair_ccd: second trip (:759-781) only after a hit with toi < 1e-6: ms = 0, not pruned, result scaled by 0.8
                        if (attempt == 0 && hit && toi < 1e-6) {
                            attempt = 1;
                            ms_in = 0.0; tolerance_in = a.tol; t_max = max_t0; iter = 0; is_impacting = false; best = nullptr;
                            restart = true;
                        }
                        else {
                            if (attempt == 1 && hit) toi *= 0.8;
                            finished = true;
                        }
                    }
                }
                if (restart) {
                    width_tolerances(vf, P, tolerance_in, tol);
#pragma unroll
                    for (int d = 0; d < 3; ++d) inv_tol[d] = 1.0 / tol[d];
                    bfs1_init(bf, bufA, bufB, tolerance_in, best);
                    out_tol = tolerance_in;
                }
                if (finished) {
                    if (hit == 1) atomicMin(min_ord, dbl_to_ord(toi));
                    busy = false;
                }
            }
        }
    }
}

__global__ void __launch_bounds__(128, 2) k_ti_stage2(NarrowArgs a, const unsigned* __restrict__ survivors, const unsigned* __restrict__ nSurvPtr, unsigned* __restrict__ work,
    DBox* __restrict__ scratch, int cap, unsigned long long* __restrict__ min_ord, int* __restrict__ warn)
{
    __shared__ DBox sLevels[kStage2WarpsPerCtaDev][2][kSmemLevel];
    __shared__ TiPair sPair[kStage2WarpsPerCtaDev];
    const int lane = threadIdx.x & 31;
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    DBox* sA = sLevels[threadIdx.x >> 5][0];
    DBox* sB = sLevels[threadIdx.x >> 5][1];
    DBox* bufA = scratch + (size_t)warp_global * 2 * cap;
    DBox* bufB = bufA + cap;
    const unsigned nSurv = *nSurvPtr;
    // diagnostics: the boxes this warp's searches evaluated (the same count on every lane), added to the pass's total once, when the warp leaves
    unsigned long long boxes = 0;
    for (;;) {
        unsigned w = 0;
        if (lane == 0) w = atomicAdd(work, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
        if (w >= nSurv) {
            if (lane == 0 && boxes) atomicAdd(reinterpret_cast<unsigned long long*>(warn + 7), boxes);
            break;
        }
        bool vf;
        {
            // the pair's 24 coordinates live in shared memory: the warp-level search only needs them 8 at a time per lane
            int v[4];
            TiPair Pl;
            load_pair(a.s, a.dir, a.cand[survivors[w]], vf, v, Pl);
            if (lane == 0) sPair[threadIdx.x >> 5] = Pl;
            __syncwarp();
        }
        const TiPair& P = sPair[threadIdx.x >> 5];
        double toi;
        const long long t0 = clock64();
        const int hit = pair_ccd(vf, P, a, bufA, bufB, cap, lane, toi, warn, boxes, sA, sB);
        if (hit && lane == 0) atomicMin(min_ord, dbl_to_ord(toi));
        if (lane == 0) { // diagnostics: the longest pair bounds this pass from below
            const unsigned dt = (unsigned)((clock64() - t0) >> 6);
            atomicMax(reinterpret_cast<unsigned*>(warn + 3), dt);
            atomicAdd(reinterpret_cast<unsigned*>(warn + 4), dt);
        }
        __syncwarp();
    }
}

// start of a narrow phase: snapshot the device-resident step as max_t and as the initial running minimum, fix this rank's slice of the
// candidate list (n32 / n64: the list size, wherever the producing stage left it), clear the per-phase counters
__global__ void k_ccd_init(IterState* st, const int* __restrict__ n32, const unsigned long long* __restrict__ n64, unsigned long long cap, int rank, int nranks, int share,
    double seed, unsigned* nSurv, unsigned* work, int* flags)
{
    if (threadIdx.x != 0) return;
    const double alpha = ord_to_dbl(st->step_ord);
    st->max_t = alpha;
    st->ccd_ord = (seed >= 0.0 && seed < alpha) ? dbl_to_ord(seed) : st->step_ord; // (seed: test hook, ipcgpu_ccd_debug_seed_bound)
    unsigned long long n = n32 ? (unsigned long long)max(*n32, 0) : *n64;
    if (n > cap) n = cap; // an overflowing producer raised its capacity flag; stay inside the list
    st->cand_range[0] = share ? n * rank / nranks : 0ull;
    st->cand_range[1] = share ? n * (rank + 1) / nranks : n;
    *nSurv = 0;
    *work = 0;
    for (int q = 0; q < 12; ++q) flags[q] = 0; // zero distance, warnings, deferred count, pad, boxes(thread pass) x2, boxes(warp pass) x2
}
// end of a narrow phase (this rank): a zero initial distance forces the step to 0 (:730-737); diagnostics go to the iteration state
__global__ void k_ccd_finish(IterState* st, const unsigned* __restrict__ nSurv, const int* __restrict__ flags, const int* __restrict__ overflow, int is_full)
{
    if (threadIdx.x != 0) return;
    if (flags[0]) {
        st->ccd_ord = 0ull;
        st->flags[FLAG_ZERO_CCD_DISTANCE] = 1;
    }
    if (overflow && *overflow) st->flags[FLAG_CCD_CAPACITY] = 1;
    st->flags[FLAG_TI_WARNINGS] += flags[1];
    st->ccd_stats[0] = *nSurv;
    st->ccd_stats[1] = (unsigned long long)flags[1];
    st->ccd_stats[2] = (unsigned)flags[2];
    st->ccd_stats[3] = (unsigned long long)(unsigned)flags[4] << 6;
    st->ccd_stats[4] = (unsigned long long)(unsigned)flags[5] << 6;
    st->ccd_stats[5] = *reinterpret_cast<const unsigned long long*>(flags + 6);
    st->ccd_stats[6] = *reinterpret_cast<const unsigned long long*>(flags + 8);
    st->ccd_stats[7] = st->cand_range[1] - st->cand_range[0];
    if (is_full) st->n_full_cand = st->ccd_stats[7];
}
// after the cross-rank min: the narrow phase's minimum becomes the step
__global__ void k_ccd_commit(IterState* st, int stage)
{
    if (threadIdx.x != 0) return;
    st->step_ord = st->ccd_ord;
    st->alpha_stage[stage] = ord_to_dbl(st->ccd_ord);
}

} // namespace ipcgpu

using namespace ipcgpu;


constexpr int kStage2WarpsPerCta = 4;
// persistent: 2 CTAs x 4 warps per SM, compiled for 2 CTAs per SM (230 registers, no spill; for 3 per SM it spilled 226 B per thread).  Fewer
// warps of this pass per SM leave room for the derivative chain that runs next to it (H100 SXM, 700 W, C5, iteration ms with budget 32:
// 1 CTA per SM 3.19, 2 -> 3.15, 3 -> 3.16; 6 CTAs of the 3-per-SM build 3.21)
constexpr int kStage2Ctas = kSMs * 2;
constexpr int kLevelCap = 4096;      // boxes per BFS level buffer (2 buffers per warp)

int ccd_alloc(ipcgpu_ctx* ctx)
{
    CcdWork& w = ctx->ccd;
    const size_t warps = (size_t)kStage2Ctas * kStage2WarpsPerCta;
    // swept grid: at most 8 entries per primitive (k_swept_cells), a dense table of kGridCells cells per primitive type
    const size_t nEnt = (size_t)8 * std::max(ctx->nSF + ctx->nSE + ctx->nSV, 1);
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, (int)(3 * kGridCells + 1));
    if (!w.arena_lock.p) {
        if (!w.arena_lock.reserve(1) || cudaMemsetAsync(w.arena_lock.p, 0, sizeof(int), ctx->stream) != cudaSuccess) {
            ctx->err = "CCD workspace allocation failed";
            return IPCGPU_ERR_CUDA;
        }
    }
    bool ok = w.arena.reserve((size_t)2 * kArenaLevel * sizeof(DBox)) && w.vmin.reserve((size_t)3 * ctx->nV) && w.vmax.reserve((size_t)3 * ctx->nV) && w.cand.reserve(ctx->ccd_capacity) && w.surv.reserve(ctx->ccd_capacity) && w.surv2.reserve(ctx->ccd_capacity)
        && w.scratch.reserve(warps * 2 * kLevelCap * sizeof(DBox)) && w.counters.reserve(16) && w.ncand.reserve(2) && w.bounds.reserve(8) && w.cells.reserve(1)
        && w.sw_keys.reserve(nEnt) && w.sw_ent.reserve(nEnt) && w.sw_cnt.reserve((size_t)3 * kGridCells + 1) && w.sw_off.reserve((size_t)3 * kGridCells + 1)
        && w.sw_tmp.reserve(scan_bytes + 256);
    if (!ok) {
        ctx->err = "CCD workspace allocation failed";
        return IPCGPU_ERR_CUDA;
    }
    return 0;
}

// Narrow phase over a device-resident candidate list.  The step is read from and written back to the device-resident iteration state
// (IterState::step_ord): nothing is read back here.  n32 / n64: device-resident list size; share: walk only this rank's contiguous
// slice of the list (replicated lists) or all of it (lists that are already this rank's own); stage: 1 = partial, 3 = full CCD.
int ccd_narrow(ipcgpu_ctx* ctx, const int2* cand, const int* n32, const unsigned long long* n64, unsigned long long cap, int share, double tol, const double* err_vf,
    const double* err_ee, int stage, const int* overflow)
{
    CcdWork& w = ctx->ccd;
    cudaStream_t st = ctx->stream;
    NarrowArgs a;
    a.s = surf_args(ctx);
    a.dir = ctx->dir.p;
    a.cand = cand;
    for (int c = 0; c < 3; ++c) { a.err_vf[c] = err_vf[c]; a.err_ee[c] = err_ee[c]; }
    a.tol = tol;
    a.max_itr = 1000000;    // TIGHT_INCLUSION_MAX_ITER (CCDUtils.hpp:14)
    a.st = ctx->iter.p;
    a.arena = reinterpret_cast<DBox*>(w.arena.p);
    a.arena_lock = w.arena_lock.p;
    IterState* ist = ctx->iter.p;
    unsigned* nSurv = reinterpret_cast<unsigned*>(w.counters.p);
    unsigned* work = nSurv + 1;
    int* flags = w.counters.p + 2; // [0] zero distance, [1] warnings, [2] deferred, [3] pass A's work counter, [4] longest, [5] total cycles, [6..7] / [8..9] boxes
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_CCD_NARROW);
    k_ccd_init<<<1, 32, 0, st>>>(ist, n32, n64, cap, ctx->rank, ctx->nranks, share, ctx->debug_prune_seed, nSurv, work, flags);
    {
        // the candidate count lives on the device: every pass is a grid-stride / persistent kernel that reads it there
        // pass 1 (thread per candidate): the root box only;
        // pass A (thread per survivor, box budget): the shallow majority dies here without holding its warp hostage;
        // pass B (warp per pair, corner-parallel box evaluation): the deep searches, compacted.
        // (measured slower or wrong, and deleted: a three-tier split -- 3-box, then 12-box thread passes; an 8-lanes-per-pair group pass between
        // A and B, or instead of A; both passes fused into one persistent kernel that starts the deep searches while the thread pass still runs:
        // DESIGN.md §3.1, §7)
        cudaEvent_t pe1 = ctx->prof_begin(IPCGPU_STAGE_CCD_ROOT_FILTER);
        k_ti_stage1<<<kSMs * 16, 128, 0, st>>>(a, w.surv.p, nSurv, flags);
        ctx->prof_end(pe1);
        unsigned* nDefA = reinterpret_cast<unsigned*>(flags + 2);
        unsigned* refill_work = reinterpret_cast<unsigned*>(flags + 3);
        // pass A (thread per survivor): the shallow majority (2-3 boxes) at 32 pairs per warp; pass B (warp per pair): the searches pass A hands on.
        // boxes a thread may evaluate before it hands its pair on (H100 SXM, 700 W, C5, iteration ms with the box counters in registers: 24 -> 2.64
        // (2,871 pairs handed on in the full CCD), 32 -> 2.58 (950), 48 -> 2.55, 64 -> 2.52 (444), 96 -> 2.49 (440), 128 -> 2.50; the eager narrow
        // phase grows from 0.79 to 0.90 ms between 32 and 96, the iteration gains because the shorter warp pass leaves the SMs to the derivative
        // chain sooner).  The test hook ipcgpu_ccd_debug_thread_budget overrides it.
        constexpr long long kThreadBudget = 96;
        const long long budget = ctx->debug_ti_budget >= 0 ? ctx->debug_ti_budget : kThreadBudget;
        constexpr int bytes = 2 * 128 * (kThreadLevel * (int)sizeof(DBox) + 8);
        static bool attr = false;
        if (!attr) { CK(cudaFuncSetAttribute(k_ti_stage15_refill, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); attr = true; }
        k_ti_stage15_refill<<<kSMs * 2, 128, bytes, st>>>(a, w.surv.p, nSurv, refill_work, w.surv2.p, nDefA, budget, &ist->ccd_ord, flags + 1);
        k_ti_stage2<<<kStage2Ctas, 32 * kStage2WarpsPerCta, 0, st>>>(a, w.surv2.p, nDefA, work, reinterpret_cast<DBox*>(w.scratch.p), kLevelCap, &ist->ccd_ord, flags + 1);
    }
    k_ccd_finish<<<1, 32, 0, st>>>(ist, nSurv, flags, overflow, stage == 3);
    ctx->prof_end(pe);
    ctx->launches += 5;
    CK(cudaGetLastError());
    int rc = nccl_min_u64(ctx, &ist->ccd_ord); // min over ranks of the step; a zero-distance flag travels as step 0
    if (rc) return rc;
    k_ccd_commit<<<1, 32, 0, st>>>(ist, stage);
    ++ctx->launches;
    return 0;
}

// sync-mode helper shared by the three step-bound entry points: copy the iteration state back and refresh the host-side diagnostics
int ccd_read_back(ipcgpu_ctx* ctx, double* alpha_out)
{
    int rc = fetch_iter_state(ctx);
    if (rc) return rc;
    CcdWork& w = ctx->ccd;
    const IterState& h = *ctx->h_iter;
    w.last_survivors = (unsigned)h.ccd_stats[0];
    w.last_warnings = (int)h.ccd_stats[1];
    w.last_deferred = h.ccd_stats[2];
    w.last_longest_cycles = h.ccd_stats[3];
    w.last_total_cycles = h.ccd_stats[4];
    w.last_boxes_thread = h.ccd_stats[5];
    w.last_boxes_warp = h.ccd_stats[6];
    w.last_candidates = h.ccd_stats[7];
    if (alpha_out) std::memcpy(alpha_out, &h.step_ord, sizeof(double));
    return 0;
}

// ---- swept hash build: SpatialHash::build(mesh, searchDir, curMaxStepSize, voxelSize) ------------------------------------
// Entirely on the stream: the span rescale of the step (:603-618), the swept bbox, the reference grid geometry and the swept grid on
// its voxel lattice all take their inputs from the device-resident iteration state.
int ccd_build_swept(ipcgpu_ctx* ctx, double h)
{
    CcdWork& w = ctx->ccd;
    cudaStream_t st = ctx->stream;
    const SurfArgs s = surf_args(ctx);
    IterState* ist = ctx->iter.p;
    if (!ctx->dir_valid) {
        ctx->err = "no search direction: pass p (or call ipcgpu_set_search_dir first)";
        return IPCGPU_ERR_STATE;
    }
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_CCD_BROAD);
    k_swept_alpha<<<1, 32, 0, st>>>(ist, ctx->pSize_dev.p, h, w.bounds.p);
    // bbox of V and of the displaced surface vertices (:627-628)
    k_swept_bounds<<<std::min(nblk(std::max(s.nV, s.nSV), 256), kSMs * 4), 256, 0, st>>>(s, ctx->dir.p, ist, w.bounds.p);
    k_refgrid_params<<<1, 32, 0, st>>>(ist, w.bounds.p, h, w.cells.p);
    ctx->launches += 3;
    const int nPrim = s.nSF + s.nSE + s.nSV;
    if (s.nSV > 0) {
        k_ref_ranges<<<nblk(s.nSV, 256), 256, 0, st>>>(s, ctx->dir.p, ist, w.vmin.p, w.vmax.p);
        k_swept_extent<<<std::min(nblk(nPrim, 256), kSMs * 4), 256, 0, st>>>(s, w.vmin.p, w.vmax.p, w.cells.p);
        k_swept_cells<<<1, 32, 0, st>>>(w.cells.p);
        const size_t nTab = (size_t)3 * kGridCells + 1;
        zero_words(w.sw_cnt.p, nTab, st); // (kernels.h: not a memset)
        k_swept_count<<<nblk(nPrim, 256), 256, 0, st>>>(s, w.vmin.p, w.vmax.p, w.cells.p, w.sw_cnt.p);
        size_t bytes = w.sw_tmp.n;
        CK(cub::DeviceScan::ExclusiveSum(w.sw_tmp.p, bytes, w.sw_cnt.p, w.sw_off.p, (int)nTab, st));
        k_swept_scatter<<<nblk(nPrim, 256), 256, 0, st>>>(s, w.vmin.p, w.vmax.p, w.cells.p, w.sw_cnt.p, w.sw_off.p, w.sw_keys.p, w.sw_ent.p);
        ctx->launches += 7;
    }
    ctx->prof_end(pe);
    CK(cudaGetLastError());
    w.swept_ready = true;
    return 0;
}

int ccd_full(ipcgpu_ctx* ctx, double tol, const double* err_vf, const double* err_ee)
{
    CcdWork& w = ctx->ccd;
    cudaStream_t st = ctx->stream;
    const SurfArgs s = surf_args(ctx);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_CCD_BROAD);
    CK(cudaMemsetAsync(w.ncand.p, 0, 2 * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(w.counters.p + 14, 0, sizeof(int), st));
    SweptArgs a{ s, ctx->dir.p, ctx->iter.p, w.vmin.p, w.vmax.p, w.cells.p, w.sw_keys.p, w.sw_ent.p, w.sw_off.p, 0, 0,
        CandOut{ w.cand.p, w.ncand.p, (unsigned long long)ctx->ccd_capacity, w.counters.p + 14 } };
    // multi-GPU: every rank keeps a disjoint share of the pairs -- PT by the surface vertex, EE by the smaller edge id (the reference's own
    // loop decomposition, :1385, :1498)
    if (s.nSF > 0 && s.nSV > 0) {
        a.lo = (int)((long long)s.nSV * ctx->rank / ctx->nranks);
        a.hi = (int)((long long)s.nSV * (ctx->rank + 1) / ctx->nranks);
        k_swept_pairs_pt<<<kSMs * 8, 32 * kSweptWarps, 0, st>>>(a);
        ++ctx->launches;
    }
    if (s.nSE > 1) {
        a.lo = (int)((long long)s.nSE * ctx->rank / ctx->nranks);
        a.hi = (int)((long long)s.nSE * (ctx->rank + 1) / ctx->nranks);
        k_swept_pairs_ee<<<kSMs * 8, 32 * kSweptWarps, 0, st>>>(a);
        ++ctx->launches;
    }
    ctx->prof_end(pe);
    // the candidate list is this rank's own (its share of the pairs): no further slicing; the list size and the capacity flag stay on the
    // device (checked at ipcgpu_fetch_iteration / by the synchronous wrapper)
    return ccd_narrow(ctx, w.cand.p, nullptr, w.ncand.p, (unsigned long long)ctx->ccd_capacity, 0, tol, err_vf, err_ee, 3, w.counters.p + 14);
}
