// constraint.cu -- barrier constraint-set build on the device (sm_90a).
//
// Replaces SelfCollisionHandler<3>::computeConstraintSet (src/CollisionObject/SelfCollisionHandler.cpp:2149-2478):
// PT loop over surface vertices (:2168-2260), EE loop over surface edges (:2271-2407), candidate list cs_PTEE
// (:2411-2424) and the serial std::map merge with PP/PE multiplicities (:2434-2476), including the three sentinel
// encodings for nearly parallel edge pairs (:2305-2311, :2383-2388, :2455-2468).
//
// Pipeline (one stream; a host sync only when the caller asks for the counts):
//   boxes+bounds -> grid params -> emit (cell,id) -> CUB radix sort -> PT / EE queries (atomic append)
//   -> merge of PP/PE duplicates -> canonical order of every output list (levels 1 and 2, sized on the device: lex_order / permute).
// The output ORDER is canonical (sorted), unlike the reference whose order depends on unordered_set iteration and TBB
// scheduling (:2176, :2282 "different constraint order will result in numerically different results").
#include "broadphase.cuh"
#include "abi.h"
#include <cub/cub.cuh>

namespace ipcgpu {

// ------------------------------------------------------------------------------------------------------------
// boxes + global bounds.  bounds[0..2] = min (flipped order), bounds[3..5] = max, bounds[6] = max extent
// ------------------------------------------------------------------------------------------------------------
DEV void grow(Box& b, V3 x)
{
    b.lo[0] = fmin(b.lo[0], x.x); b.hi[0] = fmax(b.hi[0], x.x);
    b.lo[1] = fmin(b.lo[1], x.y); b.hi[1] = fmax(b.hi[1], x.y);
    b.lo[2] = fmin(b.lo[2], x.z); b.hi[2] = fmax(b.hi[2], x.z);
}
DEV Box empty_box()
{
    Box b;
    for (int a = 0; a < 3; ++a) { b.lo[a] = 1e300; b.hi[a] = -1e300; }
    return b;
}

// prim: 0 = surface vertices, 1 = edges, 2 = triangles
__global__ void __launch_bounds__(256) k_boxes(SurfArgs s, int prim, Box* __restrict__ boxes, unsigned long long* __restrict__ bounds)
{
    const int n = prim == 0 ? s.nSV : (prim == 1 ? s.nSE : s.nSF);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    Box b = empty_box();
    double ext = 0.0;
    if (i < n) {
        int v[3], nv;
        if (prim == 0) { v[0] = s.SVI[i]; nv = 1; }
        else if (prim == 1) { v[0] = s.SE[2 * i]; v[1] = s.SE[2 * i + 1]; nv = 2; }
        else { v[0] = s.SF[i]; v[1] = s.SF[(size_t)s.nSF + i]; v[2] = s.SF[(size_t)2 * s.nSF + i]; nv = 3; }
        for (int k = 0; k < nv; ++k) grow(b, load_vertex(s.V, s.nV, v[k]));
        boxes[i] = b;
        ext = fmax(fmax(b.hi[0] - b.lo[0], b.hi[1] - b.lo[1]), b.hi[2] - b.lo[2]);
    }
    // CTA reduction then one atomic per CTA per value
    __shared__ double sm[7][8];
    double vals[7] = { b.lo[0], b.lo[1], b.lo[2], b.hi[0], b.hi[1], b.hi[2], ext };
#pragma unroll
    for (int q = 0; q < 7; ++q) {
        double x = vals[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            double y = __shfl_xor_sync(0xffffffffu, x, o);
            x = (q < 3) ? fmin(x, y) : fmax(x, y);
        }
        if ((threadIdx.x & 31) == 0) sm[q][threadIdx.x >> 5] = x;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        const int q = threadIdx.x;
        double x = sm[q][0];
        for (int w = 1; w < 8; ++w) x = (q < 3) ? fmin(x, sm[q][w]) : fmax(x, sm[q][w]);
        if (q < 3) atomicMin(bounds + q, flip_ord(x));
        else atomicMax(bounds + q, flip_ord(x));
    }
}

__global__ void k_bounds_init(unsigned long long* bounds)
{
    if (threadIdx.x < 3) bounds[threadIdx.x] = ~0ull;
    else if (threadIdx.x < 7) bounds[threadIdx.x] = 0ull;
}

// axis_bits: the cell keys of this build are sorted on 3 * axis_bits bits, so the grid gets at most 2^axis_bits - 1 cells per axis (cells
// grow when the scene would need more: the grid is only an accelerator, any cell size >= the largest inflated box is valid).  The
// number of cells per axis the scene WANTS goes to the iteration state; the host re-tunes axis_bits from it after every fetch, so that
// in the steady state the radix sort runs 2 passes (16 key bits) instead of 4.
__global__ void k_grid_params(const unsigned long long* __restrict__ bounds, double radius, int axis_bits, Grid* __restrict__ g, IterState* __restrict__ st)
{
    if (threadIdx.x != 0) return;
    double lo[3], hi[3];
    for (int a = 0; a < 3; ++a) { lo[a] = unflip_ord(bounds[a]) - radius; hi[a] = unflip_ord(bounds[3 + a]) + radius; }
    double ext = unflip_ord(bounds[6]);
    double h = (ext + 2.0 * radius) * (1.0 + 1e-9);
    const double span = fmax(fmax(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2]);
    h = fmax(h, span / 1024.0); // at most 1024 cells per axis
    if (!(h > 0.0)) h = 1.0;
    (void)axis_bits;
    // the dense cell table holds kGridCells cells: enlarge the cells until the grid fits (any cell size >= the largest inflated box is valid)
    int nx, ny, nz;
    for (int it = 0; it < 64; ++it) {
        const double inv = 1.0 / h;
        nx = max(1, (int)floor((hi[0] - lo[0]) * inv) + 1);
        ny = max(1, (int)floor((hi[1] - lo[1]) * inv) + 1);
        nz = max(1, (int)floor((hi[2] - lo[2]) * inv) + 1);
        if ((unsigned long long)nx * ny * nz <= (unsigned long long)kGridCells) break;
        h *= 1.1;
    }
    atomicMax(&st->grid_axis_cells, max(nx, max(ny, nz)));
    g->ox = lo[0]; g->oy = lo[1]; g->oz = lo[2];
    g->inv_h = 1.0 / h;
    g->q_inv = 65533.0 / fmax(span, 1e-300);
    g->nx = nx; g->ny = ny; g->nz = nz;
}

// Counting sort by cell (round 2, second half; before: CUB radix sort of (cell | type, id) pairs + an open-addressing cell table).
// One entry per primitive, registered in the cell of its box's lower corner; key = type << 20 | cell with type 0 triangles, 1 edges,
// 2 surface vertices, so the sorted array is "all triangles by cell, then all edges, then all vertices".
//   k_cell_count   : key of every primitive, its slot inside the cell from an atomic counter;
//   exclusive scan : counters -> DENSE offset table (two adjacent loads replace a hash probe per cell);
//   k_cell_scatter : primitive -> position offset[key] + slot: key, id and the quantised box (QEntry) are written in one go.
// The order of the entries inside a cell is whatever the atomics produced; nothing depends on it (pairs are reported from the entry with
// the smaller position, whichever that is; the output lists are order-free already).
__global__ void __launch_bounds__(256) k_cell_count(int nT, int nE, int nV, const Box* __restrict__ tboxes, const Box* __restrict__ eboxes, const Box* __restrict__ vboxes,
    const Grid* __restrict__ gp, int* __restrict__ cnt, unsigned* __restrict__ key_of, int* __restrict__ slot_of)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nT + nE + nV) return;
    const Grid g = *gp;
    const int type = i >= nT + nE ? 2 : (i >= nT ? 1 : 0);
    const int id = type == 2 ? i - nT - nE : (type == 1 ? i - nT : i);
    int c0[3], c1[3];
    cell_range(g, type == 2 ? vboxes[id] : (type == 1 ? eboxes[id] : tboxes[id]), c0, c1);
    const unsigned key = ((unsigned)type << kGridCellsLog2) | (unsigned)cell_key(g, c0[0], c0[1], c0[2]);
    key_of[i] = key;
    slot_of[i] = atomicAdd(cnt + key, 1);
}
__global__ void __launch_bounds__(256) k_cell_scatter(int nT, int nE, int nV, const Box* __restrict__ tboxes, const Box* __restrict__ eboxes, const Box* __restrict__ vboxes,
    const Grid* __restrict__ gp, const int* __restrict__ off, const unsigned* __restrict__ key_of, const int* __restrict__ slot_of, unsigned* __restrict__ keys,
    int* __restrict__ ids, uint4* __restrict__ sorted)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nT + nE + nV) return;
    const int type = i >= nT + nE ? 2 : (i >= nT ? 1 : 0);
    const int id = type == 2 ? i - nT - nE : (type == 1 ? i - nT : i);
    const unsigned key = key_of[i];
    const int pos = off[key] + slot_of[i];
    const QBox q = quantize_box(*gp, type == 2 ? vboxes[id] : (type == 1 ? eboxes[id] : tboxes[id]));
    keys[pos] = key;
    ids[pos] = id;
    sorted[pos] = make_uint4((unsigned)q.lo[0] | ((unsigned)q.lo[1] << 16), (unsigned)q.lo[2] | ((unsigned)q.hi[0] << 16), (unsigned)q.hi[1] | ((unsigned)q.hi[2] << 16), (unsigned)id);
}

// ------------------------------------------------------------------------------------------------------------
// queries
// ------------------------------------------------------------------------------------------------------------
struct CsOut {
    int4* act; int* nAct; int capAct;     // PT / EE entries (slot3 >= 0)
    int4* dup; int* nDup; int capDup;     // PP / PE entries to be counted (slot3 = -1)
    int4* para; int2* para_e; int* nPara; int capPara;
    int2* cand; int* nCand; int capCand;  // cs_PTEE (only when wanted)
    int* overflow;
};

DEV void push4(int4* arr, int* cnt, int cap, int* overflow, int4 v)
{
    int i = atomicAdd(cnt, 1);
    if ((unsigned)i < (unsigned)cap) arr[i] = v; // unsigned: a wrapped counter must not index backwards
    else atomicExch(overflow, 1);
}

DEV double box_gap2(const Box& a, const Box& b)
{
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double g = fmax(fmax(a.lo[k] - b.hi[k], b.lo[k] - a.hi[k]), 0.0);
        s += g * g;
    }
    return s;
}
DEV bool is_dbc_v(const SurfArgs& s, int v) { return s.dbc && s.dbc[v] != 0; }
DEV int codim_v(const SurfArgs& s, int v) { return s.vCoDim ? s.vCoDim[v] : 3; }

// ---- phase 1: broad phase proper, cell-centric pair finding (round 2, second half) ------------------------------------------------
// Only boxes are touched here: the pairs whose boxes are closer than sqrt(dHat) go to a list that phase 2 classifies.  A warp per
// query (warp_scan_candidates, the round-1 form) spends ~2 warp instructions per box test (flattened-index arithmetic, entry load,
// ballot/append per 32 tests plus ~150 instructions of set-up per query) and is ISSUE-bound (542 K edge queries x ~450 instructions;
// on C5 with H100 SXM at 400 W the constraint set took 0.69 ms with it against 0.35 ms with the kernels below).  Here a
// warp takes 32 CONSECUTIVE entries of the sorted edge grid as queries ("A"); consecutive entries share their cell, so the partner
// entries ("B") of a whole run of queries are fetched once: a lane holds one B entry and tests it against every query of the run, whose
// inflated quantised boxes sit in shared memory (one broadcast LDS.128 + LDS.64 and ~8 integer instructions per test, 16-bit SIMD min for
// two axes at a time).  Hits are rare and appended lane by lane.  One-sided: a pair is reported from the entry with
// the smaller sorted position, so only cells at or behind the run's own cell are visited.
//   Which cells: a query registered in cell c (lower corner of its box) and inflated by `radius` covers cells c0'..c1' with
//   c - 1 <= c0' <= c and c1' <= c0' + 1; its partners are registered in [c0' - 1, c1'] (broadphase.cuh).  The run uses the union over
//   its queries, computed conservatively from the quantised boxes and clamped to the provable superset [c - 2, c + 1] per axis.
struct alignas(16) AEntry {
    unsigned L01, H01, lo2, hi2; // inflated quantised box: (lo0 | lo1 << 16), (hi0 | hi1 << 16), lo2, hi2
    int pos, id, pad0, pad1;     // 32 bytes: two 128-bit shared-memory loads
};
constexpr int kCellPairWarps = 8;
// Hits are staged PER WARP (ncu on the first version, which staged per CTA: 20 % of the stall samples sat behind the CTA barrier of the final
// flush -- the eight warps of a CTA finish their chunks at very different times) and flushed by the warp itself with one global atomic.
constexpr int kWarpStageCap = 256; // pairs per warp (2 KB)
struct WarpStage {
    int2 buf[kWarpStageCap];
    unsigned count;
};
DEV void lane_push_pair(WarpStage& ws, const PairOut& o, int a, int b)
{
    const unsigned i = atomicAdd(&ws.count, 1u);
    if (i < (unsigned)kWarpStageCap) ws.buf[i] = make_int2(a, b);
    else { // stage full (a very dense neighbourhood between two flushes): straight to the global list
        const unsigned gi = atomicAdd(o.n, 1u);
        if (gi < o.cap) o.pairs[gi] = make_int2(a, b);
        else atomicExch(o.overflow, 1);
    }
}
// all 32 lanes; flushes when the stage is at least `threshold` full
DEV void warp_stage_flush(WarpStage& ws, const PairOut& o, int lane, unsigned threshold)
{
    __syncwarp();
    const unsigned n = min(ws.count, (unsigned)kWarpStageCap);
    if (n < threshold || n == 0u) return;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(o.n, n);
    base = __shfl_sync(0xffffffffu, base, 0);
    for (unsigned i = lane; i < n; i += 32) {
        if (base + i < o.cap) o.pairs[base + i] = ws.buf[i];
        else atomicExch(o.overflow, 1);
    }
    __syncwarp();
    if (lane == 0) ws.count = 0;
    __syncwarp();
}
__global__ void __launch_bounds__(32 * kCellPairWarps) k_cell_pairs_ee(const Grid* __restrict__ gp, SortedGrid eg, const int* __restrict__ SE, double radius, int first,
    int last, PairOut out)
{
    __shared__ WarpStage sStage[kCellPairWarps];
    __shared__ AEntry sA[kCellPairWarps][32];
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    WarpStage& stage = sStage[wib];
    if (lane == 0) stage.count = 0;
    __syncwarp();
    const Grid g = *gp;
    // the query is inflated by `radius` in lattice steps of the quantised entry boxes; lattice coordinate q lies in accelerator cell floor(q * S)
    const unsigned rq = (unsigned)min((int)ceil(radius * g.q_inv) + 1, 65535);
    const unsigned rq2 = rq | (rq << 16);
    const double S = g.inv_h / g.q_inv;
    const uint4* __restrict__ ent = reinterpret_cast<const uint4*>(eg.ent);
    AEntry* A = sA[wib];
    const int pos = first + (blockIdx.x * kCellPairWarps + wib) * 32 + lane;
    const bool valid = pos < last;
    unsigned key = 0xffffffffu;
    int cl[3] = { 0, 0, 0 }, ch[3] = { 0, 0, 0 }; // conservative cell range of the inflated box
    if (valid) {
        const uint4 e = __ldg(ent + pos);
        key = eg.keys[pos] & (kGridCells - 1u);
        AEntry a;
        a.L01 = __vsubus2(e.x, rq2);                                  // lo0, lo1 - rq (saturating)
        a.H01 = __vaddus2(__funnelshift_r(e.y, e.z, 16), rq2);       // hi0, hi1 + rq
        const unsigned lo2 = e.y & 0xffffu, hi2 = e.z >> 16;
        a.lo2 = lo2 > rq ? lo2 - rq : 0u;
        a.hi2 = min(hi2 + rq, 65535u);
        a.pos = pos;
        a.id = (int)e.w;
        {   // the edge's two vertices ride along: pairs of edges that share a vertex are dropped right here (the exact stages drop them
            // anyway, SelfCollisionHandler.cpp:2294; between neighbouring edges of a mesh they are the bulk of all overlapping boxes)
            const int2 av = __ldg(reinterpret_cast<const int2*>(SE) + a.id);
            a.pad0 = av.x; a.pad1 = av.y;
        }
        A[lane] = a;
        cl[0] = (int)floor((double)(a.L01 & 0xffffu) * S); ch[0] = (int)floor((double)(a.H01 & 0xffffu) * S);
        cl[1] = (int)floor((double)(a.L01 >> 16) * S);     ch[1] = (int)floor((double)(a.H01 >> 16) * S);
        cl[2] = (int)floor((double)a.lo2 * S);             ch[2] = (int)floor((double)a.hi2 * S);
    }
    __syncwarp();
    unsigned remaining = __ballot_sync(full, valid);
    while (remaining) {
        const int leader = __ffs(remaining) - 1;
        const unsigned k0 = __shfl_sync(full, key, leader);
        const unsigned m = __ballot_sync(full, valid && key == k0); // the run: consecutive lanes (the array is sorted by cell)
        remaining &= ~m;
        const int a_lo = leader, a_hi = 32 - __clz(m);              // lanes [a_lo, a_hi)
        const int p_lo = __shfl_sync(full, pos, leader);
        // the run's own cell and the union of its queries' ranges, clamped to [c - 2, c + 1] and to the grid
        const int cx = (int)(k0 % (unsigned)g.nx), cy = (int)((k0 / (unsigned)g.nx) % (unsigned)g.ny), cz = (int)(k0 / ((unsigned)g.nx * (unsigned)g.ny));
        const bool in = (m >> lane) & 1u;
        int lo[3], hi[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            lo[a] = __reduce_min_sync(full, in ? cl[a] : 0x7fffffff) - 1;
            hi[a] = __reduce_max_sync(full, in ? ch[a] : -1);
        }
        const int xlo = max(max(lo[0], cx - 2), 0), xhi = min(min(hi[0], cx + 1), g.nx - 1);
        const int ylo = max(max(lo[1], cy - 2), 0), yhi = min(min(hi[1], cy + 1), g.ny - 1);
        const int zhi = min(min(hi[2], cz + 1), g.nz - 1);
        // rows at or behind the own cell: r = 0 own row (cells cx..xhi); then (y' in (cy, yhi], z' = cz); then (y' in [ylo, yhi], z' in (cz, zhi])
        const int nUp = max(yhi - cy, 0), nY = max(yhi - ylo + 1, 0), nZ = max(zhi - cz, 0);
        const int nRows = 1 + nUp + nY * nZ; // <= 1 + 1 + 4 = 6
        // lane r < nRows: the run of row r = entries of its cells xs..xhi -- consecutive cells are consecutive in the sorted array, so the run is
        // two loads from the dense offset table (first cell's start, last cell's end)
        int rs = 0x7fffffff, re = -1;
        if (lane < nRows) {
            const int r = lane;
            int y, z, xs;
            if (r == 0) { y = cy; z = cz; xs = cx; }
            else if (r <= nUp) { y = cy + r; z = cz; xs = xlo; }
            else { const int q = r - 1 - nUp; z = cz + 1 + q / nY; y = ylo + q % nY; xs = xlo; }
            if (xs <= xhi) {
                rs = cell_lookup(eg, (unsigned)cell_key(g, xs, y, z)).x;
                re = cell_lookup(eg, (unsigned)cell_key(g, xhi, y, z)).y;
            }
        }
        if (lane == 0) rs = max(rs, p_lo + 1); // own row: nothing at or before the run's first query is ever needed
        const int rlen = (lane < 6 && lane < nRows && re > rs) ? re - rs : 0;
        int incl = rlen;
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            const int t = __shfl_up_sync(full, incl, o);
            if (lane >= o) incl += t;
        }
        int inc[6], st[6];
#pragma unroll
        for (int r = 0; r < 6; ++r) {
            inc[r] = __shfl_sync(full, incl, r);
            st[r] = __shfl_sync(full, rs, r);
        }
        const int total = inc[5];
        auto locate = [&](int j) {
            int k = st[0] + j;
#pragma unroll
            for (int r = 1; r < 6; ++r)
                if (j >= inc[r - 1]) k = st[r] + (j - inc[r - 1]);
            return k;
        };
        int kn = (lane < total) ? locate(lane) : 0;
        uint4 en = make_uint4(0u, 0u, 0u, 0u);
        if (lane < total) en = __ldg(ent + kn);
        for (int j = lane; j - lane < total; j += 32) {
            const uint4 e = en;
            const int bpos = kn;
            const bool have = j < total;
            int2 bv = make_int2(-1, -1);
            if (have) bv = __ldg(reinterpret_cast<const int2*>(SE) + (int)e.w); // the partner's vertices (in flight next to the next entry)
            if (j + 32 < total) { kn = locate(j + 32); en = __ldg(ent + kn); }
            if (have) {
                const unsigned bL01 = e.x, bH01 = __funnelshift_r(e.y, e.z, 16), blo2 = e.y & 0xffffu, bhi2 = e.z >> 16;
                for (int a = a_lo; a < a_hi; ++a) {
                    const AEntry q = A[a]; // same address on every lane: broadcast
                    const bool hit = __vminu2(q.L01, bH01) == q.L01 && __vminu2(bL01, q.H01) == bL01 && q.lo2 <= bhi2 && blo2 <= q.hi2 && bpos > q.pos
                        && q.pad0 != bv.x && q.pad0 != bv.y && q.pad1 != bv.x && q.pad1 != bv.y;
                    if (hit) lane_push_pair(stage, out, min(q.id, (int)e.w), max(q.id, (int)e.w));
                }
            }
        }
        warp_stage_flush(stage, out, lane, kWarpStageCap / 2); // (also the warp-level barrier before the queries' slots are reused)
    }
    warp_stage_flush(stage, out, lane, 1u);
}

// The point-triangle twin: queries = 32 consecutive entries of the sorted VERTEX segment (points, or swept vertex boxes for the CCD),
// partners = triangle entries of every cell a query of the run can see (both sides: up to 4 x 4 rows of <= 4 cells; typically 3 x 3 x 3).
// Rows are walked one after the other (a row of three cells holds about one warp-load of triangles); the first load of the next row is
// issued before the current row is tested.
__global__ void __launch_bounds__(32 * kCellPairWarps) k_cell_pairs_pt(const Grid* __restrict__ gp, SortedGrid vg, SortedGrid tg, const int* __restrict__ SVI,
    const int* __restrict__ SF, int nSF, double radius, int first, int last, PairOut out)
{
    __shared__ WarpStage sStage[kCellPairWarps];
    __shared__ AEntry sA[kCellPairWarps][32];
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    WarpStage& stage = sStage[wib];
    if (lane == 0) stage.count = 0;
    __syncwarp();
    const Grid g = *gp;
    // the query is inflated by `radius` in lattice steps of the quantised entry boxes; lattice coordinate q lies in accelerator cell floor(q * S)
    const unsigned rq = (unsigned)min((int)ceil(radius * g.q_inv) + 1, 65535);
    const unsigned rq2 = rq | (rq << 16);
    const double S = g.inv_h / g.q_inv;
    const uint4* __restrict__ ent = reinterpret_cast<const uint4*>(tg.ent);
    AEntry* A = sA[wib];
    const int pos = first + (blockIdx.x * kCellPairWarps + wib) * 32 + lane;
    const bool valid = pos < last;
    unsigned key = 0xffffffffu;
    int cl[3] = { 0, 0, 0 }, ch[3] = { 0, 0, 0 };
    if (valid) {
        const uint4 e = __ldg(ent + pos);
        key = vg.keys[pos] & (kGridCells - 1u);
        AEntry a;
        a.L01 = __vsubus2(e.x, rq2);
        a.H01 = __vaddus2(__funnelshift_r(e.y, e.z, 16), rq2);
        const unsigned lo2 = e.y & 0xffffu, hi2 = e.z >> 16;
        a.lo2 = lo2 > rq ? lo2 - rq : 0u;
        a.hi2 = min(hi2 + rq, 65535u);
        a.pos = pos;
        a.id = (int)e.w;
        a.pad0 = __ldg(SVI + a.id); // the vertex itself: a triangle that contains it is no partner (:2184), and those are most overlapping boxes
        a.pad1 = 0;
        A[lane] = a;
        cl[0] = (int)floor((double)(a.L01 & 0xffffu) * S); ch[0] = (int)floor((double)(a.H01 & 0xffffu) * S);
        cl[1] = (int)floor((double)(a.L01 >> 16) * S);     ch[1] = (int)floor((double)(a.H01 >> 16) * S);
        cl[2] = (int)floor((double)a.lo2 * S);             ch[2] = (int)floor((double)a.hi2 * S);
    }
    __syncwarp();
    unsigned remaining = __ballot_sync(full, valid);
    while (remaining) {
        const int leader = __ffs(remaining) - 1;
        const unsigned k0 = __shfl_sync(full, key, leader);
        const unsigned m = __ballot_sync(full, valid && key == k0);
        remaining &= ~m;
        const int a_lo = leader, a_hi = 32 - __clz(m);
        const int cx = (int)(k0 % (unsigned)g.nx), cy = (int)((k0 / (unsigned)g.nx) % (unsigned)g.ny), cz = (int)(k0 / ((unsigned)g.nx * (unsigned)g.ny));
        const bool in = (m >> lane) & 1u;
        int lo[3], hi[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            lo[a] = __reduce_min_sync(full, in ? cl[a] : 0x7fffffff) - 1;
            hi[a] = __reduce_max_sync(full, in ? ch[a] : -1);
        }
        const int xlo = max(max(lo[0], cx - 2), 0), xhi = min(min(hi[0], cx + 1), g.nx - 1);
        const int ylo = max(max(lo[1], cy - 2), 0), yhi = min(min(hi[1], cy + 1), g.ny - 1);
        const int zlo = max(max(lo[2], cz - 2), 0), zhi = min(min(hi[2], cz + 1), g.nz - 1);
        const int nY = max(yhi - ylo + 1, 0), nZ = max(zhi - zlo + 1, 0);
        const int nRows = nY * nZ; // <= 16
        {
            // lane r < nRows (<= 16): the run of row r, two loads from the dense offset table
            int rs = 0x7fffffff, re = -1;
            if (lane < nRows && xlo <= xhi) {
                const int y = ylo + lane % nY, z = zlo + lane / nY;
                rs = cell_lookup(tg, (unsigned)cell_key(g, xlo, y, z)).x;
                re = cell_lookup(tg, (unsigned)cell_key(g, xhi, y, z)).y;
            }
            // first chunk of row 0 in flight
            int cs = __shfl_sync(full, rs, 0), ce = __shfl_sync(full, re, 0);
            uint4 en = make_uint4(0u, 0u, 0u, 0u);
            if (ce > cs && lane < ce - cs) en = __ldg(ent + cs + lane); // (an empty row is [INT_MAX, -1): no index arithmetic on it)
            for (int r = 0; r < nRows; ++r) {
                const int s0 = cs, e0 = ce;
                uint4 e = en;
                if (r + 1 < nRows) { // next row's first chunk
                    cs = __shfl_sync(full, rs, r + 1);
                    ce = __shfl_sync(full, re, r + 1);
                    if (ce > cs && lane < ce - cs) en = __ldg(ent + cs + lane);
                }
                const int len = e0 > s0 ? e0 - s0 : 0;
                for (int jj = lane; jj - lane < len; jj += 32) {
                    if (jj >= 32 && jj < len) e = __ldg(ent + s0 + jj); // rows longer than one warp-load (rare)
                    if (jj < len) {
                        const unsigned bL01 = e.x, bH01 = __funnelshift_r(e.y, e.z, 16), blo2 = e.y & 0xffffu, bhi2 = e.z >> 16;
                        const int t0 = __ldg(SF + (int)e.w), t1 = __ldg(SF + nSF + (int)e.w), t2 = __ldg(SF + 2 * (size_t)nSF + (int)e.w);
                        for (int a = a_lo; a < a_hi; ++a) {
                            const AEntry q = A[a];
                            const bool hit = __vminu2(q.L01, bH01) == q.L01 && __vminu2(bL01, q.H01) == bL01 && q.lo2 <= bhi2 && blo2 <= q.hi2
                                && q.pad0 != t0 && q.pad0 != t1 && q.pad0 != t2;
                            if (hit) lane_push_pair(stage, out, q.id, (int)e.w);
                        }
                    }
                }
            }
        }
        warp_stage_flush(stage, out, lane, kWarpStageCap / 2); // (also the warp-level barrier before the queries' slots are reused)
    }
    warp_stage_flush(stage, out, lane, 1u);
}

// ---- phase 2: exact closest-feature classification, one THREAD per surviving pair (dense, convergent)
// (:2168-2260)
__global__ void __launch_bounds__(128) k_classify_pt(SurfArgs s, const int2* __restrict__ pairs, const unsigned* __restrict__ nPairs, unsigned cap, double dHat, int wantCand, CsOut out)
{
    // grid-stride over the device-resident pair count (a launch sized by the list CAPACITY spent more time retiring empty CTAs than working)
    const unsigned nP = min(*nPairs, cap);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nP; i += gridDim.x * blockDim.x) {
    const int svI = pairs[i].x, sfI = pairs[i].y;
    const int vI = s.SVI[svI];
    const int a = s.SF[sfI], b = s.SF[(size_t)s.nSF + sfI], c = s.SF[(size_t)2 * s.nSF + sfI];
    if (vI == a || vI == b || vI == c) continue;
    // mesh against itself: the self-contact filter (:2184-2190); mesh against the obstacle: none (MeshCO.cpp:1803-1990); inside the obstacle: no pairs
    const bool oP = obstacle_vertex(s, vI), oT = obstacle_vertex(s, a);
    if (oP && oT) continue;
    if (!oP && !oT && ((codim_v(s, vI) < 3 && codim_v(s, a) < 3) || (is_dbc_v(s, vI) && is_dbc_v(s, a) && is_dbc_v(s, b) && is_dbc_v(s, c)))) continue;
    const V3 p = load_vertex(s.V, s.nV, vI);
    const V3 ta = load_vertex(s.V, s.nV, a), tb_ = load_vertex(s.V, s.nV, b), tc = load_vertex(s.V, s.nV, c);
    const int ty = dType_PT(p, ta, tb_, tc);
    double d;
    int4 q;
    switch (ty) {
    case 0: d = d_PP(p, ta); q = make_int4(-vI - 1, a, -1, -1); break;
    case 1: d = d_PP(p, tb_); q = make_int4(-vI - 1, b, -1, -1); break;
    case 2: d = d_PP(p, tc); q = make_int4(-vI - 1, c, -1, -1); break;
    case 3: d = d_PE(p, ta, tb_); q = make_int4(-vI - 1, a, b, -1); break;
    case 4: d = d_PE(p, tb_, tc); q = make_int4(-vI - 1, b, c, -1); break;
    case 5: d = d_PE(p, tc, ta); q = make_int4(-vI - 1, c, a, -1); break;
    default: d = d_PT(p, ta, tb_, tc); q = make_int4(-vI - 1, a, b, c);
    }
    // an obstacle point against a mesh vertex is the same entry as that mesh vertex against the obstacle point: MeshCO writes both
    // (-meshV - 1, obstacleV, -1, .) and counts them together (MeshCO.cpp:1831, :1919, :2168-2190)
    if (ty <= 2 && oP) q = make_int4(-q.y - 1, vI, -1, -1);
    if (d < dHat) {
        if (q.w >= 0) push4(out.act, out.nAct, out.capAct, out.overflow, q);
        else push4(out.dup, out.nDup, out.capDup, out.overflow, q);
        if (wantCand) {
            int k = atomicAdd(out.nCand, 1);
            if ((unsigned)k < (unsigned)out.capCand) out.cand[k] = make_int2(-svI - 1, sfI);
            else atomicExch(out.overflow, 1);
        }
    }
    }
}

// (:2271-2407)
__global__ void __launch_bounds__(128) k_classify_ee(SurfArgs s, const int2* __restrict__ pairs, const unsigned* __restrict__ nPairs, unsigned cap, double dHat, int wantCand, CsOut out)
{
    const unsigned nP = min(*nPairs, cap);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nP; i += gridDim.x * blockDim.x) {
    const int eI = pairs[i].x, eJ = pairs[i].y;
    const int a0 = s.SE[2 * eI], a1 = s.SE[2 * eI + 1], b0 = s.SE[2 * eJ], b1 = s.SE[2 * eJ + 1];
    if (a0 == b0 || a0 == b1 || a1 == b0 || a1 == b1) continue;
    const bool oA = obstacle_vertex(s, a0), oB = obstacle_vertex(s, b0); // (:2294-2300; MeshCO.cpp:1996-2030)
    if (oA && oB) continue;
    if (!oA && !oB && ((codim_v(s, a0) < 3 && codim_v(s, b0) < 3) || (is_dbc_v(s, a0) && is_dbc_v(s, a1) && is_dbc_v(s, b0) && is_dbc_v(s, b1)))) continue;
    const V3 xa0 = load_vertex(s.V, s.nV, a0), xa1 = load_vertex(s.V, s.nV, a1), xb0 = load_vertex(s.V, s.nV, b0), xb1 = load_vertex(s.V, s.nV, b1);
    const int ty = dType_EE(xa0, xa1, xb0, xb1);
    const double cr = norm2(cross(xa1 - xa0, xb1 - xb0));
    const int add_e = (cr < eps_x_rest(s.Vrest, s.nV, a0, a1, b0, b1)) ? (-eJ - 2) : -1;
    double d;
    int4 q;
    switch (ty) {
    case 0: d = d_PP(xa0, xb0); q = make_int4(-a0 - 1, b0, -1, add_e); break;
    case 1: d = d_PP(xa0, xb1); q = make_int4(-a0 - 1, b1, -1, add_e); break;
    case 2: d = d_PE(xa0, xb0, xb1); q = make_int4(-a0 - 1, b0, b1, add_e); break;
    case 3: d = d_PP(xa1, xb0); q = make_int4(-a1 - 1, b0, -1, add_e); break;
    case 4: d = d_PP(xa1, xb1); q = make_int4(-a1 - 1, b1, -1, add_e); break;
    case 5: d = d_PE(xa1, xb0, xb1); q = make_int4(-a1 - 1, b0, b1, add_e); break;
    case 6: d = d_PE(xb0, xa0, xa1); q = make_int4(-b0 - 1, a0, a1, add_e); break;
    case 7: d = d_PE(xb1, xa0, xa1); q = make_int4(-b1 - 1, a0, a1, add_e); break;
    default: d = d_EE(xa0, xa1, xb0, xb1); q = make_int4(a0, a1, b0, b1);
    }
    if (d < dHat) {
        if (ty == 8) {
            if (add_e <= -2) { // nearly parallel EE: mollified set, keeps its own stencil (:2464-2467)
                int k = atomicAdd(out.nPara, 1);
                if ((unsigned)k < (unsigned)out.capPara) { out.para[k] = q; out.para_e[k] = make_int2(-1, -1); }
                else atomicExch(out.overflow, 1);
            }
            else push4(out.act, out.nAct, out.capAct, out.overflow, q);
        }
        else if (add_e == -1) push4(out.dup, out.nDup, out.capDup, out.overflow, q);
        else { // PP / PE that came from a nearly parallel edge pair (:2459-2462)
            int k = atomicAdd(out.nPara, 1);
            if ((unsigned)k < (unsigned)out.capPara) { out.para[k] = make_int4(q.x, q.y, q.z, -1); out.para_e[k] = make_int2(eI, eJ); }
            else atomicExch(out.overflow, 1);
        }
        if (wantCand) {
            int k = atomicAdd(out.nCand, 1);
            if ((unsigned)k < (unsigned)out.capCand) out.cand[k] = make_int2(eI, eJ);
            else atomicExch(out.overflow, 1);
        }
    }
    }
}

// ------------------------------------------------------------------------------------------------------------
// canonical order of a contact list, sized on the device: lexicographic on the signed components, the companion (eI, eJ) last.  A bucket
// pass on the first component (count, exclusive scan, scatter of positions; x + nV is the bucket: x is -v - 1 in the PT/PP/PE encodings
// and in the PT candidates, a vertex or an edge index otherwise), then an insertion sort of every bucket on the rest.
// ------------------------------------------------------------------------------------------------------------
constexpr int kLexBlocks = kSMs * 4;
DEV bool lex_less(int4 a, int2 ac, int4 b, int2 bc)
{
    if (a.y != b.y) return a.y < b.y;
    if (a.z != b.z) return a.z < b.z;
    if (a.w != b.w) return a.w < b.w;
    if (ac.x != bc.x) return ac.x < bc.x;
    return ac.y < bc.y;
}
DEV bool lex_less(int2 a, int2, int2 b, int2) { return a.y < b.y; }
template <typename T>
__global__ void __launch_bounds__(256) k_lex_count(const T* __restrict__ list, const int* __restrict__ n_ptr, int cap, int nV, int* __restrict__ cnt)
{
    const int n = min(*n_ptr, cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atomicAdd(cnt + list[i].x + nV, 1);
}
template <typename T>
__global__ void __launch_bounds__(256) k_lex_scatter(const T* __restrict__ list, const int* __restrict__ n_ptr, int cap, int nV, int* __restrict__ cur,
    int* __restrict__ perm)
{
    const int n = min(*n_ptr, cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) perm[atomicAdd(cur + list[i].x + nV, 1)] = i;
}
// one thread per bucket: insertion sort of its positions on (y, z, w, companion)
template <typename T>
__global__ void __launch_bounds__(256) k_lex_bucket_sort(int nB, const int* __restrict__ off, const T* __restrict__ list, const int2* __restrict__ comp,
    int* __restrict__ perm)
{
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nB; b += gridDim.x * blockDim.x) {
        const int s = off[b], e = off[b + 1];
        for (int i = s + 1; i < e; ++i) {
            const int pi = perm[i];
            const T key = list[pi];
            const int2 kc = comp ? comp[pi] : make_int2(0, 0);
            int j = i - 1;
            while (j >= s) {
                const int pj = perm[j];
                if (!lex_less(key, kc, list[pj], comp ? comp[pj] : make_int2(0, 0))) break;
                perm[j + 1] = pj;
                --j;
            }
            perm[j + 1] = pi;
        }
    }
}
// dst[i] = src[perm[i]] for i < n, `words` 8-byte words per element (k_copy_words then copies dst back)
__global__ void __launch_bounds__(256) k_permute_words(const unsigned long long* __restrict__ src, const int* __restrict__ perm, const int* __restrict__ n_ptr,
    int cap, int words, unsigned long long* __restrict__ dst)
{
    const long long n = (long long)min(*n_ptr, cap) * words;
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[(long long)perm[i / words] * words + i % words];
}
__global__ void __launch_bounds__(256) k_copy_words(const unsigned long long* __restrict__ src, const int* __restrict__ n_ptr, int cap, int words,
    unsigned long long* __restrict__ dst)
{
    const long long n = (long long)min(*n_ptr, cap) * words;
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i];
}
// heads of runs of equal (x,y,z) in a sorted dup list emit (x,y,z,-count) into the active list (:2434-2476)
__global__ void __launch_bounds__(256) k_merge_dups(const int* __restrict__ n_ptr, int cap, const int4* __restrict__ sorted, int4* __restrict__ act, int* __restrict__ nAct,
    int* __restrict__ overflow)
{
    const int n = min(*n_ptr, cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 v = sorted[i];
        if (i > 0) {
            const int4 u = sorted[i - 1];
            if (u.x == v.x && u.y == v.y && u.z == v.z) continue;
        }
        int cnt = 1;
        while (i + cnt < n) {
            const int4 w = sorted[i + cnt];
            if (w.x != v.x || w.y != v.y || w.z != v.z) break;
            ++cnt;
        }
        push4(act, nAct, cap, overflow, make_int4(v.x, v.y, v.z, -cnt));
    }
}

// sort-free variant of the same merge for meshes below 2^21 vertices: (x,y,z) packs into one 64-bit key, an open-addressing table
// counts the multiplicities (2 short kernels instead of sorting the list)
DEV unsigned long long dup_key(int4 v) { return ((unsigned long long)(unsigned)(-v.x - 1) << 42) | ((unsigned long long)(unsigned)v.y << 21) | (unsigned long long)(unsigned)(v.z + 1); }
__global__ void k_dup_insert(const int* __restrict__ n_ptr, int cap, const int4* __restrict__ dup, unsigned long long* __restrict__ tab_key, int* __restrict__ tab_cnt,
    unsigned mask, int* __restrict__ overflow)
{
    const int n = min(*n_ptr, cap); // the list size stays on the device
    if (2ll * n > (long long)mask + 1) { // the table must stay at most half full
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicExch(overflow, 1);
        return;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = dup_key(dup[i]);
        unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 40) & mask;
        for (;;) {
            const unsigned long long old = atomicCAS(tab_key + h, ~0ull, key);
            if (old == ~0ull || old == key) {
                atomicAdd(tab_cnt + h, 1);
                break;
            }
            h = (h + 1) & mask;
        }
    }
}
// sizes of the finished lists -> the iteration state (read back once per iteration by ipcgpu_fetch_iteration)
__global__ void k_publish_counts(const int* __restrict__ counters, int wantCand, IterState* __restrict__ st)
{
    if (threadIdx.x != 0) return;
    st->n_set[0] = counters[0];
    st->n_set[1] = counters[2];
    st->n_set[2] = wantCand ? counters[3] : 0;
    if (counters[4]) st->flags[FLAG_SET_CAPACITY] = 1;
}

// ---- multi-rank exchange of the (small) pair lists: every rank packs [header | active | mollified | (eI,eJ)] into one fixed-size
// message, one ncclAllGather moves all of them, and every rank rebuilds the GLOBAL lists (rank-major order) from the N messages.
// Message layout in int4 units: [0] = (nAct, nPara, 0, 0); [1, 1+xcap) active; [1+xcap, 1+2 xcap) mollified; then xcap int2.
__global__ void __launch_bounds__(256) k_pack_lists(const int4* __restrict__ act, const int4* __restrict__ para, const int2* __restrict__ para_e, const int* __restrict__ counters,
    int xcap, int4* __restrict__ msg, int* __restrict__ overflow)
{
    const int nA = counters[0], nP = counters[2];
    if (nA > xcap || nP > xcap) {
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            atomicExch(overflow, 1);
            msg[0] = make_int4(0, 0, 0, 0);
        }
        return;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) msg[0] = make_int4(nA, nP, 0, 0);
    int2* pe = reinterpret_cast<int2*>(msg + 1 + 2 * (size_t)xcap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(nA, nP); i += gridDim.x * blockDim.x) {
        if (i < nA) msg[1 + i] = act[i];
        if (i < nP) {
            msg[1 + xcap + i] = para[i];
            pe[i] = para_e[i];
        }
    }
}
__global__ void __launch_bounds__(256) k_unpack_lists(const int4* __restrict__ all, int nranks, int xcap, size_t stride /* int4 per message */, int4* __restrict__ gact,
    int4* __restrict__ gpara, int2* __restrict__ gpara_e, int cap, int* __restrict__ counts_out /* [0] active, [1] mollified */, int* __restrict__ overflow)
{
    for (int q = 0; q < nranks; ++q) {
        int offA = 0, offP = 0;
        for (int r = 0; r < q; ++r) {
            const int4 h = all[(size_t)r * stride];
            offA += h.x;
            offP += h.y;
        }
        const int4 * m = all + (size_t)q * stride;
        const int nA = m[0].x, nP = m[0].y;
        if (offA + nA > cap || offP + nP > cap) {
            if (blockIdx.x == 0 && threadIdx.x == 0) atomicExch(overflow, 1);
            return;
        }
        const int2* pe = reinterpret_cast<const int2*>(m + 1 + 2 * (size_t)xcap);
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(nA, nP); i += gridDim.x * blockDim.x) {
            if (i < nA) gact[offA + i] = m[1 + i];
            if (i < nP) {
                gpara[offP + i] = m[1 + xcap + i];
                gpara_e[offP + i] = pe[i];
            }
        }
        if (q == nranks - 1 && blockIdx.x == 0 && threadIdx.x == 0) {
            counts_out[0] = offA + nA;
            counts_out[1] = offP + nP;
        }
    }
}
__global__ void k_dup_emit(unsigned size, const unsigned long long* __restrict__ tab_key, const int* __restrict__ tab_cnt, int4* __restrict__ act, int* __restrict__ nAct, int cap,
    int* __restrict__ overflow)
{
    const unsigned h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= size) return;
    const unsigned long long key = tab_key[h];
    if (key == ~0ull) return;
    const int x = -(int)(key >> 42) - 1, y = (int)((key >> 21) & 0x1fffffu), z = (int)(key & 0x1fffffu) - 1;
    push4(act, nAct, cap, overflow, make_int4(x, y, z, -tab_cnt[h]));
}

} // namespace ipcgpu

using namespace ipcgpu;

static void cell_pairs_pt(const Grid* gp, const SortedGrid& vg, const SortedGrid& tg, const SurfArgs& s, double radius, int first, int last, const PairOut& out, cudaStream_t st)
{
    if (last > first) k_cell_pairs_pt<<<nblk(last - first, 32 * kCellPairWarps), 32 * kCellPairWarps, 0, st>>>(gp, vg, tg, s.SVI, s.SF, s.nSF, radius, first, last, out);
}
static void cell_pairs_ee(const Grid* gp, const SortedGrid& eg, const SurfArgs& s, double radius, int first, int last, const PairOut& out, cudaStream_t st)
{
    if (last > first) k_cell_pairs_ee<<<nblk(last - first, 32 * kCellPairWarps), 32 * kCellPairWarps, 0, st>>>(gp, eg, s.SE, radius, first, last, out);
}

int contact_scan(ipcgpu_ctx* ctx, const int* in, int* out, int n)
{
    ContactWork& w = ctx->cw;
    size_t bytes = w.cub_tmp.n;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(w.cub_tmp.p, bytes, in, out, n, ctx->stream);
    if (e != cudaSuccess) {
        ctx->err = std::string("cub scan: ") + cudaGetErrorString(e);
        return IPCGPU_ERR_CUDA;
    }
    return IPCGPU_OK;
}

// buckets of the canonical order: first components in [-nV, max(nV, nSE)) (candidates: -svI - 1 or an edge index)
static int lex_buckets(const ipcgpu_ctx* ctx) { return std::max(ctx->nV, 1) + std::max(std::max(ctx->nV, ctx->nSE), 1); }

// perm = the permutation that sorts list[0, min(*n, cap)) lexicographically (companion last)
template <typename T>
static int lex_order_impl(ipcgpu_ctx* ctx, const T* list, const int2* comp, const int* n, int cap)
{
    ContactWork& w = ctx->cw;
    cudaStream_t st = ctx->stream;
    const int nB = lex_buckets(ctx);
    zero_words(w.cnt.p, (size_t)nB + 1, st);
    k_lex_count<<<kLexBlocks, 256, 0, st>>>(list, n, cap, ctx->nV, w.cnt.p);
    int rc = contact_scan(ctx, w.cnt.p, w.off.p, nB + 1);
    if (rc) return rc;
    CK(cudaMemcpyAsync(w.cnt.p, w.off.p, (size_t)nB * sizeof(int), cudaMemcpyDeviceToDevice, st)); // scatter cursors
    k_lex_scatter<<<kLexBlocks, 256, 0, st>>>(list, n, cap, ctx->nV, w.cnt.p, w.perm.p);
    k_lex_bucket_sort<<<nblk(nB, 256), 256, 0, st>>>(nB, w.off.p, list, comp, w.perm.p);
    ctx->launches += 6;
    return IPCGPU_OK;
}
int lex_order(ipcgpu_ctx* ctx, const int4* list, const int2* comp, const int* n, int cap) { return lex_order_impl(ctx, list, comp, n, cap); }
int lex_order(ipcgpu_ctx* ctx, const int2* list, const int* n, int cap) { return lex_order_impl(ctx, list, (const int2*)nullptr, n, cap); }

// data[0, min(*n, cap)) = data[perm[i]], `words` 8-byte words per element
void permute(ipcgpu_ctx* ctx, void* data, int words, const int* n, int cap)
{
    ContactWork& w = ctx->cw;
    k_permute_words<<<kLexBlocks, 256, 0, ctx->stream>>>(static_cast<const unsigned long long*>(data), w.perm.p, n, cap, words, w.words.p);
    k_copy_words<<<kLexBlocks, 256, 0, ctx->stream>>>(w.words.p, n, cap, words, static_cast<unsigned long long*>(data));
    ctx->launches += 2;
}

// act, para (with para_e) and, when the candidates were wanted, cand in canonical order, sized by the device counters
int contact_sort_lists(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    int rc;
    if ((rc = lex_order(ctx, w.act.p, nullptr, w.counters.p + 0, w.cap))) return rc;
    permute(ctx, w.act.p, 2, w.counters.p + 0, w.cap);
    if ((rc = lex_order(ctx, w.para.p, w.para_e.p, w.counters.p + 2, w.cap))) return rc;
    permute(ctx, w.para.p, 2, w.counters.p + 2, w.cap);
    permute(ctx, w.para_e.p, 1, w.counters.p + 2, w.cap);
    if (w.want_cand) {
        if ((rc = lex_order(ctx, w.cand.p, w.counters.p + 3, 4 * w.cap))) return rc;
        permute(ctx, w.cand.p, 1, w.counters.p + 3, 4 * w.cap);
    }
    return IPCGPU_OK;
}

int contact_alloc(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    const int nSE = ctx->nSE, nSF = ctx->nSF, nSV = ctx->nSV;
    const size_t nAll = (size_t)std::max(nSE + nSF + nSV, 1); // triangles, edges and surface vertices share one sorted array
    const int cap = std::max(ctx->pair_capacity, 1024);
    bool ok = w.vbox.reserve(std::max(nSV, 1)) && w.ebox.reserve(std::max(nSE, 1)) && w.tbox.reserve(std::max(nSF, 1)) && w.bounds.reserve(8) && w.grid.reserve(2)
        && w.centries.reserve(nAll) && w.ckeys.reserve(nAll) && w.cvals.reserve(nAll) && w.key_tmp.reserve(nAll) && w.val_tmp.reserve(nAll)
        && w.act.reserve(cap) && w.dup.reserve(cap) && w.para.reserve(cap) && w.para_e.reserve(cap) && w.cand.reserve((size_t)4 * cap)
        && w.counters.reserve(16) && w.skey.reserve((size_t)4 * cap) && w.sidx.reserve((size_t)4 * cap);
    // canonical order: bucket counts and offsets, the permutation (up to 4 cap candidates), the permuted words (up to 6 per friction basis)
    const size_t nB = (size_t)lex_buckets(ctx) + 1;
    ok = ok && w.cnt.reserve(nB) && w.off.reserve(nB) && w.perm.reserve((size_t)4 * cap) && w.words.reserve((size_t)6 * cap);
    // PP/PE duplicate-merge table: the largest power of two that fits skey / sidx, at most 2^20 slots (cleared every build)
    w.dup_tab = 1024;
    while (w.dup_tab * 2 <= (unsigned)std::min<size_t>((size_t)4 * cap, (size_t)1 << 20)) w.dup_tab *= 2;
    // pair Hessians of the barrier stage (144 doubles per pair) + stencil rows + makePD flags, sized by the pair capacity so that the
    // barrier stage needs no host-side size
    ok = ok && w.bHraw.reserve((size_t)cap * 144) && w.brows.reserve((size_t)cap * 4) && w.bpsd.reserve(cap) && w.bpartials.reserve(1024);
    if (ctx->nranks > 1) { // exchange of the pair lists between ranks (ipcgpu_set_contact_partition)
        w.xcap = std::max(1, std::min(std::min(cap, 1 << 16), ctx->exchange_capacity)); // pairs per rank and list in one message (ipcgpu_set_exchange_capacity)
        w.xstride = 1 + 2 * (size_t)w.xcap + (size_t)(w.xcap + 1) / 2;
        ok = ok && w.xsend.reserve(w.xstride) && w.xrecv.reserve(w.xstride * ctx->nranks) && w.gact.reserve(cap) && w.gpara.reserve(cap) && w.gpara_e.reserve(cap);
    }
    w.bp_cap = (size_t)24 * std::max(std::max(nSE, nSV), 1024);
    ok = ok && w.bp_pairs.reserve(2 * w.bp_cap) && w.cell_cnt.reserve((size_t)3 * kGridCells + 8) && w.cell_off.reserve((size_t)3 * kGridCells + 8);
    if (!ok) {
        ctx->err = "contact workspace allocation failed";
        return IPCGPU_ERR_CUDA;
    }
    size_t b1 = 0, b2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b1, (int*)nullptr, (int*)nullptr, (int)(3 * kGridCells + 1)); // dense cell-offset table
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int*)nullptr, (int*)nullptr, (int)nB);                   // bucket offsets of the order
    if (!w.cub_tmp.reserve(std::max(b1, b2) + 256)) {
        ctx->err = "cub temp allocation failed";
        return IPCGPU_ERR_CUDA;
    }
    w.cap = cap;
    if (ctx->canonical_order == 2) return repro_alloc(ctx);
    return 0;
}

// build the sorted grids of the triangles and the edges in ONE pass: one emit, one radix sort (cell key + type bit), one gather of the
// quantised entries, one cell table
static int build_grids(ipcgpu_ctx* ctx, int nT, int nE, int nV)
{
    ContactWork& w = ctx->cw;
    cudaStream_t st = ctx->stream;
    const int n = nT + nE + nV;
    w.built_vertices = nV;
    if (n <= 0) return 0;
    const size_t nTab = (size_t)3 * kGridCells + 1;
    zero_words(w.cell_cnt.p, nTab, st); // (kernels.h: not a memset)
    k_cell_count<<<nblk(n, 256), 256, 0, st>>>(nT, nE, nV, w.tbox.p, w.ebox.p, w.vbox.p, w.grid.p, w.cell_cnt.p, w.key_tmp.p, w.val_tmp.p);
    size_t bytes = w.cub_tmp.n;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(w.cub_tmp.p, bytes, w.cell_cnt.p, w.cell_off.p, (int)nTab, st);
    if (e != cudaSuccess) {
        ctx->err = std::string("cub cell-offset scan: ") + cudaGetErrorString(e);
        return IPCGPU_ERR_CUDA;
    }
    k_cell_scatter<<<nblk(n, 256), 256, 0, st>>>(nT, nE, nV, w.tbox.p, w.ebox.p, w.vbox.p, w.grid.p, w.cell_off.p, w.key_tmp.p, w.val_tmp.p, w.ckeys.p, w.cvals.p,
        reinterpret_cast<uint4*>(w.centries.p));
    ctx->launches += 5;
    return 0;
}
// views of the combined sorted array: triangles are entries [0, nSF), edges [nSF, nSF + nSE) (positions are absolute in both views)
SortedGrid tri_grid(const ipcgpu_ctx* ctx)
{
    const ContactWork& w = ctx->cw;
    return SortedGrid{ w.ckeys.p, w.cvals.p, w.centries.p, ctx->nSF, w.cell_off.p, 0u };
}
SortedGrid edge_grid(const ipcgpu_ctx* ctx)
{
    const ContactWork& w = ctx->cw;
    return SortedGrid{ w.ckeys.p, w.cvals.p, w.centries.p, ctx->nSE, w.cell_off.p, 1u << kGridCellsLog2 };
}

SortedGrid vertex_grid(const ipcgpu_ctx* ctx) // surface-vertex entries [nSF + nSE, nSF + nSE + built_vertices) of the combined sorted array
{
    const ContactWork& w = ctx->cw;
    return SortedGrid{ w.ckeys.p, w.cvals.p, w.centries.p, w.built_vertices, w.cell_off.p, 2u << kGridCellsLog2 };
}

SurfArgs surf_args(const ipcgpu_ctx* ctx)
{
    SurfArgs s;
    s.nV = ctx->nV; s.V = ctx->V.p; s.Vrest = ctx->Vrest.p; s.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    s.vCoDim = ctx->has_codim ? ctx->vCoDim.p : nullptr;
    s.nVdof = ctx->nVdof; s.ee_as_vf = ctx->ee_as_vf;
    s.nSV = ctx->nSV; s.SVI = ctx->SVI.p; s.nSE = ctx->nSE; s.SE = ctx->SE.p; s.nSF = ctx->nSF; s.SF = ctx->SF.p;
    return s;
}

// boxes of vertices/edges/triangles at the current positions, grid parameters, and the sorted grids
int boxes_and_grid(ipcgpu_ctx* ctx, double radius, bool with_vertex_boxes)
{
    ContactWork& w = ctx->cw;
    cudaStream_t st = ctx->stream;
    const SurfArgs s = surf_args(ctx);
    k_bounds_init<<<1, 32, 0, st>>>(w.bounds.p);
    if (with_vertex_boxes && s.nSV > 0) k_boxes<<<nblk(s.nSV, 256), 256, 0, st>>>(s, 0, w.vbox.p, w.bounds.p);
    if (s.nSE > 0) k_boxes<<<nblk(s.nSE, 256), 256, 0, st>>>(s, 1, w.ebox.p, w.bounds.p);
    if (s.nSF > 0) k_boxes<<<nblk(s.nSF, 256), 256, 0, st>>>(s, 2, w.tbox.p, w.bounds.p);
    k_grid_params<<<1, 32, 0, st>>>(w.bounds.p, radius, w.axis_bits, w.grid.p, ctx->iter.p);
    ctx->launches += 5;
    return build_grids(ctx, s.nSF, s.nSE, with_vertex_boxes ? s.nSV : 0);
}

// pack this rank's lists, allgather, rebuild the global lists (called by ipcgpu_constraint_set around its all-gather)
void contact_pack_lists(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    k_pack_lists<<<kSMs, 256, 0, ctx->stream>>>(w.act.p, w.para.p, w.para_e.p, w.counters.p, w.xcap, w.xsend.p, &ctx->iter.p->flags[FLAG_EXCHANGE_CAPACITY]);
    ++ctx->launches;
}
void contact_unpack_lists(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    k_unpack_lists<<<kSMs, 256, 0, ctx->stream>>>(w.xrecv.p, ctx->nranks, w.xcap, w.xstride, w.gact.p, w.gpara.p, w.gpara_e.p, w.cap, w.counters.p + 10,
        &ctx->iter.p->flags[FLAG_EXCHANGE_CAPACITY]);
    ++ctx->launches;
}

// read the list sizes back (one synchronisation); only the host-facing calls need them
int contact_sync_counts(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    int* h = ctx->staging->contact;
    CK(cudaMemcpyAsync(h, w.counters.p, 8 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (h[4]) {
        ctx->err = "constraint-set capacity exceeded (raise it with ipcgpu_set_pair_capacity)";
        return IPCGPU_ERR_CAPACITY;
    }
    w.nC = h[0];
    w.nP = h[2];
    w.nK = w.want_cand ? h[3] : 0;
    return 0;
}

// SelfCollisionHandler::computeConstraintSet on the device.  Nothing is read back unless the caller asks for the sizes (nC / nPara /
// nCand non-NULL): the lists and their counts stay on the device and every consumer (barrier_*, partial CCD) takes the counts from there.
int contact_constraint_set(ipcgpu_ctx* ctx, double dHat, int wantCand, int* nC, int* nPara, int* nCand)
{
    ContactWork& w = ctx->cw;
    cudaStream_t st = ctx->stream;
    const SurfArgs s = surf_args(ctx);
    const double radius = sqrt(dHat);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_HASH);
    int rc;
    if ((rc = boxes_and_grid(ctx, radius, true))) return rc; // (vertex entries for the cell-centric PT kernel)
    ctx->prof_end(pe);

    pe = ctx->prof_begin(IPCGPU_STAGE_CONSTRAINT_SET);
    CK(cudaMemsetAsync(w.counters.p, 0, 16 * sizeof(int), st));
    CsOut out;
    out.act = w.act.p; out.nAct = w.counters.p + 0; out.capAct = w.cap;
    out.dup = w.dup.p; out.nDup = w.counters.p + 1; out.capDup = w.cap;
    out.para = w.para.p; out.para_e = w.para_e.p; out.nPara = w.counters.p + 2; out.capPara = w.cap;
    out.cand = w.cand.p; out.nCand = w.counters.p + 3; out.capCand = 4 * w.cap;
    out.overflow = w.counters.p + 4;
    const SortedGrid tg = tri_grid(ctx), eg = edge_grid(ctx);
    // partitioned mode (ipcgpu_set_contact_partition): this rank only issues its share of the queries (the reference's own loop
    // decomposition, :2168 / :2271), so its lists hold a disjoint part of the global sets
    int v0 = 0, v1 = s.nSV, e0 = 0, e1 = s.nSE;
    if (ctx->partition_contact && ctx->nranks > 1) {
        v0 = (int)((long long)s.nSV * ctx->rank / ctx->nranks); v1 = (int)((long long)s.nSV * (ctx->rank + 1) / ctx->nranks);
        e0 = (int)((long long)s.nSE * ctx->rank / ctx->nranks); e1 = (int)((long long)s.nSE * (ctx->rank + 1) / ctx->nranks);
    }
    // phase 1 (boxes only) -> pair lists ; phase 2 (exact classification) over the lists.  The list sizes stay on the device:
    // phase 2 is launched over the list capacity and surplus threads exit.
    unsigned* nPairs = reinterpret_cast<unsigned*>(w.counters.p + 8); // [8] PT pairs, [9] EE pairs
    PairOut ppt{ w.bp_pairs.p, nPairs, (unsigned)w.bp_cap, w.counters.p + 4 }, pee{ w.bp_pairs.p + w.bp_cap, nPairs + 1, (unsigned)w.bp_cap, w.counters.p + 4 };
    if (v1 > v0 && s.nSF > 0) {
        cell_pairs_pt(w.grid.p, vertex_grid(ctx), tg, s, radius, s.nSF + s.nSE + v0, s.nSF + s.nSE + v1, ppt, st); // vertex entries: by sorted position
        k_classify_pt<<<kSMs * 8, 128, 0, st>>>(s, ppt.pairs, ppt.n, ppt.cap, dHat, wantCand, out);
        ctx->launches += 2;
    }
    if (e1 > e0 && s.nSE > 1) {
        cell_pairs_ee(w.grid.p, eg, s, radius, s.nSF + e0, s.nSF + e1, pee, st); // edge entries sit behind the triangles
        k_classify_ee<<<kSMs * 8, 128, 0, st>>>(s, pee.pairs, pee.n, pee.cap, dHat, wantCand, out);
        ctx->launches += 2;
    }
    // merge PP/PE duplicates into the active list with negative multiplicities (:2434-2476)
    if (ctx->nV < (1 << 21) - 2) { // (x,y,z) packs into one 64-bit key: fixed-size table
        CK(cudaMemsetAsync(w.skey.p, 0xff, (size_t)w.dup_tab * sizeof(unsigned long long), st));
        CK(cudaMemsetAsync(w.sidx.p, 0, (size_t)w.dup_tab * sizeof(int), st));
        k_dup_insert<<<kSMs * 2, 256, 0, st>>>(w.counters.p + 1, w.cap, w.dup.p, w.skey.p, w.sidx.p, w.dup_tab - 1, w.counters.p + 4);
        k_dup_emit<<<nblk(w.dup_tab, 256), 256, 0, st>>>(w.dup_tab, w.skey.p, w.sidx.p, w.act.p, w.counters.p + 0, w.cap, w.counters.p + 4);
        ctx->launches += 2;
    }
    else { // huge meshes: equal entries are adjacent in canonical order
        if ((rc = lex_order(ctx, w.dup.p, nullptr, w.counters.p + 1, w.cap))) return rc;
        permute(ctx, w.dup.p, 2, w.counters.p + 1, w.cap);
        k_merge_dups<<<kLexBlocks, 256, 0, st>>>(w.counters.p + 1, w.cap, w.dup.p, w.act.p, w.counters.p + 0, w.counters.p + 4);
        ++ctx->launches;
    }
    w.want_cand = wantCand != 0;
    w.nC = w.nP = w.nK = -1; // unknown on the host until somebody asks
    if ((nC || nPara || nCand) && (rc = contact_sync_counts(ctx))) return rc;
    // deterministic output order (the reference's own order is scheduling dependent, :2176, :2282); at level 2 the gather indices too
    if (ctx->canonical_order >= 1 && (rc = contact_sort_lists(ctx))) return rc;
    ctx->rw.lists_ready = false;
    if (repro_on(ctx) && (rc = repro_contact_lists(ctx))) return rc;
    k_publish_counts<<<1, 32, 0, st>>>(w.counters.p, wantCand, ctx->iter.p);
    ++ctx->launches;
    ctx->prof_end(pe);
    if (nC) *nC = w.nC;
    if (nPara) *nPara = w.nP;
    if (nCand) *nCand = w.nK;
    return 0;
}
