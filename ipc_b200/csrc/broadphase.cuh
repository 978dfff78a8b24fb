// broadphase.cuh -- sort-based uniform grid shared by the constraint-set build and the CCD broad phase.
//
// Replaces SpatialHash<3> (src/Utils/SpatialHash.hpp:46-201 static build, :589-750 swept build, and the queries
// :203-229, :375-421, :752-832), whose std::unordered_map<int, std::vector<int>> and serial inserts do not map to a GPU.
// Design: every edge / triangle registers its AABB in at most 8 cells of a grid whose cell edge is >= the largest
// (inflated) primitive extent of this frame, the (cell,id) entries are radix-sorted by cell (CUB), and a query walks
// the <= 8 cells of its own box with a binary search per cell.  A pair is reported exactly once, from the
// lexicographically smallest common cell of the two boxes.  The grid is only an accelerator: what decides membership
// is the exact test applied afterwards (d < dHat for the constraint set; the reference's own voxel-AABB overlap for CCD
// candidates), so results do not depend on the cell size chosen here.
#pragma once
#include "common.cuh"
#include "contact.cuh"
#include "broadphase_types.h"

namespace ipcgpu {


// monotone map double -> uint64 (handles negatives) for atomicMin/Max on coordinates
DEV unsigned long long flip_ord(double x)
{
    unsigned long long u = (unsigned long long)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
DEV double unflip_ord(unsigned long long u)
{
    u = (u >> 63) ? (u & 0x7fffffffffffffffull) : ~u;
    return __longlong_as_double((long long)u);
}

DEV void cell_range(const Grid& g, const Box& b, int* c0, int* c1)
{
    const double o[3] = { g.ox, g.oy, g.oz };
    const int n[3] = { g.nx, g.ny, g.nz };
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        int lo = (int)floor((b.lo[a] - o[a]) * g.inv_h), hi = (int)floor((b.hi[a] - o[a]) * g.inv_h);
        c0[a] = min(max(lo, 0), n[a] - 1);
        c1[a] = min(max(hi, 0), n[a] - 1);
    }
}
DEV unsigned long long cell_key(const Grid& g, int ix, int iy, int iz) { return ((unsigned long long)iz * g.ny + iy) * g.nx + ix; }

DEV int lower_bound_u64(const unsigned long long* __restrict__ keys, int n, unsigned long long k)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

DEV int upper_bound_u64(const unsigned long long* __restrict__ keys, int n, unsigned long long k)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (keys[mid] <= k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Grid v2: every primitive is registered ONCE, in the cell of its box's lower corner.  With cell edge >= (largest box extent +
// 2*radius), a box starting in cell c ends in c or c+1, and a query box inflated by `radius` covers cells q0..q1 (q1 <= q0+1), so
// every partner starts in [q0-1, q1] per axis: at most 3x3 rows of <= 3 consecutive cells.  Entries are sorted by cell key; an
// open-addressing table (cell key -> index of the first entry of that cell) replaces binary searches: the <= 27 cell lookups of a
// query run on 27 lanes at once.
constexpr int kGridCellsLog2 = 20;                  // the grid holds at most 2^20 cells (k_grid_params enlarges the cells beyond that)
constexpr unsigned kGridCells = 1u << kGridCellsLog2;
struct SortedGrid {
    const unsigned* keys;   // per entry: type << 20 | cell, ascending (counting sort by cell: round 2, second half)
    const int* ids;         // primitive id per entry
    const QEntry* ent;      // quantised box + id per entry, in sorted order (coalesced 16-byte candidate scan)
    int n;
    const int* cell_off;    // DENSE table: entries of cell c of type t are positions [cell_off[t << 20 | c], cell_off[(t << 20 | c) + 1])
    unsigned type_bit;      // type << 20: triangles 0, edges 1, surface vertices 2 share ONE sorted array and ONE table
};

// entries registered in one cell: two adjacent words of the dense offset table (an empty cell is an empty range AT its place in the order)
DEV int2 cell_lookup(const SortedGrid& sg, unsigned cell)
{
    const unsigned i = sg.type_bit | cell;
    return make_int2(__ldg(sg.cell_off + i), __ldg(sg.cell_off + i + 1));
}

// conservative 16-bit quantisation of a box on the grid's lattice
struct QBox {
    int lo[3], hi[3];
};
DEV QBox quantize_box(const Grid& g, const Box& b)
{
    const double o[3] = { g.ox, g.oy, g.oz };
    QBox q;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        q.lo[a] = min(max((int)floor((b.lo[a] - o[a]) * g.q_inv) - 1, 0), 65535);
        q.hi[a] = min(max((int)ceil((b.hi[a] - o[a]) * g.q_inv) + 1, 0), 65535);
    }
    return q;
}
DEV bool qoverlap(const QBox& a, const uint4& e)
{
    // e = {lo0 | lo1 << 16, lo2 | hi0 << 16, hi1 | hi2 << 16, id}
    const int l0 = e.x & 0xffff, l1 = e.x >> 16, l2 = e.y & 0xffff, h0 = e.y >> 16, h1 = e.z & 0xffff, h2 = e.z >> 16;
    return !(a.lo[0] > h0 || l0 > a.hi[0] || a.lo[1] > h1 || l1 > a.hi[1] || a.lo[2] > h2 || l2 > a.hi[2]);
}

DEV bool boxes_overlap(const Box& a, const Box& b)
{
    return !(a.lo[0] > b.hi[0] || b.lo[0] > a.hi[0] || a.lo[1] > b.hi[1] || b.lo[1] > a.hi[1] || a.lo[2] > b.hi[2] || b.lo[2] > a.hi[2]);
}

// warp-cooperative scan: calls f(hit, id) with hit = true on every registered primitive whose (quantised) box overlaps the (already
// inflated) query box.  All 32 lanes must call this together and f is called by all 32 lanes together (hit = false on the lanes
// that have nothing), so that f can aggregate its output over the warp.
// The <= 27 cells are looked up by 27 lanes at once; the <= 9 rows (runs of consecutive entries) are then walked as ONE flattened
// index range, so that a query costs ceil(total/32) independent, coalesced loads instead of a dependent chain per row.
// `after` >= 0 restricts the walk to entries at sorted positions > after: a query that is itself entry `after` of the same grid
// then sees each of its partners from exactly one side (half the work of testing every pair twice and dropping one).
template <typename F>
DEV void warp_scan_candidates(const Grid& g, const SortedGrid& sg, const Box& qb, int lane, F f, int after = -1)
{
    const unsigned full = 0xffffffffu;
    int c0[3], c1[3];
    cell_range(g, qb, c0, c1);
    const int x0 = max(c0[0] - 1, 0), x1 = c1[0];
    const int y0 = max(c0[1] - 1, 0), z0 = max(c0[2] - 1, 0);
    const int ny = c1[1] - y0 + 1, nz = c1[2] - z0 + 1; // <= 3 each
    const int nrows = ny * nz;
    // lane 3r+dx looks up cell (x0+dx) of row r
    int2 mine = make_int2(0x7fffffff, -1);
    {
        const int r = lane / 3, dx = lane - 3 * r;
        if (r < nrows && x0 + dx <= x1) mine = cell_lookup(sg, (unsigned)cell_key(g, x0 + dx, y0 + r % ny, z0 + r / ny));
    }
    // lane L (and L+9, L+18, ...) gets the run of row L % 9: cells of one row are consecutive keys => consecutive entries
    const int rr = lane % 9;
    const int s0 = __shfl_sync(full, mine.x, 3 * rr), s1 = __shfl_sync(full, mine.x, 3 * rr + 1), s2 = __shfl_sync(full, mine.x, 3 * rr + 2);
    const int e0 = __shfl_sync(full, mine.y, 3 * rr), e1 = __shfl_sync(full, mine.y, 3 * rr + 1), e2 = __shfl_sync(full, mine.y, 3 * rr + 2);
    const int rend = max(e0, max(e1, e2));
    const int rstart = (rend > 0) ? max(min(s0, min(s1, s2)), after + 1) : 0; // empty row: harmless start
    const int rlen = (lane < 9 && rend > rstart) ? rend - rstart : 0;
    int incl = rlen; // inclusive prefix over lanes 0..8
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
        const int t = __shfl_up_sync(full, incl, o);
        if (lane >= o) incl += t;
    }
    int inc[9], st[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) {
        inc[r] = __shfl_sync(full, incl, r);
        st[r] = __shfl_sync(full, rstart, r);
    }
    const int total = inc[8];
    auto locate = [&](int j) { // flattened index -> entry
        int k = st[0] + j;
#pragma unroll
        for (int r = 1; r < 9; ++r)
            if (j >= inc[r - 1]) k = st[r] + (j - inc[r - 1]);
        return k;
    };
    // software pipeline: the load of iteration i+1 is in flight while f handles iteration i
    const QBox qq = quantize_box(g, qb);
    const uint4* __restrict__ ent = reinterpret_cast<const uint4*>(sg.ent);
    uint4 en = make_uint4(0u, 0u, 0u, 0u);
    if (lane < total) en = __ldg(ent + locate(lane));
    for (int j = lane; j - lane < total; j += 32) {
        const uint4 e = en;
        const bool in = j < total;
        if (j + 32 < total) en = __ldg(ent + locate(j + 32));
        f(in && qoverlap(qq, e), (int)e.w); // convergent: every lane calls f
    }
}

// Pair output of the broad phase: a list, its device-resident size, its capacity and the overflow flag.
struct PairOut {
    int2* pairs;
    unsigned* n;
    unsigned cap;
    int* overflow;
};
constexpr int kPairQueriesPerWarp = 8; // queries handled by one warp of a warp-per-query kernel (warp_scan_candidates)

} // namespace ipcgpu
