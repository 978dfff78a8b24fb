// pattern.cu -- the contact-augmented Hessian sparsity pattern, built and owned by the device (ipcgpu_enable_device_pattern /
// ipcgpu_update_pattern).
//
// Reference being stood in for: Optimizer::computePrecondMtr's pattern step (Optimizer.cpp:3556-3595): vNeighbor of the mesh
// (Mesh.cpp:470-493) augmented by SelfCollisionHandler::augmentConnectivity over the active set, the mollified para-EE set and, with
// friction, the lagged set (SelfCollisionHandler.cpp:330-415), then LinSysSolver::set_pattern (LinSysSolver.hpp:63-111).
//
// The mesh part is static: built once on the host at enable time as an upper-neighbour list per vertex.  An update only deals with the
// EXTRA blocks, the contact neighbour pairs (lo < hi) that are not mesh neighbours:
//   1. k_pattern_keys<false>: one thread per entry of the three sets counts its extra keys per lower vertex (a pair with a vertex of the
//      obstacle tail, or one that is already a mesh neighbour -- binary search in the mesh lists -- is dropped);
//   2. exclusive scan of the counts; k_pattern_check: do the raw keys fit the key buffer;
//   3. k_pattern_keys<true>: the same walk writes each key's upper vertex into its lower vertex's bucket;
//   4. k_pattern_rows: one thread per vertex sorts and de-duplicates its bucket and compares it with the extra neighbours of the pattern
//      in place -> the `changed` bit;
//   5. exclusive scan of the distinct counts; k_pattern_commit: new nnz, capacity check, version;
//   6. only when changed: k_pattern_write merges mesh and extra neighbours of every vertex into ia / ja and keeps the extra lists for the
//      next comparison; k_slot_offsets (elastic.cu) recomputes the CSR offsets of the elastic block slots.
// Every launch has a size fixed by nV and the capacities and reads its counts and gates from device memory, so an update is capturable.
#include "pair_common.cuh"
#include "abi.h"
#include <algorithm>
#include <cstddef>
#include <cub/cub.cuh>
#include <vector>

namespace ipcgpu {

struct PatArgs {
    const int4* cs; const int* nC;                        // active set (MMCVID) and its device count
    const int4* para; const int2* para_e; const int* nP;  // mollified set + (eI, eJ)
    const int4* fr; const int* nF;                        // lagged friction set (nullptr: not included)
    int cap, capF;                                        // list capacities (a count beyond them has raised a capacity flag already)
    const int* SE;                                        // SFEdges, interleaved
    int nVdof;
    const int* mptr; const int* mnbr;
};

DEV bool mesh_neighbour(const int* __restrict__ mptr, const int* __restrict__ mnbr, int lo, int hi)
{
    int a = mptr[lo], b = mptr[lo + 1];
    const int end = b;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (mnbr[m] < hi) a = m + 1;
        else b = m;
    }
    return a < end && mnbr[a] == hi;
}

template <bool FILL>
DEV void emit_pairs(const PatArgs& p, const int* v, int n, int* row_cnt, const int* row_off, int* bucket)
{
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j) {
            const int lo = min(v[i], v[j]), hi = max(v[i], v[j]);
            if (lo == hi || hi >= p.nVdof || mesh_neighbour(p.mptr, p.mnbr, lo, hi)) continue;
            if (FILL) bucket[row_off[lo] + atomicSub(&row_cnt[lo], 1) - 1] = hi; // (leaves row_cnt at zero for the next update)
            else atomicAdd(&row_cnt[lo], 1);
        }
}

template <bool FILL>
__global__ void __launch_bounds__(256) k_pattern_keys(PatArgs p, int* __restrict__ row_cnt, const int* __restrict__ row_off, int* __restrict__ bucket,
    const IterState* __restrict__ st)
{
    if (FILL && !st->pat_ok) return;
    const int nC = min(*p.nC, p.cap), nP = min(*p.nP, p.cap), nF = p.fr ? min(*p.nF, p.capF) : 0;
    const int total = nC + nP + nF;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const bool para = i >= nC && i < nC + nP;
        const PairStencil s = decode(i < nC ? p.cs[i] : para ? p.para[i - nC] : p.fr[i - nC - nP]);
        emit_pairs<FILL>(p, s.v, s.nv, row_cnt, row_off, bucket);
        const int2 e = para ? p.para_e[i - nC] : make_int2(-1, -1);
        if (e.x >= 0 && e.y >= 0) { // the two edges of a mollified pair
            const int v[4] = { p.SE[2 * e.x], p.SE[2 * e.x + 1], p.SE[2 * e.y], p.SE[2 * e.y + 1] };
            emit_pairs<FILL>(p, v, 4, row_cnt, row_off, bucket);
        }
    }
}

__global__ void k_pattern_check(const int* __restrict__ n_keys, long long key_cap, IterState* __restrict__ st)
{
    const int ok = (long long)*n_keys <= key_cap;
    st->pat_ok = ok;
    st->pat_diff = 0;
    if (!ok) st->flags[FLAG_PATTERN_CAPACITY] = 1;
}

// sort + de-duplicate the bucket of every vertex in place; compare with the extra neighbours of the current pattern
__global__ void __launch_bounds__(256) k_pattern_rows(int nV, const int* __restrict__ row_off, int* __restrict__ bucket, int* __restrict__ ucnt,
    const int* __restrict__ prev_ptr, const int* __restrict__ prev_nbr, IterState* __restrict__ st)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV || !st->pat_ok) return;
    int* b = bucket + row_off[v];
    const int n = row_off[v + 1] - row_off[v];
    for (int i = 1; i < n; ++i) { // (a few entries per vertex)
        const int x = b[i];
        int j = i - 1;
        while (j >= 0 && b[j] > x) { b[j + 1] = b[j]; --j; }
        b[j + 1] = x;
    }
    int u = 0;
    for (int i = 0; i < n; ++i)
        if (u == 0 || b[i] != b[u - 1]) b[u++] = b[i];
    ucnt[v] = u;
    const int p0 = prev_ptr[v];
    bool diff = prev_ptr[v + 1] - p0 != u;
    for (int i = 0; i < u && !diff; ++i) diff = prev_nbr[p0 + i] != b[i];
    if (diff) st->pat_diff = 1;
}

__global__ void k_pattern_commit(int nV, const int* __restrict__ mesh_pairs, const int* __restrict__ extra_pairs, long long nnz_cap, IterState* __restrict__ st)
{
    int changed = 0;
    if (st->pat_ok && st->pat_diff) {
        const long long nnz = 6ll * nV + 9ll * ((long long)*mesh_pairs + *extra_pairs);
        if (nnz <= nnz_cap) {
            changed = 1;
            st->pat_nnz = nnz;
            ++st->pat_version;
        }
        else st->flags[FLAG_PATTERN_CAPACITY] = 1; // the pattern in place stays, the fetch reports IPCGPU_ERR_CAPACITY
    }
    st->pat_changed = changed;
}

// LinSysSolver::set_pattern row layout: row 3v = [3v, 3v+1, 3v+2, 3n, 3n+1, 3n+2 for every neighbour n > v ascending]; rows 3v+1 and 3v+2
// drop the leading entries.  Vertex v's rows start at 6v + 9 (upper neighbours of all lower vertices).
__global__ void __launch_bounds__(256) k_pattern_write(int nV, int base, const int* __restrict__ mptr, const int* __restrict__ mnbr, const int* __restrict__ row_off,
    const int* __restrict__ bucket, const int* __restrict__ ucnt, const int* __restrict__ uoff, int* __restrict__ ia, int* __restrict__ ja, int* __restrict__ prev_ptr,
    int* __restrict__ prev_nbr, const IterState* __restrict__ st)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV || !st->pat_changed) return;
    const int m0 = mptr[v], mn = mptr[v + 1] - m0, xn = ucnt[v], x0 = uoff[v];
    const int* ex = bucket + row_off[v];
    const int k = mn + xn;
    const int r0 = 6 * v + 9 * (m0 + x0), r1 = r0 + 3 + 3 * k, r2 = r1 + 2 + 3 * k;
    ia[3 * v] = base + r0;
    ia[3 * v + 1] = base + r1;
    ia[3 * v + 2] = base + r2;
    if (v == nV - 1) ia[3 * nV] = base + r2 + 1 + 3 * k;
    const int c = base + 3 * v;
    ja[r0] = c; ja[r0 + 1] = c + 1; ja[r0 + 2] = c + 2;
    ja[r1] = c + 1; ja[r1 + 1] = c + 2;
    ja[r2] = c + 2;
    int o0 = r0 + 3, o1 = r1 + 2, o2 = r2 + 1;
    for (int i = 0, j = 0; i < mn || j < xn;) {
        const int n = (j >= xn || (i < mn && mnbr[m0 + i] < ex[j])) ? mnbr[m0 + i++] : ex[j++];
        const int cn = base + 3 * n;
#pragma unroll
        for (int q = 0; q < 3; ++q) { ja[o0 + q] = cn + q; ja[o1 + q] = cn + q; ja[o2 + q] = cn + q; }
        o0 += 3; o1 += 3; o2 += 3;
    }
    prev_ptr[v] = x0;
    for (int i = 0; i < xn; ++i) prev_nbr[x0 + i] = ex[i];
    if (v == nV - 1) prev_ptr[nV] = x0 + xn;
}

// a[ia[row0] - base, ia[row1] - base) = 0, the range read from the device-resident row starts
__global__ void __launch_bounds__(256) k_zero_csr_rows(const int* __restrict__ ia, int base, int row0, int row1, double* __restrict__ a)
{
    const long long b = ia[row0] - base, e = ia[row1] - base;
    for (long long i = b + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (long long)gridDim.x * blockDim.x) a[i] = 0.0;
}

void zero_csr_rows(const int* ia, int base, int row0, int row1, double* a, cudaStream_t st)
{
    k_zero_csr_rows<<<kSMs * 16, 256, 0, st>>>(ia, base, row0, row1, a);
}

} // namespace ipcgpu

using namespace ipcgpu;

// Mesh part + buffers + the mesh-only pattern in ia / ja (host, once per enable).  The caller refreshes the host mirrors.
int pattern_enable(ipcgpu_ctx* ctx, int index_base, uint64_t nnz_capacity)
{
    PatternWork& w = ctx->pw;
    const int nV = ctx->nV, nT = ctx->nT, nVdof = std::min(ctx->nVdof, nV);
    // vNeighbor (Mesh.cpp:470-493): tet edges and surface edges (SFEdges: the triangles' edges and the codimensional edges); pairs that
    // touch the obstacle tail are left out, its rows keep their diagonal block only
    std::vector<uint64_t> keys;
    keys.reserve((size_t)6 * nT + (size_t)ctx->nSE);
    auto add = [&](int a, int b) {
        const int lo = std::min(a, b), hi = std::max(a, b);
        if (lo != hi && hi < nVdof) keys.push_back(((uint64_t)lo << 32) | (uint32_t)hi);
    };
    const std::vector<int>& T = ctx->h_T;
    for (int t = 0; t < nT; ++t)
        for (int i = 0; i < 4; ++i)
            for (int j = i + 1; j < 4; ++j) add(T[(size_t)i * nT + t], T[(size_t)j * nT + t]);
    if (ctx->surface_ready && ctx->nSE > 0) {
        std::vector<int> se((size_t)2 * ctx->nSE);
        CK(cudaMemcpyAsync(se.data(), ctx->SE.p, se.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (int e = 0; e < ctx->nSE; ++e) add(se[2 * (size_t)e], se[2 * (size_t)e + 1]);
    }
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    const long long nPairs = (long long)keys.size();
    std::vector<int> mptr((size_t)nV + 1, 0), mnbr(std::max<size_t>(keys.size(), 1), 0);
    for (size_t i = 0; i < keys.size(); ++i) {
        ++mptr[(keys[i] >> 32) + 1];
        mnbr[i] = (int)(keys[i] & 0xffffffffu);
    }
    for (int v = 0; v < nV; ++v) mptr[v + 1] += mptr[v];
    const long long mesh_nnz = 6ll * nV + 9ll * nPairs;
    // Default capacity: the mesh pattern plus a quarter.  A contact block adds 9 entries to a vertex that already holds ~7 mesh neighbours
    // (~69 entries with its diagonal block), so a quarter is room for ~2 contact neighbours per vertex on average -- in a dense pile
    // (C5: 146 balls, every surface vertex near another ball) the contact blocks stay a few percent of the mesh's.
    const long long cap = nnz_capacity ? (long long)nnz_capacity : mesh_nnz + mesh_nnz / 4;
    if (cap < mesh_nnz || cap > 0x7fffffffll) {
        ctx->err = "ipcgpu_enable_device_pattern: the capacity must hold the mesh pattern (" + std::to_string(mesh_nnz) + " entries) and fit 32-bit offsets";
        return IPCGPU_ERR_ARG;
    }
    // raw extra keys before de-duplication: a contact block is emitted by several stencils (a PT pair's edge neighbours ...); 8 raw keys per
    // block the entry capacity leaves room for, at least 64 Ki
    const long long key_cap = std::max<long long>(8 * ((cap - mesh_nnz) / 9), 1 << 16);
    std::vector<int> ia((size_t)3 * nV + 1), ja((size_t)mesh_nnz);
    for (int v = 0; v < nV; ++v) {
        const int k = mptr[v + 1] - mptr[v];
        const int r0 = (int)(6ll * v + 9ll * mptr[v]), r1 = r0 + 3 + 3 * k, r2 = r1 + 2 + 3 * k;
        ia[3 * (size_t)v] = r0 + index_base; ia[3 * (size_t)v + 1] = r1 + index_base; ia[3 * (size_t)v + 2] = r2 + index_base;
        int o[3] = { r0, r1, r2 };
        for (int r = 0; r < 3; ++r)
            for (int c = r; c < 3; ++c) ja[o[r]++] = 3 * v + c + index_base;
        for (int i = mptr[v]; i < mptr[v + 1]; ++i)
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) ja[o[r]++] = 3 * mnbr[i] + c + index_base;
    }
    ia[(size_t)3 * nV] = (int)mesh_nnz + index_base;
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, nV + 1);
    const size_t n1 = (size_t)nV + 1;
    bool ok = w.mptr.upload(mptr.data(), n1, ctx->stream) && w.mnbr.upload(mnbr.data(), mnbr.size(), ctx->stream) && w.row_cnt.reserve(n1) && w.row_off.reserve(n1)
        && w.bucket.reserve((size_t)key_cap) && w.ucnt.reserve(n1) && w.uoff.reserve(n1) && w.prev_ptr.reserve(n1) && w.prev_nbr.reserve((size_t)key_cap)
        && w.scan_tmp.reserve(std::max<size_t>(scan_bytes, 1)) && ctx->ia.upload(ia.data(), ia.size(), ctx->stream) && ctx->ja.reserve((size_t)cap)
        && ctx->a.reserve((size_t)cap);
    if (!ok) {
        ctx->err = "ipcgpu_enable_device_pattern: allocation or upload failed";
        return IPCGPU_ERR_CUDA;
    }
    CK(cudaMemcpyAsync(ctx->ja.p, ja.data(), ja.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(ctx->a.p, 0, (size_t)cap * sizeof(double), ctx->stream));
    for (int* p : { w.row_cnt.p, w.ucnt.p, w.prev_ptr.p }) CK(cudaMemsetAsync(p, 0, n1 * sizeof(int), ctx->stream)); // no extra blocks yet
    {   // result of the "last update": the mesh pattern, unchanged, version 0
        struct { long long nnz; unsigned long long version; int changed, ok, diff, pad; } r = { mesh_nnz, 0ull, 0, 1, 0, 0 };
        static_assert(sizeof(r) == offsetof(IterState, kappa) - offsetof(IterState, pat_nnz), "IterState pattern words");
        CK(cudaMemcpyAsync(reinterpret_cast<char*>(ctx->iter.p) + offsetof(IterState, pat_nnz), &r, sizeof(r), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream)); // (host vectors and r go out of scope)
    }
    w.scan_bytes = scan_bytes;
    w.mesh_pairs = nPairs;
    w.mesh_nnz = mesh_nnz;
    w.nnz_cap = cap;
    w.key_cap = key_cap;
    w.requested_cap = nnz_capacity;
    ctx->n_rows = 3 * nV;
    ctx->nnz = (int)mesh_nnz;
    ctx->index_base = index_base;
    ctx->h_ia.assign(ia.begin(), ia.end());
    return IPCGPU_OK;
}

// enqueue one update on the main stream; the lists are those the barrier stages read (`lists`), plus the lagged friction set on request
int pattern_update(ipcgpu_ctx* ctx, const BarrierArgs& lists, bool with_friction)
{
    PatternWork& w = ctx->pw;
    ContactWork& cw = ctx->cw;
    cudaStream_t st = ctx->stream;
    const int nV = ctx->nV;
    PatArgs p;
    p.cs = lists.cs; p.nC = lists.nC; p.para = lists.para; p.para_e = lists.para_e; p.nP = lists.nP;
    p.fr = with_friction ? cw.fr_cs.p : nullptr; p.nF = with_friction ? cw.fr_n.p : nullptr;
    p.cap = std::max(cw.cap, 0); p.capF = ctx->pair_capacity; // (the exchanged global lists have the same capacity)
    p.SE = ctx->SE.p; p.nVdof = ctx->nVdof;
    p.mptr = w.mptr.p; p.mnbr = w.mnbr.p;
    IterState* it = ctx->iter.p;
    const int gv = (nV + 255) / 256;
    size_t bytes = w.scan_bytes;
    k_pattern_keys<false><<<kSMs * 4, 256, 0, st>>>(p, w.row_cnt.p, w.row_off.p, w.bucket.p, it);
    CK(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, bytes, w.row_cnt.p, w.row_off.p, nV + 1, st));
    k_pattern_check<<<1, 1, 0, st>>>(w.row_off.p + nV, w.key_cap, it);
    k_pattern_keys<true><<<kSMs * 4, 256, 0, st>>>(p, w.row_cnt.p, w.row_off.p, w.bucket.p, it);
    k_pattern_rows<<<gv, 256, 0, st>>>(nV, w.row_off.p, w.bucket.p, w.ucnt.p, w.prev_ptr.p, w.prev_nbr.p, it);
    bytes = w.scan_bytes;
    CK(cub::DeviceScan::ExclusiveSum(w.scan_tmp.p, bytes, w.ucnt.p, w.uoff.p, nV + 1, st));
    k_pattern_commit<<<1, 1, 0, st>>>(nV, w.mptr.p + nV, w.uoff.p + nV, w.nnz_cap, it);
    k_pattern_write<<<gv, 256, 0, st>>>(nV, ctx->index_base, w.mptr.p, w.mnbr.p, w.row_off.p, w.bucket.p, w.ucnt.p, w.uoff.p, ctx->ia.p, ctx->ja.p, w.prev_ptr.p,
        w.prev_nbr.p, it);
    slot_offsets(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->ia.p, ctx->ja.p, ctx->index_base, ctx->slot_off.p, ctx->flag.p, st, &it->pat_changed);
    ctx->launches += 9;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}
