// repro.cu -- the reproducible mode (ipcgpu_set_canonical_order(ctx, 2)), sm_90a: the per-vertex gather indices of the fixed-order contact
// sums (repro.cuh, DESIGN.md section 3.20).  The lists arrive in canonical order (constraint.cu's lex_order / permute).
//
// Index.  The contributions of a list (gradient: one per stencil vertex, key = list position and local vertex; Hessian: one per upper
// 3x3 block, row = its lower vertex, key = column vertex, list position, block) are counted per vertex, scanned, scattered and sorted per
// vertex on the pattern of the canonical order.  Built where the list is produced; the term calls then only stage and gather.
#include "repro.cuh"
#include "abi.h"
#include <algorithm>

namespace ipcgpu {

// ---- fixed-order gradient gather -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_repro_gather_g(int nV, VertexIndex idx, const double* __restrict__ stage, unsigned long long lo, unsigned long long hi,
    double* __restrict__ g)
{
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nV; v += gridDim.x * blockDim.x) {
        const int b = idx.ptr[v], e = idx.ptr[v + 1];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        bool any = false;
        for (int j = b; j < e; ++j) {
            const unsigned long long k = idx.key[j];
            if (k < lo || k >= hi) continue;
            s0 += stage[3 * k];
            s1 += stage[3 * k + 1];
            s2 += stage[3 * k + 2];
            any = true;
        }
        if (any) {
            g[3 * (size_t)v] += s0;
            g[3 * (size_t)v + 1] += s1;
            g[3 * (size_t)v + 2] += s2;
        }
    }
}
void repro_gather_g(int nV, const VertexIndex& idx, const double* stage, unsigned long long lo, unsigned long long hi, double* g, cudaStream_t st)
{
    k_repro_gather_g<<<kSMs * 2, 256, 0, st>>>(nV, idx, stage, lo, hi, g);
}

namespace {

constexpr int kReproBlocks = kSMs * 4;

// ---- per-vertex gather indices -------------------------------------------------------------------------------------------------------
enum { kIdxGrad = 0, kIdxBarrierH, kIdxFrictionH };
// the lists an index is built from: items [0, *nC) of cs, then [0, *nP) of para (nP nullable)
struct IndexSrc {
    const int4* cs; const int* nC;
    const int4* para; const int2* para_e; const int* nP;
    const int* SE;
    int cap;
};
template <int kMode, typename Emit>
DEV void index_item(const IndexSrc& s, int t, int nC, Emit emit)
{
    const bool is_para = t >= nC;
    const int c = is_para ? t - nC : t;
    const int4 mm = is_para ? s.para[c] : s.cs[c];
    const PairStencil ps = decode(mm);
    if (kMode == kIdxGrad) { // keys as k_barrier_gradient / k_friction_gradient stage them
        // (unrolled with a guard: the stencil arrays stay in registers)
        if (is_para) {
            int ev[4];
            para_edge_stencil(mm, s.para_e[c], s.SE, ev);
#pragma unroll
            for (int k = 0; k < 4; ++k) emit(ev[k], gkey_para_edge(s.cap, c, k));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (k < ps.nv) emit(ps.v[k], is_para ? gkey_para_dist(s.cap, c, k) : gkey_active(c, k));
    }
    else if (kMode == kIdxBarrierH) { // the blocks k_barrier_hessian_scatter adds, slot t (active, then mollified) of the fixed-slot build
        if (t >= s.cap) return;        // (beyond the slots: the build raises FLAG_SET_CAPACITY)
        int rows[4];
        hessian_rows(mm, ps, is_para, s.para_e, c, s.SE, rows);
        for (int bi = 0; bi < 4; ++bi)
            for (int bj = 0; bj < 4; ++bj)
                if (upper_block(rows, bi, bj)) emit(rows[bi], hkey(rows[bj], t, bi, bj));
    }
    else { // the blocks k_friction_hessian adds
        for (int bi = 0; bi < ps.nv; ++bi)
            for (int bj = bi; bj < ps.nv; ++bj) emit(min(ps.v[bi], ps.v[bj]), hkey(max(ps.v[bi], ps.v[bj]), c, bi, bj));
    }
}
// kScatter false: cnt[v] += entries of v; true: key[atomicAdd(cur[v], 1)] = key (the order inside a vertex is fixed by k_index_sort)
template <int kMode, bool kScatter>
__global__ void __launch_bounds__(128) k_index_emit(IndexSrc s, int* __restrict__ cnt, unsigned long long* __restrict__ key)
{
    const int nC = min(*s.nC, s.cap), n = nC + (s.nP ? min(*s.nP, s.cap) : 0);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x)
        index_item<kMode>(s, t, nC, [&](int v, unsigned long long k) {
            if (kScatter) key[atomicAdd(cnt + v, 1)] = k;
            else atomicAdd(cnt + v, 1);
        });
}
__global__ void __launch_bounds__(256) k_index_sort(int nV, const int* __restrict__ ptr, unsigned long long* __restrict__ key)
{
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nV; v += gridDim.x * blockDim.x) {
        const int s = ptr[v], e = ptr[v + 1];
        for (int i = s + 1; i < e; ++i) {
            const unsigned long long k = key[i];
            int j = i - 1;
            while (j >= s && key[j] > k) {
                key[j + 1] = key[j];
                --j;
            }
            key[j + 1] = k;
        }
    }
}

} // namespace
} // namespace ipcgpu

using namespace ipcgpu;

template <int kMode>
static int build_index(ipcgpu_ctx* ctx, const IndexSrc& s, int* ptr, unsigned long long* key)
{
    int* cnt = ctx->cw.cnt.p;
    cudaStream_t st = ctx->stream;
    const int nV = ctx->nV;
    zero_words(cnt, (size_t)nV + 1, st);
    k_index_emit<kMode, false><<<kReproBlocks, 128, 0, st>>>(s, cnt, nullptr);
    int rc = contact_scan(ctx, cnt, ptr, nV + 1);
    if (rc) return rc;
    CK(cudaMemcpyAsync(cnt, ptr, (size_t)nV * sizeof(int), cudaMemcpyDeviceToDevice, st));
    k_index_emit<kMode, true><<<kReproBlocks, 128, 0, st>>>(s, cnt, key);
    k_index_sort<<<nblk(nV, 256), 256, 0, st>>>(nV, ptr, key);
    ctx->launches += 6;
    return IPCGPU_OK;
}

int repro_alloc(ipcgpu_ctx* ctx)
{
    ReproWork& r = ctx->rw;
    const int nV = std::max(ctx->nV, 1), nSV = std::max(ctx->nSV, 1);
    const size_t cap = (size_t)std::max(ctx->cw.cap, 1);
    if (r.cap == (int)cap && r.nV == nV && r.nSV == nSV) return IPCGPU_OK;
    REQUIRE(cap <= ((size_t)1 << 27), IPCGPU_ERR_CAPACITY, "the reproducible mode keys list positions on 28 bits: a pair capacity of at most 2^27");
    bool ok = r.bg_ptr.reserve((size_t)nV + 1) && r.bh_ptr.reserve((size_t)nV + 1) && r.fg_ptr.reserve((size_t)nV + 1) && r.fh_ptr.reserve((size_t)nV + 1)
        && r.bg_key.reserve(12 * cap) && r.bh_key.reserve(10 * cap) && r.fg_key.reserve(4 * cap) && r.fh_key.reserve(10 * cap)
        && r.bstage.reserve(36 * cap) && r.fstage.reserve(12 * cap) && r.fhstage.reserve(13 * cap)
        && r.hs_mask.reserve((size_t)nV) && r.hs_pos.reserve((size_t)kMaxPlanes * nV) && r.hs_stage.reserve((size_t)6 * kMaxPlanes * nSV);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "reproducible-mode workspace allocation failed");
    CK(cudaMemsetAsync(r.hs_mask.p, 0, (size_t)nV * sizeof(int), ctx->stream)); // (k_hs_repro_add leaves it zero after every use)
    r.cap = (int)cap;
    r.nV = nV;
    r.nSV = nSV;
    r.lists_ready = r.fr_ready = false;
    return IPCGPU_OK;
}

bool repro_on(const ipcgpu_ctx* ctx) { return ctx->canonical_order == 2 && ctx->nranks == 1 && ctx->rw.cap > 0; }

// the gradient and Hessian indices of the active and mollified lists (in canonical order already)
int repro_contact_lists(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    ReproWork& r = ctx->rw;
    int rc;
    const IndexSrc s{ w.act.p, w.counters.p + 0, w.para.p, w.para_e.p, w.counters.p + 2, ctx->SE.p, r.cap };
    if ((rc = build_index<kIdxGrad>(ctx, s, r.bg_ptr.p, r.bg_key.p))) return rc;
    if ((rc = build_index<kIdxBarrierH>(ctx, s, r.bh_ptr.p, r.bh_key.p))) return rc;
    CK(cudaGetLastError());
    r.lists_ready = true;
    return IPCGPU_OK;
}

// the lagged friction list (sorted with its companions when it came from the caller), then its indices
int repro_friction_list(ipcgpu_ctx* ctx, bool sort)
{
    ContactWork& w = ctx->cw;
    ReproWork& r = ctx->rw;
    int rc;
    if (sort) {
        if ((rc = lex_order(ctx, w.fr_cs.p, nullptr, w.fr_n.p, r.cap))) return rc;
        permute(ctx, w.fr_cs.p, 2, w.fr_n.p, r.cap);
        permute(ctx, w.fr_lambda.p, 1, w.fr_n.p, r.cap);
        permute(ctx, w.fr_coord.p, 2, w.fr_n.p, r.cap);
        permute(ctx, w.fr_basis.p, 6, w.fr_n.p, r.cap);
    }
    const IndexSrc s{ w.fr_cs.p, w.fr_n.p, nullptr, nullptr, nullptr, ctx->SE.p, r.cap };
    if ((rc = build_index<kIdxGrad>(ctx, s, r.fg_ptr.p, r.fg_key.p))) return rc;
    if ((rc = build_index<kIdxFrictionH>(ctx, s, r.fh_ptr.p, r.fh_key.p))) return rc;
    CK(cudaGetLastError());
    r.fr_ready = true;
    return IPCGPU_OK;
}

ReproArgs repro_barrier_args(ipcgpu_ctx* ctx)
{
    ReproArgs a;
    ReproWork& r = ctx->rw;
    if (!repro_on(ctx) || !r.lists_ready) return a;
    a.on = 1;
    a.cap = r.cap;
    a.stage = r.bstage.p;
    a.g = VertexIndex{ r.bg_ptr.p, r.bg_key.p };
    a.h = VertexIndex{ r.bh_ptr.p, r.bh_key.p };
    return a;
}
ReproArgs repro_friction_args(ipcgpu_ctx* ctx)
{
    ReproArgs a;
    ReproWork& r = ctx->rw;
    if (!repro_on(ctx) || !r.fr_ready) return a;
    a.on = 1;
    a.cap = r.cap;
    a.stage = r.fstage.p;
    a.hstage = r.fhstage.p;
    a.g = VertexIndex{ r.fg_ptr.p, r.fg_key.p };
    a.h = VertexIndex{ r.fh_ptr.p, r.fh_key.p };
    return a;
}
