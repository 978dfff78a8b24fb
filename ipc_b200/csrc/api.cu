// api.cu -- extern "C" entry points declared in include/ipcgpu.h
//
// Execution model.  Every stage enqueues its kernels (and, with several ranks, its NCCL reductions) on the context's stream and leaves
// its scalar results in the device-resident iteration state (kernels.h: IterState).  An entry point synchronises with the host only if
// the caller hands it a host output pointer; with NULL outputs a whole Newton iteration runs without a host synchronisation, read back
// once by ipcgpu_fetch_iteration, its derivative chain on a stream of its own next to the step-bound chain (see enter() below).  The
// synchronous forms are the same code followed by that read-back (energy_result, gradient_call / hessian_call, flag_status).
#include "../../include/ipcgpu.h"
#include "context.h"
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <dlfcn.h>
#include <numeric>

using namespace ipcgpu;

#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess) {                                                                  \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                        \
            return IPCGPU_ERR_CUDA;                                                               \
        }                                                                                         \
    } while (0)
#define REQUIRE(cond, code, msg)                                                                  \
    do {                                                                                          \
        if (!(cond)) {                                                                            \
            ctx->err = (msg);                                                                     \
            return (code);                                                                        \
        }                                                                                         \
    } while (0)
#define ALLOC(buf, count) REQUIRE((buf).reserve(count), IPCGPU_ERR_CUDA, "cudaMalloc failed for " #buf)

// ---------------------------------------------------------------------------------------------------
// NCCL through dlopen: the library that torch already loaded (libnccl.so.2) is reused when present.
// ---------------------------------------------------------------------------------------------------
namespace {
struct Id128 {
    char b[128];
};
struct Nccl {
    void* h = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ Id128, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
Nccl g_nccl;
bool nccl_load(std::string& err)
{
    if (g_nccl.h) return true;
    const char* names[] = { "libnccl.so.2", "libnccl.so" };
    for (const char* n : names) {
        g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.h) break;
    }
    if (!g_nccl.h) {
        err = "dlopen(libnccl.so.2) failed";
        return false;
    }
    g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.h, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(g_nccl.h, "ncclCommInitRank");
    g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.h, "ncclAllReduce");
    g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(g_nccl.h, "ncclAllGather");
    g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.h, "ncclCommDestroy");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.h, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather) {
        err = "NCCL symbols missing";
        return false;
    }
    return true;
}
constexpr int kNcclInt32 = 2;   // ncclInt32
constexpr int kNcclFloat64 = 8; // ncclDouble
constexpr int kNcclUint64 = 5;  // ncclUint64
constexpr int kNcclSum = 0, kNcclMax = 2, kNcclMin = 3;
} // namespace

// min over ranks of a device-resident uint64 (the order-preserving image of a step), in stream; no-op on one rank
int nccl_min_u64(ipcgpu_ctx* ctx, unsigned long long* word)
{
    if (ctx->nranks <= 1) return IPCGPU_OK;
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
    int r = g_nccl.AllReduce(word, word, 1, kNcclUint64, kNcclMin, ctx->nccl_comm, ctx->stream);
    ctx->prof_end(pe);
    REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(min step) failed");
    return IPCGPU_OK;
}

// make the main stream wait for the copies ipcgpu_download_range_async forked off (a graph edge when capturing)
static int join_copy_stream(ipcgpu_ctx* ctx)
{
    if (!ctx->copy_pending) return IPCGPU_OK;
    CK(cudaEventRecord(ctx->ev_copy_join, ctx->copy));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_copy_join, 0));
    ctx->copy_pending = false;
    return IPCGPU_OK;
}

// ---- the two chains of an iteration --------------------------------------------------------------------------------------
// A device-resident iteration is two chains of work that share no written data: the DERIVATIVE chain (value-array clear, per-tet
// gradient/Hessian kernel, energy reduce/store, gradient gather, CSR assembly + diagonal, barrier gradient, barrier Hessian scatter:
// wide HBM/FP64-bound grids) and the STEP-BOUND chain (step set, inversion filter, partial CCD, swept broad phase, full CCD: strings of
// short latency-bound kernels and the Tight-Inclusion passes, the critical path).  The first derivative call in its NULL-output form
// forks the low-priority stream `deriv` off the main stream; the step-bound calls keep running on the high-priority main stream next
// to it.  While `deriv` is open only these entry points may run:
//   - ipcgpu_step_bound_set, ipcgpu_inversion_step, ipcgpu_halfspace_step, ipcgpu_ccd_partial_ti, ipcgpu_hash_build_swept, ipcgpu_ccd_full_ti
//     with every host argument NULL (a host search direction rewrites `dir`, a host step reads back);
//   - the derivative calls in their NULL-output form (they enqueue on `deriv`), among them ipcgpu_halfspace_gradient / _hessian and
//     ipcgpu_halfspace_friction_gradient / _hessian, ipcgpu_damping_gradient / _hessian, ipcgpu_neumann_gradient and
//     ipcgpu_dirichlet_gradient / _hessian;
//   - ipcgpu_allreduce_grad_hess on one rank (a no-op), and ipcgpu_download_range_async, whose copy waits on `deriv` as well.
// Every other entry point that touches the device calls enter(ctx, kSerial) first, which joins `deriv` into the main stream (the pure
// host-side getters need not).  Among them ipcgpu_update_pattern: it rewrites ia, ja and slot_off, which the derivative chain reads, so it
// runs between ipcgpu_constraint_set and the first derivative call, before the fork.  The chains stay on one stream with several ranks (the gradient sum and the step-bound min-reductions
// must keep one order per communicator), while the stage timers are on (each stage is timed alone), and in the synchronous host-output
// forms.
//
// Why the allowed calls cannot race the derivative chain (written by one side / read or written by the other):
//   - ContactWork::counters: the barrier kernels read words 0 and 2 (list sizes, written by the constraint set before the fork) and the
//     pair-Hessian build clears and counts word 12; the step-bound chain reads word 3 (partial-CCD candidates).  The step-bound chain
//     writes no ContactWork buffer.
//   - IterState: the derivative chain writes energy[kEnergyElastic] and flags[FLAG_SET_CAPACITY] / flags[FLAG_PATTERN]; the step-bound chain writes
//     step_ord, inv_ord, ccd_ord, cand_range, n_full_cand, max_t, alpha_grid, ref_lo, ref_inv_h, alpha_stage, ref_count, ccd_stats and
//     flags[FLAG_ZERO_CCD_DISTANCE] / [FLAG_CCD_CAPACITY] / [FLAG_TI_WARNINGS].  Aligned words of their own; nothing clears the struct
//     while `deriv` is open (the fetch clears the flags after joining).
//   - contact lists: the barrier kernels read act / para / para_e (written by the constraint set before the fork); the step-bound chain
//     reads ContactWork::cand and writes only the CcdWork buffers (among them the swept grid: cells, sw_keys, sw_ent, sw_cnt, sw_off,
//     sw_tmp), which the derivative chain does not touch.
//   - half-space planes: the plane constraint set, lag, energies and crossing check are kSerial (they write hs_act, hs_lag, hs_lam, hs_cnt,
//     hs_pstart and IterState::energy[kEnergyPlaneBarrier / kEnergyPlaneFriction], hs_n_*, hs_crossings); the plane derivative calls read hs_par, hs_act, hs_lag, hs_lam, hs_cnt,
//     Vprev (written before the fork) and write g / a only; ipcgpu_halfspace_step reads hs_par, SVI, dir and writes IterState::step_ord,
//     hs_alpha, hs_zero_step only (the derivative chain touches none of them).
//   - damping, Neumann forces, Dirichlet penalty (damping.cu): the gradient / Hessian calls in their NULL form (ipcgpu_damping_gradient /
//     _hessian, ipcgpu_neumann_gradient, ipcgpu_dirichlet_gradient / _hessian) run on the derivative chain; they read damp_D, damp_inc_ptr,
//     damp_inc, slot_v, slot_u, slot_off, Vprev, nbc_f, mass, dbc_vid, dbc_tgt, dbc_lam and IterState::dbc_rho (all written before the fork,
//     by kSerial calls: ipcgpu_damping_update, ipcgpu_set_neumann_forces, ipcgpu_set_dirichlet_targets / _penalty / _update_lambda) and
//     write g / a only; their energies and ipcgpu_dirichlet_completed_step (IterState::energy[kEnergyDamping / kEnergyNeumann /
//     kEnergyDirichlet], dbc_step, damp_partials, nbc_partials, dbc_partials) are kSerial.  The step-bound chain touches none of them.
//   - V, Vrest, SE, dbc, ia, ja: read by both, written by neither (ia / ja / slot_off are written only by ipcgpu_update_pattern, which joins).  g, a, gcont, hblk, e_partials2, bHraw, brows, bpsd:
//     derivative chain only.  dir, pSize_dev, inv_steps: step-bound chain only.
enum Chain { kSerial, kStepBound, kDerivative };

static int join_deriv(ipcgpu_ctx* ctx)
{
    if (!ctx->deriv_open) return IPCGPU_OK;
    ctx->deriv_open = false;
    CK(cudaEventRecord(ctx->ev_deriv_done, ctx->deriv));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_deriv_done, 0));
    return IPCGPU_OK;
}

// first call of every entry point that touches the device: the context's device, then the chain (only ipcgpu_download_range_async,
// ipcgpu_graph_kernel_priorities and ipcgpu_step_control_info without a pending result set the device themselves instead)
static int enter(ipcgpu_ctx* ctx, Chain chain)
{
    CK(cudaSetDevice(ctx->device));
    if (chain == kStepBound) return IPCGPU_OK;
    if (chain == kSerial || ctx->nranks > 1 || ctx->profiling) return join_deriv(ctx);
    if (ctx->deriv_open) return IPCGPU_OK;
    CK(cudaEventRecord(ctx->ev_deriv_fork, ctx->stream)); // everything enqueued so far (positions, contact lists) precedes the chain
    CK(cudaStreamWaitEvent(ctx->deriv, ctx->ev_deriv_fork, 0));
    ctx->deriv_open = true;
    return IPCGPU_OK;
}
#define ENTER(chain)                                                                              \
    do {                                                                                          \
        int re_ = enter(ctx, (chain));                                                            \
        if (re_) return re_;                                                                      \
    } while (0)

// one D2H copy of the iteration state + stream synchronisation
int fetch_iter_state(ipcgpu_ctx* ctx)
{
    {
        int rcj = join_copy_stream(ctx);
        if (rcj) return rcj;
    }
    CK(cudaMemcpyAsync(ctx->h_iter, ctx->iter.p, sizeof(IterState), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// ---------------------------------------------------------------------------------------------------
// map building (host, once per mesh/partition): vertex->incident (tet,local) lists and Hessian slots.
// Partition (nranks > 1): rank r owns the rows of the vertex range [v_begin, v_end) -- chosen so that the incident-tet counts
// balance -- and assembles EVERY tet that touches one of them (tets on a range boundary are computed by both neighbours), so that
// each rank's part of the CSR is complete and the Hessian needs no cross-rank reduction.
// ---------------------------------------------------------------------------------------------------
static int build_maps(ipcgpu_ctx* ctx)
{
    const int nT = ctx->nT, nV = ctx->nV;
    const std::vector<int>& T = ctx->h_T;
    ctx->t_begin = (int)((int64_t)nT * ctx->rank / ctx->nranks);
    ctx->t_end = (int)((int64_t)nT * (ctx->rank + 1) / ctx->nranks);
    // vertex ranges balanced by incident-tet count
    std::vector<int64_t> cum(nV + 1, 0);
    for (size_t i = 0; i < (size_t)4 * nT; ++i) ++cum[T[i] + 1];
    for (int v = 0; v < nV; ++v) cum[v + 1] += cum[v];
    auto boundary = [&](int r) -> int {
        if (r <= 0) return 0;
        if (r >= ctx->nranks) return nV;
        const int64_t target = cum[nV] * r / ctx->nranks;
        return (int)(std::lower_bound(cum.begin(), cum.end(), target) - cum.begin());
    };
    const int vb = std::min(boundary(ctx->rank), nV), ve = std::max(vb, std::min(boundary(ctx->rank + 1), nV));
    ctx->v_begin = vb;
    ctx->v_end = ve;
    // tets touching the owned rows, ascending
    std::vector<int> list;
    if (ctx->nranks == 1) {
        list.resize(nT);
        std::iota(list.begin(), list.end(), 0);
    }
    else {
        list.reserve((size_t)(nT / ctx->nranks) + 1024);
        for (int t = 0; t < nT; ++t) {
            bool touch = false;
            for (int k = 0; k < 4; ++k) {
                const int v = T[(size_t)k * nT + t];
                touch = touch || (v >= vb && v < ve);
            }
            if (touch) list.push_back(t);
        }
    }
    const int nL = (int)list.size();
    ctx->n_list = nL;
    if (list.empty()) list.push_back(0); // keep the upload non-empty
    REQUIRE(ctx->tet_list.upload(list.data(), list.size(), ctx->stream), IPCGPU_ERR_CUDA, "upload of the tet list failed");
    // incidence of the OWNED vertices: counting sort by vertex; entries 4*localTet+loc ascending
    std::vector<int> ptr(nV + 1, 0);
    for (int l = 0; l < nL; ++l)
        for (int k = 0; k < 4; ++k) {
            const int v = T[(size_t)k * nT + list[l]];
            if (v >= vb && v < ve) ++ptr[v + 1];
        }
    for (int v = 0; v < nV; ++v) ptr[v + 1] += ptr[v];
    std::vector<int> inc((size_t)std::max(ptr[nV], 1)), cur(ptr.begin(), ptr.end() - 1);
    for (int l = 0; l < nL; ++l)
        for (int k = 0; k < 4; ++k) {
            const int v = T[(size_t)k * nT + list[l]];
            if (v >= vb && v < ve) inc[cur[v]++] = 4 * l + k;
        }
    if (!ctx->inc_ptr.upload(ptr.data(), ptr.size(), ctx->stream) || !ctx->inc.upload(inc.data(), inc.size(), ctx->stream)) {
        ctx->err = "upload of incidence map failed";
        return IPCGPU_ERR_CUDA;
    }
    // slots: (v<=u) pairs whose ROW vertex v is owned; contributions (key, src) sorted by key then tet
    REQUIRE(((uint64_t)nL + 64ull) * 78ull < 0xffffffffull, IPCGPU_ERR_CAPACITY, "local tet count too large for 32-bit block offsets");
    struct KS {
        uint64_t key;
        unsigned src;
        unsigned tet;
    };
    std::vector<KS> ks;
    ks.reserve((size_t)10 * nL);
    static const int pa[6] = { 0, 0, 0, 1, 1, 2 }, pb[6] = { 1, 2, 3, 2, 3, 3 };
    for (int l = 0; l < nL; ++l) {
        const int t = list[l];
        int v[4];
        for (int k = 0; k < 4; ++k) v[k] = T[(size_t)k * nT + t];
        // tile-major block addresses (elastic.cu): (l/64)*64*78 + o*64 + (l%64)*len
        const unsigned tl = (unsigned)l, tile_base = (tl / 64u) * (64u * 78u), tin = tl % 64u;
        for (int a = 0; a < 4; ++a)
            if (v[a] >= vb && v[a] < ve) ks.push_back({ ((uint64_t)v[a] << 32) | (uint32_t)v[a], tile_base + 6u * a * 64u + tin * 6u, tl });
        for (int q = 0; q < 6; ++q) {
            const int lo = std::min(v[pa[q]], v[pb[q]]), hi = std::max(v[pa[q]], v[pb[q]]);
            if (lo >= vb && lo < ve) ks.push_back({ ((uint64_t)lo << 32) | (uint32_t)hi, tile_base + (24u + 9u * q) * 64u + tin * 9u, tl });
        }
    }
    std::sort(ks.begin(), ks.end(), [](const KS& a, const KS& b) { return a.key < b.key || (a.key == b.key && (a.tet < b.tet || (a.tet == b.tet && a.src < b.src))); });
    std::vector<int> sv, su, cptr;
    std::vector<unsigned> csrc(std::max<size_t>(ks.size(), 1));
    for (size_t i = 0; i < ks.size(); ++i) {
        if (i == 0 || ks[i].key != ks[i - 1].key) {
            sv.push_back((int)(ks[i].key >> 32));
            su.push_back((int)(ks[i].key & 0xffffffffu));
            cptr.push_back((int)i);
        }
        csrc[i] = ks[i].src;
    }
    cptr.push_back((int)ks.size());
    {
        // Slot order = work order of k_assemble_csr (9 threads per slot, a warp covers ~3.5 slots and runs as long as its longest
        // contribution list).  In key order every 7th slot is a diagonal block with ~23 contributions against ~5 for an off-diagonal
        // one, so half of the warps idled most lanes for 20 iterations.  Off-diagonal slots first, then the diagonal ones (key order
        // inside each group keeps the CSR writes local): warps see uniform list lengths.
        const size_t nS = sv.size();
        std::vector<int> order;
        order.reserve(nS);
        for (size_t i = 0; i < nS; ++i)
            if (sv[i] != su[i]) order.push_back((int)i);
        for (size_t i = 0; i < nS; ++i)
            if (sv[i] == su[i]) order.push_back((int)i);
        std::vector<int> sv2(nS), su2(nS), cptr2;
        std::vector<unsigned> csrc2(csrc.size());
        cptr2.reserve(nS + 1);
        size_t pos = 0;
        for (size_t k = 0; k < nS; ++k) {
            const int i = order[k];
            sv2[k] = sv[i];
            su2[k] = su[i];
            cptr2.push_back((int)pos);
            for (int c = cptr[i]; c < cptr[i + 1]; ++c) csrc2[pos++] = csrc[c];
        }
        cptr2.push_back((int)pos);
        sv.swap(sv2); su.swap(su2); cptr.swap(cptr2); csrc.swap(csrc2);
    }
    ctx->nSlots = (int)sv.size();
    if (sv.empty()) { sv.push_back(0); su.push_back(0); } // keep the uploads non-empty
    bool ok = ctx->slot_v.upload(sv.data(), sv.size(), ctx->stream) && ctx->slot_u.upload(su.data(), su.size(), ctx->stream)
        && ctx->con_ptr.upload(cptr.data(), cptr.size(), ctx->stream) && ctx->con_src.upload(csrc.data(), csrc.size(), ctx->stream)
        && ctx->slot_off.reserve((size_t)3 * std::max(1, ctx->nSlots));
    REQUIRE(ok, IPCGPU_ERR_CUDA, "upload of Hessian scatter map failed");
    ALLOC(ctx->gcont, (size_t)12 * std::max(1, nL));
    ALLOC(ctx->hblk, (size_t)78 * 64 * ((size_t)(std::max(1, nL) + 63) / 64));
    ALLOC(ctx->partials, (size_t)std::max(1, elastic_energy_blocks(ctx->t_end - ctx->t_begin)) + 8);
    CK(cudaStreamSynchronize(ctx->stream)); // host vectors go out of scope
    ctx->maps_ready = true;
    ctx->offsets_ready = false;
    // D and its incidence follow the slots, the Neumann forces and Dirichlet targets the vertices: a new mesh or partition removes them
    ctx->damp_on = ctx->damp_inc_ready = ctx->nbc_on = false;
    ctx->n_dbc = 0;
    for (int slot : { kEnergyDamping, kEnergyNeumann, kEnergyDirichlet }) // (the fetch reports 0 for a term that is not set)
        CK(cudaMemsetAsync(&ctx->iter.p->energy[slot], 0, sizeof(double), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

static void owned_value_range(ipcgpu_ctx* ctx)
{
    // CSR value range of the owned rows [3 v_begin, 3 v_end)
    if (ctx->h_ia.empty()) return;
    ctx->a_begin = (long long)ctx->h_ia[(size_t)3 * ctx->v_begin] - ctx->index_base;
    ctx->a_end = (long long)ctx->h_ia[(size_t)3 * ctx->v_end] - ctx->index_base;
}

static int ensure_offsets(ipcgpu_ctx* ctx)
{
    if (ctx->offsets_ready) return IPCGPU_OK;
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh must precede Hessian assembly");
    REQUIRE(ctx->n_rows == 3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_csr must be called with n_rows = 3*nV");
    CK(cudaMemsetAsync(ctx->flag.p, 0, sizeof(int), ctx->stream));
    slot_offsets(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->ia.p, ctx->ja.p, ctx->index_base, ctx->slot_off.p, ctx->flag.p, ctx->stream);
    ++ctx->launches;
    int h = 0;
    CK(cudaMemcpyAsync(&h, ctx->flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    REQUIRE(h == 0, IPCGPU_ERR_PATTERN, "CSR pattern misses a block of the mesh topology (row<=col entries of every tet vertex pair are required)");
    ctx->offsets_ready = true;
    return IPCGPU_OK;
}

// device-built pattern: bring the host mirrors (nnz, h_ia, owned value range) up to the device's pattern; h_iter must be fresh
static int refresh_pattern_mirror(ipcgpu_ctx* ctx)
{
    if (!ctx->device_pattern) return IPCGPU_OK;
    ctx->pat_pending = false;
    const IterState& h = *ctx->h_iter;
    ctx->pat_changed_host = h.pat_changed;
    if (h.pat_version == ctx->pat_seen_version) return IPCGPU_OK;
    ctx->pat_seen_version = h.pat_version;
    ctx->nnz = (int)h.pat_nnz;
    CK(cudaMemcpyAsync(ctx->h_ia.data(), ctx->ia.p, ctx->h_ia.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->full_pattern_ready = false;
    owned_value_range(ctx);
    return IPCGPU_OK;
}
int fetch_iter_state(ipcgpu_ctx* ctx);
// ... before a host-side use of them, when an update was enqueued since (synchronises)
static int sync_pattern_mirror(ipcgpu_ctx* ctx)
{
    if (!ctx->device_pattern || !ctx->pat_pending) return IPCGPU_OK;
    int rc = fetch_iter_state(ctx);
    return rc ? rc : refresh_pattern_mirror(ctx);
}

// C++ linkage helpers implemented in constraint.cu / ccd.cu
int contact_alloc(ipcgpu_ctx* ctx);
int contact_constraint_set(ipcgpu_ctx* ctx, double dHat, int wantCand, int* nC, int* nPara, int* nCand);
int contact_sync_counts(ipcgpu_ctx* ctx);
void contact_pack_lists(ipcgpu_ctx* ctx);
void contact_unpack_lists(ipcgpu_ctx* ctx);
int ccd_alloc(ipcgpu_ctx* ctx);
int ccd_narrow(ipcgpu_ctx* ctx, const int2* cand, const int* n32, const unsigned long long* n64, unsigned long long cap, int share, double tol, const double* err_vf,
    const double* err_ee, int stage, const int* overflow);
int ccd_build_swept(ipcgpu_ctx* ctx, double h);
int ccd_full(ipcgpu_ctx* ctx, double tol, const double* err_vf, const double* err_ee);
int ccd_read_back(ipcgpu_ctx* ctx, double* alpha_out);
int solver_build_full_pattern(ipcgpu_ctx* ctx, const int* ia, const int* ja); // solve.cu
int solver_pcg(ipcgpu_ctx* ctx, const double* rhs_dev, double sign, double rel_tol, int max_iter, int* iters_out, double* rel_res_out);
int solver_adopt_direction(ipcgpu_ctx* ctx);
int pattern_enable(ipcgpu_ctx* ctx, int index_base, uint64_t nnz_capacity); // pattern.cu
int pattern_update(ipcgpu_ctx* ctx, const BarrierArgs& lists, bool with_friction);
int safeguard_inversion(ipcgpu_ctx* ctx);     // safeguard.cu
int safeguard_intersections(ipcgpu_ctx* ctx); // safeguard.cu

// deferred error flags of the iteration state -> status code (first raised flag wins) and message
static int status_from_flags(ipcgpu_ctx* ctx, const int* f)
{
    if (f[FLAG_NONPOSITIVE_DISTANCE]) {
        ctx->err = "a constraint has d <= 0 (the reference exits here, Optimizer.cpp:3296-3306)";
        return IPCGPU_ERR_NONPOSITIVE_DISTANCE;
    }
    if (f[FLAG_SET_CAPACITY]) {
        ctx->err = "constraint-set capacity exceeded (raise it with ipcgpu_set_pair_capacity)";
        return IPCGPU_ERR_CAPACITY;
    }
    if (f[FLAG_EXCHANGE_CAPACITY]) {
        ctx->err = "pair-list exchange capacity exceeded (65536 pairs per rank and list)";
        return IPCGPU_ERR_CAPACITY;
    }
    if (f[FLAG_CCD_CAPACITY]) {
        ctx->err = "CCD candidate capacity exceeded (raise it with ipcgpu_set_ccd_capacity)";
        return IPCGPU_ERR_CAPACITY;
    }
    if (f[FLAG_PATTERN_CAPACITY]) {
        ctx->err = "device-built sparsity pattern exceeds its capacity (raise it with ipcgpu_enable_device_pattern); the previous pattern is kept";
        return IPCGPU_ERR_CAPACITY;
    }
    if (f[FLAG_PATTERN]) {
        ctx->err = "CSR pattern misses a contact block: call ipcgpu_set_csr with the augmented pattern (augmentConnectivity, SelfCollisionHandler.cpp:330-415)";
        return IPCGPU_ERR_PATTERN;
    }
    return IPCGPU_OK;
}

// ---- the tails the synchronous forms share --------------------------------------------------------------------------------
// the flags of `mask` that the (fresh) h_iter shows raised: cleared on the device, returned as a status
static int flag_status(ipcgpu_ctx* ctx, unsigned mask)
{
    int f[8] = { 0 };
    for (int i = 0; i < 8; ++i)
        if (((mask >> i) & 1u) && ctx->h_iter->flags[i]) {
            f[i] = ctx->h_iter->flags[i];
            CK(cudaMemsetAsync(&ctx->iter.p->flags[i], 0, sizeof(int), ctx->stream));
        }
    return status_from_flags(ctx, f);
}

static void set_local(ipcgpu_ctx* ctx, unsigned bits, bool local)
{
    ctx->local_scalars = local ? (ctx->local_scalars | bits) : (ctx->local_scalars & ~bits);
}

// IterState::energy[slot] once reduced.  Host E: summed across the ranks in place and read back, either the one double or (`fetch`) the
// whole iteration state, after which the flags of `check` are the status.  NULL: this rank's share, completed by the fetch's collective.
static int energy_result(ipcgpu_ctx* ctx, int slot, double* E, bool fetch = false, unsigned check = 0)
{
    set_local(ctx, 1u << slot, ctx->nranks > 1 && !E);
    if (!E) return IPCGPU_OK;
    double* out = &ctx->iter.p->energy[slot];
    if (ctx->nranks > 1) {
        int r = g_nccl.AllReduce(out, out, 1, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(energy) failed");
    }
    if (fetch) {
        int rc = fetch_iter_state(ctx);
        if (rc) return rc;
        *E = ctx->h_iter->energy[slot];
        return flag_status(ctx, check);
    }
    CK(cudaMemcpyAsync(ctx->h_scalar, out, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *E = ctx->h_scalar[0];
    return IPCGPU_OK;
}
// the tail of an energy term on the main stream: its partial sums reduced into the slot, the stage timer `pe` stopped, energy_result
static int energy_tail(ipcgpu_ctx* ctx, int slot, const double* partials, int n_partials, double scale, cudaEvent_t pe, double* E, bool fetch = false,
    unsigned check = 0)
{
    reduce_sum(partials, n_partials, scale, &ctx->iter.p->energy[slot], ctx->stream);
    ctx->prof_end(pe);
    ctx->launches += 2; // the term's partial kernel and the reduce
    CK(cudaGetLastError());
    return energy_result(ctx, slot, E, fetch, check);
}

// host gradient in/out around a kernel that accumulates into the device gradient (addCoeff-like semantics: rank 0 contributes the input)
static int gradient_roundtrip_begin(ipcgpu_ctx* ctx, const double* g_in)
{
    if (ctx->rank == 0) CK(cudaMemcpyAsync(ctx->g.p, g_in, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    else CK(cudaMemsetAsync(ctx->g.p, 0, (size_t)3 * ctx->nV * sizeof(double), ctx->stream));
    return IPCGPU_OK;
}
static int gradient_roundtrip_end(ipcgpu_ctx* ctx, double* g_out)
{
    if (ctx->nranks > 1) {
        int rc = ipcgpu_allreduce_grad_hess(ctx, 1, 0);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(g_out, ctx->g.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}
// the same for the value array
static int upload_values(ipcgpu_ctx* ctx, const double* a_host)
{
    int rc = sync_pattern_mirror(ctx);
    if (rc) return rc;
    if (ctx->rank == 0) CK(cudaMemcpyAsync(ctx->a.p, a_host, (size_t)ctx->nnz * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    else CK(cudaMemsetAsync(ctx->a.p, 0, (size_t)ctx->nnz * sizeof(double), ctx->stream));
    return IPCGPU_OK;
}
static int download_values(ipcgpu_ctx* ctx, double* a_host)
{
    int rc = sync_pattern_mirror(ctx);
    if (rc) return rc;
    if (ctx->nranks > 1 && (rc = ipcgpu_allreduce_grad_hess(ctx, 0, 1))) return rc;
    CK(cudaMemcpyAsync(a_host, ctx->a.p, (size_t)ctx->nnz * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// A gradient / Hessian term.  NULL output: the term on `chain`; host output: the caller's array in, the term added on the main stream,
// the rank-completed array out and, for a Hessian, the flags of `check` it may raise returned as its status.
// `stage`: the stage timer the term is counted under.
template <typename Launch>
static int gradient_call(ipcgpu_ctx* ctx, Chain chain, double* g_inout, Launch launch, int stage = IPCGPU_STAGE_BARRIER)
{
    ENTER(g_inout ? kSerial : chain);
    int rc;
    if (g_inout && (rc = gradient_roundtrip_begin(ctx, g_inout))) return rc;
    cudaEvent_t pe = ctx->prof_begin(stage);
    launch(ctx->deriv_stream());
    ctx->prof_end(pe);
    ++ctx->launches;
    CK(cudaGetLastError());
    return g_inout ? gradient_roundtrip_end(ctx, g_inout) : IPCGPU_OK;
}
static int hessian_begin(ipcgpu_ctx* ctx, Chain chain, const double* a_inout)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(a_inout ? kSerial : chain);
    return a_inout ? upload_values(ctx, a_inout) : IPCGPU_OK;
}
static int hessian_end(ipcgpu_ctx* ctx, double* a_inout, unsigned check)
{
    if (!a_inout) return IPCGPU_OK;
    int rc = download_values(ctx, a_inout);
    if (rc || !check || (rc = fetch_iter_state(ctx))) return rc;
    return flag_status(ctx, check);
}
template <typename Launch>
static int hessian_call(ipcgpu_ctx* ctx, Chain chain, double* a_inout, unsigned check, Launch launch, int stage = IPCGPU_STAGE_BARRIER)
{
    int rc = hessian_begin(ctx, chain, a_inout);
    if (rc) return rc;
    cudaEvent_t pe = ctx->prof_begin(stage);
    launch(ctx->deriv_stream());
    ctx->prof_end(pe);
    ++ctx->launches;
    CK(cudaGetLastError());
    return hessian_end(ctx, a_inout, check);
}

// f(node, priority attribute) on every kernel node of a graph and of the bodies of its conditional nodes, until one returns an error
template <typename F>
static cudaError_t for_each_kernel_node(cudaGraph_t top, const std::vector<cudaGraph_t>& bodies, F f)
{
    cudaError_t e = cudaSuccess;
    for (size_t b = 0; e == cudaSuccess && b <= bodies.size(); ++b) {
        cudaGraph_t g = b == 0 ? top : bodies[b - 1];
        size_t n = 0;
        e = cudaGraphGetNodes(g, nullptr, &n);
        std::vector<cudaGraphNode_t> nodes(n);
        if (e == cudaSuccess && n) e = cudaGraphGetNodes(g, nodes.data(), &n);
        for (size_t i = 0; e == cudaSuccess && i < n; ++i) {
            // (the runtime reports no type for a conditional node: cudaErrorUnknown, not sticky, but left as the last error, which a later
            // cub call would pick up -- cleared here; the node's body is in `bodies`)
            cudaGraphNodeType type;
            if (cudaGraphNodeGetType(nodes[i], &type) != cudaSuccess) {
                cudaGetLastError();
                continue;
            }
            if (type != cudaGraphNodeTypeKernel) continue;
            cudaKernelNodeAttrValue v;
            e = cudaGraphKernelNodeGetAttribute(nodes[i], cudaKernelNodeAttributePriority, &v);
            if (e == cudaSuccess) e = f(nodes[i], v);
        }
    }
    return e;
}

extern "C" {

int ipcgpu_create(int device, ipcgpu_ctx** out)
{
    if (!out) return IPCGPU_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return IPCGPU_ERR_CUDA; // no CPU fallback by design
    if (device < 0 || device >= ndev) return IPCGPU_ERR_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return IPCGPU_ERR_CUDA;
    ipcgpu_ctx* ctx = new ipcgpu_ctx();
    ctx->device = device;
    void* hi = nullptr;
    if (cudaDeviceGetStreamPriorityRange(&ctx->prio_low, &ctx->prio_high) != cudaSuccess
        || cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, ctx->prio_high) != cudaSuccess
        || cudaStreamCreateWithPriority(&ctx->deriv, cudaStreamNonBlocking, ctx->prio_low) != cudaSuccess
        || cudaEventCreateWithFlags(&ctx->ev_deriv_fork, cudaEventDisableTiming) != cudaSuccess
        || cudaEventCreateWithFlags(&ctx->ev_deriv_done, cudaEventDisableTiming) != cudaSuccess
        // side stream for the pair-Hessian build + projection.  Replayed from a graph it wins 0.13 ms per iteration next to the overlapped
        // derivative chain (H100 SXM, 700 W, C5: 3.39 -> 3.25 ms)
        || cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&ctx->ev_inputs, cudaEventDisableTiming) != cudaSuccess
        || cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&ctx->ev_scatter, cudaEventDisableTiming) != cudaSuccess
        || cudaMallocHost(&ctx->h_scalar, 512) != cudaSuccess
        || cudaMallocHost(&hi, sizeof(IterState)) != cudaSuccess || !ctx->flag.reserve(4) || !ctx->packed_scalars.reserve(kPackedScalars) || !ctx->iter.reserve(1)
        || cudaMemsetAsync(ctx->iter.p, 0, sizeof(IterState), ctx->stream) != cudaSuccess) {
        ipcgpu_destroy(ctx);
        return IPCGPU_ERR_CUDA;
    }
    ctx->h_iter = static_cast<IterState*>(hi);
    std::memset(ctx->h_iter, 0, sizeof(IterState));
    step_set(ctx->iter.p, 1.0, ctx->stream);
    *out = ctx;
    return IPCGPU_OK;
}

void ipcgpu_destroy(ipcgpu_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->side) cudaStreamSynchronize(ctx->side);
    if (ctx->deriv) cudaStreamSynchronize(ctx->deriv);
    if (ctx->copy) {
        cudaStreamSynchronize(ctx->copy);
        cudaStreamDestroy(ctx->copy);
        cudaEventDestroy(ctx->ev_copy_fork);
        cudaEventDestroy(ctx->ev_copy_join);
    }
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (auto& r : ctx->graphs) {
        if (r.exec) cudaGraphExecDestroy(r.exec);
        if (r.graph) cudaGraphDestroy(r.graph);
    }
    if (ctx->ev_inputs) cudaEventDestroy(ctx->ev_inputs);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->ev_scatter) cudaEventDestroy(ctx->ev_scatter);
    if (ctx->side) cudaStreamDestroy(ctx->side);
    if (ctx->ev_deriv_fork) cudaEventDestroy(ctx->ev_deriv_fork);
    if (ctx->ev_deriv_done) cudaEventDestroy(ctx->ev_deriv_done);
    if (ctx->deriv) cudaStreamDestroy(ctx->deriv);
    for (cudaStream_t s : ctx->cond_streams)
        if (s) cudaStreamDestroy(s);
    for (auto& v : ctx->prof)
        for (auto& pr : v) {
            cudaEventDestroy(pr.first);
            cudaEventDestroy(pr.second);
        }
    if (ctx->timer_a) cudaEventDestroy(ctx->timer_a);
    if (ctx->timer_b) cudaEventDestroy(ctx->timer_b);
    if (ctx->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->nccl_comm);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->h_scalar) cudaFreeHost(ctx->h_scalar);
    if (ctx->h_iter) cudaFreeHost(ctx->h_iter);
    delete ctx;
}

const char* ipcgpu_last_error(const ipcgpu_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int ipcgpu_host_alloc(void** ptr, uint64_t bytes) { return cudaMallocHost(ptr, bytes) == cudaSuccess ? IPCGPU_OK : IPCGPU_ERR_CUDA; }
int ipcgpu_host_free(void* ptr) { return cudaFreeHost(ptr) == cudaSuccess ? IPCGPU_OK : IPCGPU_ERR_CUDA; }
int ipcgpu_sync(ipcgpu_ctx* ctx)
{
    ENTER(kSerial);
    int rcj = join_copy_stream(ctx);
    if (rcj) return rcj;
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}
uint64_t ipcgpu_launch_count(const ipcgpu_ctx* ctx) { return ctx ? ctx->launches : 0; }

int ipcgpu_comm_unique_id(void* id128)
{
    std::string err;
    if (!id128 || !nccl_load(err)) return IPCGPU_ERR_NCCL;
    return g_nccl.GetUniqueId(id128) == 0 ? IPCGPU_OK : IPCGPU_ERR_NCCL;
}

int ipcgpu_comm_init(ipcgpu_ctx* ctx, int rank, int nranks, const void* id128)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, IPCGPU_ERR_ARG, "bad rank/nranks");
    ctx->rank = rank;
    ctx->nranks = nranks;
    if (nranks > 1) {
        REQUIRE(id128 != nullptr, IPCGPU_ERR_ARG, "nccl unique id required for nranks>1");
        REQUIRE(nccl_load(ctx->err), IPCGPU_ERR_NCCL, ctx->err);
        Id128 id;
        std::memcpy(id.b, id128, 128);
        int r = g_nccl.CommInitRank(&ctx->nccl_comm, nranks, id, rank);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
    }
    if (ctx->nT > 0) { // re-partition an already loaded mesh
        int rc = build_maps(ctx);
        if (rc) return rc;
        owned_value_range(ctx);
        if (ctx->surface_ready && (rc = contact_alloc(ctx))) return rc;
    }
    return IPCGPU_OK;
}

int ipcgpu_partition_info(ipcgpu_ctx* ctx, int* rank, int* nranks, int* tet_begin, int* tet_end, int* row_vertex_begin, int* row_vertex_end, int64_t* value_begin,
    int64_t* value_end, int* n_assembled_tets)
{
    if (rank) *rank = ctx->rank;
    if (nranks) *nranks = ctx->nranks;
    if (tet_begin) *tet_begin = ctx->t_begin;
    if (tet_end) *tet_end = ctx->t_end;
    if (row_vertex_begin) *row_vertex_begin = ctx->v_begin;
    if (row_vertex_end) *row_vertex_end = ctx->v_end;
    if (value_begin) *value_begin = ctx->a_begin;
    if (value_end) *value_end = ctx->a_end;
    if (n_assembled_tets) *n_assembled_tets = ctx->n_list;
    return IPCGPU_OK;
}

int ipcgpu_set_mesh(ipcgpu_ctx* ctx, int nV, int nT, const double* Vrest, const int* tets, const double* restTriInv, const double* vol,
    const double* mu, const double* lam, const double* mass, const uint8_t* dbc, int energy)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(nV > 0 && nT >= 0 && Vrest && tets && restTriInv && vol && mu && lam, IPCGPU_ERR_ARG, "ipcgpu_set_mesh: null or empty input");
    REQUIRE(energy == IPCGPU_NEOHOOKEAN || energy == IPCGPU_FIXED_COROT, IPCGPU_ERR_ARG, "unknown energy type");
    for (size_t i = 0; i < (size_t)4 * nT; ++i) REQUIRE(tets[i] >= 0 && tets[i] < nV, IPCGPU_ERR_ARG, "tet vertex index out of range");
    ctx->nV = nV;
    ctx->nT = nT;
    ctx->energy = energy;
    ctx->hs_set_built = ctx->hs_lag_ready = false; // the plane sets index the old vertices
    ctx->nVdof = 0x7fffffff; // a new mesh has no obstacle tail until ipcgpu_set_obstacle_tail names one
    ctx->h_T.assign(tets, tets + (size_t)4 * nT);
    ctx->h_ia.clear();
    ctx->nnz = 0;
    ctx->device_pattern = ctx->pat_pending = false;
    ctx->surface_ready = false;
    ctx->dir_valid = false;
    // Dm^-1: reference layout is per-tet column-major; device layout is SoA over the row-major index q=3i+j
    std::vector<double> A((size_t)9 * std::max(nT, 1));
    for (int t = 0; t < nT; ++t)
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) A[(size_t)(3 * i + j) * nT + t] = restTriInv[(size_t)9 * t + i + 3 * j];
    bool ok = ctx->Vrest.upload(Vrest, (size_t)3 * nV, ctx->stream) && ctx->V.upload(Vrest, (size_t)3 * nV, ctx->stream)
        && ctx->Vsaved.reserve((size_t)3 * nV) && ctx->T.upload(tets, (size_t)4 * nT, ctx->stream)
        && ctx->Ainv.upload(A.data(), (size_t)9 * nT, ctx->stream) && ctx->vol.upload(vol, nT, ctx->stream)
        && ctx->mu.upload(mu, nT, ctx->stream) && ctx->lam.upload(lam, nT, ctx->stream);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "mesh upload failed");
    ctx->has_mass = mass != nullptr;
    if (mass) REQUIRE(ctx->mass.upload(mass, nV, ctx->stream), IPCGPU_ERR_CUDA, "mass upload failed");
    ctx->has_dbc = dbc != nullptr;
    if (dbc) REQUIRE(ctx->dbc.upload(dbc, nV, ctx->stream), IPCGPU_ERR_CUDA, "dbc upload failed");
    ALLOC(ctx->g, (size_t)3 * nV);
    ALLOC(ctx->dir, (size_t)3 * nV);
    ALLOC(ctx->e_per_tet, (size_t)std::max(nT, 1));
    ALLOC(ctx->inv_steps, (size_t)std::max(nT, 1));
    CK(cudaStreamSynchronize(ctx->stream));
    return build_maps(ctx);
}

int ipcgpu_set_csr(ipcgpu_ctx* ctx, int n_rows, const int* ia, const int* ja, int index_base)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(n_rows > 0 && ia && ja && (index_base == 0 || index_base == 1), IPCGPU_ERR_ARG, "ipcgpu_set_csr: bad arguments");
    REQUIRE(ctx->nV > 0 && n_rows == 3 * ctx->nV, IPCGPU_ERR_ARG, "ipcgpu_set_csr: n_rows must be 3*nV of the mesh set before");
    const int nnz = ia[n_rows] - index_base;
    REQUIRE(nnz >= 0, IPCGPU_ERR_ARG, "ipcgpu_set_csr: negative nnz");
    ctx->n_rows = n_rows;
    ctx->nnz = nnz;
    ctx->index_base = index_base;
    ctx->device_pattern = ctx->pat_pending = false; // host mode again
    ctx->h_ia.assign(ia, ia + (size_t)n_rows + 1);
    bool ok = ctx->ia.upload(ia, (size_t)n_rows + 1, ctx->stream) && ctx->ja.upload(ja, (size_t)nnz, ctx->stream) && ctx->a.reserve((size_t)std::max(nnz, 1));
    REQUIRE(ok, IPCGPU_ERR_CUDA, "CSR upload failed");
    CK(cudaMemsetAsync(ctx->a.p, 0, (size_t)nnz * sizeof(double), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->a_all_dirty = false;
    ctx->offsets_ready = false;
    ctx->full_pattern_ready = false;
    owned_value_range(ctx);
    return IPCGPU_OK;
}

int ipcgpu_set_state(ipcgpu_ctx* ctx, const double* V)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    if (V) CK(cudaMemcpyAsync(ctx->V.p, V, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->mark_inputs();
    return IPCGPU_OK;
}

int ipcgpu_save_state(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    CK(cudaMemcpyAsync(ctx->Vsaved.p, ctx->V.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->state_saved = true;
    return IPCGPU_OK;
}

// upload the search direction; pSize = mean |p| over the surface vertices in the reference's serial order (SpatialHash.hpp:603-612),
// taken straight from the caller's array (it is only needed by the swept build and costs one pass over the surface)
static int upload_dir(ipcgpu_ctx* ctx, const double* p)
{
    if (p) {
        CK(cudaMemcpyAsync(ctx->dir.p, p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        double pSize = 0;
        // (mesh.SVI: with an obstacle attached the surface vertices of the tail do not count -- SpatialHash::build sees the mesh alone)
        int nMeshSV = 0;
        for (int i = 0; i < ctx->nSV; ++i) {
            const int v = ctx->h_SVI[i];
            if (v >= ctx->nVdof) continue;
            ++nMeshSV;
            pSize += std::abs(p[3 * (size_t)v]);
            pSize += std::abs(p[3 * (size_t)v + 1]);
            pSize += std::abs(p[3 * (size_t)v + 2]);
        }
        ctx->pSize = nMeshSV > 0 ? pSize / (double)((long long)nMeshSV * 3) : 0.0;
        // the swept-grid kernel reads it from device memory, so that a captured graph stays valid when the direction changes
        ALLOC(ctx->pSize_dev, 1);
        double* hp = ctx->h_scalar + 32; // pinned staging slot of its own (the copy is asynchronous)
        *hp = ctx->pSize;
        CK(cudaMemcpyAsync(ctx->pSize_dev.p, hp, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        ctx->pSize_surface = ctx->surface_ready;
        ctx->dir_valid = true; // (no synchronisation: like every host input of the deferred mode, p must stay untouched until the next fetch)
    }
    REQUIRE(ctx->dir_valid, IPCGPU_ERR_STATE, "no search direction uploaded yet");
    return IPCGPU_OK;
}

int ipcgpu_set_search_dir(ipcgpu_ctx* ctx, const double* p)
{
    REQUIRE(ctx->nV > 0 && p, IPCGPU_ERR_ARG, "ipcgpu_set_search_dir: mesh and p required");
    ENTER(kSerial);
    return upload_dir(ctx, p);
}

int ipcgpu_step_forward(ipcgpu_ctx* ctx, const double* p, double alpha)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(ctx->state_saved, IPCGPU_ERR_STATE, "ipcgpu_save_state must precede ipcgpu_step_forward");
    ENTER(kSerial);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    step_forward(ctx->nV, ctx->Vsaved.p, ctx->dir.p, alpha, ctx->V.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->mark_inputs();
    return IPCGPU_OK;
}

int ipcgpu_elastic_energy(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, double* E)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
    elastic_energy(ctx->eargs(), ctx->e_per_tet.p, ctx->partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyElastic, ctx->partials.p, elastic_energy_blocks(ctx->t_end - ctx->t_begin), coef, pe, E);
}

// zero the part of the value array this rank writes (everything after a cross-rank completion has filled the other rows)
static int zero_values(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->deriv_stream(); // (zero_words, not a memset: kernels.h)
    if (ctx->device_pattern) { // the range follows the device's row starts (the host mirror may lag an update in flight)
        const bool owned = ctx->nranks > 1 && !ctx->a_all_dirty;
        zero_csr_rows(ctx->ia.p, ctx->index_base, owned ? 3 * ctx->v_begin : 0, owned ? 3 * ctx->v_end : 3 * ctx->nV, ctx->a.p, st);
    }
    else if (ctx->nranks > 1 && !ctx->a_all_dirty) {
        if (ctx->a_end > ctx->a_begin) zero_words(ctx->a.p + ctx->a_begin, (size_t)(ctx->a_end - ctx->a_begin) * 2, st);
    }
    else zero_words(ctx->a.p, (size_t)ctx->nnz * 2, st);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->a_all_dirty = false;
    return IPCGPU_OK;
}

static int run_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, bool need_g, bool need_h, int add_mass, bool with_energy = false)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    if (need_h) {
        int rc = ensure_offsets(ctx);
        if (rc) return rc;
    }
    cudaStream_t st = ctx->deriv_stream(); // (stage timers are only on when it is the main stream)
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_TET);
    double* e_part = nullptr;
    if (with_energy) { // psi * vol per CTA, summed in fixed order below (computeEnergyVal at the same state: the SVD is shared)
        ALLOC(ctx->e_partials2, (size_t)elastic_grad_hess_blocks(ctx->n_list) + 8);
        e_part = ctx->e_partials2.p;
    }
    elastic_grad_hess(ctx->eargs(), coef, projectSPD, need_g, need_h, ctx->gcont.p, ctx->hblk.p, st, e_part);
    ctx->hblk_valid = need_h;
    ctx->prof_end(pe);
    ++ctx->launches;
    if (with_energy) { // (which rank's share it is: energy_result, once the call knows whether the host wants it)
        pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
        reduce_sum(e_part, elastic_grad_hess_blocks(ctx->n_list), coef, &ctx->iter.p->energy[kEnergyElastic], st);
        ctx->prof_end(pe);
        ++ctx->launches;
    }
    if (need_g) {
        // owned vertices gather their complete sums (every incident tet is in this rank's list); the other rows are written as zeros
        pe = ctx->prof_begin(IPCGPU_STAGE_GATHER_GRADIENT);
        gather_gradient(ctx->nV, ctx->inc_ptr.p, ctx->inc.p, ctx->gcont.p, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, 0, ctx->g.p, st);
        ctx->prof_end(pe);
        ++ctx->launches;
    }
    if (need_h) {
        pe = ctx->prof_begin(IPCGPU_STAGE_ASSEMBLE_CSR);
        assemble_csr(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->slot_off.p, ctx->con_ptr.p, ctx->con_src.p, ctx->hblk.p,
            ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, nullptr, 1, ctx->a.p, st);
        // per-vertex diagonal terms (mass, Dirichlet identity) of the owned rows
        const double* m = (add_mass && ctx->has_mass) ? ctx->mass.p : nullptr;
        diag_mass_dbc_range(ctx->v_begin, ctx->v_end, ctx->ia.p, ctx->index_base, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, m, ctx->a.p, st);
        ctx->prof_end(pe);
        ctx->launches += 2;
    }
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_elastic_gradient(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, int projectDBC, double* g)
{
    ENTER(g ? kSerial : kDerivative);
    int rc = run_grad_hess(ctx, coef, 1, projectDBC, true, false, 0);
    return rc || !g ? rc : gradient_roundtrip_end(ctx, g); // (the gradient is written, not accumulated: no roundtrip_begin)
}

int ipcgpu_elastic_hessian(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, int projectSPD, int projectDBC, double* a_inout)
{
    int rc = hessian_begin(ctx, kDerivative, a_inout);
    if (rc || (rc = run_grad_hess(ctx, coef, projectSPD, projectDBC, false, true, 0))) return rc;
    return hessian_end(ctx, a_inout, 0);
}

static int elastic_derivatives(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, bool with_energy, double* E, double* g, double* a)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(E || g || a ? kSerial : kDerivative);
    // the value array is rebuilt from scratch (LinSysSolver::setZero, then addCoeff of every term): slots that no local tet touches
    // -- contact-only blocks of the augmented pattern -- must not keep last iteration's values
    int rc = a ? sync_pattern_mirror(ctx) : 0; // (the host array holds the current pattern's values)
    if (rc || (rc = zero_values(ctx))) return rc;
    if ((rc = run_grad_hess(ctx, coef, projectSPD, projectDBC, true, true, add_mass, with_energy))) return rc;
    if (ctx->nranks > 1 && (g || a)) {
        rc = ipcgpu_allreduce_grad_hess(ctx, g ? 1 : 0, a ? 1 : 0);
        if (rc) return rc;
    }
    if (g) CK(cudaMemcpyAsync(g, ctx->g.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (a) CK(cudaMemcpyAsync(a, ctx->a.p, (size_t)ctx->nnz * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (with_energy && (rc = energy_result(ctx, kEnergyElastic, E))) return rc; // (a host E synchronises)
    if (!E && (g || a)) CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_elastic_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, double* g, double* a)
{
    return elastic_derivatives(ctx, coef, projectSPD, projectDBC, add_mass, false, nullptr, g, a);
}

int ipcgpu_elastic_energy_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, double* E, double* g, double* a)
{
    return elastic_derivatives(ctx, coef, projectSPD, projectDBC, add_mass, true, E, g, a);
}

// ---- step bound: device-resident chain ---------------------------------------------------------------------
int ipcgpu_step_bound_set(ipcgpu_ctx* ctx, double alpha)
{
    REQUIRE(alpha >= 0.0, IPCGPU_ERR_ARG, "the step must be non-negative");
    ENTER(kStepBound);
    step_set(ctx->iter.p, alpha, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_inversion_step(ipcgpu_ctx* ctx, const double* p, double slack, double* alpha_inout)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(p || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_INVERSION);
    inversion_step(ctx->eargs(), ctx->dir.p, slack, ctx->inv_steps.p, ctx->iter.p, ctx->stream);
    ctx->prof_end(pe);
    ctx->launches += 2;
    if ((rc = nccl_min_u64(ctx, &ctx->iter.p->inv_ord))) return rc;
    inversion_apply(ctx->iter.p, ctx->nT, ctx->stream); // Energy.cpp:576-579
    ++ctx->launches;
    CK(cudaGetLastError());
    if (alpha_inout) return ccd_read_back(ctx, alpha_inout);
    return IPCGPU_OK;
}

// ---- contact ---------------------------------------------------------------------------------------------
int ipcgpu_set_surface(ipcgpu_ctx* ctx, int nSV, const int* SVI, int nSE, const int* SE, int nSF, const int* SF, const int* vCoDim)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(nSV >= 0 && nSE >= 0 && nSF >= 0 && (nSV == 0 || SVI) && (nSE == 0 || SE) && (nSF == 0 || SF), IPCGPU_ERR_ARG, "ipcgpu_set_surface: bad arguments");
    for (int i = 0; i < nSV; ++i) REQUIRE(SVI[i] >= 0 && SVI[i] < ctx->nV, IPCGPU_ERR_ARG, "SVI out of range");
    for (int i = 0; i < 2 * nSE; ++i) REQUIRE(SE[i] >= 0 && SE[i] < ctx->nV, IPCGPU_ERR_ARG, "SFEdges out of range");
    for (size_t i = 0; i < (size_t)3 * nSF; ++i) REQUIRE(SF[i] >= 0 && SF[i] < ctx->nV, IPCGPU_ERR_ARG, "SF out of range");
    ctx->nSV = nSV; ctx->nSE = nSE; ctx->nSF = nSF;
    bool ok = ctx->SVI.upload(SVI, std::max(nSV, 0), ctx->stream) && ctx->SE.upload(SE, (size_t)2 * nSE, ctx->stream) && ctx->SF.upload(SF, (size_t)3 * nSF, ctx->stream);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "surface upload failed");
    ctx->has_codim = vCoDim != nullptr;
    if (vCoDim) REQUIRE(ctx->vCoDim.upload(vCoDim, ctx->nV, ctx->stream), IPCGPU_ERR_CUDA, "codim upload failed");
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->h_SVI.assign(SVI, SVI + nSV);
    ctx->hs_set_built = ctx->hs_lag_ready = false; // the plane sets index the old surface (and halfspace_alloc may reallocate them)
    ctx->pSize_surface = false; // pSize belongs to the surface
    int rc = contact_alloc(ctx);
    if (rc) return rc;
    if ((rc = ccd_alloc(ctx))) return rc;
    ctx->surface_ready = true;
    if (ctx->device_pattern) return ipcgpu_enable_device_pattern(ctx, ctx->index_base, ctx->pw.requested_cap); // new surface edges
    return IPCGPU_OK;
}

int ipcgpu_set_obstacle_tail(ipcgpu_ctx* ctx, int first_obstacle_vertex, int ee_through_vf_routine)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (the pair rules change)
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    if (first_obstacle_vertex < 0 || first_obstacle_vertex >= ctx->nV) { // no obstacle
        ctx->nVdof = 0x7fffffff;
        ctx->ee_as_vf = ee_through_vf_routine ? 1 : 0;
        ctx->pSize_surface = false;
        if (ctx->device_pattern) return ipcgpu_enable_device_pattern(ctx, ctx->index_base, ctx->pw.requested_cap); // the tail's pairs return
        return IPCGPU_OK;
    }
    REQUIRE(first_obstacle_vertex > 0, IPCGPU_ERR_ARG, "the mesh needs at least one vertex of its own");
    for (size_t i = 0; i < ctx->h_T.size(); ++i) REQUIRE(ctx->h_T[i] < first_obstacle_vertex, IPCGPU_ERR_ARG, "a tetrahedron uses an obstacle vertex");
    REQUIRE(ctx->has_dbc, IPCGPU_ERR_STATE, "the obstacle's vertices must be flagged Dirichlet (1) in ipcgpu_set_mesh: their rows never reach the system");
    {
        std::vector<uint8_t> tail((size_t)(ctx->nV - first_obstacle_vertex));
        CK(cudaMemcpyAsync(tail.data(), ctx->dbc.p + first_obstacle_vertex, tail.size(), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (uint8_t f : tail) REQUIRE(f == 1, IPCGPU_ERR_ARG, "the obstacle's vertices must be flagged Dirichlet (1) in ipcgpu_set_mesh");
    }
    ctx->nVdof = first_obstacle_vertex;
    ctx->ee_as_vf = ee_through_vf_routine ? 1 : 0;
    ctx->pSize_surface = false; // the mean |p| of the swept build is taken over the MESH's surface vertices: upload the direction again
    if (ctx->device_pattern) return ipcgpu_enable_device_pattern(ctx, ctx->index_base, ctx->pw.requested_cap); // the tail's pairs leave
    return IPCGPU_OK;
}

int ipcgpu_set_obstacle_positions(ipcgpu_ctx* ctx, const double* Vo_soa)
{
    REQUIRE(ctx->nV > 0 && ctx->nVdof < ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_obstacle_tail first");
    REQUIRE(Vo_soa, IPCGPU_ERR_ARG, "null argument");
    ENTER(kSerial);
    const size_t nVo = (size_t)(ctx->nV - ctx->nVdof);
    // current AND rest positions: the obstacle has no rest shape of its own, compute_eps_x takes its current edge lengths
    // (MeshCollisionUtils.hpp:2976-2981); SoA with the stride of the whole vertex array
    // (the saved line-search state keeps the old tail: move the obstacle BETWEEN line searches, or call ipcgpu_save_state again afterwards)
    for (double* dst : { ctx->V.p, ctx->Vrest.p })
        CK(cudaMemcpy2DAsync(dst + ctx->nVdof, (size_t)ctx->nV * sizeof(double), Vo_soa, nVo * sizeof(double), nVo * sizeof(double), 3, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream)); // (pageable host memory)
    ctx->mark_inputs();
    return IPCGPU_OK;
}

int ipcgpu_set_ccd_capacity(ipcgpu_ctx* ctx, uint64_t capacity)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(capacity > 0 && capacity < 0xffffffffull, IPCGPU_ERR_ARG, "capacity out of range");
    ctx->ccd_capacity = (size_t)capacity;
    if (ctx->surface_ready) return ccd_alloc(ctx);
    return IPCGPU_OK;
}

int ipcgpu_ti_error(const double* V, int nV, const double* p, double err_vf[3], double err_ee[3])
{
    if (!V || nV <= 0 || !err_vf || !err_ee) return IPCGPU_ERR_ARG;
    double lo[3] = { 1e300, 1e300, 1e300 }, hi[3] = { -1e300, -1e300, -1e300 };
    for (int v = 0; v < nV; ++v)
        for (int c = 0; c < 3; ++c) {
            const double x = V[(size_t)c * nV + v];
            lo[c] = std::min(lo[c], x);
            hi[c] = std::max(hi[c], x);
            if (p) {
                const double y = x + p[3 * (size_t)v + c];
                lo[c] = std::min(lo[c], y);
                hi[c] = std::max(hi[c], y);
            }
        }
    double diag2 = 0.0;
    for (int c = 0; c < 3; ++c) diag2 += (hi[c] - lo[c]) * (hi[c] - lo[c]);
    const double radius = 0.5 * std::sqrt(diag2);
    // Tight-Inclusion get_numerical_error with minimum separation: filter * max(1, |x|max)^3
    const double ee_filter = 7.105427357601002e-15, vf_filter = 7.549516567451064e-15;
    for (int c = 0; c < 3; ++c) {
        const double center = 0.5 * (lo[c] + hi[c]);
        const double a = center - 10.0 * radius / std::sqrt(3.0), b = center + 10.0 * radius / std::sqrt(3.0);
        double m = std::max(std::fabs(a), std::fabs(b));
        m = std::max(m, 1.0);
        err_ee[c] = m * m * m * ee_filter;
        err_vf[c] = m * m * m * vf_filter;
    }
    return IPCGPU_OK;
}

int ipcgpu_ccd_debug_seed_bound(ipcgpu_ctx* ctx, double toi)
{
    ctx->debug_prune_seed = toi;
    return IPCGPU_OK;
}

int ipcgpu_ccd_debug_thread_budget(ipcgpu_ctx* ctx, int64_t boxes)
{
    ctx->debug_ti_budget = boxes;
    return IPCGPU_OK;
}

int ipcgpu_ccd_partial_ti(ipcgpu_ctx* ctx, const double* p, double tol, const double err_vf[3], const double err_ee[3], double* alpha_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(err_vf && err_ee, IPCGPU_ERR_ARG, "null argument");
    ENTER(p || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    // CFL_FOR_CCD != 0: an empty candidate list leaves the step unchanged (:700).  Replicated lists: every rank walks a contiguous
    // slice; partitioned lists (ipcgpu_set_contact_partition) are already this rank's own.
    ContactWork& w = ctx->cw;
    const int share = (ctx->nranks > 1 && !ctx->lists_local) ? 1 : 0;
    if ((rc = ccd_narrow(ctx, w.cand.p, w.counters.p + 3, nullptr, (unsigned long long)4 * w.cap, share, tol, err_vf, err_ee, 1, nullptr))) return rc;
    if (alpha_inout) return ccd_read_back(ctx, alpha_inout);
    return IPCGPU_OK;
}

int ipcgpu_hash_build_swept(ipcgpu_ctx* ctx, const double* p, double* alpha_inout, double h)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(h > 0.0, IPCGPU_ERR_ARG, "bad arguments");
    ENTER(p || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    REQUIRE(ctx->pSize_surface, IPCGPU_ERR_STATE, "the search direction was uploaded before ipcgpu_set_surface: upload it again");
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    if ((rc = ccd_build_swept(ctx, h))) return rc;
    if (alpha_inout) return ccd_read_back(ctx, alpha_inout);
    return IPCGPU_OK;
}

int ipcgpu_ccd_full_ti(ipcgpu_ctx* ctx, double tol, const double err_vf[3], const double err_ee[3], double* alpha_inout, uint64_t* n_candidates)
{
    REQUIRE(ctx->surface_ready && ctx->ccd.swept_ready, IPCGPU_ERR_STATE, "ipcgpu_hash_build_swept first");
    REQUIRE(err_vf && err_ee, IPCGPU_ERR_ARG, "null argument");
    ENTER(alpha_inout || n_candidates ? kSerial : kStepBound);
    int rc;
    // (the swept grid was built for the step the chain held then; a host step that differs from it only lowers max_t)
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    if ((rc = ccd_full(ctx, tol, err_vf, err_ee))) return rc;
    if (alpha_inout || n_candidates) {
        if ((rc = ccd_read_back(ctx, alpha_inout))) return rc;
        if (n_candidates) *n_candidates = ctx->h_iter->n_full_cand;
        return flag_status(ctx, 1u << FLAG_CCD_CAPACITY);
    }
    return IPCGPU_OK;
}

int ipcgpu_ccd_stats(ipcgpu_ctx* ctx, uint64_t* candidates, uint64_t* survivors, uint64_t* warnings)
{
    if (candidates) *candidates = ctx->ccd.last_candidates;
    if (survivors) *survivors = ctx->ccd.last_survivors;
    if (warnings) *warnings = (uint64_t)ctx->ccd.last_warnings;
    return IPCGPU_OK;
}

int ipcgpu_ccd_stats_ex(ipcgpu_ctx* ctx, uint64_t* deferred, uint64_t* boxes_thread_pass, uint64_t* boxes_warp_pass)
{
    if (deferred) *deferred = ctx->ccd.last_deferred;
    if (boxes_thread_pass) *boxes_thread_pass = ctx->ccd.last_boxes_thread;
    if (boxes_warp_pass) *boxes_warp_pass = ctx->ccd.last_boxes_warp;
    return IPCGPU_OK;
}

int ipcgpu_ccd_stats_timing(ipcgpu_ctx* ctx, uint64_t* longest_pair_cycles, uint64_t* total_pair_cycles)
{
    if (longest_pair_cycles) *longest_pair_cycles = ctx->ccd.last_longest_cycles;
    if (total_pair_cycles) *total_pair_cycles = ctx->ccd.last_total_cycles;
    return IPCGPU_OK;
}

int ipcgpu_set_exchange_capacity(ipcgpu_ctx* ctx, int pairs_per_rank)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (the message buffers change)
    REQUIRE(pairs_per_rank > 0, IPCGPU_ERR_ARG, "capacity must be positive");
    ctx->exchange_capacity = pairs_per_rank;
    if (ctx->surface_ready) return contact_alloc(ctx);
    return IPCGPU_OK;
}

int ipcgpu_set_pair_capacity(ipcgpu_ctx* ctx, int capacity)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(capacity > 0, IPCGPU_ERR_ARG, "capacity must be positive");
    ctx->pair_capacity = capacity;
    if (ctx->surface_ready) return contact_alloc(ctx);
    return IPCGPU_OK;
}

int ipcgpu_constraint_set(ipcgpu_ctx* ctx, double dHat, int getPTEE, int* nC, int* nPara, int* nCand)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(dHat > 0.0, IPCGPU_ERR_ARG, "dHat must be positive");
    ENTER(kSerial);
    int rc = contact_constraint_set(ctx, dHat, getPTEE, nC, nPara, nCand);
    ctx->lists_local = (rc == 0) && ctx->partition_contact && ctx->nranks > 1;
    ctx->cw.lists_global = false;
    if (rc == 0 && ctx->lists_local) {
        // every rank holds a disjoint part of the sets: exchange them (one fixed-size message per rank) so that each rank can assemble
        // the Hessian rows it owns from ALL pairs that touch them
        ContactWork& w = ctx->cw;
        contact_pack_lists(ctx);
        cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
        int r = g_nccl.AllGather(w.xsend.p, w.xrecv.p, w.xstride * 4, kNcclInt32, ctx->nccl_comm, ctx->stream);
        ctx->prof_end(pe);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllGather(pair lists) failed");
        contact_unpack_lists(ctx);
        w.lists_global = true;
        CK(cudaGetLastError());
    }
    ctx->mark_inputs();
    return rc;
}

int ipcgpu_set_canonical_order(ipcgpu_ctx* ctx, int enable)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    ctx->canonical_order = enable != 0;
    return IPCGPU_OK;
}

int ipcgpu_set_contact_partition(ipcgpu_ctx* ctx, int enable)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    ctx->partition_contact = enable != 0;
    return IPCGPU_OK;
}

int ipcgpu_get_constraint_set(ipcgpu_ctx* ctx, int* mm, int* para, int* para_e, int* cand)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    ContactWork& w = ctx->cw;
    if (w.nC < 0) { // built without a read-back: fetch the sizes now
        int rc = contact_sync_counts(ctx);
        if (rc) return rc;
    }
    if (mm && w.nC) CK(cudaMemcpyAsync(mm, w.act.p, (size_t)w.nC * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
    if (para && w.nP) CK(cudaMemcpyAsync(para, w.para.p, (size_t)w.nP * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
    if (para_e && w.nP) CK(cudaMemcpyAsync(para_e, w.para_e.p, (size_t)w.nP * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    if (cand && w.nK) CK(cudaMemcpyAsync(cand, w.cand.p, (size_t)w.nK * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_constraint_set_sizes(ipcgpu_ctx* ctx, int* nC, int* nPara, int* nCand)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    ContactWork& w = ctx->cw;
    if (w.nC < 0) {
        int rc = contact_sync_counts(ctx);
        if (rc) return rc;
    }
    if (nC) *nC = w.nC;
    if (nPara) *nPara = w.nP;
    if (nCand) *nCand = w.nK;
    return IPCGPU_OK;
}

int ipcgpu_set_constraint_set(ipcgpu_ctx* ctx, int nC, const int* mm, int nP, const int* para, const int* para_e, int nK, const int* cand)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    ContactWork& w = ctx->cw;
    REQUIRE(nC >= 0 && nP >= 0 && nK >= 0 && nC <= w.cap && nP <= w.cap && nK <= 4 * w.cap, IPCGPU_ERR_CAPACITY, "set exceeds the pair capacity");
    if (nC) CK(cudaMemcpyAsync(w.act.p, mm, (size_t)nC * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
    if (nP) CK(cudaMemcpyAsync(w.para.p, para, (size_t)nP * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
    if (nP) CK(cudaMemcpyAsync(w.para_e.p, para_e, (size_t)nP * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream));
    if (nK) CK(cudaMemcpyAsync(w.cand.p, cand, (size_t)nK * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream));
    int* h = reinterpret_cast<int*>(ctx->h_scalar);
    for (int i = 0; i < 16; ++i) h[i] = 0;
    h[0] = nC; h[2] = nP; h[3] = nK;
    CK(cudaMemcpyAsync(w.counters.p, h, 16 * sizeof(int), cudaMemcpyHostToDevice, ctx->stream)); // the consumers read the sizes on the device
    CK(cudaStreamSynchronize(ctx->stream));
    w.nC = nC; w.nP = nP; w.nK = nK;
    w.want_cand = nK > 0;
    ctx->lists_local = false; // uploaded sets are the global ones
    w.lists_global = false;
    ctx->mark_inputs();
    return IPCGPU_OK;
}

static BarrierArgs barrier_args(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC)
{
    BarrierArgs p;
    ContactWork& w = ctx->cw;
    p.nV = ctx->nV; p.V = ctx->V.p; p.Vrest = ctx->Vrest.p; p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr; p.SE = ctx->SE.p;
    p.nVdof = ctx->nVdof;
    // one rank: the lists as built.  Several ranks: the GLOBAL lists (replicated build, or partitioned build + exchange); energy and
    // gradient take a contiguous share of them, the Hessian goes by row owner.
    if (ctx->nranks > 1 && w.lists_global) {
        p.cs = w.gact.p; p.nC = w.counters.p + 10; p.para = w.gpara.p; p.para_e = w.gpara_e.p; p.nP = w.counters.p + 11;
    }
    else {
        p.cs = w.act.p; p.nC = w.counters.p + 0; p.para = w.para.p; p.para_e = w.para_e.p; p.nP = w.counters.p + 2;
    }
    p.rank = ctx->rank; p.nranks = ctx->nranks; p.share = ctx->nranks > 1 ? 1 : 0;
    p.row_lo = ctx->nranks > 1 ? ctx->v_begin : 0;
    p.row_hi = ctx->nranks > 1 ? ctx->v_end : ctx->nV;
    p.dHat = dHat; p.kappa = kappa; p.projectDBC = projectDBC;
    p.ia = ctx->ia.p; p.ja = ctx->ja.p; p.base = ctx->index_base;
    return p;
}

// ---- device-built sparsity pattern (pattern.cu) -------------------------------------------------------------------------
int ipcgpu_enable_device_pattern(ipcgpu_ctx* ctx, int index_base, uint64_t nnz_capacity)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (ja / a may be reallocated)
    REQUIRE(ctx->maps_ready && ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(index_base == 0 || index_base == 1, IPCGPU_ERR_ARG, "index_base must be 0 or 1");
    ctx->device_pattern = false;
    int rc = pattern_enable(ctx, index_base, nnz_capacity);
    if (rc) return rc;
    ctx->device_pattern = true;
    ctx->pat_pending = false;
    ctx->pat_seen_version = 0;
    ctx->pat_changed_host = 0;
    ctx->a_all_dirty = false;
    ctx->offsets_ready = false;
    ctx->full_pattern_ready = false;
    owned_value_range(ctx);
    return ensure_offsets(ctx);
}

int ipcgpu_update_pattern(ipcgpu_ctx* ctx, int with_friction, int* changed, int64_t* nnz)
{
    REQUIRE(ctx->device_pattern, IPCGPU_ERR_STATE, "ipcgpu_enable_device_pattern first");
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(!with_friction || ctx->cw.fr_ready, IPCGPU_ERR_STATE, "with_friction: ipcgpu_friction_lag / ipcgpu_set_friction_data first");
    ENTER(kSerial);
    int rc = pattern_update(ctx, barrier_args(ctx, 1.0, 1.0, 0), with_friction != 0);
    if (rc) return rc;
    ctx->pat_pending = true;
    if (!changed && !nnz) return IPCGPU_OK;
    if ((rc = sync_pattern_mirror(ctx))) return rc;
    if (changed) *changed = ctx->pat_changed_host;
    if (nnz) *nnz = ctx->nnz;
    return flag_status(ctx, 1u << FLAG_PATTERN_CAPACITY);
}

int ipcgpu_pattern_info(ipcgpu_ctx* ctx, int* changed, int64_t* nnz, uint64_t* version)
{
    REQUIRE(ctx->device_pattern, IPCGPU_ERR_STATE, "ipcgpu_enable_device_pattern first");
    ENTER(kSerial);
    int rc = sync_pattern_mirror(ctx);
    if (rc) return rc;
    if (changed) *changed = ctx->pat_changed_host;
    if (nnz) *nnz = ctx->nnz;
    if (version) *version = ctx->pat_seen_version;
    return IPCGPU_OK;
}

int ipcgpu_get_pattern(ipcgpu_ctx* ctx, int* ia, int* ja)
{
    REQUIRE(ctx->n_rows > 0, IPCGPU_ERR_STATE, "no pattern: ipcgpu_set_csr or ipcgpu_enable_device_pattern first");
    ENTER(kSerial);
    int rc = sync_pattern_mirror(ctx);
    if (rc) return rc;
    if (ia) CK(cudaMemcpyAsync(ia, ctx->ia.p, ((size_t)ctx->n_rows + 1) * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (ja) CK(cudaMemcpyAsync(ja, ctx->ja.p, (size_t)ctx->nnz * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_barrier_energy(ipcgpu_ctx* ctx, double dHat, double kappa, double* E)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    BarrierArgs p = barrier_args(ctx, dHat, kappa, 0);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    barrier_energy(p, ctx->cw.bpartials.p, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE], ctx->stream);
    // synchronous form: the d <= 0 flag is checked right here (every rank checks its own share of the pairs)
    return energy_tail(ctx, kEnergyBarrier, ctx->cw.bpartials.p, barrier_energy_blocks(), kappa, pe, E, true, 1u << FLAG_NONPOSITIVE_DISTANCE);
}

int ipcgpu_barrier_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    const BarrierArgs p = barrier_args(ctx, dHat, kappa, 0);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { barrier_gradient(p, ctx->g.p, st); });
}

int ipcgpu_evaluate_constraints(ipcgpu_ctx* ctx, double* val, int n)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    ContactWork& w = ctx->cw;
    if (w.nC < 0) {
        int rc = contact_sync_counts(ctx);
        if (rc) return rc;
    }
    REQUIRE(n == w.nC && (val || n == 0), IPCGPU_ERR_ARG, "ipcgpu_evaluate_constraints: n must be the size of the active set on this context");
    ALLOC(w.bval, (size_t)std::max(w.cap, 1));
    BarrierArgs p = barrier_args(ctx, 1.0, 1.0, 0);
    p.cs = w.act.p; p.nC = w.counters.p + 0; // this context's own active list (what ipcgpu_get_constraint_set returns), not the exchanged one
    evaluate_constraints(p, w.bval.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    if (n) CK(cudaMemcpyAsync(val, w.bval.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_constraint_jacobian_t(ipcgpu_ctx* ctx, const double* input, int n, double coef, double* g_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(g_inout != nullptr, IPCGPU_ERR_ARG, "null gradient");
    ENTER(kSerial);
    ContactWork& w = ctx->cw;
    if (w.nC < 0) {
        int rc = contact_sync_counts(ctx);
        if (rc) return rc;
    }
    REQUIRE(n == w.nC && (input || n == 0), IPCGPU_ERR_ARG, "ipcgpu_constraint_jacobian_t: n must be the size of the active set on this context");
    REQUIRE(!(ctx->nranks > 1 && ctx->lists_local), IPCGPU_ERR_STATE, "per-constraint input needs the replicated sets (ipcgpu_set_contact_partition(0))");
    ALLOC(w.bval, (size_t)std::max(w.cap, 1));
    int rc = gradient_roundtrip_begin(ctx, g_inout);
    if (rc) return rc;
    if (n) CK(cudaMemcpyAsync(w.bval.p, input, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    BarrierArgs p = barrier_args(ctx, 1.0, 1.0, 0);
    p.cs = w.act.p; p.nC = w.counters.p + 0;
    constraint_jacobian_t(p, w.bval.p, coef, ctx->g.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return gradient_roundtrip_end(ctx, g_inout);
}

int ipcgpu_para_ee_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(g_inout != nullptr, IPCGPU_ERR_ARG, "null gradient");
    ENTER(kSerial);
    int rc = gradient_roundtrip_begin(ctx, g_inout);
    if (rc) return rc;
    para_gradient(barrier_args(ctx, dHat, kappa, 0), ctx->g.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return gradient_roundtrip_end(ctx, g_inout);
}

int ipcgpu_barrier_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    int rc = hessian_begin(ctx, kDerivative, a_inout);
    if (rc) return rc;
    ContactWork& w = ctx->cw;
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    const BarrierArgs bp = barrier_args(ctx, dHat, kappa, projectDBC);
    cudaStream_t st = ctx->deriv_stream();
    if (ctx->inputs_marked) {
        // build + projection on the side stream, ordered after the last change of their inputs (positions, contact sets) -- i.e. next to
        // whatever has been queued since (the elastic assembly); the scatter joins the derivative chain, after the elastic writes
        CK(cudaStreamWaitEvent(ctx->side, ctx->ev_inputs, 0));
        if (ctx->scatter_marked) CK(cudaStreamWaitEvent(ctx->side, ctx->ev_scatter, 0)); // back-to-back calls: the last scatter still reads the buffers
        barrier_hessian_build_project(bp, ctx->iter.p->flags, w.bHraw.p, w.brows.p, w.bpsd.p, w.counters.p + 12, w.cap, ctx->side);
        CK(cudaEventRecord(ctx->ev_join, ctx->side));
        CK(cudaStreamWaitEvent(st, ctx->ev_join, 0));
    }
    else barrier_hessian_build_project(bp, ctx->iter.p->flags, w.bHraw.p, w.brows.p, w.bpsd.p, w.counters.p + 12, w.cap, st);
    barrier_hessian_scatter(bp, ctx->a.p, ctx->iter.p->flags, w.bHraw.p, w.brows.p, w.bpsd.p, w.counters.p + 12, w.cap, st);
    ctx->scatter_marked = (cudaEventRecord(ctx->ev_scatter, st) == cudaSuccess);
    ctx->prof_end(pe);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return hessian_end(ctx, a_inout, (1u << FLAG_PATTERN) | (1u << FLAG_SET_CAPACITY));
}

// ---- lagged friction of the self-contact pairs (SURVEY 8 f4) --------------------------------------------------------------
int ipcgpu_set_prev_state(ipcgpu_ctx* ctx, const double* V_prev_soa)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    ALLOC(ctx->Vprev, (size_t)3 * ctx->nV);
    if (V_prev_soa) CK(cudaMemcpyAsync(ctx->Vprev.p, V_prev_soa, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    else CK(cudaMemcpyAsync(ctx->Vprev.p, ctx->V.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream)); // V_prev = V at the start of a step
    ctx->prev_set = true;
    return IPCGPU_OK;
}

static int friction_alloc(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    const size_t cap = (size_t)std::max(ctx->pair_capacity, 1);
    ALLOC(w.fr_cs, cap);
    ALLOC(w.fr_n, 1);
    ALLOC(w.fr_lambda, cap);
    ALLOC(w.fr_coord, cap);
    ALLOC(w.fr_basis, 6 * cap);
    ALLOC(w.fr_partials, (size_t)friction_energy_blocks() + 8);
    return IPCGPU_OK;
}

int ipcgpu_friction_lag(ipcgpu_ctx* ctx, double dHat, double kappa, int* n_pairs)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    int rc = friction_alloc(ctx);
    if (rc) return rc;
    ContactWork& w = ctx->cw;
    // the lagged set is the whole active set on every rank (the global list after a partitioned build)
    friction_lag(barrier_args(ctx, dHat, kappa, 0), w.fr_cs.p, w.fr_n.p, w.fr_lambda.p, w.fr_coord.p, w.fr_basis.p, ctx->pair_capacity,
        &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE], ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    w.fr_ready = true;
    w.fr_host_n = -1;
    if (n_pairs) {
        CK(cudaMemcpyAsync(ctx->h_scalar, w.fr_n.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        w.fr_host_n = *reinterpret_cast<int*>(ctx->h_scalar);
        *n_pairs = w.fr_host_n;
    }
    return IPCGPU_OK;
}

static int friction_host_count(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    if (w.fr_host_n < 0) {
        CK(cudaMemcpyAsync(ctx->h_scalar, w.fr_n.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        w.fr_host_n = *reinterpret_cast<int*>(ctx->h_scalar);
    }
    return IPCGPU_OK;
}

int ipcgpu_get_friction_data(ipcgpu_ctx* ctx, int* n_pairs, int* mmcvid4, double* lambda, double* coord2, double* basis6)
{
    REQUIRE(ctx->cw.fr_ready, IPCGPU_ERR_STATE, "ipcgpu_friction_lag / ipcgpu_set_friction_data first");
    ENTER(kSerial);
    int rc = friction_host_count(ctx);
    if (rc) return rc;
    ContactWork& w = ctx->cw;
    const size_t n = (size_t)w.fr_host_n;
    if (n_pairs) *n_pairs = w.fr_host_n;
    if (n && mmcvid4) CK(cudaMemcpyAsync(mmcvid4, w.fr_cs.p, n * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
    if (n && lambda) CK(cudaMemcpyAsync(lambda, w.fr_lambda.p, n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (n && coord2) CK(cudaMemcpyAsync(coord2, w.fr_coord.p, n * sizeof(double2), cudaMemcpyDeviceToHost, ctx->stream));
    if (n && basis6) CK(cudaMemcpyAsync(basis6, w.fr_basis.p, 6 * n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_set_friction_data(ipcgpu_ctx* ctx, int n_pairs, const int* mmcvid4, const double* lambda, const double* coord2, const double* basis6)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(n_pairs >= 0 && n_pairs <= ctx->pair_capacity, IPCGPU_ERR_CAPACITY, "friction set larger than the pair capacity");
    REQUIRE(n_pairs == 0 || (mmcvid4 && lambda && coord2 && basis6), IPCGPU_ERR_ARG, "null friction arrays");
    ENTER(kSerial);
    int rc = friction_alloc(ctx);
    if (rc) return rc;
    ContactWork& w = ctx->cw;
    const size_t n = (size_t)n_pairs;
    if (n) {
        CK(cudaMemcpyAsync(w.fr_cs.p, mmcvid4, n * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(w.fr_lambda.p, lambda, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(w.fr_coord.p, coord2, n * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(w.fr_basis.p, basis6, 6 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaMemcpyAsync(w.fr_n.p, &n_pairs, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream)); // n_pairs lives on the caller's stack
    w.fr_host_n = n_pairs;
    w.fr_ready = true;
    return IPCGPU_OK;
}

static FrictionArgs friction_args(ipcgpu_ctx* ctx, double eps2, double coef, int projectDBC)
{
    FrictionArgs p;
    ContactWork& w = ctx->cw;
    p.nV = ctx->nV; p.V = ctx->V.p; p.Vt = ctx->Vprev.p; p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    p.cs = w.fr_cs.p; p.n = w.fr_n.p; p.lambda = w.fr_lambda.p; p.coord = w.fr_coord.p; p.basis = w.fr_basis.p;
    p.eps2 = eps2; p.coef = coef; p.projectDBC = projectDBC;
    p.ia = ctx->ia.p; p.ja = ctx->ja.p; p.base = ctx->index_base;
    p.rank = ctx->rank; p.nranks = ctx->nranks;
    p.row_lo = ctx->nranks > 1 ? ctx->v_begin : 0;
    p.row_hi = ctx->nranks > 1 ? ctx->v_end : ctx->nV;
    return p;
}
#define REQUIRE_FRICTION() \
    REQUIRE(ctx->cw.fr_ready, IPCGPU_ERR_STATE, "ipcgpu_friction_lag / ipcgpu_set_friction_data first"); \
    REQUIRE(ctx->prev_set, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first")

int ipcgpu_friction_energy(ipcgpu_ctx* ctx, double eps2, double coef, double* E)
{
    REQUIRE_FRICTION();
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    friction_energy(friction_args(ctx, eps2, coef, 0), ctx->cw.fr_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyFriction, ctx->cw.fr_partials.p, friction_energy_blocks(), coef, pe, E);
}

int ipcgpu_friction_gradient(ipcgpu_ctx* ctx, double eps2, double coef, double* g_inout)
{
    REQUIRE_FRICTION();
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive");
    const FrictionArgs p = friction_args(ctx, eps2, coef, 0);
    return gradient_call(ctx, kSerial, g_inout, [&](cudaStream_t st) { friction_gradient(p, ctx->g.p, st); });
}

int ipcgpu_friction_hessian(ipcgpu_ctx* ctx, double eps2, double coef, int projectDBC, double* a_inout)
{
    REQUIRE_FRICTION();
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive");
    const FrictionArgs p = friction_args(ctx, eps2, coef, projectDBC);
    return hessian_call(ctx, kSerial, a_inout, 1u << FLAG_PATTERN,
        [&](cudaStream_t st) { friction_hessian(p, ctx->a.p, ctx->iter.p->flags + FLAG_PATTERN, st); });
}

// ---- inertia term (Optimizer.cpp:3227-3239, :3439-3450) ---------------------------------------------------------------------
int ipcgpu_set_xtilde(ipcgpu_ctx* ctx, const double* xtilde_soa)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(xtilde_soa != nullptr, IPCGPU_ERR_ARG, "null xTilta");
    ENTER(kSerial);
    ALLOC(ctx->xtilde, (size_t)3 * ctx->nV);
    CK(cudaMemcpyAsync(ctx->xtilde.p, xtilde_soa, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->xtilde_set = true;
    return IPCGPU_OK;
}

int ipcgpu_inertia_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE(ctx->xtilde_set && ctx->has_mass, IPCGPU_ERR_STATE, "ipcgpu_set_xtilde and a mass diagonal (ipcgpu_set_mesh) first");
    ENTER(kSerial);
    // vertex blocks [nV r / N, nV (r+1) / N): every vertex exactly once across the ranks
    const int v0 = (int)((long long)ctx->nV * ctx->rank / ctx->nranks), v1 = (int)((long long)ctx->nV * (ctx->rank + 1) / ctx->nranks);
    ALLOC(ctx->in_partials, (size_t)inertia_energy_blocks(ctx->nV) + 8);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
    inertia_energy(v0, v1, ctx->nV, ctx->V.p, ctx->xtilde.p, ctx->mass.p, ctx->in_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyInertia, ctx->in_partials.p, inertia_energy_blocks(v1 - v0), 1.0, pe, E);
}

int ipcgpu_inertia_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE(ctx->xtilde_set && ctx->has_mass, IPCGPU_ERR_STATE, "ipcgpu_set_xtilde and a mass diagonal (ipcgpu_set_mesh) first");
    ENTER(kSerial);
    if (g_inout) CK(cudaMemcpyAsync(ctx->g.p, g_inout, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    // Device-resident form with several ranks: the gradient is summed over the ranks later (ipcgpu_allreduce_grad_hess), so only rank 0 adds
    // the per-vertex term.  Host form: every rank holds the caller's vector and adds the full term -- no reduction needed, which is why this
    // is not a gradient_call (whose host form sums the ranks' vectors).
    if (g_inout || ctx->nranks == 1 || ctx->rank == 0) {
        inertia_gradient(ctx->nV, ctx->V.p, ctx->xtilde.p, ctx->mass.p, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, ctx->g.p, ctx->stream);
        ++ctx->launches;
    }
    CK(cudaGetLastError());
    if (g_inout) {
        CK(cudaMemcpyAsync(g_inout, ctx->g.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return IPCGPU_OK;
}

// ---- Rayleigh damping, Neumann forces, augmented-Lagrangian Dirichlet penalty (damping.cu; which chain each call runs on: see enter()) ------
#define REQUIRE_ONE_RANK() REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "damping, Neumann forces and the Dirichlet penalty run on one rank")

// a term switched on or off: graphs that bake the line search's set of terms in are refused, and the term's energy slot reads 0 while it is off
static int term_switched(ipcgpu_ctx* ctx, int slot)
{
    ++ctx->epoch;
    CK(cudaMemsetAsync(&ctx->iter.p->energy[slot], 0, sizeof(double), ctx->stream));
    return IPCGPU_OK;
}

static DampingArgs damping_args(ipcgpu_ctx* ctx)
{
    DampingArgs p;
    p.nV = ctx->nV; p.nSlots = ctx->nSlots;
    p.slot_v = ctx->slot_v.p; p.slot_u = ctx->slot_u.p;
    p.inc_ptr = ctx->damp_inc_ptr.p; p.inc = ctx->damp_inc.p;
    p.D = ctx->damp_D.p;
    p.V = ctx->V.p; p.Vprev = ctx->Vprev.p;
    p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    return p;
}

// the slot incidence of every vertex (once per mesh): the slots in which it is slot_v (entry 2s), then those in which it is the slot_u of an
// off-diagonal slot (2s + 1), each group in slot order
static int damping_incidence(ipcgpu_ctx* ctx)
{
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "run ipcgpu_damping_update once outside a capture first (it builds the slot incidence)");
    const int nS = ctx->nSlots, nV = ctx->nV;
    std::vector<int> sv((size_t)std::max(nS, 1)), su((size_t)std::max(nS, 1));
    CK(cudaMemcpyAsync(sv.data(), ctx->slot_v.p, (size_t)nS * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(su.data(), ctx->slot_u.p, (size_t)nS * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<int> ptr((size_t)nV + 1, 0);
    for (int s = 0; s < nS; ++s) {
        ++ptr[(size_t)sv[s] + 1];
        if (sv[s] != su[s]) ++ptr[(size_t)su[s] + 1];
    }
    for (int v = 0; v < nV; ++v) ptr[(size_t)v + 1] += ptr[v];
    std::vector<int> inc((size_t)std::max(ptr[nV], 1)), cur(ptr.begin(), ptr.end() - 1);
    for (int s = 0; s < nS; ++s) inc[(size_t)cur[sv[s]]++] = 2 * s;
    for (int s = 0; s < nS; ++s)
        if (sv[s] != su[s]) inc[(size_t)cur[su[s]]++] = 2 * s + 1;
    REQUIRE(ctx->damp_inc_ptr.upload(ptr.data(), ptr.size(), ctx->stream) && ctx->damp_inc.upload(inc.data(), inc.size(), ctx->stream), IPCGPU_ERR_CUDA,
        "upload of the damping incidence failed");
    CK(cudaStreamSynchronize(ctx->stream)); // host vectors go out of scope
    ctx->damp_inc_ready = true;
    return IPCGPU_OK;
}

int ipcgpu_damping_update(ipcgpu_ctx* ctx, double coef)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    int rc;
    if (coef == 0.0) { // no damping term
        if (ctx->damp_on && (rc = term_switched(ctx, kEnergyDamping))) return rc;
        ctx->damp_on = false;
        return IPCGPU_OK;
    }
    if (!ctx->damp_inc_ready && (rc = damping_incidence(ctx))) return rc;
    ALLOC(ctx->damp_D, (size_t)9 * std::max(ctx->nSlots, 1));
    ALLOC(ctx->damp_partials, (size_t)damping_energy_blocks(ctx->nSlots) + 8);
    // computeDampingMtr (Optimizer.cpp:3723-3734): the elastic Hessian at the current state, coef, projected (projectSPD = projectDBC = 1)
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    elastic_grad_hess(ctx->eargs(), coef, 1, false, true, ctx->gcont.p, ctx->hblk.p, ctx->stream);
    ctx->hblk_valid = true; // (IPCGPU_BUF_TET_HESSIANS now holds the damping's per-tet blocks)
    damping_assemble(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->con_ptr.p, ctx->con_src.p, ctx->hblk.p, ctx->has_dbc ? ctx->dbc.p : nullptr,
        ctx->damp_D.p, ctx->stream);
    ctx->prof_end(pe);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (!ctx->damp_on && (rc = term_switched(ctx, kEnergyDamping))) return rc;
    ctx->damp_on = true;
    return IPCGPU_OK;
}

#define REQUIRE_DAMPING()                                                                                                \
    REQUIRE(ctx->damp_on, IPCGPU_ERR_STATE, "ipcgpu_damping_update with a nonzero coefficient first");                  \
    REQUIRE(ctx->prev_set, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first");                                              \
    REQUIRE_ONE_RANK()

int ipcgpu_damping_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE_DAMPING();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    damping_energy(damping_args(ctx), ctx->damp_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyDamping, ctx->damp_partials.p, damping_energy_blocks(ctx->nSlots), 0.5, pe, E);
}

int ipcgpu_damping_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE_DAMPING();
    const DampingArgs p = damping_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { damping_gradient(p, projectDBC, ctx->g.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_damping_hessian(ipcgpu_ctx* ctx, double* a_inout)
{
    REQUIRE_DAMPING();
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    if (!ctx->offsets_ready) { // (the slot offsets of a new host pattern: one synchronising check, as the first elastic Hessian does)
        ENTER(kSerial);
        int rc = ensure_offsets(ctx);
        if (rc) return rc;
    }
    const DampingArgs p = damping_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { damping_hessian(p, ctx->slot_off.p, ctx->a.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_set_neumann_forces(ipcgpu_ctx* ctx, double coef, const double* f)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(!f || ctx->has_mass, IPCGPU_ERR_STATE, "Neumann forces need the mass diagonal (ipcgpu_set_mesh)");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    int rc;
    if (f) {
        ALLOC(ctx->nbc_f, (size_t)3 * ctx->nV);
        ALLOC(ctx->nbc_partials, (size_t)vertex_energy_blocks(ctx->nV) + 8);
        CK(cudaMemcpyAsync(ctx->nbc_f.p, f, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream)); // (f is the caller's: the upload completes here)
    }
    set_double(&ctx->iter.p->nbc_coef, coef, ctx->stream); // (read at run time, like the forces: a new dt needs no new capture)
    ++ctx->launches;
    CK(cudaGetLastError());
    if ((f != nullptr) != ctx->nbc_on && (rc = term_switched(ctx, kEnergyNeumann))) return rc;
    ctx->nbc_on = f != nullptr;
    return IPCGPU_OK;
}

#define REQUIRE_NEUMANN()                                                                                   \
    REQUIRE(ctx->nbc_on, IPCGPU_ERR_STATE, "ipcgpu_set_neumann_forces first");                             \
    REQUIRE_ONE_RANK()

int ipcgpu_neumann_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE_NEUMANN();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    neumann_energy(ctx->nV, ctx->V.p, ctx->nbc_f.p, ctx->mass.p, ctx->has_dbc ? ctx->dbc.p : nullptr, &ctx->iter.p->nbc_coef, ctx->nbc_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyNeumann, ctx->nbc_partials.p, vertex_energy_blocks(ctx->nV), 1.0, pe, E);
}

int ipcgpu_neumann_gradient(ipcgpu_ctx* ctx, double* g_inout)
{
    REQUIRE_NEUMANN();
    const uint8_t* dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    const double* coef = &ctx->iter.p->nbc_coef;
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { neumann_gradient(ctx->nV, ctx->nbc_f.p, ctx->mass.p, dbc, coef, ctx->g.p, st); },
        IPCGPU_STAGE_DAMPING_BC);
}

static DirichletArgs dirichlet_args(ipcgpu_ctx* ctx)
{
    DirichletArgs p;
    p.n = ctx->n_dbc; p.nV = ctx->nV;
    p.vid = ctx->dbc_vid.p; p.tgt = ctx->dbc_tgt.p; p.lam = ctx->dbc_lam.p;
    p.V = ctx->V.p; p.mass = ctx->mass.p;
    p.rho = &ctx->iter.p->dbc_rho;
    return p;
}

int ipcgpu_set_dirichlet_targets(ipcgpu_ctx* ctx, int n, const int* vid, const double* target, const double* lambda, double dist2Tol)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(n >= 0 && (n == 0 || (vid && target)), IPCGPU_ERR_ARG, "ipcgpu_set_dirichlet_targets: bad arguments");
    REQUIRE(n == 0 || ctx->has_mass, IPCGPU_ERR_STATE, "the Dirichlet penalty needs the mass diagonal (ipcgpu_set_mesh)");
    {
        // targetPos is a map: one target per vertex (the gradient / Hessian kernels update a vertex's rows from one thread)
        std::vector<char> seen((size_t)ctx->nV, 0);
        for (int i = 0; i < n; ++i) {
            REQUIRE(vid[i] >= 0 && vid[i] < ctx->nV, IPCGPU_ERR_ARG, "Dirichlet target vertex out of range");
            REQUIRE(!seen[(size_t)vid[i]], IPCGPU_ERR_ARG, "Dirichlet target vertices must be distinct");
            seen[(size_t)vid[i]] = 1;
        }
    }
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    if (n > 0) {
        ALLOC(ctx->dbc_vid, (size_t)n);
        ALLOC(ctx->dbc_tgt, (size_t)3 * n);
        ALLOC(ctx->dbc_lam, (size_t)3 * n);
        ALLOC(ctx->dbc_partials, (size_t)vertex_energy_blocks(n) + 8);
        CK(cudaMemcpyAsync(ctx->dbc_vid.p, vid, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->dbc_tgt.p, target, (size_t)3 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        if (lambda) CK(cudaMemcpyAsync(ctx->dbc_lam.p, lambda, (size_t)3 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        else CK(cudaMemsetAsync(ctx->dbc_lam.p, 0, (size_t)3 * n * sizeof(double), ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream)); // (the arrays are the caller's: the upload completes here)
    }
    // the number of targets is a launch shape (a new number needs a new capture); the same number with new values does not
    if (n != ctx->n_dbc) {
        int rc = term_switched(ctx, kEnergyDirichlet);
        if (rc) return rc;
    }
    ctx->n_dbc = n;
    set_double(&ctx->iter.p->dbc_tol, n ? dist2Tol : 0.0, ctx->stream); // (stream order: a new dist2Tol per time step needs no new capture)
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_set_dirichlet_penalty(ipcgpu_ctx* ctx, double rho)
{
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    set_double(&ctx->iter.p->dbc_rho, rho, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_get_dirichlet_lambda(ipcgpu_ctx* ctx, double* lambda)
{
    REQUIRE(lambda != nullptr, IPCGPU_ERR_ARG, "null output");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    if (ctx->n_dbc > 0) CK(cudaMemcpyAsync(lambda, ctx->dbc_lam.p, (size_t)3 * ctx->n_dbc * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

#define REQUIRE_DIRICHLET()                                                                                                   \
    REQUIRE_ONE_RANK();                                                                                                        \
    if (ctx->n_dbc == 0) return IPCGPU_OK

int ipcgpu_dirichlet_energy(ipcgpu_ctx* ctx, double* E)
{
    if (E) *E = 0.0;
    REQUIRE_DIRICHLET();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    dirichlet_energy(dirichlet_args(ctx), ctx->dbc_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyDirichlet, ctx->dbc_partials.p, vertex_energy_blocks(ctx->n_dbc), 1.0, pe, E);
}

int ipcgpu_dirichlet_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE_DIRICHLET();
    if (projectDBC) return IPCGPU_OK; // (Optimizer.cpp:3542)
    const DirichletArgs p = dirichlet_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { dirichlet_gradient(p, ctx->g.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_dirichlet_hessian(ipcgpu_ctx* ctx, int projectDBC, double* a_inout)
{
    REQUIRE_DIRICHLET();
    if (projectDBC) return IPCGPU_OK; // (:3711)
    const DirichletArgs p = dirichlet_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { dirichlet_hessian(p, ctx->ia.p, ctx->index_base, ctx->a.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_dirichlet_update_lambda(ipcgpu_ctx* ctx)
{
    REQUIRE_DIRICHLET();
    ENTER(kSerial);
    dirichlet_update_lambda(dirichlet_args(ctx), ctx->dbc_lam.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_dirichlet_completed_step(ipcgpu_ctx* ctx, double* s)
{
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    ALLOC(ctx->dbc_partials, (size_t)vertex_energy_blocks(ctx->n_dbc) + 8);
    dirichlet_completed_step(dirichlet_args(ctx), &ctx->iter.p->dbc_tol, ctx->dbc_partials.p, &ctx->iter.p->dbc_step, ctx->stream);
    ctx->launches += ctx->n_dbc ? 3 : 2;
    CK(cudaGetLastError());
    if (!s) return IPCGPU_OK;
    CK(cudaMemcpyAsync(ctx->h_scalar, &ctx->iter.p->dbc_step, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *s = ctx->h_scalar[0];
    return IPCGPU_OK;
}

// ---- analytic half-space collision objects (halfspace.cu; which chain each call runs on: see enter()) ------------------------------------
static HalfSpaceArgs halfspace_args(ipcgpu_ctx* ctx)
{
    HalfSpaceArgs p;
    p.nV = ctx->nV; p.nSV = ctx->nSV; p.nP = ctx->n_hs;
    p.SVI = ctx->SVI.p; p.V = ctx->V.p; p.Vt = ctx->Vprev.p;
    p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr; p.vCoDim = ctx->has_codim ? ctx->vCoDim.p : nullptr;
    p.par = ctx->hs_par.p;
    p.act = ctx->hs_act.p; p.n_act = ctx->hs_cnt.p;
    p.lag = ctx->hs_lag.p; p.lam = ctx->hs_lam.p; p.n_lag = ctx->hs_cnt.p + 1;
    p.row_lo = ctx->nranks > 1 ? ctx->v_begin : 0;
    p.row_hi = ctx->nranks > 1 ? ctx->v_end : ctx->nV;
    p.ia = ctx->ia.p; p.base = ctx->index_base;
    return p;
}

int ipcgpu_set_halfspaces(ipcgpu_ctx* ctx, int n, const double* origin, const double* normal, const double* velocitydt, const double* friction)
{
    REQUIRE(n >= 0 && n <= kMaxPlanes, IPCGPU_ERR_ARG, "at most 8 half-spaces");
    REQUIRE(n == 0 || (origin && normal && friction), IPCGPU_ERR_ARG, "null half-space arrays");
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    std::vector<double> par((size_t)kPlaneStride * std::max(n, 1), 0.0);
    for (int k = 0; k < n; ++k) {
        const double* o = origin + 3 * k;
        const double* nr = normal + 3 * k;
        const double z = (nr[0] * nr[0] + nr[1] * nr[1]) + nr[2] * nr[2]; // normal.normalize() (HalfSpace.cpp:49)
        REQUIRE(z > 0.0, IPCGPU_ERR_ARG, "half-space normal is zero");
        const double s = std::sqrt(z);
        double* q = par.data() + kPlaneStride * k;
        for (int r = 0; r < 3; ++r) q[r] = nr[r] / s;
        q[3] = -((q[0] * o[0] + q[1] * o[1]) + q[2] * o[2]); // D = -normal.dot(origin) (:51)
        for (int r = 0; r < 3; ++r) q[4 + r] = velocitydt ? velocitydt[3 * k + r] : 0.0;
        q[7] = friction[k];
    }
    if (n != ctx->n_hs) {
        ++ctx->epoch; // the graphs captured with the old number of planes are refused (launch shapes and calls change)
        ctx->hs_set_built = ctx->hs_lag_ready = false;
        // the plane energies and the hs_* words start from zero, and no rank-local share of the old planes is left for the fetch to sum
        IterState* ist = ctx->iter.p;
        CK(cudaMemsetAsync(&ist->energy[kEnergyPlaneBarrier], 0, sizeof(double), ctx->stream));
        CK(cudaMemsetAsync(&ist->energy[kEnergyPlaneFriction], 0, sizeof(double), ctx->stream));
        CK(cudaMemsetAsync(&ist->hs_alpha, 0, offsetof(IterState, pat_nnz) - offsetof(IterState, hs_alpha), ctx->stream));
        set_local(ctx, (1u << kEnergyPlaneBarrier) | (1u << kEnergyPlaneFriction) | kLocalCrossings, false);
    }
    ctx->n_hs = n;
    if (n > 0) {
        ALLOC(ctx->hs_par, (size_t)kPlaneStride * kMaxPlanes);
        CK(cudaMemcpyAsync(ctx->hs_par.p, par.data(), par.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream)); // `par` lives on this stack
    return IPCGPU_OK;
}

// allocations sized by the surface (lazy: the first call after ipcgpu_set_surface, which refuses older graphs, must run outside a capture)
static int halfspace_alloc(ipcgpu_ctx* ctx)
{
    const size_t n = (size_t)kMaxPlanes * std::max(ctx->nSV, 1);
    ALLOC(ctx->hs_flags, n);
    ALLOC(ctx->hs_offs, n);
    ALLOC(ctx->hs_act, n);
    ALLOC(ctx->hs_lag, n);
    ALLOC(ctx->hs_lam, n);
    ALLOC(ctx->hs_cnt, 2);
    ALLOC(ctx->hs_pstart, kMaxPlanes + 1);
    ALLOC(ctx->hs_partials, (size_t)halfspace_energy_blocks() + 8);
    // the scan's temporary storage grows with its length (decoupled look-back tile state): sized for the scan this surface and this number of
    // planes run, at every call (a host-only query), and the size handed to cub is that one
    ctx->hs_scan_bytes = halfspace_scan_bytes(ctx->n_hs * ctx->nSV);
    ALLOC(ctx->hs_scan, ctx->hs_scan_bytes);
    return IPCGPU_OK;
}

static int halfspace_sync_counts(ipcgpu_ctx* ctx)
{
    CK(cudaMemcpyAsync(ctx->h_scalar + 44, ctx->hs_cnt.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_halfspace_constraint_set(ipcgpu_ctx* ctx, double dHat, int* n_active)
{
    if (n_active) *n_active = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE(ctx->surface_ready && ctx->nSV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_surface with surface vertices first");
    ENTER(kSerial);
    int rc = halfspace_alloc(ctx);
    if (rc) return rc;
    const HalfSpaceArgs p = halfspace_args(ctx);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_CONSTRAINT_SET);
    CK(halfspace_active_set(p, dHat, ctx->hs_flags.p, ctx->hs_offs.p, ctx->hs_scan.p, ctx->hs_scan_bytes, ctx->hs_act.p, ctx->hs_cnt.p, ctx->hs_pstart.p,
        ctx->iter.p, ctx->stream));
    ctx->prof_end(pe);
    ctx->launches += 3;
    ctx->hs_set_built = true;
    ctx->mark_inputs();
    if (n_active) {
        if ((rc = halfspace_sync_counts(ctx))) return rc;
        *n_active = reinterpret_cast<int*>(ctx->h_scalar + 44)[0];
    }
    return IPCGPU_OK;
}

#define REQUIRE_HS_SET() REQUIRE(ctx->hs_set_built, IPCGPU_ERR_STATE, "ipcgpu_halfspace_constraint_set first")

int ipcgpu_halfspace_energy(ipcgpu_ctx* ctx, double dHat, double kappa, double* E)
{
    if (E) *E = 0.0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    ENTER(kSerial);
    const HalfSpaceArgs p = halfspace_args(ctx);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    halfspace_energy(p, dHat, ctx->hs_partials.p, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE], ctx->stream);
    return energy_tail(ctx, kEnergyPlaneBarrier, ctx->hs_partials.p, halfspace_energy_blocks(), kappa, pe, E, true, 1u << FLAG_NONPOSITIVE_DISTANCE);
}

int ipcgpu_halfspace_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { halfspace_gradient(p, dHat, kappa, ctx->g.p, st); });
}

int ipcgpu_halfspace_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { halfspace_hessian(p, dHat, kappa, projectDBC, ctx->a.p, st); });
}

int ipcgpu_halfspace_step(ipcgpu_ctx* ctx, const double* p_dir, double slackness, double* alpha_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(p_dir || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p_dir);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    halfspace_step(halfspace_args(ctx), ctx->dir.p, slackness, ctx->iter.p, ctx->stream);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (!alpha_inout) return IPCGPU_OK;
    if ((rc = ccd_read_back(ctx, alpha_inout))) return rc;
    if (ctx->h_iter->hs_zero_step) {
        CK(cudaMemsetAsync(&ctx->iter.p->hs_zero_step, 0, sizeof(int), ctx->stream));
        ctx->err = "step 0: a vertex is at or behind a half-space and moves further into it (Optimizer.cpp:2031-2033 would exit(-1))";
        return IPCGPU_ERR_LINE_SEARCH;
    }
    return IPCGPU_OK;
}

int ipcgpu_halfspace_crossings(ipcgpu_ctx* ctx, int* n)
{
    if (n) *n = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    ENTER(kSerial);
    halfspace_crossings(halfspace_args(ctx), ctx->iter.p, ctx->stream);
    ctx->launches += 2;
    CK(cudaGetLastError());
    set_local(ctx, kLocalCrossings, ctx->nranks > 1 && !n);
    if (!n) return IPCGPU_OK;
    if (ctx->nranks > 1) {
        int r = g_nccl.AllReduce(&ctx->iter.p->hs_crossings, &ctx->iter.p->hs_crossings, 1, kNcclInt32, kNcclSum, ctx->nccl_comm, ctx->stream);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(half-space crossings) failed");
    }
    int rc = fetch_iter_state(ctx);
    if (rc) return rc;
    *n = ctx->h_iter->hs_crossings;
    return IPCGPU_OK;
}

int ipcgpu_halfspace_friction_lag(ipcgpu_ctx* ctx, double dHat, double kappa, int* n_lagged)
{
    if (n_lagged) *n_lagged = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    ENTER(kSerial);
    halfspace_lag(halfspace_args(ctx), dHat, kappa, ctx->hs_pstart.p, ctx->hs_lag.p, ctx->hs_lam.p, ctx->hs_cnt.p + 1, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE],
        ctx->iter.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->hs_lag_ready = true;
    if (n_lagged) {
        int rc = halfspace_sync_counts(ctx);
        if (rc) return rc;
        *n_lagged = reinterpret_cast<int*>(ctx->h_scalar + 44)[1];
    }
    return IPCGPU_OK;
}

#define REQUIRE_HS_LAG()                                                                                            \
    REQUIRE(ctx->hs_lag_ready, IPCGPU_ERR_STATE, "ipcgpu_halfspace_friction_lag first");                          \
    REQUIRE(ctx->prev_set, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first");                                       \
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive")

int ipcgpu_halfspace_friction_energy(ipcgpu_ctx* ctx, double eps2, double* E)
{
    if (E) *E = 0.0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    halfspace_friction_energy(halfspace_args(ctx), eps2, ctx->hs_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyPlaneFriction, ctx->hs_partials.p, halfspace_energy_blocks(), 1.0, pe, E, true);
}

int ipcgpu_halfspace_friction_gradient(ipcgpu_ctx* ctx, double eps2, double* g_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { halfspace_friction_gradient(p, eps2, ctx->g.p, st); });
}

int ipcgpu_halfspace_friction_hessian(ipcgpu_ctx* ctx, double eps2, int projectDBC, double* a_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { halfspace_friction_hessian(p, eps2, projectDBC, ctx->a.p, st); });
}

int ipcgpu_get_halfspace_sets(ipcgpu_ctx* ctx, int* n_active, int* active2, int* n_lagged, int* lagged2, double* lambda)
{
    if (n_active) *n_active = 0;
    if (n_lagged) *n_lagged = 0;
    if (ctx->n_hs == 0 || !ctx->hs_set_built) return IPCGPU_OK;
    ENTER(kSerial);
    int rc = halfspace_sync_counts(ctx);
    if (rc) return rc;
    const int* h = reinterpret_cast<int*>(ctx->h_scalar + 44);
    const size_t na = (size_t)h[0], nl = ctx->hs_lag_ready ? (size_t)h[1] : 0;
    if (n_active) *n_active = (int)na;
    if (n_lagged) *n_lagged = (int)nl;
    if (na && active2) CK(cudaMemcpyAsync(active2, ctx->hs_act.p, na * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    if (nl && lagged2) CK(cudaMemcpyAsync(lagged2, ctx->hs_lag.p, nl * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    if (nl && lambda) CK(cudaMemcpyAsync(lambda, ctx->hs_lam.p, nl * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

// ---- CUDA graphs of device-resident call sequences ----------------------------------------------------------------------------
// An iteration in the NULL-output form is ~65 launches whose arguments do not change while the scene, the pattern, dHat / kappa and
// the tolerances stay the same: positions, search direction, list sizes and step bounds all live in device memory.  Enqueued one by
// one the front of the iteration (grid builds: ~25 short kernels) is bound by the host's launch rate; captured once and
// replayed, the whole sequence is one cudaGraphLaunch.
static ipcgpu_ctx::HostState snapshot_host_state(const ipcgpu_ctx* ctx)
{
    ipcgpu_ctx::HostState h;
    h.local_scalars = ctx->local_scalars;
    h.lists_local = ctx->lists_local;
    h.lists_global = ctx->cw.lists_global;
    h.want_cand = ctx->cw.want_cand;
    h.swept_ready = ctx->ccd.swept_ready;
    h.fr_ready = ctx->cw.fr_ready;
    h.inputs_marked = false; // events recorded inside a capture cannot be waited on outside of it
    h.scatter_marked = false;
    h.nC = ctx->cw.nC; h.nP = ctx->cw.nP; h.nK = ctx->cw.nK; h.fr_host_n = ctx->cw.fr_host_n;
    h.hs_set_built = ctx->hs_set_built;
    h.hs_lag_ready = ctx->hs_lag_ready;
    return h;
}
static void apply_host_state(ipcgpu_ctx* ctx, const ipcgpu_ctx::HostState& h)
{
    ctx->local_scalars = h.local_scalars;
    ctx->lists_local = h.lists_local;
    ctx->cw.lists_global = h.lists_global;
    ctx->cw.want_cand = h.want_cand;
    ctx->ccd.swept_ready = h.swept_ready;
    ctx->cw.fr_ready = h.fr_ready;
    ctx->inputs_marked = h.inputs_marked;
    ctx->scatter_marked = h.scatter_marked;
    ctx->cw.nC = h.nC; ctx->cw.nP = h.nP; ctx->cw.nK = h.nK; ctx->cw.fr_host_n = h.fr_host_n;
    ctx->hs_set_built = h.hs_set_built;
    ctx->hs_lag_ready = h.hs_lag_ready;
}

int ipcgpu_capture_begin(ipcgpu_ctx* ctx)
{
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is already in progress");
    REQUIRE(!ctx->profiling, IPCGPU_ERR_STATE, "switch the stage timers off (ipcgpu_profile(ctx, 0)) before capturing");
    ENTER(kSerial);
    ctx->inputs_marked = false;  // the side-stream fork of the pair Hessians must hang on an event recorded INSIDE the capture
    ctx->scatter_marked = false;
    ctx->deriv_copied = false;
    ctx->launches_at_capture = ctx->launches;
    ctx->dirty_at_capture = ctx->a_all_dirty;
    ctx->pat_pending_at_capture = ctx->pat_pending;
    ctx->pat_pending = false;
    ctx->sc_pending_at_capture = ctx->sc_pending;
    ctx->sc_pending = false;
    ctx->capture_bodies.clear();
    CK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    ctx->capturing = true;
    return IPCGPU_OK;
}

int ipcgpu_capture_end(ipcgpu_ctx* ctx, int* graph_id)
{
    REQUIRE(ctx->capturing, IPCGPU_ERR_STATE, "no capture in progress");
    REQUIRE(graph_id != nullptr, IPCGPU_ERR_ARG, "null graph id");
    ENTER(kSerial); // forked branches (derivative chain, copies) must rejoin the capturing stream
    {
        int rcj = join_copy_stream(ctx);
        if (rcj) return rcj;
    }
    ctx->capturing = false;
    ipcgpu_ctx::GraphRec rec;
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &rec.graph);
    if (e != cudaSuccess || rec.graph == nullptr) {
        cudaGetLastError();
        ctx->err = std::string("stream capture failed (a call inside the capture synchronised or copied to the host? use NULL outputs): ") + cudaGetErrorString(e);
        return IPCGPU_ERR_CUDA;
    }
    if (ctx->deriv_copied) {
        // the sequence hands the derivative chain's results to the host: that chain and the copy behind it (longer than the step-bound
        // chain) are now the critical path, so in this graph the two chains trade priorities
        e = for_each_kernel_node(rec.graph, ctx->capture_bodies, [&](cudaGraphNode_t node, cudaKernelNodeAttrValue v) {
            v.priority = (v.priority == ctx->prio_high) ? ctx->prio_low : ctx->prio_high;
            return cudaGraphKernelNodeSetAttribute(node, cudaKernelNodeAttributePriority, &v);
        });
        if (e != cudaSuccess) {
            cudaGraphDestroy(rec.graph);
            ctx->err = std::string("kernel node priorities: ") + cudaGetErrorString(e);
            return IPCGPU_ERR_CUDA;
        }
    }
    // kernel nodes carry the priority of the stream they were captured from; without this flag a replay would run every node at the
    // priority of the stream it is launched into
    e = cudaGraphInstantiateWithFlags(&rec.exec, rec.graph, cudaGraphInstantiateFlagUseNodePriority);
    if (e != cudaSuccess) {
        cudaGraphDestroy(rec.graph);
        ctx->err = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e);
        return IPCGPU_ERR_CUDA;
    }
    rec.launches = ctx->launches - ctx->launches_at_capture;
    rec.epoch = ctx->epoch;
    rec.dirty_at_begin = ctx->dirty_at_capture;
    rec.updates_pattern = ctx->pat_pending;
    ctx->pat_pending = ctx->pat_pending_at_capture; // nothing ran yet
    rec.step_control = ctx->sc_pending;
    ctx->sc_pending = ctx->sc_pending_at_capture;
    rec.bodies.swap(ctx->capture_bodies);
    rec.hs = snapshot_host_state(ctx);
    ctx->launches = ctx->launches_at_capture; // nothing ran yet
    ctx->inputs_marked = false;
    ctx->scatter_marked = false;
    ctx->graphs.push_back(rec);
    *graph_id = (int)ctx->graphs.size() - 1;
    return IPCGPU_OK;
}

int ipcgpu_graph_launch(ipcgpu_ctx* ctx, int graph_id)
{
    REQUIRE(graph_id >= 0 && graph_id < (int)ctx->graphs.size() && ctx->graphs[graph_id].exec, IPCGPU_ERR_ARG, "unknown graph id");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    const ipcgpu_ctx::GraphRec& rec = ctx->graphs[graph_id];
    REQUIRE(rec.epoch == ctx->epoch, IPCGPU_ERR_STATE, "the scene, pattern, partition or capacities changed since this graph was captured: capture it again");
    ENTER(kSerial);
    if (ctx->a_all_dirty && !rec.dirty_at_begin) // a cross-rank completion filled rows the captured clear does not cover
        CK(cudaMemsetAsync(ctx->a.p, 0, (size_t)(ctx->device_pattern ? ctx->pw.nnz_cap : ctx->nnz) * sizeof(double), ctx->stream));
    CK(cudaGraphLaunch(rec.exec, ctx->stream));
    if (rec.updates_pattern) ctx->pat_pending = true;
    if (rec.step_control) ctx->sc_pending = true;
    ctx->a_all_dirty = false;
    apply_host_state(ctx, rec.hs);
    ctx->launches += rec.launches;
    return IPCGPU_OK;
}

int ipcgpu_graph_destroy(ipcgpu_ctx* ctx, int graph_id)
{
    REQUIRE(graph_id >= 0 && graph_id < (int)ctx->graphs.size(), IPCGPU_ERR_ARG, "unknown graph id");
    ENTER(kSerial);
    ipcgpu_ctx::GraphRec& rec = ctx->graphs[graph_id];
    if (rec.exec) cudaGraphExecDestroy(rec.exec);
    if (rec.graph) cudaGraphDestroy(rec.graph);
    rec.exec = nullptr;
    rec.graph = nullptr;
    return IPCGPU_OK;
}

int ipcgpu_graph_kernel_priorities(ipcgpu_ctx* ctx, int graph_id, int* n_high, int* n_low)
{
    REQUIRE(graph_id >= 0 && graph_id < (int)ctx->graphs.size() && ctx->graphs[graph_id].graph, IPCGPU_ERR_ARG, "unknown graph id");
    REQUIRE(n_high && n_low, IPCGPU_ERR_ARG, "null argument");
    CK(cudaSetDevice(ctx->device));
    *n_high = *n_low = 0;
    CK(for_each_kernel_node(ctx->graphs[graph_id].graph, ctx->graphs[graph_id].bodies, [&](cudaGraphNode_t, cudaKernelNodeAttrValue v) {
        if (v.priority == ctx->prio_high) ++*n_high;
        else if (v.priority == ctx->prio_low) ++*n_low;
        return cudaSuccess;
    }));
    return IPCGPU_OK;
}

// ---- line-search safeguards (SURVEY 8(f) rank 2) -----------------------------------------------------------------------
static int reduce_checks(ipcgpu_ctx* ctx)
{
    if (ctx->nranks > 1 && (ctx->local_scalars & kLocalChecks)) {
        int r = g_nccl.AllReduce(ctx->iter.p->checks, ctx->iter.p->checks, 2, kNcclInt32, kNcclSum, ctx->nccl_comm, ctx->stream);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(safeguard counts) failed");
    }
    set_local(ctx, kLocalChecks, false);
    return IPCGPU_OK;
}

int ipcgpu_check_inversion(ipcgpu_ctx* ctx, int* n_inverted)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    int rc = safeguard_inversion(ctx);
    REQUIRE(rc == 0, rc, "inversion check launch failed");
    set_local(ctx, kLocalChecks, true);
    if (n_inverted) {
        CK(cudaMemsetAsync(&ctx->iter.p->checks[1], 0, sizeof(int), ctx->stream)); // (the partner count is not pending: keep the sum clean)
        if ((rc = reduce_checks(ctx))) return rc;
        if ((rc = fetch_iter_state(ctx))) return rc;
        *n_inverted = ctx->h_iter->checks[0];
    }
    return IPCGPU_OK;
}

int ipcgpu_intersection_free(ipcgpu_ctx* ctx, int* ok)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_HASH);
    int rc = safeguard_intersections(ctx);
    ctx->prof_end(pe);
    REQUIRE(rc == 0, rc, "intersection check launch failed");
    set_local(ctx, kLocalChecks, true);
    if (ok) {
        CK(cudaMemsetAsync(&ctx->iter.p->checks[0], 0, sizeof(int), ctx->stream));
        if ((rc = reduce_checks(ctx))) return rc;
        if ((rc = fetch_iter_state(ctx))) return rc;
        *ok = ctx->h_iter->checks[1] == 0 ? 1 : 0;
    }
    return IPCGPU_OK;
}

// ---- step control: CFL branch and line search (step_control.cu holds the decision kernel) ----------------------------------------
// Each loop body and loop condition is written once: a sequence of the entry points above plus one step_decide.  Outside a capture the
// host loops and reads the decision word (one synchronisation per decision); inside one the body is captured into a conditional node.
static int decide(ipcgpu_ctx* ctx, int op, double a, int b, cudaGraphConditionalHandle h, bool* word)
{
    step_decide(ctx->iter.p, op, a, b, (unsigned long long)h, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    if (word) {
        int* hw = reinterpret_cast<int*>(ctx->h_scalar + 40); // pinned staging slot of its own
        CK(cudaMemcpyAsync(hw, &ctx->iter.p->ls_cond, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *word = *hw != 0;
    }
    return IPCGPU_OK;
}

} // extern "C"

// if (decision) body  /  while (decision) body, where the decision is step_decide(op) before the node and, for a loop, at the end of each pass.
// Captured: the handle is created on the graph being captured, the decision before the node sets it, the node is added behind the
// capture's current dependencies, and the body is captured into the node's body graph on a stream of its own (ctx->stream points to it
// meanwhile, so that the entry points the body calls enqueue there).
template <typename Body>
static int cond_node(ipcgpu_ctx* ctx, bool loop, int op, double a, int b, Body body)
{
    int rc;
    if (!ctx->capturing) {
        bool go = false;
        if ((rc = decide(ctx, op, a, b, 0, &go))) return rc;
        while (go) {
            if ((rc = body())) return rc;
            if (!loop) break;
            if ((rc = decide(ctx, op, a, b, 0, &go))) return rc;
        }
        return IPCGPU_OK;
    }
    REQUIRE(ctx->cond_depth < ipcgpu_ctx::kCondDepth, IPCGPU_ERR_STATE, "conditional nodes nested too deeply");
    cudaStreamCaptureStatus cs;
    cudaGraph_t g = nullptr;
    const cudaGraphNode_t* deps = nullptr;
    size_t nd = 0;
    CK(cudaStreamGetCaptureInfo(ctx->stream, &cs, nullptr, &g, &deps, &nd));
    cudaGraphConditionalHandle h = 0;
    const cudaError_t eh = cudaGraphConditionalHandleCreate(&h, g, 0, 0);
    if (eh != cudaSuccess) {
        cudaGetLastError();
        ctx->err = std::string("conditional graph nodes need CUDA 12.4 or newer in the driver: ") + cudaGetErrorString(eh);
        return IPCGPU_ERR_CUDA;
    }
    if ((rc = decide(ctx, op, a, b, h, nullptr))) return rc;
    CK(cudaStreamGetCaptureInfo(ctx->stream, &cs, nullptr, &g, &deps, &nd));
    cudaGraphNodeParams np = {};
    np.type = cudaGraphNodeTypeConditional;
    np.conditional.handle = h;
    np.conditional.type = loop ? cudaGraphCondTypeWhile : cudaGraphCondTypeIf;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    CK(cudaGraphAddNode(&node, g, deps, nd, &np));
    cudaGraph_t bg = np.conditional.phGraph_out[0];
    ctx->capture_bodies.push_back(bg);
    cudaStream_t outer = ctx->stream, inner = ctx->cond_streams[ctx->cond_depth];
    CK(cudaStreamBeginCaptureToGraph(inner, bg, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    ctx->stream = inner;
    ++ctx->cond_depth;
    ctx->inputs_marked = false;
    rc = body();
    if (!rc && loop) rc = decide(ctx, op, a, b, h, nullptr);
    --ctx->cond_depth;
    ctx->stream = outer;
    cudaGraph_t captured = nullptr;
    const cudaError_t ee = cudaStreamEndCapture(inner, &captured);
    if (rc) return rc;
    CK(ee);
    CK(cudaStreamUpdateCaptureDependencies(outer, &node, 1, cudaStreamSetCaptureDependencies));
    ctx->mark_inputs(); // an event recorded inside the body cannot be waited on out here: the positions / sets changed at this node
    return IPCGPU_OK;
}

extern "C" {

static int step_control_prepare(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->surface_ready && ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh and ipcgpu_set_surface first");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the CFL branch and the line search run on one rank");
    REQUIRE(ctx->dir_valid && ctx->pSize_surface, IPCGPU_ERR_STATE, "no search direction for this surface: ipcgpu_set_search_dir first");
    if (!ctx->cond_streams[0]) {
        REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "run the CFL branch / line search once outside a capture first (it creates its streams)");
        for (cudaStream_t& s : ctx->cond_streams) CK(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, ctx->prio_high));
    }
    return IPCGPU_OK;
}

static int step_control_status(ipcgpu_ctx* ctx, int status)
{
    if (status == IPCGPU_ERR_LINE_SEARCH)
        ctx->err = "step 0: the line search's entry state fails a safeguard (inversion / intersection), or the step bound or the entry step is 0";
    else if (status == IPCGPU_ERR_NONPOSITIVE_DISTANCE)
        ctx->err = "a line-search trial has a constraint with d <= 0 (the reference exits here, Optimizer.cpp:3296-3306)";
    return status;
}

// host-output form: read the state back, hand out the step and the status
static int step_control_host_result(ipcgpu_ctx* ctx, double* alpha_inout)
{
    int rc = fetch_iter_state(ctx);
    if (rc) return rc;
    ctx->sc_pending = false;
    std::memcpy(alpha_inout, &ctx->h_iter->step_ord, sizeof(double));
    return step_control_status(ctx, ctx->h_iter->sc_status);
}

int ipcgpu_ccd_cfl_ti(ipcgpu_ctx* ctx, double dHat, int first_iteration, double voxel_size, double tol, const double err_vf[3], const double err_ee[3], double* alpha_inout)
{
    REQUIRE(err_vf && err_ee, IPCGPU_ERR_ARG, "null argument");
    REQUIRE(dHat > 0.0 && voxel_size > 0.0, IPCGPU_ERR_ARG, "dHat and the voxel size must be positive");
    ENTER(alpha_inout ? kSerial : kStepBound);
    int rc = step_control_prepare(ctx);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    cfl_pmax(ctx->nSV, ctx->SVI.p, ctx->nVdof, ctx->dir.p, ctx->iter.p, ctx->stream);
    ctx->launches += 2;
    CK(cudaGetLastError());
    rc = cond_node(ctx, false, kCflBranch, dHat, first_iteration ? 1 : 0, [&]() {
        int r = ccd_build_swept(ctx, voxel_size);
        if (!r) r = ccd_full(ctx, tol, err_vf, err_ee);
        if (!r) r = decide(ctx, kCflClamp, 0.0, 0, 0, nullptr);
        return r;
    });
    if (rc) return rc;
    ctx->sc_pending = true;
    return alpha_inout ? step_control_host_result(ctx, alpha_inout) : IPCGPU_OK;
}

// the energy terms of a line search: with planes set, their barrier energy, and their friction when fricDHat > 0 and a lagged plane set exists
// (Optimizer.cpp:3355-3365)
static int ls_terms(const ipcgpu_ctx* ctx, const ipcgpu_line_search_terms& t)
{
    int terms = (t.inertia ? kTermInertia : 0) | (t.fric_coef > 0.0 ? kTermFriction : 0);
    if (ctx->n_hs > 0) terms |= kTermHalfSpace;
    if (ctx->n_hs > 0 && ctx->hs_lag_ready && t.fric_eps2 > 0.0) terms |= kTermHalfSpaceFriction;
    // damping, Neumann forces and the Dirichlet penalty whenever they are set (ipcgpu_damping_update, _set_neumann_forces, _set_dirichlet_targets)
    if (ctx->damp_on) terms |= kTermDamping;
    if (ctx->nbc_on) terms |= kTermNeumann;
    if (ctx->n_dbc > 0) terms |= kTermDirichlet;
    return terms;
}
// one trial's energy: E_el, E_in, E_b, E_f (and the planes', damping, Neumann and Dirichlet-penalty terms) into IterState (summed by the decision
// that reads them)
static int ls_energy(ipcgpu_ctx* ctx, const ipcgpu_line_search_terms& t)
{
    const int terms = ls_terms(ctx, t);
    int rc = ipcgpu_elastic_energy(ctx, t.elastic_coef, 1, nullptr);
    if (!rc && t.inertia) rc = ipcgpu_inertia_energy(ctx, nullptr);
    if (!rc) rc = ipcgpu_barrier_energy(ctx, t.dHat, t.kappa, nullptr);
    if (!rc && (terms & kTermHalfSpace)) rc = ipcgpu_halfspace_energy(ctx, t.dHat, t.kappa, nullptr);
    if (!rc && (terms & kTermHalfSpaceFriction)) rc = ipcgpu_halfspace_friction_energy(ctx, t.fric_eps2, nullptr);
    if (!rc && t.fric_coef > 0.0) rc = ipcgpu_friction_energy(ctx, t.fric_eps2, t.fric_coef, nullptr);
    if (!rc && (terms & kTermDamping)) rc = ipcgpu_damping_energy(ctx, nullptr);
    if (!rc && (terms & kTermNeumann)) rc = ipcgpu_neumann_energy(ctx, nullptr);
    if (!rc && (terms & kTermDirichlet)) rc = ipcgpu_dirichlet_energy(ctx, nullptr);
    return rc;
}
// a trial's constraint sets: the self-contact set and the planes' (isIntersected and computeConstraintSet cover every collision object)
static int ls_constraint_set(ipcgpu_ctx* ctx, double dHat)
{
    int rc = ipcgpu_constraint_set(ctx, dHat, 1, nullptr, nullptr, nullptr);
    return rc ? rc : ipcgpu_halfspace_constraint_set(ctx, dHat, nullptr);
}
static int ls_intersection(ipcgpu_ctx* ctx)
{
    int rc = ipcgpu_intersection_free(ctx, nullptr);
    return rc ? rc : ipcgpu_halfspace_crossings(ctx, nullptr);
}
// V = V0 + alpha p with the device-resident step
static int ls_step(ipcgpu_ctx* ctx)
{
    step_forward(ctx->nV, ctx->Vsaved.p, ctx->dir.p, 0.0, ctx->V.p, ctx->stream, &ctx->iter.p->step_ord);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->mark_inputs();
    return IPCGPU_OK;
}

static int line_search_body(ipcgpu_ctx* ctx, const ipcgpu_line_search_terms& t)
{
    const int terms = ls_terms(ctx, t);
    CK(cudaMemcpyAsync(ctx->Vsaved.p, ctx->V.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream)); // :2692
    ctx->state_saved = true;
    int rc = ls_energy(ctx, t); // :2681
    if (!rc) rc = decide(ctx, kLsStart, 0.0, terms, 0, nullptr);
    if (!rc) rc = ls_step(ctx); // :2709
    if (!rc && ctx->energy == IPCGPU_NEOHOOKEAN) { // getNeedElemInvSafeGuard() (:2710)
        rc = ipcgpu_check_inversion(ctx, nullptr);
        if (!rc) rc = cond_node(ctx, true, kLsInversion, 0.0, 0, [&]() {
            int r = ls_step(ctx);
            return r ? r : ipcgpu_check_inversion(ctx, nullptr);
        });
    }
    if (!rc) rc = ls_intersection(ctx); // :2720
    if (!rc) rc = cond_node(ctx, true, kLsIntersection, 0.0, terms, [&]() {
        int r = ls_step(ctx);
        return r ? r : ls_intersection(ctx);
    });
    if (!rc) rc = ls_constraint_set(ctx, t.dHat); // :2741
    if (!rc) rc = ls_energy(ctx, t);              // :2744
    if (!rc) rc = cond_node(ctx, true, kLsArmijo, 0.0, terms, [&]() {
        int r = ls_step(ctx);
        if (!r) r = ls_constraint_set(ctx, t.dHat);
        return r ? r : ls_energy(ctx, t);
    });
    if (!rc) rc = cond_node(ctx, false, kLsPostCheck, 0.0, 0, [&]() {
        int r = ls_intersection(ctx);
        if (!r) r = cond_node(ctx, true, kLsPostLoop, 0.0, terms, [&]() {
            int q = ls_step(ctx);
            return q ? q : ls_intersection(ctx);
        });
        if (!r) r = cond_node(ctx, false, kLsRebuild, 0.0, 0, [&]() { return ls_constraint_set(ctx, t.dHat); });
        return r;
    });
    return rc;
}

int ipcgpu_line_search(ipcgpu_ctx* ctx, const ipcgpu_line_search_terms* t, double* alpha_inout)
{
    REQUIRE(t != nullptr, IPCGPU_ERR_ARG, "null terms");
    REQUIRE(t->dHat > 0.0 && t->kappa >= 0.0, IPCGPU_ERR_ARG, "dHat must be positive");
    REQUIRE(!t->inertia || (ctx->xtilde_set && ctx->has_mass), IPCGPU_ERR_STATE, "inertia: ipcgpu_set_xtilde and a mass diagonal first");
    REQUIRE(!(t->fric_coef > 0.0) || (ctx->cw.fr_ready && ctx->prev_set && t->fric_eps2 > 0.0), IPCGPU_ERR_STATE,
        "friction: ipcgpu_friction_lag, ipcgpu_set_prev_state and fric_eps2 > 0 first");
    REQUIRE(ctx->n_hs == 0 || ctx->hs_set_built, IPCGPU_ERR_STATE, "half-spaces: ipcgpu_halfspace_constraint_set first (E0 takes the sets held on entry)");
    REQUIRE(!(ls_terms(ctx, *t) & kTermHalfSpaceFriction) || ctx->prev_set, IPCGPU_ERR_STATE, "half-space friction: ipcgpu_set_prev_state first");
    REQUIRE(!ctx->damp_on || ctx->prev_set, IPCGPU_ERR_STATE, "damping: ipcgpu_set_prev_state first");
    REQUIRE(!(ctx->capturing && ctx->canonical_order), IPCGPU_ERR_STATE, "inside a capture the line search needs ipcgpu_set_canonical_order(ctx, 0)");
    ENTER(kSerial);
    int rc = step_control_prepare(ctx);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    if ((rc = cond_node(ctx, false, kLsEntry, 0.0, 0, [&]() { return line_search_body(ctx, *t); }))) return rc;
    ctx->sc_pending = true;
    return alpha_inout ? step_control_host_result(ctx, alpha_inout) : IPCGPU_OK;
}

int ipcgpu_step_control_info(ipcgpu_ctx* ctx, ipcgpu_step_control* out)
{
    REQUIRE(out != nullptr, IPCGPU_ERR_ARG, "null output");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    if (ctx->sc_pending) {
        ENTER(kSerial);
        int rc = fetch_iter_state(ctx);
        if (rc) return rc;
        ctx->sc_pending = false;
    }
    else CK(cudaSetDevice(ctx->device)); // (reads the host mirror: no need to join the derivative chain)
    const IterState& h = *ctx->h_iter;
    out->alpha_cfl = h.sc_alpha_cfl;
    out->alpha_feasible = h.ls_LF;
    std::memcpy(&out->alpha, &h.step_ord, sizeof(double));
    out->energy_start = h.ls_E0;
    out->energy = h.ls_Et;
    out->full_ccd = h.sc_full_ccd;
    out->stopped = h.ls_stopped;
    out->halvings_inversion = h.ls_count[0];
    out->halvings_intersection = h.ls_count[1];
    out->halvings_armijo = h.ls_count[2];
    out->halvings_post_check = h.ls_count[3];
    out->post_check_rebuilt = h.ls_rebuilt;
    out->status = h.sc_status;
    return step_control_status(ctx, h.sc_status);
}

// ---- device-resident linear solve hand-off (SURVEY 8(f) rank 1) ----------------------------------------------------------
int ipcgpu_solve_pcg(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual)
{
    REQUIRE(ctx->nnz > 0 && ctx->n_rows == 3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the built-in solver runs on one rank (a distributed solver takes each rank's rows: ipcgpu_partition_info)");
    REQUIRE(rel_tol > 0.0 && max_iter > 0, IPCGPU_ERR_ARG, "bad tolerance / iteration limit");
    ENTER(kSerial);
    {
        int rcp = sync_pattern_mirror(ctx);
        if (rcp) return rcp;
    }
    if (!ctx->full_pattern_ready) { // once per sparsity pattern: rows of both triangles, gathered through a position map
        std::vector<int> ia((size_t)ctx->n_rows + 1), ja((size_t)ctx->nnz);
        CK(cudaMemcpyAsync(ia.data(), ctx->ia.p, ia.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(ja.data(), ctx->ja.p, ja.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        int rc = solver_build_full_pattern(ctx, ia.data(), ja.data());
        if (rc) return rc;
    }
    const double* rhs_dev = ctx->g.p;
    double sign = -1.0; // Newton: H p = -g (Optimizer.cpp:2350-2352)
    if (rhs) { // a host right-hand side is staged in a buffer of its own
        ALLOC(ctx->pcg_b, (size_t)ctx->n_rows);
        CK(cudaMemcpyAsync(ctx->pcg_b.p, rhs, (size_t)ctx->n_rows * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        rhs_dev = ctx->pcg_b.p;
        sign = 1.0;
    }
    int rc = solver_pcg(ctx, rhs_dev, sign, rel_tol, max_iter, iters, rel_residual);
    if (rc) return rc;
    if (adopt_as_search_dir && (rc = solver_adopt_direction(ctx))) return rc;
    if (x) {
        CK(cudaMemcpyAsync(x, ctx->sol.p, (size_t)ctx->n_rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return IPCGPU_OK;
}

int ipcgpu_csr_set_zero(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(kSerial);
    return zero_values(ctx);
}

int ipcgpu_allreduce_grad_hess(ipcgpu_ctx* ctx, int with_gradient, int with_hessian)
{
    if (ctx->nranks <= 1) return IPCGPU_OK;
    REQUIRE(ctx->nccl_comm != nullptr, IPCGPU_ERR_STATE, "ipcgpu_comm_init first");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
    if (with_gradient) { // elastic part: every rank holds the complete rows it owns (zeros elsewhere); barrier part: partial sums
        int r = g_nccl.AllReduce(ctx->g.p, ctx->g.p, (size_t)3 * ctx->nV, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(gradient) failed");
    }
    if (with_hessian) {
        // The rows a rank owns are already complete (row-owner assembly): this only matters to a caller that wants the WHOLE matrix on
        // every rank.  Non-owned rows are zero, so a sum completes it.
        // (device-built pattern: the whole capacity -- the count is fixed when the call is captured, the pattern may grow at replay)
        const size_t n = ctx->device_pattern ? (size_t)ctx->pw.nnz_cap : (size_t)ctx->nnz;
        int r = g_nccl.AllReduce(ctx->a.p, ctx->a.p, n, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream);
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(csr values) failed");
        ctx->a_all_dirty = true; // the next rebuild must clear every row, not only the owned ones
    }
    ctx->prof_end(pe);
    return IPCGPU_OK;
}

int ipcgpu_fetch_iteration(ipcgpu_ctx* ctx, ipcgpu_iteration* out)
{
    REQUIRE(out != nullptr, IPCGPU_ERR_ARG, "null output");
    ENTER(kSerial);
    if (ctx->nranks > 1) {
        // complete the deferred scalars across ranks in ONE collective: the shares still local (local_scalars) and the error flags (so
        // that every rank returns the same status)
        double* buf = ctx->packed_scalars.p;
        cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
        pack_scalars(ctx->iter.p, ctx->local_scalars, buf, ctx->stream);
        int r = g_nccl.AllReduce(buf, buf, kPackedScalars, kNcclFloat64, kNcclSum, ctx->nccl_comm, ctx->stream);
        unpack_scalars(ctx->iter.p, ctx->local_scalars, buf, ctx->stream);
        ctx->prof_end(pe);
        ctx->launches += 2;
        REQUIRE(r == 0, IPCGPU_ERR_NCCL, "ncclAllReduce(iteration scalars) failed");
    }
    ctx->local_scalars = 0;
    int rc = ccd_read_back(ctx, nullptr);
    if (rc || (rc = refresh_pattern_mirror(ctx))) return rc;
    const IterState& h = *ctx->h_iter;
    out->energy_elastic = h.energy[kEnergyElastic];
    out->energy_barrier = h.energy[kEnergyBarrier];
    out->energy_friction = h.energy[kEnergyFriction];
    out->energy_inertia = h.energy[kEnergyInertia];
    out->alpha_inversion = h.alpha_stage[0];
    out->alpha_partial_ccd = h.alpha_stage[1];
    out->alpha_swept_grid = h.alpha_stage[2];
    out->alpha_full_ccd = h.alpha_stage[3];
    std::memcpy(&out->alpha, &h.step_ord, sizeof(double));
    out->n_active = h.n_set[0];
    out->n_mollified = h.n_set[1];
    out->n_candidates = h.n_set[2];
    out->n_full_ccd_candidates = h.n_full_cand;
    out->ti_warnings = (uint64_t)h.flags[FLAG_TI_WARNINGS];
    out->n_inverted_tets = h.checks[0];
    out->n_intersected_triangles = h.checks[1];
    out->energy_halfspace = h.energy[kEnergyPlaneBarrier];
    out->energy_halfspace_friction = h.energy[kEnergyPlaneFriction];
    out->alpha_halfspace = h.hs_alpha;
    out->n_halfspace_active = h.hs_n_active;
    out->n_halfspace_crossings = h.hs_crossings;
    out->energy_damping = h.energy[kEnergyDamping];
    out->energy_neumann = h.energy[kEnergyNeumann];
    out->energy_dirichlet = h.energy[kEnergyDirichlet];
    out->dirichlet_completed_step = h.dbc_step;
    ContactWork& w = ctx->cw;
    w.nC = h.n_set[0]; w.nP = h.n_set[1]; w.nK = h.n_set[2];
    int status = status_from_flags(ctx, h.flags);
    if (status == IPCGPU_OK && h.hs_zero_step) {
        ctx->err = "step 0: a vertex is at or behind a half-space and moves further into it (Optimizer.cpp:2031-2033 would exit(-1))";
        status = IPCGPU_ERR_LINE_SEARCH;
    }
    out->status = status;
    CK(cudaMemsetAsync(ctx->iter.p->flags, 0, 8 * sizeof(int), ctx->stream)); // flags are per fetch
    if (h.hs_zero_step) CK(cudaMemsetAsync(&ctx->iter.p->hs_zero_step, 0, sizeof(int), ctx->stream));
    if (h.grid_axis_cells > 0) { // sort width of the next iteration's grid builds: enough bits for 1.5x the cells this one wanted
        int bits = 3;
        while (bits < 10 && (1 << bits) - 2 < (h.grid_axis_cells * 3) / 2 + 2) ++bits;
        w.axis_bits = bits;
        CK(cudaMemsetAsync(&ctx->iter.p->grid_axis_cells, 0, sizeof(int), ctx->stream));
    }
    return status;
}

int ipcgpu_profile(ipcgpu_ctx* ctx, int enable)
{
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "stage timers cannot be switched inside a capture");
    ENTER(kSerial);
    CK(cudaStreamSynchronize(ctx->stream));
    for (int s = 0; s < IPCGPU_STAGE_COUNT; ++s) {
        for (auto& pr : ctx->prof[s]) {
            cudaEventDestroy(pr.first);
            cudaEventDestroy(pr.second);
        }
        ctx->prof[s].clear();
    }
    ctx->profiling = enable != 0;
    return IPCGPU_OK;
}

int ipcgpu_profile_read(ipcgpu_ctx* ctx, int stage, double* total_ms, int* count)
{
    REQUIRE(stage >= 0 && stage < IPCGPU_STAGE_COUNT && total_ms && count, IPCGPU_ERR_ARG, "bad stage");
    ENTER(kSerial);
    CK(cudaStreamSynchronize(ctx->stream));
    double tot = 0.0;
    for (auto& pr : ctx->prof[stage]) {
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, pr.first, pr.second));
        tot += ms;
    }
    *total_ms = tot;
    *count = (int)ctx->prof[stage].size();
    return IPCGPU_OK;
}

int ipcgpu_timer_start(ipcgpu_ctx* ctx)
{
    ENTER(kSerial);
    if (!ctx->timer_a) {
        CK(cudaEventCreate(&ctx->timer_a));
        CK(cudaEventCreate(&ctx->timer_b));
    }
    CK(cudaEventRecord(ctx->timer_a, ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_timer_stop(ipcgpu_ctx* ctx, double* ms)
{
    REQUIRE(ctx->timer_a && ms, IPCGPU_ERR_STATE, "ipcgpu_timer_start first");
    ENTER(kSerial);
    CK(cudaEventRecord(ctx->timer_b, ctx->stream));
    CK(cudaEventSynchronize(ctx->timer_b));
    float f = 0.f;
    CK(cudaEventElapsedTime(&f, ctx->timer_a, ctx->timer_b));
    *ms = f;
    return IPCGPU_OK;
}

static int buf_info(ipcgpu_ctx* ctx, int which, double** p, uint64_t* n)
{
    const uint64_t nL = (uint64_t)ctx->n_list;
    switch (which) {
    case IPCGPU_BUF_GRADIENT: *p = ctx->g.p; *n = (uint64_t)3 * ctx->nV; return 0;
    case IPCGPU_BUF_CSR_VALUES: *p = ctx->a.p; *n = (uint64_t)ctx->nnz; return 0;
    case IPCGPU_BUF_ENERGY_PER_TET: *p = ctx->e_per_tet.p; *n = (uint64_t)ctx->nT; return 0;
    case IPCGPU_BUF_TET_HESSIANS: *p = ctx->hblk.p; *n = 78 * 64 * ((nL + 63) / 64); return ctx->hblk_valid ? 0 : 2; /* tile-major, see elastic.cu */
    case IPCGPU_BUF_TET_GRADIENTS: *p = ctx->gcont.p; *n = 12 * nL; return 0;
    case IPCGPU_BUF_INVERSION_STEPS: *p = ctx->inv_steps.p; *n = (uint64_t)ctx->nT; return 0;
    default: return 1;
    }
}

int ipcgpu_download(ipcgpu_ctx* ctx, int which, double* dst, uint64_t count) { return ipcgpu_download_range(ctx, which, 0, count, dst); }

int ipcgpu_download_range_async(ipcgpu_ctx* ctx, int which, uint64_t offset, uint64_t count, double* dst_pinned)
{
    double* p;
    uint64_t n;
    REQUIRE(buf_info(ctx, which, &p, &n) == 0, IPCGPU_ERR_ARG, "unknown buffer id");
    REQUIRE((dst_pinned || count == 0) && offset + count <= n, IPCGPU_ERR_ARG, "download: bad destination or range");
    REQUIRE(!(ctx->capturing && ctx->device_pattern && which == IPCGPU_BUF_CSR_VALUES), IPCGPU_ERR_STATE,
        "with the device-built pattern the CSR values cannot be copied from inside a graph: the range is fixed at capture, the pattern may change at replay");
    CK(cudaSetDevice(ctx->device));
    if (!ctx->copy) {
        REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "call ipcgpu_download_range_async once outside a capture first (it creates the copy stream)");
        CK(cudaStreamCreateWithFlags(&ctx->copy, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&ctx->ev_copy_fork, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&ctx->ev_copy_join, cudaEventDisableTiming));
    }
    if (count == 0) return IPCGPU_OK;
    // everything enqueued so far, on the main stream and on an open derivative stream, produces the buffer: the copy starts after it and
    // runs next to whatever follows on the main stream (this call does not join the derivative chain, see enter())
    CK(cudaEventRecord(ctx->ev_copy_fork, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->copy, ctx->ev_copy_fork, 0));
    if (ctx->deriv_open) {
        CK(cudaEventRecord(ctx->ev_deriv_done, ctx->deriv));
        CK(cudaStreamWaitEvent(ctx->copy, ctx->ev_deriv_done, 0));
        if (ctx->capturing) ctx->deriv_copied = true;
    }
    CK(cudaMemcpyAsync(dst_pinned, p + offset, count * sizeof(double), cudaMemcpyDeviceToHost, ctx->copy));
    ctx->copy_pending = true;
    return IPCGPU_OK;
}

int ipcgpu_download_range(ipcgpu_ctx* ctx, int which, uint64_t offset, uint64_t count, double* dst)
{
    double* p;
    uint64_t n;
    ENTER(kSerial);
    {
        int rcp = sync_pattern_mirror(ctx);
        if (rcp) return rcp;
    }
    {
        const int bi = buf_info(ctx, which, &p, &n);
        REQUIRE(bi != 2, IPCGPU_ERR_STATE, "no per-tet Hessian blocks: the last elastic gradient/Hessian call computed no Hessian");
        REQUIRE(bi == 0, IPCGPU_ERR_ARG, "unknown buffer id");
    }
    REQUIRE((dst || count == 0) && offset + count <= n, IPCGPU_ERR_ARG, "download: bad destination or range");
    if (count) CK(cudaMemcpyAsync(dst, p + offset, count * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

void* ipcgpu_device_ptr(ipcgpu_ctx* ctx, int which)
{
    if (which == IPCGPU_BUF_CSR_ROW_STARTS) return ctx->ia.p;
    if (which == IPCGPU_BUF_CSR_COLUMNS) return ctx->ja.p;
    double* p;
    uint64_t n;
    return buf_info(ctx, which, &p, &n) == 0 ? p : nullptr;
}

} // extern "C"
