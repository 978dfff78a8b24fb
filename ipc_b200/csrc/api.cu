// api.cu -- extern "C" entry points declared in include/ipcgpu.h: the context, its streams, the read-back of the iteration state and the
// tails the synchronous forms share.  The entry points of each stage are in api_mesh.cu, api_contact.cu, api_terms.cu, api_step.cu and
// api_comm.cu.
//
// Execution model.  Every stage enqueues its kernels (and, with several ranks, its NCCL reductions) on the context's stream and leaves
// its scalar results in the device-resident iteration state (kernels.h: IterState).  An entry point synchronises with the host only if
// the caller hands it a host output pointer; with NULL outputs a whole Newton iteration runs without a host synchronisation, read back
// once by ipcgpu_fetch_iteration, its derivative chain on a stream of its own next to the step-bound chain (see enter() in abi.h).  The
// synchronous forms are the same code followed by that read-back (energy_result, gradient_call / hessian_call, flag_status).
#include "abi.h"
#include <cstring>

using namespace ipcgpu;

// make the main stream wait for the copies ipcgpu_download_range_async forked off (a graph edge when capturing)
int join_copy_stream(ipcgpu_ctx* ctx)
{
    if (!ctx->copy_pending) return IPCGPU_OK;
    CK(cudaEventRecord(ctx->ev_copy_join, ctx->copy));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_copy_join, 0));
    ctx->copy_pending = false;
    return IPCGPU_OK;
}

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
    owned_value_range(ctx);
    return IPCGPU_OK;
}
// ... before a host-side use of them, when an update was enqueued since (synchronises)
int sync_pattern_mirror(ipcgpu_ctx* ctx)
{
    if (!ctx->device_pattern || !ctx->pat_pending) return IPCGPU_OK;
    int rc = fetch_iter_state(ctx);
    return rc ? rc : refresh_pattern_mirror(ctx);
}

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
    if (f[FLAG_SOLVE]) {
        ctx->err = "the deferred linear solve failed: a non-positive pivot of the multilevel preconditioner or a non-finite residual (the matrix is not positive definite)";
        return IPCGPU_ERR_SOLVE;
    }
    if (f[FLAG_PATTERN]) {
        ctx->err = "CSR pattern misses a contact block: call ipcgpu_set_csr with the augmented pattern (augmentConnectivity, SelfCollisionHandler.cpp:330-415)";
        return IPCGPU_ERR_PATTERN;
    }
    return IPCGPU_OK;
}

// ---- the tails the synchronous forms share --------------------------------------------------------------------------------
// the flags of `mask` that the (fresh) h_iter shows raised: cleared on the device, returned as a status
int flag_status(ipcgpu_ctx* ctx, unsigned mask)
{
    int f[kFlagSlots] = { 0 };
    for (int i = 0; i < kFlagSlots; ++i)
        if (((mask >> i) & 1u) && ctx->h_iter->flags[i]) {
            f[i] = ctx->h_iter->flags[i];
            CK(cudaMemsetAsync(&ctx->iter.p->flags[i], 0, sizeof(int), ctx->stream));
        }
    return status_from_flags(ctx, f);
}

void set_local(ipcgpu_ctx* ctx, unsigned bits, bool local)
{
    ctx->local_scalars = local ? (ctx->local_scalars | bits) : (ctx->local_scalars & ~bits);
}

// IterState::energy[slot] once reduced.  Host E: summed across the ranks in place and read back, either the one double or (`fetch`) the
// whole iteration state, after which the flags of `check` are the status.  NULL: this rank's share, completed by the fetch's collective.
int energy_result(ipcgpu_ctx* ctx, int slot, double* E, bool fetch, unsigned check)
{
    set_local(ctx, 1u << slot, ctx->nranks > 1 && !E);
    if (!E) return IPCGPU_OK;
    double* out = &ctx->iter.p->energy[slot];
    int rc = nccl_sum(ctx, out, 1, "ncclAllReduce(energy) failed");
    if (rc) return rc;
    if (fetch) {
        if ((rc = fetch_iter_state(ctx))) return rc;
        *E = ctx->h_iter->energy[slot];
        return flag_status(ctx, check);
    }
    CK(cudaMemcpyAsync(&ctx->staging->scalar, out, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *E = ctx->staging->scalar;
    return IPCGPU_OK;
}
// the tail of an energy term on the main stream: its partial sums reduced into the slot, the stage timer `pe` stopped, energy_result
int energy_tail(ipcgpu_ctx* ctx, int slot, const double* partials, int n_partials, double scale, cudaEvent_t pe, double* E, bool fetch,
    unsigned check, const double* scale_dev)
{
    reduce_sum(partials, n_partials, scale, &ctx->iter.p->energy[slot], ctx->stream, scale_dev);
    ctx->prof_end(pe);
    ctx->launches += 2; // the term's partial kernel and the reduce
    CK(cudaGetLastError());
    return energy_result(ctx, slot, E, fetch, check);
}

// host gradient in/out around a kernel that accumulates into the device gradient (addCoeff-like semantics: rank 0 contributes the input)
int gradient_roundtrip_begin(ipcgpu_ctx* ctx, const double* g_in)
{
    if (ctx->rank == 0) CK(cudaMemcpyAsync(ctx->g.p, g_in, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    else CK(cudaMemsetAsync(ctx->g.p, 0, (size_t)3 * ctx->nV * sizeof(double), ctx->stream));
    return IPCGPU_OK;
}
int gradient_roundtrip_end(ipcgpu_ctx* ctx, double* g_out)
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

int hessian_begin(ipcgpu_ctx* ctx, Chain chain, const double* a_inout)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(a_inout ? kSerial : chain);
    return a_inout ? upload_values(ctx, a_inout) : IPCGPU_OK;
}
int hessian_end(ipcgpu_ctx* ctx, double* a_inout, unsigned check)
{
    if (!a_inout) return IPCGPU_OK;
    int rc = download_values(ctx, a_inout);
    if (rc || !check || (rc = fetch_iter_state(ctx))) return rc;
    return flag_status(ctx, check);
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
        || cudaMallocHost(&ctx->staging, sizeof(HostStaging)) != cudaSuccess
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
    nccl_comm_destroy(ctx);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->staging) cudaFreeHost(ctx->staging);
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

int ipcgpu_allreduce_grad_hess(ipcgpu_ctx* ctx, int with_gradient, int with_hessian)
{
    if (ctx->nranks <= 1) return IPCGPU_OK;
    REQUIRE(ctx->nccl_comm != nullptr, IPCGPU_ERR_STATE, "ipcgpu_comm_init first");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ALLREDUCE);
    int rc;
    // elastic part: every rank holds the complete rows it owns (zeros elsewhere); barrier part: partial sums
    if (with_gradient && (rc = nccl_sum(ctx, ctx->g.p, (size_t)3 * ctx->nV, "ncclAllReduce(gradient) failed"))) return rc;
    if (with_hessian) {
        // The rows a rank owns are already complete (row-owner assembly): this only matters to a caller that wants the WHOLE matrix on
        // every rank.  Non-owned rows are zero, so a sum completes it.
        // (device-built pattern: the whole capacity -- the count is fixed when the call is captured, the pattern may grow at replay)
        const size_t n = ctx->device_pattern ? (size_t)ctx->pw.nnz_cap : (size_t)ctx->nnz;
        if ((rc = nccl_sum(ctx, ctx->a.p, n, "ncclAllReduce(csr values) failed"))) return rc;
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
        const int r = nccl_sum(ctx, buf, kPackedScalars, "ncclAllReduce(iteration scalars) failed");
        unpack_scalars(ctx->iter.p, ctx->local_scalars, buf, ctx->stream);
        ctx->prof_end(pe);
        ctx->launches += 2;
        if (r) return r;
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
    CK(cudaMemsetAsync(ctx->iter.p->flags, 0, sizeof(ctx->iter.p->flags), ctx->stream)); // flags are per fetch
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
    case IPCGPU_BUF_POSITIONS: *p = ctx->V.p; *n = (uint64_t)3 * ctx->nV; return 0;
    case IPCGPU_BUF_SEARCH_DIR: *p = ctx->dir.p; *n = ctx->dir_valid ? (uint64_t)3 * ctx->nV : 0; return 0;
    case IPCGPU_BUF_XTILDE: *p = ctx->xtilde.p; *n = ctx->xtilde_set ? (uint64_t)3 * ctx->nV : 0; return 0;
    case IPCGPU_BUF_MULTILEVEL_INVERSES: *p = ctx->ml.inv.p; *n = ctx->ml.built ? (uint64_t)ctx->ml.tiles * 96 * 96 : 0; return 0;
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
