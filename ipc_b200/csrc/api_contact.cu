// api_contact.cu -- entry points of self-contact: surface and obstacle, capacities, the CCD step-bound stages with their statistics and
// test hooks, the constraint sets, barrier and lagged-friction terms, and the device-built sparsity pattern.
#include "abi.h"
#include <algorithm>
#include <cmath>
#include <vector>

using namespace ipcgpu;

extern "C" {

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
    int rc = safeguard_set_points(ctx, vCoDim);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->h_SVI.assign(SVI, SVI + nSV);
    ctx->hs_set_built = ctx->hs_lag_ready = false; // the plane sets index the old surface (and halfspace_alloc may reallocate them)
    ctx->pSize_surface = false; // pSize belongs to the surface
    if ((rc = contact_alloc(ctx))) return rc;
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
        const int r = nccl_all_gather(ctx, w.xsend.p, w.xrecv.p, w.xstride, "ncclAllGather(pair lists) failed");
        ctx->prof_end(pe);
        if (r) return r;
        contact_unpack_lists(ctx);
        w.lists_global = true;
        CK(cudaGetLastError());
    }
    ctx->mark_inputs();
    return rc;
}

int ipcgpu_set_canonical_order(ipcgpu_ctx* ctx, int level)
{
    REQUIRE(level >= 0 && level <= 2, IPCGPU_ERR_ARG, "ipcgpu_set_canonical_order: level 0, 1 or 2");
    REQUIRE(level != 2 || ctx->nranks == 1, IPCGPU_ERR_STATE, "the reproducible mode (level 2) runs on one rank");
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    ctx->canonical_order = level;
    // the lists held now keep the order they were built in: the fixed-order sums start with the next lists built at level 2
    ctx->rw.lists_ready = ctx->rw.fr_ready = false;
    if (level == 2 && ctx->surface_ready) return repro_alloc(ctx);
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
    int* h = ctx->staging->contact;
    for (int i = 0; i < 16; ++i) h[i] = 0;
    h[0] = nC; h[2] = nP; h[3] = nK;
    CK(cudaMemcpyAsync(w.counters.p, h, 16 * sizeof(int), cudaMemcpyHostToDevice, ctx->stream)); // the consumers read the sizes on the device
    CK(cudaStreamSynchronize(ctx->stream));
    w.nC = nC; w.nP = nP; w.nK = nK;
    w.want_cand = nK > 0;
    ctx->lists_local = false; // uploaded sets are the global ones
    w.lists_global = false;
    ctx->rw.lists_ready = false;
    if (repro_on(ctx)) {
        int rc = contact_sort_lists(ctx);
        if (!rc) rc = repro_contact_lists(ctx);
        if (rc) return rc;
    }
    ctx->mark_inputs();
    return IPCGPU_OK;
}

} // extern "C"

BarrierArgs barrier_args(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC)
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
    p.kappa_dev = kappa_ptr(ctx, kappa);
    p.rep = repro_barrier_args(ctx);
    return p;
}

extern "C" {

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
    ctx->g_assembled = ctx->a_assembled = false;
    owned_value_range(ctx);
    if ((rc = solver_forget_full_pattern(ctx))) return rc;
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
    ctx->g_assembled = ctx->a_assembled = false;
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
    REQUIRE_KAPPA(kappa);
    ENTER(kSerial);
    BarrierArgs p = barrier_args(ctx, dHat, kappa, 0);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    barrier_energy(p, ctx->cw.bpartials.p, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE], ctx->stream);
    // synchronous form: the d <= 0 flag is checked right here (every rank checks its own share of the pairs)
    return energy_tail(ctx, kEnergyBarrier, ctx->cw.bpartials.p, barrier_energy_blocks(), kappa, pe, E, true, 1u << FLAG_NONPOSITIVE_DISTANCE, p.kappa_dev);
}

int ipcgpu_barrier_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE_KAPPA(kappa);
    const BarrierArgs p = barrier_args(ctx, dHat, kappa, 0);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) {
        barrier_gradient(p, ctx->g.p, st);
        ctx->launches += p.rep.on; // (the reproducible mode's gather)
    });
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
    ctx->launches += 1 + p.rep.on;
    CK(cudaGetLastError());
    return gradient_roundtrip_end(ctx, g_inout);
}

int ipcgpu_para_ee_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE(g_inout != nullptr, IPCGPU_ERR_ARG, "null gradient");
    REQUIRE_KAPPA(kappa);
    ENTER(kSerial);
    int rc = gradient_roundtrip_begin(ctx, g_inout);
    if (rc) return rc;
    const BarrierArgs p = barrier_args(ctx, dHat, kappa, 0);
    para_gradient(p, ctx->g.p, ctx->stream);
    ctx->launches += 1 + p.rep.on;
    CK(cudaGetLastError());
    return gradient_roundtrip_end(ctx, g_inout);
}

int ipcgpu_barrier_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout)
{
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    REQUIRE_KAPPA(kappa);
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
    REQUIRE_KAPPA(kappa);
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
    ctx->rw.fr_ready = false;
    if (repro_on(ctx) && (rc = repro_friction_list(ctx, !ctx->rw.lists_ready))) return rc; // (a copy of the active list: sorted already at level 2)
    if (n_pairs) {
        CK(cudaMemcpyAsync(&ctx->staging->count, w.fr_n.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        w.fr_host_n = ctx->staging->count;
        *n_pairs = w.fr_host_n;
    }
    return IPCGPU_OK;
}

static int friction_host_count(ipcgpu_ctx* ctx)
{
    ContactWork& w = ctx->cw;
    if (w.fr_host_n < 0) {
        CK(cudaMemcpyAsync(&ctx->staging->count, w.fr_n.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        w.fr_host_n = ctx->staging->count;
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
    ctx->rw.fr_ready = false;
    if (repro_on(ctx)) return repro_friction_list(ctx, true);
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
    p.rep = repro_friction_args(ctx);
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
    return gradient_call(ctx, kSerial, g_inout, [&](cudaStream_t st) {
        friction_gradient(p, ctx->g.p, st);
        ctx->launches += p.rep.on;
    });
}

int ipcgpu_friction_hessian(ipcgpu_ctx* ctx, double eps2, double coef, int projectDBC, double* a_inout)
{
    REQUIRE_FRICTION();
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive");
    const FrictionArgs p = friction_args(ctx, eps2, coef, projectDBC);
    return hessian_call(ctx, kSerial, a_inout, 1u << FLAG_PATTERN,
        [&](cudaStream_t st) {
            friction_hessian(p, ctx->a.p, ctx->iter.p->flags + FLAG_PATTERN, st);
            ctx->launches += p.rep.on;
        });
}

} // extern "C"
