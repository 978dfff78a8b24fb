// api_step.cu -- entry points that drive a whole sequence: CUDA-graph capture and replay, the line-search safeguards, and the step control
// (CFL branch and line search) built from conditional graph nodes.
#include "abi.h"
#include <cstring>
#include <vector>

using namespace ipcgpu;

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
    if (ctx->local_scalars & kLocalChecks) {
        int rc = nccl_sum(ctx, ctx->iter.p->checks, 2, "ncclAllReduce(safeguard counts) failed");
        if (rc) return rc;
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

int ipcgpu_safeguard_debug_flags(ipcgpu_ctx* ctx, int enable, int* tri_flags, int* tet_hits)
{
    ENTER(kSerial);
    if (tri_flags || tet_hits) {
        REQUIRE(ctx->debug_safeguard_flags, IPCGPU_ERR_STATE, "ipcgpu_safeguard_debug_flags(ctx, 1, ...) before the check");
        CK(cudaStreamSynchronize(ctx->stream));
        if (tri_flags && ctx->nSF > 0) CK(cudaMemcpy(tri_flags, ctx->dbg_tri_flags.p, sizeof(int) * ctx->nSF, cudaMemcpyDeviceToHost));
        if (tet_hits && ctx->nT > 0) CK(cudaMemcpy(tet_hits, ctx->dbg_tet_hits.p, sizeof(int) * ctx->nT, cudaMemcpyDeviceToHost));
    }
    const int rc = safeguard_debug_flags(ctx, enable != 0);
    REQUIRE(rc == 0, rc, "safeguard debug buffer allocation failed");
    return IPCGPU_OK;
}

// ---- step control: CFL branch and line search (step_control.cu holds the decision kernel) ----------------------------------------
// Each loop body and loop condition is written once: a sequence of entry points plus one step_decide.  Outside a capture the
// host loops and reads the decision word (one synchronisation per decision); inside one the body is captured into a conditional node.
static int decide(ipcgpu_ctx* ctx, int op, double a, int b, cudaGraphConditionalHandle h, bool* word)
{
    step_decide(ctx->iter.p, op, a, b, (unsigned long long)h, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    if (word) {
        CK(cudaMemcpyAsync(&ctx->staging->decision, &ctx->iter.p->ls_cond, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        *word = ctx->staging->decision != 0;
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

// Optimizer::initX (:925-1233) for options 0-4 with the barrier solver (solveIP): the predictor becomes the search direction, its step is
// bounded (inversion filter, planes with slackness 0.9, swept hash + full CCD: initX always takes the full CCD, :1132) and applied with the
// two backtracking loops of the line search (kLsInversion, kLsIntersection).  Nothing here synchronises outside the host loops of cond_node.
int ipcgpu_warm_start(ipcgpu_ctx* ctx, int option, double voxel_size, double tol, const double err_vf[3], const double err_ee[3], double* alpha_out)
{
    REQUIRE(option >= 0 && option <= 4, IPCGPU_ERR_ARG, "warm start option 0-4 (initX option 5, Jacobi, is not supported)");
    REQUIRE(option == 0 || (err_vf && err_ee && voxel_size > 0.0), IPCGPU_ERR_ARG, "the warm start needs the Tight-Inclusion errors and a positive voxel size");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the warm start runs on one rank");
    REQUIRE(ctx->surface_ready && ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh and ipcgpu_set_surface first");
    ENTER(kSerial);
    DynamicsArgs dyn;
    int rc = timestep_prepare(ctx, &dyn);
    if (rc) return rc;
    timestep_predictor(dyn, option, ctx->dir.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    if ((rc = solver_adopt_direction(ctx, nullptr)) || (rc = step_control_prepare(ctx))) return rc;
    if ((rc = decide(ctx, kWsEntry, option ? 1.0 : 0.0, 0, 0, nullptr))) return rc; // stepSize = 1.0 (:1123)
    if (option) {
        if (ctx->energy == IPCGPU_NEOHOOKEAN && (rc = ipcgpu_inversion_step(ctx, nullptr, 0.2, nullptr))) return rc; // filterStepSize (:1124)
        if ((rc = ipcgpu_halfspace_step(ctx, nullptr, 0.9, nullptr))) return rc; // slackness_a (:1123, :1130-1131)
        if (ctx->n_hs > 0) CK(cudaMemsetAsync(&ctx->iter.p->hs_zero_step, 0, sizeof(int), ctx->stream)); // a zero bound is no error here
        if ((rc = ipcgpu_hash_build_swept(ctx, nullptr, nullptr, voxel_size))) return rc; // :1135
        if ((rc = ipcgpu_ccd_full_ti(ctx, tol, err_vf, err_ee, nullptr, nullptr))) return rc;
        CK(cudaMemcpyAsync(ctx->Vsaved.p, ctx->V.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream)); // V0 (:1191)
        ctx->state_saved = true;
        rc = ls_step(ctx); // :1192
        if (!rc && ctx->energy == IPCGPU_NEOHOOKEAN) { // getNeedElemInvSafeGuard() (:1194-1200)
            rc = ipcgpu_check_inversion(ctx, nullptr);
            if (!rc) rc = cond_node(ctx, true, kLsInversion, 0.0, 0, [&]() {
                int r = ls_step(ctx);
                return r ? r : ipcgpu_check_inversion(ctx, nullptr);
            });
        }
        const int terms = ctx->n_hs > 0 ? kTermHalfSpace : 0;
        if (!rc) rc = ls_intersection(ctx); // isIntersected (:1203-1210)
        if (!rc) rc = cond_node(ctx, true, kLsIntersection, 0.0, terms, [&]() {
            int r = ls_step(ctx);
            return r ? r : ls_intersection(ctx);
        });
        if (rc) return rc;
    }
    ctx->sc_pending = true;
    return alpha_out ? step_control_host_result(ctx, alpha_out) : IPCGPU_OK;
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

} // extern "C"
