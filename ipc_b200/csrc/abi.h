// abi.h -- private to the C-ABI translation units (api*.cu) and to the stage files that report errors through ctx->err: the CUDA-check
// macros, the two chains of an iteration, and the prototypes of every host helper that crosses a file boundary.  Not installed.
#pragma once
#include "../../include/ipcgpu.h"
#include "common.cuh"
#include "context.h"
#include <cstddef>
#include <string>

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

static inline int nblk(long long n, int b) { return (int)((n + b - 1) / b); }

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
//   - time integration (timestep.cu): ipcgpu_compute_xtilde, ipcgpu_end_time_step and ipcgpu_warm_start write xtilde, Vprev, V, dir and the
//     dynamic state (vel, acc, dxe), which the derivative chain reads (inertia, damping, friction) or the step-bound chain does (dir): all
//     three are kSerial.
//   - the device-resident kappa (kappa.cu): the barrier / plane derivative calls given IPCGPU_KAPPA_DEVICE read IterState::kappa; every call
//     that writes it or the other kappa words -- ipcgpu_set_kappa, _kappa_init (which also reads g and V), _kappa_clear_close_set and
//     _kappa_post_line_search (which reads V and the contact sets) -- is kSerial, which orders it before the derivative chain.  The pair-Hessian
//     build of ipcgpu_barrier_hessian runs on the side stream, which waits on ev_inputs only: the three calls that write kappa mark the
//     inputs (mark_inputs) as a position or set change does.  The step-bound chain touches none of them.
//   - end-of-step diagnostics (diagnostics.cu): ipcgpu_system_energy reads V, Vprev, mass and TimeParams and writes e_per_tet and partials
//     (the per-tet elastic energy, as ipcgpu_elastic_energy does) and diag_part / diag_sys; ipcgpu_constraint_summary reads V, the self /
//     obstacle active list, the plane set and IterState::kappa and writes cw.bval and diag_sum*.  Both are kSerial: e_per_tet and bval are
//     no input of either chain, and the chains' writes to V and the lists are ordered before them.
//   - V, Vrest, SE, dbc, ia, ja: read by both, written by neither (ia / ja / slot_off are written only by ipcgpu_update_pattern, which joins).  g, a, gcont, hblk, e_partials2, bHraw, brows, bpsd:
//     derivative chain only.  dir, pSize_dev, inv_steps: step-bound chain only.
enum Chain { kSerial, kStepBound, kDerivative };

inline int join_deriv(ipcgpu_ctx* ctx)
{
    if (!ctx->deriv_open) return IPCGPU_OK;
    ctx->deriv_open = false;
    CK(cudaEventRecord(ctx->ev_deriv_done, ctx->deriv));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_deriv_done, 0));
    return IPCGPU_OK;
}

// first call of every entry point that touches the device: the context's device, then the chain (only ipcgpu_download_range_async,
// ipcgpu_graph_kernel_priorities and ipcgpu_step_control_info without a pending result set the device themselves instead)
inline int enter(ipcgpu_ctx* ctx, Chain chain)
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

// ---- api.cu: the read-back of the iteration state and the tails the synchronous forms share ----------------------------------
int join_copy_stream(ipcgpu_ctx* ctx);
int fetch_iter_state(ipcgpu_ctx* ctx);
int sync_pattern_mirror(ipcgpu_ctx* ctx);
int flag_status(ipcgpu_ctx* ctx, unsigned mask);
void set_local(ipcgpu_ctx* ctx, unsigned bits, bool local);
int energy_result(ipcgpu_ctx* ctx, int slot, double* E, bool fetch = false, unsigned check = 0);
// scale_dev != nullptr: the scale is read on the device from there (the device-resident kappa)
int energy_tail(ipcgpu_ctx* ctx, int slot, const double* partials, int n_partials, double scale, cudaEvent_t pe, double* E, bool fetch = false,
    unsigned check = 0, const double* scale_dev = nullptr);

// ---- the barrier stiffness: a kappa argument equal to IPCGPU_KAPPA_DEVICE stands for IterState::kappa, read at run time (one rank only) ----
inline bool kappa_on_device(double kappa) { return kappa == IPCGPU_KAPPA_DEVICE; }
inline const double* kappa_ptr(ipcgpu_ctx* ctx, double kappa) { return kappa_on_device(kappa) ? &ctx->iter.p->kappa : nullptr; }
#define REQUIRE_KAPPA(kappa)                                                                                                        \
    REQUIRE(!kappa_on_device(kappa) || ctx->nranks == 1, IPCGPU_ERR_STATE, "the device-resident kappa (IPCGPU_KAPPA_DEVICE) runs on one rank")
int gradient_roundtrip_begin(ipcgpu_ctx* ctx, const double* g_in);
int gradient_roundtrip_end(ipcgpu_ctx* ctx, double* g_out);
int hessian_begin(ipcgpu_ctx* ctx, Chain chain, const double* a_inout);
int hessian_end(ipcgpu_ctx* ctx, double* a_inout, unsigned check);

// ---- api_comm.cu: the cross-rank collectives, in place on the context's stream (no-ops on one rank); `what` is the error text ----------
int nccl_sum(ipcgpu_ctx* ctx, double* buf, size_t n, const char* what);
int nccl_sum(ipcgpu_ctx* ctx, int* buf, size_t n, const char* what);
int nccl_min_u64(ipcgpu_ctx* ctx, unsigned long long* word); // min over ranks of a device-resident uint64 (the order-preserving image of a step)
int nccl_all_gather(ipcgpu_ctx* ctx, const int4* send, int4* recv, size_t n, const char* what); // n int4 per rank
void nccl_comm_destroy(ipcgpu_ctx* ctx);

// ---- api_mesh.cu ------------------------------------------------------------------------------------------------------------
int build_maps(ipcgpu_ctx* ctx);
void owned_value_range(ipcgpu_ctx* ctx);
int ensure_offsets(ipcgpu_ctx* ctx);
int upload_dir(ipcgpu_ctx* ctx, const double* p);

// ---- api_terms.cu: checks the time-integration state, sizes the dynamic state and x~, fills the kernels' arguments ----------------------
int timestep_prepare(ipcgpu_ctx* ctx, ipcgpu::DynamicsArgs* p);

// ---- constraint.cu ----------------------------------------------------------------------------------------------------------
namespace ipcgpu {
struct SortedGrid; // broadphase.cuh
}
int contact_alloc(ipcgpu_ctx* ctx);
int contact_constraint_set(ipcgpu_ctx* ctx, double dHat, int wantCand, int* nC, int* nPara, int* nCand);
int contact_sync_counts(ipcgpu_ctx* ctx);
int contact_scan(ipcgpu_ctx* ctx, const int* in, int* out, int n); // exclusive sum of n ints through the cub_tmp scratch
// canonical order (lexicographic on the signed components, companion last) of a list of min(*n, cap) entries, sized on the device:
// lex_order leaves the sorting permutation in ContactWork::perm, permute applies it to the list or a companion of `words` 8-byte words
int lex_order(ipcgpu_ctx* ctx, const int4* list, const int2* comp, const int* n, int cap);
int lex_order(ipcgpu_ctx* ctx, const int2* list, const int* n, int cap);
void permute(ipcgpu_ctx* ctx, void* data, int words, const int* n, int cap);
int contact_sort_lists(ipcgpu_ctx* ctx); // act, para + para_e and (want_cand) cand in canonical order
void contact_pack_lists(ipcgpu_ctx* ctx);
void contact_unpack_lists(ipcgpu_ctx* ctx);
ipcgpu::SurfArgs surf_args(const ipcgpu_ctx* ctx);
ipcgpu::BarrierArgs barrier_args(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC); // (api_contact.cu; kappa may be IPCGPU_KAPPA_DEVICE)
ipcgpu::HalfSpaceArgs halfspace_args(ipcgpu_ctx* ctx);                                      // (api_terms.cu)
ipcgpu::SortedGrid edge_grid(const ipcgpu_ctx* ctx);

// ---- repro.cu: the reproducible mode (canonical order level 2) -----------------------------------------------------------------------
int repro_alloc(ipcgpu_ctx* ctx);                        // its workspace, sized by the pair capacity and the mesh (outside a capture)
bool repro_on(const ipcgpu_ctx* ctx);                    // level 2 on one rank, workspace allocated
int repro_contact_lists(ipcgpu_ctx* ctx);                // the gather indices of act / para (in canonical order)
int repro_friction_list(ipcgpu_ctx* ctx, bool sort);     // fr_cs (+ companions) in canonical order if `sort`, its gather indices
ipcgpu::ReproArgs repro_barrier_args(ipcgpu_ctx* ctx);   // on = 0 unless the indices belong to the lists in act / para
ipcgpu::ReproArgs repro_friction_args(ipcgpu_ctx* ctx);  // ... to the list in fr_cs
int boxes_and_grid(ipcgpu_ctx* ctx, double radius, bool with_vertex_boxes);

// ---- ccd.cu -----------------------------------------------------------------------------------------------------------------
int ccd_alloc(ipcgpu_ctx* ctx);
int ccd_narrow(ipcgpu_ctx* ctx, const int2* cand, const int* n32, const unsigned long long* n64, unsigned long long cap, int share, double tol, const double* err_vf,
    const double* err_ee, int stage, const int* overflow);
int ccd_build_swept(ipcgpu_ctx* ctx, double h);
int ccd_full(ipcgpu_ctx* ctx, double tol, const double* err_vf, const double* err_ee);
int ccd_read_back(ipcgpu_ctx* ctx, double* alpha_out);

// ---- api_step.cu: the decisions of the step control and of the Krylov loops ----------------------------------------------------
// one step_decide(op) on the main stream; word != NULL: read back (with the solve's words, IterState::ls_cond + kDecisionBytes) and returned
int decide(ipcgpu_ctx* ctx, int op, double a, int b, cudaGraphConditionalHandle h, bool* word, const double* aux = nullptr);
int cond_prepare(ipcgpu_ctx* ctx, const char* what); // the streams of cond_node's bodies (refused inside a capture before an eager run)

// if (decision) body  /  while (decision) body, where the decision is step_decide(op) before the node and, for a loop, at the end of each pass.
// Captured: the handle is created on the graph being captured, the decision before the node sets it, the node is added behind the
// capture's current dependencies, and the body is captured into the node's body graph on a stream of its own (ctx->stream points to it
// meanwhile, so that the entry points the body calls enqueue there).
template <typename Body>
int cond_node(ipcgpu_ctx* ctx, bool loop, int op, double a, int b, Body body)
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

// ---- solve.cu, multilevel.cu, pattern.cu, safeguard.cu ----------------------------------------------------------------------
// The Krylov loops of both solvers, after their set-up and a step_decide(kSolveStart): bursts of kKrylovBurst iterations as the body of a
// WHILE whose decision (kSolveBurst) stops on a non-finite residual, on sqrt(rr) <= rel_tol sqrt(bb) or when the next burst would pass
// max_iter, then the max_iter % kKrylovBurst iterations left as a second WHILE that runs at most once.  `iteration` enqueues one iteration
// on ctx->stream (read it there: inside a capture it is the body's stream).  The set-up check (|b| > 0, no pivot <= 0) is the first
// decision of the first WHILE.  Eager: one read per burst plus the one before the first, as many as a host loop needs.
constexpr int kKrylovBurst = 25;
int solver_finish(ipcgpu_ctx* ctx); // max |x_i| into IterState::sv_xmax_ord
template <typename Iteration>
int krylov_loops(ipcgpu_ctx* ctx, int max_iter, Iteration iteration)
{
    for (const int burst : { kKrylovBurst, max_iter % kKrylovBurst }) {
        if (burst == 0 || burst > max_iter) continue;
        int rc = cond_node(ctx, true, ipcgpu::kSolveBurst, 0.0, burst, [&]() {
            for (int k = 0; k < burst; ++k) iteration();
            CK(cudaGetLastError());
            return IPCGPU_OK;
        });
        if (rc) return rc;
    }
    return solver_finish(ctx);
}
int solver_full_pattern(ipcgpu_ctx* ctx);        // fia / fja / fpos of the pattern in ia / ja, rebuilt on the device when its version moved
int solver_forget_full_pattern(ipcgpu_ctx* ctx); // a new pattern (ipcgpu_set_csr / ipcgpu_enable_device_pattern): the next solve rebuilds
// PCG with the block-Jacobi or the multilevel preconditioner; its workspace pcg_part holds kPcgSpmvBlocks SpMV partials, then 2 per CTA
// of one thread per vertex
constexpr int kPcgSpmvBlocks = ipcgpu::kSMs * 8;
enum { kPrecondJacobi = 0, kPrecondMultilevel = 1, kPrecondAmg = 2 }; // solver_pcg's preconditioner
int solver_pcg(ipcgpu_ctx* ctx, const double* rhs_dev, double sign, double rel_tol, int max_iter, int precond);
int solver_multilevel_build(ipcgpu_ctx* ctx, double* bad_pivot); // the hierarchy at the current matrix and positions (set-up)
void solver_multilevel_step(ipcgpu_ctx* ctx, bool start);        // (iteration: the CG update first) z = M^-1 r, partials of r.z and r.r
int solver_multilevel_matrices(ipcgpu_ctx* ctx, double* dst, uint64_t count);
int solver_amg_build(ipcgpu_ctx* ctx, double* bad_pivot); // the smoothed-aggregation hierarchy of the resident matrix (set-up)
void solver_amg_step(ipcgpu_ctx* ctx, bool start);        // (iteration: the CG update first) one W-cycle z = M^-1 r, partials of r.z and r.r
size_t solver_amg_bytes(const ipcgpu_ctx* ctx);           // device memory the AMG workspace holds
int solver_amg_reserve(ipcgpu_ctx* ctx, double headroom);  // ipcgpu_amg_reserve (the hierarchy of the last set-up read back first)
bool solver_amg_reserved(ipcgpu_ctx* ctx);                 // a reservation that still fits the mesh and pattern (another one is dropped)
int solver_amg_read(ipcgpu_ctx* ctx);                      // AmgDev into AmgWork::h (synchronises)
int solver_amg_coarse_enough(ipcgpu_ctx* ctx, int rows);   // the "at most rows block rows is the last level" rule, in device memory
int solver_adopt_direction(ipcgpu_ctx* ctx, const double* src); // src NULL: the direction already in ctx->dir
// (sign g_i) / a(i,i) into out; jacobi: initX option 5's predictor (0 on Dirichlet vertices and the obstacle tail, no status words)
void solver_precondition_diag(ipcgpu_ctx* ctx, double sign, double* out, bool jacobi);
int pattern_enable(ipcgpu_ctx* ctx, int index_base, uint64_t nnz_capacity);
int pattern_update(ipcgpu_ctx* ctx, const ipcgpu::BarrierArgs& lists, bool with_friction);
int safeguard_inversion(ipcgpu_ctx* ctx);
int safeguard_intersections(ipcgpu_ctx* ctx);
int safeguard_debug_flags(ipcgpu_ctx* ctx, bool on); // test hook: per-triangle flags and per-tet point counts of the intersection check
int safeguard_set_points(ipcgpu_ctx* ctx, const int* vCoDim); // the codimension-0 vertices of the point-in-tetrahedron check (vCoDim nullable)

// A gradient / Hessian term.  NULL output: the term on `chain`; host output: the caller's array in, the term added on the main stream,
// the rank-completed array out and, for a Hessian, the flags of `check` it may raise returned as its status.
// `stage`: the stage timer the term is counted under.
template <typename Launch>
int gradient_call(ipcgpu_ctx* ctx, Chain chain, double* g_inout, Launch launch, int stage = IPCGPU_STAGE_BARRIER)
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
template <typename Launch>
int hessian_call(ipcgpu_ctx* ctx, Chain chain, double* a_inout, unsigned check, Launch launch, int stage = IPCGPU_STAGE_BARRIER)
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
