// abi.h -- private to the C-ABI translation units (api*.cu) and to the stage files that report errors through ctx->err: the CUDA-check
// macros, the two chains of an iteration, and the prototypes of every host helper that crosses a file boundary.  Not installed.
#pragma once
#include "../../include/ipcgpu.h"
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
int energy_tail(ipcgpu_ctx* ctx, int slot, const double* partials, int n_partials, double scale, cudaEvent_t pe, double* E, bool fetch = false,
    unsigned check = 0);
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
void contact_pack_lists(ipcgpu_ctx* ctx);
void contact_unpack_lists(ipcgpu_ctx* ctx);
ipcgpu::SurfArgs surf_args(const ipcgpu_ctx* ctx);
ipcgpu::SortedGrid edge_grid(const ipcgpu_ctx* ctx);
int boxes_and_grid(ipcgpu_ctx* ctx, double radius, bool with_vertex_boxes);

// ---- ccd.cu -----------------------------------------------------------------------------------------------------------------
int ccd_alloc(ipcgpu_ctx* ctx);
int ccd_narrow(ipcgpu_ctx* ctx, const int2* cand, const int* n32, const unsigned long long* n64, unsigned long long cap, int share, double tol, const double* err_vf,
    const double* err_ee, int stage, const int* overflow);
int ccd_build_swept(ipcgpu_ctx* ctx, double h);
int ccd_full(ipcgpu_ctx* ctx, double tol, const double* err_vf, const double* err_ee);
int ccd_read_back(ipcgpu_ctx* ctx, double* alpha_out);

// ---- solve.cu, multilevel.cu, pattern.cu, safeguard.cu ----------------------------------------------------------------------
int solver_build_full_pattern(ipcgpu_ctx* ctx, const int* ia, const int* ja);
int solver_pcg(ipcgpu_ctx* ctx, const double* rhs_dev, double sign, double rel_tol, int max_iter, int* iters_out, double* rel_res_out);
int solver_pcg_multilevel(ipcgpu_ctx* ctx, const double* rhs_dev, double sign, double rel_tol, int max_iter, int* iters_out, double* rel_res_out);
int solver_multilevel_matrices(ipcgpu_ctx* ctx, double* dst, uint64_t count);
int solver_adopt_direction(ipcgpu_ctx* ctx, const double* src); // src NULL: the direction already in ctx->dir
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
