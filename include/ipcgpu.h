/*
 * ipcgpu.h -- C ABI of the H100-native IPC Newton hot path (libipcgpu.so).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch/Eigen types.  Each entry point
 * names the reference interface (ipc-sim/IPC @ 573d2c7, paths relative to the reference root) that a
 * maintainer would rebind to it; INTEGRATION.md shows the adapter classes.
 *
 * Conventions
 *  - One context per process per GPU (one rank = one GPU); multi-GPU runs are N processes that share
 *    an NCCL communicator handed in through ipcgpu_comm_init.
 *  - All reals are double, all indices int32.  Layouts are exactly what the reference's Eigen objects
 *    expose through .data():
 *       V, V_rest  : column-major nV x 3  => SoA [x(nV) | y(nV) | z(nV)]        (Mesh.hpp:61)
 *       F (tets)   : column-major nT x 4  => SoA [v0(nT) | v1 | v2 | v3]         (Mesh.hpp:64)
 *       SF         : column-major nSF x 3 => SoA                                 (Mesh.hpp:70)
 *       restTriInv : nT matrices 3x3, each column-major (9 doubles)              (Mesh.hpp:90)
 *       gradient / searchDir : interleaved [x0 y0 z0 x1 ...]                     (Energy.cpp:275)
 *       CSR        : upper-triangular ia/ja/a of LinSysSolver                    (LinSysSolver.hpp:34-37)
 *  - Every function returns 0 on success, otherwise an IPCGPU_ERR_* code; nothing here calls exit().
 *    ipcgpu_last_error() gives a human-readable message for the last failure on that context.
 *  - Host output pointers may be NULL: the result then stays device-resident (no D2H copy, NO host synchronisation) and
 *    is consumed by the later calls on the device.  With every output NULL a whole Newton iteration -- constraint set, E, g, H,
 *    inversion filter, partial CCD, swept grid, full CCD, and with several ranks the NCCL reductions between them -- is ONE
 *    uninterrupted stream; ipcgpu_fetch_iteration() then reads all scalars back with a single synchronisation.  In particular
 *    the step bound travels on the device: alpha_inout == NULL means "the device-resident step" (start it with
 *    ipcgpu_step_bound_set).  Host INPUT arrays handed to such calls must stay untouched until the next fetch / sync.
 *  - Several ranks: tets are block-partitioned for the energy and the inversion filter; the gradient/Hessian assembly is by ROW
 *    OWNER -- a rank owns a contiguous vertex range, assembles every tet and every contact pair that touches it and holds the
 *    complete CSR rows of that range (ipcgpu_partition_info), so the Hessian needs no cross-rank reduction; the gradient is one
 *    sum-allreduce of 3 nV doubles, every step bound one min-allreduce of a uint64.
 */
#ifndef IPCGPU_H
#define IPCGPU_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ipcgpu_ctx ipcgpu_ctx;

enum {
    IPCGPU_OK = 0,
    IPCGPU_ERR_CUDA = 1,
    IPCGPU_ERR_ARG = 2,
    IPCGPU_ERR_PATTERN = 3,
    IPCGPU_ERR_NONPOSITIVE_DISTANCE = 4, /* Optimizer.cpp:3296-3306 would exit(0) */
    IPCGPU_ERR_CAPACITY = 5,
    IPCGPU_ERR_NCCL = 6,
    IPCGPU_ERR_STATE = 7,
    IPCGPU_ERR_LINE_SEARCH = 8, /* step 0: a line search whose entry state fails a safeguard (the reference loops forever, Optimizer.cpp:2710-2811),
                                   or a zero step bound (Optimizer.cpp:2031-2033 would exit(-1)) */
    IPCGPU_ERR_SOLVE = 9 /* ipcgpu_solve_pcg_multilevel: a domain matrix of the preconditioner has a pivot <= 0 (the matrix is not positive definite) */
};

enum { IPCGPU_NEOHOOKEAN = 0, IPCGPU_FIXED_COROT = 1 };

/* device-resident result buffers that ipcgpu_download() can fetch */
enum {
    IPCGPU_BUF_GRADIENT = 0,      /* 3*nV doubles, interleaved */
    IPCGPU_BUF_CSR_VALUES = 1,    /* nnz doubles */
    IPCGPU_BUF_ENERGY_PER_TET = 2,/* nT doubles */
    IPCGPU_BUF_TET_HESSIANS = 3,  /* 78*nT doubles (block layout, see DESIGN.md) */
    IPCGPU_BUF_TET_GRADIENTS = 4, /* 12*nT doubles */
    IPCGPU_BUF_INVERSION_STEPS = 5,/* nT doubles */
    /* ipcgpu_device_ptr only (int arrays): the CSR row starts (n_rows + 1) and column indices (nnz) in the context's index base -- with
     * the device-built pattern they change when ipcgpu_pattern_info reports `changed` (a device solver re-points its matrix then) */
    IPCGPU_BUF_CSR_ROW_STARTS = 6,
    IPCGPU_BUF_CSR_COLUMNS = 7,
    /* the state a time step leaves on the device (ipcgpu_end_time_step / ipcgpu_warm_start / the line search), for the frame a binding writes
     * out: positions result.V (SoA, 3*nV), the search direction (interleaved, 3*nV; the warm start's predictor), xTilta (SoA, 3*nV) */
    IPCGPU_BUF_POSITIONS = 8,
    IPCGPU_BUF_SEARCH_DIR = 9,
    IPCGPU_BUF_XTILDE = 10,
    /* the inverses the last ipcgpu_solve_pcg_multilevel stored: 96*96 doubles per domain, row-major and symmetric, level after level
     * (ipcgpu_multilevel_info gives the domains per level) */
    IPCGPU_BUF_MULTILEVEL_INVERSES = 11
};

/* ---- lifetime ---------------------------------------------------------------------------------- */
int ipcgpu_create(int device, ipcgpu_ctx** out);
void ipcgpu_destroy(ipcgpu_ctx* ctx);
const char* ipcgpu_last_error(const ipcgpu_ctx* ctx);
/* pinned host allocations so that host<->device copies of the big result arrays run at PCIe speed */
int ipcgpu_host_alloc(void** ptr, uint64_t bytes);
int ipcgpu_host_free(void* ptr);
int ipcgpu_sync(ipcgpu_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t ipcgpu_launch_count(const ipcgpu_ctx* ctx);

/* ---- multi-GPU (tet / pair partition + NCCL) ------------------------------------------------------ */
/* 128-byte ncclUniqueId created on rank 0 and broadcast by the host (torch.distributed / MPI / file). */
int ipcgpu_comm_unique_id(void* id128);
int ipcgpu_comm_init(ipcgpu_ctx* ctx, int rank, int nranks, const void* id128);
/* what this rank owns: tets [tet_begin, tet_end) (energy, inversion filter), the rows of vertices [row_vertex_begin,
 * row_vertex_end) = CSR values [value_begin, value_end) (0-based offsets into `a`; valid after ipcgpu_set_csr), and how many
 * tets it assembles for them (boundary tets are assembled by both neighbours).  Any pointer may be NULL. */
int ipcgpu_partition_info(ipcgpu_ctx* ctx, int* rank, int* nranks, int* tet_begin, int* tet_end, int* row_vertex_begin, int* row_vertex_end,
    int64_t* value_begin, int64_t* value_end, int* n_assembled_tets);

/* ---- one read-back per Newton iteration -------------------------------------------------------------------- */
typedef struct ipcgpu_iteration {
    double energy_elastic, energy_barrier;   /* last ipcgpu_elastic_energy / ipcgpu_barrier_energy (summed over ranks) */
    double alpha_inversion, alpha_partial_ccd, alpha_swept_grid, alpha_full_ccd; /* the step after each bound of Optimizer.cpp:1884-2040 */
    double alpha;                            /* the device-resident step now */
    int n_active, n_mollified, n_candidates; /* sizes of the last constraint set (this rank's lists) */
    int status;                              /* IPCGPU_OK or the first deferred error (d <= 0, capacity, pattern) -- same on every rank */
    uint64_t n_full_ccd_candidates;          /* candidates of the last full CCD (this rank) */
    uint64_t ti_warnings;                    /* conservative early-outs of the Tight-Inclusion searches since the last fetch (should be 0) */
    int n_inverted_tets;                     /* last ipcgpu_check_inversion (summed over ranks) */
    int n_intersected_triangles;             /* last ipcgpu_intersection_free: surface triangles crossed by an edge plus (codimension-0
                                              * vertex, tet) pairs with the vertex inside (summed over ranks) */
    double energy_friction, energy_inertia;  /* last ipcgpu_friction_energy / ipcgpu_inertia_energy (summed over ranks) */
    /* half-space collision objects (ipcgpu_set_halfspaces; all 0 without planes) */
    double energy_halfspace;                 /* last ipcgpu_halfspace_energy (summed over ranks) */
    double energy_halfspace_friction;        /* last ipcgpu_halfspace_friction_energy (summed over ranks) */
    double alpha_halfspace;                  /* the step after the last ipcgpu_halfspace_step */
    int n_halfspace_active;                  /* size of the last plane active set (every rank holds all of it) */
    int n_halfspace_crossings;               /* last ipcgpu_halfspace_crossings (summed over ranks) */
    /* damping, Neumann forces, Dirichlet penalty (single rank; 0 while a term is not set) */
    double energy_damping;                   /* last ipcgpu_damping_energy */
    double energy_neumann;                   /* last ipcgpu_neumann_energy */
    double energy_dirichlet;                 /* last ipcgpu_dirichlet_energy */
    double dirichlet_completed_step;         /* last ipcgpu_dirichlet_completed_step (0 before the first) */
} ipcgpu_iteration;
/* Synchronises once, completes the deferred cross-rank scalars (collective: every rank must call it), fills `out`, clears the
 * deferred error flags and returns out->status. */
int ipcgpu_fetch_iteration(ipcgpu_ctx* ctx, ipcgpu_iteration* out);
/* start value of the device-resident step bound (Optimizer.cpp:1884: alpha = 1) */
int ipcgpu_step_bound_set(ipcgpu_ctx* ctx, double alpha);

/* ---- CUDA graphs of device-resident call sequences ---------------------------------------------------------------------
 * Everything between ipcgpu_capture_begin and ipcgpu_capture_end is recorded instead of executed (every call in between must be in its
 * NULL-output form: nothing may synchronise or copy to the host) and replayed by ipcgpu_graph_launch as ONE launch.  What a graph bakes
 * in: the host scalars handed to the calls (dHat, kappa, coef, tolerances, Tight-Inclusion errors, voxel size) and the device buffers.
 * What it does not: positions (ipcgpu_set_state), search direction (ipcgpu_set_search_dir), previous state / xTilta, the contact sets,
 * list sizes and step bounds -- they live in device memory and are read at replay time.  So one capture serves every Newton iteration
 * of a solve; capture again after ipcgpu_set_mesh / _set_surface / _set_csr / _set_*_capacity / _comm_init / _set_canonical_order /
 * _set_contact_partition (older graphs are refused with IPCGPU_ERR_STATE) or when dHat / kappa change.  Run the sequence once eagerly
 * before capturing it (lazy allocations), with ipcgpu_set_canonical_order(ctx, 0): the canonical sort of the contact lists needs their sizes
 * on the host.  Collective: with several ranks every rank captures and launches the same sequence.
 * ipcgpu_fetch_iteration stays outside the graph. */
int ipcgpu_capture_begin(ipcgpu_ctx* ctx);
int ipcgpu_capture_end(ipcgpu_ctx* ctx, int* graph_id);
int ipcgpu_graph_launch(ipcgpu_ctx* ctx, int graph_id);
int ipcgpu_graph_destroy(ipcgpu_ctx* ctx, int graph_id);
/* kernel nodes of a captured graph at the high and at the low stream priority; a replay keeps each node's priority.  The step-bound chain
 * runs at the high one and the derivative chain (gradient, Hessian, CSR assembly) at the low one -- the other way round in a graph that
 * copies derivative results to the host (ipcgpu_download_range_async), where the derivative chain and its copy are the critical path */
int ipcgpu_graph_kernel_priorities(ipcgpu_ctx* ctx, int graph_id, int* n_high, int* n_low);

/* ---- scene (once per scene; replaces what Mesh<3> precomputes, Mesh.cpp:415-527, :661-671) ------- */
int ipcgpu_set_mesh(ipcgpu_ctx* ctx, int nV, int nT,
    const double* V_rest_soa, const int* tets_soa,
    const double* restTriInv /* 9*nT */, const double* vol /* triArea */,
    const double* mu, const double* lam,
    const double* mass_diag /* nV, may be NULL */,
    const uint8_t* dbc_type /* nV: 0 NOT_DBC, 1 ZERO, 2 NONZERO; may be NULL */,
    int energy);
/* LinSysSolver::set_pattern result (LinSysSolver.hpp:46-150): ia has n_rows+1 entries.
 * Must be called again whenever the contact stencil changes the pattern (Optimizer.cpp:3556-3595) -- or let the device build the
 * pattern (ipcgpu_enable_device_pattern below).  Returns a context in device-pattern mode to host mode. */
int ipcgpu_set_csr(ipcgpu_ctx* ctx, int n_rows, const int* ia, const int* ja, int index_base);
/* ---- device-built sparsity pattern (opt-in; DESIGN.md section 3.10, INTEGRATION.md sections 4-5) ----
 * ipcgpu_enable_device_pattern: the device builds and owns the pattern from here on.  Builds the mesh part once (vNeighbor, Mesh.cpp:470-493:
 * tet edges and SFEdges, both vertices below the obstacle tail), sizes ja / a for nnz_capacity entries (0 = the mesh pattern's nnz x 1.25)
 * and sets the mesh-only pattern.  Call it after ipcgpu_set_mesh (which returns to host mode) and ipcgpu_set_surface; a later
 * ipcgpu_set_surface / ipcgpu_set_obstacle_tail rebuilds the mesh part.  Call it again to raise the capacity.  Captured graphs are refused
 * afterwards, as after ipcgpu_set_csr. */
int ipcgpu_enable_device_pattern(ipcgpu_ctx* ctx, int index_base, uint64_t nnz_capacity);
/* augmentConnectivity (SelfCollisionHandler.cpp:330-415) + LinSysSolver::set_pattern over the device-resident active set, the mollified set
 * (MMCVIDs and eIeJ) and, with_friction != 0, the lagged friction set: the pattern becomes exactly vNeighbor + these contact neighbours
 * (not the union with earlier patterns).  Its place in an iteration: right after ipcgpu_constraint_set, before the first derivative call.
 * NULL outputs: deferred and capturable; the result is read by ipcgpu_fetch_iteration / ipcgpu_pattern_info, a pattern that would exceed the
 * capacity is reported there as IPCGPU_ERR_CAPACITY (the previous pattern stays, nothing is truncated).  Host outputs: synchronises and
 * returns changed (the extra blocks differ from the previous pattern's) and nnz. */
int ipcgpu_update_pattern(ipcgpu_ctx* ctx, int with_friction, int* changed, int64_t* nnz);
/* result of the last update (synchronises when one was enqueued since the last fetch): changed, nnz, and a version that every update that
 * rewrote the pattern bumps.  Any pointer may be NULL. */
int ipcgpu_pattern_info(ipcgpu_ctx* ctx, int* changed, int64_t* nnz, uint64_t* version);
/* download the current pattern (ia: n_rows + 1 entries, ja: nnz) for a host solver's analyze_pattern; either pointer may be NULL */
int ipcgpu_get_pattern(ipcgpu_ctx* ctx, int* ia, int* ja);
/* current positions (mesh.V); NULL keeps the device copy (after ipcgpu_step_forward) */
int ipcgpu_set_state(ipcgpu_ctx* ctx, const double* V_soa);
/* x = x0 + alpha*p on the device (Optimizer::stepForward, Optimizer.cpp:2919-2938); x0 = state at the
 * time of ipcgpu_save_state */
int ipcgpu_save_state(ipcgpu_ctx* ctx);
/* upload the search direction p (interleaved 3nV) once; later calls may pass p = NULL to reuse it */
int ipcgpu_set_search_dir(ipcgpu_ctx* ctx, const double* p_interleaved);
int ipcgpu_step_forward(ipcgpu_ctx* ctx, const double* p_interleaved /* NULL = last search dir */, double alpha);

/* ---- elastic plug-in: Energy<3> virtuals (Energy.hpp:42-131) ---------------------------------------- */
/* Energy::computeEnergyVal (Energy.cpp:232-242): E = coef * sum_t psi_t * vol_t */
int ipcgpu_elastic_energy(ipcgpu_ctx* ctx, double coef, int redoSVD, double* E);
/* Energy::computeGradient (Energy.cpp:245-289): g (3nV interleaved) is overwritten */
int ipcgpu_elastic_gradient(ipcgpu_ctx* ctx, double coef, int redoSVD, int projectDBC, double* g);
/* Energy::computeHessian (Energy.cpp:292-331) into the CSR value array.
 * a_inout != NULL: host array is uploaded, accumulated into and downloaded (addCoeff semantics);
 * a_inout == NULL: device-resident values are accumulated (zero them with ipcgpu_csr_set_zero). */
int ipcgpu_elastic_hessian(ipcgpu_ctx* ctx, double coef, int redoSVD, int projectSPD, int projectDBC, double* a_inout);
/* fused variant for the Newton loop: computeGradient + computePrecondMtr's setZero, elastic and mass terms in one
 * pass over the tets (Optimizer.cpp:3416, 3439-3450, 3616-3668). The device-resident gradient and CSR values are
 * OVERWRITTEN (the value array is zeroed first, like LinSysSolver::setZero at :3616); the barrier_* calls then accumulate
 * on top.  Results stay on the device when the pointers are NULL. */
int ipcgpu_elastic_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass,
    double* g, double* a);
/* ... and computeEnergyVal in the same pass: the reference caches F / U / sigma / V between computeEnergyVal(redoSVD = 2) and the gradient /
 * Hessian of the same state (Optimizer.hpp:115-116); here the energy is a by-product of the kernel that already holds the singular values
 * (one SVD per tet and iteration instead of two).  E NULL: the energy stays on the device (ipcgpu_fetch_iteration). */
int ipcgpu_elastic_energy_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass,
    double* E, double* g, double* a);
/* Energy::filterStepSize (Energy.cpp:565-581); alpha_inout == NULL: the device-resident step */
int ipcgpu_inversion_step(ipcgpu_ctx* ctx, const double* p_interleaved, double slack, double* alpha_inout);

/* ---- contact plug-in: SelfCollisionHandler<3> statics (SelfCollisionHandler.hpp:23-232) ------------------- */
/* Surface arrays of Mesh<3>: SVI (Mesh.hpp:72), SFEdges as interleaved (first,second) pairs (Mesh.hpp:74), SF column-major
 * (Mesh.hpp:70), optional per-vertex codimension (Mesh::vICoDim; NULL = all 3). */
int ipcgpu_set_surface(ipcgpu_ctx* ctx, int nSV, const int* SVI, int nSE, const int* SFEdges, int nSF, const int* SF_soa, const int* vCoDim);
/* capacity (entries) of the device-side pair lists; default 2^20. IPCGPU_ERR_CAPACITY is returned when exceeded. */
int ipcgpu_set_pair_capacity(ipcgpu_ctx* ctx, int capacity);
/* Multi-rank, partitioned build (ipcgpu_set_contact_partition(1)): every rank ships its part of the active / mollified lists in ONE fixed-size
 * message (sizes are device-resident, so the message cannot be sized per call); this is its capacity in pairs per rank and list (default and
 * maximum 65,536 = 2.6 MB per rank).  A driver that knows the size of the contact set (it just rebuilt the sparsity pattern from it) sets a
 * few times its per-rank share; exceeding it raises IPCGPU_ERR_CAPACITY at the fetch, never truncation. */
int ipcgpu_set_exchange_capacity(ipcgpu_ctx* ctx, int pairs_per_rank);
/* SelfCollisionHandler::computeConstraintSet (SelfCollisionHandler.cpp:2149-2478) with the broad phase of
 * SpatialHash::build/query* (SpatialHash.hpp:46-229, 375-421) done on the device. The sets stay on the device (they feed the
 * barrier_* calls and the partial CCD); sizes are returned.  Output order is canonical: every list sorted lexicographically. */
int ipcgpu_constraint_set(ipcgpu_ctx* ctx, double dHat, int getPTEE, int* nC, int* nPara, int* nCand);
/* sizes of the last set (synchronises if it was built with NULL size pointers) */
int ipcgpu_constraint_set_sizes(ipcgpu_ctx* ctx, int* nC, int* nPara, int* nCand);
/* enable=1 (default): the lists are returned in canonical (lexicographic) order, so two runs give bitwise identical sets and sums.
 * enable=0: the order is whatever the atomic appends produced -- the same freedom the reference has (its order depends on
 * unordered_set iteration and TBB scheduling); saves the sorting passes when the sets are only consumed on the device. */
int ipcgpu_set_canonical_order(ipcgpu_ctx* ctx, int enable);
/* Multi-rank only. enable=1: ipcgpu_constraint_set issues only this rank's share of the PT/EE queries, so every rank holds a disjoint
 * part of the sets (PP/PE multiplicities may be split between ranks, which leaves the summed E/g/H unchanged because
 * makePD(c*M) = c*makePD(M) for c > 0); the counts returned are local.  enable=0 (default): every rank builds the whole set
 * (what the host needs to extend the sparsity pattern) and the per-pair work is split by list index. */
int ipcgpu_set_contact_partition(ipcgpu_ctx* ctx, int enable);
/* copies of constraintSet (4 ints each, MMCVID encoding), paraEEMMCVIDSet (4), paraEEeIeJSet (2), cs_PTEE (2); any may be NULL */
int ipcgpu_get_constraint_set(ipcgpu_ctx* ctx, int* mmcvid4, int* para4, int* para_eIeJ2, int* cand2);
/* upload host-built sets instead (drop-in use of only the per-pair kernels) */
int ipcgpu_set_constraint_set(ipcgpu_ctx* ctx, int nC, const int* mmcvid4, int nPara, const int* para4, const int* para_eIeJ2, int nCand, const int* cand2);
/* kappa * [ sum mult*b(d) + sum e*b(d) ]  (evaluateConstraints :64-81 + Optimizer.cpp:3290-3353).
 * Returns IPCGPU_ERR_NONPOSITIVE_DISTANCE where the reference would exit(0) (Optimizer.cpp:3296-3306). */
int ipcgpu_barrier_energy(ipcgpu_ctx* ctx, double dHat, double kappa, double* E);
/* g += kappa*J^T b' (+ mollified terms)  (leftMultiplyConstraintJacobianT :84-148, augmentParaEEGradient :2990-3045).
 * g_inout != NULL: host vector uploaded, accumulated, downloaded; NULL: the device-resident gradient is accumulated. */
int ipcgpu_barrier_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout);
/* The reference's own two-step form of the barrier gradient (Optimizer.cpp:3492-3502), for a caller that keeps that code unchanged:
 *   evaluateConstraints (:64-81): val[c] = squared distance of active pair c (n = size of the active set on this context);
 *   leftMultiplyConstraintJacobianT (:84-148): g_inout += coef * mult_c * input[c] * grad d_c  (input = b'(d) in the reference);
 *   augmentParaEEGradient (:2990-3045): the mollified pairs' term.
 * ipcgpu_barrier_gradient = the three fused (b' evaluated on the device). */
int ipcgpu_evaluate_constraints(ipcgpu_ctx* ctx, double* val, int n);
int ipcgpu_constraint_jacobian_t(ipcgpu_ctx* ctx, const double* input, int n, double coef, double* g_inout);
int ipcgpu_para_ee_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout);
/* CSR += makePD(kappa*mult*(b'' grad d grad d^T + b' hess d))  (augmentIPHessian :418-561, augmentParaEEHessian :3049-3201) */
int ipcgpu_barrier_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout);

/* ---- lagged friction of the self-contact pairs (SelfCollisionHandler.hpp: computeDistCoordAndTanBasis, computeFrictionEnergy,
 * augmentFrictionGradient, augmentFrictionHessian; SelfCollisionHandler.cpp:2481-2987; FrictionUtils.hpp; C1 clamping, Types.hpp:42) ------ */
/* result.V_prev: the positions at the start of the time step, against which the tangential slip is measured (Optimizer.cpp:3371).
 * NULL = take the current device-resident state. */
int ipcgpu_set_prev_state(ipcgpu_ctx* ctx, const double* V_prev_soa);
/* The friction update of Optimizer.cpp:1582-1600: snapshots the active set of the last ipcgpu_constraint_set (MMActiveSet_lastH) and
 * computes at the current positions lambda_c = -kappa b'(d_c) 2 sqrt(d_c) * multiplicity (MMLambda_lastH), the closest-point coordinates
 * (MMDistCoord) and the tangent bases (MMTanBasis) -- computeDistCoordAndTanBasis, a serial loop in the reference.  Everything stays on the
 * device; n_pairs (may be NULL: no synchronisation) receives the size of the lagged set. */
int ipcgpu_friction_lag(ipcgpu_ctx* ctx, double dHat, double kappa, int* n_pairs);
/* copies of the lagged data, for a caller that keeps the reference's containers (any pointer may be NULL): MMCVID x 4 ints, lambda,
 * Vector2d coordinates, Matrix<double,3,2> bases column-major (6 doubles) */
int ipcgpu_get_friction_data(ipcgpu_ctx* ctx, int* n_pairs, int* mmcvid4, double* lambda, double* coord2, double* basis6);
/* upload host-held lagged data instead (drop-in use of only the three evaluators below with the reference's own containers) */
int ipcgpu_set_friction_data(ipcgpu_ctx* ctx, int n_pairs, const int* mmcvid4, const double* lambda, const double* coord2, const double* basis6);
/* computeFrictionEnergy (:2529-2596): coef * sum_c lambda_c f0(|u_c|), u_c = tangential slip since V_prev; eps2 = fricDHat, coef = selfFric */
int ipcgpu_friction_energy(ipcgpu_ctx* ctx, double eps2, double coef, double* E);
/* augmentFrictionGradient (:2598-2735): g += coef lambda_c f1(|u|)/|u| T^T u.  g_inout NULL = the device-resident gradient */
int ipcgpu_friction_gradient(ipcgpu_ctx* ctx, double eps2, double coef, double* g_inout);
/* augmentFrictionHessian (:2745-2987): CSR += makePD(T^T S T) per pair; a_inout as in ipcgpu_barrier_hessian */
int ipcgpu_friction_hessian(ipcgpu_ctx* ctx, double eps2, double coef, int projectDBC, double* a_inout);

/* ---- inertia term of Optimizer::computeEnergyVal / computeGradient (Optimizer.cpp:3227-3239, :3439-3450); the mass diagonal is the one of
 * ipcgpu_set_mesh (also added to the Hessian diagonal by ipcgpu_elastic_grad_hess(add_mass), :3638-3668) ----------------------------- */
int ipcgpu_set_xtilde(ipcgpu_ctx* ctx, const double* xtilde_soa);
/* sum_v |x_v - xtilde_v|^2 m_v / 2 */
int ipcgpu_inertia_energy(ipcgpu_ctx* ctx, double* E);
/* g_v += m_v (x_v - xtilde_v) for every vertex that is not a projected Dirichlet vertex; g_inout NULL = the device-resident gradient */
int ipcgpu_inertia_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout);

/* ---- time integration: the frame of a time step around its Newton iterations (DESIGN.md section 3.14, INTEGRATION.md section 10) -------------
 * Per-vertex kernels over every vertex, obstacle tail included; "Dirichlet" is Mesh::isDBCVertex (dbc_type != 0).  Every expression keeps the
 * reference's evaluation order and rounding (no fused multiply-add).  No communication: every rank holds all vertices, so the calls work at any
 * rank count, except the warm start (single rank). */
/* Optimizer::setTime (Optimizer.cpp:421-428) and Config's time-integration tokens: type 0 = TIT_BE, 1 = TIT_NM (beta, gamma: Config.hpp:96).
 * Held in device memory: a replayed graph uses the current values, so changing dt needs no new capture. */
int ipcgpu_set_time_integration(ipcgpu_ctx* ctx, int type, double dt, double beta, double gamma, const double gravity[3]);
/* Optimizer's dynamic state (:175-177, restart :203-230): velocity 3nV interleaved, acceleration and dx_Elastic nV x 3 SoA; NULL = zero */
int ipcgpu_set_dynamics(ipcgpu_ctx* ctx, const double* velocity, const double* acceleration_soa, const double* dx_elastic_soa);
int ipcgpu_get_dynamics(ipcgpu_ctx* ctx, double* velocity, double* acceleration_soa, double* dx_elastic_soa); /* any NULL skipped; synchronises */
/* computeXTilta (:1236-1278) from V_prev (ipcgpu_set_prev_state) and the dynamic state, into the x~ the inertia term reads.  Capturable. */
int ipcgpu_compute_xtilde(ipcgpu_ctx* ctx);
/* end of a time step (:572-590): dx_Elastic, velocity, acceleration, V_prev = V, x~.  Capturable. */
int ipcgpu_end_time_step(ipcgpu_ctx* ctx);
/* initX(option) (:925-1233) for option 0-4: the predictor becomes the search direction (mean |p| of the swept build: the fixed-order device sum
 * of a direction adopted on the device, as ipcgpu_solve_pcg's).  Option 0: p = 0, nothing moves, the step is 0.  Options >= 1: from step 1,
 * the inversion filter (Neo-Hookean meshes), the planes' step with slackness 0.9, the swept hash with voxel_size (avgEdgeLen / 3) and the full
 * Tight-Inclusion CCD; V0 := V into the saved state, V = V0 + alpha p; while a tet is inverted (Neo-Hookean), alpha /= 2; while not
 * intersection-free (isIntersected, :2627-2659), alpha /= 2.  A bound of 0 is not an error (the reference only logs it, :1186-1188); an entry
 * state that fails a check at step 0 gives IPCGPU_ERR_LINE_SEARCH with V = V0.  Results: the stage steps in ipcgpu_iteration (alpha_inversion,
 * alpha_halfspace, alpha_swept_grid, alpha_full_ccd), the accepted step as the device-resident step, the halvings and the status in
 * ipcgpu_step_control (alpha_feasible = alpha = the accepted step).  alpha_out NULL: deferred and capturable (conditional nodes; run it once
 * outside a capture first); otherwise synchronises and returns the accepted step.  Option 5 or out of range: IPCGPU_ERR_ARG.  Single rank. */
int ipcgpu_warm_start(ipcgpu_ctx* ctx, int option, double voxel_size, double tolerance, const double err_vf[3], const double err_ee[3], double* alpha_out);

/* ---- Rayleigh damping, Neumann forces and the augmented-Lagrangian Dirichlet penalty: the last terms of Optimizer::computeEnergyVal /
 * computeGradient / computePrecondMtr (DESIGN.md section 3.13, INTEGRATION.md section 9) ------------------------------------------------
 * Conventions as everywhere: a NULL output is deferred and capturable (energies: ipcgpu_fetch_iteration), the NULL gradient / Hessian forms run
 * on the derivative chain, a host output synchronises.  New VALUES -- D rebuilt at the next time step, forces, targets, multipliers, rho --
 * need no new capture; switching a term on or off (and a new number of Dirichlet targets) refuses older graphs, because the line search bakes
 * its set of terms in.  ipcgpu_line_search includes every term that is set.  Single rank: IPCGPU_ERR_STATE with several.  A new mesh removes
 * all three. */
/* computeDampingMtr (Optimizer.cpp:3723-3734, called at the end of every time step, :593-595) at the current state:
 * D = coef sum_t makePD(H_t) with projectDBC = 1, coef = energyParams[0] dampingStiff / dt; coef = 0 removes the term.  D is held in the mesh's
 * vertex-pair order, independent of the system's sparsity pattern.  As in the reference (IglUtils.hpp:45-52, setCoeff), D holds the IDENTITY on
 * the diagonal of every Dirichlet vertex of a tet: the system matrix gets 2.0 there (identity + D), and in penalty mode (projectDBC = 0) D d adds
 * x_v - x_prev,v to a Dirichlet vertex's gradient rows.  The first call on a mesh builds a per-vertex slot list (synchronises; not in a capture). */
int ipcgpu_damping_update(ipcgpu_ctx* ctx, double coef);
/* 1/2 d^T D d, d = V - V_prev (ipcgpu_set_prev_state) with every Dirichlet row zeroed (:3381-3400) */
int ipcgpu_damping_energy(ipcgpu_ctx* ctx, double* E);
/* g += D d with the rows of isProjectDBCVertex(v, projectDBC) zeroed in d (:3519-3540); g_inout as in ipcgpu_barrier_gradient */
int ipcgpu_damping_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout);
/* addCoeff(dampingMtr, 1.0) (:3707-3709); a_inout as in ipcgpu_barrier_hessian */
int ipcgpu_damping_hessian(ipcgpu_ctx* ctx, double* a_inout);
/* Neumann forces (:3241-3250, :3452-3461): f (3nV interleaved) = per vertex, the summed force of the NBCs that are active (the scripter's
 * isNBCActive) and contain it; coef = dt^2; f = NULL removes the term.  Dirichlet vertices are skipped whatever projectDBC is. */
int ipcgpu_set_neumann_forces(ipcgpu_ctx* ctx, double coef, const double* f);
/* -sum_v coef m_v x_v . f_v */
int ipcgpu_neumann_energy(ipcgpu_ctx* ctx, double* E);
/* g_v -= coef m_v f_v */
int ipcgpu_neumann_gradient(ipcgpu_ctx* ctx, double* g_inout);
/* AnimScripter::targetPos (AnimScripter.cpp:2151-2158): n targets, vertex vid[i] (distinct, as the keys of the reference's map; a repeated
 * vertex is IPCGPU_ERR_ARG), target position target[3i..3i+2], multiplier lambda[3i..3i+2] (NULL = 0), dist2Tol (:2158, recomputed every time
 * step; held in device memory like the targets); n = 0 removes the term */
int ipcgpu_set_dirichlet_targets(ipcgpu_ctx* ctx, int n, const int* vid, const double* target, const double* lambda, double dist2Tol);
/* rho_DBC, held in device memory and set in stream order (changing it between replays needs no new capture); rho = 0 adds nothing at all */
int ipcgpu_set_dirichlet_penalty(ipcgpu_ctx* ctx, double rho);
/* copy of the multipliers (3n doubles), for a binding that keeps the reference's targetPos next to the device copy; synchronises */
int ipcgpu_get_dirichlet_lambda(ipcgpu_ctx* ctx, double* lambda);
/* augmentMDBCEnergy / Gradient / Hessian (AnimScripter.cpp:2303-2336): sum_i rho/2 m |x - t|^2 - sqrt(m) lambda . (x - t); the gradient and the
 * Hessian (rho m on the vertex's diagonal) apply only when !projectDBC (Optimizer.cpp:3542, :3711); all three add nothing while rho = 0 */
int ipcgpu_dirichlet_energy(ipcgpu_ctx* ctx, double* E);
int ipcgpu_dirichlet_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout);
int ipcgpu_dirichlet_hessian(ipcgpu_ctx* ctx, int projectDBC, double* a_inout);
/* updateLambda (:2338-2345): lambda_i -= rho sqrt(m) (x - t), on the device (capturable) */
int ipcgpu_dirichlet_update_lambda(ipcgpu_ctx* ctx);
/* computeCompletedStepSize (:2286-2300): 1 - sqrt(sum |x - t|^2 / (dist2Tol 1e6)), 1 when dist2Tol = 0.  s NULL: deferred to the fetch */
int ipcgpu_dirichlet_completed_step(ipcgpu_ctx* ctx, double* s);

/* ---- line-search safeguards (Optimizer.cpp:2709-2733, 2799-2811), so that a line-search trial -- step forward, checks, constraint set,
 * energies -- is one stream ------------------------------------------------------------------------------------------------------ */
/* Mesh::checkInversion(mute) (Mesh.cpp:715-763): number of tets with mu, lambda != 0 whose current edge matrix has det < 0 (0 = no
 * inversion).  NULL: deferred, reported by ipcgpu_fetch_iteration. */
int ipcgpu_check_inversion(ipcgpu_ctx* ctx, int* n_inverted);
/* SelfCollisionHandler::checkEdgeTriIntersectionIfAny (SelfCollisionHandler.cpp:3254-3337) with the hash query of
 * SpatialHash::queryTriangleForEdges done on the device: *ok = 1 iff no surface edge crosses a surface triangle (exact orient3d +
 * the reference's full-pivot solve, IglUtils.hpp:214-265) AND no codimension-0 vertex (vCoDim == 0 in ipcgpu_set_surface) lies in a
 * tetrahedron (IglUtils::pointInsideTetrahedron, IglUtils.hpp:276-294: four exact orientations, a point on a face, an edge or a vertex is
 * inside; every tet, no Dirichlet or Lame filter).  Rebuilds the static grid, and the grid of the codimension-0 vertices, at the current
 * positions; without codimension-0 vertices the second test launches nothing.  With several ranks each rank tests its own triangles and
 * tets.  NULL: deferred, reported by ipcgpu_fetch_iteration. */
int ipcgpu_intersection_free(ipcgpu_ctx* ctx, int* ok);
/* TEST HOOK.  enable != 0: every later ipcgpu_intersection_free also writes, on the device, a flag per surface triangle (1 = an edge crosses
 * it) and the number of codimension-0 vertices inside each tetrahedron; enable = 0 frees those buffers and leaves the check as it was (the
 * same launches).  tri_flags (nSF) and tet_hits (nT), nullable, receive the last check's values after a synchronisation; they need the
 * hook on, and are read before `enable` is applied. */
int ipcgpu_safeguard_debug_flags(ipcgpu_ctx* ctx, int enable, int* tri_flags, int* tet_hits);

/* ---- CCD step bound (Tight-Inclusion), Optimizer.cpp:1884-2040 ----------------------------------------------------- */
/* capacity (pairs) of the device CCD candidate list; default 2^23 */
int ipcgpu_set_ccd_capacity(ipcgpu_ctx* ctx, uint64_t capacity);
/* scene-wide Tight-Inclusion numerical error (computeTightInclusionError, CCDUtils.cpp:55-87): world bbox of V inflated to centre +-
 * 10*radius*(1,1,1)/sqrt(3) (computeConservativeWorldBBox, :21-52, uses mesh.V only: pass p = NULL for the reference's value; a non-NULL
 * p widens the box by V+p, an extension), then inclusion_ccd::get_numerical_error(..., use_ms = true). Host-only. */
int ipcgpu_ti_error(const double* V_soa, int nV, const double* p_interleaved /* may be NULL */, double err_vf[3], double err_ee[3]);
/* largestFeasibleStepSize_TightInclusion (SelfCollisionHandler.cpp:690-866) over the candidate list cs_PTEE of the last
 * ipcgpu_constraint_set(getPTEE=1).  alpha_inout: step on entry (max_t of every pair) -> min(alpha, earliest time of impact);
 * NULL = the device-resident step (no synchronisation). */
int ipcgpu_ccd_partial_ti(ipcgpu_ctx* ctx, const double* p_interleaved /* NULL = last uploaded */, double tolerance,
    const double err_vf[3], const double err_ee[3], double* alpha_inout);
/* SpatialHash::build(mesh, searchDir, curMaxStepSize, voxelSize) (SpatialHash.hpp:589-750): alpha_inout is scaled down when
 * spanSize = alpha*mean|p|/h > 1 exactly like the reference (:603-618). */
int ipcgpu_hash_build_swept(ipcgpu_ctx* ctx, const double* p_interleaved /* NULL = last uploaded */, double* alpha_inout, double voxel_size);
/* largestFeasibleStepSize_CCD_TightInclusion (SelfCollisionHandler.cpp:1370-1630) over the candidates of the swept hash.
 * n_candidates (may be NULL) receives the number of PT+EE pairs sent to the narrow phase. */
int ipcgpu_ccd_full_ti(ipcgpu_ctx* ctx, double tolerance, const double err_vf[3], const double err_ee[3], double* alpha_inout, uint64_t* n_candidates);

/* ---- step control: the CFL branch of the step bound and the line search (DESIGN.md section 3.11, INTEGRATION.md section 4) ---------------
 * Both run their data-dependent decisions on the device.  Inside ipcgpu_capture_begin / _end they become conditional graph nodes (CUDA 12.4
 * or newer; IPCGPU_ERR_CUDA without driver support) and nothing synchronises.  OUTSIDE a capture the host drives the loops and reads each
 * decision back: one synchronisation per decision, also with alpha_inout == NULL (the one exception to "NULL outputs never synchronise"; it is
 * also the eager run that makes the lazy allocations before a capture).  Single rank only (IPCGPU_ERR_STATE with several). */
/* CFL_FOR_CCD == 2 (Optimizer.cpp:1947-2027; src/Utils/Types.hpp:34).  Call it after ipcgpu_ccd_partial_ti, in place of
 * ipcgpu_hash_build_swept + ipcgpu_ccd_full_ti: alpha_CFL = sqrt(dHat) / (2 max_i |p_SVI[i]|) over the mesh's surface vertices (inf for p = 0);
 * if (first_iteration && alpha > alpha_CFL) || alpha > 2 alpha_CFL: swept hash + full CCD, then alpha = max(alpha, alpha_CFL); otherwise
 * alpha = min(alpha, alpha_CFL) (the swept-grid and full-CCD stages of ipcgpu_iteration then report that step).  A zero step raises
 * IPCGPU_ERR_LINE_SEARCH (ipcgpu_step_control_info; returned directly by the host-output form). */
int ipcgpu_ccd_cfl_ti(ipcgpu_ctx* ctx, double dHat, int first_iteration, double voxel_size, double tolerance, const double err_vf[3], const double err_ee[3],
    double* alpha_inout /* NULL: device-resident step */);
/* the energy of a line-search trial, ((E_el + E_in) + E_b) + E_f in the order of Optimizer::computeEnergyVal (Optimizer.cpp:3199-3378); the
 * half-space, damping, Neumann and Dirichlet-penalty terms join it whenever they are set on the context (DESIGN.md section 3.13) */
typedef struct ipcgpu_line_search_terms {
    double elastic_coef;          /* dt^2 * energyParams[0] (BE) or dt^2 * beta_NM * energyParams[0] */
    int    inertia;               /* != 0: + sum m|x - xtilde|^2 / 2 (ipcgpu_set_xtilde) */
    double dHat, kappa;           /* + kappa * sum b(d) over the sets rebuilt at every trial */
    double fric_eps2, fric_coef;  /* fric_coef > 0: + friction energy of the lagged set (ipcgpu_friction_lag) */
} ipcgpu_line_search_terms;
/* Optimizer::lineSearch (Optimizer.cpp:2662-2916) with armijoParam = 0 and lowerBound = 0, the only values the reference passes (:2059, :2614),
 * from the device-resident step (alpha_inout == NULL) or *alpha_inout, along the search direction held (ipcgpu_set_search_dir / ipcgpu_solve_pcg).
 *   V0 := V into the saved state (this OVERWRITES what ipcgpu_save_state saved), E0 := E(V) with the contact sets held;
 *   V = V0 + alpha p; Neo-Hookean meshes only: while a tet is inverted, alpha /= 2 and step again (:2710-2715);
 *   while not intersection-free, alpha /= 2 and step again (:2720-2733);  constraint set (getPTEE = 1), E_t = E(V);
 *   while E_t > E0: alpha /= 2 (alpha == 0: stopped), step, constraint set, E_t = E(V) (:2761-2797);
 *   if alpha dropped: while not intersection-free, alpha /= 2 and step, then the constraint set again if that loop ran (:2799-2811).
 * The accepted step becomes the device-resident step (ipcgpu_fetch_iteration().alpha).  An entry step of 0 runs nothing; every loop also ends
 * at alpha == 0 and then reports IPCGPU_ERR_LINE_SEARCH with V = V0; d <= 0 in a trial ends the search with IPCGPU_ERR_NONPOSITIVE_DISTANCE.
 * Results: ipcgpu_step_control_info; the host-output form returns the status directly.  Inside a capture the contact lists must be in
 * arbitrary order (ipcgpu_set_canonical_order(ctx, 0)). */
int ipcgpu_line_search(ipcgpu_ctx* ctx, const ipcgpu_line_search_terms* terms, double* alpha_inout);
typedef struct ipcgpu_step_control {
    double alpha_cfl;             /* last ipcgpu_ccd_cfl_ti */
    double alpha_feasible;        /* last line search: the step after the inversion guard and the intersection pre-check (LFStepSize, :2750) */
    double alpha;                 /* ... the accepted step */
    double energy_start, energy;  /* ... E0 and E_t of the last trial (lastEnergyVal, :2898) */
    int full_ccd;                 /* last ipcgpu_ccd_cfl_ti took the full CCD */
    int stopped;                  /* the Armijo loop halved the step to 0 (lineSearch's return value) */
    int halvings_inversion, halvings_intersection, halvings_armijo, halvings_post_check;
    int post_check_rebuilt;       /* the post-check halved the step and the constraint set was rebuilt */
    int status;                   /* IPCGPU_OK, IPCGPU_ERR_LINE_SEARCH or IPCGPU_ERR_NONPOSITIVE_DISTANCE */
} ipcgpu_step_control;
/* synchronises only when a CFL branch or a line search was enqueued since the last read; returns out->status */
int ipcgpu_step_control_info(ipcgpu_ctx* ctx, ipcgpu_step_control* out);

/* ---- kinematic mesh obstacle: MeshCO<3> (src/CollisionObject/MeshCO.hpp:39-233; SURVEY 8 row f3, barrier / Tight-Inclusion path) --------------------
 * An obstacle is a triangle mesh without degrees of freedom (MeshCO's Base::V, edges, Base::F).  It rides at the TAIL of the mesh's arrays: the
 * caller appends the obstacle's vertices to the vertex arrays of ipcgpu_set_mesh (rest = current positions, Dirichlet flag 1, mass 0, no
 * tetrahedron uses them) and its vertices / edges / triangles, re-indexed, to the arrays of ipcgpu_set_surface, then names the first obstacle
 * vertex here.  From then on the contact stages -- ipcgpu_contact_constraint_set, barrier energy / gradient / Hessian, evaluate_constraints,
 * J^T, partial and full CCD, ipcgpu_intersection_free -- cover the mesh against itself AND the mesh against the obstacle:
 *   - pairs of the mesh with the obstacle follow MeshCO.cpp: no Dirichlet / codimension filter (MeshCO.cpp:1795-2100), a mesh vertex and an
 *     obstacle vertex closest to each other form ONE point-point entry however they were found (:1831, :1919, :2168-2190), the full pair
 *     stencil is differentiated and projected (makePD of the 6x6 / 9x9 / 12x12 block, :430-560) and only the mesh vertices' rows and columns
 *     are scattered (the obstacle's rows are Dirichlet rows of the system: identity);  pairs inside the obstacle do not exist;
 *   - entries are reported in the self-contact encoding over the merged numbering (an obstacle vertex k is vertex first_obstacle_vertex + k);
 *     adapters/IpcGpuAdapters.hpp splits them into the SelfCollisionHandler's and MeshCO's own MMCVID lists;
 *   - step bounds: one minimum over both kinds of pairs (the reference takes MeshCO's bound, then the self-contact bound, each with the
 *     running step as max_t: the same minimum).  ee_through_vf_routine != 0 (what the reference does, MeshCO.cpp:900-940 and :1609-1655):
 *     Tight-Inclusion evaluates a mesh-edge / obstacle-edge pair with vertexFaceCCD_double on the four points in edge order, edge-edge error
 *     bound and initial distance; 0: with edgeEdgeCCD_double.
 * Everything sized by the vertex count (positions, search direction, gradient, CSR rows) includes the tail: the obstacle's search direction is
 * zero, its gradient rows are Dirichlet rows (whatever the barrier terms add there is discarded with them), its CSR rows hold the identity; because the tail's rows come last and no mesh row has a column in them,
 * the mesh's own upper-triangular CSR values are a PREFIX of the value array.  first_obstacle_vertex < 0 or >= nV removes the obstacle.
 * Friction: the reference implements none against a MeshCO (CollisionObject.h:403-423 throw "not implemented"); ipcgpu_friction_lag lags the pairs
 * that touch the obstacle with a zero normal force, so the friction terms stay those of the mesh's own pairs.  Not covered: the CTCD variants, SQP, and scenes that switch self contact off (Config.cpp:480
 * `selfCollisionOff`) while keeping an obstacle: the mesh's own pairs are always part of the pass. */
int ipcgpu_set_obstacle_tail(ipcgpu_ctx* ctx, int first_obstacle_vertex, int ee_through_vf_routine);
/* MeshCO::move / Base::V after a scripted motion: new positions of the obstacle's vertices, SoA [x | y | z] over the obstacle's own count;
 * current and rest positions of the tail are both replaced (an obstacle has no rest shape: compute_eps_x(mesh, Base::V, ...) uses its current
 * edge lengths, MeshCollisionUtils.hpp:2976-2981).  The state saved by ipcgpu_save_state keeps the tail it was saved with: move the obstacle between
 * line searches (as the reference does, Optimizer.cpp: the scripted motion runs before the Newton loop of a time step) or save the state again. */
int ipcgpu_set_obstacle_positions(ipcgpu_ctx* ctx, const double* Vo_soa);

/* ---- analytic half-space collision objects: HalfSpace<3> (src/CollisionObject/HalfSpace.cpp, CollisionObject.h; script tokens `ground` /
 * `halfSpace`, Config.cpp:425-447; DESIGN.md section 3.12, INTEGRATION.md section 8) ----------------------------------------------------------
 * Entries are (plane, vertex) pairs.  Every call below has a NULL-output form that is deferred and capturable; the parameters of the planes live
 * in device memory, so moving a plane between time steps (new origin / velocitydt: the caller's HalfSpace::move) needs no new capture -- only a
 * change of their number does.  Without planes (n = 0) every call returns at once and launches nothing.  Several ranks: the active set, the
 * lagged set and the step bound are replicated (each rank walks all of SVI: no collective); gradient and Hessian rows, energies and crossing
 * counts go by row owner (the counts and energies are summed by ipcgpu_fetch_iteration's single collective). */
/* HalfSpace::init (HalfSpace.cpp:42-52) for up to 8 planes: normal normalised, D = -n.origin; velocitydt (3n, NULL = 0) and friction per plane.
 * The ground token is origin (0, y, 0), normal (0, 1, 0).  n = 0 removes all planes. */
int ipcgpu_set_halfspaces(ipcgpu_ctx* ctx, int n, const double* origin, const double* normal, const double* velocitydt, const double* friction);
/* CollisionObject::computeConstraintSet (CollisionObject.h:323-352) of every plane in one pass: SVI vertices, not Dirichlet, codimension 3,
 * d = (n.x + D)^2 < dHat; plane-major, SVI order inside a plane (activeSet[coI] over coI).  n_active NULL: deferred. */
int ipcgpu_halfspace_constraint_set(ipcgpu_ctx* ctx, double dHat, int* n_active);
/* kappa sum b(d) (Optimizer.cpp:3254-3267); d <= 0 raises IPCGPU_ERR_NONPOSITIVE_DISTANCE as ipcgpu_barrier_energy does */
int ipcgpu_halfspace_energy(ipcgpu_ctx* ctx, double dHat, double kappa, double* E);
/* HalfSpace::leftMultiplyConstraintJacobianT (HalfSpace.cpp:121-143) with input b'(d) (Optimizer.cpp:3465-3472): g += kappa b'(d) 2 dist n.
 * g_inout as in ipcgpu_barrier_gradient; the NULL form runs on the derivative chain */
int ipcgpu_halfspace_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout);
/* HalfSpace::augmentIPHessian (HalfSpace.cpp:169-213): the vertex's diagonal block += kappa param n n^T where param = 4 b'' d + 2 b' > 0;
 * a_inout as in ipcgpu_barrier_hessian */
int ipcgpu_halfspace_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout);
/* HalfSpace::largestFeasibleStepSize (HalfSpace.cpp:242-269; slackness_a = 0.9 at Optimizer.cpp:1886-1890, after the inversion filter, before the
 * partial CCD): alpha = min(alpha, 1, -dist / (n.p) slackness over the non-Dirichlet SVI vertices with n.p < 0).  A bound <= 0 stores step 0
 * and reports IPCGPU_ERR_LINE_SEARCH (returned by the host form, else by ipcgpu_fetch_iteration).  p NULL: the held search direction;
 * alpha_inout NULL: the device-resident step (step-bound chain). */
int ipcgpu_halfspace_step(ipcgpu_ctx* ctx, const double* p_interleaved, double slackness, double* alpha_inout);
/* CollisionObject::isIntersected (CollisionObject.h:386-401): number of (plane, vertex) with d <= 0 over every codimension-3, non-Dirichlet
 * vertex.  The test is on the SQUARED distance, as in the reference: a vertex that tunnelled behind a plane is not counted.  n NULL: deferred. */
int ipcgpu_halfspace_crossings(ipcgpu_ctx* ctx, int* n);
/* the friction update of Optimizer.cpp:1555-1572: the active entries of the planes with friction > 0 become the lagged set, with
 * lambda = -kappa 2 sqrt(d) b'(d).  n_lagged NULL: deferred. */
int ipcgpu_halfspace_friction_lag(ipcgpu_ctx* ctx, double dHat, double kappa, int* n_lagged);
/* HalfSpace::computeFrictionEnergy / augmentFrictionGradient / augmentFrictionHessian (HalfSpace.cpp:272-380, coef 1.0 as Optimizer.cpp:3361
 * passes it) against result.V_prev (ipcgpu_set_prev_state); eps2 = fricDHat.  Outputs as in the barrier calls above. */
int ipcgpu_halfspace_friction_energy(ipcgpu_ctx* ctx, double eps2, double* E);
int ipcgpu_halfspace_friction_gradient(ipcgpu_ctx* ctx, double eps2, double* g_inout);
int ipcgpu_halfspace_friction_hessian(ipcgpu_ctx* ctx, double eps2, int projectDBC, double* a_inout);
/* copies of the active set (plane, vertex interleaved), the lagged set and its lambda (activeSet / activeSet_lastH / lambda_lastH, split by
 * plane); any pointer may be NULL (call once with NULL arrays for the sizes) */
int ipcgpu_get_halfspace_sets(ipcgpu_ctx* ctx, int* n_active, int* active2, int* n_lagged, int* lagged2, double* lambda);

/* diagnostics of the last narrow phase: candidates tested, pairs surviving the root box, conservative early-outs (should be 0) */
int ipcgpu_ccd_stats(ipcgpu_ctx* ctx, uint64_t* candidates, uint64_t* survivors, uint64_t* warnings);
/* more diagnostics: pairs handed from the thread-level to the warp-level pass, parameter boxes evaluated by each pass */
int ipcgpu_ccd_stats_ex(ipcgpu_ctx* ctx, uint64_t* deferred, uint64_t* boxes_thread_pass, uint64_t* boxes_warp_pass);
/* critical path of the warp-level pass: SM cycles spent on its longest single pair, and summed over all its pairs */
int ipcgpu_ccd_stats_timing(ipcgpu_ctx* ctx, uint64_t* longest_pair_cycles, uint64_t* total_pair_cycles);
/* TEST HOOK.  Pairs prune their interval search against the earliest impact any pair has reported so far -- which pair reports first
 * depends on scheduling.  toi >= 0 makes every later narrow phase start as if some pair had already reported `toi` (the step on entry,
 * i.e. max_t of every pair, is unchanged; the result is min(toi, the pairs' impacts)); toi < 0 switches the hook off. */
int ipcgpu_ccd_debug_seed_bound(ipcgpu_ctx* ctx, double toi);
/* TEST HOOK.  boxes >= 0: a thread may evaluate this many boxes of a search in the thread-level pass before it hands the pair on to the
 * warp-level pass, in every later narrow phase of this context (0 hands on every search that does not end at its root box); boxes < 0
 * restores the default, 32.  The step bound does not depend on it. */
int ipcgpu_ccd_debug_thread_budget(ipcgpu_ctx* ctx, int64_t boxes);

/* ---- linear-solve hand-off with the Hessian resident in HBM (LinSysSolver::factorize/solve, LinSysSolver.hpp:230-236; Optimizer.cpp:2324-2355) ----
 * The production binding is a sparse Cholesky on the device arrays (cuDSS: INTEGRATION.md; ipcgpu_device_ptr / the ia, ja uploaded by
 * ipcgpu_set_csr).  What this library itself provides is the hand-off and a reference solver that never leaves the device: block-Jacobi
 * preconditioned CG on the upper-triangular CSR.  rhs == NULL solves H p = -g with the device-resident gradient; x == NULL keeps the
 * solution on the device; adopt_as_search_dir != 0 makes it the search direction of the step-bound stages (as if uploaded by
 * ipcgpu_set_search_dir; mean|p| of SpatialHash.hpp:603-612 is then a fixed-order device sum).  Single rank.
 * iters / rel_residual (nullable) report the iteration count and |r| / |b|. */
int ipcgpu_solve_pcg(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual);
/* The same Krylov method and the same contract as ipcgpu_solve_pcg (rhs == NULL: H p = -g on the resident gradient; x == NULL: the solution
 * stays on the device; adopt_as_search_dir; iters / rel_residual nullable; single rank), preconditioned by a multilevel additive Schwarz
 * hierarchy (Wu, Wang, Wang 2022) rebuilt from the resident matrix and the current positions at every call: vertices in the Morton order
 * of their positions (obstacle tail included), domains of 32 vertices at level 0 and of 32 aggregates of 32^l vertices at level l, every
 * domain matrix (96 x 96, piecewise-constant translations as coarse space) inverted and stored dense, z = sum_l P_l^T A_l^-1 P_l r.  Every
 * sum is taken in a fixed order: two calls on the same state return identical bits.  Memory: 73,728 bytes per domain, about 2.4 KB per
 * vertex, kept for the life of the context.  Dirichlet vertices (the dbc flags of ipcgpu_set_mesh) and the obstacle tail are left out of the
 * coarse levels: with a zero right-hand side on their identity rows their solution entries are exactly 0.  A domain matrix with a pivot <= 0 (the matrix is not positive definite) returns IPCGPU_ERR_SOLVE; nothing is NaN and nothing hangs. */
int ipcgpu_solve_pcg_multilevel(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters,
    double* rel_residual);
/* what the last multilevel solve built: number of levels, domains per level (8 entries, 0 beyond the last level), bytes of the stored
 * inverses; any pointer may be NULL.  IPCGPU_ERR_STATE before the first ipcgpu_solve_pcg_multilevel and after one that failed. */
int ipcgpu_multilevel_info(ipcgpu_ctx* ctx, int* levels, int64_t* domains_per_level, uint64_t* bytes);
/* TEST HOOK.  The level matrices of the hierarchy (96*96 doubles per domain, level after level, as IPCGPU_BUF_MULTILEVEL_INVERSES) assembled
 * again from the resident matrix and the current positions and copied out before any inversion.  It overwrites the stored inverses: the
 * hierarchy counts as not built until the next ipcgpu_solve_pcg_multilevel.  count: 96*96 times the domains of ipcgpu_multilevel_info. */
int ipcgpu_multilevel_debug_matrices(ipcgpu_ctx* ctx, double* dst, uint64_t count);
/* LinSysSolver::setZero (LinSysSolver.hpp:348) on the device-resident value array */
int ipcgpu_csr_set_zero(ipcgpu_ctx* ctx);
/* cross-rank completion over NVLink (no-op on a single rank).  with_gradient: sum-allreduce of the gradient (needed every iteration).
 * with_hessian: only for a caller that wants the WHOLE matrix on every rank -- each rank's own rows are complete without it (row-owner
 * assembly); it ships the other ranks' rows (a sum over arrays that are zero outside the owned rows). */
int ipcgpu_allreduce_grad_hess(ipcgpu_ctx* ctx, int with_gradient, int with_hessian);
int ipcgpu_download(ipcgpu_ctx* ctx, int which, double* dst, uint64_t count);
/* count entries starting at `offset` (e.g. the CSR values of the rows this rank owns: ipcgpu_partition_info) */
int ipcgpu_download_range(ipcgpu_ctx* ctx, int which, uint64_t offset, uint64_t count, double* dst);
/* The same without waiting: the copy is forked onto the context's copy stream behind everything enqueued so far and runs next to whatever
 * the main stream does afterwards (a host solver wants the Hessian, the step-bound stages that follow do not touch it).  dst must be pinned
 * (ipcgpu_host_alloc) and must not be read before the next ipcgpu_fetch_iteration / ipcgpu_sync, which join the copy stream.  May be
 * captured into a graph (call it once outside a capture first). */
int ipcgpu_download_range_async(ipcgpu_ctx* ctx, int which, uint64_t offset, uint64_t count, double* dst_pinned);
/* raw device pointer of a result buffer (for a device-side linear solver) */
void* ipcgpu_device_ptr(ipcgpu_ctx* ctx, int which);

/* ---- device-side timing (CUDA events on the context's own stream; bench.py's roofline numbers) ---------- */
enum {
    IPCGPU_STAGE_ELASTIC_ENERGY = 0,
    IPCGPU_STAGE_ELASTIC_TET = 1,     /* per-tet gradient/Hessian kernel */
    IPCGPU_STAGE_GATHER_GRADIENT = 2,
    IPCGPU_STAGE_ASSEMBLE_CSR = 3,
    IPCGPU_STAGE_INVERSION = 4,
    IPCGPU_STAGE_HASH = 5,
    IPCGPU_STAGE_CONSTRAINT_SET = 6,
    IPCGPU_STAGE_BARRIER = 7,
    IPCGPU_STAGE_CCD_BROAD = 8,
    IPCGPU_STAGE_CCD_NARROW = 9,
    IPCGPU_STAGE_ALLREDUCE = 10,
    IPCGPU_STAGE_CCD_ROOT_FILTER = 11, /* first narrow-phase kernel (root-box inclusion test), nested inside CCD_NARROW */
    IPCGPU_STAGE_DAMPING_BC = 12,     /* damping (D's update, energy, gradient, Hessian), Neumann forces and the Dirichlet penalty */
    IPCGPU_STAGE_COUNT = 13
};
/* enable=1 starts recording an event pair around every stage launch (and clears old records) */
int ipcgpu_profile(ipcgpu_ctx* ctx, int enable);
/* synchronises, then returns the summed device time and launch count of one stage since ipcgpu_profile(ctx,1) */
int ipcgpu_profile_read(ipcgpu_ctx* ctx, int stage, double* total_ms, int* count);
/* whole-region device timer on the context stream */
int ipcgpu_timer_start(ipcgpu_ctx* ctx);
int ipcgpu_timer_stop(ipcgpu_ctx* ctx, double* ms);

#ifdef __cplusplus
}
#endif
#endif
