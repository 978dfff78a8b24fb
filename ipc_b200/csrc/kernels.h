// kernels.h -- launcher declarations shared between the .cu translation units and the C-ABI (api*.cu)
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace ipcgpu {

constexpr int kFlagSlots = 9; // IterState::flags (FLAG_*)

// slots of IterState::energy
enum { kEnergyElastic = 0, kEnergyBarrier, kEnergyFriction, kEnergyInertia, kEnergyPlaneBarrier, kEnergyPlaneFriction, kEnergyDamping, kEnergyNeumann,
    kEnergyDirichlet, kEnergySlots };

// Device-resident scalars of one Newton iteration.  Every stage reads its inputs from here and leaves its outputs here, so a whole
// iteration is one stream of launches (and in-stream NCCL reductions) with a single read-back at the end (ipcgpu_fetch_iteration).
struct IterState {
    unsigned long long step_ord;      // running step-size bound (order-preserving integer image of a non-negative double)
    unsigned long long inv_ord;       // min inversion step over this rank's tets (then over all ranks)
    unsigned long long ccd_ord;       // running minimum of the narrow phase in flight (every pair prunes against it)
    unsigned long long cand_range[2]; // [begin, end) of the candidate list this rank's narrow phase walks
    unsigned long long n_full_cand;   // candidates of the last full CCD (this rank)
    double max_t;                     // step on entry of the narrow phase in flight (max_t of every pair, SURVEY 8a row 10)
    double alpha_grid;                // sweep length of the last swept grid (after the span rescale of SpatialHash.hpp:603-618)
    double ref_lo[3], ref_inv_h;      // reference swept-grid geometry (SpatialHash.hpp:589-640)
    double alpha_stage[4];            // step after: inversion filter, partial CCD, swept-grid rescale, full CCD
    double energy[kEnergySlots];      // kEnergy* slots (this rank's share, then cross-rank sums)
    int ref_count[3];
    int n_set[3];                     // active / mollified / candidate counts of the last constraint set (this rank's lists)
    int flags[kFlagSlots];            // FLAG_* slots (nonzero = raised); cleared by ipcgpu_fetch_iteration
    int grid_axis_cells;              // cells per axis the broad-phase grids built since the last fetch would have liked (sort-width tuning)
    int checks[2];                    // line-search safeguards: inverted tets, surface triangles crossed by an edge (this rank's share, then sums)
    unsigned long long ccd_stats[8];  // survivors, warnings, deferred, longest / total pair cycles, boxes (thread pass, warp pass), candidates
    // step control (step_control.cu): the CFL branch of the step bound and the line search
    unsigned long long sc_pmax_ord;   // max |p| over the mesh's surface vertices
    double sc_alpha_cfl;              // sqrt(dHat) / (2 max |p|)
    double ls_E0, ls_Et, ls_LF;       // energy on entry, energy of the last trial, step after the safeguards (LFStepSize)
    int sc_full_ccd;                  // the CFL branch took the full CCD
    int sc_status;                    // IPCGPU_OK or the IPCGPU_ERR_* code that ended the last CFL branch / line search
    int ls_count[4];                  // halvings: inversion guard, intersection pre-check, Armijo loop, post-check
    int ls_stopped, ls_rebuilt, ls_post_ran;
    int ls_cond;                      // the decision word of the last step_decide
    // linear solve (solve.cu, multilevel.cu): the Krylov loops' state, read with ls_cond by the host loop of an eager solve (kDecisionWords)
    int sv_iters;                     // iterations run by the solve in flight
    int sv_status;                    // IPCGPU_OK or IPCGPU_ERR_SOLVE (a pivot <= 0 of the multilevel set-up, a non-finite residual)
    int sv_run;                       // the loop goes on: the set-up passed, no stop yet
    int sv_max_iter;
    double sv_rr, sv_bb, sv_tol;      // |r|^2 after the last iteration, |b|^2, rel_tol
    unsigned long long sv_xmax_ord;   // max |x_i| of the solution (order-preserving image)
    unsigned long long sv_fp_version; // pat_version the full-row structure (fia / fja / fpos) was built for; ~0 = none
    int sv_fp_build;                  // the full-row build in flight runs (pat_version != sv_fp_version)
    int sv_pad_;
    // Dirichlet penalty and Neumann forces (damping.cu; before the half-space words, which ipcgpu_set_halfspaces clears as one range)
    double dbc_rho;                   // rho_DBC (ipcgpu_set_dirichlet_penalty), read by the penalty kernels at run time
    double dbc_step;                  // the last computeCompletedStepSize
    double dbc_tol;                   // dist2Tol of the targets (ipcgpu_set_dirichlet_targets; 0 without targets), read at run time
    double nbc_coef;                  // dt^2 of the Neumann term (ipcgpu_set_neumann_forces)
    // half-space collision objects (halfspace.cu)
    double hs_alpha;                  // step after the plane bound
    int hs_n_active, hs_n_lagged;     // sizes of the plane active set / lagged set (replicated on every rank)
    int hs_crossings;                 // vertices with d <= 0 of the last crossing check (this rank's share, then sums)
    int hs_zero_step;                 // the plane bound (or the step entering it) was 0; cleared by ipcgpu_fetch_iteration
    // device-built sparsity pattern (pattern.cu): result of the last ipcgpu_update_pattern and its per-update control words
    long long pat_nnz;                // nnz of the pattern in ia / ja
    unsigned long long pat_version;   // bumped by every update that rewrote the pattern
    int pat_changed;                  // the last update rewrote the pattern
    int pat_ok;                       // the raw contact keys of the update in flight fit the key buffer
    int pat_diff;                     // the extra blocks of the update in flight differ from the previous ones
    int pat_pad_;
    // barrier stiffness held on the device (kappa.cu): read by the barrier / plane calls given IPCGPU_KAPPA_DEVICE, adapted by initKappa and
    // postLineSearch's close-pair doubling
    double kappa;                     // kappa
    double kappa_suggest, kappa_max;  // suggestKappa / upperBoundKappa at the current dHat (ipcgpu_set_kappa)
    double kappa_min_last;            // minKappa = -g_c.g_E / |g_c|^2 of the last initKappa (NaN for g_c = 0)
    double kappa_dot[2];              // g_c.g_E and g_c.g_c of the initKappa in flight
    unsigned long long kappa_dmin_ord;// min d^2 over the active entries of the last snapshot (order-preserving image)
    int kappa_doublings;              // doublings since the last ipcgpu_set_kappa
    int kappa_n_close[2];             // close set: self / obstacle entries, plane entries
    int kappa_needs_init;             // postLineSearch met kappa == 0: initKappa is due
    int kappa_hit;                    // a saved close entry is not farther than its snapshot (the check in flight)
    int kappa_skip;                   // the check in flight found kappa == 0: no snapshot
    // aggregation rounds of the AMG set-up (amg.cu, kAmgRound): passes run, the pass limit (0: the level is not coarsened), rows left
    // undecided by the last pass, the limit was reached
    int amg_round, amg_limit, amg_undecided, amg_stuck;
};
// step_decide operations (step_control.cu) and the energy terms of a line search.  kSolveStart / kSolveBurst: the Krylov loops of both
// built-in solvers (solve.cu, multilevel.cu); kAmgRound: the aggregation rounds of the AMG set-up (amg.cu)
enum { kCflBranch = 0, kCflClamp, kLsEntry, kLsStart, kLsInversion, kLsIntersection, kLsArmijo, kLsPostCheck, kLsPostLoop, kLsRebuild, kWsEntry, kSolveStart,
    kSolveBurst, kAmgRound };
// bytes of IterState from ls_cond on that an eager decision reads back: the decision word and the solve's words (one copy)
constexpr size_t kDecisionBytes = offsetof(IterState, sv_tol) - offsetof(IterState, ls_cond);
enum { kTermInertia = 1, kTermFriction = 2, kTermHalfSpace = 4, kTermHalfSpaceFriction = 8, kTermDamping = 16, kTermNeumann = 32, kTermDirichlet = 64 };
enum { FLAG_NONPOSITIVE_DISTANCE = 0, FLAG_SET_CAPACITY = 1, FLAG_CCD_CAPACITY = 2, FLAG_ZERO_CCD_DISTANCE = 3, FLAG_PATTERN = 4, FLAG_TI_WARNINGS = 5, FLAG_EXCHANGE_CAPACITY = 6,
    FLAG_PATTERN_CAPACITY = 7, FLAG_SOLVE = 8 };
// Scalars that may still hold this rank's share (ipcgpu_ctx::local_scalars): bit s = energy[s], then checks and hs_crossings.  The fetch
// completes them in one sum-allreduce of kPackedScalars doubles: the energies, the flags (a flag is raised iff any rank raised it), the
// 2 checks and the crossing count (integer counts are exact in a double).
enum : unsigned { kLocalChecks = 1u << kEnergySlots, kLocalCrossings = 1u << (kEnergySlots + 1) };
constexpr int kPackedScalars = kEnergySlots + kFlagSlots + 2 + 1;

struct ElasticArgs {
    int nV, nT;
    int t_begin, t_end;      // this rank's OWNED tet range (energy, inversion filter: every tet exactly once)
    int n_list;              // gradient/Hessian kernel: number of tets this rank assembles (all tets that touch its rows)
    const int* tet_list;     // their ids, ascending; nullptr = the contiguous range [t_begin, t_begin + n_list)
    const double* V;         // SoA [x|y|z] current positions
    const int* T;            // SoA [v0|v1|v2|v3]
    const double* Ainv;      // SoA 9 x nT, q = 3*i+j row-major index of Dm^-1
    const double* vol;
    const double* mu;
    const double* lam;
    int energy;              // 0 NH, 1 FCR
    int e_row_lo, e_row_hi;  // fused energy of the gradient/Hessian kernel: a tet is counted by the rank that owns its smallest vertex
};

// elastic.cu
void elastic_energy(const ElasticArgs& p, double* e_per_tet, double* partials, cudaStream_t st); // elastic_energy_blocks partial sums of psi * vol
int elastic_energy_blocks(int nTets);
// e_partials != nullptr: the kernel also leaves one partial sum of psi * vol per CTA there (elastic_grad_hess_blocks of them)
void elastic_grad_hess(const ElasticArgs& p, double coef, int projectSPD, bool need_g, bool need_h, double* gcont, double* hblk, cudaStream_t st, double* e_partials = nullptr);
int elastic_grad_hess_blocks(int n_list);
void gather_gradient(int nV, const int* inc_ptr, const int* inc, const double* gcont, const uint8_t* dbc, int projectDBC, int accumulate, double* g, cudaStream_t st);
// nOff: the off-diagonal slots come first (slots [0, nOff)), the diagonal ones after them.  accumulate == 0: a[] holds zeros at the slots'
// entries (written, not added)
void assemble_csr(int nOff, int nSlots, const int* slot_v, const int* slot_u, const int* slot_off, const int* con_ptr, const unsigned* con_src,
    const double* hblk, const uint8_t* dbc, int projectDBC, const double* mass, int accumulate, double* a, cudaStream_t st);
void diag_mass_dbc(int nV, const int* ia, int base, const uint8_t* dbc, int projectDBC, const double* mass, double* a, cudaStream_t st);
// gate != nullptr: the kernel does nothing unless *gate is nonzero (the device-built pattern recomputes the offsets only when it changed)
void slot_offsets(int nSlots, const int* slot_v, const int* slot_u, const int* ia, const int* ja, int base, int* slot_off, int* err, cudaStream_t st,
    const int* gate = nullptr);
void diag_mass_dbc_range(int v0, int v1, const int* ia, int base, const uint8_t* dbc, int projectDBC, const double* mass, double* a, cudaStream_t st);
void inversion_step(const ElasticArgs& p, const double* dir, double slack, double* per_tet, IterState* st_dev, cudaStream_t st);
void inversion_apply(IterState* st_dev, int nT, cudaStream_t st);          // Energy.cpp:576-579 on the device-resident step
void step_set(IterState* st_dev, double alpha, cudaStream_t st);           // step_ord = alpha
void pack_scalars(const IterState* st_dev, unsigned local_mask, double* buf, cudaStream_t st);   // deferred cross-rank scalars -> kPackedScalars doubles
void unpack_scalars(IterState* st_dev, unsigned local_mask, const double* buf, cudaStream_t st);


// ---- contact ------------------------------------------------------------------------------------------
struct SurfArgs {
    int nV;
    const double* V;      // SoA current positions
    const double* Vrest;  // SoA rest positions
    const uint8_t* dbc;   // nullable
    const int* vCoDim;    // nullable (=> 3)
    int nSV; const int* SVI;
    int nSE; const int* SE;   // interleaved (first, second)   [Mesh::SFEdges]
    int nSF; const int* SF;   // SoA [v0|v1|v2]                [Mesh::SF column-major]
    // kinematic obstacle (MeshCO): vertices >= nVdof belong to a triangle mesh without degrees of freedom that rides at the tail of the vertex
    // arrays (ipcgpu_set_obstacle_tail; INT_MAX = none).  Pairs between the mesh and the obstacle follow MeshCO.cpp, pairs inside the obstacle
    // do not exist.  ee_as_vf: Tight-Inclusion evaluates mesh-obstacle edge pairs through the vertex-face routine (MeshCO.cpp:1609)
    int nVdof, ee_as_vf;
};
// which body a surface primitive belongs to is decided by any one of its vertices (primitives do not straddle bodies)
__device__ __forceinline__ bool obstacle_vertex(const SurfArgs& s, int v) { return v >= s.nVdof; }

// Reproducible mode (ipcgpu_set_canonical_order(ctx, 2), repro.cu): the contact terms add into g and a in an order fixed by the lists alone.
// A term kernel writes each pair's per-vertex vectors to `stage` (3 doubles per contribution index); a gather then sums the entries of
// every vertex in ascending key order and adds the result to g once.  The Hessians go through a per-row gather of the same form.
struct VertexIndex {
    const int* ptr;                  // nV + 1 starts: the entries of vertex v are key[ptr[v], ptr[v + 1]), ascending
    const unsigned long long* key;   // gradient key or Hessian block key (repro.cuh: gkey_*, hkey)
};
struct ReproArgs {
    int on = 0;                      // 0: the atomic scatter (levels 0 and 1); nothing below is read
    int cap = 0;                     // list capacity, which places the mollified list's gradient keys (repro.cuh: para_keys)
    double* stage = nullptr;         // per-contribution gradient vectors
    double* hstage = nullptr;        // friction Hessian: M (9) and the stencil weights (4) per pair
    VertexIndex g = {}, h = {};      // gradient and Hessian indices
};

struct BarrierArgs {
    ReproArgs rep;
    int nV;
    const double* V;
    const double* Vrest;
    const uint8_t* dbc;
    const int* SE;
    const int4* cs; const int* nC;          // active set (MMCVID encoding, SURVEY appendix A) and its DEVICE-resident count
    const int4* para; const int2* para_e; const int* nP; // mollified (nearly parallel EE) set + (eI,eJ), device count
    // multi-rank: E and g are taken over a contiguous share [n*rank/nranks, n*(rank+1)/nranks) of each list (share = 1) or over the
    // whole list (share = 0: the lists are already this rank's own); the Hessian is assembled by ROW OWNER: a rank processes every
    // pair that touches a vertex in [row_lo, row_hi) and scatters only the block rows it owns
    int rank, nranks, share;
    int row_lo, row_hi;
    double dHat, kappa;
    int projectDBC;
    const int* ia; const int* ja; int base;
    int nVdof; // first obstacle vertex (SurfArgs::nVdof)
    const double* kappa_dev; // nullptr: kappa above; else the device-resident kappa (IterState::kappa), read at run time
};

// barrier.cu
void barrier_energy(const BarrierArgs& p, double* partials, int* bad, cudaStream_t st);
int barrier_energy_blocks();
void barrier_gradient(const BarrierArgs& p, double* g, cudaStream_t st);
void evaluate_constraints(const BarrierArgs& p, double* val, cudaStream_t st);
void constraint_jacobian_t(const BarrierArgs& p, const double* input, double coef, double* g, cudaStream_t st);
void para_gradient(const BarrierArgs& p, double* g, cudaStream_t st);
// Hraw: 144 doubles per owned pair; rows: 4 vertex ids per owned pair; psd: makePD "unchanged" flag per owned pair; n_owned: device counter
void barrier_hessian_build_project(const BarrierArgs& p, int* flags, double* Hraw, int* rows, int* psd, int* n_owned, int capacity, cudaStream_t st);
void barrier_hessian_scatter(const BarrierArgs& p, double* a, int* flags, const double* Hraw, const int* rows, const int* psd, const int* n_owned, int capacity, cudaStream_t st);
// repro.cu -- the reproducible mode.  g[v] += the staged contributions of v with lo <= key < hi, in index order (one thread per vertex)
void repro_gather_g(int nV, const VertexIndex& idx, const double* stage, unsigned long long lo, unsigned long long hi, double* g, cudaStream_t st);
// friction.cu -- lagged friction of the self-contact pairs (SelfCollisionHandler.cpp:2481-2987)
struct FrictionArgs {
    ReproArgs rep;
    int nV;
    const double* V;       // current positions (SoA)
    const double* Vt;      // positions at the start of the time step, result.V_prev (SoA)
    const uint8_t* dbc;
    const int4* cs; const int* n;   // LAGGED active set (MMActiveSet_lastH) and its device-resident size
    const double* lambda;           // MMLambda_lastH
    const double2* coord;           // MMDistCoord
    const double* basis;            // MMTanBasis: 6 per pair, column-major 3x2
    double eps2, coef;              // fricDHat, selfFric
    int projectDBC;
    const int* ia; const int* ja; int base;
    int rank, nranks;               // E and g: contiguous share of the list; H: by row owner [row_lo, row_hi)
    int row_lo, row_hi;
};
void friction_lag(const BarrierArgs& p, int4* cs_out, int* n_out, double* lambda, double2* coord, double* basis, int capacity, int* bad, cudaStream_t st);
void friction_energy(const FrictionArgs& p, double* partials, cudaStream_t st);
int friction_energy_blocks();
void friction_gradient(const FrictionArgs& p, double* g, cudaStream_t st);
void friction_hessian(const FrictionArgs& p, double* a, int* err, cudaStream_t st);
// pattern.cu: a[ia[row0] - base, ia[row1] - base) = 0 with the range read on the device (the value-array clear of the device-built pattern)
void zero_csr_rows(const int* ia, int base, int row0, int row1, double* a, cudaStream_t st);
// elastic.cu (shared fixed-order reduction)
// scale_dev != nullptr: the scale is read on the device from there instead of `scale`
void reduce_sum(const double* partials, int n, double scale, double* out, cudaStream_t st, const double* scale_dev = nullptr);

// misc.cu.  alpha_ord != nullptr: the step is read on the device from there (an IterState::step_ord) instead of `alpha`
void step_forward(int nV, const double* x0_soa, const double* p_interleaved, double alpha, double* x_soa, cudaStream_t st,
    const unsigned long long* alpha_ord = nullptr);
// step_control.cu: IterState::sc_pmax_ord = max |p| over the surface vertices below nVdof; one decision of the step control (handle != 0:
// also the value of that conditional graph node)
void cfl_pmax(int nSV, const int* SVI, int nVdof, const double* dir, IterState* st_dev, cudaStream_t st);
// aux: kSolveStart reads the solver's scalars there ([4] |b|^2, [6] a non-positive pivot)
void step_decide(IterState* st_dev, int op, double a, int b, unsigned long long handle, cudaStream_t st, const double* aux = nullptr);
// inertia term of Optimizer::computeEnergyVal / computeGradient (Optimizer.cpp:3227-3239, :3439-3450)
int inertia_energy_blocks(int nV);
void inertia_energy(int v0, int v1, int nV, const double* x_soa, const double* xtilde_soa, const double* mass, double* partials, cudaStream_t st);
void inertia_gradient(int nV, const double* x_soa, const double* xtilde_soa, const double* mass, const uint8_t* dbc, int projectDBC, double* g, cudaStream_t st);
// halfspace.cu -- analytic planes (HalfSpace<3>).  par: kPlaneStride doubles per plane [n0 n1 n2 D v0 v1 v2 mu]; act / lag: (plane, vertex)
constexpr int kPlaneStride = 8;
constexpr int kMaxPlanes = 8;
struct HalfSpaceArgs {
    int nV, nSV, nP;
    const int* SVI;
    const double* V;        // current positions (SoA)
    const double* Vt;       // result.V_prev (SoA), friction only
    const uint8_t* dbc;     // nullable
    const int* vCoDim;      // nullable (=> 3)
    const double* par;
    const int2* act; const int* n_act;        // active set and its device-resident size
    const int2* lag; const double* lam; const int* n_lag; // lagged set (friction planes only), lambda, size
    int row_lo, row_hi;     // rows (energies, gradient, Hessian, crossings) this rank owns
    const int* ia; int base;
    // reproducible mode: an entry (plane q, vertex v) at list position c leaves its vector / block in rep_stage[c], sets bit q of rep_mask[v]
    // and c in rep_pos[kMaxPlanes v + q]; the entry of the lowest plane of v then adds them in plane order (and clears rep_mask[v])
    int* rep_mask = nullptr;
    int* rep_pos = nullptr;
    double* rep_stage = nullptr;
};
int halfspace_energy_blocks();
size_t halfspace_scan_bytes(int n);
// n_act: the device-resident size the per-entry kernels read (also left in IterState::hs_n_active); pstart: first entry of each plane (nP + 1)
cudaError_t halfspace_active_set(const HalfSpaceArgs& p, double dHat, int* flags, int* offs, void* scan_tmp, size_t scan_bytes, int2* act, int* n_act,
    int* pstart, IterState* st_dev, cudaStream_t st);
void halfspace_energy(const HalfSpaceArgs& p, double dHat, double* partials, int* bad, cudaStream_t st);
// kappa_dev != nullptr: kappa is read on the device from there (IterState::kappa)
void halfspace_gradient(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, double* g, cudaStream_t st);
void halfspace_hessian(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, int projectDBC, double* a, cudaStream_t st);
void halfspace_step(const HalfSpaceArgs& p, const double* dir, double slack, IterState* st_dev, cudaStream_t st);
void halfspace_crossings(const HalfSpaceArgs& p, IterState* st_dev, cudaStream_t st);
void halfspace_lag(const HalfSpaceArgs& p, double dHat, double kappa, const double* kappa_dev, const int* pstart, int2* lag, double* lam, int* n_lag, int* bad, IterState* st_dev, cudaStream_t st);
void halfspace_friction_energy(const HalfSpaceArgs& p, double eps2, double* partials, cudaStream_t st);
void halfspace_friction_gradient(const HalfSpaceArgs& p, double eps2, double* g, cudaStream_t st);
void halfspace_friction_hessian(const HalfSpaceArgs& p, double eps2, int projectDBC, double* a, cudaStream_t st);

// damping.cu -- Rayleigh damping (D in elastic slot order, 9 doubles per slot), Neumann forces, augmented-Lagrangian Dirichlet penalty
struct DampingArgs {
    int nV, nSlots;
    const int* slot_v; const int* slot_u;
    const int* inc_ptr; const int* inc;   // slot incidence per vertex (nV + 1 starts; entry 2s: as slot_v, 2s + 1: as slot_u of an off-diagonal slot)
    const double* D;
    const double* V; const double* Vprev; // SoA
    const uint8_t* dbc;                   // nullable
};
struct DirichletArgs {
    int n, nV;
    const int* vid; const double* tgt; const double* lam; // targets: vertex, target position and multiplier (3 per target, interleaved)
    const double* V; const double* mass;
    const double* rho;                    // device-resident rho_DBC (IterState::dbc_rho)
};
void damping_assemble(int nSlots, const int* slot_v, const int* slot_u, const int* con_ptr, const unsigned* con_src, const double* hblk, const uint8_t* dbc,
    double* D, cudaStream_t st);
int damping_energy_blocks(int nSlots);
void damping_energy(const DampingArgs& p, double* partials, cudaStream_t st);
void damping_gradient(const DampingArgs& p, int projectDBC, double* g, cudaStream_t st);
void damping_hessian(const DampingArgs& p, const int* slot_off, double* a, cudaStream_t st);
int vertex_energy_blocks(int n); // partials of the per-vertex / per-target energies below
void neumann_energy(int nV, const double* x, const double* f, const double* mass, const uint8_t* dbc, const double* coef, double* partials, cudaStream_t st);
void neumann_gradient(int nV, const double* f, const double* mass, const uint8_t* dbc, const double* coef, double* g, cudaStream_t st);
void dirichlet_energy(const DirichletArgs& p, double* partials, cudaStream_t st);
void dirichlet_gradient(const DirichletArgs& p, double* g, cudaStream_t st);
void dirichlet_hessian(const DirichletArgs& p, const int* ia, int base, double* a, cudaStream_t st);
void dirichlet_update_lambda(const DirichletArgs& p, double* lam, cudaStream_t st);
void dirichlet_completed_step(const DirichletArgs& p, const double* dist2Tol, double* partials, double* out, cudaStream_t st); // 3 launches (dist2Tol: device)
void set_double(double* p, double v, cudaStream_t st); // a device double in stream order

// timestep.cu -- time integration (Optimizer::setTime / computeXTilta / solve's end of step / initX).  TimeParams lives in device memory
// (ipcgpu_set_time_integration): a replayed graph reads the current values.
struct TimeParams {
    double dt, dtSq, beta, gamma;      // dtSq = dt * dt (setTime, Optimizer.cpp:423)
    double gravity[3], gDtSq[3];       // gravityDtSq = dtSq * gravity (:427)
    int type;                          // 0 TIT_BE, 1 TIT_NM
    int pad_;
};
struct DynamicsArgs {
    int nV;
    const TimeParams* tp;
    const uint8_t* dbc;                // nullable: isDBCVertex = dbc != 0
    double* vel;                       // velocity, interleaved 3 nV
    double* acc;                       // acceleration, nV x 3 column-major (SoA)
    double* dxe;                       // dx_Elastic, nV x 3 column-major (SoA)
    const double* V;                   // SoA
    double* Vprev;                     // result.V_prev, SoA
    double* xtilde;                    // xTilta, SoA
};
void timestep_xtilde(const DynamicsArgs& p, cudaStream_t st);
void timestep_end(const DynamicsArgs& p, cudaStream_t st);
void timestep_predictor(const DynamicsArgs& p, int option, double* dir, cudaStream_t st); // option 0-4 into dir (interleaved)

// diagnostics.cu -- the end-of-step diagnostics: Optimizer::computeSystemEnergy per component and the constraint summary of the homotopy
// read-back.  A segment is the part of one component's tet range or vertex range inside one cell of the global chunk grid (kDiagChunk
// elements); the table lists every component's tet segments, then its vertex segments, in index order, component after component.
constexpr int kDiagChunk = 2048;
enum { kSegTets = 0, kSegVertices = 1 };
struct DiagSegment {
    int begin, end, kind, pad_;
};
struct SystemEnergyArgs {
    int nV, n_comp, n_seg;
    const DiagSegment* seg;
    const int* comp_seg;      // n_comp + 1 starts of each component's segments in `seg`
    const double* e_per_tet;  // vol psi per tet at the current V (k_elastic_energy)
    const double* V; const double* Vprev; const double* mass; // SoA, SoA, mass_diag
    const TimeParams* tp;
    double* part;             // 7 doubles per segment: E, p (3), V x p (3)
    double* out;              // sysE (n_comp), sysM (3 n_comp), sysL (3 n_comp)
};
void system_energy(const SystemEnergyArgs& p, cudaStream_t st); // 2 launches
struct SummaryArgs {
    int nV;
    const double* V;                         // SoA
    const double* par; const int2* act; const int* n_act; // planes (nullptrs without planes)
    const double* val; const int* nC;        // pair_distance of the self / obstacle active entries (k_evaluate_constraints)
    double dHat, kappa;
    const double* kappa_dev;                 // nullptr: kappa above; else IterState::kappa
    double* part;                            // kDiagSummaryBlocks partial sums of fb^2
    unsigned long long* part_ord;            // 2 kDiagSummaryBlocks: min and max image of d per CTA
    double* out;                             // n, d_min, d_max, fb_norm
};
void constraint_summary(const SummaryArgs& p, cudaStream_t st); // 2 launches
constexpr int kDiagSummaryBlocks = 264;

// zero n_words 4-byte words.  A kernel rather than cudaMemsetAsync where the two chains of an iteration overlap (abi.h: enter): replayed from a
// graph, a memset node has no priority of its own and queues behind whatever low-priority grids are pending, which held the step-bound
// chain up for the length of the CSR assembly
void zero_words(void* p, size_t n_words, cudaStream_t st);

} // namespace ipcgpu
