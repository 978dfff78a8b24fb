/*
 * oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain C++17 (Eigen-free, TBB-free) restatement of the reference
 * (ipc-sim/IPC @ 573d2c7) algorithms on the Newton hot path. Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library; the product path (ipc_b200/csrc) never links it.
 *
 * Every function cites the reference file:line it follows. Matrices are
 * row-major double[9] (M[3*i+j]) unless stated; "ref layout" means the Eigen
 * column-major layout the reference hands out with .data().
 *
 * Pinning status (see DESIGN.md "Oracle"):
 *   - pair distance / gradient / Hessian / barrier: pinned against the reference's
 *     own MATLAB-codegen scalar bodies compiled into oracle/_ref (when
 *     /root/reference is present) and against committed mpmath golden vectors.
 *   - elastic path: pinned against mpmath golden vectors generated from the
 *     closed forms (tests/golden), FD self-consistency and invariants.
 *   - Tight-Inclusion: the arithmetic lives in an un-vendored third party
 *     (CCD-Wrapper@23907da -> Tight-Inclusion); restated from the published
 *     algorithm => "parity unpinned" for that stage.
 */
#pragma once
#include <cstdint>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- elastic (oracle/elastic.cpp) ---------------------------------------- */
/* AutoFlipSVD / JIXIE implicit-QR 3x3 SVD (ImplicitQRSVD.h:687-850). Row-major. */
int orc_svd3(const double F[9], double U[9], double S[3], double V[9]);
/* Which way the same SVD left: *exit_id = 0..4 for the beta_2, beta_1, alpha_2, alpha_3, alpha_1 exits (in the order they are tested);
 * *sort_id = 0 / 1 for the sort after process(0) / process(1); *reordered = 1 when that sort took its swapping branch rather than the
 * early return. Returns the QR sweep count. */
int orc_svd3_branch(const double F[9], int* exit_id, int* sort_id, int* reordered);

/* energy_type: 0 = NeoHookean, 1 = FixedCoRot */
void orc_psi(int energy_type, const double S[3], double mu, double lam, double* E);
void orc_dpsi(int energy_type, const double S[3], double mu, double lam, double dE[3]);
void orc_d2psi(int energy_type, const double S[3], double mu, double lam, double d2E[9]);
void orc_bleft(int energy_type, const double S[3], double mu, double lam, double BL[3]);
void orc_pk1(int energy_type, const double F[9], const double U[9], const double S[3],
    const double V[9], double mu, double lam, double P[9]);
void orc_dPdF(int energy_type, const double U[9], const double S[3], const double V[9],
    double mu, double lam, double w, int projectSPD, double dPdF[81]);
void orc_makePD(int n, double* M /* n x n row-major, symmetric */);
void orc_makePD2d(double M[4]);

typedef struct {
    int nV, nT;
    const double* V;      /* SoA [x(nV) | y(nV) | z(nV)]  (Eigen col-major MatrixXd nV x 3) */
    const int* T;         /* SoA [v0(nT) | v1 | v2 | v3]  (Eigen col-major MatrixXi nT x 4) */
    const double* Ainv;   /* restTriInv, ref layout: 9 per tet, column-major */
    const double* vol;    /* triArea (rest volume) */
    const double* mu;
    const double* lam;
    const uint8_t* dbc;   /* per vertex: 0 NOT_DBC, 1 ZERO, 2 NONZERO (Mesh.hpp:135-144) */
    int energy_type;
} orc_mesh;

/* Energy.cpp:195-242 */
void orc_elastic_energy(const orc_mesh* m, double coef, double* E_per_elem /*nullable*/, double* E, int nthreads);
/* Energy.cpp:245-289 (+ :334-366) ; g interleaved [x0 y0 z0 x1 ...] */
void orc_elastic_gradient(const orc_mesh* m, double coef, int projectDBC, double* g, int nthreads);
/* Energy.cpp:368-408 ; H_all: 144 per tet, row-major 12x12 */
void orc_elastic_hessian_blocks(const orc_mesh* m, double coef, int projectSPD, double* H_all, int nthreads);
/* Energy.cpp:317-330 + IglUtils.hpp:39-116 + LinSysSolver.hpp:331-339,402-410.
 * a must be zeroed by the caller (setZero). ia/ja use index_base (0 or 1). */
void orc_elastic_hessian_csr(const orc_mesh* m, double coef, int projectSPD, int projectDBC,
    const int* ia, const int* ja, int index_base, double* a, int nthreads);
/* get_feasible_steps.cpp:110-172 + Energy.cpp:565-581 ; p interleaved */
void orc_inversion_step(const orc_mesh* m, const double* p, double slack, double* per_tet /*nullable*/, double* alpha_inout);

/* LinSysSolver.hpp:46-150: builds the upper-triangular block CSR pattern from vertex
 * adjacency given as CSR (nbr_ptr/nbr sorted ascending, no self). Returns nnz; if ia==NULL only counts. */
int orc_csr_pattern(int nV, const int* nbr_ptr, const int* nbr, int index_base, int* ia, int* ja);

/* ---- contact pair math (oracle/contact.cpp) -------------------------------- */
void orc_d_PP(const double* v, double* d);                /* v: 6 doubles  */
void orc_d_PE(const double* v, double* d);                /* v: 9 doubles  */
void orc_d_PT(const double* v, double* d);                /* v: 12 doubles */
void orc_d_EE(const double* v, double* d);
void orc_g_PP(const double* v, double* g);
void orc_g_PE(const double* v, double* g);
void orc_g_PT(const double* v, double* g);
void orc_g_EE(const double* v, double* g);
void orc_H_PP(const double* v, double* H);                /* row-major n x n */
void orc_H_PE(const double* v, double* H);
void orc_H_PT(const double* v, double* H);
void orc_H_EE(const double* v, double* H);
int orc_dType_PT(const double* v);
int orc_dType_EE(const double* v);
void orc_point_tri_d(const double* v, double* d);
void orc_edge_edge_d(const double* v, double* d);
void orc_barrier(double d, double dHat, double* b, double* db, double* d2b);
/* mollifier (MeshCollisionUtils.hpp:2409-2912) */
void orc_ee_cross(const double* v, double* c, double* g /*12, nullable*/, double* H /*144, nullable*/);
void orc_mollifier(const double* v, double eps_x, double* e, double* g /*12*/, double* H /*144*/);

typedef struct {
    int nV;
    const double* V;       /* SoA current positions */
    const double* Vrest;   /* SoA rest positions (eps_x) */
    const uint8_t* dbc;
    int nSV; const int* SVI;
    int nSE; const int* SE;  /* interleaved (first,second) */
    int nSF; const int* SF;  /* SoA [v0(nSF)|v1|v2] (Eigen col-major) */
    const int* vCoDim;       /* per vertex codimension (3 for tet bodies); nullable => 3 */
} orc_surf;

/* SelfCollisionHandler.cpp:2149-2478 (brute force over all pairs: the set does not depend on the hash).
 * Outputs are canonically sorted. Buffers sized by caps; returns 0 or -1 if a cap was exceeded. */
int orc_constraint_set(const orc_surf* s, double dHat,
    int cap, int* mmcvid /*4*cap*/, int* nC,
    int capP, int* para /*4*capP*/, int* para_eIeJ /*2*capP*/, int* nPara,
    int capK, int* cand /*2*capK*/, int* nCand, int nthreads);

/* SelfCollisionHandler.cpp:38-81, Optimizer.cpp:3290-3353 */
int orc_barrier_energy(const orc_surf* s, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara,
    double dHat, double kappa, double* E);
/* SelfCollisionHandler.cpp:84-148, :2990-3045 ; g += ... (interleaved) */
void orc_barrier_gradient(const orc_surf* s, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara,
    double dHat, double kappa, int projectDBC, double* g);
/* SelfCollisionHandler.cpp:418-561, :3049-3201 ; a += ... */
void orc_barrier_hessian_csr(const orc_surf* s, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara,
    double dHat, double kappa, int projectDBC,
    const int* ia, const int* ja, int index_base, double* a, int nthreads);
/* per-pair projected block, for kernel parity: kind/verts out, H row-major 12x12 (unused rows zero) */
void orc_barrier_pair_hessian(const orc_surf* s, const int mm[4], double dHat, double kappa, double* H144, int* nvert);

/* ---- lagged friction of the self-contact pairs (oracle/friction.cpp) ---------------------------------- */
/* Optimizer.cpp:1582-1595 (lambda) + SelfCollisionHandler.cpp:2481-2527 (closest-point coordinates, tangent bases) at s->V.
 * basis: 6 per pair = Eigen column-major Matrix<double,3,2>. */
void orc_friction_lag(const orc_surf* s, const int* mmcvid, int nC, double dHat, double kappa, double* lambda, double* coord, double* basis);
/* SelfCollisionHandler.cpp:2529-2596 ; s->V current, Vt = result.V_prev (SoA) */
void orc_friction_energy(const orc_surf* s, const double* Vt, const int* mmcvid, int nC, const double* lambda, const double* coord, const double* basis,
    double eps2, double coef, double* E);
/* SelfCollisionHandler.cpp:2598-2735 ; g += (interleaved) */
void orc_friction_gradient(const orc_surf* s, const double* Vt, const int* mmcvid, int nC, const double* lambda, const double* coord, const double* basis,
    double eps2, double coef, double* g);
/* one pair's block, row-major with leading dimension 12; project = 0 skips makePD (for the finite-difference tests) */
void orc_friction_pair_hessian(const orc_surf* s, const double* Vt, const int mm[4], double lambda, const double coord[2], const double basis[6], double eps2,
    double coef, int project, double* H144, int* nvert);
/* SelfCollisionHandler.cpp:2745-2987 ; a += */
void orc_friction_hessian_csr(const orc_surf* s, const double* Vt, const int* mmcvid, int nC, const double* lambda, const double* coord, const double* basis,
    double eps2, double coef, int projectDBC, const int* ia, const int* ja, int index_base, double* a, int nthreads);

/* ---- broad phase + CCD (oracle/ccd.cpp) -------------------------------------- */
typedef struct {
    double lo[3]; double inv_h; int count[3];
} orc_grid;
/* SpatialHash.hpp:46-58 / :589-640 (swept; alpha is scaled down in place when spanSize>1) */
void orc_grid_static(const orc_surf* s, double h, orc_grid* g);
void orc_grid_swept(const orc_surf* s, const double* p, double* alpha_inout, double h, orc_grid* g);

/* CCDUtils.cpp:21-87 + Tight-Inclusion get_numerical_error (restated) */
void orc_ti_error(const double* V, int nV, const double* p /*nullable*/, double err_vf[3], double err_ee[3]);
/* Tight-Inclusion vertexFaceCCD_double / edgeEdgeCCD_double restatement.
 * x0: 12 doubles (4 verts at t=0), x1: 12 doubles (t=1). Returns 1 on hit. */
int orc_ti_vf(const double* x0, const double* x1, const double err[3], double ms, double tol,
    double max_t, int max_itr, int no_zero_toi, double* toi, double* out_tol);
int orc_ti_ee(const double* x0, const double* x1, const double err[3], double ms, double tol,
    double max_t, int max_itr, int no_zero_toi, double* toi, double* out_tol);
/* diagnostics: 1 = boxes of a level with equal t_lo are visited in DESCENDING (u_lo, v_lo) instead of the canonical ascending order */
void orc_ti_debug_tie_order(int reversed);
/* SelfCollisionHandler.cpp:690-866 with canonical max_t = alpha on entry */
int orc_ccd_partial(const orc_surf* s, const double* p, const int* cand, int nCand, double tol,
    const double err_vf[3], const double err_ee[3], double* alpha_inout, int nthreads);
/* SelfCollisionHandler.cpp:1370-1630 ; candidate pairs = voxel-AABB overlap on the swept grid */
int orc_ccd_full(const orc_surf* s, const double* p, const orc_grid* g, double alpha_grid, double tol,
    const double err_vf[3], const double err_ee[3], double* alpha_inout, long long* nPairs, int nthreads);

/* ---- reference-style hashed drivers (oracle/hash.cpp): the faithful CPU baselines ----------------------------- */
int orc_constraint_set_hashed(const orc_surf* s, double dHat, double voxel_size,
    int cap, int* mmcvid, int* nC, int capP, int* para, int* para_eIeJ, int* nPara, int capK, int* cand, int* nCand, int nthreads);
int orc_ccd_full_hashed(const orc_surf* s, const double* p, double* alpha_inout, double voxel_size, double tol,
    const double err_vf[3], const double err_ee[3], long long* nPairs, int nthreads);

/* ---- kinematic mesh obstacles: MeshCO<3> (oracle/meshco.cpp) ------------------------------------------------------ */
typedef struct {
    int nV; const double* V;  /* SoA positions (Base::V) */
    int nE; const int* E;     /* interleaved (first, second) (MeshCO::edges) */
    int nF; const int* F;     /* SoA [v0|v1|v2] (Base::F column-major) */
} orc_obstacle;
/* MeshCO.cpp:1795-2223 in MeshCO's MMCVID encoding (negative = mesh vertex, non-negative = obstacle vertex); cand = cs_PTEE */
int orc_meshco_constraint_set(const orc_surf* s, const orc_obstacle* o, double dHat, int cap, int* mmcvid, int* nC, int capP, int* para, int* para_eIeJ, int* nPara,
    int capK, int* cand, int* nCand, int nthreads);
/* the same entries in the self-contact encoding over the merged vertex numbering (obstacle vertex k = nV + k, obstacle edge j = nSE + j) */
void orc_meshco_to_merged(int nV, int nSE, const int* mmcvid, int nC, int* out, const int* para_eIeJ, int nP, int* para_e_out);
/* Optimizer.cpp:3268-3289 / :3480-3491 / :3686-3689 with MeshCO.cpp:83-200, :407-586, :2226-2520; g and the CSR are the MESH's */
int orc_meshco_energy(const orc_surf* s, const orc_obstacle* o, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara, double dHat, double kappa, double* E);
void orc_meshco_gradient(const orc_surf* s, const orc_obstacle* o, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara, double dHat, double kappa, double* g);
void orc_meshco_hessian_csr(const orc_surf* s, const orc_obstacle* o, const int* mmcvid, int nC, const int* para, const int* para_eIeJ, int nPara, double dHat, double kappa,
    int projectDBC, const int* ia, const int* ja, int index_base, double* a, int nthreads);
/* MeshCO.cpp:742-980 and :1388-1668; ee_as_vf = 1: edge-edge pairs through the vertex-face routine, as the reference calls it */
int orc_meshco_ccd_partial(const orc_surf* s, const orc_obstacle* o, const double* p, const int* cand, int nCand, double tol, const double evf[3], const double eee[3],
    int ee_as_vf, double* alpha_inout, int nthreads);
int orc_meshco_ccd_full(const orc_surf* s, const orc_obstacle* o, const double* p, double tol, const double evf[3], const double eee[3], int ee_as_vf, double* alpha_inout,
    long long* nPairs, int nthreads);

/* ---- line-search safeguards (oracle/intersect.cpp) --------------------------------------------------------------- */
/* igl::predicates::orient3d restated (filter + exact expansion arithmetic): +1 / 0 / -1 */
int orc_orient3d(const double* pa, const double* pb, const double* pc, const double* pd);
int orc_orient3d_exact(const double* pa, const double* pb, const double* pc, const double* pd);
/* IglUtils::segTriIntersect (IglUtils.hpp:214-265) */
int orc_seg_tri_intersect(const double* ve0, const double* ve1, const double* vt0, const double* vt1, const double* vt2);
/* SelfCollisionHandler::checkEdgeTriIntersectionIfAny (:3254-3296): 1 = intersection free; hits = intersected triangles */
int orc_intersection_free(const orc_surf* s, double cell, int* hits, int* tri_flags /* nSF, nullable */, int nthreads);
/* Mesh::checkInversion (Mesh.cpp:715-763): tets with mu, lambda != 0 and det(current edge matrix) < 0 */
int orc_count_inverted(const orc_mesh* m);

#ifdef __cplusplus
}
#endif
