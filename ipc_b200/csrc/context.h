// context.h -- the ipcgpu_ctx object behind the C ABI: device buffers, scatter maps, streams, NCCL.
#pragma once
#include "kernels.h"
#include "broadphase_types.h"
#include <cuda_runtime.h>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace ipcgpu {

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    ~DevBuf() { release(); }
    void release()
    {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
    // grow-only allocation; returns false on CUDA failure
    bool reserve(size_t count)
    {
        if (count <= n) return true;
        release();
        if (cudaMalloc(&p, count * sizeof(T)) != cudaSuccess) {
            p = nullptr;
            return false;
        }
        n = count;
        return true;
    }
    bool upload(const T* h, size_t count, cudaStream_t st)
    {
        if (!reserve(count)) return false;
        return count == 0 || cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, st) == cudaSuccess;
    }
};

// device workspace of the contact stages (constraint.cu / ccd.cu)
struct ContactWork {
    DevBuf<Box> vbox, ebox, tbox;   // per-primitive boxes (primitive order)
    DevBuf<QEntry> centries;        // grid-sorted entries (triangles first, then edges): quantised box + id
    DevBuf<unsigned long long> bounds, skey, words; // skey / sidx: the PP/PE duplicate-merge table; words: permuted list entries
    DevBuf<unsigned> ckeys, key_tmp; // ckeys: sorted 32-bit cell keys (cell | type bits) of the combined triangle + edge + vertex grid
    DevBuf<Grid> grid;
    DevBuf<int> cvals, val_tmp, counters, sidx;
    DevBuf<int> cnt, off, perm;     // canonical order: bucket counts / offsets over [-nV, max(nV, nSE)), the sorting permutation
    DevBuf<int4> act, dup, para;
    DevBuf<int2> para_e, cand;
    DevBuf<unsigned char> cub_tmp;  // scans: the cell offsets, the order's bucket offsets, the reproducible mode's index offsets
    DevBuf<int> cell_cnt, cell_off; // dense per-(type, cell) counters and their exclusive prefix sum: entry range of a cell = two adjacent offsets
    DevBuf<int2> bp_pairs; // broad-phase pair lists (PT then EE), bp_cap each
    size_t bp_cap = 0;
    int cap = 0;
    // counters (device ints): [0] active, [1] PP/PE duplicates, [2] mollified, [3] candidates, [4] overflow, [8]/[9] broad-phase pairs PT/EE,
    // [10]/[11] active / mollified of the GLOBAL lists after the cross-rank exchange, [12] pair Hessians owned by this rank
    int nC = 0, nP = 0, nK = 0; // host mirrors of [0], [2], [3]; -1 = not read back (device-resident iteration)
    bool want_cand = false;
    unsigned dup_tab = 1024;    // slots of the PP/PE duplicate-merge table
    int axis_bits = 10;         // key bits per axis of the grid sorts (re-tuned from IterState::grid_axis_cells at every fetch)
    int built_axis_bits = 10;   // ... of the grids that are currently built (position of the type bit)
    int built_vertices = 0;     // surface-vertex entries in the combined sorted array (0: the build carried none)
    // barrier stage workspace, sized by the pair capacity
    DevBuf<double> bHraw, bpartials, bval; // (bval: per-constraint values of ipcgpu_evaluate_constraints / inputs of ..._jacobian_t)
    DevBuf<int> brows, bpsd;
    // multi-rank exchange of the pair lists (one fixed-size message per rank, see k_pack_lists)
    int xcap = 0;
    size_t xstride = 0;
    DevBuf<int4> xsend, xrecv, gact, gpara;
    DevBuf<int2> gpara_e;
    bool lists_global = false; // gact / gpara hold the global lists of the last partitioned build
    // lagged friction data (MMActiveSet_lastH, MMLambda_lastH, MMDistCoord, MMTanBasis): snapshot taken by ipcgpu_friction_lag
    DevBuf<int4> fr_cs;
    DevBuf<int> fr_n;
    DevBuf<double> fr_lambda, fr_basis, fr_partials;
    DevBuf<double2> fr_coord;
    int fr_host_n = -1;        // host mirror of the lagged count (-1 = not read back)
    bool fr_ready = false;
};

// reproducible mode (ipcgpu_set_canonical_order(ctx, 2), repro.cu), allocated when the level is selected: the per-vertex gather indices of
// the barrier (bg / bh) and friction (fg / fh) gradients and Hessians with their staging, and the plane terms' per-vertex masks, positions
// and staging (the index builds count and scan in ContactWork's cnt / cub_tmp).  lists_ready / fr_ready: the indices belong to the lists
// in act / para and fr_cs (built where the lists were produced at level 2)
struct ReproWork {
    DevBuf<int> bg_ptr, bh_ptr, fg_ptr, fh_ptr;
    DevBuf<unsigned long long> bg_key, bh_key, fg_key, fh_key;
    DevBuf<double> bstage, fstage, fhstage;
    DevBuf<int> hs_mask, hs_pos;
    DevBuf<double> hs_stage;
    int cap = 0, nV = 0, nSV = 0; // what the buffers are sized for
    bool lists_ready = false, fr_ready = false;
};

// device workspace of the CCD stage (ccd.cu)
struct CcdWork {
    DevBuf<int> vmin, vmax, counters;
    DevBuf<int2> cand;
    DevBuf<unsigned> surv, surv2;
    DevBuf<unsigned char> scratch, arena; // per-warp level buffers of the narrow phase's warp pass; overflow arena shared by its warps
    DevBuf<int> arena_lock;
    DevBuf<unsigned long long> ncand, bounds;
    // swept grid on the reference voxel lattice (ccd.cu): geometry, per-entry cell keys and entries (sorted by key), dense per-(type, cell)
    // counters and their exclusive prefix sum, scan scratch
    DevBuf<SweptCells> cells;
    DevBuf<unsigned> sw_keys;
    DevBuf<uint4> sw_ent;
    DevBuf<int> sw_cnt, sw_off;
    DevBuf<unsigned char> sw_tmp;
    bool swept_ready = false; // (the reference swept-grid geometry of the last build lives in IterState)
    unsigned last_survivors = 0;
    unsigned long long last_deferred = 0, last_longest_cycles = 0, last_total_cycles = 0;
    int last_warnings = 0;
    unsigned long long last_candidates = 0, last_boxes_thread = 0, last_boxes_warp = 0;
};

// device-built sparsity pattern (pattern.cu, ipcgpu_enable_device_pattern): the static mesh part (vNeighbor, upper neighbours only) and
// the per-update workspace.  Extra blocks (contact neighbours that are not mesh neighbours) are bucketed by their lower vertex.
struct PatternWork {
    DevBuf<int> mptr, mnbr;           // mesh part: upper neighbours u > v of vertex v in mnbr[mptr[v], mptr[v+1]), ascending
    DevBuf<int> row_cnt, row_off;     // raw extra keys per lower vertex (nV + 1, last entry 0) and their exclusive scan
    DevBuf<int> bucket;               // raw extra keys, upper vertex ids grouped by lower vertex (key_cap entries)
    DevBuf<int> ucnt, uoff;           // distinct extra neighbours per vertex (nV + 1) and their exclusive scan
    DevBuf<int> prev_ptr, prev_nbr;   // extra neighbours of the pattern currently in ia / ja (what the next update compares with)
    DevBuf<unsigned char> scan_tmp;
    size_t scan_bytes = 0;
    long long mesh_pairs = 0, mesh_nnz = 0, nnz_cap = 0, key_cap = 0;
    uint64_t requested_cap = 0;       // what the caller asked for (0 = default), kept to rebuild after a surface / obstacle change
};

// multilevel additive Schwarz preconditioner (multilevel.cu): the Morton order of the vertices, the stored inverses of the domain matrices
// (96 x 96 doubles per domain, the levels one after the other) and the per-level restricted / coarse-solved vectors (96 per domain)
constexpr int kMultilevelMax = 8; // levels: 32^8 vertices and more are out of reach of an int
struct MultilevelWork {
    DevBuf<double> box, inv, R, Y, chunk; // (chunk: per-chunk shares of a level's assembly)
    DevBuf<unsigned> code, code_sorted;
    DevBuf<int> id, order, rank;
    DevBuf<unsigned char> sort_tmp, fixed; // (fixed: 1 for a vertex without degrees of freedom -- Dirichlet or obstacle tail)
    bool built = false;                   // the last solve built the whole hierarchy (every pivot positive)
    int levels = 0;
    long long domains[kMultilevelMax] = {};
    size_t tile_off[kMultilevelMax] = {}, tiles = 0; // first domain of every level, domains in all
    bool smem_opted = false;              // the inversion kernel's dynamic shared memory has been opted in
};

// smoothed-aggregation multigrid preconditioner (amg.cu): per level the block CSR matrix (3 x 3 blocks), the inverses of its diagonal
// blocks, the aggregates, the prolongator P and its transpose R (block CSR), the cycle's vectors; shared scratch of the set-up
// Every size of the hierarchy lives in device memory (AmgDev), so that a reserved set-up runs inside a graph; the host reads it back
// only to grow buffers (unreserved) or to answer a getter.
constexpr int kAmgMaxLevels = 6;
constexpr int kAmgDegree = 16;
// the entry counts of one coarsening (level l -> l + 1) that a reservation bounds: blocks of P (and R), entries of the A P expansion, blocks
// of A P, entries of the R (A P) expansion, blocks of A_{l+1}
enum { kAmgQP = 0, kAmgQApExp, kAmgQAp, kAmgQRapExp, kAmgQCoarse, kAmgQty };
struct AmgDev {
    int n[kAmgMaxLevels];                 // block rows (0: not built by the last set-up)
    int nnzb[kAmgMaxLevels];              // kept blocks
    int np[kAmgMaxLevels];                // blocks of P (0 on the last level)
    int na[kAmgMaxLevels];                // aggregates of the coarsening of level l
    int go[kAmgMaxLevels];                // level l is coarsened (cleared by a stopping rule or a capacity cut)
    int levels, fail, cut_level, coarse_enough; // fail: a pivot <= 0, a non-finite rho or bound, a bad layout; cut_level: -1 = not cut
    int cut_depth, pad_;                  // cut_depth: the cut is the reserved depth (the set-up wanted one more level)
    long long need[kAmgMaxLevels][kAmgQty]; // what the last set-up needed (counted even where it was cut)
    double rho[kAmgMaxLevels], rho_g[kAmgMaxLevels], omega[kAmgMaxLevels]; // rho_g: the Gershgorin bound of D^-1 A
    double inv_theta[kAmgMaxLevels], c[kAmgMaxLevels][kAmgDegree][2]; // Chebyshev: 1 / theta, (c1, c2) of step k
};
struct AmgLevel {
    DevBuf<int> ia, ja, agg, pia, pja, ria, rja;
    DevBuf<double> blk, dinv, pblk, rblk;
    DevBuf<double> f, x, r, d0, d1, t; // (level 0 takes f and x from the Krylov loop: r and z)
    long long cap_n = 0, cap_nnzb = 0, cap[kAmgQty] = {}; // the sizes the buffers hold (rows, kept blocks, the coarsening's counts)
};
struct AmgWork {
    AmgLevel lv[kAmgMaxLevels];
    int levels = 0;                                     // levels of the cycle: the built ones (unreserved), the reserved depth otherwise
    int reserved = 0;                                   // reserved depth L_r (ipcgpu_amg_reserve); 0: the set-up reads sizes back and grows
    int res_nV = 0;                                     // the mesh the reservation was sized for (another one drops it)
    bool ran = false;                                   // a set-up was enqueued (AmgDev holds its result)
    DevBuf<AmgDev> dev;
    AmgDev h{};                                         // host copy of dev (read by the getters)
    DevBuf<int> cnt, scan_out, m1, m2, pos, lidx, ridx, spos, prow, api, apj;
    DevBuf<double> apb;                                 // A P of the coarsening in flight
    DevBuf<unsigned long long> key, skey, tkey, tkey_sorted; // (row, column) keys of a product's entries; (column, row) keys of R
    DevBuf<unsigned char> state0, state1, tmp;
    DevBuf<int> flags;                                  // [1] bad layout, [2] bad pivot
    DevBuf<unsigned long long> absrow;                  // max absolute row sum of D^-1 A (ordered bits)
    DevBuf<double> part, sq;                            // power iteration: per-chunk partials, squared norms of every step
};

// point-in-tetrahedron half of the intersection check (safeguard.cu): the codimension-0 vertices (vCoDim == 0) of ipcgpu_set_surface, and
// a grid over them rebuilt at every check -- cell key per point, the (key, vertex) pairs sorted by key, the grid's geometry, sort scratch
struct PointGrid {
    double o[3], inv_h;
    int n[3];
    double lo[3], hi[3]; // box of the points: a tetrahedron whose box misses it scans nothing
};
struct PointTetWork {
    int n = 0; // codimension-0 vertices; 0 = the check launches nothing
    DevBuf<int> pts, id, id_sorted;
    DevBuf<unsigned> key, key_sorted;
    DevBuf<PointGrid> grid;
    DevBuf<unsigned char> sort_tmp;
    size_t sort_bytes = 0;
};

// pinned host memory of the scalars the entry points copy between host and device, one member per use.  Allocated once per context
// (cudaMallocHost(sizeof(HostStaging))), freed by ipcgpu_destroy: every member keeps its own address for the context's lifetime, since a
// captured graph or a copy nobody waits on may still hold it.
struct HostStaging {
    double scalar;   // a read-back double: energy_result, ipcgpu_dirichlet_completed_step
    int count;       // a read-back count: the lagged friction pairs
    int contact[16]; // ContactWork::counters read back (contact_sync_counts) or uploaded (ipcgpu_set_constraint_set)
    double pSize;    // source of upload_dir's asynchronous H2D copy into pSize_dev, which nothing waits on: never reused for anything else
    int hs_count[2]; // half-space counts: [0] active, [1] lagged
};

} // namespace ipcgpu

struct ipcgpu_ctx {
    int device = 0;
    // main stream, high priority: everything except the derivative chain, in particular the step-bound chain (the critical path)
    cudaStream_t stream = nullptr;
    // derivative stream, low priority: the elastic gradient/Hessian, its CSR assembly and the barrier gradient / Hessian scatter of the
    // device-resident iteration run here next to the step-bound chain (abi.h: enter / join_deriv).  deriv_open: work has been forked
    // onto it that the main stream has not joined yet; deriv_copied: the capture in progress copies derivative results to the host
    cudaStream_t deriv = nullptr;
    cudaEvent_t ev_deriv_fork = nullptr, ev_deriv_done = nullptr;
    bool deriv_open = false, deriv_copied = false;
    int prio_low = 0, prio_high = 0; // the device's stream priority range (numerically lower = higher priority)
    cudaStream_t deriv_stream() const { return deriv_open ? deriv : stream; }
    // side stream: the build + projection of the pair Hessians (latency-bound, a fraction of one wave) run next to the elastic assembly
    // and join the stream of the derivative chain before the scatter; ev_inputs marks, on the main stream, the last point at which their
    // inputs (positions, contact sets) changed
    cudaStream_t side = nullptr;
    // copy stream: ipcgpu_download_range_async forks it off the main stream, so that a result (gradient, CSR values) travels to the host
    // while the later stages of the iteration run; joined by ipcgpu_fetch_iteration / ipcgpu_sync / ipcgpu_capture_end
    cudaStream_t copy = nullptr;
    cudaEvent_t ev_copy_fork = nullptr, ev_copy_join = nullptr;
    bool copy_pending = false;
    cudaEvent_t ev_inputs = nullptr, ev_join = nullptr, ev_scatter = nullptr; // (ev_scatter: the previous scatter has read the pair Hessians)
    bool scatter_marked = false;
    bool inputs_marked = false;
    void mark_inputs()
    {
        inputs_marked = (cudaEventRecord(ev_inputs, stream) == cudaSuccess);
    }
    std::string err;
    uint64_t launches = 0;

    // partition: tets [t_begin, t_end) are OWNED (energy, inversion filter); rows of vertices [v_begin, v_end) are owned, and the
    // gradient/Hessian kernel runs over every tet that touches them (tet_list, halo tets duplicated) so that the CSR needs no reduction
    int rank = 0, nranks = 1;
    void* nccl_comm = nullptr;
    int v_begin = 0, v_end = 0, n_list = 0;
    ipcgpu::DevBuf<int> tet_list;
    long long a_begin = 0, a_end = 0; // CSR value range of the owned rows

    // device-resident scalars of the iteration in flight + pinned host mirror
    ipcgpu::DevBuf<ipcgpu::IterState> iter;
    ipcgpu::IterState* h_iter = nullptr;
    double pSize = 0.0;     // mean |p| over the surface vertices (SpatialHash.hpp:603-612), computed when p is uploaded
    bool dir_valid = false, pSize_surface = false;
    unsigned local_scalars = 0;              // kLocal* bits (kernels.h): IterState scalars that still hold this rank's share
    bool a_all_dirty = false;                // a cross-rank completion filled rows this rank does not own
    std::vector<int> h_ia;                   // host copy of the CSR row starts (value range of the owned rows)

    // mesh
    int nV = 0, nT = 0, energy = 0;
    int t_begin = 0, t_end = 0;
    ipcgpu::DevBuf<double> V, Vsaved, Vrest, Ainv, vol, mu, lam, mass, Vprev, xtilde;
    bool prev_set = false, xtilde_set = false; // result.V_prev (friction) / xTilta (inertia) uploaded
    ipcgpu::DevBuf<int> T;
    ipcgpu::DevBuf<uint8_t> dbc;
    bool has_mass = false, has_dbc = false, state_saved = false;
    std::vector<int> h_T; // host copy of tets (maps are rebuilt when the partition changes)

    // surface (Mesh::SVI / SFEdges / SF) and contact workspace
    int nSV = 0, nSE = 0, nSF = 0;
    int nVdof = 0x7fffffff;  // first obstacle vertex (ipcgpu_set_obstacle_tail): vertices from here on have no degrees of freedom; INT_MAX = no obstacle
    int ee_as_vf = 1;        // Tight-Inclusion of mesh-obstacle edge pairs through the vertex-face routine, as MeshCO.cpp:1609 calls it
    ipcgpu::DevBuf<int> SVI, SE, SF, vCoDim;
    bool has_codim = false, surface_ready = false;
    int pair_capacity = 1 << 20;
    int exchange_capacity = 1 << 16; // pairs per rank and list in the fixed-size message of the cross-rank pair-list exchange
    // order of the contact lists (ipcgpu_set_canonical_order): 0 build order, 1 sorted lexicographically (lex_order), 2 sorted and every
    // contact sum taken in list order (the reproducible mode, ReproWork)
    int canonical_order = 1;
    ipcgpu::ReproWork rw;
    bool partition_contact = false, lists_local = false; // multi-rank: build only this rank's share of the contact sets
    ipcgpu::ContactWork cw;
    ipcgpu::CcdWork ccd;
    ipcgpu::PointTetWork pit;
    // half-space collision objects (halfspace.cu, ipcgpu_set_halfspaces): parameters, flags / scan of the (plane, SVI index) range, active and
    // lagged (plane, vertex) lists, per-plane starts of the active list, energy partials
    int n_hs = 0;
    ipcgpu::DevBuf<double> hs_par, hs_lam, hs_partials;
    ipcgpu::DevBuf<int> hs_flags, hs_offs, hs_cnt, hs_pstart; // hs_cnt: [0] active, [1] lagged
    ipcgpu::DevBuf<int2> hs_act, hs_lag;
    ipcgpu::DevBuf<unsigned char> hs_scan;
    size_t hs_scan_bytes = 0;
    bool hs_set_built = false, hs_lag_ready = false;
    // Rayleigh damping, Neumann forces and the Dirichlet penalty (damping.cu): D in slot order (9 doubles per slot) and its per-vertex slot
    // incidence (built once per mesh, at the first ipcgpu_damping_update); the summed Neumann force per vertex (interleaved); the Dirichlet
    // targets (vertex, target, multiplier).  A new mesh (build_maps) removes all three.
    bool damp_on = false, damp_inc_ready = false, nbc_on = false;
    int n_dbc = 0;
    ipcgpu::DevBuf<double> damp_D, damp_partials, nbc_f, nbc_partials, dbc_tgt, dbc_lam, dbc_partials;
    ipcgpu::DevBuf<int> damp_inc_ptr, damp_inc, dbc_vid;
    // time integration (timestep.cu): the parameters of ipcgpu_set_time_integration in device memory, and Optimizer's dynamic state --
    // velocity (interleaved), acceleration and dx_Elastic (SoA) -- for dyn_nV vertices (zeroed at the first use on a mesh of another size)
    ipcgpu::DevBuf<ipcgpu::TimeParams> tparams;
    ipcgpu::DevBuf<double> vel, acc, dxe;
    bool time_set = false;
    int dyn_nV = 0;
    // device-resident barrier stiffness (kappa.cu): g_c of initKappa and the per-CTA partials of its two dot products, and the close set of
    // postLineSearch (self / obstacle entries and plane entries, each with its saved d).  kp_pending: a kappa call was enqueued since the
    // last ipcgpu_kappa_info
    ipcgpu::DevBuf<double> kp_gc, kp_part, kp_close_mm_val, kp_close_hs_val;
    ipcgpu::DevBuf<int4> kp_close_mm;
    ipcgpu::DevBuf<int2> kp_close_hs;
    bool kp_pending = false, kp_pending_at_capture = false;
    // end-of-step diagnostics (diagnostics.cu): the components of ipcgpu_set_components (n_comp = 0: none; a new mesh removes them) as a
    // segment table with each component's first segment, the per-segment partials and the results of ipcgpu_system_energy (7 n_comp); the
    // partials and the result (n, d_min, d_max, |fb|) of ipcgpu_constraint_summary
    int n_comp = 0, n_seg = 0, comp_v_end = 0;
    ipcgpu::DevBuf<ipcgpu::DiagSegment> diag_seg;
    ipcgpu::DevBuf<int> diag_comp_seg;
    ipcgpu::DevBuf<double> diag_part, diag_sys, diag_sum_part, diag_sum;
    ipcgpu::DevBuf<unsigned long long> diag_sum_ord;
    size_t ccd_capacity = (size_t)1 << 23; // candidate pairs
    std::vector<int> h_SVI;                // host copy (pSize of the swept build is a serial host sum, SpatialHash.hpp:603-612)
    double debug_prune_seed = -1.0;        // test hook, see ipcgpu_ccd_debug_seed_bound
    long long debug_ti_budget = -1;        // test hook, see ipcgpu_ccd_debug_thread_budget
    bool debug_safeguard_flags = false;    // test hook, see ipcgpu_safeguard_debug_flags
    ipcgpu::DevBuf<int> dbg_tri_flags, dbg_tet_hits;

    // gradient gather map (local tets)
    ipcgpu::DevBuf<int> inc_ptr, inc;
    // Hessian slots (mesh-topology vertex pairs v<=u touched by local tets) and contributions
    int nSlots = 0, nOffSlots = 0; // (the off-diagonal slots come first: [0, nOffSlots))
    ipcgpu::DevBuf<int> slot_v, slot_u, slot_off, con_ptr;
    ipcgpu::DevBuf<unsigned> con_src;
    bool hblk_valid = false; // the last gradient/Hessian call left the per-tet Hessian blocks in hblk
    bool maps_ready = false, offsets_ready = false;

    // CSR
    int n_rows = 0, nnz = 0, index_base = 0;
    ipcgpu::DevBuf<int> ia, ja;
    ipcgpu::DevBuf<double> a;
    ipcgpu::DevBuf<int> flag; // device error flag
    // device-built pattern mode (ipcgpu_enable_device_pattern; ipcgpu_set_csr returns to host mode).  The host mirrors nnz / h_ia / a_begin,
    // a_end follow the device at every fetch (or wherever a host result needs them, see sync_pattern_mirror in api.cu); pat_pending: an
    // update was enqueued since they were last refreshed
    bool device_pattern = false, pat_pending = false;
    uint64_t pat_seen_version = 0;
    int pat_changed_host = 0;
    ipcgpu::PatternWork pw;
    // device-resident linear solve (solve.cu): full-row structure of the symmetric matrix, built on the device whenever the pattern's
    // version differs from the one it was built for (fp_cnt / fp_start / fp_cur / fp_tmp: counts, scan, scatter cursors, scan scratch),
    // + PCG workspace.  solve_epoch[m]: the epoch of the last eager solve of the block-Jacobi (0) / multilevel (1) / reserved AMG (2) solver, whose lazy
    // allocations a capture relies on; sv_pending: a solve was enqueued since ipcgpu_solve_info read it
    ipcgpu::DevBuf<int> fia, fja, fpos, fp_cnt, fp_start, fp_cur;
    ipcgpu::DevBuf<unsigned char> fp_tmp;
    ipcgpu::DevBuf<double> sol, pcg_b, pcg_r, pcg_p, pcg_q, pcg_minv, pcg_scal, pcg_part; // (pcg_part: per-CTA partials of the dot products)
    ipcgpu::MultilevelWork ml;
    ipcgpu::AmgWork amg;
    uint64_t solve_epoch[3] = { ~0ull, ~0ull, ~0ull };
    bool sv_pending = false, sv_pending_at_capture = false;
    // an elastic gradient / Hessian call wrote g / a since the last ipcgpu_set_state, ipcgpu_set_mesh or pattern change: what the diagonal
    // preconditioning (ipcgpu_precondition_diag, ipcgpu_warm_start option 5) reads is the system at the current state
    bool g_assembled = false, a_assembled = false;

    // work / result buffers
    ipcgpu::DevBuf<double> gcont, hblk, g, e_per_tet, partials, inv_steps, dir, in_partials, e_partials2;
    ipcgpu::DevBuf<double> packed_scalars; // the fetch's cross-rank sum (kPackedScalars)
    ipcgpu::DevBuf<double> pSize_dev; // mean |p| of the uploaded search direction, read by the swept-grid kernel from device memory (graph replay)

    // CUDA graphs of device-resident call sequences (ipcgpu_capture_begin / _end / ipcgpu_graph_launch).  A captured sequence mutates a
    // few host-side state words (which scalars are still rank-local, which lists are global ...); they are snapshotted at the end of the
    // capture and re-applied at every replay.  `epoch` is bumped by every call that may reallocate or re-partition: older graphs are refused.
    struct HostState {
        unsigned local_scalars;
        bool lists_local, lists_global, want_cand, swept_ready, fr_ready, inputs_marked, scatter_marked, hs_set_built, hs_lag_ready, rep_lists, rep_fr;
        bool g_assembled, a_assembled;
        int nC, nP, nK, fr_host_n;
    };
    struct GraphRec {
        cudaGraphExec_t exec = nullptr;
        cudaGraph_t graph = nullptr;
        uint64_t launches = 0, epoch = 0;
        bool dirty_at_begin = false;
        bool updates_pattern = false; // the sequence contains ipcgpu_update_pattern
        bool step_control = false;    // ... a CFL branch or a line search
        bool solve = false;           // ... a linear solve
        bool kappa = false;           // ... a call that writes the device-resident kappa
        std::vector<cudaGraph_t> bodies; // bodies of its conditional nodes (owned by `graph`)
        HostState hs;
    };
    std::vector<GraphRec> graphs;
    std::vector<cudaGraph_t> capture_bodies; // conditional-node bodies of the capture in progress
    // conditional graph nodes (abi.h: cond_node): the bodies of nested conditional nodes are captured on these high-priority streams, one per depth
    static constexpr int kCondDepth = 3;
    cudaStream_t cond_streams[kCondDepth] = { nullptr, nullptr, nullptr };
    int cond_depth = 0;
    bool sc_pending = false, sc_pending_at_capture = false; // a CFL branch / line search was enqueued since ipcgpu_step_control_info read it
    bool capturing = false, pat_pending_at_capture = false;
    uint64_t epoch = 0, launches_at_capture = 0;
    bool dirty_at_capture = false;
    ipcgpu::HostStaging* staging = nullptr; // pinned staging for scalars

    // profiling: event pairs per stage (only when enabled)
    bool profiling = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof[16];
    cudaEvent_t timer_a = nullptr, timer_b = nullptr;
    cudaEvent_t prof_begin(int stage)
    {
        if (!profiling) return nullptr;
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        prof[stage].emplace_back(a, b);
        cudaEventRecord(a, stream);
        return b;
    }
    void prof_end(cudaEvent_t b)
    {
        if (b) cudaEventRecord(b, stream);
    }

    ipcgpu::ElasticArgs eargs() const
    {
        ipcgpu::ElasticArgs p;
        p.nV = nV; p.nT = nT; p.t_begin = t_begin; p.t_end = t_end;
        p.n_list = n_list; p.tet_list = (nranks > 1) ? tet_list.p : nullptr;
        p.V = V.p; p.T = T.p; p.Ainv = Ainv.p; p.vol = vol.p; p.mu = mu.p; p.lam = lam.p; p.energy = energy;
        p.e_row_lo = (nranks > 1) ? v_begin : 0; p.e_row_hi = (nranks > 1) ? v_end : nV;
        return p;
    }
};
