// kappa.cu -- the barrier stiffness held in device memory (IterState::kappa*) and its adaptation under ADAPTIVE_KAPPA (src/Utils/Types.hpp:41):
//
//   Optimizer.cpp:2216-2233   suggestKappa / upperBoundKappa       ipcgpu_kappa_bounds (host), ipcgpu_set_kappa (stream order)
//   Optimizer.cpp:2236-2313   initKappa                            ipcgpu_kappa_init: g_c = J^T g_b(d) over the self / obstacle and plane active
//                                                                  sets, Dirichlet rows zeroed; g_c.g_E and g_c.g_c as fixed-order sums; one
//                                                                  thread takes the decision
//   Optimizer.cpp:2316-2322   initSubProb_IP                       ipcgpu_kappa_clear_close_set
//   Optimizer.cpp:2357-2445   postLineSearch                       ipcgpu_kappa_post_line_search: the saved close entries against the current
//                                                                  positions (an "any": order-free), the doubling, the new snapshot (atomic appends)
//
// No call synchronises except ipcgpu_kappa_info after a kappa call, so a whole time step with kappa on the device can be one graph.  The
// pair distances are pair_distance (the squared distance k_evaluate_constraints takes); the plane distances are rounded term by term, as the
// half-space kernels (halfspace.cu, built without contraction) evaluate them.
#include "abi.h"
#include "pair_common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

using namespace ipcgpu;

namespace {

constexpr int kKappaThreads = 256;
constexpr int kKappaBlocks = kSMs * 2;

// the squared distance of plane entry (plane, vertex) as k_hs_energy evaluates it
DEV double plane_d2(const double* __restrict__ par, const double* __restrict__ V, int nV, int2 e)
{
    const double* pl = par + kPlaneStride * e.x;
    const double x = V[e.y], y = V[(size_t)nV + e.y], z = V[(size_t)2 * nV + e.y];
    const double dist = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(pl[0], x), __dmul_rn(pl[1], y)), __dmul_rn(pl[2], z)), pl[3]);
    return __dmul_rn(dist, dist);
}

// the plane active set of postLineSearch / initKappa (nullptrs without planes)
struct PlaneSet {
    const double* par;
    const int2* act;
    const int* n;
};

__global__ void k_kappa_set(IterState* st, double kappa, double suggest, double max)
{
    if (threadIdx.x != 0) return;
    st->kappa = kappa;
    st->kappa_suggest = suggest;
    st->kappa_max = max;
    st->kappa_doublings = 0;
}

// ---- initKappa ---------------------------------------------------------------------------------------------------------------
// val[c] = g_b(d_c) in place (compute_g_b, Optimizer.cpp:2252-2273)
__global__ void __launch_bounds__(kKappaThreads) k_kappa_gb(const int* __restrict__ nC, double dHat, double* __restrict__ val)
{
    const int n = *nC;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        double b, db, d2b;
        barrier_all(val[c], dHat, b, db, d2b);
        val[c] = db;
    }
}
// g_c.segment<dim>(vI * dim).setZero() for every Dirichlet vertex (:2276-2278; result.DBCVertexIds: dbc != 0, the obstacle tail included)
__global__ void __launch_bounds__(kKappaThreads) k_kappa_zero_dbc(int nV, const uint8_t* __restrict__ dbc, double* __restrict__ gc)
{
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nV; v += gridDim.x * blockDim.x)
        if (dbc[v] != 0)
            for (int r = 0; r < 3; ++r) gc[3 * (size_t)v + r] = 0.0;
}
// per-CTA partials of g_c.g_E (partials[b]) and g_c.g_c (partials[nb + b]), fixed order
__global__ void __launch_bounds__(kKappaThreads) k_kappa_dots(int n, const double* __restrict__ gc, const double* __restrict__ gE, double* __restrict__ partials)
{
    __shared__ double tot[2];
    double v[2] = { 0.0, 0.0 };
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double c = gc[i];
        v[0] += c * gE[i];
        v[1] += c * c;
    }
    cta_sum<2>(v, tot);
    __syncthreads();
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = tot[0];
        partials[gridDim.x + blockIdx.x] = tot[1];
    }
}
// the decision of initKappa (:2240, :2281-2290) on IterState::kappa_dot
__global__ void k_kappa_init_decide(const int* __restrict__ nC, const int* __restrict__ n_plane, IterState* st)
{
    if (threadIdx.x != 0) return;
    st->kappa_needs_init = 0;
    if (*nC + (n_plane ? *n_plane : 0) == 0) return; // constraintStartInds.back() == 0: "start with default kappa"
    const double minKappa = -st->kappa_dot[0] / st->kappa_dot[1];
    st->kappa_min_last = minKappa;
    double kappa = st->kappa;
    if (minKappa > 0.0) kappa = minKappa;
    if (kappa < st->kappa_suggest) kappa = st->kappa_suggest; // suggestKappa(minKappa); if (kappa < minKappa) kappa = minKappa
    if (kappa > st->kappa_max) kappa = st->kappa_max;         // upperBoundKappa(kappa)
    st->kappa = kappa;
}

// ---- postLineSearch ----------------------------------------------------------------------------------------------------------
// any saved entry with d <= its saved d raises kappa_hit (nothing runs while kappa == 0)
__global__ void __launch_bounds__(kKappaThreads) k_kappa_check(BarrierArgs p, PlaneSet ps, const int4* __restrict__ mm, const double* __restrict__ mm_val, int cap_mm,
    const int2* __restrict__ hs, const double* __restrict__ hs_val, int cap_hs, IterState* st)
{
    if (st->kappa == 0.0) return;
    const int n_mm = min(st->kappa_n_close[0], cap_mm), n = n_mm + min(st->kappa_n_close[1], cap_hs);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const bool plane = i >= n_mm;
        const double d = plane ? plane_d2(ps.par, p.V, p.nV, hs[i - n_mm]) : pair_distance(mm[i], p.V, p.nV);
        if (d <= (plane ? hs_val[i - n_mm] : mm_val[i])) st->kappa_hit = 1;
    }
}
// kappa == 0: needs_init (initKappa is the caller's, and the snapshot is skipped).  Otherwise the doubling, capped (:2393-2396), and the close
// set emptied for the snapshot that follows
__global__ void k_kappa_double(IterState* st)
{
    if (threadIdx.x != 0) return;
    if (st->kappa == 0.0) {
        st->kappa_needs_init = 1;
        st->kappa_skip = 1;
    }
    else {
        st->kappa_skip = 0;
        if (st->kappa_hit) {
            double kappa = st->kappa * 2.0;
            if (kappa > st->kappa_max) kappa = st->kappa_max;
            st->kappa = kappa;
            ++st->kappa_doublings;
        }
        st->kappa_n_close[0] = st->kappa_n_close[1] = 0;
        st->kappa_dmin_ord = dbl_to_ord(INFINITY);
    }
    st->kappa_hit = 0;
}
// the new snapshot: every active entry with d < dTol (:2400-2440), and the least d over all of them (the reference logs it)
__global__ void __launch_bounds__(kKappaThreads) k_kappa_snapshot(BarrierArgs p, PlaneSet ps, double dTol, int4* __restrict__ mm, double* __restrict__ mm_val, int cap_mm,
    int2* __restrict__ hs, double* __restrict__ hs_val, int cap_hs, IterState* st)
{
    if (st->kappa_skip) return;
    const int nC = *p.nC, n = nC + (ps.n ? *ps.n : 0);
    double dmin = INFINITY;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const bool plane = i >= nC;
        const int4 e = plane ? make_int4(0, 0, 0, 0) : p.cs[i];
        const int2 q = plane ? ps.act[i - nC] : make_int2(0, 0);
        const double d = plane ? plane_d2(ps.par, p.V, p.nV, q) : pair_distance(e, p.V, p.nV);
        dmin = fmin(dmin, d);
        if (!(d < dTol)) continue;
        if (!plane) {
            const int s = atomicAdd(&st->kappa_n_close[0], 1);
            if (s < cap_mm) {
                mm[s] = e;
                mm_val[s] = d;
            }
        }
        else {
            const int s = atomicAdd(&st->kappa_n_close[1], 1);
            if (s < cap_hs) {
                hs[s] = q;
                hs_val[s] = d;
            }
        }
    }
    dmin = warp_min(dmin);
    if ((threadIdx.x & 31) == 0 && dmin < INFINITY) atomicMin(&st->kappa_dmin_ord, dbl_to_ord(fmax(dmin, 0.0)));
}

__global__ void k_kappa_clear(IterState* st)
{
    if (threadIdx.x != 0) return;
    st->kappa_n_close[0] = st->kappa_n_close[1] = 0;
}

// H_bC2 (BarrierFunctions.hpp:73-83)
double H_b(double d1, double dHat1)
{
    const double t2 = d1 - dHat1;
    return (std::log(d1 / dHat1) * -2.0 - t2 * 4.0 / d1) + 1.0 / (d1 * d1) * (t2 * t2);
}

} // namespace

#define REQUIRE_KAPPA_CTX()                                                                                                         \
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the device-resident kappa runs on one rank");                                    \
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");                                                     \
    REQUIRE(ctx->n_hs == 0 || ctx->hs_set_built, IPCGPU_ERR_STATE, "half-spaces: ipcgpu_halfspace_constraint_set first")

static PlaneSet plane_set(ipcgpu_ctx* ctx)
{
    if (ctx->n_hs == 0) return PlaneSet{ nullptr, nullptr, nullptr };
    return PlaneSet{ ctx->hs_par.p, ctx->hs_act.p, ctx->hs_cnt.p };
}

// the close set sized for the active lists it snapshots (ContactWork::cap entries, the planes' kMaxPlanes * nSV): no entry can be dropped.
// A reallocation empties it
static int close_set_alloc(ipcgpu_ctx* ctx)
{
    const size_t cap_mm = (size_t)std::max({ ctx->cw.cap, ctx->pair_capacity, 1 }), cap_hs = (size_t)kMaxPlanes * std::max(ctx->nSV, 1);
    if (ctx->kp_close_mm.n >= cap_mm && ctx->kp_close_hs.n >= cap_hs) return IPCGPU_OK;
    ALLOC(ctx->kp_close_mm, cap_mm);
    ALLOC(ctx->kp_close_mm_val, cap_mm);
    ALLOC(ctx->kp_close_hs, cap_hs);
    ALLOC(ctx->kp_close_hs_val, cap_hs);
    CK(cudaMemsetAsync(ctx->iter.p->kappa_n_close, 0, sizeof(ctx->iter.p->kappa_n_close), ctx->stream));
    return IPCGPU_OK;
}

// after a call that writes IterState::kappa: the pair-Hessian build of the next ipcgpu_barrier_hessian runs on the side stream, ordered only
// after ev_inputs (api_contact.cu), so the kappa it reads with IPCGPU_KAPPA_DEVICE is one of its inputs and is marked like the positions
static void kappa_written(ipcgpu_ctx* ctx)
{
    ctx->kp_pending = true;
    ctx->mark_inputs();
}

extern "C" {

int ipcgpu_kappa_bounds(double dHat, double kappa_min_multiplier, double avg_node_mass, double bbox_diag2, double* suggest, double* max)
{
    if (!(dHat > 0.0) || !(bbox_diag2 > 0.0) || !suggest || !max) return IPCGPU_ERR_ARG;
    const double Hb = H_b(1.0e-16 * bbox_diag2, dHat);
    *suggest = kappa_min_multiplier * avg_node_mass / (4.0e-16 * bbox_diag2 * Hb);
    *max = 100 * kappa_min_multiplier * avg_node_mass / (4.0e-16 * bbox_diag2 * Hb);
    return IPCGPU_OK;
}

int ipcgpu_set_kappa(ipcgpu_ctx* ctx, double kappa, double suggest, double max)
{
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the device-resident kappa runs on one rank");
    REQUIRE(kappa >= 0.0 && suggest >= 0.0 && max >= 0.0, IPCGPU_ERR_ARG, "kappa and its bounds must be >= 0");
    ENTER(kSerial);
    k_kappa_set<<<1, 32, 0, ctx->stream>>>(ctx->iter.p, kappa, suggest, max);
    ++ctx->launches;
    CK(cudaGetLastError());
    kappa_written(ctx);
    return IPCGPU_OK;
}

int ipcgpu_kappa_init(ipcgpu_ctx* ctx, double dHat)
{
    REQUIRE_KAPPA_CTX();
    REQUIRE(dHat > 0.0, IPCGPU_ERR_ARG, "dHat must be positive");
    ENTER(kSerial);
    const size_t n = (size_t)3 * ctx->nV;
    ALLOC(ctx->kp_gc, n);
    ALLOC(ctx->kp_part, 2 * (size_t)kKappaBlocks);
    REQUIRE(ctx->g.n >= n, IPCGPU_ERR_STATE, "no device gradient g_E: the NULL-output gradient calls first");
    ALLOC(ctx->cw.bval, (size_t)std::max(ctx->cw.cap, 1));
    const BarrierArgs p = barrier_args(ctx, dHat, 1.0, 0);
    const PlaneSet ps = plane_set(ctx);
    cudaStream_t st = ctx->stream;
    double* gc = ctx->kp_gc.p;
    // g_c (:2250-2279): the self / obstacle active set through evaluateConstraints and leftMultiplyConstraintJacobianT with input g_b(d),
    // the planes' through HalfSpace::leftMultiplyConstraintJacobianT with coefficient 1, then the Dirichlet rows
    CK(cudaMemsetAsync(gc, 0, n * sizeof(double), st));
    evaluate_constraints(p, ctx->cw.bval.p, st);
    k_kappa_gb<<<kKappaBlocks, kKappaThreads, 0, st>>>(p.nC, dHat, ctx->cw.bval.p);
    constraint_jacobian_t(p, ctx->cw.bval.p, 1.0, gc, st);
    ctx->launches += 3 + p.rep.on; // (+ the reproducible mode's gather)
    if (ps.n) {
        const HalfSpaceArgs hp = halfspace_args(ctx);
        halfspace_gradient(hp, dHat, 1.0, nullptr, gc, st);
        ctx->launches += 1 + (hp.rep_mask != nullptr);
    }
    if (ctx->has_dbc) {
        k_kappa_zero_dbc<<<std::min(nblk(ctx->nV, kKappaThreads), kKappaBlocks), kKappaThreads, 0, st>>>(ctx->nV, ctx->dbc.p, gc);
        ++ctx->launches;
    }
    const int nb = std::min(nblk((long long)n, kKappaThreads), kKappaBlocks);
    double* part = ctx->kp_part.p;
    IterState* ist = ctx->iter.p;
    k_kappa_dots<<<nb, kKappaThreads, 0, st>>>((int)n, gc, ctx->g.p, part);
    reduce_sum(part, nb, 1.0, &ist->kappa_dot[0], st);
    reduce_sum(part + nb, nb, 1.0, &ist->kappa_dot[1], st);
    k_kappa_init_decide<<<1, 32, 0, st>>>(p.nC, ps.n, ist);
    ctx->launches += 4;
    CK(cudaGetLastError());
    kappa_written(ctx);
    return IPCGPU_OK;
}

int ipcgpu_kappa_clear_close_set(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the device-resident kappa runs on one rank");
    ENTER(kSerial);
    k_kappa_clear<<<1, 32, 0, ctx->stream>>>(ctx->iter.p);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->kp_pending = true;
    return IPCGPU_OK;
}

int ipcgpu_kappa_post_line_search(ipcgpu_ctx* ctx, double dTol)
{
    REQUIRE_KAPPA_CTX();
    ENTER(kSerial);
    int rc = close_set_alloc(ctx);
    if (rc) return rc;
    const BarrierArgs p = barrier_args(ctx, 1.0, 1.0, 0);
    const PlaneSet ps = plane_set(ctx);
    const int cap_mm = (int)ctx->kp_close_mm.n, cap_hs = (int)ctx->kp_close_hs.n;
    cudaStream_t st = ctx->stream;
    IterState* ist = ctx->iter.p;
    k_kappa_check<<<kKappaBlocks, kKappaThreads, 0, st>>>(p, ps, ctx->kp_close_mm.p, ctx->kp_close_mm_val.p, cap_mm, ctx->kp_close_hs.p, ctx->kp_close_hs_val.p,
        cap_hs, ist);
    k_kappa_double<<<1, 32, 0, st>>>(ist);
    k_kappa_snapshot<<<kKappaBlocks, kKappaThreads, 0, st>>>(p, ps, dTol, ctx->kp_close_mm.p, ctx->kp_close_mm_val.p, cap_mm, ctx->kp_close_hs.p,
        ctx->kp_close_hs_val.p, cap_hs, ist);
    ctx->launches += 3;
    CK(cudaGetLastError());
    kappa_written(ctx);
    return IPCGPU_OK;
}

int ipcgpu_kappa_info(ipcgpu_ctx* ctx, ipcgpu_kappa* out)
{
    REQUIRE(out != nullptr, IPCGPU_ERR_ARG, "null output");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    if (ctx->kp_pending) {
        ENTER(kSerial);
        int rc = fetch_iter_state(ctx);
        if (rc) return rc;
        ctx->kp_pending = false;
    }
    const IterState& h = *ctx->h_iter;
    out->kappa = h.kappa;
    out->min_kappa = h.kappa_min_last;
    out->suggest = h.kappa_suggest;
    out->max = h.kappa_max;
    out->doublings = h.kappa_doublings;
    out->n_close = h.kappa_n_close[0] + h.kappa_n_close[1];
    out->needs_init = h.kappa_needs_init;
    // (the word is 0 before the first snapshot: reported as no entry)
    out->close_min_dist2 = INFINITY;
    if (h.kappa_dmin_ord) std::memcpy(&out->close_min_dist2, &h.kappa_dmin_ord, sizeof(double));
    return IPCGPU_OK;
}

} // extern "C"
