// api_terms.cu -- entry points of the remaining terms of the incremental potential: inertia, Rayleigh damping, Neumann forces, the
// augmented-Lagrangian Dirichlet penalty and the analytic half-space collision objects.
#include "abi.h"
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

using namespace ipcgpu;

// the dynamic state for the current mesh, zero when it was never set for a mesh of this size
static int dynamics_alloc(ipcgpu_ctx* ctx)
{
    if (ctx->dyn_nV == ctx->nV) return IPCGPU_OK;
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "set the dynamic state (ipcgpu_set_dynamics) outside a capture first");
    const size_t n = (size_t)3 * ctx->nV;
    ALLOC(ctx->vel, n);
    ALLOC(ctx->acc, n);
    ALLOC(ctx->dxe, n);
    for (double* b : { ctx->vel.p, ctx->acc.p, ctx->dxe.p }) CK(cudaMemsetAsync(b, 0, n * sizeof(double), ctx->stream));
    ctx->dyn_nV = ctx->nV;
    return IPCGPU_OK;
}

// the state every per-vertex time-integration call needs: the parameters, V_prev of this mesh, and the dynamic state
int timestep_prepare(ipcgpu_ctx* ctx, DynamicsArgs* p)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(ctx->time_set, IPCGPU_ERR_STATE, "ipcgpu_set_time_integration first");
    REQUIRE(ctx->prev_set && ctx->Vprev.n >= (size_t)3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first");
    int rc = dynamics_alloc(ctx);
    if (rc) return rc;
    ALLOC(ctx->xtilde, (size_t)3 * ctx->nV);
    p->nV = ctx->nV;
    p->tp = ctx->tparams.p;
    p->dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    p->vel = ctx->vel.p; p->acc = ctx->acc.p; p->dxe = ctx->dxe.p;
    p->V = ctx->V.p; p->Vprev = ctx->Vprev.p; p->xtilde = ctx->xtilde.p;
    return IPCGPU_OK;
}

extern "C" {

// ---- inertia term (Optimizer.cpp:3227-3239, :3439-3450) ---------------------------------------------------------------------
int ipcgpu_set_xtilde(ipcgpu_ctx* ctx, const double* xtilde_soa)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(xtilde_soa != nullptr, IPCGPU_ERR_ARG, "null xTilta");
    ENTER(kSerial);
    ALLOC(ctx->xtilde, (size_t)3 * ctx->nV);
    CK(cudaMemcpyAsync(ctx->xtilde.p, xtilde_soa, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->xtilde_set = true;
    return IPCGPU_OK;
}

// ---- time integration (timestep.cu): Optimizer::setTime (:421-428), computeXTilta (:1236-1278), the end of a time step (:572-590) -------------
int ipcgpu_set_time_integration(ipcgpu_ctx* ctx, int type, double dt, double beta, double gamma, const double gravity[3])
{
    REQUIRE(type == 0 || type == 1, IPCGPU_ERR_ARG, "time integration type: 0 (TIT_BE) or 1 (TIT_NM)");
    REQUIRE(gravity != nullptr, IPCGPU_ERR_ARG, "null gravity");
    REQUIRE(dt > 0.0 && (type == 0 || beta > 0.0), IPCGPU_ERR_ARG, "dt, and beta of a Newmark integration, must be positive");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "set the time integration outside a capture (a replay reads the values held on the device)");
    ENTER(kSerial);
    TimeParams q = {};
    q.type = type;
    q.dt = dt;
    q.dtSq = dt * dt;
    q.beta = beta;
    q.gamma = gamma;
    for (int d = 0; d < 3; ++d) {
        q.gravity[d] = gravity[d];
        q.gDtSq[d] = q.dtSq * gravity[d];
    }
    ALLOC(ctx->tparams, 1);
    CK(cudaMemcpyAsync(ctx->tparams.p, &q, sizeof q, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream)); // `q` lives on this stack
    ctx->time_set = true;
    return IPCGPU_OK;
}

int ipcgpu_set_dynamics(ipcgpu_ctx* ctx, const double* velocity, const double* acceleration_soa, const double* dx_elastic_soa)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    ctx->dyn_nV = 0; // (re)sized and zeroed, then the given arrays
    int rc = dynamics_alloc(ctx);
    if (rc) return rc;
    const size_t bytes = (size_t)3 * ctx->nV * sizeof(double);
    if (velocity) CK(cudaMemcpyAsync(ctx->vel.p, velocity, bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (acceleration_soa) CK(cudaMemcpyAsync(ctx->acc.p, acceleration_soa, bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (dx_elastic_soa) CK(cudaMemcpyAsync(ctx->dxe.p, dx_elastic_soa, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream)); // (the arrays are the caller's: the upload completes here)
    return IPCGPU_OK;
}

int ipcgpu_get_dynamics(ipcgpu_ctx* ctx, double* velocity, double* acceleration_soa, double* dx_elastic_soa)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    int rc = dynamics_alloc(ctx);
    if (rc) return rc;
    const size_t bytes = (size_t)3 * ctx->nV * sizeof(double);
    if (velocity) CK(cudaMemcpyAsync(velocity, ctx->vel.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (acceleration_soa) CK(cudaMemcpyAsync(acceleration_soa, ctx->acc.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (dx_elastic_soa) CK(cudaMemcpyAsync(dx_elastic_soa, ctx->dxe.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_compute_xtilde(ipcgpu_ctx* ctx)
{
    ENTER(kSerial);
    DynamicsArgs p;
    int rc = timestep_prepare(ctx, &p);
    if (rc) return rc;
    timestep_xtilde(p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->xtilde_set = true;
    return IPCGPU_OK;
}

int ipcgpu_end_time_step(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->xtilde_set, IPCGPU_ERR_STATE, "no xTilta for the step that ends: ipcgpu_compute_xtilde (or ipcgpu_set_xtilde) first");
    ENTER(kSerial);
    DynamicsArgs p;
    int rc = timestep_prepare(ctx, &p);
    if (rc) return rc;
    timestep_end(p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_inertia_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE(ctx->xtilde_set && ctx->has_mass, IPCGPU_ERR_STATE, "ipcgpu_set_xtilde and a mass diagonal (ipcgpu_set_mesh) first");
    ENTER(kSerial);
    // vertex blocks [nV r / N, nV (r+1) / N): every vertex exactly once across the ranks
    const int v0 = (int)((long long)ctx->nV * ctx->rank / ctx->nranks), v1 = (int)((long long)ctx->nV * (ctx->rank + 1) / ctx->nranks);
    ALLOC(ctx->in_partials, (size_t)inertia_energy_blocks(ctx->nV) + 8);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
    inertia_energy(v0, v1, ctx->nV, ctx->V.p, ctx->xtilde.p, ctx->mass.p, ctx->in_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyInertia, ctx->in_partials.p, inertia_energy_blocks(v1 - v0), 1.0, pe, E);
}

int ipcgpu_inertia_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE(ctx->xtilde_set && ctx->has_mass, IPCGPU_ERR_STATE, "ipcgpu_set_xtilde and a mass diagonal (ipcgpu_set_mesh) first");
    ENTER(kSerial);
    if (g_inout) CK(cudaMemcpyAsync(ctx->g.p, g_inout, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    // Device-resident form with several ranks: the gradient is summed over the ranks later (ipcgpu_allreduce_grad_hess), so only rank 0 adds
    // the per-vertex term.  Host form: every rank holds the caller's vector and adds the full term -- no reduction needed, which is why this
    // is not a gradient_call (whose host form sums the ranks' vectors).
    if (g_inout || ctx->nranks == 1 || ctx->rank == 0) {
        inertia_gradient(ctx->nV, ctx->V.p, ctx->xtilde.p, ctx->mass.p, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, ctx->g.p, ctx->stream);
        ++ctx->launches;
    }
    CK(cudaGetLastError());
    if (g_inout) {
        CK(cudaMemcpyAsync(g_inout, ctx->g.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return IPCGPU_OK;
}

// ---- Rayleigh damping, Neumann forces, augmented-Lagrangian Dirichlet penalty (damping.cu; which chain each call runs on: see enter()) ------
#define REQUIRE_ONE_RANK() REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "damping, Neumann forces and the Dirichlet penalty run on one rank")

// a term switched on or off: graphs that bake the line search's set of terms in are refused, and the term's energy slot reads 0 while it is off
static int term_switched(ipcgpu_ctx* ctx, int slot)
{
    ++ctx->epoch;
    CK(cudaMemsetAsync(&ctx->iter.p->energy[slot], 0, sizeof(double), ctx->stream));
    return IPCGPU_OK;
}

static DampingArgs damping_args(ipcgpu_ctx* ctx)
{
    DampingArgs p;
    p.nV = ctx->nV; p.nSlots = ctx->nSlots;
    p.slot_v = ctx->slot_v.p; p.slot_u = ctx->slot_u.p;
    p.inc_ptr = ctx->damp_inc_ptr.p; p.inc = ctx->damp_inc.p;
    p.D = ctx->damp_D.p;
    p.V = ctx->V.p; p.Vprev = ctx->Vprev.p;
    p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    return p;
}

// the slot incidence of every vertex (once per mesh): the slots in which it is slot_v (entry 2s), then those in which it is the slot_u of an
// off-diagonal slot (2s + 1), each group in slot order
static int damping_incidence(ipcgpu_ctx* ctx)
{
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "run ipcgpu_damping_update once outside a capture first (it builds the slot incidence)");
    const int nS = ctx->nSlots, nV = ctx->nV;
    std::vector<int> sv((size_t)std::max(nS, 1)), su((size_t)std::max(nS, 1));
    CK(cudaMemcpyAsync(sv.data(), ctx->slot_v.p, (size_t)nS * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(su.data(), ctx->slot_u.p, (size_t)nS * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<int> ptr((size_t)nV + 1, 0);
    for (int s = 0; s < nS; ++s) {
        ++ptr[(size_t)sv[s] + 1];
        if (sv[s] != su[s]) ++ptr[(size_t)su[s] + 1];
    }
    for (int v = 0; v < nV; ++v) ptr[(size_t)v + 1] += ptr[v];
    std::vector<int> inc((size_t)std::max(ptr[nV], 1)), cur(ptr.begin(), ptr.end() - 1);
    for (int s = 0; s < nS; ++s) inc[(size_t)cur[sv[s]]++] = 2 * s;
    for (int s = 0; s < nS; ++s)
        if (sv[s] != su[s]) inc[(size_t)cur[su[s]]++] = 2 * s + 1;
    REQUIRE(ctx->damp_inc_ptr.upload(ptr.data(), ptr.size(), ctx->stream) && ctx->damp_inc.upload(inc.data(), inc.size(), ctx->stream), IPCGPU_ERR_CUDA,
        "upload of the damping incidence failed");
    CK(cudaStreamSynchronize(ctx->stream)); // host vectors go out of scope
    ctx->damp_inc_ready = true;
    return IPCGPU_OK;
}

int ipcgpu_damping_update(ipcgpu_ctx* ctx, double coef)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    int rc;
    if (coef == 0.0) { // no damping term
        if (ctx->damp_on && (rc = term_switched(ctx, kEnergyDamping))) return rc;
        ctx->damp_on = false;
        return IPCGPU_OK;
    }
    if (!ctx->damp_inc_ready && (rc = damping_incidence(ctx))) return rc;
    ALLOC(ctx->damp_D, (size_t)9 * std::max(ctx->nSlots, 1));
    ALLOC(ctx->damp_partials, (size_t)damping_energy_blocks(ctx->nSlots) + 8);
    // computeDampingMtr (Optimizer.cpp:3723-3734): the elastic Hessian at the current state, coef, projected (projectSPD = projectDBC = 1)
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    elastic_grad_hess(ctx->eargs(), coef, 1, false, true, ctx->gcont.p, ctx->hblk.p, ctx->stream);
    ctx->hblk_valid = true; // (IPCGPU_BUF_TET_HESSIANS now holds the damping's per-tet blocks)
    damping_assemble(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->con_ptr.p, ctx->con_src.p, ctx->hblk.p, ctx->has_dbc ? ctx->dbc.p : nullptr,
        ctx->damp_D.p, ctx->stream);
    ctx->prof_end(pe);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (!ctx->damp_on && (rc = term_switched(ctx, kEnergyDamping))) return rc;
    ctx->damp_on = true;
    return IPCGPU_OK;
}

#define REQUIRE_DAMPING()                                                                                                \
    REQUIRE(ctx->damp_on, IPCGPU_ERR_STATE, "ipcgpu_damping_update with a nonzero coefficient first");                  \
    REQUIRE(ctx->prev_set, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first");                                              \
    REQUIRE_ONE_RANK()

int ipcgpu_damping_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE_DAMPING();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    damping_energy(damping_args(ctx), ctx->damp_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyDamping, ctx->damp_partials.p, damping_energy_blocks(ctx->nSlots), 0.5, pe, E);
}

int ipcgpu_damping_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE_DAMPING();
    const DampingArgs p = damping_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { damping_gradient(p, projectDBC, ctx->g.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_damping_hessian(ipcgpu_ctx* ctx, double* a_inout)
{
    REQUIRE_DAMPING();
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    if (!ctx->offsets_ready) { // (the slot offsets of a new host pattern: one synchronising check, as the first elastic Hessian does)
        ENTER(kSerial);
        int rc = ensure_offsets(ctx);
        if (rc) return rc;
    }
    const DampingArgs p = damping_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { damping_hessian(p, ctx->slot_off.p, ctx->a.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_set_neumann_forces(ipcgpu_ctx* ctx, double coef, const double* f)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(!f || ctx->has_mass, IPCGPU_ERR_STATE, "Neumann forces need the mass diagonal (ipcgpu_set_mesh)");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    int rc;
    if (f) {
        ALLOC(ctx->nbc_f, (size_t)3 * ctx->nV);
        ALLOC(ctx->nbc_partials, (size_t)vertex_energy_blocks(ctx->nV) + 8);
        CK(cudaMemcpyAsync(ctx->nbc_f.p, f, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream)); // (f is the caller's: the upload completes here)
    }
    set_double(&ctx->iter.p->nbc_coef, coef, ctx->stream); // (read at run time, like the forces: a new dt needs no new capture)
    ++ctx->launches;
    CK(cudaGetLastError());
    if ((f != nullptr) != ctx->nbc_on && (rc = term_switched(ctx, kEnergyNeumann))) return rc;
    ctx->nbc_on = f != nullptr;
    return IPCGPU_OK;
}

#define REQUIRE_NEUMANN()                                                                                   \
    REQUIRE(ctx->nbc_on, IPCGPU_ERR_STATE, "ipcgpu_set_neumann_forces first");                             \
    REQUIRE_ONE_RANK()

int ipcgpu_neumann_energy(ipcgpu_ctx* ctx, double* E)
{
    REQUIRE_NEUMANN();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    neumann_energy(ctx->nV, ctx->V.p, ctx->nbc_f.p, ctx->mass.p, ctx->has_dbc ? ctx->dbc.p : nullptr, &ctx->iter.p->nbc_coef, ctx->nbc_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyNeumann, ctx->nbc_partials.p, vertex_energy_blocks(ctx->nV), 1.0, pe, E);
}

int ipcgpu_neumann_gradient(ipcgpu_ctx* ctx, double* g_inout)
{
    REQUIRE_NEUMANN();
    const uint8_t* dbc = ctx->has_dbc ? ctx->dbc.p : nullptr;
    const double* coef = &ctx->iter.p->nbc_coef;
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { neumann_gradient(ctx->nV, ctx->nbc_f.p, ctx->mass.p, dbc, coef, ctx->g.p, st); },
        IPCGPU_STAGE_DAMPING_BC);
}

static DirichletArgs dirichlet_args(ipcgpu_ctx* ctx)
{
    DirichletArgs p;
    p.n = ctx->n_dbc; p.nV = ctx->nV;
    p.vid = ctx->dbc_vid.p; p.tgt = ctx->dbc_tgt.p; p.lam = ctx->dbc_lam.p;
    p.V = ctx->V.p; p.mass = ctx->mass.p;
    p.rho = &ctx->iter.p->dbc_rho;
    return p;
}

int ipcgpu_set_dirichlet_targets(ipcgpu_ctx* ctx, int n, const int* vid, const double* target, const double* lambda, double dist2Tol)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(n >= 0 && (n == 0 || (vid && target)), IPCGPU_ERR_ARG, "ipcgpu_set_dirichlet_targets: bad arguments");
    REQUIRE(n == 0 || ctx->has_mass, IPCGPU_ERR_STATE, "the Dirichlet penalty needs the mass diagonal (ipcgpu_set_mesh)");
    {
        // targetPos is a map: one target per vertex (the gradient / Hessian kernels update a vertex's rows from one thread)
        std::vector<char> seen((size_t)ctx->nV, 0);
        for (int i = 0; i < n; ++i) {
            REQUIRE(vid[i] >= 0 && vid[i] < ctx->nV, IPCGPU_ERR_ARG, "Dirichlet target vertex out of range");
            REQUIRE(!seen[(size_t)vid[i]], IPCGPU_ERR_ARG, "Dirichlet target vertices must be distinct");
            seen[(size_t)vid[i]] = 1;
        }
    }
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    if (n > 0) {
        ALLOC(ctx->dbc_vid, (size_t)n);
        ALLOC(ctx->dbc_tgt, (size_t)3 * n);
        ALLOC(ctx->dbc_lam, (size_t)3 * n);
        ALLOC(ctx->dbc_partials, (size_t)vertex_energy_blocks(n) + 8);
        CK(cudaMemcpyAsync(ctx->dbc_vid.p, vid, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->dbc_tgt.p, target, (size_t)3 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        if (lambda) CK(cudaMemcpyAsync(ctx->dbc_lam.p, lambda, (size_t)3 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        else CK(cudaMemsetAsync(ctx->dbc_lam.p, 0, (size_t)3 * n * sizeof(double), ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream)); // (the arrays are the caller's: the upload completes here)
    }
    // the number of targets is a launch shape (a new number needs a new capture); the same number with new values does not
    if (n != ctx->n_dbc) {
        int rc = term_switched(ctx, kEnergyDirichlet);
        if (rc) return rc;
    }
    ctx->n_dbc = n;
    set_double(&ctx->iter.p->dbc_tol, n ? dist2Tol : 0.0, ctx->stream); // (stream order: a new dist2Tol per time step needs no new capture)
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_set_dirichlet_penalty(ipcgpu_ctx* ctx, double rho)
{
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    set_double(&ctx->iter.p->dbc_rho, rho, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_get_dirichlet_lambda(ipcgpu_ctx* ctx, double* lambda)
{
    REQUIRE(lambda != nullptr, IPCGPU_ERR_ARG, "null output");
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    if (ctx->n_dbc > 0) CK(cudaMemcpyAsync(lambda, ctx->dbc_lam.p, (size_t)3 * ctx->n_dbc * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_dirichlet_energy(ipcgpu_ctx* ctx, double* E)
{
    if (E) *E = 0.0;
    REQUIRE_ONE_RANK();
    if (ctx->n_dbc == 0) return IPCGPU_OK;
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_DAMPING_BC);
    dirichlet_energy(dirichlet_args(ctx), ctx->dbc_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyDirichlet, ctx->dbc_partials.p, vertex_energy_blocks(ctx->n_dbc), 1.0, pe, E);
}

int ipcgpu_dirichlet_gradient(ipcgpu_ctx* ctx, int projectDBC, double* g_inout)
{
    REQUIRE_ONE_RANK();
    if (ctx->n_dbc == 0) return IPCGPU_OK;
    if (projectDBC) return IPCGPU_OK; // (Optimizer.cpp:3542)
    const DirichletArgs p = dirichlet_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) { dirichlet_gradient(p, ctx->g.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_dirichlet_hessian(ipcgpu_ctx* ctx, int projectDBC, double* a_inout)
{
    REQUIRE_ONE_RANK();
    if (ctx->n_dbc == 0) return IPCGPU_OK;
    if (projectDBC) return IPCGPU_OK; // (:3711)
    const DirichletArgs p = dirichlet_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) { dirichlet_hessian(p, ctx->ia.p, ctx->index_base, ctx->a.p, st); }, IPCGPU_STAGE_DAMPING_BC);
}

int ipcgpu_dirichlet_update_lambda(ipcgpu_ctx* ctx)
{
    REQUIRE_ONE_RANK();
    if (ctx->n_dbc == 0) return IPCGPU_OK;
    ENTER(kSerial);
    dirichlet_update_lambda(dirichlet_args(ctx), ctx->dbc_lam.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_dirichlet_completed_step(ipcgpu_ctx* ctx, double* s)
{
    REQUIRE_ONE_RANK();
    ENTER(kSerial);
    ALLOC(ctx->dbc_partials, (size_t)vertex_energy_blocks(ctx->n_dbc) + 8);
    dirichlet_completed_step(dirichlet_args(ctx), &ctx->iter.p->dbc_tol, ctx->dbc_partials.p, &ctx->iter.p->dbc_step, ctx->stream);
    ctx->launches += ctx->n_dbc ? 3 : 2;
    CK(cudaGetLastError());
    if (!s) return IPCGPU_OK;
    CK(cudaMemcpyAsync(&ctx->staging->scalar, &ctx->iter.p->dbc_step, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *s = ctx->staging->scalar;
    return IPCGPU_OK;
}

// ---- analytic half-space collision objects (halfspace.cu; which chain each call runs on: see enter()) ------------------------------------
} // extern "C"

HalfSpaceArgs halfspace_args(ipcgpu_ctx* ctx)
{
    HalfSpaceArgs p;
    p.nV = ctx->nV; p.nSV = ctx->nSV; p.nP = ctx->n_hs;
    p.SVI = ctx->SVI.p; p.V = ctx->V.p; p.Vt = ctx->Vprev.p;
    p.dbc = ctx->has_dbc ? ctx->dbc.p : nullptr; p.vCoDim = ctx->has_codim ? ctx->vCoDim.p : nullptr;
    p.par = ctx->hs_par.p;
    p.act = ctx->hs_act.p; p.n_act = ctx->hs_cnt.p;
    p.lag = ctx->hs_lag.p; p.lam = ctx->hs_lam.p; p.n_lag = ctx->hs_cnt.p + 1;
    p.row_lo = ctx->nranks > 1 ? ctx->v_begin : 0;
    p.row_hi = ctx->nranks > 1 ? ctx->v_end : ctx->nV;
    p.ia = ctx->ia.p; p.base = ctx->index_base;
    if (repro_on(ctx) && ctx->rw.nV >= ctx->nV && ctx->rw.nSV >= ctx->nSV) { // the reproducible mode: every vertex adds its planes in plane order
        p.rep_mask = ctx->rw.hs_mask.p;
        p.rep_pos = ctx->rw.hs_pos.p;
        p.rep_stage = ctx->rw.hs_stage.p;
    }
    return p;
}

extern "C" {

int ipcgpu_set_halfspaces(ipcgpu_ctx* ctx, int n, const double* origin, const double* normal, const double* velocitydt, const double* friction)
{
    REQUIRE(n >= 0 && n <= kMaxPlanes, IPCGPU_ERR_ARG, "at most 8 half-spaces");
    REQUIRE(n == 0 || (origin && normal && friction), IPCGPU_ERR_ARG, "null half-space arrays");
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    std::vector<double> par((size_t)kPlaneStride * std::max(n, 1), 0.0);
    for (int k = 0; k < n; ++k) {
        const double* o = origin + 3 * k;
        const double* nr = normal + 3 * k;
        const double z = (nr[0] * nr[0] + nr[1] * nr[1]) + nr[2] * nr[2]; // normal.normalize() (HalfSpace.cpp:49)
        REQUIRE(z > 0.0, IPCGPU_ERR_ARG, "half-space normal is zero");
        const double s = std::sqrt(z);
        double* q = par.data() + kPlaneStride * k;
        for (int r = 0; r < 3; ++r) q[r] = nr[r] / s;
        q[3] = -((q[0] * o[0] + q[1] * o[1]) + q[2] * o[2]); // D = -normal.dot(origin) (:51)
        for (int r = 0; r < 3; ++r) q[4 + r] = velocitydt ? velocitydt[3 * k + r] : 0.0;
        q[7] = friction[k];
    }
    if (n != ctx->n_hs) {
        ++ctx->epoch; // the graphs captured with the old number of planes are refused (launch shapes and calls change)
        ctx->hs_set_built = ctx->hs_lag_ready = false;
        // the plane energies and the hs_* words start from zero, and no rank-local share of the old planes is left for the fetch to sum
        IterState* ist = ctx->iter.p;
        CK(cudaMemsetAsync(&ist->energy[kEnergyPlaneBarrier], 0, sizeof(double), ctx->stream));
        CK(cudaMemsetAsync(&ist->energy[kEnergyPlaneFriction], 0, sizeof(double), ctx->stream));
        CK(cudaMemsetAsync(&ist->hs_alpha, 0, offsetof(IterState, pat_nnz) - offsetof(IterState, hs_alpha), ctx->stream));
        set_local(ctx, (1u << kEnergyPlaneBarrier) | (1u << kEnergyPlaneFriction) | kLocalCrossings, false);
    }
    ctx->n_hs = n;
    if (n > 0) {
        ALLOC(ctx->hs_par, (size_t)kPlaneStride * kMaxPlanes);
        CK(cudaMemcpyAsync(ctx->hs_par.p, par.data(), par.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream)); // `par` lives on this stack
    return IPCGPU_OK;
}

// allocations sized by the surface (lazy: the first call after ipcgpu_set_surface, which refuses older graphs, must run outside a capture)
static int halfspace_alloc(ipcgpu_ctx* ctx)
{
    const size_t n = (size_t)kMaxPlanes * std::max(ctx->nSV, 1);
    ALLOC(ctx->hs_flags, n);
    ALLOC(ctx->hs_offs, n);
    ALLOC(ctx->hs_act, n);
    ALLOC(ctx->hs_lag, n);
    ALLOC(ctx->hs_lam, n);
    ALLOC(ctx->hs_cnt, 2);
    ALLOC(ctx->hs_pstart, kMaxPlanes + 1);
    ALLOC(ctx->hs_partials, (size_t)halfspace_energy_blocks() + 8);
    // the scan's temporary storage grows with its length (decoupled look-back tile state): sized for the scan this surface and this number of
    // planes run, at every call (a host-only query), and the size handed to cub is that one
    ctx->hs_scan_bytes = halfspace_scan_bytes(ctx->n_hs * ctx->nSV);
    ALLOC(ctx->hs_scan, ctx->hs_scan_bytes);
    return IPCGPU_OK;
}

static int halfspace_sync_counts(ipcgpu_ctx* ctx)
{
    CK(cudaMemcpyAsync(ctx->staging->hs_count, ctx->hs_cnt.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_halfspace_constraint_set(ipcgpu_ctx* ctx, double dHat, int* n_active)
{
    if (n_active) *n_active = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE(ctx->surface_ready && ctx->nSV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_surface with surface vertices first");
    ENTER(kSerial);
    int rc = halfspace_alloc(ctx);
    if (rc) return rc;
    const HalfSpaceArgs p = halfspace_args(ctx);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_CONSTRAINT_SET);
    CK(halfspace_active_set(p, dHat, ctx->hs_flags.p, ctx->hs_offs.p, ctx->hs_scan.p, ctx->hs_scan_bytes, ctx->hs_act.p, ctx->hs_cnt.p, ctx->hs_pstart.p,
        ctx->iter.p, ctx->stream));
    ctx->prof_end(pe);
    ctx->launches += 3;
    ctx->hs_set_built = true;
    ctx->mark_inputs();
    if (n_active) {
        if ((rc = halfspace_sync_counts(ctx))) return rc;
        *n_active = ctx->staging->hs_count[0];
    }
    return IPCGPU_OK;
}

#define REQUIRE_HS_SET() REQUIRE(ctx->hs_set_built, IPCGPU_ERR_STATE, "ipcgpu_halfspace_constraint_set first")

int ipcgpu_halfspace_energy(ipcgpu_ctx* ctx, double dHat, double kappa, double* E)
{
    if (E) *E = 0.0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    REQUIRE_KAPPA(kappa);
    ENTER(kSerial);
    const HalfSpaceArgs p = halfspace_args(ctx);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    halfspace_energy(p, dHat, ctx->hs_partials.p, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE], ctx->stream);
    return energy_tail(ctx, kEnergyPlaneBarrier, ctx->hs_partials.p, halfspace_energy_blocks(), kappa, pe, E, true, 1u << FLAG_NONPOSITIVE_DISTANCE,
        kappa_ptr(ctx, kappa));
}

int ipcgpu_halfspace_gradient(ipcgpu_ctx* ctx, double dHat, double kappa, double* g_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    REQUIRE_KAPPA(kappa);
    const HalfSpaceArgs p = halfspace_args(ctx);
    const double* kd = kappa_ptr(ctx, kappa);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) {
        halfspace_gradient(p, dHat, kappa, kd, ctx->g.p, st);
        ctx->launches += p.rep_mask != nullptr; // (the reproducible mode's per-vertex add)
    });
}

int ipcgpu_halfspace_hessian(ipcgpu_ctx* ctx, double dHat, double kappa, int projectDBC, double* a_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    REQUIRE_KAPPA(kappa);
    const HalfSpaceArgs p = halfspace_args(ctx);
    const double* kd = kappa_ptr(ctx, kappa);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) {
        halfspace_hessian(p, dHat, kappa, kd, projectDBC, ctx->a.p, st);
        ctx->launches += p.rep_mask != nullptr;
    });
}

int ipcgpu_halfspace_step(ipcgpu_ctx* ctx, const double* p_dir, double slackness, double* alpha_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE(ctx->surface_ready, IPCGPU_ERR_STATE, "ipcgpu_set_surface first");
    ENTER(p_dir || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p_dir);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    halfspace_step(halfspace_args(ctx), ctx->dir.p, slackness, ctx->iter.p, ctx->stream);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (!alpha_inout) return IPCGPU_OK;
    if ((rc = ccd_read_back(ctx, alpha_inout))) return rc;
    if (ctx->h_iter->hs_zero_step) {
        CK(cudaMemsetAsync(&ctx->iter.p->hs_zero_step, 0, sizeof(int), ctx->stream));
        ctx->err = "step 0: a vertex is at or behind a half-space and moves further into it (Optimizer.cpp:2031-2033 would exit(-1))";
        return IPCGPU_ERR_LINE_SEARCH;
    }
    return IPCGPU_OK;
}

int ipcgpu_halfspace_crossings(ipcgpu_ctx* ctx, int* n)
{
    if (n) *n = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    ENTER(kSerial);
    halfspace_crossings(halfspace_args(ctx), ctx->iter.p, ctx->stream);
    ctx->launches += 2;
    CK(cudaGetLastError());
    set_local(ctx, kLocalCrossings, ctx->nranks > 1 && !n);
    if (!n) return IPCGPU_OK;
    int rc = nccl_sum(ctx, &ctx->iter.p->hs_crossings, 1, "ncclAllReduce(half-space crossings) failed");
    if (rc || (rc = fetch_iter_state(ctx))) return rc;
    *n = ctx->h_iter->hs_crossings;
    return IPCGPU_OK;
}

int ipcgpu_halfspace_friction_lag(ipcgpu_ctx* ctx, double dHat, double kappa, int* n_lagged)
{
    if (n_lagged) *n_lagged = 0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_SET();
    REQUIRE_KAPPA(kappa);
    ENTER(kSerial);
    halfspace_lag(halfspace_args(ctx), dHat, kappa, kappa_ptr(ctx, kappa), ctx->hs_pstart.p, ctx->hs_lag.p, ctx->hs_lam.p, ctx->hs_cnt.p + 1, &ctx->iter.p->flags[FLAG_NONPOSITIVE_DISTANCE],
        ctx->iter.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->hs_lag_ready = true;
    if (n_lagged) {
        int rc = halfspace_sync_counts(ctx);
        if (rc) return rc;
        *n_lagged = ctx->staging->hs_count[1];
    }
    return IPCGPU_OK;
}

#define REQUIRE_HS_LAG()                                                                                            \
    REQUIRE(ctx->hs_lag_ready, IPCGPU_ERR_STATE, "ipcgpu_halfspace_friction_lag first");                          \
    REQUIRE(ctx->prev_set, IPCGPU_ERR_STATE, "ipcgpu_set_prev_state first");                                       \
    REQUIRE(eps2 > 0.0, IPCGPU_ERR_ARG, "fricDHat must be positive")

int ipcgpu_halfspace_friction_energy(ipcgpu_ctx* ctx, double eps2, double* E)
{
    if (E) *E = 0.0;
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_BARRIER);
    halfspace_friction_energy(halfspace_args(ctx), eps2, ctx->hs_partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyPlaneFriction, ctx->hs_partials.p, halfspace_energy_blocks(), 1.0, pe, E, true);
}

int ipcgpu_halfspace_friction_gradient(ipcgpu_ctx* ctx, double eps2, double* g_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return gradient_call(ctx, kDerivative, g_inout, [&](cudaStream_t st) {
        halfspace_friction_gradient(p, eps2, ctx->g.p, st);
        ctx->launches += p.rep_mask != nullptr;
    });
}

int ipcgpu_halfspace_friction_hessian(ipcgpu_ctx* ctx, double eps2, int projectDBC, double* a_inout)
{
    if (ctx->n_hs == 0) return IPCGPU_OK;
    REQUIRE_HS_LAG();
    const HalfSpaceArgs p = halfspace_args(ctx);
    return hessian_call(ctx, kDerivative, a_inout, 0, [&](cudaStream_t st) {
        halfspace_friction_hessian(p, eps2, projectDBC, ctx->a.p, st);
        ctx->launches += p.rep_mask != nullptr;
    });
}

int ipcgpu_get_halfspace_sets(ipcgpu_ctx* ctx, int* n_active, int* active2, int* n_lagged, int* lagged2, double* lambda)
{
    if (n_active) *n_active = 0;
    if (n_lagged) *n_lagged = 0;
    if (ctx->n_hs == 0 || !ctx->hs_set_built) return IPCGPU_OK;
    ENTER(kSerial);
    int rc = halfspace_sync_counts(ctx);
    if (rc) return rc;
    const int* h = ctx->staging->hs_count;
    const size_t na = (size_t)h[0], nl = ctx->hs_lag_ready ? (size_t)h[1] : 0;
    if (n_active) *n_active = (int)na;
    if (n_lagged) *n_lagged = (int)nl;
    if (na && active2) CK(cudaMemcpyAsync(active2, ctx->hs_act.p, na * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    if (nl && lagged2) CK(cudaMemcpyAsync(lagged2, ctx->hs_lag.p, nl * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
    if (nl && lambda) CK(cudaMemcpyAsync(lambda, ctx->hs_lam.p, nl * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

} // extern "C"
