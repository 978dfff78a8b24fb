// api_mesh.cu -- entry points of the mesh and its Hessian layout: the host-side maps (build_maps), mesh / CSR / state / search-direction
// uploads, the elastic terms, the device-resident step bound and its inversion filter, and the built-in PCG solve.
#include "abi.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

using namespace ipcgpu;

// ---------------------------------------------------------------------------------------------------
// map building (host, once per mesh/partition): vertex->incident (tet,local) lists and Hessian slots.
// Partition (nranks > 1): rank r owns the rows of the vertex range [v_begin, v_end) -- chosen so that the incident-tet counts
// balance -- and assembles EVERY tet that touches one of them (tets on a range boundary are computed by both neighbours), so that
// each rank's part of the CSR is complete and the Hessian needs no cross-rank reduction.
// ---------------------------------------------------------------------------------------------------
int build_maps(ipcgpu_ctx* ctx)
{
    const int nT = ctx->nT, nV = ctx->nV;
    const std::vector<int>& T = ctx->h_T;
    ctx->t_begin = (int)((int64_t)nT * ctx->rank / ctx->nranks);
    ctx->t_end = (int)((int64_t)nT * (ctx->rank + 1) / ctx->nranks);
    // vertex ranges balanced by incident-tet count
    std::vector<int64_t> cum(nV + 1, 0);
    for (size_t i = 0; i < (size_t)4 * nT; ++i) ++cum[T[i] + 1];
    for (int v = 0; v < nV; ++v) cum[v + 1] += cum[v];
    auto boundary = [&](int r) -> int {
        if (r <= 0) return 0;
        if (r >= ctx->nranks) return nV;
        const int64_t target = cum[nV] * r / ctx->nranks;
        return (int)(std::lower_bound(cum.begin(), cum.end(), target) - cum.begin());
    };
    const int vb = std::min(boundary(ctx->rank), nV), ve = std::max(vb, std::min(boundary(ctx->rank + 1), nV));
    ctx->v_begin = vb;
    ctx->v_end = ve;
    // tets touching the owned rows, ascending
    std::vector<int> list;
    if (ctx->nranks == 1) {
        list.resize(nT);
        std::iota(list.begin(), list.end(), 0);
    }
    else {
        list.reserve((size_t)(nT / ctx->nranks) + 1024);
        for (int t = 0; t < nT; ++t) {
            bool touch = false;
            for (int k = 0; k < 4; ++k) {
                const int v = T[(size_t)k * nT + t];
                touch = touch || (v >= vb && v < ve);
            }
            if (touch) list.push_back(t);
        }
    }
    const int nL = (int)list.size();
    ctx->n_list = nL;
    if (list.empty()) list.push_back(0); // keep the upload non-empty
    REQUIRE(ctx->tet_list.upload(list.data(), list.size(), ctx->stream), IPCGPU_ERR_CUDA, "upload of the tet list failed");
    // incidence of the OWNED vertices: counting sort by vertex; entries 4*localTet+loc ascending
    std::vector<int> ptr(nV + 1, 0);
    for (int l = 0; l < nL; ++l)
        for (int k = 0; k < 4; ++k) {
            const int v = T[(size_t)k * nT + list[l]];
            if (v >= vb && v < ve) ++ptr[v + 1];
        }
    for (int v = 0; v < nV; ++v) ptr[v + 1] += ptr[v];
    std::vector<int> inc((size_t)std::max(ptr[nV], 1)), cur(ptr.begin(), ptr.end() - 1);
    for (int l = 0; l < nL; ++l)
        for (int k = 0; k < 4; ++k) {
            const int v = T[(size_t)k * nT + list[l]];
            if (v >= vb && v < ve) inc[cur[v]++] = 4 * l + k;
        }
    if (!ctx->inc_ptr.upload(ptr.data(), ptr.size(), ctx->stream) || !ctx->inc.upload(inc.data(), inc.size(), ctx->stream)) {
        ctx->err = "upload of incidence map failed";
        return IPCGPU_ERR_CUDA;
    }
    // slots: (v<=u) pairs whose ROW vertex v is owned; contributions (key, src) sorted by key then tet
    REQUIRE(((uint64_t)nL + 64ull) * 78ull < 0xffffffffull, IPCGPU_ERR_CAPACITY, "local tet count too large for 32-bit block offsets");
    struct KS {
        uint64_t key;
        unsigned src;
        unsigned tet;
    };
    std::vector<KS> ks;
    ks.reserve((size_t)10 * nL);
    static const int pa[6] = { 0, 0, 0, 1, 1, 2 }, pb[6] = { 1, 2, 3, 2, 3, 3 };
    for (int l = 0; l < nL; ++l) {
        const int t = list[l];
        int v[4];
        for (int k = 0; k < 4; ++k) v[k] = T[(size_t)k * nT + t];
        // tile-major block addresses (elastic.cu): (l/64)*64*78 + o*64 + (l%64)*len
        const unsigned tl = (unsigned)l, tile_base = (tl / 64u) * (64u * 78u), tin = tl % 64u;
        for (int a = 0; a < 4; ++a)
            if (v[a] >= vb && v[a] < ve) ks.push_back({ ((uint64_t)v[a] << 32) | (uint32_t)v[a], tile_base + 6u * a * 64u + tin * 6u, tl });
        for (int q = 0; q < 6; ++q) {
            const int lo = std::min(v[pa[q]], v[pb[q]]), hi = std::max(v[pa[q]], v[pb[q]]);
            if (lo >= vb && lo < ve) ks.push_back({ ((uint64_t)lo << 32) | (uint32_t)hi, tile_base + (24u + 9u * q) * 64u + tin * 9u, tl });
        }
    }
    std::sort(ks.begin(), ks.end(), [](const KS& a, const KS& b) { return a.key < b.key || (a.key == b.key && (a.tet < b.tet || (a.tet == b.tet && a.src < b.src))); });
    std::vector<int> sv, su, cptr;
    std::vector<unsigned> csrc(std::max<size_t>(ks.size(), 1));
    for (size_t i = 0; i < ks.size(); ++i) {
        if (i == 0 || ks[i].key != ks[i - 1].key) {
            sv.push_back((int)(ks[i].key >> 32));
            su.push_back((int)(ks[i].key & 0xffffffffu));
            cptr.push_back((int)i);
        }
        csrc[i] = ks[i].src;
    }
    cptr.push_back((int)ks.size());
    {
        // Slot order = work order of k_assemble_csr (one thread per stored entry: 9 per off-diagonal slot, 6 per diagonal one; a warp
        // covers ~3.5 / ~5.3 slots and runs as long as its longest contribution list).  In key order every 7th slot is a diagonal block
        // with ~23 contributions against ~5 for an off-diagonal one, so half of the warps idled most lanes for 20 iterations.
        // Off-diagonal slots first, then the diagonal ones (key order inside each group keeps the CSR writes local): warps see uniform
        // list lengths, and the kernel knows from nOffSlots where the 6-thread slots begin.
        const size_t nS = sv.size();
        std::vector<int> order;
        order.reserve(nS);
        for (size_t i = 0; i < nS; ++i)
            if (sv[i] != su[i]) order.push_back((int)i);
        ctx->nOffSlots = (int)order.size();
        for (size_t i = 0; i < nS; ++i)
            if (sv[i] == su[i]) order.push_back((int)i);
        std::vector<int> sv2(nS), su2(nS), cptr2;
        std::vector<unsigned> csrc2(csrc.size());
        cptr2.reserve(nS + 1);
        size_t pos = 0;
        for (size_t k = 0; k < nS; ++k) {
            const int i = order[k];
            sv2[k] = sv[i];
            su2[k] = su[i];
            cptr2.push_back((int)pos);
            for (int c = cptr[i]; c < cptr[i + 1]; ++c) csrc2[pos++] = csrc[c];
        }
        cptr2.push_back((int)pos);
        sv.swap(sv2); su.swap(su2); cptr.swap(cptr2); csrc.swap(csrc2);
    }
    ctx->nSlots = (int)sv.size();
    if (sv.empty()) { sv.push_back(0); su.push_back(0); } // keep the uploads non-empty
    bool ok = ctx->slot_v.upload(sv.data(), sv.size(), ctx->stream) && ctx->slot_u.upload(su.data(), su.size(), ctx->stream)
        && ctx->con_ptr.upload(cptr.data(), cptr.size(), ctx->stream) && ctx->con_src.upload(csrc.data(), csrc.size(), ctx->stream)
        && ctx->slot_off.reserve((size_t)3 * std::max(1, ctx->nSlots));
    REQUIRE(ok, IPCGPU_ERR_CUDA, "upload of Hessian scatter map failed");
    ALLOC(ctx->gcont, (size_t)12 * std::max(1, nL));
    ALLOC(ctx->hblk, (size_t)78 * 64 * ((size_t)(std::max(1, nL) + 63) / 64));
    ALLOC(ctx->partials, (size_t)std::max(1, elastic_energy_blocks(ctx->t_end - ctx->t_begin)) + 8);
    CK(cudaStreamSynchronize(ctx->stream)); // host vectors go out of scope
    ctx->maps_ready = true;
    ctx->offsets_ready = false;
    // D and its incidence follow the slots, the Neumann forces and Dirichlet targets the vertices: a new mesh or partition removes them
    ctx->damp_on = ctx->damp_inc_ready = ctx->nbc_on = false;
    ctx->n_dbc = 0;
    for (int slot : { kEnergyDamping, kEnergyNeumann, kEnergyDirichlet }) // (the fetch reports 0 for a term that is not set)
        CK(cudaMemsetAsync(&ctx->iter.p->energy[slot], 0, sizeof(double), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

void owned_value_range(ipcgpu_ctx* ctx)
{
    // CSR value range of the owned rows [3 v_begin, 3 v_end)
    if (ctx->h_ia.empty()) return;
    ctx->a_begin = (long long)ctx->h_ia[(size_t)3 * ctx->v_begin] - ctx->index_base;
    ctx->a_end = (long long)ctx->h_ia[(size_t)3 * ctx->v_end] - ctx->index_base;
}

int ensure_offsets(ipcgpu_ctx* ctx)
{
    if (ctx->offsets_ready) return IPCGPU_OK;
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh must precede Hessian assembly");
    REQUIRE(ctx->n_rows == 3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_csr must be called with n_rows = 3*nV");
    CK(cudaMemsetAsync(ctx->flag.p, 0, sizeof(int), ctx->stream));
    slot_offsets(ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->ia.p, ctx->ja.p, ctx->index_base, ctx->slot_off.p, ctx->flag.p, ctx->stream);
    ++ctx->launches;
    int h = 0;
    CK(cudaMemcpyAsync(&h, ctx->flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    REQUIRE(h == 0, IPCGPU_ERR_PATTERN, "CSR pattern misses a block of the mesh topology (row<=col entries of every tet vertex pair are required)");
    ctx->offsets_ready = true;
    return IPCGPU_OK;
}

// upload the search direction; pSize = mean |p| over the surface vertices in the reference's serial order (SpatialHash.hpp:603-612),
// taken straight from the caller's array (it is only needed by the swept build and costs one pass over the surface)
int upload_dir(ipcgpu_ctx* ctx, const double* p)
{
    if (p) {
        CK(cudaMemcpyAsync(ctx->dir.p, p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        double pSize = 0;
        // (mesh.SVI: with an obstacle attached the surface vertices of the tail do not count -- SpatialHash::build sees the mesh alone)
        int nMeshSV = 0;
        for (int i = 0; i < ctx->nSV; ++i) {
            const int v = ctx->h_SVI[i];
            if (v >= ctx->nVdof) continue;
            ++nMeshSV;
            pSize += std::abs(p[3 * (size_t)v]);
            pSize += std::abs(p[3 * (size_t)v + 1]);
            pSize += std::abs(p[3 * (size_t)v + 2]);
        }
        ctx->pSize = nMeshSV > 0 ? pSize / (double)((long long)nMeshSV * 3) : 0.0;
        // the swept-grid kernel reads it from device memory, so that a captured graph stays valid when the direction changes
        ALLOC(ctx->pSize_dev, 1);
        ctx->staging->pSize = ctx->pSize; // (its own pinned slot: nothing waits on this copy)
        CK(cudaMemcpyAsync(ctx->pSize_dev.p, &ctx->staging->pSize, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        ctx->pSize_surface = ctx->surface_ready;
        ctx->dir_valid = true; // (no synchronisation: like every host input of the deferred mode, p must stay untouched until the next fetch)
    }
    REQUIRE(ctx->dir_valid, IPCGPU_ERR_STATE, "no search direction uploaded yet");
    return IPCGPU_OK;
}

extern "C" {

int ipcgpu_set_mesh(ipcgpu_ctx* ctx, int nV, int nT, const double* Vrest, const int* tets, const double* restTriInv, const double* vol,
    const double* mu, const double* lam, const double* mass, const uint8_t* dbc, int energy)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(nV > 0 && nT >= 0 && Vrest && tets && restTriInv && vol && mu && lam, IPCGPU_ERR_ARG, "ipcgpu_set_mesh: null or empty input");
    REQUIRE(energy == IPCGPU_NEOHOOKEAN || energy == IPCGPU_FIXED_COROT, IPCGPU_ERR_ARG, "unknown energy type");
    for (size_t i = 0; i < (size_t)4 * nT; ++i) REQUIRE(tets[i] >= 0 && tets[i] < nV, IPCGPU_ERR_ARG, "tet vertex index out of range");
    ctx->nV = nV;
    ctx->nT = nT;
    ctx->energy = energy;
    ctx->hs_set_built = ctx->hs_lag_ready = false; // the plane sets index the old vertices
    ctx->nVdof = 0x7fffffff; // a new mesh has no obstacle tail until ipcgpu_set_obstacle_tail names one
    ctx->n_comp = 0;         // ... and no components until ipcgpu_set_components names them
    ctx->h_T.assign(tets, tets + (size_t)4 * nT);
    ctx->h_ia.clear();
    ctx->nnz = 0;
    ctx->device_pattern = ctx->pat_pending = false;
    ctx->surface_ready = false;
    ctx->dir_valid = false;
    ctx->g_assembled = ctx->a_assembled = false;
    // Dm^-1: reference layout is per-tet column-major; device layout is SoA over the row-major index q=3i+j
    std::vector<double> A((size_t)9 * std::max(nT, 1));
    for (int t = 0; t < nT; ++t)
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) A[(size_t)(3 * i + j) * nT + t] = restTriInv[(size_t)9 * t + i + 3 * j];
    bool ok = ctx->Vrest.upload(Vrest, (size_t)3 * nV, ctx->stream) && ctx->V.upload(Vrest, (size_t)3 * nV, ctx->stream)
        && ctx->Vsaved.reserve((size_t)3 * nV) && ctx->T.upload(tets, (size_t)4 * nT, ctx->stream)
        && ctx->Ainv.upload(A.data(), (size_t)9 * nT, ctx->stream) && ctx->vol.upload(vol, nT, ctx->stream)
        && ctx->mu.upload(mu, nT, ctx->stream) && ctx->lam.upload(lam, nT, ctx->stream);
    REQUIRE(ok, IPCGPU_ERR_CUDA, "mesh upload failed");
    ctx->has_mass = mass != nullptr;
    if (mass) REQUIRE(ctx->mass.upload(mass, nV, ctx->stream), IPCGPU_ERR_CUDA, "mass upload failed");
    ctx->has_dbc = dbc != nullptr;
    if (dbc) REQUIRE(ctx->dbc.upload(dbc, nV, ctx->stream), IPCGPU_ERR_CUDA, "dbc upload failed");
    ALLOC(ctx->g, (size_t)3 * nV);
    ALLOC(ctx->dir, (size_t)3 * nV);
    ALLOC(ctx->e_per_tet, (size_t)std::max(nT, 1));
    ALLOC(ctx->inv_steps, (size_t)std::max(nT, 1));
    CK(cudaStreamSynchronize(ctx->stream));
    return build_maps(ctx);
}

int ipcgpu_set_csr(ipcgpu_ctx* ctx, int n_rows, const int* ia, const int* ja, int index_base)
{
    ENTER(kSerial);
    ++ctx->epoch; // graphs captured before this call are refused (buffers, partition or list order may change)
    REQUIRE(n_rows > 0 && ia && ja && (index_base == 0 || index_base == 1), IPCGPU_ERR_ARG, "ipcgpu_set_csr: bad arguments");
    REQUIRE(ctx->nV > 0 && n_rows == 3 * ctx->nV, IPCGPU_ERR_ARG, "ipcgpu_set_csr: n_rows must be 3*nV of the mesh set before");
    const int nnz = ia[n_rows] - index_base;
    REQUIRE(nnz >= 0, IPCGPU_ERR_ARG, "ipcgpu_set_csr: negative nnz");
    ctx->n_rows = n_rows;
    ctx->nnz = nnz;
    ctx->index_base = index_base;
    ctx->device_pattern = ctx->pat_pending = false; // host mode again
    ctx->h_ia.assign(ia, ia + (size_t)n_rows + 1);
    bool ok = ctx->ia.upload(ia, (size_t)n_rows + 1, ctx->stream) && ctx->ja.upload(ja, (size_t)nnz, ctx->stream) && ctx->a.reserve((size_t)std::max(nnz, 1));
    REQUIRE(ok, IPCGPU_ERR_CUDA, "CSR upload failed");
    CK(cudaMemsetAsync(ctx->a.p, 0, (size_t)nnz * sizeof(double), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->a_all_dirty = false;
    ctx->offsets_ready = false;
    ctx->g_assembled = ctx->a_assembled = false;
    owned_value_range(ctx);
    return solver_forget_full_pattern(ctx);
}

int ipcgpu_set_state(ipcgpu_ctx* ctx, const double* V)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    if (V) CK(cudaMemcpyAsync(ctx->V.p, V, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->mark_inputs();
    ctx->g_assembled = ctx->a_assembled = false;
    return IPCGPU_OK;
}

int ipcgpu_save_state(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    CK(cudaMemcpyAsync(ctx->Vsaved.p, ctx->V.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->state_saved = true;
    return IPCGPU_OK;
}

int ipcgpu_set_search_dir(ipcgpu_ctx* ctx, const double* p)
{
    REQUIRE(ctx->nV > 0 && p, IPCGPU_ERR_ARG, "ipcgpu_set_search_dir: mesh and p required");
    ENTER(kSerial);
    return upload_dir(ctx, p);
}

int ipcgpu_step_forward(ipcgpu_ctx* ctx, const double* p, double alpha)
{
    REQUIRE(ctx->nV > 0, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    REQUIRE(ctx->state_saved, IPCGPU_ERR_STATE, "ipcgpu_save_state must precede ipcgpu_step_forward");
    ENTER(kSerial);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    step_forward(ctx->nV, ctx->Vsaved.p, ctx->dir.p, alpha, ctx->V.p, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->mark_inputs();
    return IPCGPU_OK;
}

int ipcgpu_elastic_energy(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, double* E)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(kSerial);
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
    elastic_energy(ctx->eargs(), ctx->e_per_tet.p, ctx->partials.p, ctx->stream);
    return energy_tail(ctx, kEnergyElastic, ctx->partials.p, elastic_energy_blocks(ctx->t_end - ctx->t_begin), coef, pe, E);
}

// zero the part of the value array this rank writes (everything after a cross-rank completion has filled the other rows)
static int zero_values(ipcgpu_ctx* ctx)
{
    cudaStream_t st = ctx->deriv_stream(); // (zero_words, not a memset: kernels.h)
    if (ctx->device_pattern) { // the range follows the device's row starts (the host mirror may lag an update in flight)
        const bool owned = ctx->nranks > 1 && !ctx->a_all_dirty;
        zero_csr_rows(ctx->ia.p, ctx->index_base, owned ? 3 * ctx->v_begin : 0, owned ? 3 * ctx->v_end : 3 * ctx->nV, ctx->a.p, st);
    }
    else if (ctx->nranks > 1 && !ctx->a_all_dirty) {
        if (ctx->a_end > ctx->a_begin) zero_words(ctx->a.p + ctx->a_begin, (size_t)(ctx->a_end - ctx->a_begin) * 2, st);
    }
    else zero_words(ctx->a.p, (size_t)ctx->nnz * 2, st);
    ++ctx->launches;
    CK(cudaGetLastError());
    ctx->a_all_dirty = false;
    return IPCGPU_OK;
}

// cleared: the value array holds zeros at every entry of the slots (zero_values), so the assembly writes its sums instead of adding them
static int run_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, bool need_g, bool need_h, int add_mass, bool with_energy = false,
    bool cleared = false)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    if (need_h) {
        int rc = ensure_offsets(ctx);
        if (rc) return rc;
    }
    cudaStream_t st = ctx->deriv_stream(); // (stage timers are only on when it is the main stream)
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_TET);
    double* e_part = nullptr;
    if (with_energy) { // psi * vol per CTA, summed in fixed order below (computeEnergyVal at the same state: the SVD is shared)
        ALLOC(ctx->e_partials2, (size_t)elastic_grad_hess_blocks(ctx->n_list) + 8);
        e_part = ctx->e_partials2.p;
    }
    elastic_grad_hess(ctx->eargs(), coef, projectSPD, need_g, need_h, ctx->gcont.p, ctx->hblk.p, st, e_part);
    ctx->hblk_valid = need_h;
    ctx->g_assembled = ctx->g_assembled || need_g;
    ctx->a_assembled = ctx->a_assembled || need_h;
    ctx->prof_end(pe);
    ++ctx->launches;
    if (with_energy) { // (which rank's share it is: energy_result, once the call knows whether the host wants it)
        pe = ctx->prof_begin(IPCGPU_STAGE_ELASTIC_ENERGY);
        reduce_sum(e_part, elastic_grad_hess_blocks(ctx->n_list), coef, &ctx->iter.p->energy[kEnergyElastic], st);
        ctx->prof_end(pe);
        ++ctx->launches;
    }
    if (need_g) {
        // owned vertices gather their complete sums (every incident tet is in this rank's list); the other rows are written as zeros
        pe = ctx->prof_begin(IPCGPU_STAGE_GATHER_GRADIENT);
        gather_gradient(ctx->nV, ctx->inc_ptr.p, ctx->inc.p, ctx->gcont.p, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, 0, ctx->g.p, st);
        ctx->prof_end(pe);
        ++ctx->launches;
    }
    if (need_h) {
        pe = ctx->prof_begin(IPCGPU_STAGE_ASSEMBLE_CSR);
        assemble_csr(ctx->nOffSlots, ctx->nSlots, ctx->slot_v.p, ctx->slot_u.p, ctx->slot_off.p, ctx->con_ptr.p, ctx->con_src.p, ctx->hblk.p,
            ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, nullptr, cleared ? 0 : 1, ctx->a.p, st);
        // per-vertex diagonal terms (mass, Dirichlet identity) of the owned rows
        const double* m = (add_mass && ctx->has_mass) ? ctx->mass.p : nullptr;
        diag_mass_dbc_range(ctx->v_begin, ctx->v_end, ctx->ia.p, ctx->index_base, ctx->has_dbc ? ctx->dbc.p : nullptr, projectDBC, m, ctx->a.p, st);
        ctx->prof_end(pe);
        ctx->launches += 2;
    }
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_elastic_gradient(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, int projectDBC, double* g)
{
    ENTER(g ? kSerial : kDerivative);
    int rc = run_grad_hess(ctx, coef, 1, projectDBC, true, false, 0);
    return rc || !g ? rc : gradient_roundtrip_end(ctx, g); // (the gradient is written, not accumulated: no roundtrip_begin)
}

int ipcgpu_elastic_hessian(ipcgpu_ctx* ctx, double coef, int /*redoSVD*/, int projectSPD, int projectDBC, double* a_inout)
{
    int rc = hessian_begin(ctx, kDerivative, a_inout);
    if (rc || (rc = run_grad_hess(ctx, coef, projectSPD, projectDBC, false, true, 0))) return rc;
    return hessian_end(ctx, a_inout, 0);
}

static int elastic_derivatives(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, bool with_energy, double* E, double* g, double* a)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(E || g || a ? kSerial : kDerivative);
    // the value array is rebuilt from scratch (LinSysSolver::setZero, then addCoeff of every term): slots that no local tet touches
    // -- contact-only blocks of the augmented pattern -- must not keep last iteration's values
    int rc = a ? sync_pattern_mirror(ctx) : 0; // (the host array holds the current pattern's values)
    if (rc || (rc = zero_values(ctx))) return rc;
    if ((rc = run_grad_hess(ctx, coef, projectSPD, projectDBC, true, true, add_mass, with_energy, true))) return rc;
    if (ctx->nranks > 1 && (g || a)) {
        rc = ipcgpu_allreduce_grad_hess(ctx, g ? 1 : 0, a ? 1 : 0);
        if (rc) return rc;
    }
    if (g) CK(cudaMemcpyAsync(g, ctx->g.p, (size_t)3 * ctx->nV * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (a) CK(cudaMemcpyAsync(a, ctx->a.p, (size_t)ctx->nnz * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (with_energy && (rc = energy_result(ctx, kEnergyElastic, E))) return rc; // (a host E synchronises)
    if (!E && (g || a)) CK(cudaStreamSynchronize(ctx->stream));
    return IPCGPU_OK;
}

int ipcgpu_elastic_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, double* g, double* a)
{
    return elastic_derivatives(ctx, coef, projectSPD, projectDBC, add_mass, false, nullptr, g, a);
}

int ipcgpu_elastic_energy_grad_hess(ipcgpu_ctx* ctx, double coef, int projectSPD, int projectDBC, int add_mass, double* E, double* g, double* a)
{
    return elastic_derivatives(ctx, coef, projectSPD, projectDBC, add_mass, true, E, g, a);
}

// ---- step bound: device-resident chain ---------------------------------------------------------------------
int ipcgpu_step_bound_set(ipcgpu_ctx* ctx, double alpha)
{
    REQUIRE(alpha >= 0.0, IPCGPU_ERR_ARG, "the step must be non-negative");
    ENTER(kStepBound);
    step_set(ctx->iter.p, alpha, ctx->stream);
    ++ctx->launches;
    CK(cudaGetLastError());
    return IPCGPU_OK;
}

int ipcgpu_inversion_step(ipcgpu_ctx* ctx, const double* p, double slack, double* alpha_inout)
{
    REQUIRE(ctx->maps_ready, IPCGPU_ERR_STATE, "ipcgpu_set_mesh first");
    ENTER(p || alpha_inout ? kSerial : kStepBound);
    int rc = upload_dir(ctx, p);
    if (rc) return rc;
    if (alpha_inout && (rc = ipcgpu_step_bound_set(ctx, *alpha_inout))) return rc;
    cudaEvent_t pe = ctx->prof_begin(IPCGPU_STAGE_INVERSION);
    inversion_step(ctx->eargs(), ctx->dir.p, slack, ctx->inv_steps.p, ctx->iter.p, ctx->stream);
    ctx->prof_end(pe);
    ctx->launches += 2;
    if ((rc = nccl_min_u64(ctx, &ctx->iter.p->inv_ord))) return rc;
    inversion_apply(ctx->iter.p, ctx->nT, ctx->stream); // Energy.cpp:576-579
    ++ctx->launches;
    CK(cudaGetLastError());
    if (alpha_inout) return ccd_read_back(ctx, alpha_inout);
    return IPCGPU_OK;
}

// ---- device-resident linear solve hand-off (SURVEY 8(f) rank 1) ----------------------------------------------------------
// (the three built-in solvers: the preconditioner is the only difference).  The deferred form (rhs, x, iters, rel_residual all NULL) enqueues
// everything, the Krylov loops as conditional graph nodes inside a capture; its result is read by ipcgpu_solve_info, its failure raises
// FLAG_SOLVE.  Any other form synchronises and returns what it always did.
static int solve_pcg(ipcgpu_ctx* ctx, int precond, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual)
{
    REQUIRE(ctx->nnz > 0 && ctx->n_rows == 3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the built-in solver runs on one rank (a distributed solver takes each rank's rows: ipcgpu_partition_info)");
    REQUIRE(rel_tol > 0.0 && max_iter > 0, IPCGPU_ERR_ARG, "bad tolerance / iteration limit");
    const bool deferred = !rhs && !x && !iters && !rel_residual;
    REQUIRE(deferred || !ctx->capturing, IPCGPU_ERR_STATE, "inside a capture the solve takes its deferred form: rhs, x, iters and rel_residual all NULL");
    static const char* const name[] = { "ipcgpu_solve_pcg", "ipcgpu_solve_pcg_multilevel", "ipcgpu_solve_pcg_amg" };
    const bool multilevel = precond == kPrecondMultilevel;
    // (the unreserved AMG set-up reads its sizes back: it cannot be captured)
    REQUIRE(!ctx->capturing || precond != kPrecondAmg || solver_amg_reserved(ctx), IPCGPU_ERR_STATE,
        "ipcgpu_solve_pcg_amg runs inside a capture after ipcgpu_amg_reserve (the unreserved set-up reads sizes back)");
    static const char* const first[] = { "run ipcgpu_solve_pcg once outside a capture first (it makes its allocations and creates its streams)",
        "run ipcgpu_solve_pcg_multilevel once outside a capture first (it makes its allocations and creates its streams)",
        "run ipcgpu_solve_pcg_amg once outside a capture after ipcgpu_amg_reserve first (it creates its streams)" };
    REQUIRE(!ctx->capturing || ctx->solve_epoch[precond] == ctx->epoch, IPCGPU_ERR_STATE, first[precond]);
    ENTER(kSerial);
    int rc = cond_prepare(ctx, name[precond]);
    if (rc) return rc;
    const int n = ctx->n_rows;
    bool ok = ctx->sol.reserve(n) && ctx->pcg_r.reserve(n) && ctx->pcg_p.reserve(n) && ctx->pcg_q.reserve(n) && ctx->pcg_scal.reserve(8)
        && ctx->pcg_part.reserve((size_t)kPcgSpmvBlocks + 2 * nblk(ctx->nV, 256)) && (precond != kPrecondJacobi || ctx->pcg_minv.reserve((size_t)6 * ctx->nV));
    REQUIRE(ok, IPCGPU_ERR_CUDA, "PCG workspace allocation failed");
    if ((rc = solver_full_pattern(ctx))) return rc; // (rows of both triangles, gathered through a position map; rebuilt when the pattern moved)
    const double* rhs_dev = ctx->g.p;
    double sign = -1.0; // Newton: H p = -g (Optimizer.cpp:2350-2352)
    if (rhs) { // a host right-hand side is staged in a buffer of its own
        ALLOC(ctx->pcg_b, (size_t)n);
        CK(cudaMemcpyAsync(ctx->pcg_b.p, rhs, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        rhs_dev = ctx->pcg_b.p;
        sign = 1.0;
    }
    rc = solver_pcg(ctx, rhs_dev, sign, rel_tol, max_iter, precond);
    if (rc) return rc;
    ctx->sv_pending = true;
    if (!ctx->capturing && (precond != kPrecondAmg || ctx->amg.reserved)) ctx->solve_epoch[precond] = ctx->epoch;
    // outside a capture the host loops have read the solve's words (h_iter) with their last decision; inside one they are in device memory
    const IterState& h = *ctx->h_iter;
    const bool bad_pivot = !ctx->capturing && precond != kPrecondJacobi && h.sv_status != 0 && h.sv_iters == 0; // (the set-up failed: no iteration ran)
    if (multilevel) ctx->ml.built = !bad_pivot;
    if (!deferred) { // the host-output forms report a failure by their return value alone, as before: no deferred flag
        if (h.sv_status != 0) CK(cudaMemsetAsync(&ctx->iter.p->flags[FLAG_SOLVE], 0, sizeof(int), ctx->stream));
        REQUIRE(!bad_pivot || precond == kPrecondAmg, IPCGPU_ERR_SOLVE, "multilevel preconditioner: a domain matrix has a non-positive pivot (the matrix is not positive definite)");
        REQUIRE(!bad_pivot, IPCGPU_ERR_SOLVE, "AMG preconditioner: a diagonal block with a non-positive pivot or a non-finite spectral radius (the matrix is not positive definite)");
    }
    if (adopt_as_search_dir && (rc = solver_adopt_direction(ctx, ctx->sol.p))) return rc;
    if (iters) *iters = h.sv_iters;
    if (rel_residual) *rel_residual = h.sv_bb > 0.0 ? std::sqrt(h.sv_rr / h.sv_bb) : 0.0;
    if (x) {
        CK(cudaMemcpyAsync(x, ctx->sol.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return IPCGPU_OK;
}

int ipcgpu_solve_pcg(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual)
{
    return solve_pcg(ctx, kPrecondJacobi, rhs, rel_tol, max_iter, x, adopt_as_search_dir, iters, rel_residual);
}

int ipcgpu_solve_pcg_multilevel(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual)
{
    return solve_pcg(ctx, kPrecondMultilevel, rhs, rel_tol, max_iter, x, adopt_as_search_dir, iters, rel_residual);
}

// smoothed-aggregation multigrid (amg.cu, AMGCLSolver.cpp:24-44, :173-191): single rank; capturable after ipcgpu_amg_reserve
int ipcgpu_solve_pcg_amg(ipcgpu_ctx* ctx, const double* rhs, double rel_tol, int max_iter, double* x, int adopt_as_search_dir, int* iters, double* rel_residual)
{
    return solve_pcg(ctx, kPrecondAmg, rhs, rel_tol, max_iter, x, adopt_as_search_dir, iters, rel_residual);
}

// LinSysSolver::precondition_diag on the resident system: computeSearchDir's fallback (sign -1, Optimizer.cpp:2331-2346) and the friction
// convergence test's (sign +1, :1724).  Its result takes the solvers' words (kSolveStart with |b|^2 = 0: 0 iterations, rel_residual 0) and
// their max |x_i| (solver_finish), so ipcgpu_solve_info reads it as it reads a solve's.
int ipcgpu_precondition_diag(ipcgpu_ctx* ctx, int sign, double* x, int adopt_as_search_dir)
{
    REQUIRE(sign == 1 || sign == -1, IPCGPU_ERR_ARG, "ipcgpu_precondition_diag: sign must be +1 or -1");
    REQUIRE(ctx->nnz > 0 && ctx->n_rows == 3 * ctx->nV, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the diagonal preconditioning runs on one rank, like the built-in solvers");
    REQUIRE(ctx->g_assembled && ctx->a_assembled, IPCGPU_ERR_STATE,
        "no gradient and matrix assembled since the last ipcgpu_set_state, ipcgpu_set_mesh or pattern change");
    REQUIRE(!x || !ctx->capturing, IPCGPU_ERR_STATE, "inside a capture the diagonal preconditioning takes its deferred form: x NULL");
    const int n = ctx->n_rows;
    REQUIRE(!ctx->capturing || (ctx->sol.n >= (size_t)n && ctx->pcg_scal.n >= 8), IPCGPU_ERR_STATE,
        "run ipcgpu_precondition_diag once outside a capture first (it sizes its workspace)");
    ENTER(kSerial);
    REQUIRE(ctx->sol.reserve(n) && ctx->pcg_scal.reserve(8), IPCGPU_ERR_CUDA, "diagonal preconditioning workspace allocation failed");
    CK(cudaMemsetAsync(ctx->pcg_scal.p, 0, 8 * sizeof(double), ctx->stream));
    int rc = decide(ctx, kSolveStart, 0.0, 0, 0, nullptr, ctx->pcg_scal.p);
    if (rc) return rc;
    solver_precondition_diag(ctx, (double)sign, ctx->sol.p, false);
    CK(cudaGetLastError());
    if ((rc = solver_finish(ctx))) return rc;
    ctx->sv_pending = true;
    if (adopt_as_search_dir && (rc = solver_adopt_direction(ctx, ctx->sol.p))) return rc;
    if (x) { // the host form reports a non-finite result by its return value alone, as the solvers' host forms do: no deferred flag
        IterState& h = *ctx->h_iter;
        CK(cudaMemcpyAsync(x, ctx->sol.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(&h.sv_status, &ctx->iter.p->sv_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (h.sv_status != 0) CK(cudaMemsetAsync(&ctx->iter.p->flags[FLAG_SOLVE], 0, sizeof(int), ctx->stream));
        REQUIRE(h.sv_status == 0, IPCGPU_ERR_SOLVE, "diagonal preconditioning: a non-finite entry (a zero or non-finite diagonal or gradient entry)");
    }
    return IPCGPU_OK;
}

int ipcgpu_solve_info(ipcgpu_ctx* ctx, ipcgpu_solve_result* out)
{
    REQUIRE(out != nullptr, IPCGPU_ERR_ARG, "null output");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    if (ctx->sv_pending) {
        ENTER(kSerial);
        int rc = fetch_iter_state(ctx);
        if (rc) return rc;
        ctx->sv_pending = false;
    }
    else CK(cudaSetDevice(ctx->device)); // (reads the host mirror)
    const IterState& h = *ctx->h_iter;
    out->iterations = h.sv_iters;
    out->rel_residual = h.sv_bb > 0.0 ? std::sqrt(h.sv_rr / h.sv_bb) : 0.0;
    std::memcpy(&out->max_abs_x, &h.sv_xmax_ord, sizeof(double));
    out->status = h.sv_status;
    if (h.sv_status) ctx->err = "the linear solve failed: a non-positive pivot of the multilevel preconditioner or a non-finite residual (the matrix is not positive definite)";
    return h.sv_status;
}

int ipcgpu_multilevel_info(ipcgpu_ctx* ctx, int* levels, int64_t* domains_per_level, uint64_t* bytes)
{
    const ipcgpu::MultilevelWork& w = ctx->ml;
    REQUIRE(w.built, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_multilevel first (a call that failed leaves no hierarchy)");
    if (levels) *levels = w.levels;
    if (domains_per_level)
        for (int l = 0; l < ipcgpu::kMultilevelMax; ++l) domains_per_level[l] = l < w.levels ? w.domains[l] : 0;
    if (bytes) *bytes = (uint64_t)w.tiles * 96 * 96 * sizeof(double);
    return IPCGPU_OK;
}

int ipcgpu_multilevel_debug_matrices(ipcgpu_ctx* ctx, double* dst, uint64_t count)
{
    REQUIRE(ctx->ml.built, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_multilevel first");
    ENTER(kSerial);
    return solver_multilevel_matrices(ctx, dst, count);
}

int ipcgpu_amg_info(ipcgpu_ctx* ctx, int* levels, int64_t* rows, int64_t* blocks, double* rho, double* omega, uint64_t* bytes)
{
    REQUIRE(ctx->amg.ran, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    int rc = solver_amg_read(ctx);
    if (rc) return rc;
    const ipcgpu::AmgDev& h = ctx->amg.h;
    REQUIRE(!h.fail && h.levels > 0, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    if (levels) *levels = h.levels;
    for (int l = 0; l < ipcgpu::kAmgMaxLevels; ++l) {
        const bool in = l < h.levels;
        if (rows) rows[l] = in ? h.n[l] : 0;
        if (blocks) blocks[l] = in ? h.nnzb[l] : 0;
        if (rho) rho[l] = in ? h.rho[l] : 0.0;
        if (omega) omega[l] = in ? h.omega[l] : 0.0;
    }
    if (bytes) *bytes = solver_amg_bytes(ctx);
    return IPCGPU_OK;
}

int ipcgpu_amg_debug_level(ipcgpu_ctx* ctx, int level, int* aggregate, int* ia, int* ja, double* blocks)
{
    REQUIRE(ctx->amg.ran, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    int rc = solver_amg_read(ctx);
    if (rc) return rc;
    const ipcgpu::AmgDev& h = ctx->amg.h;
    REQUIRE(!h.fail && h.levels > 0, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first (a call that failed leaves no hierarchy)");
    REQUIRE(level >= 0 && level < h.levels, IPCGPU_ERR_ARG, "level out of range (ipcgpu_amg_info gives the levels)");
    const ipcgpu::AmgLevel& L = ctx->amg.lv[level];
    const int n = h.n[level], nnzb = h.nnzb[level];
    cudaStream_t st = ctx->stream;
    if (aggregate) {
        if (h.np[level] > 0) CK(cudaMemcpyAsync(aggregate, L.agg.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
        else std::fill(aggregate, aggregate + n, -1); // (the last level is not aggregated)
    }
    if (ia) CK(cudaMemcpyAsync(ia, L.ia.p, ((size_t)n + 1) * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (ja && nnzb) CK(cudaMemcpyAsync(ja, L.ja.p, (size_t)nnzb * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (blocks && nnzb) CK(cudaMemcpyAsync(blocks, L.blk.p, 9 * (size_t)nnzb * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return IPCGPU_OK;
}

int ipcgpu_amg_reserve(ipcgpu_ctx* ctx, double headroom)
{
    REQUIRE(std::isfinite(headroom) && headroom >= 1.0, IPCGPU_ERR_ARG, "ipcgpu_amg_reserve: headroom must be finite and >= 1");
    REQUIRE(ctx->nranks == 1, IPCGPU_ERR_STATE, "the built-in solver runs on one rank");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    REQUIRE(ctx->amg.ran, IPCGPU_ERR_STATE, "ipcgpu_amg_reserve: an eager ipcgpu_solve_pcg_amg first");
    ENTER(kSerial);
    return solver_amg_reserve(ctx, headroom);
}

int ipcgpu_amg_capacity_info(ipcgpu_ctx* ctx, int* cut_at_level, int64_t* needed, int64_t* reserved)
{
    REQUIRE(ctx->amg.ran, IPCGPU_ERR_STATE, "ipcgpu_solve_pcg_amg first");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    int rc = solver_amg_read(ctx);
    if (rc) return rc;
    const ipcgpu::AmgWork& w = ctx->amg;
    if (cut_at_level) *cut_at_level = w.h.cut_level;
    for (int l = 0; l < ipcgpu::kAmgMaxLevels; ++l)
        for (int q = 0; q < ipcgpu::kAmgQty; ++q) {
            if (needed) needed[l * ipcgpu::kAmgQty + q] = w.h.need[l][q];
            if (reserved) reserved[l * ipcgpu::kAmgQty + q] = w.lv[l].cap[q];
        }
    return IPCGPU_OK;
}

int ipcgpu_amg_debug_coarse_enough(ipcgpu_ctx* ctx, int rows)
{
    REQUIRE(rows >= 0, IPCGPU_ERR_ARG, "ipcgpu_amg_debug_coarse_enough: rows must be >= 0");
    REQUIRE(!ctx->capturing, IPCGPU_ERR_STATE, "a capture is in progress");
    ENTER(kSerial);
    return solver_amg_coarse_enough(ctx, rows);
}

int ipcgpu_csr_set_zero(ipcgpu_ctx* ctx)
{
    REQUIRE(ctx->nnz > 0, IPCGPU_ERR_STATE, "ipcgpu_set_csr first");
    ENTER(kSerial);
    return zero_values(ctx);
}

} // extern "C"
