// abi_driver.cpp -- a C++ caller of the C ABI (include/ipcgpu.h), no Python in the loop: what the reference-side adapters do.
// Reads a scene (binary, written by tests/test_gpu_cpp_driver.py), drives one Newton iteration's hot path through libipcgpu.so twice --
// once with host outputs (synchronous calls), once device-resident as a replayed CUDA graph with a single ipcgpu_fetch_iteration -- and writes the results back
// for the test to compare with the oracle.   build: g++ -std=c++17 -I include tests/cpp/abi_driver.cpp -L ipc_b200 -lipcgpu -o abi_driver
#include "ipcgpu.h"
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

template <typename T>
static std::vector<T> rd(FILE* f, size_t n)
{
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}
#define CHECK(call)                                                                                         \
    do {                                                                                                    \
        int rc_ = (call);                                                                                   \
        if (rc_) { fprintf(stderr, "%s -> %d: %s\n", #call, rc_, ipcgpu_last_error(ctx)); return 1; }     \
    } while (0)

int main(int argc, char** argv)
{
    if (argc < 3) { fprintf(stderr, "usage: abi_driver scene.bin out.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("scene"); return 2; }
    const std::vector<int32_t> hd = rd<int32_t>(f, 8); // nV nT nSV nSE nSF nnz energy pad
    const int nV = hd[0], nT = hd[1], nSV = hd[2], nSE = hd[3], nSF = hd[4], nnz = hd[5], energy = hd[6];
    const std::vector<double> par = rd<double>(f, 6); // dHat kappa dt2 voxel tol pad
    const auto Vrest = rd<double>(f, 3 * (size_t)nV), V = rd<double>(f, 3 * (size_t)nV), p = rd<double>(f, 3 * (size_t)nV);
    const auto T = rd<int32_t>(f, 4 * (size_t)nT);
    const auto Ainv = rd<double>(f, 9 * (size_t)nT), vol = rd<double>(f, nT), mu = rd<double>(f, nT), lam = rd<double>(f, nT), mass = rd<double>(f, nV);
    const auto SVI = rd<int32_t>(f, nSV), SE = rd<int32_t>(f, 2 * (size_t)nSE), SF = rd<int32_t>(f, 3 * (size_t)nSF);
    const auto ia = rd<int32_t>(f, 3 * (size_t)nV + 1), ja = rd<int32_t>(f, nnz);
    fclose(f);
    const double dHat = par[0], kappa = par[1], dt2 = par[2], voxel = par[3], tol = par[4];

    ipcgpu_ctx* ctx = nullptr;
    if (ipcgpu_create(0, &ctx)) { fprintf(stderr, "ipcgpu_create failed: a CUDA device is required\n"); return 3; }
    CHECK(ipcgpu_set_mesh(ctx, nV, nT, Vrest.data(), T.data(), Ainv.data(), vol.data(), mu.data(), lam.data(), mass.data(), nullptr, energy));
    CHECK(ipcgpu_set_surface(ctx, nSV, SVI.data(), nSE, SE.data(), nSF, SF.data(), nullptr));
    CHECK(ipcgpu_set_csr(ctx, 3 * nV, ia.data(), ja.data(), 1));
    CHECK(ipcgpu_set_state(ctx, V.data()));
    double evf[3], eee[3];
    if (ipcgpu_ti_error(V.data(), nV, nullptr, evf, eee)) return 4;

    // ---- synchronous calls: every result on the host ---------------------------------------------------------------
    int nC = 0, nP = 0, nK = 0;
    CHECK(ipcgpu_constraint_set(ctx, dHat, 1, &nC, &nP, &nK));
    double E_el = 0, E_b = 0;
    CHECK(ipcgpu_elastic_energy(ctx, dt2, 1, &E_el));
    CHECK(ipcgpu_barrier_energy(ctx, dHat, kappa, &E_b));
    std::vector<double> g(3 * (size_t)nV), a(nnz);
    CHECK(ipcgpu_elastic_grad_hess(ctx, dt2, 1, 1, 1, g.data(), a.data()));
    CHECK(ipcgpu_barrier_gradient(ctx, dHat, kappa, g.data()));
    CHECK(ipcgpu_barrier_hessian(ctx, dHat, kappa, 1, a.data()));
    double alpha = 1.0;
    CHECK(ipcgpu_inversion_step(ctx, p.data(), 0.2, &alpha));
    const double a_inv = alpha;
    CHECK(ipcgpu_ccd_partial_ti(ctx, nullptr, tol, evf, eee, &alpha));
    const double a_part = alpha;
    CHECK(ipcgpu_hash_build_swept(ctx, nullptr, &alpha, voxel));
    uint64_t ncand = 0;
    CHECK(ipcgpu_ccd_full_ti(ctx, tol, evf, eee, &alpha, &ncand));
    int n_inv = -1, ok = -1;
    CHECK(ipcgpu_check_inversion(ctx, &n_inv));
    CHECK(ipcgpu_intersection_free(ctx, &ok));

    // ---- the same iteration device-resident, the way a Newton loop runs it: NULL outputs everywhere, the sequence captured ONCE into a CUDA
    // graph (after one eager run) and replayed with one launch + one fetch per iteration -------------------------------------------------
    auto enqueue = [&]() -> int {
        CHECK(ipcgpu_constraint_set(ctx, dHat, 1, nullptr, nullptr, nullptr));
        CHECK(ipcgpu_barrier_energy(ctx, dHat, kappa, nullptr));
        CHECK(ipcgpu_elastic_energy_grad_hess(ctx, dt2, 1, 1, 1, nullptr, nullptr, nullptr)); // computeEnergyVal + computeGradient + computePrecondMtr, one SVD per tet
        CHECK(ipcgpu_barrier_gradient(ctx, dHat, kappa, nullptr));
        CHECK(ipcgpu_barrier_hessian(ctx, dHat, kappa, 1, nullptr));
        CHECK(ipcgpu_step_bound_set(ctx, 1.0));
        CHECK(ipcgpu_inversion_step(ctx, nullptr, 0.2, nullptr));
        CHECK(ipcgpu_ccd_partial_ti(ctx, nullptr, tol, evf, eee, nullptr));
        CHECK(ipcgpu_hash_build_swept(ctx, nullptr, nullptr, voxel));
        CHECK(ipcgpu_ccd_full_ti(ctx, tol, evf, eee, nullptr, nullptr));
        return 0;
    };
    CHECK(ipcgpu_set_canonical_order(ctx, 0)); // the sets are consumed on the device: no canonical sort
    ipcgpu_iteration it;
    if (enqueue()) return 1; // eager once (lazy allocations)
    CHECK(ipcgpu_fetch_iteration(ctx, &it));
    int graph = -1;
    CHECK(ipcgpu_capture_begin(ctx));
    if (enqueue()) return 1;
    CHECK(ipcgpu_capture_end(ctx, &graph));
    CHECK(ipcgpu_set_state(ctx, V.data()));      // what changes between iterations travels through device memory
    CHECK(ipcgpu_set_search_dir(ctx, p.data()));
    CHECK(ipcgpu_graph_launch(ctx, graph));
    CHECK(ipcgpu_fetch_iteration(ctx, &it));
    std::vector<double> g2(3 * (size_t)nV), a2(nnz);
    CHECK(ipcgpu_download(ctx, IPCGPU_BUF_GRADIENT, g2.data(), g2.size()));
    CHECK(ipcgpu_download(ctx, IPCGPU_BUF_CSR_VALUES, a2.data(), a2.size()));

    FILE* o = fopen(argv[2], "wb");
    if (!o) { perror("out"); return 2; }
    const int32_t ints[8] = { nC, nP, nK, (int32_t)ncand, n_inv, ok, it.status, (int32_t)it.n_full_ccd_candidates };
    const double dbl[12] = { E_el, E_b, a_inv, a_part, alpha, it.energy_elastic, it.energy_barrier, it.alpha_inversion, it.alpha_partial_ccd, it.alpha_full_ccd, it.alpha, 0.0 };
    fwrite(ints, sizeof(int32_t), 8, o);
    fwrite(dbl, sizeof(double), 12, o);
    fwrite(g.data(), sizeof(double), g.size(), o);
    fwrite(a.data(), sizeof(double), a.size(), o);
    fwrite(g2.data(), sizeof(double), g2.size(), o);
    fwrite(a2.data(), sizeof(double), a2.size(), o);
    fclose(o);
    ipcgpu_destroy(ctx);
    printf("abi_driver ok: nC=%d nPara=%d nCand=%d E=%.12e alpha=%.17g launches ok\n", nC, nP, nK, E_el + E_b, alpha);
    return 0;
}
