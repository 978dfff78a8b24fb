// elastic.cu -- per-tetrahedron elastic energy / gradient / PSD-projected Hessian kernels (sm_90a).
//
// Reference path being replaced: Energy<3>::getEnergyValPerElemBySVD / computeGradientByPK /
// computeHessianByPK (src/Energy/Energy.cpp:195-242, 245-289, 292-331, 334-408, 448-562) and
// computeInjectiveStepSize_3d (src/Utils/get_feasible_steps.cpp:110-172).
//
// Design (not a translation): one thread per tet, everything in registers.
//  * loads: SoA tet indices / Dm^-1 / vol / mu / lam are fully coalesced; the 4-vertex stencil is
//    a gather from the SoA position array (L2-resident: 24 B/vertex).
//  * the 9x9 dP/dF of the reference is never formed.  With G the 4x3 shape-gradient matrix
//    (G[i+1][j] = Dm^-1(i,j), G[0] = -sum) and W = G V, every 3x3 vertex block is
//        H_ab = U * Ht_ab * U^T,
//        Ht_ab[k][m] = a_km W_ak W_bm + [k!=m] o_km W_am W_bk + [k==m] sum_{l!=k} d_kl W_al W_bl
//    where a = projected d2psi/dsigma2 (A block), and d/o the diagonal/off-diagonal entries of the
//    three projected 2x2 B blocks -- ~0.9 kflop instead of the ~5 kflop 21-term contraction, which
//    keeps the kernel on the HBM side of the FP64 ridge.
//  * output: only the 78 upper-triangular scalars per tet (what the CSR sink accepts), as 4 diagonal
//    blocks (6 each) + 6 off-diagonal blocks (9 each, oriented so rows belong to the smaller global
//    vertex id).  Each CTA stages its 64 x 624 B tile in shared memory and ships it with ONE TMA bulk
//    store (cp.async.bulk.global.shared::cta), so HBM sees only full-line writes.
#include "elastic.cuh"
#include "kernels.h"

namespace ipcgpu {

constexpr int kHessTile = 64; // tets per CTA in the gradient/Hessian kernel

struct TetIn {
    int v[4];
    double x[4][3];
    M3 A; // Dm^-1 row-major
    double vol, mu, lam;
};

DEV void load_tet(const ElasticArgs& p, int t, TetIn& in)
{
#pragma unroll
    for (int k = 0; k < 4; ++k) in.v[k] = __ldg(p.T + (size_t)k * p.nT + t);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) in.x[k][c] = __ldg(p.V + (size_t)c * p.nV + in.v[k]);
#pragma unroll
    for (int q = 0; q < 9; ++q) in.A.m[q] = __ldg(p.Ainv + (size_t)q * p.nT + t);
    in.vol = __ldg(p.vol + t);
    in.mu = __ldg(p.mu + t);
    in.lam = __ldg(p.lam + t);
}

DEV void def_grad(const TetIn& in, M3& F)
{
    double e[3][3]; // e[c] = x_{c+1} - x_0
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r) e[c][r] = in.x[c + 1][r] - in.x[0][r];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) F(i, j) = e[0][i] * in.A(0, j) + e[1][i] * in.A(1, j) + e[2][i] * in.A(2, j);
}

// ---------------------------------------------------------------------------------------------
// energy: per-tet psi*vol (optional) + deterministic two-level sum
// ---------------------------------------------------------------------------------------------
template <int ENERGY>
__global__ void __launch_bounds__(256) k_elastic_energy(ElasticArgs p, double* __restrict__ e_per_tet, double* __restrict__ partials)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    double e = 0.0;
    if (t < p.t_end - p.t_begin) {
        const int tt = p.t_begin + t;
        TetIn in;
        load_tet(p, tt, in);
        M3 F, U, V;
        double s[3];
        def_grad(in, F);
        svd3<false>(F, U, s, V);
        e = psi<ENERGY>(s, in.mu, in.lam) * in.vol;
        if (e_per_tet) e_per_tet[tt] = e;
    }
    cta_sum(&e, partials + blockIdx.x);
}

// single-CTA fixed-order reduction of the per-CTA partials: out[0] = scale * sum.  kDevScale: the scale is read from scale_dev (the
// device-resident kappa of a barrier energy); a template parameter, so that the host-scale instantiation compiles as without it
template <bool kDevScale>
__global__ void __launch_bounds__(1024) k_reduce_sum(const double* __restrict__ partials, int n, double scale, double* __restrict__ out,
    const double* __restrict__ scale_dev)
{
    __shared__ double sm[32];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
        v = warp_sum(v);
        if (threadIdx.x == 0) out[0] = (kDevScale ? *scale_dev : scale) * v;
    }
}

// ---------------------------------------------------------------------------------------------
// gradient + Hessian
// ---------------------------------------------------------------------------------------------
DEV void tma_store_tile(void* gdst, const void* ssrc, unsigned bytes)
{
    // cp.async.bulk moves multiples of 16 bytes: a partial tile with an odd tet count and 9-double blocks (ntile * 72 B) is rounded UP --
    // the extra 8 bytes land in the next tet's (unused) place inside the same slot region of the tile, which always has room for 64 tets.
    // (Round 1 passed the raw size: the last block entry of the last tet was dropped whenever nT % 64 was odd -- found by the C3 scene.)
    bytes = (bytes + 15u) & ~15u;
    // make the generic-proxy smem writes visible to the async proxy, then one bulk copy
    unsigned saddr = (unsigned)__cvta_generic_to_shared(ssrc);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(gdst), "r"(saddr), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
}

// Output layout of the per-tet Hessian blocks ("tile-major"): tets are grouped in tiles of kHessTile = 64; inside a tile the
// 10 block slots follow each other (4 diagonal blocks of 6 upper scalars, then the 6 off-diagonal 3x3 blocks of the vertex pairs
// (0,1)(0,2)(0,3)(1,2)(1,3)(2,3)), and inside a slot the 64 tets are contiguous:
//     address(t, slot offset o, entry q) = (t/64)*64*78 + o*64 + (t%64)*len(o) + q,   o in {0,6,12,18,24,33,...,69}, len = 6 or 9.
// Every (tile, slot) region is therefore one contiguous 3 KB / 4.5 KB run that a CTA ships with a single TMA bulk store as soon
// as the slot is computed; only two such regions live in shared memory at a time (9 KB instead of 46 KB per CTA), which lifts the
// shared-memory occupancy limit of the first version of this kernel.
// block slots of a tet in emission order: (a, b) local vertex pair, offset of the slot inside a tile (in units of 64 doubles), length

// One 64-tet tile per CTA, compiled for 8 CTAs per SM (128 registers).  DESIGN.md ("Defaults re-checked on H100") keeps the timings
// of 2- and 4-tile CTAs and of 6, 10 and 12 CTAs per SM: none was faster.
template <int ENERGY, bool NEED_G, bool NEED_H>
__global__ void __launch_bounds__(kHessTile, 8) k_elastic_grad_hess(ElasticArgs p, double coef, int projectSPD,
    double* __restrict__ gcont /* 12 per LOCAL tet */, double* __restrict__ hblk /* tile-major, 78 per LOCAL tet */, double* __restrict__ e_partials /* nullable */)
{
    double e_tet = 0.0; // fused energy: psi * vol of this thread's tet (computeEnergyVal at the same state shares the SVD, like the reference's cache)
    extern __shared__ __align__(128) double smem[];
    const int tx = threadIdx.x;
    double* sHb[2] = { smem, smem + kHessTile * 9 };          // two slot buffers (ping-pong)
    double* sG = smem + (NEED_H ? 2 * kHessTile * 9 : 0);     // kHessTile * 12
    const int nLocal = p.n_list;
    const int tileI = blockIdx.x;
    const int tile0 = tileI * kHessTile;
    const int t = tile0 + tx;
    const bool active = t < nLocal;
    const int ntile = max(min(kHessTile, nLocal - tile0), 0);
    TetIn in;
    M3 U;
    double W[4][3];
    double a00 = 0, a01 = 0, a02 = 0, a11 = 0, a12 = 0, a22 = 0, d01 = 0, d10 = 0, o01 = 0, d12 = 0, d21 = 0, o12 = 0, d20 = 0, d02 = 0, o02 = 0;
    if (active) {
        const int tt = p.tet_list ? __ldg(p.tet_list + t) : p.t_begin + t;
        load_tet(p, tt, in);
        M3 F, V;
        double s[3];
        def_grad(in, F);
        svd3<true>(F, U, s, V);
        const double w = coef * in.vol;
        if (e_partials) {
            const int vmin = min(min(in.v[0], in.v[1]), min(in.v[2], in.v[3]));
            if (vmin >= p.e_row_lo && vmin < p.e_row_hi) e_tet = psi<ENERGY>(s, in.mu, in.lam) * in.vol;
        }

        if (NEED_G) {
            M3 P;
            pk1<ENERGY>(F, U, s, V, in.mu, in.lam, P);
            // g[3(i+1)+k] = w * sum_j A(i,j) P(k,j) ; g[k] = -sum_i   (IglUtils.cpp:656-667)
            double* g = sG + tx * 12;
            double g0 = 0.0, g1 = 0.0, g2 = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                double a = w * (in.A(i, 0) * P(0, 0) + in.A(i, 1) * P(0, 1) + in.A(i, 2) * P(0, 2));
                double b = w * (in.A(i, 0) * P(1, 0) + in.A(i, 1) * P(1, 1) + in.A(i, 2) * P(1, 2));
                double c = w * (in.A(i, 0) * P(2, 0) + in.A(i, 1) * P(2, 1) + in.A(i, 2) * P(2, 2));
                g[3 + 3 * i] = a;
                g[4 + 3 * i] = b;
                g[5 + 3 * i] = c;
                g0 -= a;
                g1 -= b;
                g2 -= c;
            }
            g[0] = g0;
            g[1] = g1;
            g[2] = g2;
        }

        if (NEED_H) {
            SigmaDerivs sd;
            sigma_derivs<ENERGY>(s, in.mu, in.lam, sd);
            if (projectSPD) make_pd3(sd.A);
            // B blocks for sigma pairs (0,1), (1,2), (2,0)   [Energy.cpp:468-491]
            double bd0[3], bd1[3], bo[3]; // B(0,0), B(1,1), B(0,1)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int cp = (c + 1) % 3;
                double right = sd.dE[c] + sd.dE[cp];
                const double sum = s[c] + s[cp];
                right /= 2.0 * ((sum < 1.0e-6) ? 1.0e-6 : sum);
                double pp = sd.BL[c] + right, qq = sd.BL[c] - right, rr = pp;
                if (projectSPD) make_pd2(pp, qq, rr);
                bd0[c] = pp;
                bd1[c] = rr;
                bo[c] = qq;
            }
            // weights in (k,l) index space   [Energy.cpp:497-528; note the transposed (2,0) block]
            //   d[k][l] = M(kl,kl), o[k][m] = M(km,mk)
            a00 = w * sd.A[0]; a01 = w * sd.A[1]; a02 = w * sd.A[2]; a11 = w * sd.A[3]; a12 = w * sd.A[4]; a22 = w * sd.A[5];
            d01 = w * bd0[0]; d10 = w * bd1[0]; o01 = w * bo[0];
            d12 = w * bd0[1]; d21 = w * bd1[1]; o12 = w * bo[1];
            d20 = w * bd0[2]; d02 = w * bd1[2]; o02 = w * bo[2];
            // W = G V
#pragma unroll
            for (int l = 0; l < 3; ++l) {
                double s0 = 0.0;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    double v = in.A(a, 0) * V(0, l) + in.A(a, 1) * V(1, l) + in.A(a, 2) * V(2, l);
                    W[a + 1][l] = v;
                    s0 -= v;
                }
                W[0][l] = s0;
            }
        }
    }
    if (NEED_H) {
        int slot = 0;
        int offd = 24; // old-style offset of the next off-diagonal block
#pragma unroll
        for (int a = 0; a < 4; ++a) {
#pragma unroll
            for (int b = a; b < 4; ++b) {
                const int len = (a == b) ? 6 : 9;
                const int o = (a == b) ? 6 * a : offd;
                if (a != b) offd += 9;
                double* buf = sHb[slot & 1];
                if (active) {
                    const double wa0 = W[a][0], wa1 = W[a][1], wa2 = W[a][2];
                    const double wb0 = W[b][0], wb1 = W[b][1], wb2 = W[b][2];
                    // Ht (U-frame) 3x3
                    M3 Ht;
                    Ht(0, 0) = a00 * wa0 * wb0 + d01 * wa1 * wb1 + d02 * wa2 * wb2;
                    Ht(1, 1) = a11 * wa1 * wb1 + d10 * wa0 * wb0 + d12 * wa2 * wb2;
                    Ht(2, 2) = a22 * wa2 * wb2 + d20 * wa0 * wb0 + d21 * wa1 * wb1;
                    Ht(0, 1) = a01 * wa0 * wb1 + o01 * wa1 * wb0;
                    Ht(1, 0) = a01 * wa1 * wb0 + o01 * wa0 * wb1;
                    Ht(0, 2) = a02 * wa0 * wb2 + o02 * wa2 * wb0;
                    Ht(2, 0) = a02 * wa2 * wb0 + o02 * wa0 * wb2;
                    Ht(1, 2) = a12 * wa1 * wb2 + o12 * wa2 * wb1;
                    Ht(2, 1) = a12 * wa2 * wb1 + o12 * wa1 * wb2;
                    // T = U * Ht ; H = T * U^T
                    M3 Tm;
#pragma unroll
                    for (int i = 0; i < 3; ++i)
#pragma unroll
                        for (int m = 0; m < 3; ++m) Tm(i, m) = U(i, 0) * Ht(0, m) + U(i, 1) * Ht(1, m) + U(i, 2) * Ht(2, m);
                    double* oo = buf + tx * len;
                    if (a == b) {
                        int q = 0;
#pragma unroll
                        for (int i = 0; i < 3; ++i)
#pragma unroll
                            for (int r = i; r < 3; ++r) oo[q++] = Tm(i, 0) * U(r, 0) + Tm(i, 1) * U(r, 1) + Tm(i, 2) * U(r, 2);
                    }
                    else {
                        const bool flip = in.v[a] > in.v[b]; // rows must belong to the smaller global vertex
#pragma unroll
                        for (int i = 0; i < 3; ++i)
#pragma unroll
                            for (int r = 0; r < 3; ++r) {
                                double h = Tm(i, 0) * U(r, 0) + Tm(i, 1) * U(r, 1) + Tm(i, 2) * U(r, 2);
                                oo[flip ? (3 * r + i) : (3 * i + r)] = h;
                            }
                    }
                }
                // ship this slot: generic-proxy writes -> async-proxy fence -> CTA barrier -> one elected TMA store
                asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
                __syncthreads();
                if (tx == 0 && ntile > 0) {
                    tma_store_tile(hblk + (size_t)tileI * (kHessTile * 78) + (size_t)o * kHessTile, buf, (unsigned)ntile * (unsigned)len * 8u);
                    asm volatile("cp.async.bulk.wait_group.read 1;\n" ::: "memory"); // the other buffer's store has been read out
                }
                __syncthreads();
                ++slot;
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
    __syncthreads();
    if (tx == 0) {
        if (NEED_G && ntile > 0) tma_store_tile(gcont + (size_t)tile0 * 12, sG, (unsigned)ntile * 12u * 8u);
        asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory");
    }
    if (e_partials) { // fixed-order CTA sum: warp sums, then warp 0 adds them in warp order
        __shared__ double sE[2];
        const double ws = warp_sum(e_tet);
        if ((threadIdx.x & 31) == 0) sE[threadIdx.x >> 5] = ws;
        __syncthreads();
        if (threadIdx.x == 0) {
            double acc = 0.0;
#pragma unroll
            for (int i = 0; i < 2; ++i) acc += sE[i];
            e_partials[blockIdx.x] = acc;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// vertex gather of the per-tet gradients (Energy.cpp:270-282): ascending (tet, local) order
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gather_gradient(int nV, const int* __restrict__ inc_ptr, const int* __restrict__ inc /* 4*tet+loc */,
    const double* __restrict__ gcont, const uint8_t* __restrict__ dbc, int projectDBC, int accumulate, double* __restrict__ g)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    double gx = 0.0, gy = 0.0, gz = 0.0;
    const int e = inc_ptr[v + 1];
    for (int q = inc_ptr[v]; q < e; ++q) {
        const int id = __ldg(inc + q);
        const double* s = gcont + (size_t)(id >> 2) * 12 + 3 * (id & 3);
        gx += s[0];
        gy += s[1];
        gz += s[2];
    }
    if (projectDBC && dbc && dbc[v]) gx = gy = gz = 0.0; // Energy.cpp:284-288
    if (accumulate) {
        g[3 * (size_t)v] += gx;
        g[3 * (size_t)v + 1] += gy;
        g[3 * (size_t)v + 2] += gz;
    }
    else {
        g[3 * (size_t)v] = gx;
        g[3 * (size_t)v + 1] = gy;
        g[3 * (size_t)v + 2] = gz;
    }
}

// ---------------------------------------------------------------------------------------------
// CSR assembly (Energy.cpp:317-330 -> IglUtils::addBlockToMatrix -> LinSysSolver::addCoeff):
// one thread per entry of a block-slot (vertex pair v<=u of the mesh topology); contributions are summed in
// ascending tet order (the reference's vFLoc order), then written to the three CSR rows.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(288) k_assemble_csr(int nOff, int nSlots, const int* __restrict__ slot_v, const int* __restrict__ slot_u,
    const int* __restrict__ slot_off /* 3 per slot */, const int* __restrict__ con_ptr, const unsigned* __restrict__ con_src,
    const double* __restrict__ hblk, const uint8_t* __restrict__ dbc, int projectDBC, const double* __restrict__ mass,
    int accumulate, double* __restrict__ a)
{
    // Consecutive threads per slot, one per stored entry: 9 for the off-diagonal slots [0, nOff), 6 for the diagonal ones after them
    // (build_maps orders them so; a diagonal block stores its 6 upper entries).  Thread q sums entry q of every contributing block
    // (ascending tet order: the reference's vFLoc order, so the sum is bitwise reproducible); the loads of one block are one contiguous run
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, tOff = 9ll * nOff;
    int sIdx, q;
    if (tid < tOff) {
        sIdx = (int)(tid / 9);
        q = (int)(tid - 9ll * sIdx);
    }
    else {
        const int k = (int)((tid - tOff) / 6);
        sIdx = nOff + k;
        q = (int)(tid - tOff - 6ll * k);
    }
    if (sIdx >= nSlots) return;
    const int v = slot_v[sIdx], u = slot_u[sIdx];
    const bool diag = (v == u);
    if (diag && q >= 6) return;
    const bool pv = dbc && (dbc[v] == 1 || (dbc[v] == 2 && projectDBC));
    const bool pu = dbc && (dbc[u] == 1 || (dbc[u] == 2 && projectDBC));
    const bool dropped = pv || pu; // projected Dirichlet vertex: block dropped; the identity is written by k_diag_mass_dbc
    double h = 0.0;
    if (!dropped) {
        const int b = con_ptr[sIdx], e = con_ptr[sIdx + 1];
        // (round 1: an explicit 8-deep load batch was slower -- but slot lists were then mixed 5- and 23-long inside a warp)
#pragma unroll 4
        for (int k = b; k < e; ++k) h += hblk[__ldg(con_src + k) + q];
    }
    int r, c;
    if (diag) { r = (q < 3) ? 0 : (q < 5 ? 1 : 2); c = (q < 3) ? q : (q < 5 ? q - 3 : 0); }
    else { r = q / 3; c = q - 3 * r; }
    const int o = slot_off[3 * sIdx + r] + c;
    // accumulate == 0: the value array was cleared before, so a[o] = h is 0 + h without reading a[o] (a sum from +0.0 is never -0.0)
    if (accumulate) {
        if (!dropped) a[o] += h;
        else if (diag) a[o] = 0.0;
    }
    else a[o] = h;
    (void)mass;
}

// per-vertex diagonal terms of computePrecondMtr (Optimizer.cpp:3638-3668): mass on free vertices, identity on projected
// Dirichlet vertices (setCoeff, also IglUtils.hpp:44-53).  The diagonal is the first stored entry of an upper-triangular row.
__global__ void __launch_bounds__(256) k_diag_mass_dbc(int v0, int nV, const int* __restrict__ ia, int base, const uint8_t* __restrict__ dbc, int projectDBC,
    const double* __restrict__ mass, double* __restrict__ a)
{
    const int v = v0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nV) return;
    const bool pv = dbc && (dbc[v] == 1 || (dbc[v] == 2 && projectDBC));
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int o = ia[3 * v + r] - base;
        if (pv) a[o] = 1.0;
        else if (mass) a[o] += mass[v];
    }
}

// slot -> CSR offsets (binary search of column 3u in rows 3v, 3v+1, 3v+2)
__global__ void __launch_bounds__(256) k_slot_offsets(int nSlots, const int* __restrict__ slot_v, const int* __restrict__ slot_u,
    const int* __restrict__ ia, const int* __restrict__ ja, int base, int* __restrict__ slot_off, int* __restrict__ err, const int* __restrict__ gate)
{
    const int sIdx = blockIdx.x * blockDim.x + threadIdx.x;
    if (sIdx >= nSlots || (gate && !*gate)) return;
    const int v = slot_v[sIdx], u = slot_u[sIdx];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int row = 3 * v + r;
        const int col = (v == u) ? row : 3 * u;
        int lo = ia[row] - base, hi = ia[row + 1] - base;
        const int target = col + base;
        int found = -1;
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            int c = ja[mid];
            if (c < target) lo = mid + 1;
            else hi = mid;
        }
        if (lo < ia[row + 1] - base && ja[lo] == target) found = lo;
        if (found < 0) atomicExch(err, 1);
        slot_off[3 * sIdx + r] = found;
    }
}

// ---------------------------------------------------------------------------------------------
// inversion step bound (get_feasible_steps.cpp:75-172 + Energy.cpp:565-581)
// ---------------------------------------------------------------------------------------------
struct Cplx {
    double re, im;
};
DEV Cplx cmul(Cplx a, Cplx b) { return { a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re }; }
DEV Cplx cdiv(Cplx a, Cplx b)
{
    // Smith's algorithm (the scaling libgcc's __divdc3 effectively provides for finite operands)
    if (fabs(b.re) >= fabs(b.im)) {
        double r = b.im / b.re, den = b.re + b.im * r;
        return { (a.re + a.im * r) / den, (a.im - a.re * r) / den };
    }
    else {
        double r = b.re / b.im, den = b.re * r + b.im;
        return { (a.re * r + a.im) / den, (a.im * r - a.re) / den };
    }
}
DEV Cplx csqrt_(Cplx z)
{
    if (z.re == 0.0 && z.im == 0.0) return { 0.0, z.im };
    double m = hypot(z.re, z.im);
    if (z.re >= 0.0) {
        double t = sqrt(0.5 * (m + z.re));
        return { t, z.im / (2.0 * t) };
    }
    else {
        double t = sqrt(0.5 * (m - z.re));
        return { fabs(z.im) / (2.0 * t), copysign(t, z.im) };
    }
}
DEV Cplx cpow_third(Cplx z)
{
    if (z.im == 0.0 && z.re > 0.0) return { pow(z.re, 1.0 / 3.0), 0.0 };
    if (z.re == 0.0 && z.im == 0.0) return { 0.0, 0.0 };
    double lr = log(hypot(z.re, z.im)), th = atan2(z.im, z.re);
    double rho = exp((1.0 / 3.0) * lr), ang = (1.0 / 3.0) * th;
    return { rho * cos(ang), rho * sin(ang) };
}
DEV double quad_root(double a, double b, double c, double tol)
{
    double t;
    if (fabs(a) <= tol) t = -c / b;
    else {
        double desc = b * b - 4 * a * c;
        if (desc > 0) {
            t = (-b - sqrt(desc)) / (2 * a);
            if (t < 0) t = (-b + sqrt(desc)) / (2 * a);
        }
        else t = -1;
    }
    return t;
}
DEV double cubic_root(double a, double b, double c, double d, double tol)
{
    double t = -1;
    if (fabs(a) <= tol) return quad_root(b, c, d, tol);
    const double delta0 = b * b - 3 * a * c;
    const double delta1 = 2 * b * b * b - 9 * a * b * c + 27 * a * a * d;
    Cplx rad = csqrt_({ delta1 * delta1 - 4.0 * delta0 * delta0 * delta0, 0.0 });
    Cplx C = cpow_third({ (delta1 + rad.re) / 2.0, rad.im / 2.0 });
    if (hypot(C.re, C.im) == 0.0) C = cpow_third({ (delta1 - rad.re) / 2.0, -rad.im / 2.0 });
    const double h = sqrt(3.0) / 2.0;
    const Cplx u2 = { -0.5, h }, u3 = { -0.5, -h };
    const Cplx d0 = { delta0, 0.0 };
    const double den = -3.0 * a;
    Cplx q1 = cdiv(d0, C);
    Cplx t1 = { (b + C.re + q1.re) / den, (C.im + q1.im) / den };
    Cplx c2 = cmul(u2, C), q2 = cdiv(d0, c2);
    Cplx t2 = { (b + c2.re + q2.re) / den, (c2.im + q2.im) / den };
    Cplx c3 = cmul(u3, C), q3 = cdiv(d0, c3);
    Cplx t3 = { (b + c3.re + q3.re) / den, (c3.im + q3.im) / den };
    if (fabs(t1.im) < tol && t1.re > 0) t = t1.re;
    if (fabs(t2.im) < tol && t2.re > 0 && (t2.re < t || t < 0)) t = t2.re;
    if (fabs(t3.im) < tol && t3.re > 0 && (t3.re < t || t < 0)) t = t3.re;
    return t;
}
DEV double det3v(const double* a, const double* b, const double* c)
{
    return a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) + a[2] * (b[0] * c[1] - b[1] * c[0]);
}

__global__ void k_inversion_init(IterState* st)
{
    if (threadIdx.x == 0) st->inv_ord = 0x7ff0000000000000ull; // +inf
}
// Energy.cpp:576-579 on the device-resident step: "if (0 < min && min < stepSize) stepSize = min"
__global__ void k_inversion_apply(IterState* st, int nT)
{
    if (threadIdx.x != 0) return;
    const double m = ord_to_dbl(st->inv_ord), alpha = ord_to_dbl(st->step_ord);
    if (nT > 0 && m > 0.0 && m < alpha) st->step_ord = dbl_to_ord(m);
    st->alpha_stage[0] = ord_to_dbl(st->step_ord);
}
__global__ void k_step_set(IterState* st, double alpha)
{
    if (threadIdx.x == 0) st->step_ord = dbl_to_ord(alpha);
}

__global__ void __launch_bounds__(256) k_inversion_step(ElasticArgs p, const double* __restrict__ dir /* interleaved 3nV */, double slack,
    double* __restrict__ per_tet, unsigned long long* __restrict__ min_ord)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    double out = 1e300;
    if (t < p.t_end - p.t_begin) {
        const int tt = p.t_begin + t;
        int v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = __ldg(p.T + (size_t)k * p.nT + tt);
        double x[4][3], d[4][3];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                x[k][c] = __ldg(p.V + (size_t)c * p.nV + v[k]);
                d[k][c] = __ldg(dir + 3 * (size_t)v[k] + c);
            }
        double e[3][3], f[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                e[k][c] = x[k + 1][c] - x[0][c];
                f[k][c] = d[k + 1][c] - d[0][c];
            }
        const double ca = det3v(f[0], f[1], f[2]);
        const double cb = det3v(e[0], f[1], f[2]) + det3v(f[0], e[1], f[2]) + det3v(f[0], f[1], e[2]);
        const double cc = det3v(f[0], e[1], e[2]) + det3v(e[0], f[1], e[2]) + det3v(e[0], e[1], f[2]);
        const double cd = (1.0 - slack) * det3v(e[0], e[1], e[2]);
        const double r = cubic_root(ca, cb, cc, cd, 1.0e-6);
        out = (r >= 0) ? r : 1e20;
        if (per_tet) per_tet[tt] = out;
    }
    // min over the CTA of out + 0.0.  A bound is r >= 0 or 1e20, but r can be -0.0 (-0/c in the linear exit, +0/(2a) with a < 0 in the
    // quadratic one), whose bits would order above every positive bound.  Energy.cpp:576-579 takes minCoeff with `<`, where either zero is
    // the minimum wherever it lies and fails `0 < min`; adding +0.0 makes both zeros +0.0, the smallest key of the ordered-uint atomicMin
    // (here and across ranks), so k_inversion_apply rejects it the same way.  per_tet keeps the signed value.
    double m = warp_min(__dadd_rn(out, 0.0));
    __shared__ double sm[8];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        double mm = sm[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) mm = fmin(mm, sm[i]);
        atomicMin(min_ord, dbl_to_ord(mm));
    }
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
void elastic_energy(const ElasticArgs& p, double* e_per_tet, double* partials, cudaStream_t st)
{
    const int nb = elastic_energy_blocks(p.t_end - p.t_begin);
    if (nb <= 0) return;
    if (p.energy == 0) k_elastic_energy<0><<<nb, 256, 0, st>>>(p, e_per_tet, partials);
    else k_elastic_energy<1><<<nb, 256, 0, st>>>(p, e_per_tet, partials);
}
int elastic_energy_blocks(int nTets) { return (nTets + 255) / 256; }
void reduce_sum(const double* partials, int n, double scale, double* out, cudaStream_t st, const double* scale_dev)
{
    if (scale_dev) k_reduce_sum<true><<<1, 1024, 0, st>>>(partials, n, scale, out, scale_dev);
    else k_reduce_sum<false><<<1, 1024, 0, st>>>(partials, n, scale, out, nullptr);
}

int elastic_grad_hess_blocks(int n_list) { return (n_list + kHessTile - 1) / kHessTile; }
template <int ENERGY, bool G, bool H>
static void launch_gh(const ElasticArgs& p, double coef, int projectSPD, double* gcont, double* hblk, cudaStream_t st, double* e_partials)
{
    const int n = p.n_list;
    if (n <= 0) return;
    const size_t smem = (size_t)kHessTile * 8 * ((H ? 18 : 0) + (G ? 12 : 0));
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(k_elastic_grad_hess<ENERGY, G, H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_set = true;
    }
    k_elastic_grad_hess<ENERGY, G, H><<<elastic_grad_hess_blocks(n), kHessTile, smem, st>>>(p, coef, projectSPD, gcont, hblk, e_partials);
}
void elastic_grad_hess(const ElasticArgs& p, double coef, int projectSPD, bool need_g, bool need_h, double* gcont, double* hblk, cudaStream_t st, double* e_partials)
{
    if (p.energy == 0) {
        if (need_g && need_h) launch_gh<0, true, true>(p, coef, projectSPD, gcont, hblk, st, e_partials);
        else if (need_g) launch_gh<0, true, false>(p, coef, projectSPD, gcont, hblk, st, e_partials);
        else if (need_h) launch_gh<0, false, true>(p, coef, projectSPD, gcont, hblk, st, e_partials);
    }
    else {
        if (need_g && need_h) launch_gh<1, true, true>(p, coef, projectSPD, gcont, hblk, st, e_partials);
        else if (need_g) launch_gh<1, true, false>(p, coef, projectSPD, gcont, hblk, st, e_partials);
        else if (need_h) launch_gh<1, false, true>(p, coef, projectSPD, gcont, hblk, st, e_partials);
    }
}

void gather_gradient(int nV, const int* inc_ptr, const int* inc, const double* gcont, const uint8_t* dbc, int projectDBC, int accumulate, double* g, cudaStream_t st)
{
    if (nV <= 0) return;
    k_gather_gradient<<<(nV + 255) / 256, 256, 0, st>>>(nV, inc_ptr, inc, gcont, dbc, projectDBC, accumulate, g);
}
void assemble_csr(int nOff, int nSlots, const int* slot_v, const int* slot_u, const int* slot_off, const int* con_ptr, const unsigned* con_src,
    const double* hblk, const uint8_t* dbc, int projectDBC, const double* mass, int accumulate, double* a, cudaStream_t st)
{
    if (nSlots <= 0) return;
    const int nb = (int)(((long long)nOff * 9 + (long long)(nSlots - nOff) * 6 + 287) / 288);
    k_assemble_csr<<<nb, 288, 0, st>>>(nOff, nSlots, slot_v, slot_u, slot_off, con_ptr, con_src, hblk, dbc, projectDBC, mass, accumulate, a);
}
void diag_mass_dbc(int nV, const int* ia, int base, const uint8_t* dbc, int projectDBC, const double* mass, double* a, cudaStream_t st)
{
    if (nV > 0 && (dbc || mass)) k_diag_mass_dbc<<<(nV + 255) / 256, 256, 0, st>>>(0, nV, ia, base, dbc, projectDBC, mass, a);
}
// the same over the vertex range [v0, v1) (row-owner partition: every rank writes the diagonal terms of its own rows)
void diag_mass_dbc_range(int v0, int v1, const int* ia, int base, const uint8_t* dbc, int projectDBC, const double* mass, double* a, cudaStream_t st)
{
    if (v1 > v0 && (dbc || mass)) k_diag_mass_dbc<<<(v1 - v0 + 255) / 256, 256, 0, st>>>(v0, v1, ia, base, dbc, projectDBC, mass, a);
}
void slot_offsets(int nSlots, const int* slot_v, const int* slot_u, const int* ia, const int* ja, int base, int* slot_off, int* err, cudaStream_t st, const int* gate)
{
    if (nSlots <= 0) return;
    k_slot_offsets<<<(nSlots + 255) / 256, 256, 0, st>>>(nSlots, slot_v, slot_u, ia, ja, base, slot_off, err, gate);
}
void inversion_step(const ElasticArgs& p, const double* dir, double slack, double* per_tet, IterState* st_dev, cudaStream_t st)
{
    k_inversion_init<<<1, 32, 0, st>>>(st_dev);
    const int n = p.t_end - p.t_begin;
    if (n <= 0) return;
    k_inversion_step<<<(n + 255) / 256, 256, 0, st>>>(p, dir, slack, per_tet, &st_dev->inv_ord);
}
void inversion_apply(IterState* st_dev, int nT, cudaStream_t st) { k_inversion_apply<<<1, 32, 0, st>>>(st_dev, nT); }
void step_set(IterState* st_dev, double alpha, cudaStream_t st) { k_step_set<<<1, 32, 0, st>>>(st_dev, alpha); }

// Deferred cross-rank scalars of one iteration in ONE collective (kernels.h: kPackedScalars): buf = the energies, the flags, the checks and
// the crossing count; a scalar that is not a local share (local_mask) packs as 0 and keeps its value.
constexpr int kFlags = kEnergySlots, kChecks = kFlags + kFlagSlots, kCrossings = kChecks + 2;
static_assert(kCrossings + 1 == kPackedScalars && kPackedScalars <= 32, "one warp packs the scalars");
__global__ void k_pack_scalars(const IterState* __restrict__ st, unsigned local_mask, double* __restrict__ buf)
{
    const int i = threadIdx.x;
    if (i < kFlags) buf[i] = ((local_mask >> i) & 1u) ? st->energy[i] : 0.0;
    else if (i < kChecks) buf[i] = (double)st->flags[i - kFlags];
    else if (i < kCrossings) buf[i] = (local_mask & kLocalChecks) ? (double)st->checks[i - kChecks] : 0.0;
    else if (i == kCrossings) buf[i] = (local_mask & kLocalCrossings) ? (double)st->hs_crossings : 0.0;
}
__global__ void k_unpack_scalars(IterState* __restrict__ st, unsigned local_mask, const double* __restrict__ buf)
{
    const int i = threadIdx.x;
    if (i < kFlags) { if ((local_mask >> i) & 1u) st->energy[i] = buf[i]; }
    else if (i < kChecks) st->flags[i - kFlags] = (int)fmin(buf[i], 2147483647.0);
    else if (i < kCrossings) { if (local_mask & kLocalChecks) st->checks[i - kChecks] = (int)buf[i]; }
    else if (i == kCrossings) { if (local_mask & kLocalCrossings) st->hs_crossings = (int)buf[i]; }
}
void pack_scalars(const IterState* st_dev, unsigned local_mask, double* buf, cudaStream_t st) { k_pack_scalars<<<1, 32, 0, st>>>(st_dev, local_mask, buf); }
void unpack_scalars(IterState* st_dev, unsigned local_mask, const double* buf, cudaStream_t st) { k_unpack_scalars<<<1, 32, 0, st>>>(st_dev, local_mask, buf); }

} // namespace ipcgpu
