// repro.cuh -- the fixed-order sums of the reproducible mode (ipcgpu_set_canonical_order(ctx, 2)), shared by the term kernels.
//
// A term kernel leaves each contribution where its list position puts it (stage), and one thread per vertex adds the contributions of its
// vertex in the order of VertexIndex (ascending key, i.e. list position, then local vertex), then adds the sum to g or to a CSR block once.
// The index depends on the lists alone (repro.cu builds it where a list is produced), so the sums are the same bits for every schedule
// and for every order the lists arrived in.
#pragma once
#include "pair_common.cuh"
#include "kernels.h"

namespace ipcgpu {

// Gradient keys: the staging slot of a contribution and its place in a vertex's sum.  Active entry c, stencil vertex k: 4c + k.  Mollified
// entry c: 4 cap + 8c + k on its edge stencil, 4 cap + 8c + 4 + k on its distance stencil.  So the active list's keys are [0, para_keys(cap))
// and the mollified list's [para_keys(cap), kAllKeys).
constexpr unsigned long long kAllKeys = ~0ull;
__host__ __device__ inline unsigned long long para_keys(int cap) { return 4ull * cap; }
DEV unsigned long long gkey_active(int c, int k) { return 4ull * c + k; }
DEV unsigned long long gkey_para_edge(int cap, int c, int k) { return para_keys(cap) + 8ull * c + k; }
DEV unsigned long long gkey_para_dist(int cap, int c, int k) { return para_keys(cap) + 8ull * c + 4 + k; }

// kStage: contribution (key, component q) goes to its own slot of the staging array, for k_repro_gather_g to sum; otherwise it is added at
// its vertex
template <bool kStage>
DEV void put_g(double* __restrict__ g, int v, unsigned long long key, int q, double val)
{
    if (kStage) g[3 * key + q] = val;
    else atomicAdd(g + 3 * (size_t)v + q, val);
}

// Hessian block key: column vertex << 32 | list index << 4 | block (bi << 2 | bj), so a row's entries sort by column vertex, then list
// position.  The list index is kept on 28 bits (repro_alloc caps the pair capacity at 2^27).
DEV unsigned long long hkey(int vj, int c, int bi, int bj) { return ((unsigned long long)vj << 32) | ((unsigned)c << 4) | (unsigned)(bi << 2 | bj); }
DEV int hkey_col(unsigned long long key) { return (int)(key >> 32); }
DEV void hkey_block(unsigned long long key, int& c, int& bi, int& bj)
{
    const unsigned low = (unsigned)key;
    c = (int)(low >> 4);
    bi = (int)((low >> 2) & 3u);
    bj = (int)(low & 3u);
}

// g[v] += sum of stage[k] over the entries k of v with lo <= k < hi, in index order
__global__ void __launch_bounds__(256) k_repro_gather_g(int nV, VertexIndex idx, const double* __restrict__ stage, unsigned long long lo, unsigned long long hi,
    double* __restrict__ g);

// one row vertex v of a Hessian gather: the entries of v grouped by column vertex (the index is sorted on it), each group summed into one
// 3x3 block in index order by block(list index, bi, bj, acc) and added to the upper-triangular CSR once.  A row or column without degrees of
// freedom is skipped, as the atomic scatters skip it.
template <typename Block>
DEV void repro_gather_row(int v, const VertexIndex& idx, const uint8_t* __restrict__ dbc, int projectDBC, const int* __restrict__ ia, const int* __restrict__ ja,
    int base, double* __restrict__ a, int* __restrict__ err, Block block)
{
    const int b = idx.ptr[v], e = idx.ptr[v + 1];
    if (b == e || proj_dbc(dbc, v, projectDBC)) return;
    for (int j = b; j < e;) {
        const int vj = hkey_col(idx.key[j]);
        double acc[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) acc[i] = 0.0;
        for (; j < e && hkey_col(idx.key[j]) == vj; ++j) {
            int c, bi, bj;
            hkey_block(idx.key[j], c, bi, bj);
            block(c, bi, bj, acc);
        }
        if (proj_dbc(dbc, vj, projectDBC)) continue;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int c0 = (vj == v) ? r : 0; // a diagonal block: its upper part only
            const int o = csr_find(ia, ja, base, 3 * v + r, 3 * vj + c0);
            if (o < 0) {
                atomicExch(err, 1);
                continue;
            }
#pragma unroll
            for (int q = 0; q < 3; ++q) // (unrolled: acc stays in registers)
                if (q >= c0) a[o + (q - c0)] += acc[3 * r + q];
        }
    }
}

} // namespace ipcgpu
