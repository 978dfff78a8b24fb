// pair_common.cuh -- MMCVID decoding, pair loading, pair-Hessian rows, CSR lookup and Dirichlet helpers shared by the per-pair kernels
// (barrier.cu, friction.cu, kappa.cu, pattern.cu) and the reproducible mode's indices (repro.cu)
#pragma once
#include "contact.cuh"

namespace ipcgpu {

struct PairStencil {
    int v[4];
    int nv;   // 2 PP, 3 PE, 4 PT/EE
    int kind; // 0 PT, 1 EE, 2 PE, 3 PP
    double mult;
};

DEV PairStencil decode(int4 mm)
{
    PairStencil s;
    s.mult = 1.0;
    if (mm.x >= 0) {
        s.v[0] = mm.x; s.v[1] = mm.y; s.v[2] = mm.z; s.v[3] = mm.w;
        s.nv = 4; s.kind = 1;
    }
    else {
        s.v[0] = -mm.x - 1; s.v[1] = mm.y; s.v[2] = mm.z; s.v[3] = mm.w;
        if (mm.z < 0) { s.nv = 2; s.kind = 3; s.mult = (double)(-mm.w); }
        else if (mm.w < 0) { s.nv = 3; s.kind = 2; s.mult = (double)(-mm.w); }
        else { s.nv = 4; s.kind = 0; }
    }
    return s;
}

DEV double pair_distance(const PairStencil& s, const V3* x)
{
    switch (s.kind) {
    case 0: return d_PT(x[0], x[1], x[2], x[3]);
    case 1: return d_EE(x[0], x[1], x[2], x[3]);
    case 2: return d_PE(x[0], x[1], x[2]);
    default: return d_PP(x[0], x[1]);
    }
}

DEV int csr_find(const int* __restrict__ ia, const int* __restrict__ ja, int base, int row, int col)
{
    int lo = ia[row] - base, hi = ia[row + 1] - base;
    const int end = hi, target = col + base;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (ja[mid] < target) lo = mid + 1;
        else hi = mid;
    }
    return (lo < end && ja[lo] == target) ? lo : -1;
}

// the vertices x of a decoded distance stencil.  (decode stays with the caller: a stencil returned from a loader changes the code of the
// barrier kernels, registers and stack frame)
DEV void load_stencil(const PairStencil& s, const double* __restrict__ V, int nV, V3* x)
{
    for (int k = 0; k < s.nv; ++k) x[k] = load_vertex(V, nV, s.v[k]);
}

// the squared distance of list entry mm at positions V
DEV double pair_distance(int4 mm, const double* __restrict__ V, int nV)
{
    const PairStencil s = decode(mm);
    V3 x[4];
    load_stencil(s, V, nV, x);
    return pair_distance(s, x);
}

// the two-edge stencil of a mollified (nearly parallel EE) entry: its own four vertices, or the edges (eI, eJ) it came from
DEV void para_edge_stencil(int4 mm, int2 e, const int* __restrict__ SE, int* ev)
{
    if (mm.w >= 0 && mm.x >= 0) { ev[0] = mm.x; ev[1] = mm.y; ev[2] = mm.z; ev[3] = mm.w; }
    else {
        ev[0] = SE[2 * e.x]; ev[1] = SE[2 * e.x + 1];
        ev[2] = SE[2 * e.y]; ev[3] = SE[2 * e.y + 1];
    }
}
// the edge stencil of a mollified entry with its vertices ex and the mollifier threshold eps_x of its rest edges
DEV double load_para_edges(int4 mm, int2 e, const int* __restrict__ SE, const double* __restrict__ V, const double* __restrict__ Vrest, int nV, int* ev, V3* ex)
{
    para_edge_stencil(mm, e, SE, ev);
    for (int k = 0; k < 4; ++k) ex[k] = load_vertex(V, nV, ev[k]);
    return eps_x_rest(Vrest, nV, ev[0], ev[1], ev[2], ev[3]);
}

// the vertex rows of an entry's pair-Hessian block (12x12, four 3-row blocks): an active entry's own stencil padded with -1, a mollified
// entry's edge stencil
DEV void hessian_rows(int4 mm, const PairStencil& s, bool is_para, const int2* __restrict__ para_e, int c, const int* __restrict__ SE, int* rows)
{
    if (!is_para)
        for (int k = 0; k < 4; ++k) rows[k] = (k < s.nv) ? s.v[k] : -1;
    else para_edge_stencil(mm, para_e[c], SE, rows);
}
// the 3x3 blocks (bi, bj) of a pair Hessian that go to the upper-triangular CSR: both rows present, vi <= vj, and on a repeated vertex the
// diagonal block only
DEV bool upper_block(const int* rows, int bi, int bj)
{
    const int vi = rows[bi], vj = rows[bj];
    return vi >= 0 && vj >= 0 && vi <= vj && !(vi == vj && bi != bj);
}

DEV bool proj_dbc(const uint8_t* dbc, int v, int projectDBC) { return dbc && (dbc[v] == 1 || (dbc[v] == 2 && projectDBC)); }

} // namespace ipcgpu
