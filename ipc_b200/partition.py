"""Host-side mirror of the multi-rank partition rule that libipcgpu.so applies (csrc/api_mesh.cu: build_maps), for callers that need to know
who owns what (which CSR rows to fetch from which rank) and for the CPU-side tests of the rule.

  tets      : block partition [nT*r/N, nT*(r+1)/N)            -- energy, inversion filter: every tet exactly once
  rows      : vertex ranges [b_r, b_{r+1}) with b_r = the first vertex whose cumulative incident-tet count reaches total*r/N
  assembly  : rank r assembles every tet that touches one of its vertices (boundary tets are assembled by both neighbours) and keeps
              the blocks (v, u), v <= u, whose ROW vertex v it owns; the owned rows of the CSR are then complete without any reduction
  contact   : a pair is assembled by every rank that owns one of its stencil vertices; each keeps the block rows it owns
  fused E   : in ipcgpu_elastic_energy_grad_hess a tet's energy is counted by the rank that owns its SMALLEST vertex: every tet exactly once,
              and that rank assembles the tet anyway
"""
import numpy as np


def tet_range(nT, rank, world):
    return nT * rank // world, nT * (rank + 1) // world


def vertex_boundaries(T, nV, world):
    """b[0..world]: rank r owns the rows of vertices [b[r], b[r+1])"""
    cnt = np.bincount(np.asarray(T).ravel(), minlength=nV).astype(np.int64)
    cum = np.concatenate([[0], np.cumsum(cnt)])
    b = [0]
    for r in range(1, world):
        b.append(int(np.searchsorted(cum, cum[-1] * r // world, side="left")))
    b.append(nV)
    b = [min(x, nV) for x in b]
    for r in range(1, world + 1):
        b[r] = max(b[r], b[r - 1])
    return b


def assembled_tets(T, vb, ve):
    """ids (ascending) of the tets that touch a vertex in [vb, ve)"""
    T = np.asarray(T)
    return np.nonzero(((T >= vb) & (T < ve)).any(axis=1))[0]


def owned_value_range(ia, index_base, vb, ve):
    """[begin, end) of the CSR values of rows 3*vb .. 3*ve-1"""
    return int(ia[3 * vb]) - index_base, int(ia[3 * ve]) - index_base


def energy_tets(T, vb, ve):
    """ids of the tets whose energy rank [vb, ve) counts in the fused energy + gradient + Hessian pass: smallest vertex owned"""
    vmin = np.asarray(T).min(axis=1)
    return np.nonzero((vmin >= vb) & (vmin < ve))[0]
