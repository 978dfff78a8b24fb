"""ipcgpu_elastic_grad_hess clears the value array and then WRITES every slot's sum into it, without reading it back; the diagonal slots
take 6 threads each, the off-diagonal ones 9.  Every CSR entry must hold exactly the sum, from +0.0 in ascending tet order, of the
per-tet blocks the kernel left in IPCGPU_BUF_TET_HESSIANS -- bit for bit, signs of zeros included -- and the blocks of projected
Dirichlet vertices must be dropped (+0.0), with 1.0 on their diagonal."""
import numpy as np
import pytest

from gpu_common import shared_ctx
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

pytestmark = pytest.mark.gpu

DT2 = 0.025 ** 2
PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def reference(m, ia, ja, hblk, dropped):
    """the CSR values from the tile-major per-tet blocks (elastic.cu), summed on the host in ascending tet order"""
    pos = {}
    for row in range(3 * m.nV):
        for k in range(ia[row] - 1, ia[row + 1] - 1):
            pos[(row, ja[k] - 1)] = k
    T = m.T_soa.reshape(4, -1)
    idx, val = [], []
    for t in range(m.nT):
        base, tin = (t // 64) * 64 * 78, t % 64
        v = T[:, t]
        for a in range(4):
            if dropped[v[a]]:
                continue
            blk = hblk[base + 6 * a * 64 + tin * 6: base + 6 * a * 64 + tin * 6 + 6]
            q = 0
            for i in range(3):
                for r in range(i, 3):
                    idx.append(pos[(3 * v[a] + i, 3 * v[a] + r)])
                    val.append(blk[q])
                    q += 1
        for p, (a, b) in enumerate(PAIRS):
            lo, hi = min(v[a], v[b]), max(v[a], v[b])
            if dropped[lo] or dropped[hi]:
                continue
            o = base + (24 + 9 * p) * 64 + tin * 9
            for i in range(3):
                for r in range(3):
                    idx.append(pos[(3 * lo + i, 3 * hi + r)])
                    val.append(hblk[o + 3 * i + r])
    a_ref = np.zeros(ja.size)
    np.add.at(a_ref, np.asarray(idx), np.asarray(val))  # (unbuffered: in the order given)
    for vtx in np.nonzero(dropped)[0]:
        for r in range(3):
            a_ref[ia[3 * vtx + r] - 1] = 1.0
    return a_ref


@pytest.mark.parametrize("energy", [0, 1])
def test_written_assembly_is_the_ordered_sum_of_the_tet_blocks(shared_ctx, energy):
    V, T = M.grid_tets(9, 8, 7)
    m = M.Mesh(V, T, energy=energy)
    M.deform(m, 2)
    m.dbc[::17] = 1
    m.dbc[5::23] = 2
    shared_ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ia, ja = m.csr_pattern(1)
    shared_ctx.set_csr(ia, ja, 1)
    shared_ctx.set_state(m.V_soa)
    for projectDBC in (0, 1):
        g, a = np.empty(3 * m.nV), np.full(ja.size, np.nan)
        shared_ctx.elastic_grad_hess(DT2, 1, projectDBC, 0, g, a)
        hblk = shared_ctx.download(L.BUF_TET_HESSIANS, 78 * 64 * ((m.nT + 63) // 64))
        dropped = (m.dbc == 1) | ((m.dbc == 2) & bool(projectDBC))
        a_ref = reference(m, ia, ja, hblk, dropped)
        assert np.array_equal(a.view(np.uint64), a_ref.view(np.uint64)), projectDBC
        assert np.count_nonzero(a) > ja.size // 2
