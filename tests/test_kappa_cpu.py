"""ipcgpu_kappa_bounds (suggestKappa / upperBoundKappa, Optimizer.cpp:2216-2233) against the float64 restatement, bit for bit, over a grid
of dHat, bounding box, node mass and multiplier (host-only: no GPU needed)."""
import itertools

import pytest

import oracle_kappa as ok
from gpu_common import scalar_bits
from ipc_b200 import lib as L


@pytest.mark.parametrize("dHat", [1e-8, 3.7e-6, 1e-4, 2.5e-3])
def test_bounds_bits(dHat):
    for bbox2, mass, mult in itertools.product([1e-2, 1.0, 3.3, 250.0], [1e-6, 0.013, 2.0], [1e-11, 0.1, 1.0]):
        s, m = L.Context.kappa_bounds(dHat, mult, mass, bbox2)
        rs, rm = ok.bounds(dHat, mult, mass, bbox2)
        assert scalar_bits(s) == scalar_bits(rs) and scalar_bits(m) == scalar_bits(rm), (dHat, bbox2, mass, mult, s, rs, m, rm)
        assert 0.0 < s < m


def test_bounds_reject_bad_input():
    with pytest.raises(L.IpcGpuError):
        L.Context.kappa_bounds(0.0, 0.1, 1.0, 1.0)
    with pytest.raises(L.IpcGpuError):
        L.Context.kappa_bounds(1e-6, 0.1, 1.0, 0.0)
