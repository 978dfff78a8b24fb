"""The point-in-tetrahedron half of the intersection check at full size: the C5 pile (146 x sphere1K.msh, 1M tets) with a cloud of 10^5
codimension-0 points in its box, some inside tets, the device count against the host count
(tests/oracle_codim.py: a k-d tree for the candidates, the oracle's exact orient3d for the decision)."""
import os

import numpy as np
import pytest

import oracle as orc
import oracle_codim as oc
from gpu_common import load_scene, shared_ctx
from ipc_b200 import codim

pytestmark = pytest.mark.gpu


class _Args:
    tets, res, scene = 1_000_000, 10, "c5"


def pile_with_points(n_points=100_000, seed=3):
    import bench
    m, info = bench.build_scene(_Args())
    rng = np.random.default_rng(seed)
    lo, hi = m.V.min(0), m.V.max(0)
    P = lo + (hi - lo) * rng.uniform(0.0, 1.0, (n_points, 3))
    mc = codim.codim_scene([dict(codim=3, V=m.V_rest, T=m.T, SF=m.SF), dict(codim=0, V=P)], energy=m.energy)
    mc.V[: m.nV] = m.V
    return mc, info


def test_c5_point_cloud_count(shared_ctx):
    m, _ = pile_with_points()
    pts = np.flatnonzero(m.vCoDim == 0).astype(np.int32)
    n_ref = oc.points_in_tets(m.V, m.T, pts, os.cpu_count() or 8)
    assert 1000 < n_ref < len(pts)
    _, hits_r = orc.Surf(m).intersection_free(nthreads=os.cpu_count() or 8)
    load_scene(shared_ctx, m)
    shared_ctx.intersection_free(want=False)
    assert shared_ctx.fetch_iteration().n_intersected_triangles == n_ref + hits_r
    assert shared_ctx.intersection_free() is False
