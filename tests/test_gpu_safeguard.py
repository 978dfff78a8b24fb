"""GPU parity of the line-search safeguards (SURVEY 8(f) rank 2): element inversion count and edge-triangle intersection check,
through the C ABI against the oracle (exact predicate: the COUNTS must be identical)."""
import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, shared_ctx
from ipc_b200 import mesh as M
from ipc_b200 import scenes

pytestmark = pytest.mark.gpu


def two_cubes(dz, n=3):
    V1, T1 = M.grid_tets(n, n, n, h=1.0 / n)
    V2, T2 = M.grid_tets(n, n, n, h=1.0 / n, origin=(0.13, 0.21, dz))
    return M.merge_meshes([(V1, T1), (V2, T2)])


@pytest.mark.parametrize("dz,free", [(1.05, True), (0.8, False), (0.999, False)])
def test_intersection_check_matches_oracle(shared_ctx, dz, free):
    m = two_cubes(dz)
    rng = np.random.default_rng(3)
    m.V = m.V_rest + 0.01 * rng.standard_normal(m.V_rest.shape)
    load_scene(shared_ctx, m)
    ok_ref, hits_ref = orc.Surf(m).intersection_free(nthreads=4)
    assert ok_ref == free
    assert shared_ctx.intersection_free() == ok_ref
    shared_ctx.intersection_free(want=False)  # deferred form: the count comes back with the iteration
    shared_ctx.check_inversion(want=False)
    it = shared_ctx.fetch_iteration()
    assert it.n_intersected_triangles == hits_ref and it.n_inverted_tets == orc.Elastic(m).count_inverted()
    # all-Dirichlet pairs are skipped (:3282)
    m.dbc[:] = 1
    load_scene(shared_ctx, m)
    assert shared_ctx.intersection_free() is True
    m.dbc[:] = 0


def test_inversion_count_matches_oracle(shared_ctx):
    m = scenes.twisted_mat(nx=10, ny=10, nz=8, energy=1, invert_frac=0.02)  # FCR scene with flipped tets
    load_scene(shared_ctx, m)
    n_ref = orc.Elastic(m).count_inverted()
    assert n_ref > 0 and shared_ctx.check_inversion() == n_ref
    m.V = m.V_rest.copy()
    load_scene(shared_ctx, m)
    assert shared_ctx.check_inversion() == 0


def check_intersection_counts(ctx, m):
    load_scene(ctx, m)
    ok_ref, hits_ref = orc.Surf(m).intersection_free(nthreads=64)
    ctx.intersection_free(want=False)
    ctx.check_inversion(want=False)
    it = ctx.fetch_iteration()
    assert it.n_intersected_triangles == hits_ref and (hits_ref == 0) == ok_ref
    assert it.n_inverted_tets == 0


def test_c5_pile_intersection_counts(shared_ctx):
    """C5 (1M tets) is intersection free: the device must agree with the oracle at the full size."""
    import bench

    class A:
        tets, res, scene = 1_000_000, 10, "c5"

    check_intersection_counts(shared_ctx, bench.build_scene(A)[0])


@pytest.mark.skipif(not scenes.have_squeeze_out_bodies(), reason=scenes.SQUEEZE_OUT_MISSING)
def test_full_size_scenes_intersection_counts(shared_ctx):
    """C4's manufactured shell crosses its core in places (scenes.squeeze_out_tiled): the device must find exactly the triangles the
    oracle finds, degenerate near-coplanar configurations included.  (C5 is test_c5_pile_intersection_counts.)"""
    check_intersection_counts(shared_ctx, scenes.squeeze_out_tiled()[0])
