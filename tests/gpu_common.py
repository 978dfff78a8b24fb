"""Scaffolding shared by the test modules: array layout, bit comparisons, scene upload and the C-ABI contexts."""
import contextlib
import struct

import numpy as np
import pytest

from ipc_b200 import lib as L


def soa(V):
    """(n, 3) rows to the structure-of-arrays layout of the C ABI (x..., y..., z...)."""
    return np.ascontiguousarray(np.asarray(V).T).ravel()


def scalar_bits(x):
    """The bit image of one float64, for == tests."""
    return struct.pack("<d", float(x))


def same_bits(x, y):
    """True when two float64 arrays have equal shapes and equal bits."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    return np.array_equal(x.view(np.uint64), y.view(np.uint64))  # (False when the shapes differ)


def rel(a, b):
    """‖a − b‖ / max(‖b‖, 1e-300), for arrays and scalars."""
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


def load_scene(ctx, m, *, mass=True, dbc=True, vcodim=True):
    """Upload m's mesh, surface and current positions, in that order."""
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass if mass else None, m.dbc if dbc else None, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim if vcodim else None)
    ctx.set_state(m.V_soa)


@contextlib.contextmanager
def own_context():
    """A context of the test's own on cuda:0, closed on exit."""
    ctx = L.Context(0)
    try:
        yield ctx
    finally:
        ctx.close()


def _start_state(ctx):
    # a fresh context's value of every setting that survives ipcgpu_set_mesh; planes and an obstacle tail exist only with a mesh
    ctx.set_canonical_order(1)
    ctx.set_contact_partition(0)
    if ctx.nV:
        ctx.set_halfspaces([], [])
        ctx.set_obstacle_tail(-1)
    ctx.ccd_debug_thread_budget(-1)
    ctx.ccd_debug_seed_bound(-1.0)
    ctx.safeguard_debug_flags(0)
    ctx.profile(0)


@pytest.fixture(scope="module")
def shared_ctx(gpu_ctx):
    """The session context with a fresh context's settings, put back to them when the module ends, whether its tests passed or not."""
    _start_state(gpu_ctx)
    yield gpu_ctx
    _start_state(gpu_ctx)
