"""ctypes binding of the C ABI in include/ipcgpu.h (libipcgpu.so).

The product path has NO CPU fallback: if the CUDA library is missing or no GPU is visible, construction
fails loudly.  torch is used nowhere here; device memory is owned by the context behind the C ABI.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libipcgpu.so")

ERR_NAMES = {0: "OK", 1: "CUDA", 2: "ARG", 3: "PATTERN", 4: "NONPOSITIVE_DISTANCE", 5: "CAPACITY", 6: "NCCL", 7: "STATE", 8: "LINE_SEARCH", 9: "SOLVE"}
ERR_NONPOSITIVE_DISTANCE, ERR_STATE, ERR_LINE_SEARCH, ERR_SOLVE = 4, 7, 8, 9

BUF_GRADIENT, BUF_CSR_VALUES, BUF_ENERGY_PER_TET, BUF_TET_HESSIANS, BUF_TET_GRADIENTS, BUF_INVERSION_STEPS = range(6)
BUF_CSR_ROW_STARTS, BUF_CSR_COLUMNS = 6, 7  # ipcgpu_device_ptr only
BUF_POSITIONS, BUF_SEARCH_DIR, BUF_XTILDE = 8, 9, 10
BUF_MULTILEVEL_INVERSES = 11

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_u8p = C.POINTER(C.c_uint8)
_ctxp = C.c_void_p

# name -> (restype, argtypes); tests check that every symbol of include/ipcgpu.h is exported
SIGNATURES = {
    "ipcgpu_create": (C.c_int, [C.c_int, C.POINTER(_ctxp)]),
    "ipcgpu_destroy": (None, [_ctxp]),
    "ipcgpu_last_error": (C.c_char_p, [_ctxp]),
    "ipcgpu_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint64]),
    "ipcgpu_host_free": (C.c_int, [C.c_void_p]),
    "ipcgpu_sync": (C.c_int, [_ctxp]),
    "ipcgpu_launch_count": (C.c_uint64, [_ctxp]),
    "ipcgpu_comm_unique_id": (C.c_int, [C.c_void_p]),
    "ipcgpu_comm_init": (C.c_int, [_ctxp, C.c_int, C.c_int, C.c_void_p]),
    "ipcgpu_partition_info": (C.c_int, [_ctxp, _ip, _ip, _ip, _ip, _ip, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _ip]),
    "ipcgpu_fetch_iteration": (C.c_int, [_ctxp, C.c_void_p]),
    "ipcgpu_step_bound_set": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_check_inversion": (C.c_int, [_ctxp, _ip]),
    "ipcgpu_intersection_free": (C.c_int, [_ctxp, _ip]),
    "ipcgpu_safeguard_debug_flags": (C.c_int, [_ctxp, C.c_int, _ip, _ip]),
    "ipcgpu_constraint_set_sizes": (C.c_int, [_ctxp, _ip, _ip, _ip]),
    "ipcgpu_ccd_debug_seed_bound": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_ccd_debug_thread_budget": (C.c_int, [_ctxp, C.c_int64]),
    "ipcgpu_download_range": (C.c_int, [_ctxp, C.c_int, C.c_uint64, C.c_uint64, _dp]),
    "ipcgpu_download_range_async": (C.c_int, [_ctxp, C.c_int, C.c_uint64, C.c_uint64, _dp]),
    "ipcgpu_set_mesh": (C.c_int, [_ctxp, C.c_int, C.c_int, _dp, _ip, _dp, _dp, _dp, _dp, _dp, _u8p, C.c_int]),
    "ipcgpu_set_csr": (C.c_int, [_ctxp, C.c_int, _ip, _ip, C.c_int]),
    "ipcgpu_enable_device_pattern": (C.c_int, [_ctxp, C.c_int, C.c_uint64]),
    "ipcgpu_update_pattern": (C.c_int, [_ctxp, C.c_int, _ip, C.POINTER(C.c_int64)]),
    "ipcgpu_pattern_info": (C.c_int, [_ctxp, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
    "ipcgpu_get_pattern": (C.c_int, [_ctxp, _ip, _ip]),
    "ipcgpu_set_state": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_save_state": (C.c_int, [_ctxp]),
    "ipcgpu_set_search_dir": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_step_forward": (C.c_int, [_ctxp, _dp, C.c_double]),
    "ipcgpu_elastic_energy": (C.c_int, [_ctxp, C.c_double, C.c_int, _dp]),
    "ipcgpu_elastic_gradient": (C.c_int, [_ctxp, C.c_double, C.c_int, C.c_int, _dp]),
    "ipcgpu_elastic_hessian": (C.c_int, [_ctxp, C.c_double, C.c_int, C.c_int, C.c_int, _dp]),
    "ipcgpu_elastic_grad_hess": (C.c_int, [_ctxp, C.c_double, C.c_int, C.c_int, C.c_int, _dp, _dp]),
    "ipcgpu_elastic_energy_grad_hess": (C.c_int, [_ctxp, C.c_double, C.c_int, C.c_int, C.c_int, _dp, _dp, _dp]),
    "ipcgpu_inversion_step": (C.c_int, [_ctxp, _dp, C.c_double, _dp]),
    "ipcgpu_set_surface": (C.c_int, [_ctxp, C.c_int, _ip, C.c_int, _ip, C.c_int, _ip, _ip]),
    "ipcgpu_set_pair_capacity": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_set_exchange_capacity": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_constraint_set": (C.c_int, [_ctxp, C.c_double, C.c_int, _ip, _ip, _ip]),
    "ipcgpu_set_contact_partition": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_set_canonical_order": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_get_constraint_set": (C.c_int, [_ctxp, _ip, _ip, _ip, _ip]),
    "ipcgpu_set_constraint_set": (C.c_int, [_ctxp, C.c_int, _ip, C.c_int, _ip, _ip, C.c_int, _ip]),
    "ipcgpu_barrier_energy": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_barrier_gradient": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_barrier_hessian": (C.c_int, [_ctxp, C.c_double, C.c_double, C.c_int, _dp]),
    "ipcgpu_evaluate_constraints": (C.c_int, [_ctxp, _dp, C.c_int]),
    "ipcgpu_constraint_jacobian_t": (C.c_int, [_ctxp, _dp, C.c_int, C.c_double, _dp]),
    "ipcgpu_para_ee_gradient": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_set_ccd_capacity": (C.c_int, [_ctxp, C.c_uint64]),
    "ipcgpu_ti_error": (C.c_int, [_dp, C.c_int, _dp, _dp, _dp]),
    "ipcgpu_ccd_partial_ti": (C.c_int, [_ctxp, _dp, C.c_double, _dp, _dp, _dp]),
    "ipcgpu_hash_build_swept": (C.c_int, [_ctxp, _dp, _dp, C.c_double]),
    "ipcgpu_ccd_full_ti": (C.c_int, [_ctxp, C.c_double, _dp, _dp, _dp, C.POINTER(C.c_uint64)]),
    "ipcgpu_ccd_stats": (C.c_int, [_ctxp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "ipcgpu_ccd_stats_ex": (C.c_int, [_ctxp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "ipcgpu_ccd_stats_timing": (C.c_int, [_ctxp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "ipcgpu_set_obstacle_tail": (C.c_int, [_ctxp, C.c_int, C.c_int]),
    "ipcgpu_set_obstacle_positions": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_set_prev_state": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_friction_lag": (C.c_int, [_ctxp, C.c_double, C.c_double, _ip]),
    "ipcgpu_get_friction_data": (C.c_int, [_ctxp, _ip, _ip, _dp, _dp, _dp]),
    "ipcgpu_set_friction_data": (C.c_int, [_ctxp, C.c_int, _ip, _dp, _dp, _dp]),
    "ipcgpu_friction_energy": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_friction_gradient": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_friction_hessian": (C.c_int, [_ctxp, C.c_double, C.c_double, C.c_int, _dp]),
    "ipcgpu_set_xtilde": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_inertia_energy": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_inertia_gradient": (C.c_int, [_ctxp, C.c_int, _dp]),
    "ipcgpu_capture_begin": (C.c_int, [_ctxp]),
    "ipcgpu_capture_end": (C.c_int, [_ctxp, _ip]),
    "ipcgpu_graph_launch": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_graph_destroy": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_graph_kernel_priorities": (C.c_int, [_ctxp, C.c_int, _ip, _ip]),
    "ipcgpu_csr_set_zero": (C.c_int, [_ctxp]),
    "ipcgpu_solve_pcg": (C.c_int, [_ctxp, _dp, C.c_double, C.c_int, _dp, C.c_int, _ip, _dp]),
    "ipcgpu_solve_pcg_multilevel": (C.c_int, [_ctxp, _dp, C.c_double, C.c_int, _dp, C.c_int, _ip, _dp]),
    "ipcgpu_solve_info": (C.c_int, [_ctxp, C.c_void_p]),
    "ipcgpu_precondition_diag": (C.c_int, [_ctxp, C.c_int, _dp, C.c_int]),
    "ipcgpu_multilevel_info": (C.c_int, [_ctxp, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
    "ipcgpu_multilevel_debug_matrices": (C.c_int, [_ctxp, _dp, C.c_uint64]),
    "ipcgpu_solve_pcg_amg": (C.c_int, [_ctxp, _dp, C.c_double, C.c_int, _dp, C.c_int, _ip, _dp]),
    "ipcgpu_amg_info": (C.c_int, [_ctxp, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _dp, _dp, C.POINTER(C.c_uint64)]),
    "ipcgpu_amg_debug_level": (C.c_int, [_ctxp, C.c_int, _ip, _ip, _ip, _dp]),
    "ipcgpu_amg_reserve": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_amg_capacity_info": (C.c_int, [_ctxp, _ip, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "ipcgpu_amg_debug_coarse_enough": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_allreduce_grad_hess": (C.c_int, [_ctxp, C.c_int, C.c_int]),
    "ipcgpu_download": (C.c_int, [_ctxp, C.c_int, _dp, C.c_uint64]),
    "ipcgpu_device_ptr": (C.c_void_p, [_ctxp, C.c_int]),
    "ipcgpu_profile": (C.c_int, [_ctxp, C.c_int]),
    "ipcgpu_profile_read": (C.c_int, [_ctxp, C.c_int, _dp, _ip]),
    "ipcgpu_timer_start": (C.c_int, [_ctxp]),
    "ipcgpu_timer_stop": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_ccd_cfl_ti": (C.c_int, [_ctxp, C.c_double, C.c_int, C.c_double, C.c_double, _dp, _dp, _dp]),
    "ipcgpu_line_search": (C.c_int, [_ctxp, C.c_void_p, _dp]),
    "ipcgpu_step_control_info": (C.c_int, [_ctxp, C.c_void_p]),
    "ipcgpu_set_halfspaces": (C.c_int, [_ctxp, C.c_int, _dp, _dp, _dp, _dp]),
    "ipcgpu_halfspace_constraint_set": (C.c_int, [_ctxp, C.c_double, _ip]),
    "ipcgpu_halfspace_energy": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_halfspace_gradient": (C.c_int, [_ctxp, C.c_double, C.c_double, _dp]),
    "ipcgpu_halfspace_hessian": (C.c_int, [_ctxp, C.c_double, C.c_double, C.c_int, _dp]),
    "ipcgpu_halfspace_step": (C.c_int, [_ctxp, _dp, C.c_double, _dp]),
    "ipcgpu_halfspace_crossings": (C.c_int, [_ctxp, _ip]),
    "ipcgpu_halfspace_friction_lag": (C.c_int, [_ctxp, C.c_double, C.c_double, _ip]),
    "ipcgpu_halfspace_friction_energy": (C.c_int, [_ctxp, C.c_double, _dp]),
    "ipcgpu_halfspace_friction_gradient": (C.c_int, [_ctxp, C.c_double, _dp]),
    "ipcgpu_halfspace_friction_hessian": (C.c_int, [_ctxp, C.c_double, C.c_int, _dp]),
    "ipcgpu_get_halfspace_sets": (C.c_int, [_ctxp, _ip, _ip, _ip, _ip, _dp]),
    "ipcgpu_damping_update": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_damping_energy": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_damping_gradient": (C.c_int, [_ctxp, C.c_int, _dp]),
    "ipcgpu_damping_hessian": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_set_neumann_forces": (C.c_int, [_ctxp, C.c_double, _dp]),
    "ipcgpu_neumann_energy": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_neumann_gradient": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_set_dirichlet_targets": (C.c_int, [_ctxp, C.c_int, _ip, _dp, _dp, C.c_double]),
    "ipcgpu_set_dirichlet_penalty": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_get_dirichlet_lambda": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_dirichlet_energy": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_dirichlet_gradient": (C.c_int, [_ctxp, C.c_int, _dp]),
    "ipcgpu_dirichlet_hessian": (C.c_int, [_ctxp, C.c_int, _dp]),
    "ipcgpu_dirichlet_update_lambda": (C.c_int, [_ctxp]),
    "ipcgpu_dirichlet_completed_step": (C.c_int, [_ctxp, _dp]),
    "ipcgpu_set_time_integration": (C.c_int, [_ctxp, C.c_int, C.c_double, C.c_double, C.c_double, _dp]),
    "ipcgpu_set_dynamics": (C.c_int, [_ctxp, _dp, _dp, _dp]),
    "ipcgpu_get_dynamics": (C.c_int, [_ctxp, _dp, _dp, _dp]),
    "ipcgpu_compute_xtilde": (C.c_int, [_ctxp]),
    "ipcgpu_end_time_step": (C.c_int, [_ctxp]),
    "ipcgpu_warm_start": (C.c_int, [_ctxp, C.c_int, C.c_double, C.c_double, _dp, _dp, _dp]),
    "ipcgpu_kappa_bounds": (C.c_int, [C.c_double, C.c_double, C.c_double, C.c_double, _dp, _dp]),
    "ipcgpu_set_kappa": (C.c_int, [_ctxp, C.c_double, C.c_double, C.c_double]),
    "ipcgpu_kappa_init": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_kappa_clear_close_set": (C.c_int, [_ctxp]),
    "ipcgpu_kappa_post_line_search": (C.c_int, [_ctxp, C.c_double]),
    "ipcgpu_kappa_info": (C.c_int, [_ctxp, C.c_void_p]),
    "ipcgpu_set_components": (C.c_int, [_ctxp, C.c_int, _ip, _ip]),
    "ipcgpu_system_energy": (C.c_int, [_ctxp, _dp, _dp, _dp]),
    "ipcgpu_get_system_energy": (C.c_int, [_ctxp, _dp, _dp, _dp]),
    "ipcgpu_constraint_summary": (C.c_int, [_ctxp, C.c_double, C.c_double, C.c_void_p]),
    "ipcgpu_get_constraint_summary": (C.c_int, [_ctxp, C.c_void_p]),
}
# IPCGPU_KAPPA_DEVICE: as a kappa argument, the barrier stiffness held in device memory (Context.set_kappa)
KAPPA_DEVICE = -1.0
TIT_BE, TIT_NM = 0, 1

STAGES = ["elastic_energy", "elastic_tet", "gather_gradient", "assemble_csr", "inversion", "hash", "constraint_set", "barrier",
          "ccd_broad", "ccd_narrow", "allreduce", "ccd_root_filter", "damping_bc"]

_lib = None


class Iteration(C.Structure):
    """ipcgpu_iteration (include/ipcgpu.h)"""
    _fields_ = [("energy_elastic", C.c_double), ("energy_barrier", C.c_double), ("alpha_inversion", C.c_double), ("alpha_partial_ccd", C.c_double),
                ("alpha_swept_grid", C.c_double), ("alpha_full_ccd", C.c_double), ("alpha", C.c_double), ("n_active", C.c_int), ("n_mollified", C.c_int),
                ("n_candidates", C.c_int), ("status", C.c_int), ("n_full_ccd_candidates", C.c_uint64), ("ti_warnings", C.c_uint64),
                ("n_inverted_tets", C.c_int), ("n_intersected_triangles", C.c_int), ("energy_friction", C.c_double), ("energy_inertia", C.c_double),
                ("energy_halfspace", C.c_double), ("energy_halfspace_friction", C.c_double), ("alpha_halfspace", C.c_double),
                ("n_halfspace_active", C.c_int), ("n_halfspace_crossings", C.c_int), ("energy_damping", C.c_double), ("energy_neumann", C.c_double),
                ("energy_dirichlet", C.c_double), ("dirichlet_completed_step", C.c_double)]


class LineSearchTerms(C.Structure):
    """ipcgpu_line_search_terms (include/ipcgpu.h)"""
    _fields_ = [("elastic_coef", C.c_double), ("inertia", C.c_int), ("dHat", C.c_double), ("kappa", C.c_double), ("fric_eps2", C.c_double),
                ("fric_coef", C.c_double)]


class StepControl(C.Structure):
    """ipcgpu_step_control (include/ipcgpu.h)"""
    _fields_ = [("alpha_cfl", C.c_double), ("alpha_feasible", C.c_double), ("alpha", C.c_double), ("energy_start", C.c_double), ("energy", C.c_double),
                ("full_ccd", C.c_int), ("stopped", C.c_int), ("halvings_inversion", C.c_int), ("halvings_intersection", C.c_int),
                ("halvings_armijo", C.c_int), ("halvings_post_check", C.c_int), ("post_check_rebuilt", C.c_int), ("status", C.c_int)]


class KappaInfo(C.Structure):
    """ipcgpu_kappa (include/ipcgpu.h)"""
    _fields_ = [("kappa", C.c_double), ("min_kappa", C.c_double), ("suggest", C.c_double), ("max", C.c_double), ("close_min_dist2", C.c_double),
                ("doublings", C.c_int), ("n_close", C.c_int), ("needs_init", C.c_int)]


class ConstraintSummary(C.Structure):
    """ipcgpu_constraint_summary_result (include/ipcgpu.h)"""
    _fields_ = [("n", C.c_int), ("d_min", C.c_double), ("d_max", C.c_double), ("fb_norm", C.c_double)]


class SolveResult(C.Structure):
    """ipcgpu_solve_result (include/ipcgpu.h)"""
    _fields_ = [("iterations", C.c_int), ("rel_residual", C.c_double), ("max_abs_x", C.c_double), ("status", C.c_int)]


class IpcGpuError(RuntimeError):
    pass


def load():
    """Load libipcgpu.so and declare signatures. Raises if the library is missing (never falls back)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise IpcGpuError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a)")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(_ip)


def f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


class PinnedArray:
    """numpy view over cudaMallocHost memory (so D2H/H2D of the big arrays runs at PCIe speed)."""

    def __init__(self, n, dtype=np.float64):
        lib = load()
        self._ptr = C.c_void_p()
        nbytes = int(n) * np.dtype(dtype).itemsize
        rc = lib.ipcgpu_host_alloc(C.byref(self._ptr), max(nbytes, 8))
        if rc:
            raise IpcGpuError("ipcgpu_host_alloc failed")
        buf = (C.c_char * max(nbytes, 8)).from_address(self._ptr.value)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(n))

    def free(self):
        if self._ptr:
            load().ipcgpu_host_free(self._ptr)
            self._ptr = None


class Context:
    """Thin OO wrapper: one context per process per GPU."""

    def __init__(self, device=0):
        self.lib = load()
        self.h = _ctxp()
        rc = self.lib.ipcgpu_create(int(device), C.byref(self.h))
        if rc:
            raise IpcGpuError(f"ipcgpu_create(device={device}) failed with {ERR_NAMES.get(rc, rc)}: a CUDA device is required (no CPU fallback)")
        self.nV = self.nT = self.nnz = 0
        self.n_components = 0
        self._keep = []

    def close(self):
        if self.h:
            self.lib.ipcgpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            msg = self.lib.ipcgpu_last_error(self.h)
            raise IpcGpuError(f"{ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")

    # ---- scene --------------------------------------------------------------------------------
    def comm_init(self, rank, nranks, unique_id):
        buf = (C.c_char * 128).from_buffer_copy(bytes(unique_id)) if unique_id is not None else None
        self._ck(self.lib.ipcgpu_comm_init(self.h, rank, nranks, buf))

    @staticmethod
    def comm_unique_id():
        buf = (C.c_char * 128)()
        rc = load().ipcgpu_comm_unique_id(buf)
        if rc:
            raise IpcGpuError("ipcgpu_comm_unique_id failed")
        return bytes(buf)

    def set_mesh(self, Vrest_soa, tets_soa, restTriInv, vol, mu, lam, mass=None, dbc=None, energy=0):
        Vr, T = f64(Vrest_soa).ravel(), i32(tets_soa).ravel()
        self.nV, self.nT = Vr.size // 3, T.size // 4
        A, vol, mu, lam, mass = f64(restTriInv).ravel(), f64(vol), f64(mu), f64(lam), f64(mass)
        dbc = None if dbc is None else np.ascontiguousarray(dbc, dtype=np.uint8)
        self._ck(self.lib.ipcgpu_set_mesh(self.h, self.nV, self.nT, _d(Vr), _i(T), _d(A), _d(vol), _d(mu), _d(lam), _d(mass),
                                          None if dbc is None else dbc.ctypes.data_as(_u8p), int(energy)))

    def set_csr(self, ia, ja, index_base):
        ia, ja = i32(ia), i32(ja)
        self.nnz = int(ia[-1]) - index_base
        self._ck(self.lib.ipcgpu_set_csr(self.h, ia.size - 1, _i(ia), _i(ja), index_base))

    def enable_device_pattern(self, index_base=1, nnz_capacity=0):
        """the device builds the sparsity pattern from here on (mesh part now, contact part at every update_pattern)"""
        self._ck(self.lib.ipcgpu_enable_device_pattern(self.h, int(index_base), int(nnz_capacity)))
        self.nnz = self.pattern_info()[1]

    def update_pattern(self, with_friction=0, want=True):
        """want=True: (changed, nnz) after one synchronisation; want=False: enqueued only (read it with fetch_iteration / pattern_info)"""
        if not want:
            self._ck(self.lib.ipcgpu_update_pattern(self.h, int(with_friction), None, None))
            return None
        ch, n = C.c_int(), C.c_int64()
        self._ck(self.lib.ipcgpu_update_pattern(self.h, int(with_friction), C.byref(ch), C.byref(n)))
        self.nnz = n.value
        return ch.value, n.value

    def pattern_info(self):
        """(changed, nnz, version) of the last pattern update"""
        ch, n, ver = C.c_int(), C.c_int64(), C.c_uint64()
        self._ck(self.lib.ipcgpu_pattern_info(self.h, C.byref(ch), C.byref(n), C.byref(ver)))
        self.nnz = n.value
        return ch.value, n.value, ver.value

    def get_pattern(self):
        """(ia, ja) of the current pattern"""
        nnz = self.pattern_info()[1]
        ia, ja = np.empty(3 * self.nV + 1, np.int32), np.empty(max(nnz, 1), np.int32)
        self._ck(self.lib.ipcgpu_get_pattern(self.h, _i(ia), _i(ja)))
        return ia, ja[:nnz]

    def device_ptr(self, which):
        return self.lib.ipcgpu_device_ptr(self.h, int(which))

    def set_state(self, V_soa):
        self._ck(self.lib.ipcgpu_set_state(self.h, _d(f64(V_soa).ravel()) if V_soa is not None else None))

    def save_state(self):
        self._ck(self.lib.ipcgpu_save_state(self.h))

    def set_search_dir(self, p):
        self._ck(self.lib.ipcgpu_set_search_dir(self.h, _d(f64(p))))

    def step_forward(self, p, alpha):
        self._ck(self.lib.ipcgpu_step_forward(self.h, _d(f64(p)) if p is not None else None, float(alpha)))

    def sync(self):
        self._ck(self.lib.ipcgpu_sync(self.h))

    def launch_count(self):
        return int(self.lib.ipcgpu_launch_count(self.h))

    # ---- elastic ------------------------------------------------------------------------------
    def elastic_energy(self, coef, redoSVD=1, want=True):
        E = C.c_double(0.0)
        self._ck(self.lib.ipcgpu_elastic_energy(self.h, coef, redoSVD, C.byref(E) if want else None))
        return E.value

    def elastic_gradient(self, coef, redoSVD=1, projectDBC=1, out=None, want=True):
        if want and out is None:
            out = np.empty(3 * self.nV)
        self._ck(self.lib.ipcgpu_elastic_gradient(self.h, coef, redoSVD, projectDBC, _d(out) if want else None))
        return out

    def elastic_hessian(self, coef, redoSVD=1, projectSPD=1, projectDBC=1, a_inout=None):
        self._ck(self.lib.ipcgpu_elastic_hessian(self.h, coef, redoSVD, projectSPD, projectDBC, _d(a_inout)))
        return a_inout

    def elastic_grad_hess(self, coef, projectSPD=1, projectDBC=1, add_mass=0, g=None, a=None):
        self._ck(self.lib.ipcgpu_elastic_grad_hess(self.h, coef, projectSPD, projectDBC, add_mass, _d(g), _d(a)))

    def elastic_energy_grad_hess(self, coef, projectSPD=1, projectDBC=1, add_mass=0, g=None, a=None, want_energy=False):
        """fused computeEnergyVal + computeGradient + computePrecondMtr (one SVD per tet); returns E when want_energy"""
        E = C.c_double()
        self._ck(self.lib.ipcgpu_elastic_energy_grad_hess(self.h, coef, projectSPD, projectDBC, add_mass, C.byref(E) if want_energy else None, _d(g), _d(a)))
        return E.value if want_energy else None

    def inversion_step(self, p, slack, alpha):
        """alpha=None: chained on the device (no synchronisation)"""
        a = C.c_double(alpha if alpha is not None else 0.0)
        self._ck(self.lib.ipcgpu_inversion_step(self.h, _d(f64(p)) if p is not None else None, slack, C.byref(a) if alpha is not None else None))
        return a.value if alpha is not None else None

    def check_inversion(self, want=True):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_check_inversion(self.h, C.byref(n) if want else None))
        return n.value if want else None

    def intersection_free(self, want=True):
        """checkEdgeTriIntersectionIfAny: no surface edge crosses a surface triangle and no codimension-0 vertex (vCoDim == 0) lies in a
        tetrahedron (faces included).  want=False: deferred, the count comes back with fetch_iteration (n_intersected_triangles)."""
        ok = C.c_int()
        self._ck(self.lib.ipcgpu_intersection_free(self.h, C.byref(ok) if want else None))
        return bool(ok.value) if want else None

    def safeguard_debug_flags(self, enable, read=False):
        """test hook: enable the per-triangle flags / per-tet point counts of the intersection check; read=True returns the last check's
        (tri_flags[nSF], tet_hits[nT]) before applying `enable`"""
        out = (np.zeros(max(self.nSF, 1), np.int32), np.zeros(max(self.nT, 1), np.int32)) if read else (None, None)
        self._ck(self.lib.ipcgpu_safeguard_debug_flags(self.h, int(enable), *(None if x is None else _i(x) for x in out)))
        return (out[0][: self.nSF], out[1][: self.nT]) if read else None

    def step_bound_set(self, alpha):
        self._ck(self.lib.ipcgpu_step_bound_set(self.h, float(alpha)))

    def fetch_iteration(self):
        it = Iteration()
        self._ck(self.lib.ipcgpu_fetch_iteration(self.h, C.byref(it)))
        return it

    def partition_info(self):
        v = [C.c_int() for _ in range(6)]
        a0, a1, nl = C.c_int64(), C.c_int64(), C.c_int()
        self._ck(self.lib.ipcgpu_partition_info(self.h, *[C.byref(x) for x in v], C.byref(a0), C.byref(a1), C.byref(nl)))
        return dict(rank=v[0].value, nranks=v[1].value, tet_begin=v[2].value, tet_end=v[3].value, row_vertex_begin=v[4].value, row_vertex_end=v[5].value,
                    value_begin=a0.value, value_end=a1.value, n_assembled_tets=nl.value)

    def ccd_debug_seed_bound(self, toi):
        self._ck(self.lib.ipcgpu_ccd_debug_seed_bound(self.h, float(toi)))

    def ccd_debug_thread_budget(self, boxes):
        self._ck(self.lib.ipcgpu_ccd_debug_thread_budget(self.h, int(boxes)))

    def constraint_set_sizes(self):
        nC, nP, nK = C.c_int(), C.c_int(), C.c_int()
        self._ck(self.lib.ipcgpu_constraint_set_sizes(self.h, C.byref(nC), C.byref(nP), C.byref(nK)))
        return nC.value, nP.value, nK.value

    def download_range_async(self, which, offset, out):
        """out: a PinnedArray view; valid after the next fetch_iteration() / sync()"""
        self._ck(self.lib.ipcgpu_download_range_async(self.h, which, int(offset), int(out.size), _d(out)))

    def download_range_into(self, which, offset, out):
        self._ck(self.lib.ipcgpu_download_range(self.h, which, int(offset), int(out.size), _d(out)))

    # ---- CUDA graphs of device-resident call sequences -----------------------------------------
    def capture_begin(self):
        self._ck(self.lib.ipcgpu_capture_begin(self.h))

    def capture_end(self):
        gid = C.c_int(-1)
        self._ck(self.lib.ipcgpu_capture_end(self.h, C.byref(gid)))
        return gid.value

    def graph_launch(self, gid):
        self._ck(self.lib.ipcgpu_graph_launch(self.h, int(gid)))

    def graph_destroy(self, gid):
        self._ck(self.lib.ipcgpu_graph_destroy(self.h, int(gid)))

    def graph_kernel_priorities(self, gid):
        """(kernel nodes at the high stream priority, kernel nodes at the low one) of a captured graph"""
        a, b = C.c_int(), C.c_int()
        self._ck(self.lib.ipcgpu_graph_kernel_priorities(self.h, int(gid), C.byref(a), C.byref(b)))
        return a.value, b.value

    # ---- friction / inertia -------------------------------------------------------------------
    def set_prev_state(self, V_prev_soa=None):
        self._ck(self.lib.ipcgpu_set_prev_state(self.h, _d(f64(V_prev_soa).ravel()) if V_prev_soa is not None else None))

    def friction_lag(self, dHat, kappa, want=True):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_friction_lag(self.h, dHat, kappa, C.byref(n) if want else None))
        return n.value if want else None

    def get_friction_data(self):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_get_friction_data(self.h, C.byref(n), None, None, None, None))
        k = max(n.value, 1)
        mm, lam, co, ba = np.empty((k, 4), np.int32), np.empty(k), np.empty((k, 2)), np.empty((k, 6))
        self._ck(self.lib.ipcgpu_get_friction_data(self.h, C.byref(n), _i(mm), _d(lam), _d(co), _d(ba)))
        return mm[:n.value], lam[:n.value], co[:n.value], ba[:n.value]

    def set_friction_data(self, mm, lam, co, ba):
        mm, lam, co, ba = i32(mm), f64(lam), f64(co), f64(ba)
        self._ck(self.lib.ipcgpu_set_friction_data(self.h, len(mm), _i(mm), _d(lam), _d(co), _d(ba)))

    def friction_energy(self, eps2, coef, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_friction_energy(self.h, eps2, coef, C.byref(E) if want else None))
        return E.value if want else None

    def friction_gradient(self, eps2, coef, g_inout=None):
        self._ck(self.lib.ipcgpu_friction_gradient(self.h, eps2, coef, _d(g_inout)))
        return g_inout

    def friction_hessian(self, eps2, coef, projectDBC=1, a_inout=None):
        self._ck(self.lib.ipcgpu_friction_hessian(self.h, eps2, coef, projectDBC, _d(a_inout)))
        return a_inout

    def set_xtilde(self, xtilde_soa):
        self._ck(self.lib.ipcgpu_set_xtilde(self.h, _d(f64(xtilde_soa).ravel())))

    def inertia_energy(self, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_inertia_energy(self.h, C.byref(E) if want else None))
        return E.value if want else None

    def inertia_gradient(self, projectDBC=1, g_inout=None):
        self._ck(self.lib.ipcgpu_inertia_gradient(self.h, projectDBC, _d(g_inout)))
        return g_inout

    # ---- time integration (Optimizer::setTime / computeXTilta / end of a time step / initX) ------------------
    def set_time_integration(self, type, dt, beta=0.25, gamma=0.5, gravity=(0.0, -9.81, 0.0)):
        """type TIT_BE (0) or TIT_NM (1); the values live in device memory (a replayed graph reads the current ones)"""
        g = f64(np.asarray(gravity, dtype=np.float64).reshape(3))
        self._ck(self.lib.ipcgpu_set_time_integration(self.h, int(type), float(dt), float(beta), float(gamma), _d(g)))

    def set_dynamics(self, velocity=None, acceleration_soa=None, dx_elastic_soa=None):
        """velocity 3nV interleaved, acceleration and dx_Elastic nV x 3 SoA (3nV); None = zero"""
        v, a, dx = (None if x is None else f64(np.asarray(x, dtype=np.float64).ravel()) for x in (velocity, acceleration_soa, dx_elastic_soa))
        self._ck(self.lib.ipcgpu_set_dynamics(self.h, _d(v), _d(a), _d(dx)))

    def get_dynamics(self):
        """(velocity interleaved, acceleration SoA, dx_Elastic SoA), 3nV doubles each"""
        v, a, dx = np.empty(3 * self.nV), np.empty(3 * self.nV), np.empty(3 * self.nV)
        self._ck(self.lib.ipcgpu_get_dynamics(self.h, _d(v), _d(a), _d(dx)))
        return v, a, dx

    def compute_xtilde(self):
        self._ck(self.lib.ipcgpu_compute_xtilde(self.h))

    def end_time_step(self):
        self._ck(self.lib.ipcgpu_end_time_step(self.h))

    def warm_start(self, option, voxel_size, tol, err_vf, err_ee, want=True, check=True):
        """initX(option): want=True returns (status, accepted step) after one synchronisation (check=True raises on an error instead);
        want=False: deferred and capturable, returns the status of the enqueue"""
        a = C.c_double()
        evf, eee = (None if e is None else f64(e) for e in (err_vf, err_ee))
        rc = self.lib.ipcgpu_warm_start(self.h, int(option), float(voxel_size), float(tol), _d(evf), _d(eee), C.byref(a) if want else None)
        if check:
            self._ck(rc)
        return (rc, a.value) if want else rc

    # ---- half-space collision objects (HalfSpace<3>) -----------------------------------------------
    def set_halfspaces(self, origin, normal, velocitydt=None, friction=None):
        """up to 8 planes: origin, normal (n, 3), velocitydt (n, 3) or None, friction (n,); an empty list removes them"""
        o = f64(np.asarray(origin, dtype=np.float64).reshape(-1, 3))
        n = len(o)
        nr = f64(np.asarray(normal, dtype=np.float64).reshape(-1, 3))
        v = None if velocitydt is None else f64(np.asarray(velocitydt, dtype=np.float64).reshape(-1, 3))
        fr = f64(np.zeros(n) if friction is None else np.asarray(friction, dtype=np.float64).reshape(-1))
        self._ck(self.lib.ipcgpu_set_halfspaces(self.h, n, _d(o) if n else None, _d(nr) if n else None, _d(v) if n else None, _d(fr) if n else None))

    def halfspace_constraint_set(self, dHat, want=True):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_halfspace_constraint_set(self.h, float(dHat), C.byref(n) if want else None))
        return n.value if want else None

    def halfspace_energy(self, dHat, kappa, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_halfspace_energy(self.h, float(dHat), float(kappa), C.byref(E) if want else None))
        return E.value if want else None

    def halfspace_gradient(self, dHat, kappa, g_inout=None):
        self._ck(self.lib.ipcgpu_halfspace_gradient(self.h, float(dHat), float(kappa), _d(g_inout)))
        return g_inout

    def halfspace_hessian(self, dHat, kappa, projectDBC=1, a_inout=None):
        self._ck(self.lib.ipcgpu_halfspace_hessian(self.h, float(dHat), float(kappa), int(projectDBC), _d(a_inout)))
        return a_inout

    def halfspace_step(self, p, slackness, alpha):
        """alpha=None: the device-resident step (step-bound chain); p=None: the held search direction"""
        a = C.c_double(alpha if alpha is not None else 0.0)
        rc = self.lib.ipcgpu_halfspace_step(self.h, _d(f64(p)) if p is not None else None, float(slackness), C.byref(a) if alpha is not None else None)
        if rc != ERR_LINE_SEARCH:
            self._ck(rc)
        return (a.value if alpha is not None else None), rc

    def halfspace_crossings(self, want=True):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_halfspace_crossings(self.h, C.byref(n) if want else None))
        return n.value if want else None

    def halfspace_friction_lag(self, dHat, kappa, want=True):
        n = C.c_int()
        self._ck(self.lib.ipcgpu_halfspace_friction_lag(self.h, float(dHat), float(kappa), C.byref(n) if want else None))
        return n.value if want else None

    def halfspace_friction_energy(self, eps2, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_halfspace_friction_energy(self.h, float(eps2), C.byref(E) if want else None))
        return E.value if want else None

    def halfspace_friction_gradient(self, eps2, g_inout=None):
        self._ck(self.lib.ipcgpu_halfspace_friction_gradient(self.h, float(eps2), _d(g_inout)))
        return g_inout

    def halfspace_friction_hessian(self, eps2, projectDBC=1, a_inout=None):
        self._ck(self.lib.ipcgpu_halfspace_friction_hessian(self.h, float(eps2), int(projectDBC), _d(a_inout)))
        return a_inout

    def get_halfspace_sets(self):
        """(active (n, 2) [plane, vertex], lagged (m, 2), lambda (m,))"""
        na, nl = C.c_int(), C.c_int()
        self._ck(self.lib.ipcgpu_get_halfspace_sets(self.h, C.byref(na), None, C.byref(nl), None, None))
        act, lag, lam = np.empty((max(na.value, 1), 2), np.int32), np.empty((max(nl.value, 1), 2), np.int32), np.empty(max(nl.value, 1))
        self._ck(self.lib.ipcgpu_get_halfspace_sets(self.h, C.byref(na), _i(act), C.byref(nl), _i(lag), _d(lam)))
        return act[:na.value], lag[:nl.value], lam[:nl.value]

    # ---- damping, Neumann forces, Dirichlet penalty --------------------------------------------------
    def damping_update(self, coef):
        """computeDampingMtr at the current state (coef = energyParams[0] dampingStiff / dt); 0 removes the term"""
        self._ck(self.lib.ipcgpu_damping_update(self.h, float(coef)))

    def damping_energy(self, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_damping_energy(self.h, C.byref(E) if want else None))
        return E.value if want else None

    def damping_gradient(self, projectDBC=1, g_inout=None):
        self._ck(self.lib.ipcgpu_damping_gradient(self.h, int(projectDBC), _d(g_inout)))
        return g_inout

    def damping_hessian(self, a_inout=None):
        self._ck(self.lib.ipcgpu_damping_hessian(self.h, _d(a_inout)))
        return a_inout

    def set_neumann_forces(self, coef, f):
        """f: per-vertex summed force of the active NBCs (nV, 3) or None (removes the term); coef = dt^2"""
        f = None if f is None else f64(np.asarray(f, dtype=np.float64).reshape(-1))
        self._ck(self.lib.ipcgpu_set_neumann_forces(self.h, float(coef), _d(f)))

    def neumann_energy(self, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_neumann_energy(self.h, C.byref(E) if want else None))
        return E.value if want else None

    def neumann_gradient(self, g_inout=None):
        self._ck(self.lib.ipcgpu_neumann_gradient(self.h, _d(g_inout)))
        return g_inout

    def set_dirichlet_targets(self, vid, target, lam=None, dist2Tol=0.0):
        """targetPos: vertices (n,), target positions (n, 3), multipliers (n, 3) or None (0); an empty list removes the term"""
        vid = i32(np.asarray(vid).reshape(-1))
        n = int(vid.size)
        t = f64(np.asarray(target, dtype=np.float64).reshape(-1))
        lam = None if lam is None else f64(np.asarray(lam, dtype=np.float64).reshape(-1))
        self._ck(self.lib.ipcgpu_set_dirichlet_targets(self.h, n, _i(vid) if n else None, _d(t) if n else None, _d(lam) if n else None, float(dist2Tol)))
        self.n_dbc = n

    def set_dirichlet_penalty(self, rho):
        self._ck(self.lib.ipcgpu_set_dirichlet_penalty(self.h, float(rho)))

    def get_dirichlet_lambda(self):
        out = np.empty(3 * max(getattr(self, "n_dbc", 0), 1))
        self._ck(self.lib.ipcgpu_get_dirichlet_lambda(self.h, _d(out)))
        return out[:3 * getattr(self, "n_dbc", 0)].reshape(-1, 3)

    def dirichlet_energy(self, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_dirichlet_energy(self.h, C.byref(E) if want else None))
        return E.value if want else None

    def dirichlet_gradient(self, projectDBC=0, g_inout=None):
        self._ck(self.lib.ipcgpu_dirichlet_gradient(self.h, int(projectDBC), _d(g_inout)))
        return g_inout

    def dirichlet_hessian(self, projectDBC=0, a_inout=None):
        self._ck(self.lib.ipcgpu_dirichlet_hessian(self.h, int(projectDBC), _d(a_inout)))
        return a_inout

    def dirichlet_update_lambda(self):
        self._ck(self.lib.ipcgpu_dirichlet_update_lambda(self.h))

    def dirichlet_completed_step(self, want=True):
        s = C.c_double()
        self._ck(self.lib.ipcgpu_dirichlet_completed_step(self.h, C.byref(s) if want else None))
        return s.value if want else None

    # ---- contact ------------------------------------------------------------------------------
    def set_surface(self, SVI, SFEdges, SF_soa, vCoDim=None):
        SVI, SE, SF = i32(SVI).ravel(), i32(SFEdges).ravel(), i32(SF_soa).ravel()
        self.nSF = SF.size // 3
        self._ck(self.lib.ipcgpu_set_surface(self.h, SVI.size, _i(SVI), SE.size // 2, _i(SE), SF.size // 3, _i(SF), _i(i32(vCoDim))))

    def set_obstacle_tail(self, first_obstacle_vertex, ee_through_vf_routine=1):
        """MeshCO hand-off: vertices from first_obstacle_vertex on are a kinematic obstacle (ipc_b200/obstacle.py builds the merged arrays);
        a negative value removes the obstacle"""
        self._ck(self.lib.ipcgpu_set_obstacle_tail(self.h, int(first_obstacle_vertex), int(ee_through_vf_routine)))

    def set_obstacle_positions(self, Vo):
        """Vo: (nVo, 3) new positions of the obstacle's vertices (MeshCO::move)"""
        self._ck(self.lib.ipcgpu_set_obstacle_positions(self.h, _d(f64(np.ascontiguousarray(np.asarray(Vo, dtype=np.float64).T).ravel()))))

    def set_canonical_order(self, level):
        """0: contact lists in build order; 1 (default): sorted lexicographically (sorts sized on the device, also inside a capture);
        2: the reproducible mode -- the same order, and every contact sum (E, g, H) in an order fixed by the lists alone, so a captured
        time step gives the same bits on every run.  One rank only."""
        self._ck(self.lib.ipcgpu_set_canonical_order(self.h, int(level)))

    def set_contact_partition(self, enable):
        self._ck(self.lib.ipcgpu_set_contact_partition(self.h, int(enable)))

    def set_exchange_capacity(self, pairs_per_rank):
        self._ck(self.lib.ipcgpu_set_exchange_capacity(self.h, int(pairs_per_rank)))

    def set_pair_capacity(self, cap):
        self._ck(self.lib.ipcgpu_set_pair_capacity(self.h, int(cap)))

    def constraint_set(self, dHat, getPTEE=1, fetch=True, sizes=True):
        """fetch=True: returns the four lists; fetch=False, sizes=True: returns the sizes (one synchronisation);
        fetch=False, sizes=False: nothing is read back (device-resident iteration)"""
        if not fetch and not sizes:
            self._ck(self.lib.ipcgpu_constraint_set(self.h, dHat, getPTEE, None, None, None))
            return None
        nC, nP, nK = C.c_int(), C.c_int(), C.c_int()
        self._ck(self.lib.ipcgpu_constraint_set(self.h, dHat, getPTEE, C.byref(nC), C.byref(nP), C.byref(nK)))
        self.nC, self.nP, self.nK = nC.value, nP.value, nK.value
        if not fetch:
            return self.nC, self.nP, self.nK
        mm = np.empty((self.nC, 4), dtype=np.int32); pa = np.empty((self.nP, 4), dtype=np.int32)
        pe = np.empty((self.nP, 2), dtype=np.int32); cand = np.empty((self.nK, 2), dtype=np.int32)
        self._ck(self.lib.ipcgpu_get_constraint_set(self.h, _i(mm), _i(pa), _i(pe), _i(cand)))
        return mm, pa, pe, cand

    def set_constraint_set(self, mm, pa, pe, cand=None):
        mm, pa, pe = i32(mm), i32(pa), i32(pe)
        cand = i32(cand) if cand is not None else np.empty((0, 2), dtype=np.int32)
        self._ck(self.lib.ipcgpu_set_constraint_set(self.h, len(mm), _i(mm), len(pa), _i(pa), _i(pe), len(cand), _i(cand)))

    def barrier_energy(self, dHat, kappa, want=True):
        E = C.c_double()
        self._ck(self.lib.ipcgpu_barrier_energy(self.h, dHat, kappa, C.byref(E) if want else None))
        return E.value

    def barrier_gradient(self, dHat, kappa, g_inout=None):
        self._ck(self.lib.ipcgpu_barrier_gradient(self.h, dHat, kappa, _d(g_inout)))
        return g_inout

    def evaluate_constraints(self, n):
        val = np.empty(int(n))
        self._ck(self.lib.ipcgpu_evaluate_constraints(self.h, _d(val), int(n)))
        return val

    def constraint_jacobian_t(self, inp, coef, g_inout):
        inp = f64(inp)
        self._ck(self.lib.ipcgpu_constraint_jacobian_t(self.h, _d(inp), int(inp.size), float(coef), _d(g_inout)))
        return g_inout

    def para_ee_gradient(self, dHat, kappa, g_inout):
        self._ck(self.lib.ipcgpu_para_ee_gradient(self.h, dHat, kappa, _d(g_inout)))
        return g_inout

    def barrier_hessian(self, dHat, kappa, projectDBC=1, a_inout=None):
        self._ck(self.lib.ipcgpu_barrier_hessian(self.h, dHat, kappa, projectDBC, _d(a_inout)))
        return a_inout

    # ---- CCD ----------------------------------------------------------------------------------
    @staticmethod
    def ti_error(V_soa, nV, p=None):
        evf, eee = np.empty(3), np.empty(3)
        rc = load().ipcgpu_ti_error(_d(f64(V_soa).ravel()), int(nV), _d(f64(p)) if p is not None else None, _d(evf), _d(eee))
        if rc:
            raise IpcGpuError("ipcgpu_ti_error failed")
        return evf, eee

    def set_ccd_capacity(self, cap):
        self._ck(self.lib.ipcgpu_set_ccd_capacity(self.h, int(cap)))

    def ccd_partial(self, p, tol, err_vf, err_ee, alpha):
        """alpha=None (here and in the next two): chained on the device, nothing is read back"""
        a = C.c_double(alpha if alpha is not None else 0.0)
        self._ck(self.lib.ipcgpu_ccd_partial_ti(self.h, _d(f64(p)) if p is not None else None, tol, _d(f64(err_vf)), _d(f64(err_ee)),
                                                C.byref(a) if alpha is not None else None))
        return a.value if alpha is not None else None

    def ccd_cfl(self, dHat, first_iteration, voxel_size, tol, err_vf, err_ee, alpha):
        """CFL branch of the step bound (CFL_FOR_CCD == 2) after ccd_partial; alpha=None: the device-resident step"""
        a = C.c_double(alpha if alpha is not None else 0.0)
        self._ck(self.lib.ipcgpu_ccd_cfl_ti(self.h, float(dHat), int(first_iteration), float(voxel_size), float(tol), _d(f64(err_vf)), _d(f64(err_ee)),
                                            C.byref(a) if alpha is not None else None))
        return a.value if alpha is not None else None

    def line_search(self, elastic_coef, dHat, kappa, inertia=False, fric_eps2=0.0, fric_coef=0.0, alpha=None, check=True):
        """Optimizer::lineSearch (armijoParam = 0) along the held search direction; alpha=None: from / into the device-resident step.
        Returns the status code (check=True raises on an error instead)"""
        t = LineSearchTerms(float(elastic_coef), int(bool(inertia)), float(dHat), float(kappa), float(fric_eps2), float(fric_coef))
        a = C.c_double(alpha if alpha is not None else 0.0)
        rc = self.lib.ipcgpu_line_search(self.h, C.byref(t), C.byref(a) if alpha is not None else None)
        if check:
            self._ck(rc)
        return (rc, a.value) if alpha is not None else rc

    def step_control_info(self):
        """ipcgpu_step_control of the last CFL branch / line search (its status is out.status, not raised)"""
        out = StepControl()
        self.lib.ipcgpu_step_control_info(self.h, C.byref(out))
        return out

    # ---- adaptive barrier stiffness (kappa held on the device; pass KAPPA_DEVICE as the kappa of the barrier calls) --------------
    @staticmethod
    def kappa_bounds(dHat, kappa_min_multiplier, avg_node_mass, bbox_diag2):
        """(suggestKappa, upperBoundKappa's kappaMax); host-only"""
        s, m = C.c_double(), C.c_double()
        rc = load().ipcgpu_kappa_bounds(float(dHat), float(kappa_min_multiplier), float(avg_node_mass), float(bbox_diag2), C.byref(s), C.byref(m))
        if rc:
            raise IpcGpuError(f"ipcgpu_kappa_bounds failed with {ERR_NAMES.get(rc, rc)}")
        return s.value, m.value

    def set_kappa(self, kappa, suggest, kmax):
        self._ck(self.lib.ipcgpu_set_kappa(self.h, float(kappa), float(suggest), float(kmax)))

    def kappa_init(self, dHat):
        self._ck(self.lib.ipcgpu_kappa_init(self.h, float(dHat)))

    def kappa_clear_close_set(self):
        self._ck(self.lib.ipcgpu_kappa_clear_close_set(self.h))

    def kappa_post_line_search(self, dTol):
        self._ck(self.lib.ipcgpu_kappa_post_line_search(self.h, float(dTol)))

    def kappa_info(self):
        out = KappaInfo()
        self._ck(self.lib.ipcgpu_kappa_info(self.h, C.byref(out)))
        return out

    # ---- end-of-step diagnostics (computeSystemEnergy, the constraint summary after solveSub_IP) ----------------------------------
    def set_components(self, vertex_end, tet_end):
        """the cumulative compVAccSize / compFAccSize: one entry per component, in order"""
        ve, te = i32(np.asarray(vertex_end).ravel()), i32(np.asarray(tet_end).ravel())
        if ve.size != te.size:
            raise ValueError("vertex_end and tet_end must have one entry per component")
        self._ck(self.lib.ipcgpu_set_components(self.h, int(ve.size), _i(ve), _i(te)))
        self.n_components = int(ve.size)

    def _system_energy_arrays(self):
        n = self.n_components
        return np.empty(n), np.empty((n, 3)), np.empty((n, 3))

    def system_energy(self, want=True):
        """(sysE (n,), sysM (n, 3), sysL (n, 3)); want=False: deferred and capturable (get_system_energy reads it)"""
        if not want:
            self._ck(self.lib.ipcgpu_system_energy(self.h, None, None, None))
            return None
        E, Mo, Lo = self._system_energy_arrays()
        self._ck(self.lib.ipcgpu_system_energy(self.h, _d(E), _d(Mo), _d(Lo)))
        return E, Mo, Lo

    def get_system_energy(self):
        E, Mo, Lo = self._system_energy_arrays()
        self._ck(self.lib.ipcgpu_get_system_energy(self.h, _d(E), _d(Mo), _d(Lo)))
        return E, Mo, Lo

    def constraint_summary(self, dHat, kappa, want=True):
        """ConstraintSummary (n, d_min, d_max, fb_norm); want=False: deferred and capturable (get_constraint_summary reads it)"""
        out = ConstraintSummary()
        self._ck(self.lib.ipcgpu_constraint_summary(self.h, float(dHat), float(kappa), C.byref(out) if want else None))
        return out if want else None

    def get_constraint_summary(self):
        out = ConstraintSummary()
        self._ck(self.lib.ipcgpu_get_constraint_summary(self.h, C.byref(out)))
        return out

    def hash_build_swept(self, p, alpha, h):
        a = C.c_double(alpha if alpha is not None else 0.0)
        self._ck(self.lib.ipcgpu_hash_build_swept(self.h, _d(f64(p)) if p is not None else None, C.byref(a) if alpha is not None else None, h))
        return a.value if alpha is not None else None

    def ccd_full(self, tol, err_vf, err_ee, alpha):
        a = C.c_double(alpha if alpha is not None else 0.0)
        n = C.c_uint64()
        self._ck(self.lib.ipcgpu_ccd_full_ti(self.h, tol, _d(f64(err_vf)), _d(f64(err_ee)), C.byref(a) if alpha is not None else None,
                                             C.byref(n) if alpha is not None else None))
        return (a.value, n.value) if alpha is not None else None

    def ccd_stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._ck(self.lib.ipcgpu_ccd_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def ccd_stats_ex(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._ck(self.lib.ipcgpu_ccd_stats_ex(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def ccd_stats_timing(self):
        a, b = C.c_uint64(), C.c_uint64()
        self._ck(self.lib.ipcgpu_ccd_stats_timing(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def profile(self, enable):
        self._ck(self.lib.ipcgpu_profile(self.h, int(enable)))

    def profile_read(self):
        out = {}
        for k, name in enumerate(STAGES):
            ms, n = C.c_double(), C.c_int()
            self._ck(self.lib.ipcgpu_profile_read(self.h, k, C.byref(ms), C.byref(n)))
            if n.value:
                out[name] = (ms.value, n.value)
        return out

    def timer_start(self):
        self._ck(self.lib.ipcgpu_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_double()
        self._ck(self.lib.ipcgpu_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def allreduce_grad_hess(self, with_gradient=1, with_hessian=1):
        self._ck(self.lib.ipcgpu_allreduce_grad_hess(self.h, with_gradient, with_hessian))

    def _solve(self, fn, rhs, rel_tol, max_iter, want_x, adopt, deferred):
        if deferred:  # H x = -g on the device, capturable; the result comes from solve_info()
            if rhs is not None or want_x is True:
                raise ValueError("the deferred solve takes the resident gradient and leaves x on the device: rhs=None, want_x=False")
            self._ck(fn(self.h, None, rel_tol, int(max_iter), None, int(adopt), None, None))
            return None
        x = np.empty(3 * self.nV) if want_x else None
        it, res = C.c_int(), C.c_double()
        self._ck(fn(self.h, _d(f64(rhs)) if rhs is not None else None, rel_tol, int(max_iter), _d(x) if want_x else None, int(adopt), C.byref(it),
                    C.byref(res)))
        return x, it.value, res.value

    def solve_pcg(self, rhs=None, rel_tol=1e-8, max_iter=2000, want_x=True, adopt=False, deferred=False):
        """H x = rhs (None: -gradient, both device resident); returns (x or None, iterations, relative residual).  deferred=True (rhs=None,
        want_x=False): enqueued only, capturable; returns None, the result is solve_info()"""
        return self._solve(self.lib.ipcgpu_solve_pcg, rhs, rel_tol, max_iter, want_x, adopt, deferred)

    def solve_pcg_multilevel(self, rhs=None, rel_tol=1e-8, max_iter=2000, want_x=True, adopt=False, deferred=False):
        """solve_pcg with the multilevel additive Schwarz preconditioner (rebuilt from the resident matrix and positions at every call)"""
        return self._solve(self.lib.ipcgpu_solve_pcg_multilevel, rhs, rel_tol, max_iter, want_x, adopt, deferred)

    def precondition_diag(self, sign=-1, want_x=True, adopt=False):
        """(sign g_i) / a(i,i) over the resident gradient and CSR values; want_x=True returns it (3 nV), want_x=False is deferred and
        capturable and returns None.  Either way solve_info() reads max_abs_x and the status"""
        x = np.empty(3 * self.nV) if want_x else None
        self._ck(self.lib.ipcgpu_precondition_diag(self.h, int(sign), _d(x), int(adopt)))
        return x

    def solve_info(self):
        """ipcgpu_solve_result of the last solve (its status is out.status, not raised)"""
        out = SolveResult()
        self.lib.ipcgpu_solve_info(self.h, C.byref(out))
        return out

    def multilevel_info(self):
        """(domains per level, bytes of the stored inverses) of the last multilevel solve"""
        lv, dom, nb = C.c_int(), (C.c_int64 * 8)(), C.c_uint64()
        self._ck(self.lib.ipcgpu_multilevel_info(self.h, C.byref(lv), dom, C.byref(nb)))
        return list(dom[: lv.value]), nb.value

    def multilevel_debug_matrices(self):
        """test hook: the level matrices before inversion, one (domains, 96, 96) array per level; the stored inverses are lost"""
        domains, _ = self.multilevel_info()
        out = np.empty(9216 * sum(domains))
        self._ck(self.lib.ipcgpu_multilevel_debug_matrices(self.h, _d(out), out.size))
        return [a.reshape(-1, 96, 96) for a in np.split(out, np.cumsum([9216 * d for d in domains])[:-1])]

    def solve_pcg_amg(self, rhs=None, rel_tol=1e-8, max_iter=2000, want_x=True, adopt=False, deferred=False):
        """solve_pcg with the smoothed-aggregation multigrid preconditioner (linearSolver AMGCL, rebuilt from the resident matrix at every
        call; capturable in its deferred form after amg_reserve()).  want_x=False with rhs=None leaves the solution on the device; the
        result is also solve_info()"""
        return self._solve(self.lib.ipcgpu_solve_pcg_amg, rhs, rel_tol, max_iter, want_x, adopt, deferred)

    def amg_reserve(self, headroom=1.5):
        """size every AMG set-up buffer from the last hierarchy (headroom x its entry counts): the solve then runs inside a capture"""
        self._ck(self.lib.ipcgpu_amg_reserve(self.h, float(headroom)))

    def amg_capacity_info(self):
        """(cut_at_level, needed, reserved) of the last AMG set-up: needed / reserved are (6 levels, 5 counts) arrays"""
        cut, need, res = C.c_int(), (C.c_int64 * 30)(), (C.c_int64 * 30)()
        self._ck(self.lib.ipcgpu_amg_capacity_info(self.h, C.byref(cut), need, res))
        return cut.value, np.array(need[:]).reshape(6, 5), np.array(res[:]).reshape(6, 5)

    def amg_debug_coarse_enough(self, rows=1000):
        """test hook: a level with at most `rows` block rows is the last"""
        self._ck(self.lib.ipcgpu_amg_debug_coarse_enough(self.h, int(rows)))

    def amg_info(self):
        """dict of the last AMG hierarchy: rows, blocks, rho, omega (one entry per level) and bytes"""
        lv, rows, blocks = C.c_int(), (C.c_int64 * 6)(), (C.c_int64 * 6)()
        rho, omega, nb = (C.c_double * 6)(), (C.c_double * 6)(), C.c_uint64()
        self._ck(self.lib.ipcgpu_amg_info(self.h, C.byref(lv), rows, blocks, rho, omega, C.byref(nb)))
        n = lv.value
        return {"rows": list(rows[:n]), "blocks": list(blocks[:n]), "rho": list(rho[:n]), "omega": list(omega[:n]), "bytes": nb.value}

    def amg_debug_level(self, level):
        """test hook: (aggregate, ia, ja, blocks (nnzb, 3, 3)) of level `level` of the last AMG hierarchy"""
        info = self.amg_info()
        n, nb = info["rows"][level], info["blocks"][level]
        agg, ia = np.empty(n, dtype=np.int32), np.empty(n + 1, dtype=np.int32)
        ja, blk = np.empty(max(nb, 1), dtype=np.int32), np.empty(9 * max(nb, 1))
        self._ck(self.lib.ipcgpu_amg_debug_level(self.h, int(level), _i(agg), _i(ia), _i(ja), _d(blk)))
        return agg, ia, ja[:nb], blk[: 9 * nb].reshape(-1, 3, 3)

    def csr_set_zero(self):
        self._ck(self.lib.ipcgpu_csr_set_zero(self.h))

    def download_into(self, which, out):
        self._ck(self.lib.ipcgpu_download(self.h, which, _d(out), int(out.size)))

    def download(self, which, count):
        out = np.empty(int(count))
        self._ck(self.lib.ipcgpu_download(self.h, which, _d(out), int(count)))
        return out


def untile_hessians(raw, nT):
    """BUF_TET_HESSIANS is tile-major (64-tet tiles, slot-major inside a tile; csrc/elastic.cu). Returns the (nT, 78) per-tet view:
    4 diagonal blocks (6 upper scalars) then the 6 oriented off-diagonal 3x3 blocks."""
    out = np.empty((nT, 78))
    ntile = (nT + 63) // 64
    r = np.asarray(raw).reshape(ntile, 64 * 78)
    t = np.arange(nT)
    tile, tin = t // 64, t % 64
    for o, ln in [(0, 6), (6, 6), (12, 6), (18, 6)] + [(24 + 9 * q, 9) for q in range(6)]:
        for q in range(ln):
            out[:, o + q] = r[tile, o * 64 + tin * ln + q]
    return out
