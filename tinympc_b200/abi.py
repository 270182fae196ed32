"""ctypes mirror of include/tinympc_b200.h (POD structs only).

Kept byte-for-byte in sync with the header; tests/test_abi.py checks sizes/offsets against a C probe
and that the shared library exports every symbol the header declares.
"""
import ctypes as C

F32, F64 = 0, 1
MODE_STRICT, MODE_FAST = 0, 1
KERNEL_AUTO, KERNEL_TPI, KERNEL_GPI, KERNEL_GPS = 0, 1, 2, 4

OK = 0
ERR_ARG, ERR_UNSUPPORTED, ERR_CUDA, ERR_NO_BOUNDS, ERR_CONE_DIM, ERR_SINGULAR = -1, -2, -3, -4, -5, -6

vp = C.c_void_p
i32p = C.POINTER(C.c_int32)


class Problem(C.Structure):
    _fields_ = [
        ("nx", C.c_int32), ("nu", C.c_int32), ("N", C.c_int32), ("dtype", C.c_int32),
        ("rho", C.c_double),
        ("Adyn", vp), ("Bdyn", vp), ("fdyn", vp), ("Q", vp), ("R", vp),
        ("Kinf", vp), ("Pinf", vp), ("Quu_inv", vp), ("AmBKt", vp), ("APf", vp), ("BPf", vp),
        ("x_min", vp), ("x_max", vp), ("u_min", vp), ("u_max", vp),
        ("num_state_cones", C.c_int32), ("num_input_cones", C.c_int32),
        ("Acx", vp), ("qcx", vp), ("cx", vp), ("Acu", vp), ("qcu", vp), ("cu", vp),
        ("num_state_linear", C.c_int32), ("num_input_linear", C.c_int32),
        ("Alin_x", vp), ("blin_x", vp), ("Alin_u", vp), ("blin_u", vp),
        ("num_tv_state_linear", C.c_int32), ("num_tv_input_linear", C.c_int32),
        ("tv_Alin_x", vp), ("tv_blin_x", vp), ("tv_Alin_u", vp), ("tv_blin_u", vp),
    ]


class Settings(C.Structure):
    _fields_ = [
        ("abs_pri_tol", C.c_double), ("abs_dua_tol", C.c_double),
        ("max_iter", C.c_int32), ("check_termination", C.c_int32),
        ("en_state_bound", C.c_int32), ("en_input_bound", C.c_int32),
        ("en_state_soc", C.c_int32), ("en_input_soc", C.c_int32),
        ("en_state_linear", C.c_int32), ("en_input_linear", C.c_int32),
        ("en_tv_state_linear", C.c_int32), ("en_tv_input_linear", C.c_int32),
    ]


STATE_FIELDS = [
    "x", "u", "v", "z", "vnew", "znew", "g", "y",
    "vcnew", "zcnew", "gc", "yc",
    "vlnew", "zlnew", "gl", "yl",
    "vlnew_tv", "zlnew_tv", "gl_tv", "yl_tv",
]
# which state fields are state-shaped (nx x N); the others are input-shaped (nu x (N-1))
STATE_IS_X = {f: (f[0] in "xvg") for f in STATE_FIELDS}


class State(C.Structure):
    _fields_ = [(f, vp) for f in STATE_FIELDS]


class Batch(C.Structure):
    _fields_ = [
        ("B", C.c_int64),
        ("x0", vp),
        ("Xref", vp), ("xref_per_instance", C.c_int32),
        ("Uref", vp), ("uref_per_instance", C.c_int32),
        ("cold_start", C.c_int32),
        ("state", State),
        ("sol_x", vp), ("sol_u", vp),
        ("iter", vp), ("solved", vp), ("residuals", vp),
        ("u0", vp),
        ("models", vp),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("instances", C.c_int64), ("kernel_launches", C.c_int64),
        ("kernel_ms", C.c_float),
        ("kernel_family", C.c_int32), ("lanes_per_instance", C.c_int32),
        ("instances_per_cta", C.c_int32), ("smem_bytes_per_cta", C.c_int32),
        ("ctas", C.c_int32), ("threads_per_cta", C.c_int32),
        ("gpi_instances", C.c_int64),
        ("tmem_cols_per_cta", C.c_int32), ("reserved0", C.c_int32),
        ("workspace_bytes", C.c_int64),
    ]


class AdaptiveRho(C.Structure):
    """tinympc_adaptive_rho_t: adaptive-rho settings, sensitivity tables (host pointers) and the in/out model blobs."""
    _fields_ = [
        ("rho_min", C.c_double), ("rho_max", C.c_double),
        ("enable_clipping", C.c_int32), ("reserved", C.c_int32),
        ("dKinf_drho", vp), ("dPinf_drho", vp),
        ("models", vp),
    ]


# every entry point declared in include/tinympc_b200.h
EXPORTS = [
    "tinympc_b200_default_settings",
    "tinympc_b200_precompute_cache",
    "tinympc_b200_model_blob_elems",
    "tinympc_b200_precompute_cache_batch",
    "tinympc_b200_precompute_cache_batch_device",
    "tinympc_b200_create",
    "tinympc_b200_destroy",
    "tinympc_b200_update_settings",
    "tinympc_b200_get_settings",
    "tinympc_b200_set_mode",
    "tinympc_b200_solve",
    "tinympc_b200_solve_host",
    "tinympc_b200_solve_adaptive",
    "tinympc_b200_solve_adaptive_host",
    "tinympc_b200_get_stats",
    "tinympc_b200_advance",
    "tinympc_b200_supported",
    "tinympc_b200_last_error",
    "tinympc_b200_version",
]
