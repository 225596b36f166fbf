"""
ctypes binding of libphicuda.so (include/phicuda.h).  This is the only place that touches the C ABI.

There is NO CPU fallback: if the shared library is missing or no CUDA device is visible, every operation raises.
(Precedent for "compile a .so and load it lazily": PhiML/phiml/backend/tensorflow/_tf_cuda_resample.py:8-35 - but the
reference silently falls back to a slow path there; this package deliberately does not.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('PHICUDA_LIB', os.path.join(_HERE, 'lib', 'libphicuda.so'))   # override: diagnostics only

BC_CONST, BC_ZERO_GRADIENT, BC_PERIODIC, BC_HALO = 0, 1, 2, 3
ERR_INVALID, ERR_UNSUPPORTED, ERR_WORKSPACE = -1, -2, -3


class PhiGrid(C.Structure):
    _fields_ = [('dim', C.c_int32), ('batch', C.c_int32), ('n', C.c_int32 * 3), ('cext', C.c_int32 * 3),
                ('fext', C.c_int32 * 3), ('dx', C.c_float * 3), ('halo', C.c_int32)]


class PhiBC(C.Structure):
    _fields_ = [('lo', C.c_uint8 * 3), ('hi', C.c_uint8 * 3), ('clo', C.c_float * 3), ('chi', C.c_float * 3)]


class PhiVBC(C.Structure):
    _fields_ = [('comp', PhiBC * 3)]


class PhiCgParams(C.Structure):
    _fields_ = [('rtol', C.c_float), ('atol', C.c_float), ('max_iter', C.c_int32), ('balance_rhs', C.c_int32),
                ('project_mean', C.c_int32), ('matrix_offset', C.c_float), ('method', C.c_int32)]


class PhiCgResult(C.Structure):
    _fields_ = [('iterations', C.c_int32), ('converged', C.c_int32), ('diverged', C.c_int32),
                ('residual_sq', C.c_float), ('tol_sq', C.c_float), ('initial_residual_sq', C.c_float)]


class PhiLaunchInfo(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ('kernel', 'generic', 'dist', 'adaptive', 'masked', 'TY', 'stages', 'ZC', 'nzc', 'groups',
                                         'total_units', 'grid_ctas', 'split')]


KERNEL_NONE, KERNEL_LAPLACE_RING, KERNEL_LAPLACE_MARCH, KERNEL_CG_RING, KERNEL_CG_MARCH, KERNEL_STENCIL_RING, KERNEL_RD_RING, KERNEL_WAVE_RING, KERNEL_JULIA, KERNEL_POINTS, KERNEL_SPH = range(11)
INTEGRATOR_EULER, INTEGRATOR_RK4 = 0, 1


class PhiWaveDisc(C.Structure):
    _fields_ = [('center', C.c_float * 3), ('value', C.c_float), ('present', C.c_int32)]


class PhiPlumeParams(C.Structure):
    _fields_ = [('dt', C.c_float), ('inflow_rate', C.c_float), ('buoyancy', C.c_float * 3), ('mac_cormack', C.c_int32), ('static_scalar', C.c_int32),
                ('cg_start_event', C.c_void_p), ('cg_stop_event', C.c_void_p)]


class PhiPointMap(C.Structure):
    _fields_ = [('lower', (C.c_float * 3) * 3), ('size', (C.c_float * 3) * 3), ('res', (C.c_float * 3) * 3)]     # [component][axis]


class PhiSphParams(C.Structure):
    _fields_ = [('lower', C.c_float * 3), ('upper', C.c_float * 3), ('support', C.c_float), ('smoothing_length', C.c_float),
                ('kernel_norm', C.c_float), ('mass', C.c_float), ('pressure_norm', C.c_float), ('viscous_norm', C.c_float),
                ('isotropic_exp', C.c_float), ('base_density', C.c_float), ('dt', C.c_float), ('damping', C.c_float),
                ('gravity', C.c_float * 3)]


class PhiValues64(C.Structure):
    _fields_ = [('dx', C.c_double * 3), ('clo', (C.c_double * 3) * 3), ('chi', (C.c_double * 3) * 3)]


class PhiCgParams64(C.Structure):
    _fields_ = [('rtol', C.c_double), ('atol', C.c_double), ('max_iter', C.c_int32), ('balance_rhs', C.c_int32),
                ('project_mean', C.c_int32), ('matrix_offset', C.c_double), ('method', C.c_int32)]


class PhiCgResult64(C.Structure):
    _fields_ = [('iterations', C.c_int32), ('converged', C.c_int32), ('diverged', C.c_int32),
                ('residual_sq', C.c_double), ('tol_sq', C.c_double), ('initial_residual_sq', C.c_double)]


F3 = C.c_void_p * 3          # float* const v[3]
_P = C.POINTER

# name -> (restype, argtypes); kept in one table so tests can check it against include/phicuda.h
PROTOTYPES = {
    'phicuda_abi_version': (C.c_int, []),
    'phicuda_last_error': (C.c_size_t, [C.c_char_p, C.c_size_t]),
    'phicuda_device_info': (C.c_int, [C.c_char_p, C.c_size_t, _P(C.c_int), _P(C.c_int), _P(C.c_int)]),
    'phicuda_last_launch_info': (C.c_int, [_P(PhiLaunchInfo)]),
    'phicuda_last_cg_passes': (C.c_int, []),
    'phicuda_last_cg_operator': (C.c_int, []),
    'phicuda_max_abs_velocity_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p]),
    'phicuda_laplace_f32': (C.c_int, [_P(PhiGrid), _P(PhiBC), C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_laplace_axpy_f32': (C.c_int, [_P(PhiGrid), _P(PhiBC), C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]),
    'phicuda_divergence_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p]),
    'phicuda_grad_sub_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p]),
    'phicuda_advect_centered_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, _P(PhiBC), C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]),
    'phicuda_advect_staggered_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, _P(PhiVBC), F3, F3, C.c_float, C.c_void_p]),
    'phicuda_grid_sample_f32': (C.c_int, [_P(PhiGrid), _P(PhiBC), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'phicuda_mac_cormack_centered_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, _P(PhiBC), C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_float, C.c_float, C.c_void_p]),
    'phicuda_axpy_centered_f32': (C.c_int, [_P(PhiGrid), C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_add_buoyancy_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiBC), C.c_void_p, C.c_float * 3, C.c_float, F3, C.c_void_p]),
    'phicuda_cg_workspace_bytes': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_cg_poisson_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, _P(PhiCgParams), C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_diffuse_implicit_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_int32, C.c_float, C.c_void_p, C.c_void_p, _P(PhiCgParams),
                                               C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_diffuse_implicit_varying_f32': (C.c_int, [_P(PhiGrid), _P(PhiBC), C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p,
                                                       _P(PhiCgParams), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_make_incompressible_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p, _P(PhiCgParams),
                                                  C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_divergence_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_grad_sub_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_collocated_workspace_bytes': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_wide_laplace_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_make_incompressible_centered_host_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, _P(PhiCgParams), C.c_void_p,
                                                                C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_mul_faces_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, F3, C.c_void_p]),
    'phicuda_cg_poisson_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, C.c_void_p, _P(PhiCgParams),
                                                C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_make_incompressible_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         _P(PhiCgParams), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_comm_create': (C.c_int, [C.c_int, C.c_int, _P(PhiGrid), _P(C.c_void_p), C.c_void_p]),
    'phicuda_comm_connect': (C.c_int, [C.c_void_p, C.c_void_p]),
    'phicuda_comm_destroy': (C.c_int, [C.c_void_p]),
    'phicuda_cg_poisson_dist_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, _P(PhiCgParams), C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    'phicuda_cg_poisson_dist_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, C.c_void_p, _P(PhiCgParams), C.c_void_p,
                                                     C.c_void_p, C.c_void_p]),
    'phicuda_plume_scratch_bytes': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_plume_step_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiBC), F3, C.c_void_p, C.c_void_p, C.c_void_p,
                                         _P(PhiPlumeParams), _P(PhiCgParams), C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_void_p]),
    'phicuda_plume_step_masked_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiBC), F3, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, F3, _P(PhiPlumeParams), _P(PhiCgParams), C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_reaction_diffusion_scratch_bytes': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_reaction_diffusion_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
                                                 C.c_float, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_wave_scratch_bytes': (C.c_size_t, [_P(PhiGrid), C.c_int32]),
    'phicuda_wave_f32': (C.c_int, [_P(PhiGrid), _P(PhiBC), C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, _P(PhiWaveDisc),
                                   C.c_float, _P(C.c_float), C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_julia_scratch_bytes': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_julia_f32': (C.c_int, [_P(PhiGrid), _P(C.c_float), _P(C.c_float), C.c_int32, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_advect_points_f32': (C.c_int, [_P(PhiGrid), _P(PhiVBC), F3, _P(PhiPointMap), C.c_void_p, C.c_int64, C.c_int32, C.c_float,
                                            C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_sph_scratch_bytes': (C.c_size_t, [C.c_int64, C.c_int32, _P(PhiSphParams)]),
    'phicuda_sph_f32': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, _P(PhiSphParams), C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_laplace_f64': (C.c_int, [_P(PhiGrid), _P(PhiBC), _P(PhiValues64), C.c_void_p, C.c_void_p, C.c_void_p]),
    'phicuda_laplace_axpy_f64': (C.c_int, [_P(PhiGrid), _P(PhiBC), _P(PhiValues64), C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]),
    'phicuda_divergence_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), F3, C.c_void_p, C.c_void_p]),
    'phicuda_grad_sub_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), F3, C.c_void_p, C.c_void_p]),
    'phicuda_advect_centered_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), F3, _P(PhiBC), _P(PhiValues64), C.c_void_p,
                                              C.c_void_p, C.c_double, C.c_void_p]),
    'phicuda_advect_staggered_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), F3, _P(PhiVBC), _P(PhiValues64), F3, F3,
                                               C.c_double, C.c_void_p]),
    'phicuda_cg_workspace_bytes_f64': (C.c_size_t, [_P(PhiGrid)]),
    'phicuda_cg_poisson_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), C.c_void_p, C.c_void_p, _P(PhiCgParams64), C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    'phicuda_make_incompressible_f64': (C.c_int, [_P(PhiGrid), _P(PhiVBC), _P(PhiValues64), F3, C.c_void_p, C.c_void_p,
                                                  _P(PhiCgParams64), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}


class PhiCudaError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"libphicuda error {code}: {message}")
        self.code = code


class Unsupported(PhiCudaError):
    """The case is valid in the reference but outside this fast path (PHI_ERR_UNSUPPORTED)."""


_lib = None


def load():
    """Loads libphicuda.so (no GPU needed for loading; compute calls need one)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           f"or `make -C phiflow_b200/csrc`. phiflow_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.phicuda_abi_version() != 2:
        raise RuntimeError("libphicuda ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    buf = C.create_string_buffer(512)
    load().phicuda_last_error(buf, 512)
    return buf.value.decode()


def check(code: int):
    if code == 0:
        return
    msg = last_error()
    if code == ERR_UNSUPPORTED:
        raise Unsupported(code, msg)
    raise PhiCudaError(code, msg)
