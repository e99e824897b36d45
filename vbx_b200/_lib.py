"""ctypes binding of libvbx_b200.so (the C ABI declared in include/vbx_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or no sm_90 (H100) device is visible,
every product entry point raises.  (The CPU oracle lives under oracle/ and is test infrastructure.)
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('VBX_B200_LIB', os.path.join(_HERE, 'libvbx_b200.so'))   # override: A/B builds

EXPORTS = ['vbx_version', 'vbx_padded_states', 'vbx_create', 'vbx_destroy', 'vbx_last_error',
           'vbx_set_option', 'vbx_plan', 'vbx_bind_workspace', 'vbx_prepare_scale',
           'vbx_prepare_project', 'vbx_prepare_xvectors', 'vbx_run', 'vbx_hard_labels', 'vbx_ahc_workspace_bytes', 'vbx_ahc', 'vbx_launch_count', 'vbx_get_timings', 'vbx_f64_workspace_bytes',
           'vbx_run_f64', 'vbx_plan_f64', 'vbx_forward_backward', 'vbx_attach_comm', 'vbx_elbo_trace']

FLAG_NONFINITE, FLAG_ELBO_DECREASED, FLAG_CONVERGED = 1, 2, 4
KERNEL_CLASSES = ['project', 'prepare', 'run_init', 'mstep_partial', 'speaker_model', 'loglik', 'forward_backward', 'exact64']


class VbxError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen the library and declare the prototypes of include/vbx_b200.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VbxError(f'{LIB_PATH} is missing - run `python -c "import __graft_entry__ as g; g.build()"` '
                       '(there is no CPU fallback for the VB-HMM path)')
    lib = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, dbl = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double
    lib.vbx_version.restype = ctypes.c_char_p
    lib.vbx_version.argtypes = []
    lib.vbx_padded_states.restype = i32
    lib.vbx_padded_states.argtypes = [i32]
    lib.vbx_create.restype = ctypes.c_int
    lib.vbx_create.argtypes = [i32, ctypes.POINTER(vp)]
    lib.vbx_destroy.restype = ctypes.c_int
    lib.vbx_destroy.argtypes = [vp]
    lib.vbx_last_error.restype = ctypes.c_char_p
    lib.vbx_last_error.argtypes = [vp]
    lib.vbx_set_option.restype = ctypes.c_int
    lib.vbx_set_option.argtypes = [vp, ctypes.c_char_p, i32]
    lib.vbx_plan.restype = ctypes.c_int
    lib.vbx_plan.argtypes = [vp, ctypes.POINTER(i64), i32, i32, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_plan_f64.restype = ctypes.c_int
    lib.vbx_plan_f64.argtypes = [vp, ctypes.POINTER(i64), i32, i32, i32]
    lib.vbx_bind_workspace.restype = ctypes.c_int
    lib.vbx_bind_workspace.argtypes = [vp, vp, ctypes.c_size_t]
    lib.vbx_prepare_scale.restype = ctypes.c_int
    lib.vbx_prepare_scale.argtypes = [vp, vp, vp, vp, vp]
    lib.vbx_prepare_project.restype = ctypes.c_int
    lib.vbx_prepare_project.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_ahc_workspace_bytes.restype = ctypes.c_int
    lib.vbx_ahc_workspace_bytes.argtypes = [vp, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_ahc.restype = ctypes.c_int
    lib.vbx_ahc.argtypes = [vp, vp, i32, i32, vp, ctypes.c_size_t, vp, vp, vp]
    lib.vbx_hard_labels.restype = ctypes.c_int
    lib.vbx_hard_labels.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.vbx_prepare_xvectors.restype = ctypes.c_int
    lib.vbx_prepare_xvectors.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_run.restype = ctypes.c_int
    lib.vbx_run.argtypes = [vp, vp, vp, vp, vp, vp, dbl, dbl, dbl, i32, dbl, vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_launch_count.restype = i64
    lib.vbx_launch_count.argtypes = [vp]
    lib.vbx_f64_workspace_bytes.restype = ctypes.c_int
    lib.vbx_f64_workspace_bytes.argtypes = [vp, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_run_f64.restype = ctypes.c_int
    lib.vbx_run_f64.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, dbl, dbl, dbl, i32, dbl, vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_forward_backward.restype = ctypes.c_int
    lib.vbx_forward_backward.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.vbx_attach_comm.restype = ctypes.c_int
    lib.vbx_attach_comm.argtypes = [vp, vp, i32, ctypes.c_char_p]
    lib.vbx_elbo_trace.restype = ctypes.c_int
    lib.vbx_elbo_trace.argtypes = [vp, vp, i32, vp, vp]
    lib.vbx_get_timings.restype = ctypes.c_int
    lib.vbx_get_timings.argtypes = [vp, ctypes.POINTER(dbl), ctypes.POINTER(i64), i32]
    _lib = lib
    return lib


def padded_states(n):
    s = load().vbx_padded_states(int(n))
    if s < 0:
        raise VbxError(f'unsupported number of HMM states {n} (1..64)')
    return s
