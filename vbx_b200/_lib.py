"""ctypes binding of libvbx_b200.so (the C ABI declared in include/vbx_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or no sm_90 (H100) device is visible,
every product entry point raises.  (The CPU oracle lives under oracle/ and is test infrastructure.)
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('VBX_B200_LIB', os.path.join(_HERE, 'libvbx_b200.so'))   # override: A/B builds

EXPORTS = ['vbx_version', 'vbx_padded_states', 'vbx_padded_states_wide', 'vbx_create', 'vbx_destroy', 'vbx_last_error',
           'vbx_set_option', 'vbx_plan', 'vbx_bind_workspace', 'vbx_prepare_scale',
           'vbx_prepare_project', 'vbx_prepare_xvectors', 'vbx_run', 'vbx_run_per_recording', 'vbx_hard_labels', 'vbx_hard_labels_keep', 'vbx_ahc_workspace_bytes', 'vbx_ahc', 'vbx_launch_count', 'vbx_get_timings', 'vbx_f64_workspace_bytes',
           'vbx_run_f64', 'vbx_plan_f64', 'vbx_forward_backward', 'vbx_attach_comm', 'vbx_elbo_trace', 'vbx_get_gsum',
           'vbx_score', 'vbx_score_overlap', 'vbx_score_jer', 'vbx_link_batch_workspace_bytes', 'vbx_link_batch',
           'vbx_enroll_batch_workspace_bytes', 'vbx_enroll_batch', 'vbx_cohort_stats_batch_workspace_bytes',
           'vbx_cohort_stats_batch', 'vbx_init_turns', 'vbx_combine_workspace_bytes', 'vbx_combine',
           'vbx_init_random', 'vbx_run_prior', 'vbx_run_f64_prior', 'vbx_class_scatter_workspace_bytes',
           'vbx_class_scatter', 'vbx_stream_window', 'vbx_stream_commit', 'vbx_verify_score_workspace_bytes',
           'vbx_verify_score', 'vbx_verify_metrics_workspace_bytes', 'vbx_verify_metrics',
           'vbx_verify_calibrate_workspace_bytes', 'vbx_verify_calibrate']

FLAG_NONFINITE, FLAG_ELBO_DECREASED, FLAG_CONVERGED = 1, 2, 4
SCORE_BAD_LABEL, SCORE_BAD_REGION, SCORE_BAD_RECORDING = 1, 2, 4      # vbx_score / vbx_score_overlap / vbx_score_jer flags
COMBINE_BAD_LABEL, COMBINE_TOO_MANY_LABELS = 1, 2                  # vbx_combine flags
LINK_MAX_SPEAKERS = 1 << 29                                        # VBX_LINK_MAX_SPEAKERS
KERNEL_CLASSES = ['project', 'prepare', 'run_init', 'mstep_partial', 'speaker_model', 'loglik', 'forward_backward', 'exact64', 'em_contract']


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
    lib.vbx_padded_states_wide.restype = i32
    lib.vbx_padded_states_wide.argtypes = [i32]
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
    lib.vbx_hard_labels_keep.restype = ctypes.c_int
    lib.vbx_hard_labels_keep.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_prepare_xvectors.restype = ctypes.c_int
    lib.vbx_prepare_xvectors.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_run.restype = ctypes.c_int
    lib.vbx_run.argtypes = [vp, vp, vp, vp, vp, vp, dbl, dbl, dbl, i32, dbl, vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_run_per_recording.restype = ctypes.c_int
    lib.vbx_run_per_recording.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, dbl, vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_run_prior.restype = ctypes.c_int
    lib.vbx_run_prior.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, dbl, vp, vp, i32, vp, vp, vp, vp, vp, vp]
    lib.vbx_launch_count.restype = i64
    lib.vbx_launch_count.argtypes = [vp]
    lib.vbx_f64_workspace_bytes.restype = ctypes.c_int
    lib.vbx_f64_workspace_bytes.argtypes = [vp, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_run_f64.restype = ctypes.c_int
    lib.vbx_run_f64.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, dbl, dbl, dbl, i32, dbl, vp, vp, i32, vp, vp, vp, vp]
    lib.vbx_run_f64_prior.restype = ctypes.c_int
    lib.vbx_run_f64_prior.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, dbl, dbl, dbl, i32, dbl, vp, vp, i32, vp, vp,
                                      vp, vp, vp, vp]
    lib.vbx_forward_backward.restype = ctypes.c_int
    lib.vbx_forward_backward.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.vbx_attach_comm.restype = ctypes.c_int
    lib.vbx_attach_comm.argtypes = [vp, vp, i32, ctypes.c_char_p]
    lib.vbx_elbo_trace.restype = ctypes.c_int
    lib.vbx_elbo_trace.argtypes = [vp, vp, i32, vp, vp]
    lib.vbx_get_gsum.restype = ctypes.c_int
    lib.vbx_get_gsum.argtypes = [vp, vp, vp]
    lib.vbx_score.restype = ctypes.c_int
    lib.vbx_score.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp]
    lib.vbx_score_overlap.restype = ctypes.c_int
    lib.vbx_score_overlap.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, i64, vp, vp,
                                      vp, vp, vp]
    lib.vbx_score_jer.restype = ctypes.c_int
    lib.vbx_score_jer.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, i64, vp, vp, vp,
                                  vp, vp, vp, vp]
    lib.vbx_link_batch_workspace_bytes.restype = ctypes.c_int
    lib.vbx_link_batch_workspace_bytes.argtypes = [vp, i32, vp, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_link_batch.restype = ctypes.c_int
    lib.vbx_link_batch.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, vp, vp, vp, ctypes.c_size_t, vp, vp, vp, vp, vp,
                                   vp, vp]
    lib.vbx_enroll_batch_workspace_bytes.restype = ctypes.c_int
    lib.vbx_enroll_batch_workspace_bytes.argtypes = [vp, i32, vp, i64, i64, i64, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_enroll_batch.restype = ctypes.c_int
    lib.vbx_enroll_batch.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, i32, vp, i64, vp, i64, vp, vp, vp, i32, vp,
                                     ctypes.c_size_t, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_cohort_stats_batch_workspace_bytes.restype = ctypes.c_int
    lib.vbx_cohort_stats_batch_workspace_bytes.argtypes = [vp, i32, vp, i64, i64, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_cohort_stats_batch.restype = ctypes.c_int
    lib.vbx_cohort_stats_batch.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, i64, vp, i64, vp, vp, i32, vp,
                                           ctypes.c_size_t, vp, vp, vp, vp]
    lib.vbx_init_turns.restype = ctypes.c_int
    lib.vbx_init_turns.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    lib.vbx_init_random.restype = ctypes.c_int
    lib.vbx_init_random.argtypes = [vp, vp, vp, vp, vp, vp, i32, vp]
    lib.vbx_combine_workspace_bytes.restype = ctypes.c_int
    lib.vbx_combine_workspace_bytes.argtypes = [vp, i32, i32, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_combine.restype = ctypes.c_int
    lib.vbx_combine.argtypes = [vp, i32, vp, i64, vp, vp, i32, vp, vp, vp, i32, vp, vp, ctypes.c_size_t, vp, vp, vp, vp,
                                vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_class_scatter_workspace_bytes.restype = ctypes.c_int
    lib.vbx_class_scatter_workspace_bytes.argtypes = [vp, i64, i32, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_class_scatter.restype = ctypes.c_int
    lib.vbx_class_scatter.argtypes = [vp, vp, i64, i32, i32, vp, vp, ctypes.c_size_t, vp, vp, vp]
    lib.vbx_stream_window.restype = ctypes.c_int
    lib.vbx_stream_window.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, dbl, vp, vp, vp, vp, vp, vp, vp,
                                      vp, vp, vp, vp, vp, vp]
    lib.vbx_stream_commit.restype = ctypes.c_int
    lib.vbx_stream_commit.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.vbx_verify_score_workspace_bytes.restype = ctypes.c_int
    lib.vbx_verify_score_workspace_bytes.argtypes = [vp, i32, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_verify_score.restype = ctypes.c_int
    lib.vbx_verify_score.argtypes = [vp, vp, i64, vp, i32, vp, i64, vp, i32, i32, vp, dbl, dbl, vp, vp, i64, vp, vp, vp,
                                     vp, vp, ctypes.c_size_t, vp, vp]
    lib.vbx_verify_metrics_workspace_bytes.restype = ctypes.c_int
    lib.vbx_verify_metrics_workspace_bytes.argtypes = [vp, i64, i32, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_verify_metrics.restype = ctypes.c_int
    lib.vbx_verify_metrics.argtypes = [vp, vp, vp, i64, i32, vp, dbl, dbl, vp, ctypes.c_size_t, vp, vp, vp, vp, vp, vp,
                                       vp]
    lib.vbx_verify_calibrate_workspace_bytes.restype = ctypes.c_int
    lib.vbx_verify_calibrate_workspace_bytes.argtypes = [vp, i64, ctypes.POINTER(ctypes.c_size_t)]
    lib.vbx_verify_calibrate.restype = ctypes.c_int
    lib.vbx_verify_calibrate.argtypes = [vp, vp, vp, i64, dbl, vp, ctypes.c_size_t, vp, vp, vp]
    lib.vbx_get_timings.restype = ctypes.c_int
    lib.vbx_get_timings.argtypes = [vp, ctypes.POINTER(dbl), ctypes.POINTER(i64), i32]
    _lib = lib
    return lib


MAX_STATES = 128     # largest live state count of the float32 kernels (65 .. 128 pad to the S = 128 tier)


def padded_states(n):
    s = load().vbx_padded_states_wide(int(n))
    if s < 0:
        raise VbxError(f'unsupported number of HMM states {n} (1..{MAX_STATES})')
    return s
