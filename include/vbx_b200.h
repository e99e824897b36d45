/*
 * vbx_b200 -- C ABI of the H100-native VB-HMM EM loop (the hot path of BUTSpeechFIT/VBx).
 *
 * The reference has no FFI: its boundary for this path is the Python function
 *     VBx(X, Phi, loopProb, Fa, Fb, pi, gamma, maxIters, epsilon, alphaQInit, ref, plot,
 *         return_model, alpha, invL) -> (gamma, pi, Li[, alpha, invL])        VBx/VBx.py:27-29,126
 * called once per recording from VBx/vbhmm.py:154-158.  This header is what a ctypes/cffi binding of
 * that function binds instead (see INTEGRATION.md); every entry point cites the reference lines whose
 * work it replaces.  A *batch* of independent recordings (the reference runs one OS process per
 * recording, AMI_run.sh:53-58) is processed per call.
 *
 * Conventions
 *  - every function returns 0 on success, a negative vbx_status otherwise; nothing throws or aborts;
 *    vbx_last_error() gives a human readable message for the last failure on that handle.
 *  - all array arguments are DEVICE pointers owned by the caller unless the name ends in `_host`;
 *    row-major, packed ragged: recording b owns frame rows offsets[b] .. offsets[b+1]-1.
 *  - `S` below is the padded state count returned by vbx_padded_states(); the live state count of
 *    recording b is n_states[b] <= S (columns >= n_states[b] hold zeros).
 *  - calls are asynchronous on `stream` (a cudaStream_t passed as void*); there is no host
 *    synchronisation inside vbx_prepare_* / vbx_run.  One handle per (device, stream); a handle must
 *    not be used from two threads at once.
 *  - arithmetic is float32 on the device with float64 accumulation of the ELBO scalars; the reference
 *    is float64 numpy (parity: SURVEY.md section 8c, tests/test_parity_gpu.py).
 */
#ifndef VBX_B200_H
#define VBX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vbx_handle_s *vbx_handle_t;

enum vbx_status {
    VBX_OK = 0,
    VBX_ERR_ARG = -1,       /* bad argument (shape, null pointer, unsupported size)           */
    VBX_ERR_CUDA = -2,      /* a CUDA runtime call or kernel launch failed                    */
    VBX_ERR_STATE = -3,     /* call order violated (no plan / workspace not bound / too small) */
    VBX_ERR_NO_DEVICE = -4  /* no usable sm_90 device                                         */
};

/* per-recording bits written to flags_out by vbx_run */
enum vbx_flag {
    VBX_FLAG_NONFINITE = 1,      /* ELBO became NaN/Inf (the reference has no such check)                    */
    VBX_FLAG_ELBO_DECREASED = 2, /* "WARNING: Value of auxiliary function has decreased!" VBx/VBx.py:123-124 */
    VBX_FLAG_CONVERGED = 4       /* stopped by the epsilon test VBx/VBx.py:122 before max_iters              */
};

const char *vbx_version(void);

/* Smallest supported padded state count >= n_states (4, 8, 16, 32 or 64); -1 if n_states > 64 or < 1.
 * (Limits of the float32 kernels: S <= 64, R <= 128 and a multiple of 4.  vbx_plan_f64 / vbx_run_f64 have no such limits.) */
int32_t vbx_padded_states(int32_t n_states);

int vbx_create(int32_t device, vbx_handle_t *out);
int vbx_destroy(vbx_handle_t h);
const char *vbx_last_error(vbx_handle_t h);

/* Options (ints).  "exact_stop" (default 1; read by the next vbx_plan): 1 = the workspace also holds the buffers of the
 * float64 finishing phase and vbx_run applies the stop rule of VBx/VBx.py:122-125 at float64 resolution (a recording
 * leaves the float32 kernels when its ELBO step comes within a guard band of epsilon, see vbx_run); 0 = float32 only.
 * "stop_noise_c" (default 2) / "stop_guard_mult" (default 16): the guard band = epsilon + guard_mult * nb with
 * nb = noise_c * 2^-24 * |ELBO|, the bound used for the float32 noise of an ELBO difference.
 * "fb_split" (read by the next vbx_plan): 0 = auto, 1 = always, 2 = never run the forward and the backward sweep of a
 * recording concurrently on separate warps followed by a combine pass (the choice for batches too small to fill the GPU;
 * results differ from the fused sweep by float32 rounding only, so pin it to 1 or 2 where bit-identical results for a
 * recording alone / inside a large batch matter).
 * "graph": 0 = auto (small batches: plans on the split schedule), 1 = always, 2 = never replay a whole vbx_run as ONE CUDA
 * graph launch.  The second call with identical arguments (pointers and scalars) is captured on a stream of the handle,
 * later identical calls replay it (ordered against `stream` with events, no host synchronisation); any other call, and
 * any failure to capture, launches the kernels directly.  Off while "timing" is on.
 * "fb_priority": 0 = auto (large batches), 1 = always, 2 = never launch the forward-backward sweep on a high-priority side
 * stream of the handle (ordered against `stream` with events, still no host synchronisation), so that it interleaves with
 * the bandwidth-bound kernels of ANOTHER handle working on the same device (vbx_b200/parts.py runs two halves of a batch).
 * Tuning knobs: "fb_states_per_lane" (0 = auto, 1, 2, 4), "fb_classic" (forward-backward sweep: 0 = one-step
 * look-ahead recurrences, 1 = normalise-every-frame), "projection" (0 = auto, 1 = FFMA tiles,
 * 2 = wgmma 3xTF32), "gemm" (in-loop contractions: 0 = tensor cores in split-precision 3xTF32, 1 = FFMA),
 * "timing" (0/1, see vbx_get_timings).  Unknown names return VBX_ERR_ARG. */
int vbx_set_option(vbx_handle_t h, const char *name, int32_t value);

/* Describe a batch: offsets_host[n_rec+1] (HOST, int64, offsets_host[0] == 0), feature dim R
 * (VBx/VBx.py:74 `D`; multiple of 4, <= 128), padded state count S.  Builds the tile lists on the device
 * and reports the workspace the caller must provide through vbx_bind_workspace (256-byte aligned). */
int vbx_plan(vbx_handle_t h, const int64_t *offsets_host, int32_t n_rec, int32_t R, int32_t S,
             size_t *workspace_bytes_out);
int vbx_bind_workspace(vbx_handle_t h, void *workspace, size_t bytes);

/* VBx/VBx.py:87-89:  rho = fea * sqrt(Phi)  and the per-frame constant G (kept as one float64 sum per
 * recording inside the workspace, since G is state independent and only shifts the ELBO).
 * fea [N,R], Phi [R], rho_out [N,R] (may alias fea). */
int vbx_prepare_scale(vbx_handle_t h, const float *fea, const float *Phi, float *rho_out, void *stream);

/* The caller-side projection folded with the scale (VBx/vbhmm.py:129,153 composed with VBx/VBx.py:88-89,
 * as defined for synthetic batches in SURVEY.md section 8d):  rho = X . V  with X [N,D], V [D,R]
 * (V = V0 * sqrt(Phi)), D a multiple of 32;  G is recovered from rho and Phi. */
int vbx_prepare_project(vbx_handle_t h, const float *X, int32_t D, const float *V, const float *Phi,
                        float *rho_out, void *stream);

/* The real-data caller chain in front of VBx() (VBx/vbhmm.py:125-129 x-vector transform, :153 PLDA projection)
 * fused with the scale of VBx/VBx.py:88-89, as two wgmma passes (R must be 128, Dx a multiple of 32):
 *   x_norm = l2norm(l2norm(x_raw - mean1) . lda - mean2)          x_raw [N,Dx], lda [Dx,128], x_norm [N,128]
 *   rho    = ((x_norm - plda_mu) . plda_tr^T) * sqrt(plda_psi)    plda_tr [128,128] and plda_psi [128] are the
 *            DIAGONALISED model (VBx/vbhmm.py:136-143; row n of plda_tr is output dimension n), Phi = plda_psi.
 * x_norm_out and rho_out are distinct [N,128] device arrays; all pointers are device pointers. */
int vbx_prepare_xvectors(vbx_handle_t h, const float *x_raw, int32_t Dx, const float *mean1, const float *lda,
                         const float *mean2, const float *plda_mu, const float *plda_tr, const float *plda_psi,
                         float *x_norm_out, float *rho_out, void *stream);

/* The EM loop VBx/VBx.py:91-125 for every recording of the planned batch.
 *   rho       [N,R]   from vbx_prepare_*                                (VBx/VBx.py:89)
 *   Phi       [R]                                                        (VBx/VBx.py:30 `Phi`)
 *   gamma_io  [N,S]   in: initial responsibilities; out: final ones     (VBx/VBx.py:47,82-83,126)
 *   pi_io     [n_rec,S] in: initial speaker priors; out: learned ones    (VBx/VBx.py:44-46,104)
 *   n_states  [n_rec] live states per recording, or NULL = S for all
 *   Fa, Fb, loop_prob, max_iters, epsilon                                (VBx/VBx.py:27-28)
 *   alpha_io, invL_io [n_rec,S,R] or NULL: speaker models; read for iteration 0 iff warm_start != 0
 *             (VBx/VBx.py:94), written with the last M-step's values (return_model, VBx/VBx.py:126)
 *   Li_out    [n_rec,max_iters] float64 ELBO trace, NaN after the last executed iteration (VBx/VBx.py:105)
 *   n_iters_out [n_rec] iterations executed (the epsilon stop of VBx/VBx.py:122-125 is per recording)
 *   flags_out [n_rec] vbx_flag bits */
/* Stop rule: with a finite epsilon (and option "exact_stop") the test `ELBO_i - ELBO_{i-1} < epsilon` is decided on
 * float32 ELBO values only while the step is far from epsilon; a recording whose step comes near it re-evaluates its
 * last two iterations and all following ones in float64 (inputs: the same float32 rho / gamma), so iteration counts
 * and results follow the float64 reference.  epsilon = -inf runs exactly max_iters float32 iterations. */
int vbx_run(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
            const int32_t *n_states, double Fa, double Fb, double loop_prob, int32_t max_iters, double epsilon,
            float *alpha_io, float *invL_io, int32_t warm_start, double *Li_out, int32_t *n_iters_out,
            int32_t *flags_out, void *stream);

/* AHC initialisation, VBx/vbhmm.py:131-146, for every recording of the planned batch, in float64 like the reference:
 *   cosine similarity of the recording's rows of x (VBx/diarization_lib.py:190-213; x [N,dim], float32 or float64),
 *   thr_out[b] = twoGMMcalib_lin(similarities)[0] (VBx/diarization_lib.py:13-31, 20 iterations),
 *   Z_out = fastcluster.linkage(squareform(-similarity), method='average') in the scipy layout
 *           (cluster id, cluster id, height, size): rows offsets[b] .. offsets[b] + T_b - 2 of Z_out [N,4] belong to
 *           recording b (one unused row per recording).
 * The flat clusters of VBx/vbhmm.py:144-146 are fcluster(Z, -(thr + threshold), 'distance') (the `adjust` shift of
 * :142-143 cancels); vbx_b200/ahc.py holds that O(T) traversal.  workspace: vbx_ahc_workspace_bytes() bytes of
 * device memory (dominated by 8 * sum_b T_b^2), 256-byte aligned.  At most 65535 recordings per call. */
int vbx_ahc_workspace_bytes(vbx_handle_t h, size_t *bytes_out);
int vbx_ahc(vbx_handle_t h, const void *x, int32_t x_is_f64, int32_t dim, void *workspace, size_t workspace_bytes,
            double *Z_out, double *thr_out, void *stream);

/* Output step, VBx/vbhmm.py:160-162: first_out[t] = argsort(-gamma[t])[0], second_out[t] = argsort(-gamma[t])[1]
 * over the live states of the frame's recording (second_out may be NULL; -1 when the recording has one state).
 * gamma [N,S] as left by vbx_run, n_states [n_rec] or NULL, outputs int32 [N]; all device pointers. */
int vbx_hard_labels(vbx_handle_t h, const float *gamma, const int32_t *n_states, int32_t *first_out,
                    int32_t *second_out, void *stream);

/* Float64 evaluation of the same EM loop ("exact" mode for the one-recording-per-call use of VBx/vbhmm.py:154-158,
 * where the reference stops on an ELBO improvement < 1e-6, VBx/vbhmm.py:157 -- below float32 resolution).
 * All arrays float64: fea [N,R] (the reference's X, VBx/VBx.py:30), Phi [R], gamma_io [N,S], pi_io [n_rec,S],
 * alpha_io / invL_io [n_rec,S,R] or NULL, Li_out [n_rec,max_iters].  Needs vbx_plan only (no vbx_prepare_*, no float32
 * workspace); `workspace` must hold vbx_f64_workspace_bytes() bytes.  Simple kernels, not tuned for throughput. */
/* vbx_plan_f64: a plan for vbx_run_f64 ONLY, for any feature dimension R >= 1 and any state count S <= 3600 (no padding:
 * gamma_io [N,S], pi_io [n_rec,S]) - the reference accepts any size, and so does the float64 path of the drop-in. */
int vbx_plan_f64(vbx_handle_t h, const int64_t *offsets_host, int32_t n_rec, int32_t R, int32_t S);
int vbx_f64_workspace_bytes(vbx_handle_t h, size_t *bytes_out);
int vbx_run_f64(vbx_handle_t h, void *workspace, size_t workspace_bytes, const double *fea, const double *Phi,
                double *gamma_io, double *pi_io, const int32_t *n_states, double Fa, double Fb, double loop_prob,
                int32_t max_iters, double epsilon, double *alpha_io, double *invL_io, int32_t warm_start,
                double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream);

/* The module-level forward_backward(lls, tr, ip) of the reference (VBx/VBx.py:146-175) for an arbitrary transition
 * matrix, float64, log domain, dense S x S log-sum-exp per frame as the reference computes it (the EM loop itself never
 * takes this route: its transition matrix is diagonal + rank one).  lls [T,S], tr [S,S] (row = from), ip [S];
 * outputs post [T,S] (state posteriors, the reference's first return value), tll [1], lfw [T,S], lbw [T,S].
 * All device pointers, float64; needs no plan.  1 <= S <= 1024. */
int vbx_forward_backward(vbx_handle_t h, const double *lls, const double *tr, const double *ip, int32_t T, int32_t S,
                         double *post_out, double *tll_out, double *lfw_out, double *lbw_out, void *stream);

/* Multi-GPU (SURVEY.md section 8e): recordings are independent (the reference runs one OS process per recording,
 * AMI_run.sh:53-58), every rank owns a shard and the only exchange is the batch-wide ELBO trace.
 * vbx_attach_comm: hand the library an NCCL communicator the CALLER owns (an ncclComm_t, e.g. torch.distributed's; NULL
 *   detaches).  libnccl_path may be NULL: the library resolves ncclAllReduce from the libnccl.so.2 already loaded in the
 *   process.
 * vbx_elbo_trace: trace_out[i] = sum over this handle's recordings of Li[rec][i], trace_out[max_iters + i] = how many
 *   recordings ran iteration i (Li as written by vbx_run, NaN padded); with a communicator attached the 2*max_iters
 *   doubles are then all-reduced (sum) over the ranks, on `stream`.  Li and trace_out are device pointers. */
int vbx_attach_comm(vbx_handle_t h, void *nccl_comm, int32_t n_ranks, const char *libnccl_path);
int vbx_elbo_trace(vbx_handle_t h, const double *Li, int32_t max_iters, double *trace_out, void *stream);

/* Number of kernels launched by this handle since creation (bench.py reports it as gpu_launches). */
int64_t vbx_launch_count(vbx_handle_t h);

/* Kernel classes for vbx_get_timings (measurement aid; no reference counterpart). */
enum vbx_kernel_class {
    VBX_K_PROJECT = 0,       /* rho = X.V                                   */
    VBX_K_PREPARE = 1,       /* scale / G constant                          */
    VBX_K_RUN_INIT = 2,
    VBX_K_MSTEP = 3,         /* gamma^T rho tiles          VBx/VBx.py:96    */
    VBX_K_SPEAKER_MODEL = 4, /* invL, alpha, bias, reg     VBx/VBx.py:95-96 */
    VBX_K_LOGLIK = 5,        /* log_p_ + row softmax       VBx/VBx.py:97    */
    VBX_K_FWDBWD = 6,        /* forward-backward, pi, ELBO VBx/VBx.py:98-105 */
    VBX_K_EXACT64 = 7,       /* snapshot + float64 finishing phase (stop rule at float64 resolution) */
    VBX_N_KERNEL_CLASSES = 8
};
/* With option "timing" = 1 every kernel class is bracketed by CUDA events on the launching stream.
 * Fills ms_out[VBX_N_KERNEL_CLASSES] / count_out[...] with the accumulated device time and launch counts
 * (HOST arrays; synchronises on the recorded events); reset != 0 clears the accumulators. */
int vbx_get_timings(vbx_handle_t h, double *ms_out, int64_t *count_out, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* VBX_B200_H */
