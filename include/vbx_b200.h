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
 *    not be used from two threads at once.  Handles on different devices may be used in one process,
 *    each from its own thread.
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

/* Smallest padded state count >= n_states of the tiers up to 64 (4, 8, 16, 32 or 64); -1 if n_states > 64 or < 1.
 * (Limits of the float32 kernels: S <= 128, R <= 128 and a multiple of 4.  vbx_plan_f64 / vbx_run_f64 have no such limits.) */
int32_t vbx_padded_states(int32_t n_states);
/* The same with the wide tier: 4, 8, 16, 32, 64, or 128 for 65 <= n_states <= 128; -1 if n_states > 128 or < 1.
 * S = 128 plans always run the split forward-backward schedule (see option "fb_split"). */
int32_t vbx_padded_states_wide(int32_t n_states);

int vbx_create(int32_t device, vbx_handle_t *out);
int vbx_destroy(vbx_handle_t h);
const char *vbx_last_error(vbx_handle_t h);

/* Options (ints).  "exact_stop" (default 1; read by the next vbx_plan): 1 = the workspace also holds the buffers of the
 * float64 finishing phase and vbx_run applies the stop rule of VBx/VBx.py:122-125 at float64 resolution (a recording
 * leaves the float32 kernels when its ELBO step comes below epsilon + 16 nb, nb = 2 * 2^-24 * |ELBO| being the bound
 * used for the float32 noise of an ELBO difference; see vbx_run); 0 = float32 only.
 * "fb_split" (read by the next vbx_plan): 0 = auto, 1 = always, 2 = never run the forward and the backward sweep of a
 * recording concurrently on separate warps followed by a combine pass (the choice for batches too small to fill the GPU;
 * results differ from the fused sweep by float32 rounding only, so pin it to 1 or 2 where bit-identical results for a
 * recording alone / inside a large batch matter).  S = 128 plans always split: 0 and 1 mean the same there, and
 * vbx_plan refuses S = 128 with VBX_ERR_ARG while fb_split = 2.
 * "graph": 0 = auto (small batches: plans on the split schedule), 1 = always, 2 = never replay a whole vbx_run as ONE CUDA
 * graph launch.  The second call with identical arguments (pointers and scalars) is captured on a stream of the handle,
 * later identical calls replay it (ordered against `stream` with events, no host synchronisation); any other call, and
 * any failure to capture, launches the kernels directly.  Off while "timing" is on.
 * Tuning knobs: "fb_states_per_lane" (0 = auto, 1, 2, 4; at S = 64 values below 2 and at S = 128 values below 4 are
 * raised to those, since a recording's lane group must fit in a warp), "fb_classic" (forward-backward sweep: 0 = one-step
 * look-ahead recurrences, 1 = normalise-every-frame), "fb_ring" (look-ahead sweep fed from shared-memory rings by bulk
 * copies that recomputes the forward variables from checkpoints instead of parking them in gamma: 1 = default, used when
 * no recording of the plan exceeds 2048 frames; 0 = register bursts; results are bit-identical), "projection" (0 = auto, 1 = FFMA tiles,
 * 2 = wgmma 3xTF32), "gemm" (in-loop contractions: 0 = tensor cores in split-precision 3xTF32, 1 = FFMA),
 * "timing" (0/1, see vbx_get_timings).  Unknown names return VBX_ERR_ARG. */
int vbx_set_option(vbx_handle_t h, const char *name, int32_t value);

/* Describe a batch: offsets_host[n_rec+1] (HOST, int64, offsets_host[0] == 0), feature dim R
 * (VBx/VBx.py:74 `D`; multiple of 4, <= 128), padded state count S (4, 8, 16, 32, 64 or 128, from vbx_padded_states_wide;
 * S = 128 always takes the split forward-backward schedule).  Builds the tile lists on the device
 * and reports the workspace the caller must provide through vbx_bind_workspace (256-byte aligned). */
int vbx_plan(vbx_handle_t h, const int64_t *offsets_host, int32_t n_rec, int32_t R, int32_t S,
             size_t *workspace_bytes_out);
int vbx_bind_workspace(vbx_handle_t h, void *workspace, size_t bytes);

/* VBx/VBx.py:87-89:  rho = fea * sqrt(Phi)  and the per-frame constant G (kept as one float64 sum per
 * recording inside the workspace, since G is state independent and only shifts the ELBO).
 * fea [N,R], Phi [R], rho_out [N,R] (may alias fea).
 * Alignment: the kernels access rho and gamma arrays (and fea, Phi, X, V) with 16-byte vectors, so vbx_prepare_scale,
 * vbx_prepare_project, vbx_run, vbx_run_per_recording, vbx_hard_labels and vbx_hard_labels_keep return VBX_ERR_ARG,
 * before anything is launched, for any of those device pointers that is not 16-byte aligned (a view that starts
 * inside an allocation, for example). */
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
 *   flags_out [n_rec] vbx_flag bits
 * A recording with no frames (or n_states 0) runs no iteration: n_iters 0, flags 0, its Li row all NaN, and its rows of
 * pi_io, alpha_io and invL_io are left as passed in. */
/* Stop rule: with a finite epsilon (and option "exact_stop") the test `ELBO_i - ELBO_{i-1} < epsilon` is decided on
 * float32 ELBO values only while the step is far from epsilon; a recording whose step comes near it re-evaluates its
 * last two iterations and all following ones in float64 (inputs: the same float32 rho / gamma), so iteration counts
 * and results follow the float64 reference.  epsilon = -inf runs exactly max_iters float32 iterations. */
int vbx_run(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
            const int32_t *n_states, double Fa, double Fb, double loop_prob, int32_t max_iters, double epsilon,
            float *alpha_io, float *invL_io, int32_t warm_start, double *Li_out, int32_t *n_iters_out,
            int32_t *flags_out, void *stream);

/* vbx_run with per-recording hyperparameters: Fa, Fb and loop_prob are float64 DEVICE arrays [n_rec] (recording b runs
 * with Fa[b], Fb[b], loop_prob[b]); every other argument and the stop rule are as in vbx_run.  One batch can so hold a
 * whole hyperparameter grid (one entry per recording and setting) or recordings tuned for different domains.  A recording
 * whose values equal vbx_run's scalars gets bit-identical results on the same plan and options.
 * Null arrays return VBX_ERR_ARG.  The values are read on the device, so they are not validated: a recording whose
 * values make its ELBO non-finite (Fb = 0, for example) ends with VBX_FLAG_NONFINITE, and the other recordings of the
 * batch are not affected.  Option "graph": the identity of a call covers the three array POINTERS, not their contents;
 * the arrays are read inside the replayed launch sequence, so a replay uses their contents at the time it runs (change
 * them in place on `stream` between calls and the replay sees the new values).  vbx_run_f64 has no per-recording form. */
int vbx_run_per_recording(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
                          const int32_t *n_states, const double *Fa, const double *Fb, const double *loop_prob,
                          int32_t max_iters, double epsilon, float *alpha_io, float *invL_io, int32_t warm_start,
                          double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream);

/* vbx_run_per_recording with a Gaussian prior on each state's speaker latent (DESIGN.md section 5.23): state s of
 * recording b starts from the posterior of y ~ N(0, I) given prior_n[b,s] x-vectors whose feature sum is prior_F[b,s,:]
 * (the fea units of vbx_prepare_scale, NOT rho: the kernels multiply by sqrt(Phi) themselves), for example the float64
 * statistics n_enroll / F_enroll of an enrolled speaker (vbx_enroll_batch).  With c = Fa[b] / Fb[b]:
 *   lambda0 = 1 + c n_e Phi      mu0 = c sqrt(Phi) F_e / lambda0
 *   invL = 1 / (1 + c (N_s + n_e) Phi)      alpha = c invL (rho^T gamma_s + sqrt(Phi) F_e)
 *   ELBO regulariser  Fb/2 sum_{s,r} [log(lambda0 invL) - lambda0 invL - lambda0 (alpha - mu0)^2 + 1]
 * which is the ELBO of the recording with those x-vectors appended as frames held on state s, minus a constant.  The
 * log-likelihoods, the forward-backward, pi and the stop rule are vbx_run's; warm_start reads alpha_io / invL_io as
 * given and puts the prior into the regulariser.  prior_n [n_rec,S] and prior_F [n_rec,S,R] are float64 DEVICE arrays
 * (S, R of the plan; columns s >= n_states[b] are not read); null arrays return VBX_ERR_ARG.  Their values are read on
 * the device and not validated (n_e >= 0 and finite values are the caller's to check).  A recording whose prior is
 * all zero gets bit-identical results to vbx_run_per_recording (gamma, pi, Li, n_iters, flags, alpha, invL), whatever
 * the other recordings' priors.  Stream ordered, no allocation, no host synchronisation.  Option
 * "graph": the two prior POINTERS are part of a call's identity, and a replay reads their contents as it runs. */
int vbx_run_prior(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
                  const int32_t *n_states, const double *Fa, const double *Fb, const double *loop_prob,
                  int32_t max_iters, double epsilon, float *alpha_io, float *invL_io, int32_t warm_start,
                  double *Li_out, int32_t *n_iters_out, int32_t *flags_out, const double *prior_n,
                  const double *prior_F, void *stream);

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

/* Output step under an upper bound on the speaker count (DESIGN.md section 5.14).  mass_out [n_rec,S] float64 is written
 * with N_s = sum_t gamma[t,s] of every live state (0 for the padded columns; a recording without frames has a row of
 * zeros), summed in an order that depends on the recording's length only.  Of recording b the keep[b] live states of
 * largest mass survive (ties: the lower index); first_out / second_out are vbx_hard_labels' outputs over the surviving
 * states only (second_out may be NULL; -1 when one state survives).  keep >= n_states gives vbx_hard_labels' labels.
 * keep [n_rec] int32; every keep[b] must be >= 1 (VBX_ERR_ARG otherwise: the call reads keep back, so it waits for
 * `stream`).  All other arguments as vbx_hard_labels; all device pointers. */
int vbx_hard_labels_keep(vbx_handle_t h, const float *gamma, const int32_t *n_states, const int32_t *keep,
                         int32_t *first_out, int32_t *second_out, double *mass_out, void *stream);

/* Initial responsibilities from speaker turns (VB resegmentation of an existing diarization, DESIGN.md section 5.20),
 * the generalisation of VBx/vbhmm.py:150-152's qinit to segments covered by several speakers or by none.  Runs on the
 * handle's plan (vbx_plan or vbx_plan_f64: offsets, n_rec, S).  All arrays are DEVICE arrays:
 *   seg [N,2] int64               x-vector t's segment [lo, hi) in ticks
 *   spk_off [n_rec+1] int64       recording b has the speakers spk_off[b] .. spk_off[b+1]-1, K_b = their number <= S
 *   turn_off [n_spk+1] int64      speaker k has the turns turn_off[k] .. turn_off[k+1]-1 (n_spk = spk_off[n_rec])
 *   turn_lo, turn_hi [n_turns]    each speaker's turns [lo, hi) in ticks, sorted and disjoint
 *   turn_cum [n_turns] int64      the exclusive prefix sum of the turn lengths within each speaker
 *   smoothing [n_rec] float64
 * With c_k = (ticks of [lo, hi) inside speaker k's turns) / (hi - lo) (0 when hi <= lo), the outputs are
 *   gamma_out [N,S]   softmax_k(smoothing_b c_k) over k < K_b, 0 in the other columns (a segment no speaker covers gets
 *                     a uniform row; a recording with K_b = 0 a row of zeros)
 *   pi_out [n_rec,S]  1 / K_b in the first K_b columns, 0 in the others
 * float64 (out_is_f64 != 0) or float32; the softmax is evaluated in float64 and rounded once.  A group of lanes per
 * x-vector (S rounded up to a power of two, at most a warp) runs over the recording's speakers; the covered time is P(hi) - P(lo), P(x) = the speaker's turn time before x
 * (binary search over turn_lo plus turn_cum, int64).  spk_off and turn_off are read back to check them (K_b > S or a
 * negative count returns VBX_ERR_ARG), so the call waits for `stream`; otherwise stream ordered, no allocation. */
int vbx_init_turns(vbx_handle_t h, const int64_t *seg, const int64_t *spk_off, const int64_t *turn_off,
                   const int64_t *turn_lo, const int64_t *turn_hi, const int64_t *turn_cum, const double *smoothing,
                   void *gamma_out, void *pi_out, int32_t out_is_f64, void *stream);

/* Random initial responsibilities (the VB-HMM started without AHC, DESIGN.md section 5.22): the flat-Dirichlet rows of
 * VBx/VBx.py:79-83 drawn from a counter-based generator, so that every restart of every recording can share one batch.
 * Runs on the handle's plan (vbx_plan or vbx_plan_f64: offsets, n_rec, S).  All arrays are DEVICE arrays:
 *   rec_key [n_rec] uint64   the recording's stream (the first 8 bytes, little-endian, of SHA-256 of its name)
 *   seed [n_rec] uint64      the restart's seed
 *   n_states [n_rec] int32   live states N_b <= S per recording, or NULL = S for all (as for vbx_run)
 * For x-vector t of recording b (its index inside the recording) and state block j = s / 4, Philox4x64-10 (Salmon et
 * al. 2011) on counter (t, j, rec_key[b], 0) with key (seed[b], 0) gives four words; word i belongs to state 4j + i:
 *   u = ((w >> 11) + 0.5) 2^-53,  e_s = -log u,  gamma_out[t, s] = e_s / sum_{s' < N_b} e_s'  (0 in the other columns)
 *   pi_out [n_rec,S] = 1 / N_b in the first N_b columns, 0 in the others
 * float64 (out_is_f64 != 0) or float32; evaluated in float64 and rounded once.  A row's bits depend on (rec_key, seed,
 * t, N_b) only, not on S or the rest of the batch.  Stream ordered, no allocation, no host synchronisation. */
int vbx_init_random(vbx_handle_t h, const uint64_t *rec_key, const uint64_t *seed, const int32_t *n_states,
                    void *gamma_out, void *pi_out, int32_t out_is_f64, void *stream);

/* Speaker linking across the recordings of an archive (DESIGN.md sections 5.15, 5.18, 5.19) for G independent
 * problems in one set of launches, e.g. one per setting of a sweep; one archive is G = 1.  Needs a handle, no plan.  The
 * problems share fea [N,R] float32 and Phi [R] (DEVICE: the features and between-speaker variances the VB-HMM ran with,
 * R <= 128); problem g has
 *   speaker [G,N] int32 (DEVICE)   row g: the speaker of x-vector t in [0, M[g]), or -1 (other values count as -1)
 *   M [G] (HOST)                   its number of speakers (a recording's VB-HMM labels, numbered across the archive)
 *   speaker_rec [sum M] (DEVICE)   the recording of each speaker (speakers of one recording are never linked), problem
 *                                  g's at off_g = M[0] + .. + M[g-1]
 *   Fa [G], Fb [G] (HOST)          the VB-HMM's scalars; every c_g = Fa[g] / Fb[g] must be finite and >= 0
 * Per speaker s, n_s = #{t : speaker[g,t] = s} and F_s = sum of those rows of fea, float64, summed in an order fixed by
 * the positions of s's x-vectors relative to its first one.  Each speaker's CTA reads its row of speaker[] over the
 * whole span from its first to its last x-vector, so the statistics cost sum_s (span_s + n_s R) reads: about (K + R) N
 * per problem for speakers packed by recording with K speakers each, but up to M N when speakers spread across the
 * whole array.  With L_s,r = 1 + c_g n_s Phi_r and b_s,r = c_g sqrt(Phi_r) F_s,r
 *   LLR(s,u) = 1/2 sum_r [ (b_s,r + b_u,r)^2 / (L_s,r + L_u,r - 1) - b_s,r^2 / L_s,r - b_u,r^2 / L_u,r
 *                          + log L_s,r + log L_u,r - log(L_s,r + L_u,r - 1) ]
 * (0 when n_s or n_u is 0), and the distance of two speakers is -LLR; 1e30 between two speakers of one recording, 0 on
 * the diagonal.  With mean, std [sum M] (DEVICE, problem g's at off_g: cohort statistics of the same speakers from
 * vbx_cohort_stats_batch; every std must be finite and > 0) the distance of two speakers of different recordings is
 * -S(s, u) instead, the adaptive symmetric normalisation (AS-norm) of DESIGN.md section 5.17
 *   S(s, u) = 1/2 [ (LLR(s,u) - mean[s]) / std[s] + (LLR(s,u) - mean[u]) / std[u] ],
 * with 1e30 within a recording and 0 on the diagonal as before; the matrix stays symmetric bit for bit.  Give both of
 * mean and std or neither.  Z_out [sum M, 4] holds problem g's average linkage of those distances (M[g] - 1 rows from
 * row off_g, scipy's layout), computed by vbx_ahc's linkage kernel (ties: the lowest slot); it is needed when some
 * M[g] >= 2.  Optional outputs (NULL: not written): n_out [sum M], F_out [sum M, R] and dist_out with problem g's
 * M[g] x M[g] distances from element M[0]^2 + .. + M[g-1]^2, float64.  Problem g's n, F, distances and Z do not depend
 * on the other problems: they are the same bits in one launch or over several.  workspace:
 * vbx_link_batch_workspace_bytes(G, M) bytes, 256-byte aligned: about 8 M[g]^2 + 1.1 KB M[g] per problem, and the
 * size of a batch is at most the sum of the sizes of its problems alone, so problems packed by those sizes fit a
 * budget.  Stream ordered, no allocation, no host synchronisation; the problems' offsets and c_g go to the device in
 * one copy from the host, as vbx_ahc's offsets do.  R outside 1..128, an M[g] outside [0, VBX_LINK_MAX_SPEAKERS] (the
 * linkage kernel keeps 4 (M - 1) in int32), more than 2^31 - 1 speakers in all, a bad c_g, mean without std (or std
 * without mean), null pointers or a workspace too small return VBX_ERR_ARG. */
#define VBX_LINK_MAX_SPEAKERS 536870912 /* 2^29 */
int vbx_link_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, size_t *bytes_out);
int vbx_link_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                   const int32_t *speaker, const int64_t *M, const int32_t *speaker_rec, const double *Fa,
                   const double *Fb, void *workspace, size_t workspace_bytes, double *n_out, double *F_out,
                   double *dist_out, double *Z_out, const double *mean, const double *std, void *stream);

/* Enrolment and cohort statistics of G independent problems in one set of launches (DESIGN.md sections 5.16, 5.17,
 * 5.19), e.g. the settings of a sweep; one archive is G = 1.  Each needs a handle, no plan.  The problems share fea
 * [N,R] and Phi [R] (DEVICE, as for vbx_link_batch); problem g has its row g of speaker [G,N] (DEVICE, local speakers
 * in [0, M[g]), -1 = none), M [G] (HOST) and Fa [g], Fb [g] (HOST; every c_g = Fa[g] / Fb[g] finite and >= 0).
 * Per-speaker arrays are packed by the speaker offsets off_g = M[0] + .. + M[g-1].  Every speaker set gets
 * vbx_link_batch's statistics n, F (and the b, e of its LLR) with c_g.  Problem g's outputs do not depend on the other
 * problems: they are the same bits in one launch or over several.  Stream ordered, no allocation, no host
 * synchronisation: the problems' offsets and scalars go to the device in one copy from pageable host memory.
 * VBX_ERR_ARG: R outside 1..128, a bad c_g, G < 0, an M[g] outside [0, VBX_LINK_MAX_SPEAKERS], more than 2^31 - 1
 * speakers in all, null pointers, misaligned or short workspace, and the conditions given below.
 *
 * vbx_enroll_batch: every problem's archive speakers against one set of E known speakers (enroll_fea [N_e,R] through
 * the same front end, enroll_speaker [N_e] in [0, E), DEVICE; packed by speaker the enrolled statistics cost about
 * (E + R) N_e reads per problem) at n_thr >= 1 thresholds (HOST, each |t| <= 1e15).  Problem g's archive speakers are
 * packed by recording: row g of speaker_rec_offsets [G, n_rec + 1] (HOST int64, from 0 to M[g], non-decreasing) holds
 * recording b's speakers at [b] .. [b+1]-1.  Every archive speaker s is scored against every enrolled speaker e,
 *   llr [s][e] = LLR(s, e) of vbx_link_batch, bit-identical to -dist of vbx_link_batch run on the same speakers.
 * Per recording with K speakers and threshold t, the minimum-cost assignment of the K x (E + K) matrix
 * C[k][e] = t - llr[k][e] (e < E), C[k][E + j] = 0 ("unknown" columns), by shortest augmenting paths; ties go to the
 * lowest column, so a real column at cost 0 wins over the unknown ones.  Outputs (DEVICE):
 *   assign_out [n_thr, sum M] int32   the enrolled speaker of each archive speaker, -1 = unknown (plane h: threshold h)
 *   best_llr_out [n_thr, sum M]       llr of the assigned pair; for an unknown speaker its largest llr
 *   llr_out [sum M, E], n_out [sum M], F_out [sum M, R], n_enroll_out [G, E], F_enroll_out [G, E, R]: optional (NULL:
 *   not written)
 * mean, std [sum M] and enroll_mean, enroll_std [G, E] (DEVICE, all four or none, except that mean and std may be NULL
 * when sum M = 0; cohort statistics from vbx_cohort_stats_batch): the assignment runs on S(s, e) of vbx_link_batch in place of LLR(s, e), problem g with its
 * own rows; the thresholds are on S, and best_llr_out and llr_out hold S.  workspace:
 * vbx_enroll_batch_workspace_bytes(G, M, E, N_e, max_k, n_thr) bytes with max_k >= the largest K of any recording of
 * any problem, 256-byte aligned: about 8 sum M E + 1.1 KB (sum M + G E) + 4 G N_e + 2 x SMs x 50 (E + max_k) bytes.
 * Further VBX_ERR_ARG: E, N_e or n_thr < 1, n_rec < 0, offsets not from 0 to M[g] or decreasing. */
int vbx_enroll_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, int64_t E, int64_t N_e,
                                     int64_t max_k, int32_t n_thr, size_t *bytes_out);
int vbx_enroll_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                     const int32_t *speaker, const int64_t *M, const int64_t *speaker_rec_offsets, int32_t n_rec,
                     const float *enroll_fea, int64_t N_e, const int32_t *enroll_speaker, int64_t E, const double *Fa,
                     const double *Fb, const double *thresholds, int32_t n_thr, void *workspace,
                     size_t workspace_bytes, int32_t *assign_out, double *best_llr_out, double *llr_out, double *n_out,
                     double *F_out, double *n_enroll_out, double *F_enroll_out, const double *mean, const double *std,
                     const double *enroll_mean, const double *enroll_std, void *stream);
/* vbx_cohort_stats_batch: the statistics that score normalisation (AS-norm, DESIGN.md section 5.17) needs, for every
 * problem against one cohort of C >= 2 speakers known to be someone else (cohort_fea [N_c,R] through the same front
 * end, cohort_speaker [N_c] in [0, C), DEVICE).  Every scored speaker x is scored against every cohort speaker with
 * vbx_link_batch's LLR (the kernel of vbx_enroll_batch: bit-identical to its llr against the same speakers), and with
 * the top K = min(top_k, C) of x's cohort scores, top_k >= 2,
 *   mean_out [x] = mean of x's K largest cohort scores, std_out [x] = their population standard deviation (ddof 0)
 * (DEVICE float64 [sum M]; ties at the K-th value count as many copies as needed), by fixed-order sums.  scores_out
 * [sum M, C] (DEVICE): the cohort scores, optional (NULL: not written).  The enrolled speakers' statistics per problem
 * come from the same entry with fea = enroll_fea and speaker = enroll_speaker repeated G times.  workspace:
 * vbx_cohort_stats_batch_workspace_bytes(G, M, C, N_c) bytes, 256-byte aligned: about 8 sum M C + 1.1 KB (sum M + G C)
 * + 4 G N_c bytes.  Further VBX_ERR_ARG: C < 2, top_k < 2, N_c < 1. */
int vbx_cohort_stats_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, int64_t C, int64_t N_c,
                                           size_t *bytes_out);
int vbx_cohort_stats_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                           const int32_t *speaker, const int64_t *M, const float *cohort_fea, int64_t N_c,
                           const int32_t *cohort_speaker, int64_t C, const double *Fa, const double *Fb, int32_t top_k,
                           void *workspace, size_t workspace_bytes, double *mean_out, double *std_out,
                           double *scores_out, void *stream);

/* Speaker-verification trials (DESIGN.md section 5.27).  Each needs a handle, no plan; stream ordered, no allocation,
 * no host synchronisation; small scalars go to the device in one copy from pageable host memory.
 *
 * vbx_verify_score: T trials, each an enrolment item against a test item.  The enrolment side is enroll_fea [N_e,R]
 * float32 with enroll_item [N_e] int32 in [0, M_e) (-1: none), the test side test_fea [N_t,R] with test_item [N_t] in
 * [0, M_t), Phi [R] (all DEVICE: x-vectors through the front end, R <= 128; every item should own an x-vector).  Each
 * item gets vbx_link_batch's statistics n, F, b, e with c = Fa / Fb (Fa, Fb finite and > 0); pack each item's x-vectors
 * together, as for vbx_link_batch (spread-out items cost up to M N reads).  Trial t = (trial_enroll[t], trial_test[t])
 * (DEVICE int32) writes score_out [T] (DEVICE float64) in trial order:
 *   LLR(i, j) of vbx_link_batch, bit-identical to vbx_enroll_batch's and vbx_cohort_stats_batch's score of the pair
 *   (enrolment item as the row) and to the swapped trial's score with the sides swapped,
 * or with enroll_mean, enroll_std [M_e] and test_mean, test_std [M_t] (DEVICE, all four or none: cohort statistics
 * from vbx_cohort_stats_batch, every std finite and > 0) the AS-norm score
 *   S = 1/2 [ (LLR - enroll_mean[i]) / enroll_std[i] + (LLR - test_mean[j]) / test_std[j] ].
 * A trial whose index lies outside its side scores NaN.  workspace: vbx_verify_score_workspace_bytes(M_e, M_t) bytes,
 * 256-byte aligned: about 1.1 KB per item.  VBX_ERR_ARG: M_e, M_t, N_e or N_t < 1, T < 0, R outside 1 .. 128, a bad
 * Fa or Fb, some but not all of the four statistics, null pointers, a misaligned or short workspace.
 *
 * vbx_verify_metrics: the error rates of T >= 1 scores [T] (DEVICE float64) with is_target [T] (DEVICE uint8, nonzero =
 * target trial) at n_op operating points p_target [n_op] (HOST, each in (0, 1)) with costs c_miss, c_fa (finite, > 0).
 * Candidate thresholds are the distinct scores (-0.0 and +0.0 one value) and +inf; at threshold t a trial is accepted
 * when score >= t, P_miss(t) = #targets below t / N_tar and P_fa(t) = #nontargets at or above t / N_non (exact counts,
 * one float64 division each).  Outputs (DEVICE):
 *   counts_out [3] int64      N_tar, N_non and the number of non-finite scores (the metrics are meaningless then)
 *   eer_out [1]               with k the first candidate where P_miss >= P_fa, a and b = P_miss - P_fa at k - 1 and k:
 *                             P_fa(k-1) + a / (a - b) (P_fa(k) - P_fa(k-1))
 *   min_dcf_out [n_op]        min over the candidates of (c_miss p P_miss + c_fa (1-p) P_fa) / min(c_miss p, c_fa (1-p))
 *   threshold_out [n_op]      the lowest candidate attaining it
 *   act_dcf_out [n_op]        the same cost at the Bayes threshold log(c_fa (1-p) / (c_miss p)), score >= it accepted
 *   cllr_out [1]              1 / (2 ln 2) [mean over targets of softplus(-s) + mean over nontargets of softplus(s)]
 * The metrics need N_tar, N_non >= 1 (NaN otherwise).  The sort is cub::DeviceRadixSort; every reduction runs in a
 * fixed order without floating-point atomics, so a call is bit-identical from run to run and for any order of the trials.
 * workspace: vbx_verify_metrics_workspace_bytes(T, n_op) bytes (the sort's temporary storage included; sized for the
 * handle's device), 256-byte aligned: about 34 T bytes plus the sort's.  VBX_ERR_ARG: T < 1, n_op outside 1 ..
 * VBX_VERIFY_MAX_OPS, a p_target outside (0, 1), bad costs, null pointers, a misaligned or short workspace. */
#define VBX_VERIFY_MAX_OPS 64
int vbx_verify_score_workspace_bytes(vbx_handle_t h, int32_t M_e, int32_t M_t, size_t *bytes_out);
int vbx_verify_score(vbx_handle_t h, const float *enroll_fea, int64_t N_e, const int32_t *enroll_item, int32_t M_e,
                     const float *test_fea, int64_t N_t, const int32_t *test_item, int32_t M_t, int32_t R,
                     const float *Phi, double Fa, double Fb, const int32_t *trial_enroll, const int32_t *trial_test,
                     int64_t T, const double *enroll_mean, const double *enroll_std, const double *test_mean,
                     const double *test_std, void *workspace, size_t workspace_bytes, double *score_out, void *stream);
int vbx_verify_metrics_workspace_bytes(vbx_handle_t h, int64_t T, int32_t n_op, size_t *bytes_out);
int vbx_verify_metrics(vbx_handle_t h, const double *scores, const uint8_t *is_target, int64_t T, int32_t n_op,
                       const double *p_target, double c_miss, double c_fa, void *workspace, size_t workspace_bytes,
                       int64_t *counts_out, double *eer_out, double *cllr_out, double *min_dcf_out,
                       double *threshold_out, double *act_dcf_out, void *stream);

/* vbx_verify_calibrate (DESIGN.md section 5.28): the linear calibration llr = a s + b of T >= 1 scores [T] (DEVICE
 * float64) with is_target [T] (DEVICE uint8, nonzero = target trial) at the prior in (0, 1): (a, b) minimise the
 * prior-weighted logistic cost
 *   C(a, b) = prior / N_tar sum_tar softplus(-z) + (1 - prior) / N_non sum_non softplus(z),  z = a s + b + logit(prior),
 * by Newton's method with step halving from (0, 0) on the device (at most 64 passes; once the predicted decrease is
 * <= 2^-52 C one last full step is taken and the fit ends), and min_cllr is the Cllr of the optimal monotone (PAV) transform of the scores at prior 1/2, from the
 * upper hull of the ROC points of the distinct scores (exact integer arithmetic).  Outputs (DEVICE):
 *   info_out [5] int64    status (0 fitted, 1 separable classes or a missing class: no finite minimiser, the fit is not
 *                         run, 2 non-finite scores, 3 the pass limit reached), passes, N_tar, N_non, hull vertices
 *   out [4] float64       a, b, cllr_prior = C(a, b) / ln 2 (NaN for status 1 and 2), min_cllr (NaN for status 2)
 * Every sum runs in an order fixed by the sorted scores, so a call is bit-identical from run to run and for any order of
 * the trials.  Stream ordered, no allocation, no host synchronisation; a fixed number of launches.  workspace:
 * vbx_verify_calibrate_workspace_bytes(T) bytes (the sort's temporary storage included; sized for the handle's device),
 * 256-byte aligned: about 42 T bytes plus the sort's.  VBX_ERR_ARG: T < 1, a prior outside (0, 1), null pointers, a
 * misaligned or short workspace. */
int vbx_verify_calibrate_workspace_bytes(vbx_handle_t h, int64_t T, size_t *bytes_out);
int vbx_verify_calibrate(vbx_handle_t h, const double *scores, const uint8_t *is_target, int64_t T, double prior,
                         void *workspace, size_t workspace_bytes, int64_t *info_out, double *out, void *stream);

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
/* vbx_run_f64 with the enrolment prior of vbx_run_prior (same formulas, all in float64, with the scalar Fa / Fb):
 * prior_n [n_rec,S], prior_F [n_rec,S,R] float64 DEVICE arrays of this plan's S and R; null arrays return VBX_ERR_ARG.
 * An all-zero prior gives bit-identical results to vbx_run_f64. */
int vbx_run_f64_prior(vbx_handle_t h, void *workspace, size_t workspace_bytes, const double *fea, const double *Phi,
                      double *gamma_io, double *pi_io, const int32_t *n_states, double Fa, double Fb, double loop_prob,
                      int32_t max_iters, double epsilon, double *alpha_io, double *invL_io, int32_t warm_start,
                      double *Li_out, int32_t *n_iters_out, int32_t *flags_out, const double *prior_n,
                      const double *prior_F, void *stream);

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

/* Diagnostic: the per-recording ELBO constant G_b = sum_t -0.5 (sum_r rho_tr^2 / Phi_r + R log 2pi) that the last
 * vbx_prepare_* call computed (the term of VBx/VBx.py:87 that vbx_run adds to every ELBO), copied device to device into
 * gsum_out [n_rec] (float64, device pointer) on `stream`.  A recording with no frames has G_b = 0.
 * VBX_ERR_STATE before a vbx_prepare_* call on the current plan and workspace. */
int vbx_get_gsum(vbx_handle_t h, double *gsum_out, void *stream);

/* per-entry bits written to flags_out by vbx_score, vbx_score_overlap and vbx_score_jer */
enum vbx_score_flag {
    VBX_SCORE_BAD_LABEL = 1,     /* a label outside [0, n_labels[e]) (a second label outside [-1, n_labels[e]) or
                                    equal to the first): that interval was not counted                            */
    VBX_SCORE_BAD_REGION = 2,    /* a region mask names a speaker >= n_ref[rec]: that overlap was not counted    */
    VBX_SCORE_BAD_RECORDING = 4  /* entry_rec[e] outside [0, n_rec), n_ref > 64 or n_ref x n_labels > max_cells:
                                    nothing of the entry was counted (covered 0, fa 0, O not written)             */
};

/* Diarization error rate accumulation (DESIGN.md section 5.11) for many (setting, recording) entries in one launch.
 * Times are int64 microseconds ("ticks").  Per recording r of n_rec (all DEVICE arrays):
 *   sys_offsets [n_rec+1]        the system intervals of r are sys_lo/sys_hi[sys_offsets[r] .. sys_offsets[r+1]-1]:
 *                                one owned interval [lo, hi) per x-vector (empty when hi <= lo)
 *   sys_join_hi                  same layout: where interval i is followed by interval i+1 of the SAME label, it ends at
 *                                sys_join_hi[i] instead of sys_hi[i] (bridges the pauses that the RTTM writer merges;
 *                                sys_join_hi = sys_hi where there is none)
 *   reg_offsets [n_rec+1]        the scored regions of r are reg_lo/reg_hi/reg_mask[reg_offsets[r] .. reg_offsets[r+1]-1]:
 *                                sorted, disjoint [lo, hi) with the bitmask of the active reference speakers (bit k =
 *                                speaker k; 0 = scored non-speech).  Time outside every region is not scored.
 *   n_ref [n_rec]                reference speakers of r, 0 .. 64
 * Per entry e of n_entries:
 *   entry_rec [n_entries]        its recording
 *   label_offsets [n_entries]    labels[label_offsets[e] + i] (int32) is the label of the recording's interval i
 *   n_labels [n_entries]         labels lie in [0, n_labels[e])
 *   o_offsets [n_entries]        its overlap block O_out[o_offsets[e] ..] of n_ref[rec] x n_labels[e] int64 (row = reference
 *                                speaker); blocks of different entries must not overlap
 * Outputs (all written by the call, no zeroing needed): covered_out[e] = scored time in which the system speaks and a
 *   reference speaker is active, fa_out[e] = scored time in which the system speaks over non-speech, O[k, s] = scored time
 *   in which reference speaker k is active while the system says s, flags_out[e] = vbx_score_flag bits.
 * max_cells (HOST): at least the largest n_ref x n_labels of any entry; blocks of up to min(max_cells, 64 x 128) cells
 *   are accumulated in shared memory, larger ones in place in O_out (same results).  O_out may be NULL if max_cells is 0.
 * Integer sums only: results are bit-identical whatever the batch and the launch order.  Needs no plan; does not
 * synchronise with the host.  VBX_ERR_ARG for negative counts, max_cells < 0 or null pointers. */
int vbx_score(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo, const int64_t *sys_hi,
              const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo, const int64_t *reg_hi, const uint64_t *reg_mask,
              const int32_t *n_ref, int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets,
              const int32_t *labels, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
              int64_t *covered_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, void *stream);

/* Overlap-aware DER accumulation (DESIGN.md section 5.12): vbx_score with a second system label per interval, counted
 * inside overlap regions only.  Arguments as for vbx_score, plus (DEVICE arrays):
 *   reg_overlap [same layout as reg_lo]  1 where the region lies inside the recording's overlap regions, else 0 (the
 *                                        caller splits the scored regions at the overlap boundaries)
 *   labels2 [same layout as labels]      the interval's second label, -1 = none; otherwise in [0, n_labels[e]) and
 *                                        different from labels[] of the same interval
 * Stream 1 is vbx_score's output.  Stream 2 is interval i saying labels2[i] from its lo to sys_join_hi[i] where interval
 * i+1 has the same second label (sys_hi[i] elsewhere), in regions with reg_overlap set.  Over scored time with N_ref
 * reference speakers and N_sys in {0, 1, 2} system labels:
 *   both_out[e] = sum of min(N_ref, N_sys) x time, fa_out[e] = sum of max(0, N_sys - N_ref) x time,
 *   O[k, s] = scored time in which reference speaker k is active while the system says s in either stream.
 * With no reg_overlap set, or labels2 all -1, the results equal vbx_score's (both_out = covered_out).  A second label
 * outside [-1, n_labels[e]) or equal to the first sets VBX_SCORE_BAD_LABEL (that interval is not counted).
 * Integer sums only: results are bit-identical whatever the batch and the launch order.  VBX_ERR_ARG as for vbx_score. */
int vbx_score_overlap(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo,
                      const int64_t *sys_hi, const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo,
                      const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_overlap, const int32_t *n_ref,
                      int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets, const int32_t *labels,
                      const int32_t *labels2, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
                      int64_t *both_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, void *stream);

/* DER accumulation plus the per-label time that the Jaccard error rate needs (DESIGN.md section 5.13).  Arguments and
 * outputs as for vbx_score_overlap; reg_overlap and labels2 may both be NULL for single-label entries (then everything
 * vbx_score writes is written, bit-identical to it).  Plus:
 *   t_offsets [n_entries] (DEVICE)   label_time_out[t_offsets[e] ..] is entry e's block of n_labels[e] int64; blocks of
 *                                    different entries must not overlap
 *   label_time_out (DEVICE, output)  S[s] = scored time in which the system says label s, in either stream (a label is
 *                                    never said twice at one instant: labels2 differs from labels), non-speech included.
 * Blocks of up to 128 labels are accumulated in shared memory, larger ones in place in label_time_out (same results).
 * An entry flagged VBX_SCORE_BAD_RECORDING leaves its label-time block unwritten.  For the Jaccard error rate the
 * scored regions are those of collar 0 with overlaps scored: O[k, s] is then |ref_k intersect sys_s|.
 * Integer sums only: results are bit-identical whatever the batch and the launch order.  VBX_ERR_ARG as for vbx_score,
 * and when only one of reg_overlap and labels2 is NULL. */
int vbx_score_jer(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo,
                  const int64_t *sys_hi, const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo,
                  const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_overlap, const int32_t *n_ref,
                  int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets, const int32_t *labels,
                  const int32_t *labels2, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
                  int64_t *both_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, const int64_t *t_offsets,
                  int64_t *label_time_out, void *stream);

/* per-recording bits written to flags_out by vbx_combine */
enum vbx_combine_flag {
    VBX_COMBINE_BAD_LABEL = 1,       /* a label of some hypothesis outside [-1, n_labels), a second label without a
                                        first or equal to it: that interval of that hypothesis counted as silent   */
    VBX_COMBINE_TOO_MANY_LABELS = 2  /* more than 255 global labels: n_global 0, every output label of the recording
                                        -1, its map rows incomplete                                                */
};

/* Combination of K diarizations of the same intervals into one by label mapping and weighted voting (DESIGN.md section
 * 5.21; DOVER with up to two labels per interval), many recordings per call; needs a handle, no plan.
 * Times are int64 microseconds ("ticks").  DEVICE arrays unless marked HOST:
 *   offsets [n_rec+1]            recording r owns intervals offsets[r] .. offsets[r+1]-1 of the N = offsets[n_rec] packed
 *                                ones (N is passed on the host as well)
 *   lo, hi [N]                   interval i is [lo, hi), sorted and disjoint inside a recording; empty when hi <= lo
 *   labels, labels2 [K, N] int32 row k: hypothesis k's first and second label of every interval, -1 = none
 *   n_labels [n_rec, K] (HOST)   hypothesis k's labels in recording r lie in [-1, n_labels[r, k]); 0 <= it <= max_labels
 *   max_labels (HOST)            1 .. 128: the row length of the O and L blocks
 *   weights [K] (HOST) or NULL   w_k, finite and > 0; NULL: rank ** -0.1 by ascending summed disagreement
 * Per recording: O_ab[s, u] = ticks in which hypothesis a says s and b says u (either stream), L_a[s] = ticks in which a
 * says s; D[a, b] = sum L_a + sum L_b - 2 x the maximum one-to-one matching of O_ab; the hypotheses ordered by their row
 * sum of D (ties: the lower index), the first being the anchor; global labels = the anchor's labels with time, then
 * every later hypothesis in that order assigned one-to-one to the global labels by the ticks it shares with the labels
 * already mapped to them (no pair without shared ticks; its unmatched labels with time get new ids in label order);
 * per interval n = floor(0.5 + sum_k w_k c_k / sum_k w_k) labels are kept (c_k = labels hypothesis k gives it), those
 * of largest summed weight, ties to the lower global id.  Outputs:
 *   labels_out, labels2_out [N] int32        the combined first and second global label, -1 = none
 *   order_out [n_rec, K] int32               hypotheses by rank (order_out[r, 0] is the anchor)
 *   weights_out [n_rec, K]                   w_k by hypothesis index
 *   D_out [n_rec, K, K] int64                the disagreements, symmetric, zero diagonal
 *   map_out [n_rec, K, 128] int32            the global label of label s of hypothesis k, -1 for a label without time
 *   n_global_out [n_rec] int32, flags_out [n_rec] int32 (vbx_combine_flag bits)
 *   O_out [n_rec, K (K-1)/2, max_labels, max_labels], L_out [n_rec, K, max_labels] int64: optional (NULL: kept in the
 *     workspace); pair (a, b), a < b, is block a (2 K - a - 1) / 2 + b - a - 1, rows = a's labels
 * Integer sums and fixed-order float64 sums: a recording's outputs are bit-identical whatever else shares the call.
 * Where an assignment has several optima the one returned is that of shortest augmenting paths over the rows in label
 * order with ties in a step going to the lowest column (global ids before "unmatched").
 * workspace: vbx_combine_workspace_bytes(n_rec, K, max_labels) bytes, 256-byte aligned.  Stream ordered, no allocation,
 * no host synchronisation: n_labels goes to the device in one copy from pageable host memory.  VBX_ERR_ARG: null
 * pointers, K outside 2..32, negative counts, max_labels outside 1..128, an n_labels outside [0, max_labels], a weight
 * that is not finite and > 0, n_rec (K (K-1)/2 + K) above 2^31 - 1, a short or misaligned workspace. */
int vbx_combine_workspace_bytes(vbx_handle_t h, int32_t n_rec, int32_t K, int32_t max_labels, size_t *bytes_out);
int vbx_combine(vbx_handle_t h, int32_t n_rec, const int64_t *offsets, int64_t N, const int64_t *lo, const int64_t *hi,
                int32_t K, const int32_t *labels, const int32_t *labels2, const int32_t *n_labels, int32_t max_labels,
                const double *weights, void *workspace, size_t workspace_bytes, int32_t *labels_out,
                int32_t *labels2_out, int32_t *order_out, double *weights_out, int64_t *D_out, int32_t *map_out,
                int32_t *n_global_out, int32_t *flags_out, int64_t *O_out, int64_t *L_out, void *stream);

/* Class statistics for training the x-vector transform and the PLDA (DESIGN.md section 5.24).  Needs a handle, no plan.
 *   X [N, D] float32 DEVICE, contiguous, 16-byte aligned base (may be NULL when N = 0); rows packed by class, D in
 *     1 .. 1024
 *   offsets [K+1] int64 HOST: class i is rows offsets[i] .. offsets[i+1] - 1; from 0 to N, not decreasing; empty
 *     classes are allowed (mean row 0, no contribution)
 * Outputs (DEVICE, float64):
 *   means_out [K, D]     m_i = the float64 mean of class i's rows
 *   scatter_out [D, D]   sum over rows r of (x_r - m_class(r)) (x_r - m_class(r))^T; both triangles, mirror images bit
 *                        for bit
 * Rows are centred by their float64 class mean before the products, which accumulate on the FP64 tensor cores (DMMA)
 * over the tiles on or above the diagonal only.  Partial tiles of row splits (their number a function of N and D) are
 * summed in a fixed order without atomics: a call is bit-identical from run to run and independent of what the
 * workspace held.  workspace: vbx_class_scatter_workspace_bytes(N, D, K) bytes, 256-byte aligned: about 8 K + 4 N bytes
 * plus 32 KB per (split, tile pair), at most about 36 MB of partial tiles.  Stream ordered, no allocation, no host
 * synchronisation beyond the one copy of offsets from pageable host memory.  VBX_ERR_ARG: null pointers, D outside
 * 1 .. 1024, K < 1, N < 0, offsets not from 0 to N or decreasing, a misaligned X or workspace, a short workspace. */
int vbx_class_scatter_workspace_bytes(vbx_handle_t h, int64_t N, int32_t D, int32_t K, size_t *bytes_out);
int vbx_class_scatter(vbx_handle_t h, const float *X, int64_t N, int32_t D, int32_t K, const int64_t *offsets,
                      void *workspace, size_t workspace_bytes, double *means_out, double *scatter_out, void *stream);

/* Streaming diarization (DESIGN.md section 5.25): live streams diarized block by block, each stream's speakers carried
 * into the VB-HMM as priors.  Needs a handle, no plan.  The state of every stream lives in DEVICE memory that the
 * caller owns, one row per slot:
 *   ctx_fea [slots, C, R] float32, ctx_lab [slots, C] int32   a ring of the stream's last min(C, count) projected
 *                                                             x-vectors and their final labels; x-vector g (0-based,
 *                                                             in push order) sits at position g mod C
 *   count [slots] int64                                       x-vectors pushed so far
 *   K [slots] int32                                           speakers so far (labels 0 .. K-1)
 *   n_hist [slots, S_max] float64, F_hist [slots, S_max, R]   per speaker, the number and the feature sum of the
 *     float64                                                 x-vectors that have left the ring, summed in time order
 * A fresh slot is all zero.  A push delivers blocks of h >= 1 new x-vectors to n streams with DISTINCT slots; all the
 * per-stream arrays below are DEVICE arrays in push order:
 *   slot [n] int32                  the stream's slot
 *   blk_off [n+1] int64             its block is rows blk_off[i] .. blk_off[i+1]-1 of blk_fea [*, R] float32 (projected)
 *   win_off [n+1] int64             its window is rows win_off[i] .. win_off[i+1]-1, min(C, count) + h of them
 *   blk_lab [*] int32, n_clusters [n] int32   the block's clusters 0 .. c-1 and c, with K + c <= S_max and K + c <= S
 *                                   (c = 0 when K = S_max: the block rows then start uniform over the K states)
 * These contents are read on the device and not validated.
 * vbx_stream_window writes, at the tier's S (the window plan's padded state count):
 *   fea_out [Nw, R] float32         [context rows, oldest first; block rows]
 *   gamma_out [Nw, S] float32       softmax(smoothing * onehot(label)) over the K + c states, 0 in the other columns;
 *                                   a context row's label is its final label, block row t's is K + blk_lab[t]; evaluated
 *                                   in float64 and rounded once
 *   pi_out [n, S] float32           1 / (K + c) in the first K + c columns, 0 in the others
 *   n_states_out [n] int32          K + c
 *   prior_n_out [n, S], prior_F_out [n, S, R] float64   n_hist, F_hist for the states k < K, 0 for the others
 * vbx_stream_commit takes first [Nw] int32, the window's first labels (vbx_hard_labels on the window plan), and writes
 * labels_out [*] int32, the block's final labels on blk_off: a block row on a state k < K is speaker k, and the fresh
 * states that hold block rows become speakers K, K+1, ... in order of their first row.  It then adds the rows that
 * leave the ring (the oldest first) to n_hist / F_hist, one sequential float64 sum per (slot, state, feature) without
 * atomics, writes the block into the ring and advances count and K.  Context rows are never relabelled.  A stream's
 * results are bit-identical from run to run, whatever the outputs held before and whatever else the push carries.
 * Stream ordered, no allocation, no host synchronisation.  VBX_ERR_ARG: a null pointer, n < 0, C < 0, R outside
 * 1 .. 128, S_max or S outside 1 .. 128. */
int vbx_stream_window(vbx_handle_t h, int32_t n, int32_t C, int32_t R, int32_t S_max, int32_t S, const int32_t *slot,
                      const int64_t *blk_off, const int64_t *win_off, const int32_t *blk_lab, const int32_t *n_clusters,
                      const float *blk_fea, double smoothing, const float *ctx_fea, const int32_t *ctx_lab,
                      const int64_t *count, const int32_t *K, const double *n_hist, const double *F_hist, float *fea_out,
                      float *gamma_out, float *pi_out, int32_t *n_states_out, double *prior_n_out, double *prior_F_out,
                      void *stream);
int vbx_stream_commit(vbx_handle_t h, int32_t n, int32_t C, int32_t R, int32_t S_max, const int32_t *slot,
                      const int64_t *blk_off, const int64_t *win_off, const float *blk_fea, const int32_t *first,
                      float *ctx_fea, int32_t *ctx_lab, int64_t *count, int32_t *K, double *n_hist, double *F_hist,
                      int32_t *labels_out, void *stream);

/* Enrolled speakers in streams (DESIGN.md section 5.29), called after a push's vbx_stream_commit.  The enrolment state
 * is one more DEVICE array the caller owns beside the stream state: named [slots, S_max] int32, the enrolled speaker
 * (0 .. E-1) each stream speaker is named by, or -1 (a fresh slot is all -1).  The enrolled speakers' statistics
 * n_enroll [E], F_enroll [E, R] float64 (DEVICE) are vbx_enroll_batch's n_enroll_out / F_enroll_out.  The candidates
 * are HOST arrays: n streams with distinct slot [n] in [0, slots), each with cand_off[i+1] - cand_off[i] >= 1 distinct
 * speakers cand_k [M] in [0, S_max) (M = cand_off[n]), packed in stream order; they should be the stream's unnamed
 * speakers (named = -1, k < K) that hold rows of the push (not validated: read on the device).  For every candidate:
 *   n = n_hist[k] + ring rows labelled k, F = F_hist[k] + those rows (oldest first, one sequential float64 sum), and
 *   b, e of vbx_link_batch with c = Fa / Fb; the LLR against every enrolled speaker (section 5.15's score, the kernel of
 *   vbx_enroll_batch: bit-identical to its llr for the same statistics); -inf for the enrolled speakers the stream
 *   has already named a speaker by; then each stream's candidates are assigned one-to-one as vbx_enroll_batch assigns
 *   a recording's speakers at `threshold`.
 * Outputs (DEVICE): assign_out [M] int32 the enrolled index or -1; best_llr_out [M] the assigned pair's LLR, or for an
 * unassigned candidate its largest LLR over the enrolled speakers the stream has not claimed (-inf when it claimed
 * them all); optional (null: not written) llr_out [M, E] the LLRs before the claimed ones are masked, n_out [M],
 * F_out [M, R].  Then named[slot, k] = assign for every assigned candidate and, with prior = 1, n_hist[slot, k] +=
 * n_enroll[a], F_hist[slot, k] += F_enroll[a].  A stream's results do not depend on the rest of the batch.
 * workspace: vbx_stream_enroll_workspace_bytes(n, M, E, max_k) bytes, max_k >= the largest candidate count of a
 * stream, 256-byte aligned.  Stream ordered, no allocation, no host synchronisation beyond one copy of the candidate
 * lists from pageable host memory.  VBX_ERR_ARG: a null pointer, sizes as vbx_stream_commit's, slots < n, E < 1,
 * |threshold| > 1e15, Fa / Fb not finite and >= 0, prior not 0 / 1, candidate lists as above violated, a misaligned or
 * short workspace. */
int vbx_stream_enroll_workspace_bytes(vbx_handle_t h, int32_t n, int64_t M, int64_t E, int32_t max_k,
                                      size_t *bytes_out);
int vbx_stream_enroll(vbx_handle_t h, int32_t n, int32_t slots, int32_t C, int32_t R, int32_t S_max,
                      const int32_t *slot, const int64_t *cand_off, const int32_t *cand_k, const float *Phi, double Fa,
                      double Fb, const float *ctx_fea, const int32_t *ctx_lab, const int64_t *count, double *n_hist,
                      double *F_hist, int32_t *named, const double *n_enroll, const double *F_enroll, int64_t E,
                      double threshold, int32_t prior, void *workspace, size_t workspace_bytes, int32_t *assign_out,
                      double *best_llr_out, double *llr_out, double *n_out, double *F_out, void *stream);

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
    VBX_K_EM_CONTRACT = 8,   /* M-step + speaker model + log_p_ in one cluster kernel (large batches) */
    VBX_N_KERNEL_CLASSES = 9
};
/* With option "timing" = 1 every kernel class is bracketed by CUDA events on the launching stream.
 * Fills ms_out[VBX_N_KERNEL_CLASSES] / count_out[...] with the accumulated device time and launch counts
 * (HOST arrays; synchronises on the recorded events); reset != 0 clears the accumulators. */
int vbx_get_timings(vbx_handle_t h, double *ms_out, int64_t *count_out, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* VBX_B200_H */
