// Internal declarations shared by the kernel translation units and the C ABI (not installed).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#define VBX_EPS_TR 1e-8f  // additive floor inside the HMM logs of the reference, VBx/VBx.py:158

namespace vbx {

constexpr int kLTile = 64;    // frames per CTA tile of the log-likelihood kernel
constexpr int kMTile = 512;   // frames per CTA tile of the M-step accumulation / mma log-likelihood kernels
constexpr int kLongT = 4096;   // recordings at least this long take the chunked-scan forward-backward
constexpr int kChunk = 256;    // frames per chunk of that scan
constexpr int kMaxR = 128;
constexpr int kMaxS = 64;
constexpr int kTcMaxD = 2048;  // largest raw dimension of the tensor-core front end (bounds its scratch in the workspace)

// Device-resident description of a planned batch (arrays owned by the handle).
struct Plan {
    int32_t n_rec = 0, R = 0, S = 0;
    int32_t exact = 0;                  // 1 = the workspace holds the buffers of the float64 finishing phase
    int32_t split = 0;                  // 1 = forward and backward sweeps on separate warps + combine pass (vbx_fb_split.cu)
    int64_t n_frames = 0;
    int32_t n_ltiles = 0, n_mtiles = 0;
    int64_t max_T = 0;
    const int64_t *offsets = nullptr;   // [n_rec+1]
    const int32_t *order = nullptr;     // [n_rec] recordings sorted by length, longest first
    const int32_t *ltile_rec = nullptr; // [n_ltiles]
    const int64_t *ltile_f0 = nullptr;  // [n_ltiles] first (global) frame of the tile
    const int32_t *mtile_rec = nullptr; // [n_mtiles]
    const int64_t *mtile_f0 = nullptr;  // [n_mtiles]
    const int32_t *mtile_begin = nullptr; // [n_rec+1] first M-tile of each recording
    // long recordings (T >= kLongT): chunked-scan forward-backward (vbx_long_kernels.cu)
    int32_t n_lrec = 0, n_lchunks = 0;
    const int32_t *lrec_list = nullptr;    // [n_lrec]   recording ids
    const int32_t *lrec_first = nullptr;   // [n_rec]    first chunk index of the recording (long ones only)
    const int32_t *lrec_nchunks = nullptr; // [n_rec]    number of chunks, 0 for short recordings
    const int32_t *lchunk_rec = nullptr;   // [n_lchunks]
    const int32_t *lchunk_idx = nullptr;   // [n_lchunks] chunk number inside its recording
};

// Caller-provided workspace, carved by the handle.
struct Workspace {
    float *p = nullptr;        // [N,S]  exp(ll - rowmax)
    float *rowmax = nullptr;   // [N]
    float *rsigma = nullptr;   // [N]    1 / forward scale
    float *cvec = nullptr;     // [N]    c_t = sum_j p[t,j] w_j, w = (1-loopP) pi + 1e-8: the one reduction of the look-ahead
                               //        sweeps that does not depend on the recursion, taken out of them (written by loglik)
    float *partial = nullptr;  // [n_mtiles,S,R] per-tile gamma^T rho
    float *A = nullptr;        // [n_rec,S,R]  Fa * alpha
    float *Afrag_hi = nullptr; // [n_rec,NT,KS,32] float2: Fa*alpha split to TF32 hi/lo, mma fragment-major
    float *Afrag_lo = nullptr; //   (NT = max(1,S/8) n-tiles, KS = ceil(R/8) k-steps; see vbx_mma_kernels.cu)
    float *bias = nullptr;     // [n_rec,S]    Fa * 0.5 * sum_r (invL + alpha^2) Phi_r ; +inf for dead columns
    float *occ = nullptr;      // [n_rec,S]    N_s = sum_t gamma
    double *regp = nullptr;    // [n_rec,S]    per speaker: sum_r (log invL - invL - alpha^2 + 1)
    double *gsum = nullptr;    // [n_rec]      sum_t G_t
    double *gpart = nullptr;   // [n_mtiles]
    double *prev_elbo = nullptr; // [n_rec]
    int32_t *active = nullptr; // [n_rec]  1 = the recording is iterating in the float32 kernels
    int32_t *tile_done = nullptr; // [n_rec] M-tiles of the running M-step finished so far (last one computes the speaker model)
    // float64 finishing phase (vbx_exact64.cu); null when the plan was made with option "exact_stop" = 0
    int32_t *active64 = nullptr; // [n_rec] 1 = iterating in the float64 kernels
    int32_t *fresh = nullptr;    // [n_rec] 1/2 = the next float64 iteration is the recording's first (restore the snapshot);
                                 //         1: its stop test is already decided (no stop), 2: test against the float32 ELBO
    float *gamma_snap = nullptr; // [2][N,S]   gamma at the start of float32 iteration i lives in slot i % 2
    float *pi_snap = nullptr;    // [2][n_rec,S]
    double *p64 = nullptr;       // [N,S]
    double *rowmax64 = nullptr;  // [N]
    double *rsig64 = nullptr;    // [N]
    double *partial64 = nullptr; // [n_mtiles,S,R]
    double *occp64 = nullptr;    // [n_mtiles,S]
    double *alpha64 = nullptr;   // [n_rec,S,R]
    double *bias64 = nullptr;    // [n_rec,S]
    double *reg64 = nullptr;     // [n_rec]
    double *pi64 = nullptr;      // [n_rec,S]
    float *scratch = nullptr;  // [2*kMaxS] write sink for warp lanes that own no recording
    // split forward-backward (vbx_fb_split.cu); null unless the plan chose it
    float *ahat = nullptr, *bhat = nullptr;   // [N,S] normalised forward variables / self-scaled backward variables
    float *socc = nullptr, *sent = nullptr;   // [n_mtiles,S] per-tile sums of gamma / of the re-entry terms of eq. (24)
    float *tc_scratch = nullptr; // operand images of the tensor-core front end (vbx_project_tc.cu); null unless R == 128
    // chunked scan of long recordings: per (chunk, basis) operators and per-chunk boundary vectors / partial sums
    float *fa_u = nullptr, *fa_lam = nullptr, *fa_exp = nullptr, *astart = nullptr;   // [LC,S,S], [LC,S] mantissa, [LC,S] exponent, [LC,S]
    float *bb_v = nullptr, *bb_mu = nullptr, *bb_exp = nullptr, *beta = nullptr;      // same shapes, backward sweep
    float *occp = nullptr, *entp = nullptr;                        // [n_lchunks,S]
};

struct RunParams {
    float Fa, Fb, FaFb, loopP;
    double dFa, dFb, dFaFb, dloopP, epsilon;
    int32_t max_iters;
    // stop rule at float64 resolution (vbx_exact64.cu): a recording leaves the float32 kernels when its ELBO step is
    // below epsilon + guard_mult * nb, nb = noise_c * 2^-24 * |ELBO| (bound on the float32 noise of an ELBO difference)
    int32_t hybrid, warm;
    double noise_c, guard_mult;
};

#ifdef __CUDACC__
// small vector load/store helpers shared by the kernel translation units
template <int N>
struct Vec {
    float v[N];
};
template <int N>
__device__ __forceinline__ Vec<N> ld_vec(const float *p);
template <>
__device__ __forceinline__ Vec<1> ld_vec<1>(const float *p) {
    Vec<1> r;
    r.v[0] = *p;
    return r;
}
template <>
__device__ __forceinline__ Vec<2> ld_vec<2>(const float *p) {
    float2 t = *reinterpret_cast<const float2 *>(p);
    Vec<2> r;
    r.v[0] = t.x;
    r.v[1] = t.y;
    return r;
}
template <>
__device__ __forceinline__ Vec<4> ld_vec<4>(const float *p) {
    float4 t = *reinterpret_cast<const float4 *>(p);
    Vec<4> r;
    r.v[0] = t.x;
    r.v[1] = t.y;
    r.v[2] = t.z;
    r.v[3] = t.w;
    return r;
}
template <int N>
__device__ __forceinline__ Vec<N> ldg_vec(const float *p);
template <>
__device__ __forceinline__ Vec<1> ldg_vec<1>(const float *p) {
    Vec<1> r;
    r.v[0] = __ldg(p);
    return r;
}
template <>
__device__ __forceinline__ Vec<2> ldg_vec<2>(const float *p) {
    float2 t = __ldg(reinterpret_cast<const float2 *>(p));
    Vec<2> r;
    r.v[0] = t.x;
    r.v[1] = t.y;
    return r;
}
template <>
__device__ __forceinline__ Vec<4> ldg_vec<4>(const float *p) {
    float4 t = __ldg(reinterpret_cast<const float4 *>(p));
    Vec<4> r;
    r.v[0] = t.x;
    r.v[1] = t.y;
    r.v[2] = t.z;
    r.v[3] = t.w;
    return r;
}
template <int N>
__device__ __forceinline__ void st_vec(float *p, const float *v);
template <>
__device__ __forceinline__ void st_vec<1>(float *p, const float *v) {
    *p = v[0];
}
template <>
__device__ __forceinline__ void st_vec<2>(float *p, const float *v) {
    *reinterpret_cast<float2 *>(p) = make_float2(v[0], v[1]);
}
template <>
__device__ __forceinline__ void st_vec<4>(float *p, const float *v) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

#endif  // __CUDACC__

// launchers (vbx_kernels.cu); each returns the number of kernels launched or -1 on launch error
int launch_prepare_scale(const Plan &pl, const Workspace &ws, const float *fea, const float *Phi, float *rho,
                         cudaStream_t st);
int launch_project_ffma(const Plan &pl, const float *X, int D, const float *V, float *rho, cudaStream_t st);
int launch_g_from_rho(const Plan &pl, const Workspace &ws, const float *rho, const float *Phi, cudaStream_t st);
int launch_run_init(const Plan &pl, const Workspace &ws, const float *gamma, const int32_t *n_states, double *Li,
                    int32_t *n_iters, int32_t *flags, int max_iters, cudaStream_t st);
int launch_mstep_partial(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, cudaStream_t st);
int launch_speaker_model(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *Phi,
                         const int32_t *n_states, float *alpha_io, float *invL_io, bool from_given,
                         cudaStream_t st);
int launch_loglik(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states, float loopP,
                  cudaStream_t st);
int launch_forward_backward(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                            const int32_t *n_states, double *Li, int32_t *n_iters, int32_t *flags, int iter,
                            int spl, int classic, cudaStream_t st);
int launch_elbo_trace(const Plan &pl, const double *Li, int max_iters, double *out, cudaStream_t st);
// forward and backward sweeps on separate warps + combine pass, any recording length (vbx_fb_split.cu)
int launch_forward_backward_split(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                  const int32_t *n_states, int spl, cudaStream_t st);
// chunked-scan forward-backward for long recordings (vbx_long_kernels.cu)
int launch_forward_backward_long(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                 const int32_t *n_states, cudaStream_t st);
// tensor-core (mma.sync 3xTF32) versions of the two in-loop contractions (vbx_mma_kernels.cu)
int launch_mstep_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, bool fold, const RunParams &rp,
                     const float *Phi, const int32_t *n_states, float *alpha_io, float *invL_io, cudaStream_t st);
int launch_loglik_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states, float loopP,
                      cudaStream_t st);
// float64 finishing phase of vbx_run (vbx_exact64.cu)
int launch_snapshot(const Plan &pl, const Workspace &ws, const float *gamma, const float *pi, int iter, cudaStream_t st);
int launch_exact64_round(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *rho, const float *Phi,
                         float *gamma, float *pi, const int32_t *n_states, float *alpha_io, float *invL_io, double *Li,
                         int32_t *n_iters, int32_t *flags, cudaStream_t st);
// float64 "exact" path (vbx_f64.cu)
size_t f64_workspace_bytes(const Plan &pl);
int launch_run_f64(const Plan &pl, void *workspace, const double *fea, const double *Phi, double *gamma, double *pi,
                   const int32_t *n_states, double Fa, double Fb, double loopP, int max_iters, double epsilon,
                   double *alpha_io, double *invL_io, int warm, double *Li, int32_t *n_iters, int32_t *flags,
                   cudaStream_t st);
int launch_hard_labels(const Plan &pl, const float *gamma, const int32_t *n_states, int32_t *first, int32_t *second,
                       cudaStream_t st);
// reference-module forward_backward() for a general transition matrix (vbx_fb_dense.cu)
int launch_fb_dense(const double *lls, const double *tr, const double *ip, int T, int S, double *post, double *tll,
                    double *lfw, double *lbw, cudaStream_t st);
// AHC initialisation (vbx_ahc.cu)
size_t ahc_workspace_bytes(const int64_t *offsets_host, int n_rec, std::vector<int64_t> *d_off_host);
int launch_ahc(const Plan &pl, const std::vector<int64_t> &d_off, const void *x, int x_is_f64, int dim, void *workspace,
               size_t workspace_bytes, double *Z_out, double *thr_out, cudaStream_t st, std::string *err);
// wgmma projection (vbx_project_tc.cu)
size_t tc_scratch_floats();
int launch_project_wgmma(const Plan &pl, float *tc_scratch, const float *X, int D, const float *V, const float *Phi, float *rho,
                         float *gframe, cudaStream_t st, std::string *err);
int launch_xvector_chain_wgmma(const Plan &pl, float *tc_scratch, const float *x_raw, int Dx, const float *mean1, const float *lda,
                               const float *mean2, const float *plda_mu, const float *plda_tr, const float *psi,
                               float *x_norm, float *rho, float *gframe, cudaStream_t st, std::string *err);
int launch_gsum_from_frames(const Plan &pl, const Workspace &ws, const float *gframe, cudaStream_t st);

}  // namespace vbx
