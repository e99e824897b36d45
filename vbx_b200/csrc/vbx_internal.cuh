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
// The wide tier: 65 .. 128 live states run as S = 128 plans, always on the split forward-backward schedule
// (vbx_fb_split.cu).  Buffers sized by kMaxS keep their size for S <= 64; the S = 128 instantiations size theirs by S.
constexpr int kMaxSWide = 128;
constexpr int kTcMaxD = 2048;  // largest raw dimension of the tensor-core front end (bounds its scratch in the workspace)

// Device-resident description of a planned batch (arrays owned by the handle).
struct Plan {
    int32_t n_rec = 0, R = 0, S = 0;
    int32_t exact = 0;                  // 1 = the workspace holds the buffers of the float64 finishing phase
    int32_t split = 0;                  // 1 = forward and backward sweeps on separate warps + combine pass (vbx_fb_split.cu)
    int32_t em_cluster = 0;             // > 0: cluster size of em_contract_kernel, which then runs the iteration's
                                        // M-step, speaker model and log-likelihood (vbx_em_contract.cu); 0 = three kernels
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

// The VB-HMM hyperparameters of one recording, derived from the double inputs by run_init_kernel exactly as vbx_run
// derived its batch-wide scalars before they became per recording: a scalar run and a per-recording run with equal
// values do bit-identical arithmetic.
struct RecParams {
    float Fa, Fb, FaFb, loopP;
    double dFa, dFb, dFaFb, dloopP;
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
    float *scratch = nullptr;  // [2*max(S,kMaxS)] write sink for warp lanes that own no recording
    // split forward-backward (vbx_fb_split.cu); null unless the plan chose it
    float *ahat = nullptr, *bhat = nullptr;   // [N,S] normalised forward variables / self-scaled backward variables
    float *socc = nullptr, *sent = nullptr;   // [n_mtiles,S] per-tile sums of gamma / of the re-entry terms of eq. (24)
    float *tc_scratch = nullptr; // operand images of the tensor-core front end (vbx_project_tc.cu); null unless R == 128
    // chunked scan of long recordings: per (chunk, basis) operators and per-chunk boundary vectors / partial sums
    float *fa_u = nullptr, *fa_lam = nullptr, *fa_exp = nullptr, *astart = nullptr;   // [LC,S,S], [LC,S] mantissa, [LC,S] exponent, [LC,S]
    float *bb_v = nullptr, *bb_mu = nullptr, *bb_exp = nullptr, *beta = nullptr;      // same shapes, backward sweep
    float *occp = nullptr, *entp = nullptr;                        // [n_lchunks,S]
    RecParams *hp = nullptr;   // [n_rec]  hyperparameters, filled by run_init_kernel from the scalars or arrays of the call
};

// Batch-wide run settings (the hyperparameters Fa, Fb, loopP are per recording: Workspace::hp).
struct RunParams {
    double epsilon;
    int32_t max_iters;
    int32_t hybrid, warm;   // hybrid: the stop rule at float64 resolution (vbx_exact64.cu)
};
// Stop rule at float64 resolution: a recording leaves the float32 kernels when its ELBO step is below
// epsilon + kStopGuardMult * nb, nb = kStopNoiseC * 2^-24 * |ELBO| (bound on the float32 noise of an ELBO difference).
constexpr double kStopNoiseC = 2.0;
constexpr double kStopGuardMult = 16.0;

// Lets `kernel` launch with up to `bytes` of dynamic shared memory on the current device.  The attribute belongs to the
// device's context, not to the process, so it is set once per (kernel, device) that has not yet been given `bytes`
// (thread-safe).  False when the runtime refuses; its error is left for cudaGetLastError.
bool allow_dynamic_smem(const void *kernel, int bytes);
template <class... Args>
bool allow_dynamic_smem(void (*kernel)(Args...), int bytes) {
    return allow_dynamic_smem(reinterpret_cast<const void *>(kernel), bytes);
}

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

// mbarrier and bulk-copy (cp.async.bulk) primitives of the shared-memory pipelines (vbx_project_tc.cu, vbx_kernels.cu)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// raise the expected transaction bytes of the current phase without arriving
__device__ __forceinline__ void mbar_add_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

// mma.sync.m16n8k8 TF32 and the hi/lo split of the "3xTF32" contractions (vbx_mma_kernels.cu, vbx_em_contract.cu)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t b0, const uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// x = hi + lo.  hi = x rounded to nearest TF32 (add half an ulp of the 13 dropped bits, then clear them: ties
// away from zero, i.e. cvt.rna.tf32.f32, on the integer pipe); lo = x - hi is exact and is handed to the tensor
// core as is (it keeps lo's top 19 bits), so |x - hi - lo'| <= 2^-22 |x| with errors of either sign.
// The rounding is a volatile asm so that the compiler keeps each split next to the mma that consumes it (volatile
// asms are not reordered among themselves); hoisting all splits of a tile up front doubles the register footprint.
__device__ __forceinline__ void split_tf32(const float x, uint32_t &hi, uint32_t &lo) {
    asm volatile("{\n\t.reg .b32 t;\n\tadd.u32 t, %1, 0x1000;\n\tand.b32 %0, t, 0xffffe000;\n\t}" : "=r"(hi) : "r"(__float_as_uint(x)));
    lo = (__float_as_uint(x - __uint_as_float(hi)) + 0x1000u) & 0xffffe000u;
}
template <int LANES>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// The problem g whose range [pref[g], pref[g+1]) holds x, for non-decreasing pref with pref[0] = 0 <= x < pref[G]:
// the largest g with pref[g] <= x (never an empty problem's, whose range is empty).  The batched speaker kernels
// (vbx_link_batch, vbx_enroll_batch, vbx_cohort_stats_batch) decode their flat indices with it.
__device__ __forceinline__ int find_problem(const int64_t *__restrict__ pref, int G, int64_t x) {
    int lo = 0, hi = G;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (pref[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

#endif  // __CUDACC__

// launchers (vbx_kernels.cu); each returns the number of kernels launched or -1 on launch error
int launch_prepare_scale(const Plan &pl, const Workspace &ws, const float *fea, const float *Phi, float *rho,
                         cudaStream_t st);
int launch_project_ffma(const Plan &pl, const float *X, int D, const float *V, float *rho, cudaStream_t st);
int launch_g_from_rho(const Plan &pl, const Workspace &ws, const float *rho, const float *Phi, cudaStream_t st);
// Fa_v / Fb_v / loopP_v: per-recording double arrays [n_rec] (any of them null: that parameter's scalar for every recording)
int launch_run_init(const Plan &pl, const Workspace &ws, const float *gamma, const int32_t *n_states, double *Li,
                    int32_t *n_iters, int32_t *flags, int max_iters, double Fa, double Fb, double loopP,
                    const double *Fa_v, const double *Fb_v, const double *loopP_v, cudaStream_t st);
int launch_mstep_partial(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, cudaStream_t st);
// prior_n [n_rec,S], prior_F [n_rec,S,R] (DEVICE, both or neither): the enrolment prior of DESIGN.md section 5.23
int launch_speaker_model(const Plan &pl, const Workspace &ws, const float *Phi,
                         const int32_t *n_states, float *alpha_io, float *invL_io, bool from_given,
                         cudaStream_t st, const double *prior_n = nullptr, const double *prior_F = nullptr);
int launch_loglik(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states,
                  cudaStream_t st);
int launch_forward_backward(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                            const int32_t *n_states, double *Li, int32_t *n_iters, int32_t *flags, int iter,
                            int spl, int classic, int ring, cudaStream_t st);
int launch_elbo_trace(const Plan &pl, const double *Li, int max_iters, double *out, cudaStream_t st);
// forward and backward sweeps on separate warps + combine pass, any recording length (vbx_fb_split.cu)
int launch_forward_backward_split(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                  const int32_t *n_states, int spl, cudaStream_t st);
// chunked-scan forward-backward for long recordings (vbx_long_kernels.cu)
int launch_forward_backward_long(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                 const int32_t *n_states, cudaStream_t st);
// tensor-core (mma.sync 3xTF32) versions of the two in-loop contractions (vbx_mma_kernels.cu)
int launch_mstep_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, cudaStream_t st);
int launch_loglik_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states,
                      cudaStream_t st);
// M-step, speaker model and log-likelihood in one cluster kernel (vbx_em_contract.cu): the cluster size for a plan of
// these dimensions (0 = not available: split plans, S > 16, R != 128, max_T > 1024, or no cluster fits on the device)
int em_contract_cluster(int S, int R, int64_t max_T, bool split);
int launch_em_contract(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, const float *Phi,
                       const int32_t *n_states, float *alpha_io, float *invL_io, cudaStream_t st);
// float64 finishing phase of vbx_run (vbx_exact64.cu)
int launch_snapshot(const Plan &pl, const Workspace &ws, const float *gamma, const float *pi, int iter, cudaStream_t st);
int launch_exact64_round(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *rho, const float *Phi,
                         float *gamma, float *pi, const int32_t *n_states, float *alpha_io, float *invL_io, double *Li,
                         int32_t *n_iters, int32_t *flags, cudaStream_t st, const double *prior_n = nullptr,
                         const double *prior_F = nullptr);
// float64 "exact" path (vbx_f64.cu)
size_t f64_workspace_bytes(const Plan &pl);
int launch_run_f64(const Plan &pl, void *workspace, const double *fea, const double *Phi, double *gamma, double *pi,
                   const int32_t *n_states, double Fa, double Fb, double loopP, int max_iters, double epsilon,
                   double *alpha_io, double *invL_io, int warm, double *Li, int32_t *n_iters, int32_t *flags,
                   cudaStream_t st, const double *prior_n = nullptr, const double *prior_F = nullptr);
int launch_hard_labels(const Plan &pl, const float *gamma, const int32_t *n_states, int32_t *first, int32_t *second,
                       cudaStream_t st);
// labels over the keep[b] states of largest posterior mass (vbx_count.cu)
int launch_hard_labels_keep(const Plan &pl, const float *gamma, const int32_t *n_states, const int32_t *keep,
                            int32_t *first, int32_t *second, double *mass, cudaStream_t st);
// initial responsibilities and priors from speaker turns (vbx_init.cu); gamma / pi are float64 when f64, else float32
int launch_init_turns(const Plan &pl, const int64_t *seg, const int64_t *spk_off, const int64_t *turn_off,
                      const int64_t *turn_lo, const int64_t *turn_hi, const int64_t *turn_cum, const double *smoothing,
                      void *gamma, void *pi, bool f64, cudaStream_t st);
// random initial responsibilities (Philox4x64-10 exponentials, normalised) and uniform priors (vbx_init.cu)
int launch_init_random(const Plan &pl, const uint64_t *rec_key, const uint64_t *seed, const int32_t *n_states,
                       void *gamma, void *pi, bool f64, cudaStream_t st);
// reference-module forward_backward() for a general transition matrix (vbx_fb_dense.cu)
int launch_fb_dense(const double *lls, const double *tr, const double *ip, int T, int S, double *post, double *tll,
                    double *lfw, double *lbw, cudaStream_t st);
// DER accumulation (vbx_score.cu)
int launch_score(int n_rec, const int64_t *sys_off, const int64_t *sys_lo, const int64_t *sys_hi, const int64_t *sys_join_hi,
                 const int64_t *reg_off,
                 const int64_t *reg_lo, const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_ovl,
                 const int32_t *n_ref, int n_entries, const int32_t *entry_rec, const int64_t *label_off,
                 const int32_t *labels, const int32_t *labels2,      // labels2 == nullptr: the single-label kernel
                 const int32_t *n_labels, const int64_t *o_off, int64_t max_cells, int64_t *covered_out,
                 int64_t *fa_out, int64_t *O_out, int32_t *flags_out,
                 const int64_t *t_off, int64_t *T_out,                // T_out == nullptr: no label time
                 cudaStream_t st);
// combination of K diarizations (vbx_combine.cu): n_labels_host [n_rec, K] and weights_host [K] (or null) on the HOST
size_t combine_workspace_bytes(int64_t n_rec, int K, int max_labels);
int launch_combine(int64_t n_rec, const int64_t *offsets, int64_t N, const int64_t *lo, const int64_t *hi, int K,
                   const int32_t *labels, const int32_t *labels2, const int32_t *n_labels_host, int max_labels,
                   const double *weights_host, void *workspace, int32_t *labels_out, int32_t *labels2_out,
                   int32_t *order_out, double *weights_out, int64_t *D_out, int32_t *map_out, int32_t *n_global_out,
                   int32_t *flags_out, int64_t *O_out, int64_t *L_out, cudaStream_t st);
// AHC initialisation (vbx_ahc.cu)
size_t ahc_workspace_bytes(const int64_t *offsets_host, int n_rec, std::vector<int64_t> *d_off_host);
int launch_ahc(const Plan &pl, const std::vector<int64_t> &d_off, const void *x, int x_is_f64, int dim, void *workspace,
               size_t workspace_bytes, double *Z_out, double *thr_out, cudaStream_t st, std::string *err);
// ahc_linkage_kernel with one CTA per problem over the n problems described by the DEVICE arrays offsets [n+1] and
// d_off [n]; problem b's region of ws (linkage_workspace_bytes(T_b) bytes at d_off[b], the T_b x T_b distances first) is
// laid out as vbx_ahc's, and its Z rows start at row offsets[b] of Z_out
size_t linkage_workspace_bytes(int64_t T);
void launch_linkage(const int64_t *offsets, const int64_t *d_off, int n, void *ws, double *Z_out, cudaStream_t st);
// speaker linking across recordings (vbx_link.cu): G problems in one set of launches (vbx_link_batch), M_host [G]
// speakers and c_host [G] = Fa_g / Fb_g on the HOST; lk_off (when not null) gets the byte offsets [G+1] of the
// problems' linkage regions.  mean, std [sum M] (DEVICE, both or neither): normalised distances
size_t link_batch_workspace_bytes(int G, const int64_t *M_host, std::vector<int64_t> *lk_off = nullptr);
int launch_link_batch(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, const int32_t *spk_rec,
                      int G, const int64_t *M_host, const double *c_host, void *workspace, double *n_out,
                      double *F_out, double *dist_out, double *Z_out, cudaStream_t st, const double *mean,
                      const double *std);
// Caller-owned DEVICE arrays for the statistics of vbx_link_batch's span and statistics kernels: n, e [M],
// b [M, kMaxR] float64; first, last [M] int64 scratch.
struct SpeakerStats {
    double *n, *e, *b;
    long long *first, *last;
};
// The statistics of n speakers carved from a workspace by take(bytes) (host), as the enrolment and cohort layouts hold them
template <class Take>
SpeakerStats take_stats(Take &take, int64_t n) {
    SpeakerStats s;
    s.n = reinterpret_cast<double *>(take(n * 8));
    s.e = reinterpret_cast<double *>(take(n * 8));
    s.b = reinterpret_cast<double *>(take(n * kMaxR * 8));
    s.first = reinterpret_cast<long long *>(take(n * 8));
    s.last = reinterpret_cast<long long *>(take(n * 8));
    take(4 * 8);             // unused; kept so that the published batched workspace sizes stay the same
    return s;
}
// n_s, F_s, b_s and e_s of G problems into s as vbx_link_batch computes them: spk [G,N] (row g: local speakers of
// problem g), off [G+1] and c [G] DEVICE; s holds M = off[G] speakers.  Problem g's statistics do not depend on the
// other problems.  Returns the number of launches, -1 on a launch error.
int launch_speaker_stats_batch(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, int G,
                               const int64_t *off, const double *c, int64_t M, const SpeakerStats &s, double *n_out,
                               double *F_out, cudaStream_t st);
// Several problems of norm_scores_kernel (DESIGN.md section 5.19), DEVICE arrays [G+1].  Rectangle (blk null): x holds
// the rows of every problem, problem g's off[g] .. off[g+1]-1, with row statistics at the row and column statistics at
// g * cols + column.  Square blocks (blk set): problem g's off[g+1] - off[g] square block starts at element blk[g] of
// copy_out and at byte x_bytes[g] of x, its statistics at off[g] + row and off[g] + column; rows * cols = blk[G].
struct NormProblems {
    int G;
    const int64_t *off, *blk, *x_bytes;
};
// enrolment against known speakers (vbx_enroll.cu)
// enroll_score_kernel over G problems whose statistics are already in a and co: rows off[g] .. off[g+1]-1 of a against
// columns g C .. g C + C - 1 of co with c[g], flat tiles tile_off [G+1] (every array DEVICE; n_tiles = tile_off[G] on
// the host) into llr [off[G], C] (and llr_out when not null), bit-identical to vbx_enroll_batch's llr against the same
// speakers.  Returns 1, 0 for n_tiles == 0.
int launch_cohort_scores_batch(const SpeakerStats &a, const SpeakerStats &co, const float *Phi, int G,
                               const int64_t *off, const int64_t *tile_off, const double *c, int64_t n_tiles, int64_t C,
                               int R, double *llr, double *llr_out, cudaStream_t st);
// score tiles of an M x C rectangle (host)
int64_t rect_tiles(int64_t M, int64_t C);
// dst [G, n] = G copies of src [n] (DEVICE)
int launch_repeat_index(const int32_t *src, int64_t n, int G, int32_t *dst, cudaStream_t st);
// G enrolment problems (vbx_enroll_batch): M_host [G], rec_off_host [G, n_rec + 1], c_host [G], thresholds [n_thr] HOST
size_t enroll_batch_workspace_bytes(int G, const int64_t *M_host, int64_t E, int64_t N_e, int64_t max_k, int64_t n_thr,
                                    int sms);
int launch_enroll_batch(const float *fea, const float *Phi, int64_t N, int R, const int32_t *spk, int G,
                        const int64_t *M_host, const int64_t *rec_off_host, int n_rec, const float *enroll_fea,
                        int64_t N_e, const int32_t *enroll_spk, int64_t E, const double *c_host,
                        const double *thresholds, int64_t n_thr, void *workspace, int sms, int32_t *assign_out,
                        double *best_llr_out, double *llr_out, double *n_out, double *F_out, double *n_enroll_out,
                        double *F_enroll_out, cudaStream_t st, const double *mean, const double *std,
                        const double *enroll_mean, const double *enroll_std);
// score normalisation against a cohort (vbx_cohort.cu): G problems against one cohort (vbx_cohort_stats_batch),
// M_host [G], c_host [G] HOST; scores_out [sum M, C] optional
size_t cohort_batch_workspace_bytes(int G, const int64_t *M_host, int64_t C, int64_t N_c);
int launch_cohort_batch(const float *fea, const float *Phi, int64_t N, int R, const int32_t *spk, int G,
                        const int64_t *M_host, const float *cohort_fea, int64_t N_c, const int32_t *cohort_spk,
                        int64_t C, const double *c_host, int64_t top_k, void *workspace, double *mean_out,
                        double *std_out, double *scores_out, cudaStream_t st);
// x [rows, cols] of LLRs (link: of distances -LLR, diagonal and `skip` entries kept) replaced by the normalised scores
// of the problems q
int launch_norm_scores(double *x, int64_t rows, int64_t cols, const double *mean_r, const double *std_r,
                       const double *mean_c, const double *std_c, bool link, double skip, double *copy_out,
                       cudaStream_t st, const NormProblems &q);
// speaker-verification trials (vbx_verify.cu): statistics of both sides, the trial scores (mean_e .. std_t all DEVICE,
// all four or none: AS-norm), and the error rates of a scored list; ops_host [n_op, 4] = C_miss p, C_fa (1 - p), their
// min and the Bayes threshold of every operating point (HOST)
size_t verify_score_workspace_bytes(int64_t M_e, int64_t M_t);
int launch_verify_score(const float *enroll_fea, int64_t N_e, const int32_t *enroll_item, int64_t M_e,
                        const float *test_fea, int64_t N_t, const int32_t *test_item, int64_t M_t, int R,
                        const float *Phi, double c, const int32_t *ti, const int32_t *tj, int64_t T,
                        const double *mean_e, const double *std_e, const double *mean_t, const double *std_t,
                        void *workspace, double *score_out, cudaStream_t st);
size_t verify_metrics_workspace_bytes(int64_t T, int n_op);
int launch_verify_metrics(const double *scores, const uint8_t *is_target, int64_t T, const double *ops_host, int n_op,
                          void *workspace, long long *counts_out, double *eer_out, double *cllr_out,
                          double *min_dcf_out, double *threshold_out, double *act_dcf_out, cudaStream_t st);
// the calibration of a scored list (vbx_verify.cu, section 5.28): info_out [5] status, passes, N_tar, N_non, hull vertices;
// out [4] a, b, cllr_prior, min_cllr (both DEVICE)
size_t verify_calibrate_workspace_bytes(int64_t T);
int launch_verify_calibrate(const double *scores, const uint8_t *is_target, int64_t T, double prior, void *workspace,
                            long long *info_out, double *out, cudaStream_t st);
// wgmma projection (vbx_project_tc.cu)
size_t tc_scratch_floats();
int launch_project_wgmma(const Plan &pl, float *tc_scratch, const float *X, int D, const float *V, const float *Phi, float *rho,
                         float *gframe, cudaStream_t st, std::string *err);
int launch_xvector_chain_wgmma(const Plan &pl, float *tc_scratch, const float *x_raw, int Dx, const float *mean1, const float *lda,
                               const float *mean2, const float *plda_mu, const float *plda_tr, const float *psi,
                               float *x_norm, float *rho, float *gframe, cudaStream_t st, std::string *err);
int launch_gsum_from_frames(const Plan &pl, const Workspace &ws, const float *gframe, cudaStream_t st);
// class means and within-class scatter on the FP64 tensor cores (vbx_train.cu, vbx_class_scatter); offsets_host [K+1]
size_t class_scatter_workspace_bytes(int64_t N, int D, int64_t K);
int launch_class_scatter(const float *X, int64_t N, int D, int64_t K, const int64_t *offsets_host, void *workspace,
                         double *means_out, double *scatter_out, cudaStream_t st);
// streaming diarization: a push's window from the streams' state, and its result folded back (vbx_stream.cu)
int launch_stream_window(int n, int C, int R, int S_max, int S, const int32_t *slot, const int64_t *blk_off,
                         const int64_t *win_off, const int32_t *blk_lab, const int32_t *n_clusters, const float *blk_fea,
                         double smoothing, const float *ctx_fea, const int32_t *ctx_lab, const int64_t *count,
                         const int32_t *K, const double *n_hist, const double *F_hist, float *fea_out, float *gamma_out,
                         float *pi_out, int32_t *n_states_out, double *prior_n_out, double *prior_F_out,
                         cudaStream_t st);
int launch_stream_commit(int n, int C, int R, int S_max, const int32_t *slot, const int64_t *blk_off,
                         const int64_t *win_off, const float *blk_fea, const int32_t *first, float *ctx_fea,
                         int32_t *ctx_lab, int64_t *count, int32_t *K, double *n_hist, double *F_hist,
                         int32_t *labels_out, cudaStream_t st);

}  // namespace vbx
