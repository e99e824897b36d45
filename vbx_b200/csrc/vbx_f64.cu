// Float64 evaluation of the VB-HMM EM loop on the GPU ("exact" mode of the reference-facing call).
//
// The reference computes in float64 (VBx/VBx.py is plain numpy on float64 inputs) and vbhmm.py stops on an ELBO
// improvement below 1e-6 (VBx/vbhmm.py:157) -- far below what float32 frame log-likelihoods can resolve on
// |ELBO| ~ 1e5.  This path keeps every quantity in float64 so that the drop-in VBx() reproduces the reference's
// iteration count and its gamma / pi / Li to ~1e-9.  It is deliberately simple (a handful of straightforward
// kernels, scaled linear-domain recursion with the same O(S) transition structure as the float32 path): it is meant
// for the one-recording-per-call use of VBx/vbhmm.py:154-158, not for throughput.  Like the reference it accepts ANY number
// of HMM states and ANY feature dimension (vbx_plan_f64): every kernel loops over states / features instead of fixing a
// lane per state.
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {
namespace f64 {

struct Buffers {
    double *rho;     // [N,R]
    double *p;       // [N,S]   exp(ll - rowmax)
    double *rowmax;  // [N]
    double *rsig;    // [N]
    double *alpha;   // [B,S,R]
    double *invL;    // [B,S,R]
    double *bias;    // [B,S]
    double *reg;     // [B]
    double *gsum;    // [B]
    double *prev;    // [B]
    int32_t *active; // [B]
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}
__device__ __forceinline__ double block_sum(double v, double *sh) {   // blockDim.x == 128
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    return sh[0] + sh[1] + sh[2] + sh[3];
}

// rho = fea * sqrt(Phi), G sum, reset of the per-recording state               VBx/VBx.py:87-89
__global__ void __launch_bounds__(128) prep_kernel(Plan pl, Buffers b, const double *__restrict__ fea,
                                                   const double *__restrict__ Phi, const int32_t *n_states, double *Li,
                                                   int32_t *n_iters, int32_t *flags, int max_iters) {
    __shared__ double sh[4];
    const int rec = blockIdx.x, R = pl.R, tid = threadIdx.x;
    const int64_t f0 = pl.offsets[rec];
    const int64_t T = pl.offsets[rec + 1] - f0;
    double acc = 0.0;
    for (int64_t i = tid; i < T * R; i += 128) {
        const int r = (int)(i % R);
        const double x = fea[f0 * R + i];
        b.rho[f0 * R + i] = x * sqrt(Phi[r]);
        acc += x * x;
    }
    acc = block_sum(acc, sh);
    for (int i = tid; i < max_iters; i += 128) Li[(int64_t)rec * max_iters + i] = CUDART_NAN;
    if (tid == 0) {
        b.gsum[rec] = -0.5 * (acc + (double)T * R * 1.8378770664093454835606594728112);
        const int ns = n_states ? n_states[rec] : pl.S;
        b.active[rec] = (T > 0 && ns > 0) ? 1 : 0;
        b.prev[rec] = 0.0;
        n_iters[rec] = 0;
        flags[rec] = 0;
    }
}

// M-step for one (recording, speaker): invL, alpha over r (threads stride the features)      VBx/VBx.py:95-96
// PRIOR (here and in bias_body): the enrolment prior of prior_n [B,S], prior_F [B,S,R] (DESIGN.md section 5.23)
template <bool PRIOR>
__device__ __forceinline__ void mstep_body(const Plan &pl, const Buffers &b, const double *__restrict__ gamma,
                                           const double *__restrict__ Phi, const int32_t *n_states, double FaFb,
                                           const double *__restrict__ prior_n, const double *__restrict__ prior_F) {
    const int rec = blockIdx.x / pl.S, s = blockIdx.x % pl.S;
    if (!b.active[rec]) return;
    const int R = pl.R, S = pl.S;
    const int ns = n_states ? n_states[rec] : S;
    const int64_t f0 = pl.offsets[rec];
    const int64_t T = pl.offsets[rec + 1] - f0;
    for (int r = threadIdx.x; r < R; r += 128) {
        const int64_t o = ((int64_t)rec * S + s) * R + r;
        if (s >= ns) {
            b.alpha[o] = 0.0;
            b.invL[o] = 0.0;
            continue;
        }
        double Ns = 0.0, gr = 0.0;
        for (int64_t t = 0; t < T; ++t) {
            const double g = gamma[(f0 + t) * S + s];
            Ns += g;
            gr += g * b.rho[(f0 + t) * R + r];
        }
        if constexpr (PRIOR) {
            Ns += prior_n[(int64_t)rec * S + s];
            gr += sqrt(Phi[r]) * prior_F[o];
        }
        const double iL = 1.0 / (1.0 + FaFb * Ns * Phi[r]);
        b.invL[o] = iL;
        b.alpha[o] = FaFb * iL * gr;
    }
}

__global__ void __launch_bounds__(128) mstep_kernel(Plan pl, Buffers b, const double *__restrict__ gamma,
                                                    const double *__restrict__ Phi, const int32_t *n_states, double FaFb) {
    mstep_body<false>(pl, b, gamma, Phi, n_states, FaFb, nullptr, nullptr);
}

__global__ void __launch_bounds__(128) mstep_prior_kernel(Plan pl, Buffers b, const double *__restrict__ gamma,
                                                          const double *__restrict__ Phi, const int32_t *n_states,
                                                          double FaFb, const double *__restrict__ prior_n,
                                                          const double *__restrict__ prior_F) {
    mstep_body<true>(pl, b, gamma, Phi, n_states, FaFb, prior_n, prior_F);
}

// per-speaker bias of eq. (23) and the ELBO regulariser of eq. (25)           VBx/VBx.py:97,100
template <bool PRIOR>
__device__ __forceinline__ void bias_body(const Plan &pl, const Buffers &b, const double *__restrict__ Phi,
                                          const int32_t *n_states, double Fb, double FaFb,
                                          const double *__restrict__ prior_n, const double *__restrict__ prior_F) {
    __shared__ double sh[4];
    const int rec = blockIdx.x;
    if (!b.active[rec]) return;
    const int R = pl.R, S = pl.S;
    const int ns = n_states ? n_states[rec] : S;
    double reg = 0.0;
    for (int s = 0; s < S; ++s) {
        double c = 0.0;
        if (s < ns) {
            for (int r = threadIdx.x; r < R; r += 128) {
                const int64_t o = ((int64_t)rec * S + s) * R + r;
                const double iL = b.invL[o], a = b.alpha[o];
                c += (iL + a * a) * Phi[r];
                reg += log(iL) - iL - a * a + 1.0;
                if constexpr (PRIOR) {   // log(lambda0 iL) - lambda0 iL - lambda0 (a - mu0)^2 + 1: the terms of
                    // speaker_model_body, each with a factor lambda0 - 1 or mu0 (exactly 0 without a prior)
                    const double ne = prior_n[(int64_t)rec * S + s], Fe = prior_F[o];
                    if (ne != 0.0 || Fe != 0.0) {
                        const double lam0 = 1.0 + FaFb * ne * Phi[r];
                        const double mu0 = FaFb * sqrt(Phi[r]) * Fe / lam0, d = a - mu0;
                        reg += log(lam0) - (lam0 - 1.0) * (iL + d * d) + mu0 * (a + d);
                    }
                }
            }
        }
        c = block_sum(c, sh);
        if (threadIdx.x == 0) b.bias[(int64_t)rec * S + s] = s < ns ? 0.5 * c : CUDART_INF;
    }
    reg = block_sum(reg, sh);
    if (threadIdx.x == 0) b.reg[rec] = 0.5 * Fb * reg;
}

__global__ void __launch_bounds__(128) bias_kernel(Plan pl, Buffers b, const double *__restrict__ Phi,
                                                   const int32_t *n_states, double Fb) {
    bias_body<false>(pl, b, Phi, n_states, Fb, 0.0, nullptr, nullptr);
}

__global__ void __launch_bounds__(128) bias_prior_kernel(Plan pl, Buffers b, const double *__restrict__ Phi,
                                                         const int32_t *n_states, double Fb, double FaFb,
                                                         const double *__restrict__ prior_n,
                                                         const double *__restrict__ prior_F) {
    bias_body<true>(pl, b, Phi, n_states, Fb, FaFb, prior_n, prior_F);
}

// log-likelihoods, row max, exp: one thread per frame                          VBx/VBx.py:97
__global__ void __launch_bounds__(128) loglik_kernel(Plan pl, Buffers b, double Fa) {
    const int64_t f = (int64_t)blockIdx.x * 128 + threadIdx.x;
    if (f >= pl.n_frames) return;
    // recording of this frame by binary search over the offsets
    int lo = 0, hi = pl.n_rec - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pl.offsets[mid] <= f) lo = mid; else hi = mid - 1;
    }
    const int rec = lo;
    if (!b.active[rec]) return;
    const int R = pl.R, S = pl.S;
    double m = -CUDART_INF;
    for (int s = 0; s < S; ++s) {
        const double bias = b.bias[(int64_t)rec * S + s];
        double d = -CUDART_INF;
        if (bias < CUDART_INF) {
            d = 0.0;
            const double *a = b.alpha + ((int64_t)rec * S + s) * R;
            const double *x = b.rho + f * R;
            for (int r = 0; r < R; ++r) d += x[r] * a[r];
            d = Fa * (d - bias);
        }
        b.p[f * S + s] = d;
        m = fmax(m, d);
    }
    for (int s = 0; s < S; ++s) b.p[f * S + s] = exp(b.p[f * S + s] - m);
    b.rowmax[f] = m;
}

// forward-backward, pi, ELBO, stop rule for S <= 64: one warp per recording, lane = state (two states per lane for
// S > 32), everything in registers
// VBx/VBx.py:98-105,122-125,146-175 in the scaled linear domain (see vbx_kernels.cu for the derivation)
__global__ void __launch_bounds__(32) fb_kernel_small(Plan pl, Buffers b, double *gamma, double *pi_io, const int32_t *n_states,
                                                double Fa, double loopP, double epsilon, double *Li, int32_t *n_iters,
                                                int32_t *flags, int iter, int max_iters) {
    const int rec = blockIdx.x, lane = threadIdx.x;
    if (!b.active[rec]) return;
    const int S = pl.S;
    const int ns = n_states ? n_states[rec] : S;
    const int64_t f0 = pl.offsets[rec];
    const int T = (int)(pl.offsets[rec + 1] - f0);
    const double P = loopP, Q = 1.0 - loopP, eps = 1e-8;
    double pi[2], w[2], a[2], base[2];
    for (int k = 0; k < 2; ++k) {
        const int s = lane + 32 * k;
        const bool live = s < ns;
        pi[k] = live ? pi_io[(int64_t)rec * S + s] : 0.0;
        w[k] = live ? Q * pi[k] + eps : 0.0;
        base[k] = live ? pi[k] + eps : 0.0;
        a[k] = 0.0;
    }
    const double *pp = b.p + f0 * S;
    double *ga = gamma + f0 * S;
    double tll = 0.0;
    for (int t = 0; t < T; ++t) {
        double v[2], loc = 0.0;
        for (int k = 0; k < 2; ++k) {
            const int s = lane + 32 * k;
            v[k] = s < S ? pp[(int64_t)t * S + s] * base[k] : 0.0;
            loc += v[k];
        }
        const double sig = warp_sum(loc);
        const double r = 1.0 / sig;
        for (int k = 0; k < 2; ++k) {
            const int s = lane + 32 * k;
            a[k] = v[k] * r;
            base[k] = P * a[k] + w[k] * 1.0;
            if (s < S) ga[(int64_t)t * S + s] = a[k];
        }
        if (lane == 0) b.rsig[f0 + t] = r;
        tll += log(sig) + b.rowmax[f0 + t];
    }
    __syncwarp();
    double bb[2] = {1.0, 1.0}, g0[2] = {a[0], a[1]}, occ[2] = {a[0], a[1]}, enter[2] = {0.0, 0.0};
    for (int t = T - 2; t >= 0; --t) {
        const double cr = b.rsig[f0 + t + 1];
        double u[2], loc = 0.0;
        for (int k = 0; k < 2; ++k) {
            const int s = lane + 32 * k;
            u[k] = s < S ? pp[(int64_t)(t + 1) * S + s] * bb[k] * cr : 0.0;
            loc += w[k] * u[k];
        }
        const double dot = warp_sum(loc);
        for (int k = 0; k < 2; ++k) {
            const int s = lane + 32 * k;
            enter[k] += u[k];
            bb[k] = P * u[k] + dot;
            if (s < S) {
                g0[k] = ga[(int64_t)t * S + s] * bb[k];
                ga[(int64_t)t * S + s] = g0[k];
                occ[k] += g0[k];
            }
        }
    }
    double pn[2], loc = 0.0;
    for (int k = 0; k < 2; ++k) {
        pn[k] = g0[k] + Q * pi[k] * enter[k];
        loc += pn[k];
    }
    const double tot = warp_sum(loc);
    for (int k = 0; k < 2; ++k) {
        const int s = lane + 32 * k;
        if (s < S) pi_io[(int64_t)rec * S + s] = pn[k] / tot;
    }
    if (lane == 0) {
        const double elbo = tll + Fa * b.gsum[rec] + b.reg[rec];
        Li[(int64_t)rec * max_iters + iter] = elbo;
        n_iters[rec] = iter + 1;
        int fl = flags[rec];
        if (!isfinite(elbo)) fl |= 1;
        if (iter > 0) {
            const double d = elbo - b.prev[rec];
            if (d < epsilon) {
                b.active[rec] = 0;
                if (iter + 1 < max_iters) fl |= 4;
                if (d < 0.0) fl |= 2;
            }
        }
        b.prev[rec] = elbo;
        flags[rec] = fl;
    }
}

// forward-backward, pi, ELBO, stop rule: one warp per recording, lanes stride the states (any S: the per-state vectors
// live in shared memory)            VBx/VBx.py:98-105,122-125,146-175 in the scaled linear domain (see vbx_kernels.cu)
__global__ void __launch_bounds__(32) fb_kernel(Plan pl, Buffers b, double *gamma, double *pi_io, const int32_t *n_states,
                                                double Fa, double loopP, double epsilon, double *Li, int32_t *n_iters,
                                                int32_t *flags, int iter, int max_iters) {
    extern __shared__ double shv[];
    const int rec = blockIdx.x, lane = threadIdx.x;
    if (!b.active[rec]) return;
    const int S = pl.S;
    double *pi = shv, *w = shv + S, *base = shv + 2 * S, *a = shv + 3 * S, *bb = shv + 4 * S, *enter = shv + 5 * S, *g0 = shv + 6 * S;
    const int ns = n_states ? n_states[rec] : S;
    const int64_t f0 = pl.offsets[rec];
    const int T = (int)(pl.offsets[rec + 1] - f0);
    const double P = loopP, Q = 1.0 - loopP, eps = 1e-8;
    for (int s = lane; s < S; s += 32) {
        const bool live = s < ns;
        pi[s] = live ? pi_io[(int64_t)rec * S + s] : 0.0;
        w[s] = live ? Q * pi[s] + eps : 0.0;
        base[s] = live ? pi[s] + eps : 0.0;
        a[s] = 0.0;
        enter[s] = 0.0;
    }
    __syncwarp();
    const double *pp = b.p + f0 * S;
    double *ga = gamma + f0 * S;
    double tll = 0.0;
    for (int t = 0; t < T; ++t) {
        double loc = 0.0;
        for (int s = lane; s < S; s += 32) {
            const double v = pp[(int64_t)t * S + s] * base[s];
            a[s] = v;
            loc += v;
        }
        const double sig = warp_sum(loc);
        const double r = 1.0 / sig;
        for (int s = lane; s < S; s += 32) {
            const double av = a[s] * r;
            a[s] = av;
            base[s] = P * av + w[s];
            ga[(int64_t)t * S + s] = av;
        }
        if (lane == 0) b.rsig[f0 + t] = r;
        tll += log(sig) + b.rowmax[f0 + t];
    }
    __syncwarp();
    for (int s = lane; s < S; s += 32) {
        bb[s] = 1.0;
        g0[s] = a[s];
    }
    for (int t = T - 2; t >= 0; --t) {
        const double cr = b.rsig[f0 + t + 1];
        double loc = 0.0;
        for (int s = lane; s < S; s += 32) {
            const double u = pp[(int64_t)(t + 1) * S + s] * bb[s] * cr;
            a[s] = u;                       // a[] is free now: holds u for the second pass
            loc += w[s] * u;
        }
        const double dot = warp_sum(loc);
        for (int s = lane; s < S; s += 32) {
            const double u = a[s];
            enter[s] += u;
            bb[s] = P * u + dot;
            g0[s] = ga[(int64_t)t * S + s] * bb[s];
            ga[(int64_t)t * S + s] = g0[s];
        }
    }
    double loc = 0.0;
    for (int s = lane; s < S; s += 32) {
        const double pn = g0[s] + Q * pi[s] * enter[s];
        a[s] = pn;
        loc += pn;
    }
    const double tot = warp_sum(loc);
    for (int s = lane; s < S; s += 32) pi_io[(int64_t)rec * S + s] = a[s] / tot;
    if (lane == 0) {
        const double elbo = tll + Fa * b.gsum[rec] + b.reg[rec];
        Li[(int64_t)rec * max_iters + iter] = elbo;
        n_iters[rec] = iter + 1;
        int fl = flags[rec];
        if (!isfinite(elbo)) fl |= 1;
        if (iter > 0) {
            const double d = elbo - b.prev[rec];
            if (d < epsilon) {
                b.active[rec] = 0;
                if (iter + 1 < max_iters) fl |= 4;
                if (d < 0.0) fl |= 2;
            }
        }
        b.prev[rec] = elbo;
        flags[rec] = fl;
    }
}

}  // namespace f64

size_t f64_workspace_bytes(const Plan &pl) {
    const size_t N = (size_t)pl.n_frames, S = (size_t)pl.S, R = (size_t)pl.R, B = (size_t)pl.n_rec;
    return sizeof(double) * (N * R + N * S + 2 * N + 2 * B * S * R + B * S + 3 * B) + sizeof(int32_t) * B + 4096;
}

int launch_run_f64(const Plan &pl, void *workspace, const double *fea, const double *Phi, double *gamma, double *pi,
                   const int32_t *n_states, double Fa, double Fb, double loopP, int max_iters, double epsilon,
                   double *alpha_io, double *invL_io, int warm, double *Li, int32_t *n_iters, int32_t *flags,
                   cudaStream_t st, const double *prior_n, const double *prior_F) {
    if (pl.n_rec == 0) return 0;
    const size_t N = (size_t)pl.n_frames, S = (size_t)pl.S, R = (size_t)pl.R, B = (size_t)pl.n_rec;
    f64::Buffers b;
    double *w = static_cast<double *>(workspace);
    b.rho = w; w += N * R;
    b.p = w; w += N * S;
    b.rowmax = w; w += N;
    b.rsig = w; w += N;
    b.alpha = w; w += B * S * R;
    b.invL = w; w += B * S * R;
    b.bias = w; w += B * S;
    b.reg = w; w += B;
    b.gsum = w; w += B;
    b.prev = w; w += B;
    b.active = reinterpret_cast<int32_t *>(w);
    int launches = 0;
    f64::prep_kernel<<<pl.n_rec, 128, 0, st>>>(pl, b, fea, Phi, n_states, Li, n_iters, flags, max_iters);
    ++launches;
    if (warm) {
        cudaMemcpyAsync(b.alpha, alpha_io, sizeof(double) * B * S * R, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(b.invL, invL_io, sizeof(double) * B * S * R, cudaMemcpyDeviceToDevice, st);
    }
    const int fblocks = (int)((pl.n_frames + 127) / 128);
    const size_t fb_smem = (size_t)7 * pl.S * sizeof(double);     // per-state vectors of the sweep
    if (fb_smem > 48 * 1024) {
        if (!allow_dynamic_smem(f64::fb_kernel, 200 * 1024)) return -1;
        if (fb_smem > 200 * 1024) return -1;                      // more than 3600 states
    }
    for (int it = 0; it < max_iters; ++it) {
        if (!(it == 0 && warm)) {
            if (prior_n)
                f64::mstep_prior_kernel<<<pl.n_rec * pl.S, 128, 0, st>>>(pl, b, gamma, Phi, n_states, Fa / Fb, prior_n, prior_F);
            else
                f64::mstep_kernel<<<pl.n_rec * pl.S, 128, 0, st>>>(pl, b, gamma, Phi, n_states, Fa / Fb);
            ++launches;
        }
        if (prior_n)
            f64::bias_prior_kernel<<<pl.n_rec, 128, 0, st>>>(pl, b, Phi, n_states, Fb, Fa / Fb, prior_n, prior_F);
        else
            f64::bias_kernel<<<pl.n_rec, 128, 0, st>>>(pl, b, Phi, n_states, Fb);
        if (fblocks) f64::loglik_kernel<<<fblocks, 128, 0, st>>>(pl, b, Fa);
        if (pl.S <= 64)
            f64::fb_kernel_small<<<pl.n_rec, 32, 0, st>>>(pl, b, gamma, pi, n_states, Fa, loopP, epsilon, Li, n_iters, flags, it, max_iters);
        else
            f64::fb_kernel<<<pl.n_rec, 32, fb_smem, st>>>(pl, b, gamma, pi, n_states, Fa, loopP, epsilon, Li, n_iters, flags, it, max_iters);
        launches += 3;
    }
    if (alpha_io && invL_io) {
        cudaMemcpyAsync(alpha_io, b.alpha, sizeof(double) * B * S * R, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(invL_io, b.invL, sizeof(double) * B * S * R, cudaMemcpyDeviceToDevice, st);
    }
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace vbx
