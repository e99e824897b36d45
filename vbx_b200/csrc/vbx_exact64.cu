// Float64 finishing phase of the batched EM loop: the reference's stop rule at float64 resolution.
//
// The reference stops when the ELBO improves by less than epsilon (VBx/VBx.py:122-125); vbhmm.py passes
// epsilon = 1e-6 on |ELBO| ~ 1e5 (VBx/vbhmm.py:157), three orders of magnitude below what float32 frame
// log-likelihoods resolve.  vbx_run therefore runs a recording through the float32 kernels only while its ELBO
// step is safely above float32 noise; once the step of iteration k comes within a guard band of epsilon the recording
// SWITCHES: iterations k-1 and k are discarded, the state that entered iteration k-1 is restored (gamma and pi are
// snapshotted at the start of every float32 iteration, two deep), and the remaining iterations -- beginning with
// k-1, so that the test of iteration k already compares two float64 values -- are evaluated by the kernels of this
// file: every quantity in float64 (inputs: the float32 rho and the float32-stored gamma and pi, exact in float64),
// with the reference's test on exact ELBO values.  A switched recording lags one round behind the others.  Two values
// are stored in float32: gamma between iterations (the output precision) and the normalised forward variables, which
// fb64 parks in gamma for the backward sweep (their rounding reaches gamma and pi); pi stays float64 across rounds.  That
// perturbs the ELBO steps by < 1e-9 near the fixed point, three orders below epsilon.
// Each kernel handles only recordings with ws.active64 != 0; a round of these launches costs a few microseconds
// when no recording is in this phase.
//
//   restore64   snapshot -> gamma, pi64                              (first float64 iteration of a recording)
//   mstep64     per 512-frame tile: gamma^T rho, N_s                 VBx/VBx.py:95-96
//   speaker64   invL, alpha, bias, ELBO regulariser                  VBx/VBx.py:95-97,100
//   loglik64    log_p_ - rowmax, exp                                 VBx/VBx.py:97
//   fb64        forward-backward, gamma, pi (eq. 24)                 VBx/VBx.py:98-104,146-175
//   elbo64      ELBO, trace, stop test                               VBx/VBx.py:100,105,122-125
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {
namespace x64 {

template <int LANES>
__device__ __forceinline__ double gsum(double v) {
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// ---------------------------------------------------------------------------------------------------------
// snapshot (float32 phase) and restore (first float64 iteration): one CTA per M-tile
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) snapshot_kernel(Plan pl, Workspace ws, const float *__restrict__ gamma,
                                                       const float *__restrict__ pi, int parity) {
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int S = pl.S;
    const float4 *src = reinterpret_cast<const float4 *>(gamma + f0 * S);
    float4 *dst = reinterpret_cast<float4 *>(ws.gamma_snap + (parity * pl.n_frames + f0) * S);
    const int n4 = len * S / 4;
    for (int i = threadIdx.x; i < n4; i += 256) dst[i] = src[i];
    if (tile == pl.mtile_begin[rec] && (int)threadIdx.x < S)
        ws.pi_snap[((int64_t)parity * pl.n_rec + rec) * S + threadIdx.x] = pi[(int64_t)rec * S + threadIdx.x];
}

// the state that entered iteration n_iters[rec] (the first one to be redone in float64) lives in snapshot n_iters[rec] % 2
__global__ void __launch_bounds__(256) restore64_kernel(Plan pl, Workspace ws, float *__restrict__ gamma,
                                                        const int32_t *__restrict__ n_iters) {
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active64[rec] || !ws.fresh[rec]) return;
    const int parity = n_iters[rec] & 1;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int S = pl.S;
    const float4 *src = reinterpret_cast<const float4 *>(ws.gamma_snap + (parity * pl.n_frames + f0) * S);
    float4 *dst = reinterpret_cast<float4 *>(gamma + f0 * S);
    const int n4 = len * S / 4;
    for (int i = threadIdx.x; i < n4; i += 256) dst[i] = src[i];
    if (tile == pl.mtile_begin[rec] && (int)threadIdx.x < S)
        ws.pi64[(int64_t)rec * S + threadIdx.x] = (double)ws.pi_snap[((int64_t)parity * pl.n_rec + rec) * S + threadIdx.x];
}

// ---------------------------------------------------------------------------------------------------------
// M-step accumulation in float64: partial64[tile][s][r] = sum_t gamma[t,s] rho[t,r], occp64[tile][s] = sum_t gamma
// 256 threads: r = tid % 128, h = tid / 128 takes the frames of parity h; gamma is staged per 64-frame block in
// shared memory and read as broadcast float4.  S = 128: h takes the states of half h instead (every frame), so that a
// thread keeps 64 accumulators and the two halves need no reduction.
// ---------------------------------------------------------------------------------------------------------
template <int S_PAD>
__global__ void __launch_bounds__(256) mstep64_kernel(Plan pl, Workspace ws, const float *__restrict__ rho,
                                                      const float *__restrict__ gamma) {
    constexpr int FB = 64;
    constexpr bool HALVES = S_PAD > kMaxS;
    constexpr int SA = HALVES ? S_PAD / 2 : S_PAD;   // accumulators per thread
    __shared__ __align__(16) float gs[FB][S_PAD];
    __shared__ double occs[S_PAD];
    extern __shared__ double red[];   // [S_PAD][kMaxR] reduction of the two frame parities (not used with HALVES)
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active64[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int R = pl.R;
    const int tid = threadIdx.x, r = tid & 127, h = tid >> 7;
    const bool rlive = r < R;
    double acc[SA];
#pragma unroll
    for (int s = 0; s < SA; ++s) acc[s] = 0.0;
    double occ = 0.0;
    for (int b0 = 0; b0 < len; b0 += FB) {
        const int bl = min(FB, len - b0);
        __syncthreads();
        {
            const float4 *src = reinterpret_cast<const float4 *>(gamma + (f0 + b0) * S_PAD);
            float4 *dst = reinterpret_cast<float4 *>(&gs[0][0]);
            for (int i = tid; i < bl * S_PAD / 4; i += 256) dst[i] = src[i];
        }
        __syncthreads();
        if (tid < S_PAD) {
            double o = 0.0;
            for (int f = 0; f < bl; ++f) o += (double)gs[f][tid];
            occ += o;
        }
        if (rlive) {
            const float *xr = rho + (f0 + b0) * R + r;
            constexpr int FSTEP = HALVES ? 1 : 2;
            const int s0 = HALVES ? h * SA : 0;
#pragma unroll 2
            for (int f = HALVES ? 0 : h; f < bl; f += FSTEP) {
                const double x = (double)__ldg(xr + (int64_t)f * R);
#pragma unroll
                for (int q = 0; q < SA / 4; ++q) {
                    const float4 g = *reinterpret_cast<const float4 *>(&gs[f][s0 + 4 * q]);
                    acc[4 * q + 0] = fma((double)g.x, x, acc[4 * q + 0]);
                    acc[4 * q + 1] = fma((double)g.y, x, acc[4 * q + 1]);
                    acc[4 * q + 2] = fma((double)g.z, x, acc[4 * q + 2]);
                    acc[4 * q + 3] = fma((double)g.w, x, acc[4 * q + 3]);
                }
            }
        }
    }
    if constexpr (HALVES) {
        if (rlive) {
            double *out = ws.partial64 + (int64_t)tile * S_PAD * R;
#pragma unroll
            for (int s = 0; s < SA; ++s) out[(int64_t)(h * SA + s) * R + r] = acc[s];
        }
        if (tid < S_PAD) ws.occp64[(int64_t)tile * S_PAD + tid] = occ;
    } else {
    if (tid < S_PAD) occs[tid] = occ;
    if (h == 1) {
#pragma unroll
        for (int s = 0; s < S_PAD; ++s) red[s * kMaxR + r] = acc[s];
    }
    __syncthreads();
    if (h == 0 && rlive) {
        double *out = ws.partial64 + (int64_t)tile * S_PAD * R;
#pragma unroll
        for (int s = 0; s < S_PAD; ++s) out[(int64_t)s * R + r] = acc[s] + red[s * kMaxR + r];
    }
    if (tid < S_PAD) ws.occp64[(int64_t)tile * S_PAD + tid] = occs[tid];
    }
}

// ---------------------------------------------------------------------------------------------------------
// speaker model in float64: one CTA per recording, thread = r, speakers in sequence   VBx/VBx.py:95-97,100
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) speaker64_kernel(Plan pl, Workspace ws, RunParams rp, const float *__restrict__ Phi,
                                                        const int32_t *__restrict__ n_states, float *alpha_io,
                                                        float *invL_io) {
    __shared__ double sh[2][4];
    const int rec = blockIdx.x;
    if (!ws.active64[rec]) return;
    const int S = pl.S, R = pl.R, r = threadIdx.x, lane = r & 31, warp = r >> 5;
    const bool live = r < R;
    const int ns = n_states ? n_states[rec] : S;
    const double phi = live ? (double)Phi[r] : 0.0;
    const int t_lo = pl.mtile_begin[rec], t_hi = pl.mtile_begin[rec + 1];
    double regsum = 0.0;
    for (int s = 0; s < S; ++s) {
        const int64_t o = ((int64_t)rec * S + s) * R + r;
        const bool dead = s >= ns;
        double c = 0.0, reg = 0.0, a = 0.0, iL = 0.0;
        if (!dead) {
            double Ns = 0.0, gr = 0.0;
            for (int t = t_lo; t < t_hi; ++t) {
                Ns += ws.occp64[(int64_t)t * S + s];
                if (live) gr += ws.partial64[((int64_t)t * S + s) * R + r];
            }
            if (live) {
                iL = 1.0 / (1.0 + ws.hp[rec].dFaFb * Ns * phi);
                a = ws.hp[rec].dFaFb * iL * gr;
                c = (iL + a * a) * phi;
                reg = log(iL) - iL - a * a + 1.0;
            }
        }
        if (live) {
            ws.alpha64[o] = a;
            if (alpha_io) alpha_io[o] = (float)a;
            if (invL_io) invL_io[o] = (float)iL;
        }
        c = gsum<32>(c);
        reg = gsum<32>(reg);
        __syncthreads();
        if (lane == 0) {
            sh[0][warp] = c;
            sh[1][warp] = reg;
        }
        __syncthreads();
        if (r == 0) {
            ws.bias64[(int64_t)rec * S + s] = dead ? CUDART_INF : 0.5 * ((sh[0][0] + sh[0][1]) + (sh[0][2] + sh[0][3]));
            regsum += (sh[1][0] + sh[1][1]) + (sh[1][2] + sh[1][3]);
        }
    }
    if (r == 0) ws.reg64[rec] = 0.5 * ws.hp[rec].dFb * regsum;
}

// ---------------------------------------------------------------------------------------------------------
// enrolment prior (DESIGN.md section 5.23) around the unchanged speaker64_kernel.  prior_stats64 adds n_e to the
// first M-tile's N_s and sqrt(Phi) F_e to its gamma^T rho, so that speaker64_kernel's tile sums give invL and alpha of
// the prior; prior_reg64 then adds the prior's terms of the regulariser to reg64.  Both leave every value as it is
// where the prior is zero: a recording without a prior gets the bits of a run without one.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) prior_stats64_kernel(Plan pl, Workspace ws, const float *__restrict__ Phi,
                                                            const int32_t *__restrict__ n_states,
                                                            const double *__restrict__ prior_n,
                                                            const double *__restrict__ prior_F) {
    const int rec = blockIdx.x;
    if (!ws.active64[rec]) return;
    const int t = pl.mtile_begin[rec];
    if (t == pl.mtile_begin[rec + 1]) return;
    const int S = pl.S, R = pl.R, r = threadIdx.x;
    const int ns = n_states ? n_states[rec] : S;
    const double sphi = r < R ? sqrt((double)Phi[r]) : 0.0;
    for (int s = 0; s < ns; ++s) {
        const double ne = prior_n[(int64_t)rec * S + s];
        if (r == 0 && ne != 0.0) ws.occp64[(int64_t)t * S + s] += ne;
        if (r < R) {
            const double Fe = prior_F[((int64_t)rec * S + s) * R + r];
            if (Fe != 0.0) ws.partial64[((int64_t)t * S + s) * R + r] += sphi * Fe;
        }
    }
}

// reg64 += Fb/2 sum_{s,r} [log lambda0 - (lambda0 - 1)(invL + d^2) + mu0 (alpha + d)], d = alpha - mu0: the KL divergence
// to N(mu0, 1/lambda0) minus the one to N(0, I) that speaker64_kernel wrote
__global__ void __launch_bounds__(128) prior_reg64_kernel(Plan pl, Workspace ws, const float *__restrict__ Phi,
                                                          const int32_t *__restrict__ n_states,
                                                          const double *__restrict__ prior_n,
                                                          const double *__restrict__ prior_F) {
    __shared__ double sh[4];
    const int rec = blockIdx.x;
    if (!ws.active64[rec]) return;
    const int S = pl.S, R = pl.R, r = threadIdx.x, lane = r & 31, warp = r >> 5;
    const bool live = r < R;
    const int ns = n_states ? n_states[rec] : S;
    const double phi = live ? (double)Phi[r] : 0.0, c = ws.hp[rec].dFaFb;
    const int t_lo = pl.mtile_begin[rec], t_hi = pl.mtile_begin[rec + 1];
    double cor = 0.0;
    for (int s = 0; s < ns && live; ++s) {
        const int64_t o = ((int64_t)rec * S + s) * R + r;
        const double ne = prior_n[(int64_t)rec * S + s], Fe = prior_F[o];
        if (ne == 0.0 && Fe == 0.0) continue;
        double Ns = 0.0;   // N_s + n_e, as speaker64_kernel summed it
        for (int t = t_lo; t < t_hi; ++t) Ns += ws.occp64[(int64_t)t * S + s];
        const double iL = 1.0 / (1.0 + c * Ns * phi), a = ws.alpha64[o];
        const double lam0 = 1.0 + c * ne * phi, mu0 = c * sqrt(phi) * Fe / lam0, d = a - mu0;
        cor += log(lam0) - (lam0 - 1.0) * (iL + d * d) + mu0 * (a + d);
    }
    cor = gsum<32>(cor);
    if (lane == 0) sh[warp] = cor;
    __syncthreads();
    if (r == 0) {
        const double tot = (sh[0] + sh[1]) + (sh[2] + sh[3]);
        if (tot != 0.0) ws.reg64[rec] += 0.5 * ws.hp[rec].dFb * tot;
    }
}

// ---------------------------------------------------------------------------------------------------------
// log-likelihoods in float64.  One CTA per M-tile, processed in blocks of 64 frames: rho block transposed in
// shared memory, alpha [r][s] in shared memory, warp = (state quarter, frame half), lane = frame.  S = 128: blocks of 32
// frames and warp = state eighth (the 64-frame layout would need 225 KB of shared memory).
//   ll[t,s] = Fa (sum_r rho[t,r] alpha[s,r] - bias[s]);  rowmax; p64 = exp(ll - rowmax)       VBx/VBx.py:97
// ---------------------------------------------------------------------------------------------------------
template <int S_PAD>
__host__ __device__ constexpr int loglik64_frames() { return S_PAD > kMaxS ? 32 : 64; }

template <int S_PAD>
__global__ void __launch_bounds__(256) loglik64_kernel(Plan pl, Workspace ws, RunParams rp, const float *__restrict__ rho) {
    constexpr int FB = loglik64_frames<S_PAD>(), SJ = S_PAD > kMaxS ? S_PAD / 8 : (S_PAD / 4 > 0 ? S_PAD / 4 : 1), NSG = S_PAD / SJ;
    extern __shared__ double sm64[];
    const int R = pl.R;
    double *aS = sm64;                                   // [S_PAD][kMaxR]
    double *llS = aS + kMaxR * S_PAD;                    // [FB][S_PAD]
    float *xS = reinterpret_cast<float *>(llS + FB * S_PAD);   // [R][FB + 1]
    __shared__ double mxS[FB];
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active64[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < S_PAD * R; i += 256) {
        const int s = i / R, r = i - s * R;
        aS[s * kMaxR + r] = ws.alpha64[((int64_t)rec * S_PAD + s) * R + r];
    }
    const int sg = warp % NSG, fh = warp / NSG;          // NSG = 4 (S >= 4): fh in 0..1
    double nb[SJ];
#pragma unroll
    for (int j = 0; j < SJ; ++j) nb[j] = ws.bias64[(int64_t)rec * S_PAD + sg * SJ + j];
    for (int b0 = 0; b0 < len; b0 += FB) {
        const int bl = min(FB, len - b0);
        __syncthreads();
        for (int i = tid; i < FB * R; i += 256) {
            const int f = i / R, r = i - f * R;
            xS[r * (FB + 1) + f] = f < bl ? __ldg(rho + (f0 + b0 + f) * R + r) : 0.f;
        }
        __syncthreads();
        const int f = fh * 32 + lane;
        double acc[SJ];
#pragma unroll
        for (int j = 0; j < SJ; ++j) acc[j] = 0.0;
        for (int r = 0; r < R; ++r) {
            const double x = (double)xS[r * (FB + 1) + f];
            const double *ar = aS + sg * SJ * kMaxR + r;
#pragma unroll
            for (int j = 0; j < SJ; ++j) acc[j] = fma(x, ar[j * kMaxR], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < SJ; ++j) llS[f * S_PAD + sg * SJ + j] = nb[j] < CUDART_INF ? ws.hp[rec].dFa * (acc[j] - nb[j]) : -CUDART_INF;
        __syncthreads();
        if (tid < FB) {
            double m = -CUDART_INF;
            for (int s = 0; s < S_PAD; ++s) m = fmax(m, llS[tid * S_PAD + s]);
            mxS[tid] = m;
            if (tid < bl) ws.rowmax64[f0 + b0 + tid] = m;
        }
        __syncthreads();
        double *out = ws.p64 + (f0 + b0) * S_PAD;
        for (int i = tid; i < bl * S_PAD; i += 256) {
            const double v = llS[i];
            out[i] = v > -CUDART_INF ? exp(v - mxS[i / S_PAD]) : 0.0;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// forward-backward in float64 (scaled linear domain, O(S) transition structure; see vbx_kernels.cu for the
// derivation).  A group of LPR lanes owns one recording, SPL states per lane.  The normalised forward variables
// are parked in gamma (float32: gamma = a o b is rounded to float32 anyway), the scales stay float64.
// ---------------------------------------------------------------------------------------------------------
template <int N>
struct DVec {
    double v[N];
};
template <int N>
__device__ __forceinline__ DVec<N> ld_d(const double *p) {
    DVec<N> r;
    if (N == 2) {
        const double2 t = *reinterpret_cast<const double2 *>(p);
        r.v[0] = t.x;
        r.v[N - 1] = t.y;
    } else {
#pragma unroll
        for (int k = 0; k < N; ++k) r.v[k] = p[k];
    }
    return r;
}

template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) fb64_kernel(Plan pl, Workspace ws, RunParams rp, float *gamma, float *pi_io,
                                                   const int32_t *__restrict__ n_states) {
    constexpr int LPR = S_PAD / SPL;
    constexpr int RPW = 32 / LPR;
    constexpr int PF = 8;
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int g = lane / LPR, l = lane % LPR;
    const int slot = warp_global * RPW + g;
    int rec = -1;
    if (slot < pl.n_rec) rec = pl.order[slot];
    const bool live = rec >= 0 && ws.active64[rec] != 0;
    int64_t f0 = 0;
    int T = 0;
    if (live) {
        f0 = pl.offsets[rec];
        T = (int)(pl.offsets[rec + 1] - f0);
    }
    int Tmax = T;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) Tmax = max(Tmax, __shfl_xor_sync(0xffffffffu, Tmax, off));
    if (Tmax == 0) return;
    const int Tlast = max(T - 1, 0);
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    const double P = rec >= 0 ? ws.hp[rec].dloopP : 0.0, Q = 1.0 - P, eps = 1e-8;
    double pi[SPL], w[SPL], base[SPL], a[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        pi[k] = sl ? ws.pi64[(int64_t)rec * S_PAD + s] : 0.0;
        w[k] = sl ? Q * pi[k] + eps : 0.0;          // VBx/VBx.py:98,159
        base[k] = sl ? pi[k] + eps : 0.0;           // VBx/VBx.py:164
        a[k] = 0.0;
    }
    const double *pp = ws.p64 + f0 * S_PAD + l * SPL;
    float *ga = gamma + f0 * S_PAD + l * SPL;
    double *rs = ws.rsig64 + f0;

    // ---------------- forward, VBx/VBx.py:164,167-168 ----------------
    {
        DVec<SPL> bufA[PF], bufB[PF];      // ping-pong register bursts (named, so that they stay in registers)
        auto fchunk = [&](const int t0, DVec<SPL>(&cur)[PF], DVec<SPL>(&nxt)[PF]) {
#pragma unroll
            for (int i = 0; i < PF; ++i) nxt[i] = ld_d<SPL>(pp + (int64_t)min(t0 + PF + i, Tlast) * S_PAD);
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                const int t = t0 + i;
                double v[SPL], loc = 0.0;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    v[k] = cur[i].v[k] * base[k];
                    loc += v[k];
                }
                const double sig = gsum<LPR>(loc);
                const double r = 1.0 / sig;
                const bool act = t < T;
                float an[SPL];
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    const double av = v[k] * r;
                    a[k] = act ? av : a[k];
                    base[k] = act ? fma(P, av, w[k]) : base[k];
                    an[k] = (float)av;
                }
                if (act) {
                    st_vec<SPL>(ga + (int64_t)t * S_PAD, an);
                    if (l == 0) rs[t] = r;
                }
            }
        };
#pragma unroll
        for (int i = 0; i < PF; ++i) bufA[i] = ld_d<SPL>(pp + (int64_t)min(i, Tlast) * S_PAD);
        for (int t0 = 0; t0 < Tmax; t0 += 2 * PF) {
            fchunk(t0, bufA, bufB);
            fchunk(t0 + PF, bufB, bufA);
        }
    }
    __syncwarp();

    // ---------------- backward, VBx/VBx.py:165,170-171,174 and the statistics of eq. (24) ----------------
    double b[SPL], g0[SPL], enter[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        b[k] = 1.0;
        g0[k] = a[k];
        enter[k] = 0.0;
    }
    {
        constexpr int PB = 4;
        struct Slot {
            DVec<SPL> p;
            Vec<SPL> a;
            double r;
        };
        auto load_slot = [&](const int ii) {
            const int t = max(T - 2 - ii, 0);
            const int t1 = min(t + 1, Tlast);
            Slot sl;
            sl.p = ld_d<SPL>(pp + (int64_t)t1 * S_PAD);
            sl.a = ld_vec<SPL>(ga + (int64_t)t * S_PAD);
            sl.r = rs[t1];
            return sl;
        };
        Slot bufA[PB], bufB[PB];
        auto bchunk = [&](const int i0, Slot(&cur)[PB], Slot(&nxt)[PB]) {
#pragma unroll
            for (int i = 0; i < PB; ++i) nxt[i] = load_slot(i0 + PB + i);
#pragma unroll
            for (int i = 0; i < PB; ++i) {
                const Slot &c = cur[i];
                const int t = T - 2 - (i0 + i);
                const bool act = t >= 0;
                double u[SPL], loc = 0.0;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    u[k] = (c.p.v[k] * c.r) * b[k];
                    loc = fma(w[k], u[k], loc);
                }
                const double dot = gsum<LPR>(loc);
                double gn[SPL], bn[SPL], gsl = 0.0;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    bn[k] = fma(P, u[k], dot);
                    gn[k] = (double)c.a.v[k] * bn[k];
                    gsl += gn[k];
                }
                const double sc = 1.0 / gsum<LPR>(gsl);      // rows of gamma sum to one
                float gf[SPL];
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    gn[k] *= sc;
                    gf[k] = (float)gn[k];
                    b[k] = act ? bn[k] : b[k];
                    g0[k] = act ? gn[k] : g0[k];
                    enter[k] += act ? u[k] : 0.0;
                }
                if (act) st_vec<SPL>(ga + (int64_t)t * S_PAD, gf);
            }
        };
#pragma unroll
        for (int i = 0; i < PB; ++i) bufA[i] = load_slot(i);
        for (int i0 = 0; i0 < Tmax - 1; i0 += 2 * PB) {
            bchunk(i0, bufA, bufB);
            bchunk(i0 + PB, bufB, bufA);
        }
    }
    // ---------------- eq. (24), VBx/VBx.py:101-104 ----------------
    double pn[SPL], loc = 0.0;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        pn[k] = g0[k] + Q * pi[k] * enter[k];
        loc += pn[k];
    }
    const double tot = gsum<LPR>(loc);
    if (live) {
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            const int s = l * SPL + k;
            const double v = pn[k] / tot;
            ws.pi64[(int64_t)rec * S_PAD + s] = v;
            pi_io[(int64_t)rec * S_PAD + s] = (float)v;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// ELBO, trace and the reference's stop test on float64 values                VBx/VBx.py:100,105,122-125,173
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) elbo64_kernel(Plan pl, Workspace ws, RunParams rp, double *Li, int32_t *n_iters,
                                                     int32_t *flags) {
    const int rec = blockIdx.x;
    if (!ws.active64[rec]) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t f0 = pl.offsets[rec];
    const int T = (int)(pl.offsets[rec + 1] - f0);
    double acc = 0.0;
    for (int t = tid; t < T; t += 128) acc += ws.rowmax64[f0 + t] - log(ws.rsig64[f0 + t]);
    acc = gsum<32>(acc);
    __shared__ double part[4];
    if (lane == 0) part[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        const double elbo = (part[0] + part[1]) + (part[2] + part[3]) + ws.hp[rec].dFa * ws.gsum[rec] + ws.reg64[rec];
        const int idx = n_iters[rec];
        Li[(int64_t)rec * rp.max_iters + idx] = elbo;
        n_iters[rec] = idx + 1;
        int fl = flags[rec];
        if (!isfinite(elbo)) fl |= 1;
        const int fr = ws.fresh[rec];
        ws.fresh[rec] = 0;
        bool stop = false;
        if (idx > 0 && fr != 1) {       // fr == 1: the float32 kernels saw this step safely above epsilon -> no test here
            const double d = elbo - ws.prev_elbo[rec];
            if (d < rp.epsilon) {
                stop = true;
                if (idx + 1 < rp.max_iters) fl |= 4;
                if (d < 0.0) fl |= 2;
            }
        }
        if (stop || idx + 1 >= rp.max_iters) ws.active64[rec] = 0;
        ws.prev_elbo[rec] = elbo;
        flags[rec] = fl;
    }
}

}  // namespace x64

int launch_snapshot(const Plan &pl, const Workspace &ws, const float *gamma, const float *pi, int iter, cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    x64::snapshot_kernel<<<pl.n_mtiles, 256, 0, st>>>(pl, ws, gamma, pi, iter & 1);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <int S_PAD>
static int launch_exact64_t(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *rho, const float *Phi,
                            float *gamma, float *pi, const int32_t *n_states, float *alpha_io, float *invL_io, double *Li,
                            int32_t *n_iters, int32_t *flags, cudaStream_t st, const double *prior_n,
                            const double *prior_F) {
    constexpr int SPL = S_PAD > kMaxS ? 4 : (S_PAD >= 16 ? 2 : 1);
    constexpr int RPW = 32 / (S_PAD / SPL);
    constexpr int FB = x64::loglik64_frames<S_PAD>();
    const size_t sm_m = S_PAD > kMaxS ? 0 : (size_t)S_PAD * kMaxR * sizeof(double);   // S = 128: no parity reduction
    const size_t sm_l = (size_t)(kMaxR * S_PAD + FB * S_PAD) * sizeof(double) + (size_t)kMaxR * (FB + 1) * sizeof(float);
    if (!allow_dynamic_smem(x64::mstep64_kernel<S_PAD>, (int)sm_m) || !allow_dynamic_smem(x64::loglik64_kernel<S_PAD>, (int)sm_l))
        return -1;
    x64::restore64_kernel<<<pl.n_mtiles, 256, 0, st>>>(pl, ws, gamma, n_iters);
    x64::mstep64_kernel<S_PAD><<<pl.n_mtiles, 256, sm_m, st>>>(pl, ws, rho, gamma);
    if (prior_n) x64::prior_stats64_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, Phi, n_states, prior_n, prior_F);
    x64::speaker64_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, rp, Phi, n_states, alpha_io, invL_io);
    if (prior_n) x64::prior_reg64_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, Phi, n_states, prior_n, prior_F);
    x64::loglik64_kernel<S_PAD><<<pl.n_mtiles, 256, sm_l, st>>>(pl, ws, rp, rho);
    const int warps = (pl.n_rec + RPW - 1) / RPW;
    x64::fb64_kernel<S_PAD, SPL><<<(warps + 3) / 4, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    x64::elbo64_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, rp, Li, n_iters, flags);
    return cudaGetLastError() == cudaSuccess ? (prior_n ? 8 : 6) : -1;
}

// One float64 iteration for every recording in the finishing phase (ws.active64).
int launch_exact64_round(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *rho, const float *Phi,
                         float *gamma, float *pi, const int32_t *n_states, float *alpha_io, float *invL_io, double *Li,
                         int32_t *n_iters, int32_t *flags, cudaStream_t st, const double *prior_n,
                         const double *prior_F) {
    if (pl.n_rec == 0 || pl.n_mtiles == 0) return 0;
#define VBX_X64(S_) return launch_exact64_t<S_>(pl, ws, rp, rho, Phi, gamma, pi, n_states, alpha_io, invL_io, Li, n_iters, flags, st, \
                                                prior_n, prior_F)
    switch (pl.S) {
        case 4: VBX_X64(4);
        case 8: VBX_X64(8);
        case 16: VBX_X64(16);
        case 32: VBX_X64(32);
        case 64: VBX_X64(64);
        case kMaxSWide: VBX_X64(kMaxSWide);
        default: return -1;
    }
#undef VBX_X64
}

}  // namespace vbx
