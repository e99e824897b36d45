// Forward-backward with the two sweeps running CONCURRENTLY on different warps           VBx/VBx.py:98-104,146-175
//
// The fused kernel (vbx_kernels.cu) walks a recording forward and then backward on the same lanes: 2 T dependent steps.
// When the batch cannot fill the GPU with recordings (BASELINE configs 2, 4, 5 and the one-recording drop-in call) that
// sequential latency IS the iteration time.  Here the backward sweep does not wait for the forward scales: it carries
// its own scaling, both sweeps start together on separate warps, and a fully T-parallel pass combines them
// (SURVEY.md section 7, hard part 1; verified exact there):
//     forward   a_t  = normalised forward variables, 1/sigma_t             (as in the fused kernel, look-ahead form)
//     backward  bh_t = backward variables up to a per-frame factor         (look-ahead form, self-scaled)
//     combine   gamma_t = a_t o bh_t / sum ;   Z_t = sum_j p_tj bh_tj (P a_{t-1,j} + w_j) ;
//               re-entry statistics of eq. (24): enter_j = sum_{t>=1} p_tj bh_tj / Z_t ;   N_s = sum_t gamma_ts
// Every quantity the rest of the iteration reads (gamma, pi, N_s, 1/sigma_t for the ELBO) has the same meaning as in
// the fused kernel; results differ from it by float32 rounding only.  Recordings of any length take this path (no
// chunked scan needed: a 12 000-frame recording costs 12 000 look-ahead steps, ~0.4 ms).
//
// Backward scaling.  Unscaled, B_t = P p_{t+1} o B_{t+1} + D_t with D_t = w . (p_{t+1} o B_{t+1}) shrinks by the factor
// tau_t = D_t / D_{t+1} in [1e-8, S] per frame.  The sweep multiplies step t by rho_t = 1 / tau_{t+3} (the true factor
// of three frames earlier, so its reciprocal is off the dependency chain); then d_t = tau_t tau_{t+1} tau_{t+2} stays
// within [1e-24, S^3] and b_t / d_t within [1, 1e8] for any recording length.
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

template <int LANES>
__device__ __forceinline__ float gsum(float v) {
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}
// index shuffle pinned in program order (see vbx_kernels.cu: keeps each hand-out of a per-frame scalar inside its step)
__device__ __forceinline__ float shfl_pin(const float v, const int src) {
    float r;
    asm volatile("shfl.sync.idx.b32 %0, %1, %2, 0x1f, 0xffffffff;" : "=f"(r) : "f"(v), "r"(src));
    return r;
}
__device__ __forceinline__ float rcpf(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// ordered loads / stores (see vbx_kernels.cu: volatile accesses keep a prefetch burst ahead of the first store of its chunk)
template <int N>
__device__ __forceinline__ Vec<N> ldo(const float *p);
template <>
__device__ __forceinline__ Vec<1> ldo<1>(const float *p) {
    Vec<1> r;
    asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(r.v[0]) : "l"(p) : "memory");
    return r;
}
template <>
__device__ __forceinline__ Vec<2> ldo<2>(const float *p) {
    Vec<2> r;
    asm volatile("ld.volatile.global.v2.f32 {%0, %1}, [%2];" : "=f"(r.v[0]), "=f"(r.v[1]) : "l"(p) : "memory");
    return r;
}
template <>
__device__ __forceinline__ Vec<4> ldo<4>(const float *p) {
    Vec<4> r;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3]) : "l"(p) : "memory");
    return r;
}
template <int N>
__device__ __forceinline__ void sto(float *p, const float *v);
template <>
__device__ __forceinline__ void sto<1>(float *p, const float *v) {
    asm volatile("st.volatile.global.f32 [%0], %1;" ::"l"(p), "f"(v[0]) : "memory");
}
template <>
__device__ __forceinline__ void sto<2>(float *p, const float *v) {
    asm volatile("st.volatile.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
}
template <>
__device__ __forceinline__ void sto<4>(float *p, const float *v) {
    asm volatile("st.volatile.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
}

// ------------------------------------------------------------------------------------------------
// sweeps: warps [0, n_warps) run the forward sweep of their recordings, warps [n_warps, 2 n_warps) the backward sweep
// ------------------------------------------------------------------------------------------------
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) fb_sweeps_kernel(Plan pl, Workspace ws, RunParams rp, const float *__restrict__ pi_io,
                                                        const int32_t *__restrict__ n_states, int n_warps) {
    constexpr int LPR = S_PAD / SPL;
    constexpr int RPW = 32 / LPR;
    constexpr int PF = (SPL == 4) ? 10 : (SPL == 2 ? 20 : 24);   // frames per prefetch burst (ping-pong register sets)
    const int lane = threadIdx.x & 31;
    int warp_global = blockIdx.x * 4 + (threadIdx.x >> 5);
    const bool backward = warp_global >= n_warps;               // warp-uniform role
    if (backward) warp_global -= n_warps;
    const int g = lane / LPR, l = lane % LPR;
    const int slot = warp_global * RPW + g;
    int rec = -1;
    if (slot < pl.n_rec) rec = pl.order[slot];
    const bool live = rec >= 0 && ws.active[rec] != 0;
    int64_t f0 = 0;
    int T = 0;
    if (live) {
        f0 = pl.offsets[rec];
        T = (int)(pl.offsets[rec + 1] - f0);
    }
    int Tmax = T, Tmin = live ? T : 0x7fffffff;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        Tmax = max(Tmax, __shfl_xor_sync(0xffffffffu, Tmax, off));
        Tmin = min(Tmin, __shfl_xor_sync(0xffffffffu, Tmin, off));
    }
    if (Tmax == 0) return;  // warp-uniform: no live recording in this warp
    const int Tlast = max(T - 1, 0);
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    const float P = rec >= 0 ? ws.hp[rec].loopP : 0.f, Q = 1.f - P;
    float pi[SPL], w[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        pi[k] = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pi[k], VBX_EPS_TR) : 0.f;   // VBx/VBx.py:98,159
    }
    // groups without a recording read row 0 of the batch and write into a scratch row (stride 0): no predicates in the loops
    const float *pp = ws.p + f0 * S_PAD + l * SPL;
    const float *cv = ws.cvec + f0;         // c_t = p_t . w from the log-likelihood kernel
    const int64_t ostr = live ? S_PAD : 0;
    const int gl0 = lane - l;               // first lane of this group
    constexpr int NC = (PF + LPR - 1) / LPR; // per burst every lane keeps NC of the c values, handed out by shuffle

    if (!backward) {
        // ---------------- forward sweep, VBx/VBx.py:164,167-168 (look-ahead recurrences, see vbx_kernels.cu) ----------------
        float *ah = live ? ws.ahat + f0 * S_PAD + l * SPL : ws.scratch + l * SPL;
        float *rs = live ? ws.rsigma + f0 : ws.scratch + (S_PAD > kMaxS ? S_PAD : kMaxS);
        const int rstr = live ? 1 : 0;
        float y[SPL];
        const Vec<SPL> p0 = ldg_vec<SPL>(pp);
        const Vec<SPL> p1 = ldg_vec<SPL>(pp + (int64_t)min(1, Tlast) * S_PAD);
        float loc = 0.f, locq = 0.f;
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            const int s = l * SPL + k;
            y[k] = (live && s < ns) ? p0.v[k] * (pi[k] + VBX_EPS_TR) : 0.f;   // VBx/VBx.py:164
            loc += y[k];
            locq = fmaf(p1.v[k], y[k], locq);
        }
        float Yc = gsum<LPR>(loc);     // Y_0 = sigma_0
        float q = gsum<LPR>(locq);     // q_0 = p_1 . y_0
        float c = __ldg(cv + min(1, Tlast));   // c_1 = p_1 . w
        float rn = 1.f;                 // r_1
        float rs1 = rcpf(Yc);           // 1/sigma_0 (becomes r_2)
        {
            float an[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) an[k] = y[k] * rs1;
            st_vec<SPL>(ah, an);
            if (l == 0) rs[0] = rs1;
        }
        auto fstep = [&](const int j, const Vec<SPL> &ps, const Vec<SPL> &pn, const float cn, const bool check) {
            const int s = j + 1;
            float ys[SPL], lq = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                ys[k] = (rn * ps.v[k]) * fmaf(P, y[k], w[k] * Yc);
                lq = fmaf(pn.v[k], ys[k], lq);
            }
            const float qn = gsum<LPR>(lq);                    // consumed by the NEXT step
            const float Ys = rn * fmaf(P, q, c * Yc);           // Y_s = sum_i y_s,i
            const float inv = rcpf(Ys);
            const float rsig = rn * Yc * inv;                   // 1 / sigma_s
            float an[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                an[k] = ys[k] * inv;
                y[k] = ys[k];
            }
            Yc = Ys;
            q = qn;
            c = cn;
            rn = rs1;
            rs1 = rsig;
            if (!check || s < T) {
                sto<SPL>(ah + s * ostr, an);
                if (l == 0) rs[s * rstr] = rsig;
            }
        };
        Vec<SPL> bufA[PF], bufB[PF];
        float cbA[NC], cbB[NC];             // lane l keeps c of the frames (burst start) + k LPR + l
        Vec<SPL> ps = p1;
        // slot i of a burst starting at step j0 holds the row (and c) of frame j0 + i + 2
        auto fchunk = [&](const int j0, Vec<SPL>(&cur)[PF], Vec<SPL>(&nxt)[PF], const float (&cc)[NC], float (&nc)[NC], const bool check) {
#pragma unroll
            for (int i = 0; i < PF; ++i) nxt[i] = ldo<SPL>(pp + (int64_t)min(j0 + PF + i + 2, Tlast) * S_PAD);
#pragma unroll
            for (int k = 0; k < NC; ++k) nc[k] = ldo<1>(cv + min(j0 + PF + 2 + k * LPR + l, Tlast)).v[0];
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                fstep(j0 + i, ps, cur[i], shfl_pin(cc[i / LPR], gl0 + i % LPR), check);
                ps = cur[i];
            }
        };
#pragma unroll
        for (int i = 0; i < PF; ++i) bufA[i] = ldg_vec<SPL>(pp + (int64_t)min(i + 2, Tlast) * S_PAD);
#pragma unroll
        for (int k = 0; k < NC; ++k) cbA[k] = __ldg(cv + min(2 + k * LPR + l, Tlast));
        int j0 = 0;
        for (; j0 + 2 * PF <= Tmin - 1; j0 += 2 * PF) {
            fchunk(j0, bufA, bufB, cbA, cbB, false);
            fchunk(j0 + PF, bufB, bufA, cbB, cbA, false);
        }
        for (; j0 < Tmax - 1; j0 += 2 * PF) {
            fchunk(j0, bufA, bufB, cbA, cbB, true);
            fchunk(j0 + PF, bufB, bufA, cbB, cbA, true);
        }
    } else {
        // ---------------- backward sweep, VBx/VBx.py:165,170-171 (self-scaled look-ahead recurrences) ----------------
        //   v_t = kappa_{t+1} o b_{t+1},  kappa_{t+1} = rho_t p_{t+1};   b_t = P v_t + d_t;
        //   d_t = w . v_t = P e_{t+1} + d_{t+1} f_{t+1},   e_{t+1} = (w o kappa_{t+1}) . v_{t+1},   f_{t+1} = w . kappa_{t+1}
        float *bh = live ? ws.bhat + f0 * S_PAD + l * SPL : ws.scratch + l * SPL;
        float b[SPL], kap[SPL];
        // frame T-1: b = 1 = P * 0 + 1, i.e. v_{T-1} = 0, d_{T-1} = 1, e_{T-1} = 0
        {
            float one[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) one[k] = 1.f;
            st_vec<SPL>(bh + (int64_t)Tlast * ostr, one);
        }
        float dprev = 1.f, e = 0.f, f;
        float rho0 = 1.f, rho1 = 1.f, rho2 = 1.f;   // rho_t (forms kappa_{t+1} of the running step), rho_{t-1}, rho_{t-2}
        const Vec<SPL> plast = ldg_vec<SPL>(pp + (int64_t)Tlast * S_PAD);
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            b[k] = 1.f;
            kap[k] = plast.v[k];                     // rho_{T-2} = 1
        }
        f = __ldg(cv + Tlast);                       // f_{T-1} = w . kappa_{T-1} = c_{T-1}
        // step ii handles frame t = T-2-ii with pt = p_t (row of frame t, needed for kappa_t) and ct = c_t = p_t . w
        auto bstep = [&](const int ii, const Vec<SPL> &pt, const float ct, const bool check) {
            const int t = T - 2 - ii;
            float v[SPL], kapn[SPL], loce = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                v[k] = kap[k] * b[k];                               // v_t
                kapn[k] = rho1 * pt.v[k];                           // kappa_t = rho_{t-1} p_t
                loce = fmaf(w[k] * kapn[k], v[k], loce);
            }
            const float en = gsum<LPR>(loce);                       // e_t, consumed by the NEXT step
            const float fn = rho1 * ct;                             // f_t = w . kappa_t (no reduction: c is precomputed)
            const float d = fmaf(P, e, dprev * f);                  // d_t = w . v_t
            float bn[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) bn[k] = fmaf(P, v[k], d);
            // rho_{t-3} = 1 / tau_t = rho_t d_{t+1} / d_t  (off the chain: used three steps from now)
            const float rho3 = rho0 * dprev * rcpf(d);
            if (!check || t >= 0) sto<SPL>(bh + t * ostr, bn);
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                b[k] = bn[k];
                kap[k] = kapn[k];
            }
            dprev = d;
            e = en;
            f = fn;
            rho0 = rho1;
            rho1 = rho2;
            rho2 = rho3;
        };
        Vec<SPL> bufA[PF], bufB[PF];
        float cbA[NC], cbB[NC];
        // slot i of a burst starting at step i0 holds the row (and c) of frame T-2-(i0+i)
        auto bchunk = [&](const int i0, Vec<SPL>(&cur)[PF], Vec<SPL>(&nxt)[PF], const float (&cc)[NC], float (&nc)[NC], const bool check) {
#pragma unroll
            for (int i = 0; i < PF; ++i) nxt[i] = ldo<SPL>(pp + (int64_t)max(T - 2 - (i0 + PF + i), 0) * S_PAD);
#pragma unroll
            for (int k = 0; k < NC; ++k) nc[k] = ldo<1>(cv + max(T - 2 - (i0 + PF + k * LPR + l), 0)).v[0];
#pragma unroll
            for (int i = 0; i < PF; ++i) bstep(i0 + i, cur[i], shfl_pin(cc[i / LPR], gl0 + i % LPR), check);
        };
#pragma unroll
        for (int i = 0; i < PF; ++i) bufA[i] = ldg_vec<SPL>(pp + (int64_t)max(T - 2 - i, 0) * S_PAD);
#pragma unroll
        for (int k = 0; k < NC; ++k) cbA[k] = __ldg(cv + max(T - 2 - (k * LPR + l), 0));
        int i0 = 0;
        for (; i0 + 2 * PF <= Tmin - 1; i0 += 2 * PF) {
            bchunk(i0, bufA, bufB, cbA, cbB, false);
            bchunk(i0 + PF, bufB, bufA, cbB, cbA, false);
        }
        for (; i0 < Tmax - 1; i0 += 2 * PF) {
            bchunk(i0, bufA, bufB, cbA, cbB, true);
            bchunk(i0 + PF, bufB, bufA, cbB, cbA, true);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// combine: one CTA per M-tile (512 frames of one recording), sub-blocks of FBK frames; LPF lanes share a frame
// ------------------------------------------------------------------------------------------------
template <int S_PAD>
__global__ void __launch_bounds__(256) fb_combine_kernel(Plan pl, Workspace ws, RunParams rp, float *__restrict__ gamma,
                                                         const float *__restrict__ pi_io, const int32_t *__restrict__ n_states) {
    constexpr int SC = S_PAD < 16 ? S_PAD : 16;   // states per lane
    constexpr int LPF = S_PAD / SC;               // lanes per frame: 1, 2 (S=32), 4 (S=64)
    constexpr int FBK = 256 / LPF;                // frames per sub-block
    constexpr int LD = 2 * S_PAD + 1;             // row: gamma[S_PAD], u[S_PAD], pad
    constexpr int NCOL = 2 * S_PAD;
    constexpr int NPART = 256 / NCOL;             // row groups of the column sums
    extern __shared__ float smf[];
    float *rows = smf;                            // [FBK][LD]
    float *psum = smf + FBK * LD;                 // [NPART][NCOL]
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t rf0 = pl.offsets[rec];
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int ns = n_states ? n_states[rec] : S_PAD;
    const int tid = threadIdx.x;
    const int fl = tid / LPF, sc = tid % LPF;     // frame slot, state chunk
    const float P = ws.hp[rec].loopP, Q = 1.f - P;
    float w[SC];
#pragma unroll
    for (int k = 0; k < SC; ++k) {
        const int s = sc * SC + k;
        w[k] = s < ns ? fmaf(Q, pi_io[(int64_t)rec * S_PAD + s], VBX_EPS_TR) : 0.f;
    }
    double tot = 0.0;                             // running column sum of this thread's column (tid < NCOL)
    for (int b0 = 0; b0 < len; b0 += FBK) {
        const int bl = min(FBK, len - b0);
        float g[SC], u[SC];
#pragma unroll
        for (int k = 0; k < SC; ++k) g[k] = u[k] = 0.f;
        const bool on = fl < bl;
        const int64_t fr = f0 + b0 + (on ? fl : 0);                   // global frame (lanes past the block end idle on frame b0)
        const bool first = fr == rf0;                                 // frame 0 of the recording: no re-entry term
        float gs = 0.f, z = 0.f;
        if (on) {
            const float *pa = ws.ahat + fr * S_PAD + sc * SC;
            const float *pb = ws.bhat + fr * S_PAD + sc * SC;
            const float *pq = ws.p + fr * S_PAD + sc * SC;
            const float *pm = ws.ahat + (first ? fr : fr - 1) * S_PAD + sc * SC;
#pragma unroll
            for (int k4 = 0; k4 < SC / 4; ++k4) {
                const float4 a = *reinterpret_cast<const float4 *>(pa + 4 * k4);
                const float4 bb = *reinterpret_cast<const float4 *>(pb + 4 * k4);
                const float4 pp = *reinterpret_cast<const float4 *>(pq + 4 * k4);
                const float4 am = *reinterpret_cast<const float4 *>(pm + 4 * k4);
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w}, pv[4] = {pp.x, pp.y, pp.z, pp.w},
                            mv[4] = {am.x, am.y, am.z, am.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int k = 4 * k4 + i;
                    g[k] = av[i] * bv[i];
                    u[k] = pv[i] * bv[i];
                    gs += g[k];
                    z = fmaf(u[k], fmaf(P, mv[i], w[k]), z);
                }
            }
        }
        // the LPF lanes of a frame are adjacent and on/off together, but a warp may hold both kinds: the shuffles run
        // unconditionally (a full-mask shuffle inside `if (on)` deadlocks as soon as a tile ends inside a warp)
        gs = gsum<LPF>(gs);
        z = gsum<LPF>(z);
        if (on) {
            const float ig = 1.f / gs, iz = first ? 0.f : 1.f / z;
#pragma unroll
            for (int k = 0; k < SC; ++k) {
                g[k] *= ig;
                u[k] *= iz;
            }
            float *go = gamma + fr * S_PAD + sc * SC;
#pragma unroll
            for (int k4 = 0; k4 < SC / 4; ++k4)
                *reinterpret_cast<float4 *>(go + 4 * k4) = make_float4(g[4 * k4], g[4 * k4 + 1], g[4 * k4 + 2], g[4 * k4 + 3]);
        }
        __syncthreads();                                          // previous sub-block's column sums are done
#pragma unroll
        for (int k = 0; k < SC; ++k) {
            rows[fl * LD + sc * SC + k] = g[k];                   // frames >= bl contribute zeros
            rows[fl * LD + S_PAD + sc * SC + k] = u[k];
        }
        __syncthreads();
        if (tid < NPART * NCOL) {
            const int col = tid % NCOL, part = tid / NCOL;
            float s = 0.f;
            for (int r = part; r < FBK; r += NPART) s += rows[r * LD + col];
            psum[part * NCOL + col] = s;
        }
        __syncthreads();
        if (tid < NCOL) {
            double s = 0.0;
#pragma unroll 4
            for (int part = 0; part < NPART; ++part) s += (double)psum[part * NCOL + tid];
            tot += s;
        }
    }
    if (tid < S_PAD)
        ws.socc[(int64_t)tile * S_PAD + tid] = (float)tot;
    else if (tid < NCOL)
        ws.sent[(int64_t)tile * S_PAD + tid - S_PAD] = (float)tot;
}

// ------------------------------------------------------------------------------------------------
// tail: N_s and eq. (24) per recording (one warp, tile partials in tile order)            VBx/VBx.py:95,101-104
// ------------------------------------------------------------------------------------------------
template <int S_PAD>
__global__ void __launch_bounds__(128) fb_split_tail_kernel(Plan pl, Workspace ws, RunParams rp, const float *__restrict__ gamma,
                                                            float *pi_io, const int32_t *__restrict__ n_states) {
    const int rec = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (rec >= pl.n_rec || !ws.active[rec]) return;       // warp-uniform
    const int lane = threadIdx.x & 31;
    const int ns = n_states ? n_states[rec] : S_PAD;
    const int64_t f0 = pl.offsets[rec];
    const int t_lo = pl.mtile_begin[rec], t_hi = pl.mtile_begin[rec + 1];
    constexpr int SPLc = S_PAD > 32 ? S_PAD / 32 : 1;
    const double Q = 1.0 - (double)ws.hp[rec].loopP;
    double pn[SPLc];
    float loc = 0.f;
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        pn[k] = 0.0;
        if (s < S_PAD) {
            double occ = 0.0, ent = 0.0;
            for (int t = t_lo; t < t_hi; ++t) {
                occ += (double)ws.socc[(int64_t)t * S_PAD + s];
                ent += (double)ws.sent[(int64_t)t * S_PAD + s];
            }
            ws.occ[(int64_t)rec * S_PAD + s] = (float)occ;
            const double pik = s < ns ? (double)pi_io[(int64_t)rec * S_PAD + s] : 0.0;
            pn[k] = (double)gamma[f0 * S_PAD + s] + Q * pik * ent;
            loc += (float)pn[k];
        }
    }
    const float tot = gsum<32>(loc);
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        if (s < S_PAD) pi_io[(int64_t)rec * S_PAD + s] = (float)(pn[k] / (double)tot);
    }
}

template <int S_PAD, int SPL>
int launch_split_t(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi, const int32_t *n_states,
                   cudaStream_t st) {
    constexpr int RPW = 32 / (S_PAD / SPL);
    constexpr int LPF = S_PAD / (S_PAD < 16 ? S_PAD : 16), FBK = 256 / LPF, LD = 2 * S_PAD + 1, NCOL = 2 * S_PAD, NPART = 256 / NCOL;
    const int n_warps = (pl.n_rec + RPW - 1) / RPW;
    const int blocks = (2 * n_warps + 3) / 4;
    const size_t smem = (size_t)(FBK * LD + NPART * NCOL) * sizeof(float);
    if (!allow_dynamic_smem(fb_combine_kernel<S_PAD>, (int)smem)) return -1;
    fb_sweeps_kernel<S_PAD, SPL><<<blocks, 128, 0, st>>>(pl, ws, rp, pi, n_states, n_warps);
    fb_combine_kernel<S_PAD><<<pl.n_mtiles, 256, smem, st>>>(pl, ws, rp, gamma, pi, n_states);
    fb_split_tail_kernel<S_PAD><<<(pl.n_rec + 3) / 4, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    return cudaGetLastError() == cudaSuccess ? 3 : -1;
}

}  // namespace

// spl: states per lane of the sweeps (0 = default: 2 from 16 states up, else 1)
int launch_forward_backward_split(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                  const int32_t *n_states, int spl, cudaStream_t st) {
    if (pl.n_rec == 0 || pl.n_mtiles == 0) return 0;
#define VBX_SP(S_, L_) return launch_split_t<S_, L_>(pl, ws, rp, gamma, pi, n_states, st)
    switch (pl.S) {
        case 4: VBX_SP(4, 1);
        case 8:
            if (spl == 2) VBX_SP(8, 2);
            VBX_SP(8, 1);
        case 16:
            if (spl == 1) VBX_SP(16, 1);
            if (spl == 4) VBX_SP(16, 4);
            VBX_SP(16, 2);
        case 32:
            if (spl == 1) VBX_SP(32, 1);
            if (spl == 4) VBX_SP(32, 4);
            VBX_SP(32, 2);
        case 64:
            if (spl == 4) VBX_SP(64, 4);
            VBX_SP(64, 2);
        case 128: VBX_SP(128, 4);   // a lane group must fit in a warp: 32 lanes x 4 states
        default: return -1;
    }
#undef VBX_SP
}

}  // namespace vbx
