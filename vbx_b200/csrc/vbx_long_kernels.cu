// Forward-backward for LONG recordings (T >= kLongT) as an exact chunked scan   VBx/VBx.py:98-104,146-175
//
// One warp-group per recording walks the frames sequentially (vbx_kernels.cu); with few, long recordings (DIHARD-
// shaped batches: 24 recordings x 12 000 frames per GPU) that leaves the GPU idle.  Both recursions are linear in the
// carried vector, so a recording is cut into chunks of kChunk frames and each sweep becomes three phases:
//   A  per (chunk, basis vector e_i): run the chunk from e_i with per-step renormalisation -> the chunk's transfer
//      operator as S columns  exp(lambda_i) * u_i   (S independent tasks per chunk, embarrassingly parallel)
//   B  per recording: combine the operators sequentially over the chunks (one small S x S mat-vec per chunk) -> the
//      true vector entering every chunk
//   C  per chunk: re-run the chunk from its true entry vector, now writing the per-frame outputs
// Exact (no approximation): products of positive operators with renormalisation lose no accuracy.  The per-frame
// results (normalised forward variables, scales, gamma, statistics) have the same meaning as in the sequential kernel;
// they differ from it only by float32 rounding.  Whether a recording takes this path depends on its own length only,
// never on the batch it is in.
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
__device__ __forceinline__ float rcpf(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Common per-task setup: a task group of LPR lanes, SPL states per lane.
template <int S_PAD, int SPL>
struct Group {
    static constexpr int LPR = S_PAD / SPL;
    static constexpr int GPW = 32 / LPR;   // task groups per warp
};

// ------------------------------------------------------------------ forward, phase A (operators) ----------------
// task = (long chunk j, basis i).  Chunk 0 of a recording runs once from the initial distribution (i == 0 only) and the
// last chunk of a recording needs no operator.  Output: fa_u[j][i][:] (normalised end vector), fa_lam[j][i].
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) long_fwd_basis_kernel(Plan pl, Workspace ws, RunParams rp, const float *pi_io,
                                                             const int32_t *__restrict__ n_states) {
    using G = Group<S_PAD, SPL>;
    constexpr int LPR = G::LPR, GPW = G::GPW;
    const int lane = threadIdx.x & 31;
    const int g = lane / LPR, l = lane % LPR;
    const int64_t task = ((int64_t)blockIdx.x * 4 + (threadIdx.x >> 5)) * GPW + g;
    const int64_t n_tasks = (int64_t)pl.n_lchunks * S_PAD;
    bool live = task < n_tasks;
    int j = 0, i = 0, rec = 0, c = 0, K = 1;
    if (live) {
        j = (int)(task / S_PAD);
        i = (int)(task % S_PAD);
        rec = pl.lchunk_rec[j];
        c = pl.lchunk_idx[j];
        K = pl.lrec_nchunks[rec];
        live = ws.active[rec] != 0 && c < K - 1 && (c > 0 || i == 0);
    }
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    live = live && (c == 0 || i < ns);
    const int64_t f0 = live ? pl.offsets[rec] : 0;
    const int t0 = c * kChunk, t1 = t0 + kChunk;   // c < K-1: full chunk
    const float P = ws.hp[rec].loopP, Q = 1.f - P;   // rec = 0 on lanes without a chunk
    float w[SPL], base[SPL], a[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        const float pik = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pik, VBX_EPS_TR) : 0.f;
        // entry vector: initial distribution for chunk 0, the basis vector e_i otherwise (sum = 1)
        base[k] = c == 0 ? (sl ? pik + VBX_EPS_TR : 0.f) : (sl ? fmaf(P, s == i ? 1.f : 0.f, w[k]) : 0.f);
        a[k] = 0.f;
    }
    const float *pp = ws.p + (f0 + t0) * S_PAD + l * SPL;
    // the chunk's total scale = product of the per-frame scales, kept as mantissa * 2^exponent (a float log would
    // cost ~1e-5 relative in the combination weights)
    float lam = 1.f;
    int lexp = 0;
    // any warp-uniform trip count works: dead groups just run on row 0 of the batch
    if (!live) pp = ws.p + l * SPL;
    constexpr int PFB = 8;   // frames per load burst (the chunk length is a multiple of it)
    Vec<SPL> buf[PFB];
    for (int t8 = 0; t8 < kChunk; t8 += PFB) {
#pragma unroll
      for (int i = 0; i < PFB; ++i) buf[i] = ldg_vec<SPL>(pp + (live ? (int64_t)(t8 + i) * S_PAD : 0));
#pragma unroll
      for (int i = 0; i < PFB; ++i) {
        const int t = t8 + i;
        const Vec<SPL> cur = buf[i];
        float v[SPL];
#pragma unroll
        for (int k = 0; k < SPL; ++k) v[k] = cur.v[k] * base[k];
        float loc = v[0];
#pragma unroll
        for (int k = 1; k < SPL; ++k) loc += v[k];
        const float sig = gsum<LPR>(loc);
        const float r = __frcp_rn(sig);   // correctly rounded: the factor taken out of the vector is sig up to 6e-8, unbiased
        lam *= sig;
        if ((t & 3) == 3) {
            int ex;
            lam = frexpf(lam, &ex);
            lexp += ex;
        }
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            a[k] = v[k] * r;
            base[k] = fmaf(P, a[k], w[k]);
        }
      }
    }
    (void)t1;
    if (live) {
        float *u = ws.fa_u + ((int64_t)j * S_PAD + i) * S_PAD + l * SPL;
        st_vec<SPL>(u, a);
        if (l == 0) {
            ws.fa_lam[(int64_t)j * S_PAD + i] = lam;
            ws.fa_exp[(int64_t)j * S_PAD + i] = (float)lexp;
        }
    }
}

// ------------------------------------------------------------------ forward, phase B (combine) -------------------
// one warp per long recording, lane = state (two per lane for S = 64).  astart[j][:] = normalised forward vector
// entering chunk j (for chunk 0 it is unused: phase C starts from the initial distribution).
// Operator of one chunk as seen by one lane: column entries u_i[s] for this lane's state(s) and, distributed over the
// lanes, the scale (mantissa, exponent) of basis i = lane (+32).  All loads are independent, so a chunk costs one
// memory latency; the next chunk's operator is fetched while the current one is applied.
template <int S_PAD, int SPLc>
struct ChunkOp {
    float u[SPLc][S_PAD];
    float m[SPLc], e[SPLc];
};
template <int S_PAD, int SPLc>
__device__ __forceinline__ void load_op(ChunkOp<S_PAD, SPLc> &op, const float *U, const float *M, const float *E,
                                        const int64_t j, const int lane) {
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        const int sc = s < S_PAD ? s : 0;
#pragma unroll
        for (int i = 0; i < S_PAD; ++i) op.u[k][i] = U[((int64_t)j * S_PAD + i) * S_PAD + sc];
        op.m[k] = M[(int64_t)j * S_PAD + sc];
        op.e[k] = E[(int64_t)j * S_PAD + sc];
    }
}

template <int S_PAD>
__global__ void __launch_bounds__(32) long_fwd_combine_kernel(Plan pl, Workspace ws, const int32_t *__restrict__ n_states) {
    const int lr = blockIdx.x;
    const int rec = pl.lrec_list[lr];
    if (!ws.active[rec]) return;
    const int lane = threadIdx.x;
    const int K = pl.lrec_nchunks[rec], j0 = pl.lrec_first[rec];
    const int ns = n_states ? n_states[rec] : S_PAD;
    constexpr int SPLc = S_PAD > 32 ? 2 : 1;
    float a[SPLc];
    // chunk 0 was run from the initial distribution: its end vector is the entry of chunk 1
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        a[k] = s < S_PAD ? ws.fa_u[((int64_t)j0 * S_PAD + 0) * S_PAD + s] : 0.f;
        if (s < S_PAD && K > 1) ws.astart[(int64_t)(j0 + 1) * S_PAD + s] = a[k];
    }
    ChunkOp<S_PAD, SPLc> cur, nxt;
    if (K > 2) load_op<S_PAD, SPLc>(cur, ws.fa_u, ws.fa_lam, ws.fa_exp, j0 + 1, lane);
    for (int c = 1; c < K - 1; ++c) {
        const int j = j0 + c;
        if (c + 1 < K - 1) load_op<S_PAD, SPLc>(nxt, ws.fa_u, ws.fa_lam, ws.fa_exp, j + 1, lane);
        // weights a_i * scale_i, relative to the largest exponent among the contributing basis vectors
        float wgt[SPLc], ex[SPLc], emax = -CUDART_INF_F;
#pragma unroll
        for (int k = 0; k < SPLc; ++k) {
            const bool on = lane + 32 * k < ns && a[k] > 0.f;
            ex[k] = on ? cur.e[k] : -CUDART_INF_F;
            emax = fmaxf(emax, ex[k]);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) emax = fmaxf(emax, __shfl_xor_sync(0xffffffffu, emax, off));
#pragma unroll
        for (int k = 0; k < SPLc; ++k) wgt[k] = ex[k] > -CUDART_INF_F ? ldexpf(a[k] * cur.m[k], (int)(ex[k] - emax)) : 0.f;
        float acc[SPLc];
#pragma unroll
        for (int k = 0; k < SPLc; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < S_PAD; ++i) {
            const float wi = __shfl_sync(0xffffffffu, wgt[i >> 5], i & 31);
#pragma unroll
            for (int k = 0; k < SPLc; ++k) acc[k] = wi != 0.f ? fmaf(wi, cur.u[k][i], acc[k]) : acc[k];   // columns of dead states are never written
        }
        float loc = 0.f;
#pragma unroll
        for (int k = 0; k < SPLc; ++k) loc += (lane + 32 * k < S_PAD) ? acc[k] : 0.f;
        const float tot = gsum<32>(loc);
        const float r = 1.f / tot;
#pragma unroll
        for (int k = 0; k < SPLc; ++k) {
            const int s = lane + 32 * k;
            a[k] = s < S_PAD ? acc[k] * r : 0.f;
            if (s < S_PAD) ws.astart[(int64_t)(j + 1) * S_PAD + s] = a[k];
        }
        cur = nxt;
    }
}

// ------------------------------------------------------------------ forward, phase C (re-run, write outputs) -----
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) long_fwd_rerun_kernel(Plan pl, Workspace ws, RunParams rp, float *gamma,
                                                             const float *pi_io, const int32_t *__restrict__ n_states) {
    using G = Group<S_PAD, SPL>;
    constexpr int LPR = G::LPR, GPW = G::GPW;
    const int lane = threadIdx.x & 31;
    const int g = lane / LPR, l = lane % LPR;
    const int64_t j = ((int64_t)blockIdx.x * 4 + (threadIdx.x >> 5)) * GPW + g;
    bool live = j < pl.n_lchunks;
    int rec = 0, c = 0;
    if (live) {
        rec = pl.lchunk_rec[j];
        c = pl.lchunk_idx[j];
        live = ws.active[rec] != 0;
    }
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    const int64_t f0 = live ? pl.offsets[rec] : 0;
    const int T = live ? (int)(pl.offsets[rec + 1] - f0) : 0;
    const int t0 = c * kChunk;
    const int len = live ? min(kChunk, T - t0) : 0;
    int lenmax = len;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) lenmax = max(lenmax, __shfl_xor_sync(0xffffffffu, lenmax, off));
    const float P = ws.hp[rec].loopP, Q = 1.f - P;   // rec = 0 on lanes without a chunk
    float w[SPL], base[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        const float pik = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pik, VBX_EPS_TR) : 0.f;
        if (c == 0)
            base[k] = sl ? pik + VBX_EPS_TR : 0.f;
        else
            base[k] = sl ? fmaf(P, ws.astart[j * S_PAD + s], w[k]) : 0.f;
    }
    const float *pp = ws.p + (f0 + t0) * S_PAD + l * SPL;
    float *ga = gamma + (f0 + t0) * S_PAD + l * SPL;
    float *rs = ws.rsigma + f0 + t0;
    constexpr int PFB = 8;   // frames per load burst
    const int lclamp = max(len - 1, 0);
    for (int t8 = 0; t8 < lenmax; t8 += PFB) {
        Vec<SPL> buf[PFB];
#pragma unroll
        for (int i = 0; i < PFB; ++i) buf[i] = ldg_vec<SPL>(pp + (int64_t)min(t8 + i, lclamp) * S_PAD);
#pragma unroll
        for (int i = 0; i < PFB; ++i) {
            const int t = t8 + i;
            const bool act = t < len;
            float v[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) v[k] = buf[i].v[k] * base[k];
            float loc = v[0];
#pragma unroll
            for (int k = 1; k < SPL; ++k) loc += v[k];
            const float sig = gsum<LPR>(loc);
            if (act) {
                const float r = rcpf(sig);
                float an[SPL];
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    an[k] = v[k] * r;
                    base[k] = fmaf(P, an[k], w[k]);
                }
                st_vec<SPL>(ga + (int64_t)t * S_PAD, an);
                if (l == 0) rs[t] = r;
            }
        }
    }
}

// ------------------------------------------------------------------ backward, phase A (operators) ---------------
// The backward operator of chunk c maps beta_c = b(t1-1) to beta_{c-1} = b(t0-1): steps t = t1-2 .. t0-1, each
//   u = p(t+1) * b(t+1) * rsigma(t+1);  b(t) = loopP*u + sum_j w_j u_j .
// Chunk 0 needs no operator; the last chunk runs once from b = 1 (basis index 0 only).
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) long_bwd_basis_kernel(Plan pl, Workspace ws, RunParams rp, const float *pi_io,
                                                             const int32_t *__restrict__ n_states) {
    using G = Group<S_PAD, SPL>;
    constexpr int LPR = G::LPR, GPW = G::GPW;
    const int lane = threadIdx.x & 31;
    const int g = lane / LPR, l = lane % LPR;
    const int64_t task = ((int64_t)blockIdx.x * 4 + (threadIdx.x >> 5)) * GPW + g;
    const int64_t n_tasks = (int64_t)pl.n_lchunks * S_PAD;
    bool live = task < n_tasks;
    int j = 0, i = 0, rec = 0, c = 0, K = 1;
    if (live) {
        j = (int)(task / S_PAD);
        i = (int)(task % S_PAD);
        rec = pl.lchunk_rec[j];
        c = pl.lchunk_idx[j];
        K = pl.lrec_nchunks[rec];
        live = ws.active[rec] != 0 && c > 0 && (c < K - 1 || i == 0);
    }
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    live = live && (c == K - 1 || i < ns);
    const int64_t f0 = live ? pl.offsets[rec] : 0;
    const int T = live ? (int)(pl.offsets[rec + 1] - f0) : 0;
    const int t0 = c * kChunk;
    const int t1 = live ? min(T, t0 + kChunk) : 0;
    const int steps = live ? t1 - t0 : 0;          // t = t1-2 .. t0-1
    int smax = steps;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) smax = max(smax, __shfl_xor_sync(0xffffffffu, smax, off));
    const float P = ws.hp[rec].loopP, Q = 1.f - P;   // rec = 0 on lanes without a chunk
    float w[SPL], b[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        const float pik = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pik, VBX_EPS_TR) : 0.f;
        b[k] = (c == K - 1) ? 1.f : (s == i ? 1.f : 0.f);
    }
    const float *prow = ws.p + f0 * S_PAD + l * SPL;
    const float *rs = ws.rsigma + f0;
    float mu = 1.f;
    int mexp = 0;
    constexpr int PFB = 8;   // frames per load burst
    for (int q8 = 0; q8 < smax; q8 += PFB) {
        Vec<SPL> pbuf[PFB];
        float rbuf[PFB];
#pragma unroll
        for (int ii = 0; ii < PFB; ++ii) {
            const int fr = max(t1 - 1 - (q8 + ii), t0);          // frame t+1 of step q, clamped into the chunk
            pbuf[ii] = ldg_vec<SPL>(prow + (int64_t)fr * S_PAD);
            rbuf[ii] = rs[fr];
        }
#pragma unroll
        for (int ii = 0; ii < PFB; ++ii) {
            const int q = q8 + ii;
            const bool act = q < steps;                          // produces b(t1-2-q) from frame t1-1-q
            const float cr = act ? rbuf[ii] : 0.f;
            float u[SPL], loc = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                u[k] = (pbuf[ii].v[k] * cr) * b[k];
                loc = fmaf(w[k], u[k], loc);
            }
            const float dot = gsum<LPR>(loc);
            float bn[SPL], bs = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                bn[k] = fmaf(P, u[k], dot);
                bs += bn[k];
            }
            const float tot = gsum<LPR>(bs);             // own normalisation keeps the basis run in range
            if (act) {
                // A basis state whose likelihood is (numerically) 0 at the first frame maps to the zero vector: keep it
                // at 0.  The threshold also keeps 1/tot finite (0 * inf = NaN otherwise); a column that small
                // contributes less than 1e-22 relative to the combined vector (beta <= 1e8).
                const bool pos = tot > 1e-30f;
                const float r = pos ? __frcp_rn(tot) : 0.f;
                mu *= pos ? tot : 0.f;
                if ((q & 3) == 3) {
                    int ex;
                    mu = frexpf(mu, &ex);
                    mexp += ex;
                }
#pragma unroll
                for (int k = 0; k < SPL; ++k) b[k] = bn[k] * r;
            }
        }
    }
    if (live) {
        st_vec<SPL>(ws.bb_v + ((int64_t)j * S_PAD + i) * S_PAD + l * SPL, b);
        if (l == 0) {
            ws.bb_mu[(int64_t)j * S_PAD + i] = mu;
            ws.bb_exp[(int64_t)j * S_PAD + i] = (float)mexp;
        }
    }
}

// ------------------------------------------------------------------ backward, phase B (combine) ------------------
// beta[j][:] = backward vector at the LAST frame of chunk j (exact scale; 1 for the last chunk of a recording).
template <int S_PAD>
__global__ void __launch_bounds__(32) long_bwd_combine_kernel(Plan pl, Workspace ws, const int32_t *__restrict__ n_states) {
    const int lr = blockIdx.x;
    const int rec = pl.lrec_list[lr];
    if (!ws.active[rec]) return;
    const int ns = n_states ? n_states[rec] : S_PAD;   // dead states carry b > 0 but contribute nothing (p = 0)
    const int lane = threadIdx.x;
    const int K = pl.lrec_nchunks[rec], j0 = pl.lrec_first[rec];
    constexpr int SPLc = S_PAD > 32 ? 2 : 1;
    float b[SPLc];
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        if (s < S_PAD) ws.beta[(int64_t)(j0 + K - 1) * S_PAD + s] = 1.f;
        // the last chunk was run from b = 1: scale * v is beta of the chunk before it
        b[k] = 0.f;
        if (s < S_PAD && K > 1) {
            const int64_t o = (int64_t)(j0 + K - 1) * S_PAD;
            b[k] = ldexpf(ws.bb_mu[o], (int)ws.bb_exp[o]) * ws.bb_v[o * S_PAD + s];
            ws.beta[(int64_t)(j0 + K - 2) * S_PAD + s] = b[k];
        }
    }
    ChunkOp<S_PAD, SPLc> cur, nxt;
    if (K > 2) load_op<S_PAD, SPLc>(cur, ws.bb_v, ws.bb_mu, ws.bb_exp, j0 + K - 2, lane);
    for (int c = K - 2; c >= 1; --c) {
        const int j = j0 + c;
        if (c - 1 >= 1) load_op<S_PAD, SPLc>(nxt, ws.bb_v, ws.bb_mu, ws.bb_exp, j - 1, lane);
        float wgt[SPLc];
#pragma unroll
        for (int k = 0; k < SPLc; ++k) {
            const bool on = lane + 32 * k < ns && b[k] > 0.f;
            wgt[k] = on ? ldexpf(b[k] * cur.m[k], (int)cur.e[k]) : 0.f;   // bounded: beta stays in [1e-8, 1e8]
        }
        float acc[SPLc];
#pragma unroll
        for (int k = 0; k < SPLc; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < S_PAD; ++i) {
            const float wi = __shfl_sync(0xffffffffu, wgt[i >> 5], i & 31);
#pragma unroll
            for (int k = 0; k < SPLc; ++k) acc[k] = wi != 0.f ? fmaf(wi, cur.u[k][i], acc[k]) : acc[k];   // columns of dead states are never written
        }
#pragma unroll
        for (int k = 0; k < SPLc; ++k) {
            const int s = lane + 32 * k;
            b[k] = s < S_PAD ? acc[k] : 0.f;
            if (s < S_PAD) ws.beta[(int64_t)(j - 1) * S_PAD + s] = b[k];
        }
        cur = nxt;
    }
}

// ------------------------------------------------------------------ backward, phase C (re-run, write outputs) ----
// gamma over the chunk, partial N_s and re-entry statistics per chunk (summed in chunk order by the tail kernel).
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) long_bwd_rerun_kernel(Plan pl, Workspace ws, RunParams rp, float *gamma,
                                                             const float *pi_io, const int32_t *__restrict__ n_states) {
    using G = Group<S_PAD, SPL>;
    constexpr int LPR = G::LPR, GPW = G::GPW;
    const int lane = threadIdx.x & 31;
    const int g = lane / LPR, l = lane % LPR;
    const int64_t j = ((int64_t)blockIdx.x * 4 + (threadIdx.x >> 5)) * GPW + g;
    bool live = j < pl.n_lchunks;
    int rec = 0, c = 0;
    if (live) {
        rec = pl.lchunk_rec[j];
        c = pl.lchunk_idx[j];
        live = ws.active[rec] != 0;
    }
    const int ns = live ? (n_states ? n_states[rec] : S_PAD) : 0;
    const int64_t f0 = live ? pl.offsets[rec] : 0;
    const int T = live ? (int)(pl.offsets[rec + 1] - f0) : 0;
    const int t0 = c * kChunk;
    const int t1 = live ? min(T, t0 + kChunk) : 0;
    const int steps = live ? t1 - t0 : 0;   // q = 0: frame t1-1 (uses beta as is); q >= 1: b(t1-1-q) from frame t1-q
    int smax = steps;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) smax = max(smax, __shfl_xor_sync(0xffffffffu, smax, off));
    const float P = ws.hp[rec].loopP, Q = 1.f - P;   // rec = 0 on lanes without a chunk
    float w[SPL], b[SPL], occ[SPL], ent[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        const float pik = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pik, VBX_EPS_TR) : 0.f;
        b[k] = live ? ws.beta[j * S_PAD + s] : 0.f;
        occ[k] = 0.f;
        ent[k] = 0.f;
    }
    const float *prow = ws.p + f0 * S_PAD + l * SPL;
    float *grow = gamma + f0 * S_PAD + l * SPL;
    const float *rs = ws.rsigma + f0;
    constexpr int PFB = 8;   // frames per load burst
    for (int q8 = 0; q8 < smax; q8 += PFB) {
        Vec<SPL> pbuf[PFB], abuf[PFB];
        float rbuf[PFB];
#pragma unroll
        for (int ii = 0; ii < PFB; ++ii) {
            const int t = max(t1 - 1 - (q8 + ii), t0);          // frame whose gamma is produced in step q (clamped)
            const int tn = min(t + 1, max(t1 - 1, t0));          // frame t+1 feeding b(t)
            pbuf[ii] = ldg_vec<SPL>(prow + (int64_t)tn * S_PAD);
            rbuf[ii] = rs[tn];
            abuf[ii] = ld_vec<SPL>(grow + (int64_t)t * S_PAD);
        }
#pragma unroll
        for (int ii = 0; ii < PFB; ++ii) {
            const int q = q8 + ii;
            const bool act = q < steps;
            const int t = t1 - 1 - q;
            float u[SPL], loc = 0.f;
            const bool stepb = q > 0 && act;                     // b(t) from frame t+1
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                u[k] = stepb ? (pbuf[ii].v[k] * rbuf[ii]) * b[k] : 0.f;
                loc = fmaf(w[k], u[k], loc);
            }
            const float dot = gsum<LPR>(loc);
            if (stepb) {
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    ent[k] += u[k];                    // u of frame t+1 >= 1
                    b[k] = fmaf(P, u[k], dot);
                }
            }
            float gn[SPL], gs = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                gn[k] = act ? abuf[ii].v[k] * b[k] : 0.f;
                gs += gn[k];
            }
            const float tot = gsum<LPR>(gs);
            if (act) {
                const float sc = rcpf(tot);
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    gn[k] *= sc;
                    occ[k] += gn[k];
                }
                st_vec<SPL>(grow + (int64_t)t * S_PAD, gn);
            }
        }
    }
    // the step across the chunk boundary contributes u of frame t0 (t0 >= 1) to the re-entry statistics
    {
        Vec<SPL> cp;
        float cr = 0.f;
        const bool act = live && c > 0;
        if (act) {
            cp = ldg_vec<SPL>(prow + (int64_t)t0 * S_PAD);
            cr = rs[t0];
        } else {
#pragma unroll
            for (int k = 0; k < SPL; ++k) cp.v[k] = 0.f;
        }
#pragma unroll
        for (int k = 0; k < SPL; ++k) ent[k] += act ? (cp.v[k] * cr) * b[k] : 0.f;
    }
    if (live) {
        st_vec<SPL>(ws.occp + j * S_PAD + l * SPL, occ);
        st_vec<SPL>(ws.entp + j * S_PAD + l * SPL, ent);
    }
}

// ------------------------------------------------------------------ tail: eq. (24) and N_s -----------------------
template <int S_PAD>
__global__ void __launch_bounds__(32) long_tail_kernel(Plan pl, Workspace ws, RunParams rp, const float *gamma, float *pi_io,
                                                       const int32_t *__restrict__ n_states) {
    const int lr = blockIdx.x;
    const int rec = pl.lrec_list[lr];
    if (!ws.active[rec]) return;
    const int lane = threadIdx.x;
    const int K = pl.lrec_nchunks[rec], j0 = pl.lrec_first[rec];
    const int ns = n_states ? n_states[rec] : S_PAD;
    const int64_t f0 = pl.offsets[rec];
    constexpr int SPLc = S_PAD > 32 ? 2 : 1;
    const double Q = 1.0 - (double)ws.hp[rec].loopP;
    double pn[SPLc];
    float loc = 0.f;
#pragma unroll
    for (int k = 0; k < SPLc; ++k) {
        const int s = lane + 32 * k;
        pn[k] = 0.0;
        if (s < S_PAD) {
            double occ = 0.0, ent = 0.0;
            for (int c = 0; c < K; ++c) {
                occ += (double)ws.occp[(int64_t)(j0 + c) * S_PAD + s];
                ent += (double)ws.entp[(int64_t)(j0 + c) * S_PAD + s];
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

template <int S_PAD>
int launch_long_t(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi, const int32_t *n_states,
                  cudaStream_t st) {
    constexpr int SPL = S_PAD > 32 ? 2 : 1;
    constexpr int GPW = 32 / (S_PAD / SPL);
    const int64_t basis_tasks = (int64_t)pl.n_lchunks * S_PAD;
    const int basis_blocks = (int)((basis_tasks + 4 * GPW - 1) / (4 * GPW));
    const int chunk_blocks = (pl.n_lchunks + 4 * GPW - 1) / (4 * GPW);
    long_fwd_basis_kernel<S_PAD, SPL><<<basis_blocks, 128, 0, st>>>(pl, ws, rp, pi, n_states);
    long_fwd_combine_kernel<S_PAD><<<pl.n_lrec, 32, 0, st>>>(pl, ws, n_states);
    long_fwd_rerun_kernel<S_PAD, SPL><<<chunk_blocks, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    long_bwd_basis_kernel<S_PAD, SPL><<<basis_blocks, 128, 0, st>>>(pl, ws, rp, pi, n_states);
    long_bwd_combine_kernel<S_PAD><<<pl.n_lrec, 32, 0, st>>>(pl, ws, n_states);
    long_bwd_rerun_kernel<S_PAD, SPL><<<chunk_blocks, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    long_tail_kernel<S_PAD><<<pl.n_lrec, 32, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    return cudaGetLastError() == cudaSuccess ? 7 : -1;
}

}  // namespace

int launch_forward_backward_long(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                                 const int32_t *n_states, cudaStream_t st) {
    if (pl.n_lrec == 0) return 0;
    switch (pl.S) {
        case 4: return launch_long_t<4>(pl, ws, rp, gamma, pi, n_states, st);
        case 8: return launch_long_t<8>(pl, ws, rp, gamma, pi, n_states, st);
        case 16: return launch_long_t<16>(pl, ws, rp, gamma, pi, n_states, st);
        case 32: return launch_long_t<32>(pl, ws, rp, gamma, pi, n_states, st);
        case 64: return launch_long_t<64>(pl, ws, rp, gamma, pi, n_states, st);
        default: return -1;
    }
}

}  // namespace vbx
