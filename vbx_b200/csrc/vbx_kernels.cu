// Hand-written sm_90a kernels of the VB-HMM EM loop (reference: VBx/VBx.py:74-126,146-175).
//
// Data layout (all float32, row-major, packed ragged over the batch):
//   rho    [N,R]   x-vectors scaled into the PLDA space           VBx/VBx.py:89
//   gamma  [N,S]   responsibilities; doubles as the store of the normalised forward variables
//   p      [N,S]   exp(log_p - rowmax)   rowmax [N]               VBx/VBx.py:97 (without the common G_t)
//   rsigma [N]     reciprocal forward scales
// One EM iteration = 4 launches:
//   mstep_partial  -> per-tile gamma^T rho                (VBx/VBx.py:96, the T-long contraction)
//   speaker_model  -> invL, alpha, bias, ELBO regulariser (VBx/VBx.py:95-96,100)
//   loglik         -> p, rowmax                           (VBx/VBx.py:97)
//   forward_backward -> gamma, pi, N_s, ELBO, stop test   (VBx/VBx.py:98-105,122-125,146-175)
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {

// ------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
}

template <int LANES>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}
template <int LANES>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
    for (int off = LANES / 2; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// ------------------------------------------------------------------------------------------------
// prepare: rho = fea * sqrt(Phi), G partial sums per M-tile          VBx/VBx.py:87-89
// MODE 0: in = fea, writes rho, ||x||^2 from fea.   MODE 1: in = rho (read only), ||x||^2 = sum rho^2/Phi.
// ------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256) prepare_kernel(Plan pl, Workspace ws, const float *__restrict__ in,
                                                      const float *__restrict__ Phi, float *rho) {
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int R = pl.R;
    const bool rlive = 4 * lane < R;
    float4 sc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rlive) {
        float4 ph = __ldg(reinterpret_cast<const float4 *>(Phi) + lane);
        if (MODE == 0)
            sc = make_float4(sqrtf(ph.x), sqrtf(ph.y), sqrtf(ph.z), sqrtf(ph.w));
        else
            sc = make_float4(1.f / ph.x, 1.f / ph.y, 1.f / ph.z, 1.f / ph.w);
    }
    const double cst = (double)R * 1.8378770664093454835606594728112;  // R * log(2*pi)
    double gw = 0.0;
    for (int t = warp; t < len; t += 8) {
        float n2 = 0.f;
        if (rlive) {
            const int64_t idx = (f0 + t) * R + 4 * lane;
            float4 x = *reinterpret_cast<const float4 *>(in + idx);
            if (MODE == 0) {
                n2 = x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
                *reinterpret_cast<float4 *>(rho + idx) = make_float4(x.x * sc.x, x.y * sc.y, x.z * sc.z, x.w * sc.w);
            } else {
                n2 = x.x * x.x * sc.x + x.y * x.y * sc.y + x.z * x.z * sc.z + x.w * x.w * sc.w;
            }
        }
        n2 = group_sum<32>(n2);
        gw += -0.5 * ((double)n2 + cst);
    }
    __shared__ double sg[8];
    if (lane == 0) sg[warp] = gw;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < 8; ++i) s += sg[i];
        ws.gpart[tile] = s;
    }
}

__global__ void gsum_kernel(Plan pl, Workspace ws) {
    const int rec = blockIdx.x * blockDim.x + threadIdx.x;
    if (rec >= pl.n_rec) return;
    double s = 0.0;
    for (int t = pl.mtile_begin[rec]; t < pl.mtile_begin[rec + 1]; ++t) s += ws.gpart[t];
    ws.gsum[rec] = s;
}

// per-recording sum of the per-frame constants written by the wgmma projection epilogue (float64, fixed order)
__global__ void __launch_bounds__(128) gsum_frames_kernel(Plan pl, Workspace ws, const float *__restrict__ gframe) {
    const int rec = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (rec >= pl.n_rec) return;
    const int64_t f0 = pl.offsets[rec];
    const int T = (int)(pl.offsets[rec + 1] - f0);
    double acc = 0.0;
    for (int t = lane; t < T; t += 32) acc += (double)gframe[f0 + t];
    acc = warp_sum_d(acc);
    if (lane == 0) ws.gsum[rec] = acc;
}
int launch_gsum_from_frames(const Plan &pl, const Workspace &ws, const float *gframe, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    gsum_frames_kernel<<<(pl.n_rec + 3) / 4, 128, 0, st>>>(pl, ws, gframe);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_prepare_scale(const Plan &pl, const Workspace &ws, const float *fea, const float *Phi, float *rho,
                         cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    prepare_kernel<0><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, fea, Phi, rho);
    gsum_kernel<<<(pl.n_rec + 127) / 128, 128, 0, st>>>(pl, ws);
    return cudaGetLastError() == cudaSuccess ? 2 : -1;
}
int launch_g_from_rho(const Plan &pl, const Workspace &ws, const float *rho, const float *Phi, cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    prepare_kernel<1><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, Phi, nullptr);
    gsum_kernel<<<(pl.n_rec + 127) / 128, 128, 0, st>>>(pl, ws);
    return cudaGetLastError() == cudaSuccess ? 2 : -1;
}

// ------------------------------------------------------------------------------------------------
// projection, FFMA tiles:  rho[N,R] = X[N,D] . V[D,R]     (vbhmm.py:129,153 folded; SURVEY 8d)
// 128 x 128 block tile, 8 x 8 per thread, k-chunks of 16 through shared memory.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) project_ffma_kernel(const float *__restrict__ X, const float *__restrict__ V,
                                                            float *__restrict__ rho, int64_t N, int D, int R) {
    constexpr int BM = 128, BN = 128, BK = 16;
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int64_t row0 = (int64_t)blockIdx.x * BM;
    const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 8 rows x 8 cols (strided by 16)
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < D; k0 += BK) {
        // A tile: 128 rows x 16 k -> 512 float4, 2 per thread
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + i * 256;
            const int r = idx >> 2, c4 = idx & 3;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row0 + r < N) v = __ldg(reinterpret_cast<const float4 *>(X + (row0 + r) * D + k0) + c4);
            As[c4 * 4 + 0][r] = v.x;
            As[c4 * 4 + 1][r] = v.y;
            As[c4 * 4 + 2][r] = v.z;
            As[c4 * 4 + 3][r] = v.w;
        }
        // B tile: 16 k x 128 cols -> 512 float4
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int idx = tid + i * 256;
            const int kk = idx >> 5, c4 = idx & 31;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (4 * c4 < R) v = __ldg(reinterpret_cast<const float4 *>(V + (int64_t)(k0 + kk) * R) + c4);
            *reinterpret_cast<float4 *>(&Bs[kk][4 * c4]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[8], b[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 8; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t r = row0 + ty + 16 * i;
        if (r < N) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = tx + 16 * j;
                if (c < R) rho[r * R + c] = acc[i][j];
            }
        }
    }
}

int launch_project_ffma(const Plan &pl, const float *X, int D, const float *V, float *rho, cudaStream_t st) {
    if (pl.n_frames == 0) return 0;
    const int64_t blocks = (pl.n_frames + 127) / 128;
    project_ffma_kernel<<<(unsigned)blocks, 256, 0, st>>>(X, V, rho, pl.n_frames, D, pl.R);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// run_init: per recording reset + initial occupancies N_s = sum_t gamma[t,s]   (VBx/VBx.py:95 for ii=0)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) run_init_kernel(Plan pl, Workspace ws, const float *__restrict__ gamma,
                                                       const int32_t *__restrict__ n_states, double *Li,
                                                       int32_t *n_iters, int32_t *flags, int max_iters) {
    const int rec = blockIdx.x;
    const int S = pl.S;
    const int tid = threadIdx.x;
    const int64_t f0 = pl.offsets[rec];
    const int64_t T = pl.offsets[rec + 1] - f0;
    const int ns = n_states ? n_states[rec] : S;
    const bool ok = T > 0 && ns > 0;
    if (tid == 0) {
        ws.active[rec] = ok ? 1 : 0;
        ws.tile_done[rec] = 0;
        if (ws.active64) {
            ws.active64[rec] = 0;
            ws.fresh[rec] = 0;
        }
        ws.prev_elbo[rec] = 0.0;
        n_iters[rec] = 0;
        flags[rec] = 0;
    }
    for (int i = tid; i < max_iters; i += 128) Li[(int64_t)rec * max_iters + i] = CUDART_NAN;
    __shared__ double part[128];
    const int s = tid % S, k = tid / S, nk = 128 / S;
    double acc = 0.0;
    for (int64_t t = k; t < T; t += nk) acc += (double)gamma[(f0 + t) * S + s];
    part[tid] = acc;
    __syncthreads();
    if (tid < S) {
        double tot = 0.0;
        for (int i = 0; i < nk; ++i) tot += part[i * S + tid];
        ws.occ[(int64_t)rec * S + tid] = (float)tot;
    }
}

int launch_run_init(const Plan &pl, const Workspace &ws, const float *gamma, const int32_t *n_states, double *Li,
                    int32_t *n_iters, int32_t *flags, int max_iters, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    run_init_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, gamma, n_states, Li, n_iters, flags, max_iters);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// Output step (SURVEY 8f.2): the most and second most likely speaker per frame,
// labels1st = argsort(-q)[:, 0], labels2nd = argsort(-q)[:, 1]                       VBx/vbhmm.py:160-162
// One thread per frame of a 64-frame tile; only the recording's live states compete (ties: lowest index).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLTile) hard_labels_kernel(Plan pl, const float *__restrict__ gamma,
                                                             const int32_t *__restrict__ n_states,
                                                             int32_t *__restrict__ first, int32_t *__restrict__ second) {
    const int tile = blockIdx.x;
    const int rec = pl.ltile_rec[tile];
    const int64_t f0 = pl.ltile_f0[tile];
    const int len = (int)min((int64_t)kLTile, pl.offsets[rec + 1] - f0);
    if ((int)threadIdx.x >= len) return;
    const int S = pl.S, ns = n_states ? n_states[rec] : S;
    const float4 *row = reinterpret_cast<const float4 *>(gamma + (f0 + threadIdx.x) * S);
    float b1 = -INFINITY, b2 = -INFINITY;
    int i1 = -1, i2 = -1;
    for (int q = 0; q < S / 4; ++q) {
        const float4 v = row[q];
        const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int s = 4 * q + e;
            if (s >= ns) break;
            if (x[e] > b1) {
                b2 = b1, i2 = i1;
                b1 = x[e], i1 = s;
            } else if (x[e] > b2) {
                b2 = x[e], i2 = s;
            }
        }
    }
    first[f0 + threadIdx.x] = i1;
    if (second) second[f0 + threadIdx.x] = i2;
}

int launch_hard_labels(const Plan &pl, const float *gamma, const int32_t *n_states, int32_t *first, int32_t *second,
                       cudaStream_t st) {
    if (pl.n_ltiles == 0) return 0;
    hard_labels_kernel<<<pl.n_ltiles, kLTile, 0, st>>>(pl, gamma, n_states, first, second);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// M-step accumulation: partial[tile][s][r] = sum_{t in tile} gamma[t,s] * rho[t,r]      VBx/VBx.py:96
// One CTA per <=256-frame tile of one recording.  A warp owns a frame slot and SPT states; lane owns
// 4 consecutive r (the rho row is one coalesced 512 B request), gamma values are warp-uniform loads.
// ------------------------------------------------------------------------------------------------
template <int S_PAD>
__global__ void __launch_bounds__(256) mstep_partial_kernel(Plan pl, Workspace ws, const float *__restrict__ rho,
                                                            const float *__restrict__ gamma) {
    constexpr int SPT = S_PAD < 16 ? S_PAD : 16;
    constexpr int NG = S_PAD / SPT;
    constexpr int FS = 8 / NG;
    __shared__ __align__(16) float red[S_PAD][kMaxR];
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sg = warp % NG, fs = warp / NG;
    const int R = pl.R;
    const bool rlive = 4 * lane < R;
    float acc[SPT][4];
#pragma unroll
    for (int s = 0; s < SPT; ++s)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[s][c] = 0.f;
    const float *grow = gamma + f0 * S_PAD + sg * SPT;
    const float *xrow = rho + f0 * R + 4 * lane;
#pragma unroll 2
    for (int t = fs; t < len; t += FS) {
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rlive) x = __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)t * R));
        const float4 *g4 = reinterpret_cast<const float4 *>(grow + (int64_t)t * S_PAD);
#pragma unroll
        for (int q = 0; q < SPT / 4; ++q) {
            const float4 g = __ldg(g4 + q);
            acc[4 * q + 0][0] = fmaf(g.x, x.x, acc[4 * q + 0][0]);
            acc[4 * q + 0][1] = fmaf(g.x, x.y, acc[4 * q + 0][1]);
            acc[4 * q + 0][2] = fmaf(g.x, x.z, acc[4 * q + 0][2]);
            acc[4 * q + 0][3] = fmaf(g.x, x.w, acc[4 * q + 0][3]);
            acc[4 * q + 1][0] = fmaf(g.y, x.x, acc[4 * q + 1][0]);
            acc[4 * q + 1][1] = fmaf(g.y, x.y, acc[4 * q + 1][1]);
            acc[4 * q + 1][2] = fmaf(g.y, x.z, acc[4 * q + 1][2]);
            acc[4 * q + 1][3] = fmaf(g.y, x.w, acc[4 * q + 1][3]);
            acc[4 * q + 2][0] = fmaf(g.z, x.x, acc[4 * q + 2][0]);
            acc[4 * q + 2][1] = fmaf(g.z, x.y, acc[4 * q + 2][1]);
            acc[4 * q + 2][2] = fmaf(g.z, x.z, acc[4 * q + 2][2]);
            acc[4 * q + 2][3] = fmaf(g.z, x.w, acc[4 * q + 2][3]);
            acc[4 * q + 3][0] = fmaf(g.w, x.x, acc[4 * q + 3][0]);
            acc[4 * q + 3][1] = fmaf(g.w, x.y, acc[4 * q + 3][1]);
            acc[4 * q + 3][2] = fmaf(g.w, x.z, acc[4 * q + 3][2]);
            acc[4 * q + 3][3] = fmaf(g.w, x.w, acc[4 * q + 3][3]);
        }
    }
    // fixed-order reduction over the frame slots (deterministic)
#pragma unroll 1
    for (int k = 0; k < FS; ++k) {
        if (fs == k) {
#pragma unroll
            for (int s = 0; s < SPT; ++s) {
                float4 *dst = reinterpret_cast<float4 *>(&red[sg * SPT + s][4 * lane]);
                float4 v = make_float4(acc[s][0], acc[s][1], acc[s][2], acc[s][3]);
                if (k > 0) {
                    const float4 o = *dst;
                    v.x += o.x;
                    v.y += o.y;
                    v.z += o.z;
                    v.w += o.w;
                }
                *dst = v;
            }
        }
        __syncthreads();
    }
    const int R4 = R >> 2;
    float *out = ws.partial + (int64_t)tile * S_PAD * R;
    for (int i = threadIdx.x; i < S_PAD * R4; i += 256) {
        const int s = i / R4, c4 = i - s * R4;
        *reinterpret_cast<float4 *>(out + (int64_t)s * R + 4 * c4) = *reinterpret_cast<const float4 *>(&red[s][4 * c4]);
    }
}

int launch_mstep_partial(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    switch (pl.S) {
        case 4: mstep_partial_kernel<4><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, gamma); break;
        case 8: mstep_partial_kernel<8><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, gamma); break;
        case 16: mstep_partial_kernel<16><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, gamma); break;
        case 32: mstep_partial_kernel<32><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, gamma); break;
        case 64: mstep_partial_kernel<64><<<pl.n_mtiles, 256, 0, st>>>(pl, ws, rho, gamma); break;
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// speaker model: invL, alpha (eqs 17,16; VBx/VBx.py:95-96), the per-speaker bias of eq. (23)
// (VBx/VBx.py:97) and the per-speaker parts of the ELBO regulariser of eq. (25) (VBx/VBx.py:100).  One CTA per
// recording, four 128-thread warp-groups each taking every 4th speaker, thread = r.  Sums over tiles run in tile order in float64 (deterministic).
// ------------------------------------------------------------------------------------------------
template <int S8, bool R128>
__global__ void __launch_bounds__(512) speaker_model_kernel(Plan pl, Workspace ws, RunParams rp,
                                                            const float *__restrict__ Phi,
                                                            const int32_t *__restrict__ n_states, float *alpha_io,
                                                            float *invL_io, int from_given) {
    // one CTA per recording; four 128-thread warp-groups, each takes every 4th speaker, thread = r
    const int S = pl.S, R = pl.R;
    constexpr int NT = S8 / 8, NSP = S8 / 4;   // speakers per warp-group
    const int rec = blockIdx.x;
    if (!ws.active[rec]) return;            // CTA-uniform
    const int wg = threadIdx.x >> 7;
    const int r = threadIdx.x & 127, warp = r >> 5, lane = r & 31;
    const bool live = r < R;
    const int ns = n_states ? n_states[rec] : S;
    const float phi = live ? Phi[r] : 0.f;
    const int t_lo = pl.mtile_begin[rec], t_hi = pl.mtile_begin[rec + 1];
    extern __shared__ float sAv[];                       // [S8][kMaxR] Fa*alpha, staged for the coalesced fragment writes
    __shared__ double cpart[kMaxS][4], rpart[kMaxS][4];
    // all tile sums of this thread's speakers first (independent loads in flight), then the per-speaker math
    double grs[NSP];
#pragma unroll
    for (int k = 0; k < NSP; ++k) {
        const int s = wg + 4 * k;
        double gr = 0.0;
        if (live && s < ns && !from_given)
            for (int t = t_lo; t < t_hi; ++t) gr += (double)__ldg(ws.partial + ((int64_t)t * S + s) * R + r);
        grs[k] = gr;
    }
#pragma unroll
    for (int k = 0; k < NSP; ++k) {
        const int s = wg + 4 * k;
        const int64_t o = ((int64_t)rec * S + s) * R + r;
        const bool dead = s >= ns;   // dead (or padding) column: never wins, never contributes
        float invL = 1.f, alpha = 0.f, Av = 0.f;
        float c = 0.f, reg = 0.f;
        if (live && !dead) {
            if (from_given) {
                alpha = alpha_io[o];
                invL = invL_io[o];
            } else {
                const double gr = grs[k];
                const float Ns = ws.occ[(int64_t)rec * S + s];
                invL = 1.f / (1.f + rp.FaFb * Ns * phi);
                alpha = (float)((double)(rp.FaFb * invL) * gr);
            }
            Av = rp.Fa * alpha;
            const float a2 = alpha * alpha;
            reg = logf(invL) - invL - a2 + 1.f;
            c = (invL + a2) * phi;
        }
        if (live && s < S) {
            ws.A[o] = Av;
            if (!from_given || dead) {
                if (alpha_io) alpha_io[o] = dead ? 0.f : alpha;
                if (invL_io) invL_io[o] = dead ? 0.f : invL;
            }
        }
        sAv[s * kMaxR + r] = Av;                          // columns >= R hold 0
        c = group_sum<32>(c);                             // 32 terms in float, the rest in float64
        reg = group_sum<32>(reg);
        if (lane == 0) {
            cpart[s][warp] = (double)c;
            rpart[s][warp] = (double)reg;
        }
    }
    __syncthreads();
    if (threadIdx.x < S) {
        const int s = threadIdx.x;
        const bool dead = s >= ns;
        ws.bias[(int64_t)rec * S + s] =
            dead ? CUDART_INF_F : (float)(rp.dFa * 0.5 * ((cpart[s][0] + cpart[s][1]) + (cpart[s][2] + cpart[s][3])));
        ws.regp[(int64_t)rec * S + s] = dead ? 0.0 : (rpart[s][0] + rpart[s][1]) + (rpart[s][2] + rpart[s][3]);
    }
    // mma fragment-major copy of Fa*alpha, split into TF32 hi/lo (consumed by loglik_mma_kernel): linear, coalesced
    // writes; element q = ((i*KS + j)*32 + lane)*2 + e  <->  state 8i + lane/4, column col(j, lane%4, e)
    const int KS = R128 ? 16 : (R + 7) >> 3, KQ = 2 * KS;
    float *fh = ws.Afrag_hi + (int64_t)rec * NT * KS * 64, *fl = ws.Afrag_lo + (int64_t)rec * NT * KS * 64;
    for (int q = threadIdx.x; q < NT * KS * 64; q += 512) {
        const int e = q & 1, ln = (q >> 1) & 31, ij = q >> 6;
        const int j = R128 ? (ij & 15) : ij % KS, i = R128 ? (ij >> 4) : ij / KS;
        const int st = 8 * i + (ln >> 2), fq = ln & 3;
        // R = 128 uses the coalesced column permutation of loglik_mma_kernel, other R the plain one
        const int col = R128 ? 16 * (j >> 1) + 4 * fq + 2 * (j & 1) + e : KQ * fq + 2 * j + e;
        const float Av = col < kMaxR ? sAv[st * kMaxR + col] : 0.f;
        const float hi = __uint_as_float(__float_as_uint(Av) & 0xffffe000u);
        fh[q] = hi;
        fl[q] = Av - hi;
    }
}

int launch_speaker_model(const Plan &pl, const Workspace &ws, const RunParams &rp, const float *Phi,
                         const int32_t *n_states, float *alpha_io, float *invL_io, bool from_given,
                         cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    const int S8 = pl.S > 8 ? pl.S : 8;
    const size_t smem = (size_t)S8 * kMaxR * sizeof(float);
    const int fg = from_given ? 1 : 0;
#define VBX_SM(S8_, R_) speaker_model_kernel<S8_, R_><<<pl.n_rec, 512, smem, st>>>(pl, ws, rp, Phi, n_states, alpha_io, invL_io, fg)
    if (pl.R == 128) {
        switch (S8) {
            case 8: VBX_SM(8, true); break;
            case 16: VBX_SM(16, true); break;
            case 32: VBX_SM(32, true); break;
            default: VBX_SM(64, true); break;
        }
    } else {
        switch (S8) {
            case 8: VBX_SM(8, false); break;
            case 16: VBX_SM(16, false); break;
            case 32: VBX_SM(32, false); break;
            default: VBX_SM(64, false); break;
        }
    }
#undef VBX_SM
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// log-likelihood + row softmax numerator, fused:                               VBx/VBx.py:97
//   ll[t,s] = sum_r rho[t,r] * A[s,r] - bias[s] ;  rowmax[t] = max_s ll ;  p[t,s] = exp(ll - rowmax)
// One CTA = 64 frames of one recording.  rho tile and the recording's A are staged once in shared
// memory (cp.async, rows padded by 4 floats -> conflict-free LDS.128); each thread owns FJ frames x SJ
// states and walks k in float4 steps.
// ------------------------------------------------------------------------------------------------
template <int S_PAD>
__global__ void __launch_bounds__(128) loglik_kernel(Plan pl, Workspace ws, const float *__restrict__ rho,
                                                     const float *__restrict__ pi, const int32_t *__restrict__ n_states, const float Q) {
    constexpr int SL = S_PAD < 8 ? S_PAD : 8;  // state lanes
    constexpr int SJ = S_PAD / SL;             // states per thread (strided by SL)
    constexpr int FL = 128 / SL;               // frame lanes
    constexpr int FJ = kLTile / FL;            // frames per thread (strided by FL)
    extern __shared__ float4 smem4[];
    float *smem = reinterpret_cast<float *>(smem4);
    const int R = pl.R, RP = R + 4, R4 = R >> 2;
    float *rhoS = smem;             // [kLTile][RP]
    float *AS = smem + kLTile * RP; // [S_PAD][RP]
    const int tile = blockIdx.x;
    const int rec = pl.ltile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t f0 = pl.ltile_f0[tile];
    const int len = (int)min((int64_t)kLTile, pl.offsets[rec + 1] - f0);
    const int tid = threadIdx.x;
    {
        const float *src = rho + f0 * R;
        for (int i = tid; i < len * R4; i += 128) {
            const int row = i / R4, c4 = i - row * R4;
            cp_async16(rhoS + row * RP + 4 * c4, src + (int64_t)row * R + 4 * c4);
        }
        const float *Ab = ws.A + (int64_t)rec * S_PAD * R;
        for (int i = tid; i < S_PAD * R4; i += 128) {
            const int row = i / R4, c4 = i - row * R4;
            cp_async16(AS + row * RP + 4 * c4, Ab + (int64_t)row * R + 4 * c4);
        }
        cp_async_wait_all();
    }
    __syncthreads();
    const int sl = tid % SL, fl = tid / SL;
    float acc[FJ][SJ];
#pragma unroll
    for (int j = 0; j < SJ; ++j) {
        const float b = ws.bias[(int64_t)rec * S_PAD + sl + SL * j];
#pragma unroll
        for (int i = 0; i < FJ; ++i) acc[i][j] = -b;
    }
#pragma unroll 4
    for (int k4 = 0; k4 < R4; ++k4) {
        float4 x[FJ], a[SJ];
#pragma unroll
        for (int i = 0; i < FJ; ++i) x[i] = *reinterpret_cast<const float4 *>(rhoS + (fl + FL * i) * RP + 4 * k4);
#pragma unroll
        for (int j = 0; j < SJ; ++j) a[j] = *reinterpret_cast<const float4 *>(AS + (sl + SL * j) * RP + 4 * k4);
#pragma unroll
        for (int i = 0; i < FJ; ++i)
#pragma unroll
            for (int j = 0; j < SJ; ++j) {
                acc[i][j] = fmaf(x[i].x, a[j].x, acc[i][j]);
                acc[i][j] = fmaf(x[i].y, a[j].y, acc[i][j]);
                acc[i][j] = fmaf(x[i].z, a[j].z, acc[i][j]);
                acc[i][j] = fmaf(x[i].w, a[j].w, acc[i][j]);
            }
    }
    float wv[SJ];                    // transition weights w = Q pi + 1e-8 of this thread's states (VBx/VBx.py:98,159)
    {
        const int ns = n_states ? n_states[rec] : S_PAD;
#pragma unroll
        for (int j = 0; j < SJ; ++j) {
            const int s = sl + SL * j;
            wv[j] = s < ns ? fmaf(Q, pi[(int64_t)rec * S_PAD + s], VBX_EPS_TR) : 0.f;
        }
    }
#pragma unroll
    for (int i = 0; i < FJ; ++i) {
        float m = acc[i][0];
#pragma unroll
        for (int j = 1; j < SJ; ++j) m = fmaxf(m, acc[i][j]);
        m = group_max<SL>(m);
        const int fr = fl + FL * i;
        float pv[SJ], c = 0.f;
#pragma unroll
        for (int j = 0; j < SJ; ++j) {
            pv[j] = expf(acc[i][j] - m);
            c = fmaf(pv[j], wv[j], c);
        }
        if (pl.split) c = group_sum<SL>(c);   // c_t = sum_j p[t,j] w_j, consumed by the split sweeps (CTA-uniform branch)
        if (fr < len) {
            float *dst = ws.p + (f0 + fr) * S_PAD + sl;
#pragma unroll
            for (int j = 0; j < SJ; ++j) dst[SL * j] = pv[j];
            if (sl == 0) {
                ws.rowmax[f0 + fr] = m;
                if (pl.split) ws.cvec[f0 + fr] = c;
            }
        }
    }
}

static size_t loglik_smem(int S_pad, int R) { return (size_t)(kLTile + S_pad) * (R + 4) * sizeof(float); }

template <int S_PAD>
static int launch_loglik_t(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states, float loopP,
                           cudaStream_t st) {
    const size_t smem = loglik_smem(S_PAD, pl.R);
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(loglik_kernel<S_PAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)loglik_smem(S_PAD, kMaxR)) != cudaSuccess)
            return -1;
        configured = true;
    }
    loglik_kernel<S_PAD><<<pl.n_ltiles, 128, smem, st>>>(pl, ws, rho, pi, n_states, 1.f - loopP);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_loglik(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states, float loopP,
                  cudaStream_t st) {
    if (pl.n_ltiles == 0) return 0;
    switch (pl.S) {
        case 4: return launch_loglik_t<4>(pl, ws, rho, pi, n_states, loopP, st);
        case 8: return launch_loglik_t<8>(pl, ws, rho, pi, n_states, loopP, st);
        case 16: return launch_loglik_t<16>(pl, ws, rho, pi, n_states, loopP, st);
        case 32: return launch_loglik_t<32>(pl, ws, rho, pi, n_states, loopP, st);
        case 64: return launch_loglik_t<64>(pl, ws, rho, pi, n_states, loopP, st);
        default: return -1;
    }
}

// ------------------------------------------------------------------------------------------------
// forward-backward in the scaled linear domain                     VBx/VBx.py:98-104,146-175
//
// The transition matrix of VBx/VBx.py:98 is  loopP*I + (1-loopP)*1*pi^T ; with the reference's +1e-8
// inside every log (VBx/VBx.py:159,164) it acts on a vector a as  loopP*a + w*sum(a),  w = (1-loopP)*pi + 1e-8,
// so each frame costs O(S).  A group of LPR lanes owns one recording (SPL states per lane), 32/LPR
// recordings share a warp (recordings are sorted by length, so the groups of a warp finish together).
// Forward variables are normalised per frame (scale sigma_t, its reciprocal is kept for the backward sweep and
// for the ELBO kernel); the backward variables are scaled by the forward scales, so gamma_t = a_t * b_t sums to
// one up to rounding and b_t stays within [1e-8, 1e8] (w >= 1e-8 bounds the spread of b_t).  The same sweep
// accumulates N_s (VBx/VBx.py:95) and the re-entry statistics of eq. (24) (VBx/VBx.py:101-103); the tail applies
// eq. (24) (VBx/VBx.py:101-104).
//
// Latency notes: every global load is an unconditional, index-clamped prefetch PF/PB frames ahead (a predicated
// load turns into load+select and stalls on the spot); the main loops carry no per-group predicates, only the
// ragged tail does; the reciprocal is a single MUFU.RCP.
// ------------------------------------------------------------------------------------------------
#ifndef VBX_LDO
#define VBX_LDO "ld.volatile.global"
#define VBX_STO "st.volatile.global"
#endif
// Ordered prefetch loads: ptxas sinks plain (reorderable) LDGs of a burst towards their first use, which shrinks the
// prefetch window; volatile accesses keep their program order, so a burst issued before the first volatile store of
// a chunk stays there.
template <int N>
__device__ __forceinline__ Vec<N> ldo_vec(const float *p);
template <>
__device__ __forceinline__ Vec<1> ldo_vec<1>(const float *p) {
    Vec<1> r;
    asm volatile(VBX_LDO ".f32 %0, [%1];" : "=f"(r.v[0]) : "l"(p) : "memory");
    return r;
}
template <>
__device__ __forceinline__ Vec<2> ldo_vec<2>(const float *p) {
    Vec<2> r;
    asm volatile(VBX_LDO ".v2.f32 {%0, %1}, [%2];" : "=f"(r.v[0]), "=f"(r.v[1]) : "l"(p) : "memory");
    return r;
}
template <>
__device__ __forceinline__ Vec<4> ldo_vec<4>(const float *p) {
    Vec<4> r;
    asm volatile(VBX_LDO ".v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3]) : "l"(p) : "memory");
    return r;
}
template <int N>
__device__ __forceinline__ void sto_vec(float *p, const float *v);
template <>
__device__ __forceinline__ void sto_vec<1>(float *p, const float *v) {
    asm volatile(VBX_STO ".f32 [%0], %1;" ::"l"(p), "f"(v[0]) : "memory");
}
template <>
__device__ __forceinline__ void sto_vec<2>(float *p, const float *v) {
    asm volatile(VBX_STO ".v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]), "f"(v[1]) : "memory");
}
template <>
__device__ __forceinline__ void sto_vec<4>(float *p, const float *v) {
    asm volatile(VBX_STO ".v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
}

__device__ __forceinline__ float rcp_fast(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

template <int S_PAD, int SPL, bool NORM>
__global__ void __launch_bounds__(128) forward_backward_kernel(Plan pl, Workspace ws, RunParams rp, float *gamma,
                                                               float *pi_io, const int32_t *__restrict__ n_states) {
    constexpr int LPR = S_PAD / SPL;
    constexpr int RPW = 32 / LPR;
    constexpr int PF = (SPL == 4) ? 8 : (SPL == 2 ? 24 : 16);  // frames per prefetch burst, forward sweep (ping-pong register sets)
    constexpr int PB = (SPL == 4) ? 4 : (SPL == 2 ? 10 : 8);   // ... backward sweep (three arrays per frame)
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int g = lane / LPR, l = lane % LPR;
    const int slot = warp_global * RPW + g;
    int rec = -1;
    if (slot < pl.n_rec) rec = pl.order[slot];
    // long recordings are handled by the chunked scan (vbx_long_kernels.cu)
    const bool live = rec >= 0 && ws.active[rec] != 0 && pl.lrec_nchunks[rec] == 0;
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
    const float P = rp.loopP, Q = 1.f - rp.loopP;

    float pi[SPL], w[SPL], base[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        pi[k] = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pi[k], VBX_EPS_TR) : 0.f;   // VBx/VBx.py:98,159
        base[k] = sl ? pi[k] + VBX_EPS_TR : 0.f;          // VBx/VBx.py:164 (initial state probabilities)
    }
    // Groups without a recording read row 0 of the batch and write into a scratch row (stride 0), so that the
    // main loops need no predicates at all.
    const float *pp = ws.p + f0 * S_PAD + l * SPL;
    float *ga = live ? gamma + f0 * S_PAD + l * SPL : ws.scratch + l * SPL;
    float *rs = live ? ws.rsigma + f0 : ws.scratch + kMaxS;
    const int64_t gstr = live ? S_PAD : 0;
    const int rstr = live ? 1 : 0;

    // ---------------- forward sweep, VBx/VBx.py:164,167-168 ----------------
    float a[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) a[k] = 0.f;
    {
        Vec<SPL> bufA[PF], bufB[PF];
        auto fstep = [&](const int t, const Vec<SPL> &cur, const bool check) {
            float v[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) v[k] = cur.v[k] * base[k];
            float loc = v[0];
#pragma unroll
            for (int k = 1; k < SPL; ++k) loc += v[k];
            const float sig = group_sum<LPR>(loc);
            const float r = rcp_fast(sig);
            float an[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) an[k] = v[k] * r;
            if (!check) {
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    a[k] = an[k];
                    base[k] = fmaf(P, an[k], w[k]);
                }
                sto_vec<SPL>(ga + t * gstr, an);
                if (l == 0) rs[t * rstr] = r;
            } else {
                const bool act = t < T;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    a[k] = act ? an[k] : a[k];
                    base[k] = act ? fmaf(P, an[k], w[k]) : base[k];
                }
                if (act) {
                    sto_vec<SPL>(ga + t * gstr, an);
                    if (l == 0) rs[t * rstr] = r;
                }
            }
        };
        // one chunk = PF frames: first issue the burst of loads for the NEXT chunk, then run this chunk's steps
        auto fchunk = [&](const int t0, Vec<SPL>(&cur)[PF], Vec<SPL>(&nxt)[PF], const bool check) {
#pragma unroll
            for (int i = 0; i < PF; ++i) nxt[i] = ldo_vec<SPL>(pp + (int64_t)min(t0 + PF + i, Tlast) * S_PAD);
#pragma unroll
            for (int i = 0; i < PF; ++i) fstep(t0 + i, cur[i], check);
        };
#pragma unroll
        for (int i = 0; i < PF; ++i) bufA[i] = ldg_vec<SPL>(pp + (int64_t)min(i, Tlast) * S_PAD);
        int t0 = 0;
        for (; t0 + 2 * PF <= Tmin; t0 += 2 * PF) {
            fchunk(t0, bufA, bufB, false);
            fchunk(t0 + PF, bufB, bufA, false);
        }
        for (; t0 < Tmax; t0 += 2 * PF) {
            fchunk(t0, bufA, bufB, true);
            fchunk(t0 + PF, bufB, bufA, true);
        }
    }
    __syncwarp();  // rsigma written by lane l==0 of each group is read by the whole group below

    // ---------------- backward sweep, VBx/VBx.py:165,170-171,174 + eq. (24) statistics ----------------
    float b[SPL], g0[SPL], occf[SPL], entf[SPL];
    double enter[SPL], occ[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        b[k] = 1.f;
        g0[k] = a[k];            // gamma_{T-1} = forward variable (already stored)
        occ[k] = (double)a[k];
        enter[k] = 0.0;
        occf[k] = 0.f;
        entf[k] = 0.f;
    }
    {
        struct Slot {
            Vec<SPL> p, a;
            float r;
        };
        Slot bufA[PB], bufB[PB];
        auto load_slot = [&](const int ii) {   // data of backward step ii (frame t = T-2-ii)
            const int t = max(T - 2 - ii, 0);
            const int t1 = min(t + 1, Tlast);
            Slot sl;
            sl.p = ldo_vec<SPL>(pp + (int64_t)t1 * S_PAD);
            sl.a = ldo_vec<SPL>(ga + t * gstr);
            sl.r = ldo_vec<1>(rs + t1 * rstr).v[0];
            return sl;
        };
        auto bstep = [&](const int ii, const Slot &c, const bool check) {
            const int t = T - 2 - ii;
            float u[SPL], loc = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                u[k] = (c.p.v[k] * c.r) * b[k];
                loc = fmaf(w[k], u[k], loc);
            }
            const float dot = group_sum<LPR>(loc);
            float gn[SPL], bn[SPL], gs = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                bn[k] = fmaf(P, u[k], dot);
                gn[k] = c.a.v[k] * bn[k];
                gs += gn[k];
            }
            if (NORM) {  // remove the common-mode rounding drift: rows of gamma sum to one
                const float sc = rcp_fast(group_sum<LPR>(gs));
#pragma unroll
                for (int k = 0; k < SPL; ++k) gn[k] *= sc;
            }
            if (!check) {
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    b[k] = bn[k];
                    g0[k] = gn[k];
                    occf[k] += gn[k];
                    entf[k] += u[k];
                }
                sto_vec<SPL>(ga + t * gstr, gn);
            } else {
                const bool act = t >= 0;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    b[k] = act ? bn[k] : b[k];
                    g0[k] = act ? gn[k] : g0[k];
                    occf[k] += act ? gn[k] : 0.f;
                    entf[k] += act ? u[k] : 0.f;
                }
                if (act) sto_vec<SPL>(ga + t * gstr, gn);
            }
        };
        auto bchunk = [&](const int i0, Slot(&cur)[PB], Slot(&nxt)[PB], const bool check) {
#pragma unroll
            for (int i = 0; i < PB; ++i) nxt[i] = load_slot(i0 + PB + i);
#pragma unroll
            for (int i = 0; i < PB; ++i) bstep(i0 + i, cur[i], check);
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                occ[k] += (double)occf[k];
                enter[k] += (double)entf[k];
                occf[k] = 0.f;
                entf[k] = 0.f;
            }
        };
#pragma unroll
        for (int i = 0; i < PB; ++i) bufA[i] = load_slot(i);
        int i0 = 0;
        for (; i0 + 2 * PB <= Tmin - 1; i0 += 2 * PB) {
            bchunk(i0, bufA, bufB, false);
            bchunk(i0 + PB, bufB, bufA, false);
        }
        for (; i0 < Tmax - 1; i0 += 2 * PB) {
            bchunk(i0, bufA, bufB, true);
            bchunk(i0 + PB, bufB, bufA, true);
        }
    }

    // ---------------- tail: eq. (24), VBx/VBx.py:101-104 ----------------
    double pn[SPL];
    float loc = 0.f;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        pn[k] = (double)g0[k] + (double)Q * (double)pi[k] * enter[k];
        loc += (float)pn[k];
    }
    const float tot = group_sum<LPR>(loc);
    if (live) {
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            const int s = l * SPL + k;
            pi_io[(int64_t)rec * S_PAD + s] = (float)(pn[k] / (double)tot);
            ws.occ[(int64_t)rec * S_PAD + s] = (float)occ[k];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// forward-backward with one step of look-ahead: the group reduction leaves the per-frame dependency chain.
//
// The kernel above needs  sigma_t = sum_i p_t,i (P a_{t-1,i} + w_i)  before it can touch frame t+1: a multiply, a
// 3-level shuffle reduction, a reciprocal and two more multiplies, ~125 cycles per frame with nothing else to do
// (at most 7 warps per SM exist for 4096 recordings).  Here the forward vector is carried with a lagging scale,
//     y_{t+1} = r_{t+1} p_{t+1} o (P y_t + w Y_t),      Y_t = sum_i y_t,i,
// and Y is advanced by a scalar recurrence fed by a reduction that only needs the PREVIOUS vector:
//     Y_{t+1} = r_{t+1} (P q_t + c_{t+1} Y_t),   q_t = p_{t+1} . y_t,   c_{t+1} = p_{t+1} . w   (c does not depend on y).
// q_t is launched as soon as y_t exists and is consumed one frame later, so two frames share one reduction latency
// and the reductions for c fill the gaps.  r_{t+1} = 1/sigma_{t-1} keeps Y_t = sigma_t sigma_{t-1} (no under/overflow:
// sigma >= ~1e-8).  Outputs are unchanged: a_t = y_t / Y_t,  1/sigma_t = r_t Y_{t-1} / Y_t.
// Backward, same idea:  v_t = kappa_{t+1} o b_{t+1} (kappa_t = p_t / sigma_t),  b_t = P v_t + d_t,
//     d_t = w . v_t = P e_{t+1} + d_{t+1} f_{t+1},   e_{t+1} = (w o kappa_{t+1}) . v_{t+1},   f_{t+1} = w . kappa_{t+1}.
// ------------------------------------------------------------------------------------------------
template <int S_PAD, int SPL>
__global__ void __launch_bounds__(128) forward_backward_la_kernel(Plan pl, Workspace ws, RunParams rp, float *gamma,
                                                                  float *pi_io, const int32_t *__restrict__ n_states) {
    constexpr int LPR = S_PAD / SPL;
    constexpr int RPW = 32 / LPR;
    // Ping-pong register bursts (see the kernel above): one burst must cover the DRAM latency under load, and the
    // look-ahead steps are about half as long as the normalise-every-frame ones, so the bursts are deeper.
    constexpr int PF = (SPL == 4) ? 10 : (SPL == 2 ? 24 : 32); // frames per prefetch burst, forward sweep
    constexpr int PB = (SPL == 4) ? 5 : (SPL == 2 ? 10 : 16);  // ... backward sweep (three arrays per frame)
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * 4 + (threadIdx.x >> 5);
    const int g = lane / LPR, l = lane % LPR;
    const int slot = warp_global * RPW + g;
    int rec = -1;
    if (slot < pl.n_rec) rec = pl.order[slot];
    const bool live = rec >= 0 && ws.active[rec] != 0 && pl.lrec_nchunks[rec] == 0;
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
    const float P = rp.loopP, Q = 1.f - rp.loopP;

    float pi[SPL], w[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        const int s = l * SPL + k;
        const bool sl = live && s < ns;
        pi[k] = sl ? pi_io[(int64_t)rec * S_PAD + s] : 0.f;
        w[k] = sl ? fmaf(Q, pi[k], VBX_EPS_TR) : 0.f;   // VBx/VBx.py:98,159
    }
    const float *pp = ws.p + f0 * S_PAD + l * SPL;
    float *ga = live ? gamma + f0 * S_PAD + l * SPL : ws.scratch + l * SPL;
    float *rs = live ? ws.rsigma + f0 : ws.scratch + kMaxS;
    const int64_t gstr = live ? S_PAD : 0;
    const int rstr = live ? 1 : 0;

    // ---------------- forward sweep, VBx/VBx.py:164,167-168 ----------------
    float alast[SPL];                       // forward variable of the recording's last frame
    {
        // frame 0: y_0 = p_0 o (pi + eps)  (VBx/VBx.py:164), normalised directly
        float y[SPL];
        const Vec<SPL> p0 = ldg_vec<SPL>(pp);
        const Vec<SPL> p1 = ldg_vec<SPL>(pp + (int64_t)min(1, Tlast) * S_PAD);
        float loc = 0.f, locq = 0.f, locc = 0.f;
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            const int s = l * SPL + k;
            y[k] = (live && s < ns) ? p0.v[k] * (pi[k] + VBX_EPS_TR) : 0.f;
            loc += y[k];
            locq = fmaf(p1.v[k], y[k], locq);
            locc = fmaf(p1.v[k], w[k], locc);
        }
        float Yc = group_sum<LPR>(loc);     // Y_0 = sigma_0
        float q = group_sum<LPR>(locq);     // q_0 = p_1 . y_0
        float c = group_sum<LPR>(locc);     // c_1 = p_1 . w
        float rn = 1.f;                     // r_1
        float rs1 = rcp_fast(Yc);           // 1/sigma_0 (becomes r_2)
        {
            float an[SPL];
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                an[k] = y[k] * rs1;
                alast[k] = an[k];
            }
            st_vec<SPL>(ga, an);
            if (l == 0) rs[0] = rs1;
        }
        // step j handles frame s = j + 1 with ps = p_s (slot j) and pn = p_{s+1} (slot j + 1)
        auto fstep = [&](const int j, const Vec<SPL> &ps, const Vec<SPL> &pn, const bool check) {
            const int s = j + 1;
            float ys[SPL], locq = 0.f, locc = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                ys[k] = (rn * ps.v[k]) * fmaf(P, y[k], w[k] * Yc);
                locq = fmaf(pn.v[k], ys[k], locq);
                locc = fmaf(pn.v[k], w[k], locc);
            }
            const float qn = group_sum<LPR>(locq);              // consumed by the NEXT step
            const float cn = group_sum<LPR>(locc);
            const float Ys = rn * fmaf(P, q, c * Yc);           // Y_s = sum_i y_s,i
            const float inv = rcp_fast(Ys);
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
            if (!check) {
#pragma unroll
                for (int k = 0; k < SPL; ++k) alast[k] = an[k];
                sto_vec<SPL>(ga + s * gstr, an);
                if (l == 0) rs[s * rstr] = rsig;
            } else {
                const bool act = s < T;
#pragma unroll
                for (int k = 0; k < SPL; ++k) alast[k] = act ? an[k] : alast[k];
                if (act) {
                    sto_vec<SPL>(ga + s * gstr, an);
                    if (l == 0) rs[s * rstr] = rsig;
                }
            }
        };
        Vec<SPL> bufA[PF], bufB[PF];
        Vec<SPL> ps = p1;                   // row of frame 1
        // slot i of a burst starting at step j0 holds the row of frame j0 + i + 2 (`pn` of step j0 + i)
        auto fchunk = [&](const int j0, Vec<SPL>(&cur)[PF], Vec<SPL>(&nxt)[PF], const bool check) {
#pragma unroll
            for (int i = 0; i < PF; ++i) nxt[i] = ldo_vec<SPL>(pp + (int64_t)min(j0 + PF + i + 2, Tlast) * S_PAD);
#pragma unroll
            for (int i = 0; i < PF; ++i) {
                fstep(j0 + i, ps, cur[i], check);
                ps = cur[i];
            }
        };
#pragma unroll
        for (int i = 0; i < PF; ++i) bufA[i] = ldg_vec<SPL>(pp + (int64_t)min(i + 2, Tlast) * S_PAD);
        int j0 = 0;
        for (; j0 + 2 * PF <= Tmin - 1; j0 += 2 * PF) {
            fchunk(j0, bufA, bufB, false);
            fchunk(j0 + PF, bufB, bufA, false);
        }
        for (; j0 < Tmax - 1; j0 += 2 * PF) {
            fchunk(j0, bufA, bufB, true);
            fchunk(j0 + PF, bufB, bufA, true);
        }
    }
    __syncwarp();  // rsigma written by lane l==0 of each group is read by the whole group below

    // ---------------- backward sweep, VBx/VBx.py:165,170-171,174 + eq. (24) statistics ----------------
    float g0[SPL], occf[SPL], entf[SPL];
    double enter[SPL], occ[SPL];
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        g0[k] = alast[k];        // gamma_{T-1} = forward variable (already stored)
        occ[k] = (double)alast[k];
        enter[k] = 0.0;
        occf[k] = 0.f;
        entf[k] = 0.f;
    }
    {
        struct Slot {             // data of backward step ii (frame t = T-2-ii): p_{t+1}, 1/sigma_{t+1}, a_t
            Vec<SPL> p, a;
            float r;
        };
        auto load_slot = [&](const int ii) {
            const int t = max(T - 2 - ii, 0);
            const int t1 = min(t + 1, Tlast);
            Slot sl;
            sl.p = ldo_vec<SPL>(pp + (int64_t)t1 * S_PAD);
            sl.a = ldo_vec<SPL>(ga + t * gstr);
            sl.r = ldo_vec<1>(rs + t1 * rstr).v[0];
            return sl;
        };
        Slot bufA[PB], bufB[PB];
        Slot cur = load_slot(0);
#pragma unroll
        for (int i = 0; i < PB; ++i) bufA[i] = load_slot(i + 1);       // slot i of a burst at i0 = data of step i0 + i + 1
        // state entering step ii: b = b_{t+1}, dprev = d_{t+1}, e = e_{t+1}, kap = kappa_{t+1}, f = f_{t+1}
        // (b_{T-1} = 1 = P * 0 + 1, i.e. v_{T-1} = 0, d_{T-1} = 1, e_{T-1} = 0)
        float b[SPL], kap[SPL];
        float dprev = 1.f, e = 0.f, f;
        {
            float locf = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                b[k] = 1.f;
                kap[k] = cur.p.v[k] * cur.r;
                locf = fmaf(w[k], kap[k], locf);
            }
            f = group_sum<LPR>(locf);
        }
        auto bstep = [&](const int ii, const Slot &c, const Slot &nx, const bool check) {
            const int t = T - 2 - ii;
            float v[SPL], kapn[SPL], loce = 0.f, locf = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                v[k] = kap[k] * b[k];                               // v_t = p_{t+1} b_{t+1} / sigma_{t+1}
                kapn[k] = nx.p.v[k] * nx.r;                          // kappa_t
                const float wk = w[k] * kapn[k];
                loce = fmaf(wk, v[k], loce);
                locf += wk;
            }
            const float en = group_sum<LPR>(loce);                   // e_t, consumed by the NEXT step
            const float fn = group_sum<LPR>(locf);                   // f_t
            const float d = fmaf(P, e, dprev * f);                   // d_t = w . v_t
            float gn[SPL], bn[SPL], gs = 0.f;
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                bn[k] = fmaf(P, v[k], d);
                gn[k] = c.a.v[k] * bn[k];
                gs += gn[k];
            }
            {   // rows of gamma sum to one (removes the common-mode rounding drift)
                const float sc = rcp_fast(group_sum<LPR>(gs));
#pragma unroll
                for (int k = 0; k < SPL; ++k) gn[k] *= sc;
            }
            if (!check) {
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    g0[k] = gn[k];
                    occf[k] += gn[k];
                    entf[k] += v[k];
                }
                sto_vec<SPL>(ga + t * gstr, gn);
            } else {
                const bool act = t >= 0;
#pragma unroll
                for (int k = 0; k < SPL; ++k) {
                    g0[k] = act ? gn[k] : g0[k];
                    occf[k] += act ? gn[k] : 0.f;
                    entf[k] += act ? v[k] : 0.f;
                }
                if (act) sto_vec<SPL>(ga + t * gstr, gn);
            }
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                b[k] = bn[k];
                kap[k] = kapn[k];
            }
            dprev = d;
            e = en;
            f = fn;
        };
        auto bchunk = [&](const int i0, Slot(&cb)[PB], Slot(&nb)[PB], const bool check) {
#pragma unroll
            for (int i = 0; i < PB; ++i) nb[i] = load_slot(i0 + PB + i + 1);
#pragma unroll
            for (int i = 0; i < PB; ++i) {
                bstep(i0 + i, cur, cb[i], check);
                cur = cb[i];
            }
#pragma unroll
            for (int k = 0; k < SPL; ++k) {
                occ[k] += (double)occf[k];
                enter[k] += (double)entf[k];
                occf[k] = 0.f;
                entf[k] = 0.f;
            }
        };
        int i0 = 0;
        for (; i0 + 2 * PB <= Tmin - 1; i0 += 2 * PB) {
            bchunk(i0, bufA, bufB, false);
            bchunk(i0 + PB, bufB, bufA, false);
        }
        for (; i0 < Tmax - 1; i0 += 2 * PB) {
            bchunk(i0, bufA, bufB, true);
            bchunk(i0 + PB, bufB, bufA, true);
        }
    }

    // ---------------- tail: eq. (24), VBx/VBx.py:101-104 ----------------
    double pn[SPL];
    float loc = 0.f;
#pragma unroll
    for (int k = 0; k < SPL; ++k) {
        pn[k] = (double)g0[k] + (double)Q * (double)pi[k] * enter[k];
        loc += (float)pn[k];
    }
    const float tot = group_sum<LPR>(loc);
    if (live) {
#pragma unroll
        for (int k = 0; k < SPL; ++k) {
            const int s = l * SPL + k;
            pi_io[(int64_t)rec * S_PAD + s] = (float)(pn[k] / (double)tot);
            ws.occ[(int64_t)rec * S_PAD + s] = (float)occ[k];
        }
    }
}

template <int S_PAD, int SPL>
static int launch_fb_t(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                       const int32_t *n_states, bool classic, cudaStream_t st) {
    constexpr int RPW = 32 / (S_PAD / SPL);
    const int warps = (pl.n_rec + RPW - 1) / RPW;
    const int blocks = (warps + 3) / 4;
    if (classic)
        forward_backward_kernel<S_PAD, SPL, true><<<blocks, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    else
        forward_backward_la_kernel<S_PAD, SPL><<<blocks, 128, 0, st>>>(pl, ws, rp, gamma, pi, n_states);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// ELBO + stop test: one CTA per recording                           VBx/VBx.py:100,105,122-125,173
//   tll = sum_t (log sigma_t + rowmax_t) + Fa * sum_t G_t ;  ELBO = tll + reg
// float64, fixed summation order (lane-strided partial sums, xor tree) => deterministic.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) elbo_kernel(Plan pl, Workspace ws, RunParams rp, double *Li, int32_t *n_iters,
                                                   int32_t *flags, int iter) {
    const int rec = blockIdx.x;
    if (!ws.active[rec]) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t f0 = pl.offsets[rec];
    const int T = (int)(pl.offsets[rec + 1] - f0);
    const float *rs = ws.rsigma + f0;
    const float *mx = ws.rowmax + f0;
    double acc = 0.0;
    for (int t = tid; t < T; t += 128) acc += (double)mx[t] - log((double)rs[t]);
    acc = warp_sum_d(acc);
    __shared__ double part[4];
    if (lane == 0) part[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        double reg = 0.0;                         // eq. (25) regulariser: per-speaker parts in speaker order
        for (int s = 0; s < pl.S; ++s) reg += ws.regp[(int64_t)rec * pl.S + s];
        const double elbo = (part[0] + part[1]) + (part[2] + part[3]) + rp.dFa * ws.gsum[rec] + 0.5 * rp.dFb * reg;
        const double d = elbo - ws.prev_elbo[rec];
        if (rp.hybrid && iter > 0 && isfinite(elbo)) {
            // float32 resolves an ELBO difference to about nb; decide here only what is decided safely
            const double nb = rp.noise_c * 5.9604644775390625e-8 * fabs(elbo);
            const bool go_on = d >= rp.epsilon + rp.guard_mult * nb;     // far above epsilon: keep iterating in float32
            const bool stop = d < rp.epsilon - 4.0 * nb;                  // clearly below epsilon: the reference stops too
            if (!go_on && !stop) {
                // Hand the recording to the float64 kernels (vbx_exact64.cu).  This iteration AND the previous one are
                // discarded and redone there from the snapshot that entered iteration iter-1, so that the test of
                // iteration iter compares two float64 ELBO values; iteration iter-1 itself was seen safely above
                // epsilon one round ago (fresh = 1: no test).  Only a warm-started iteration 0 cannot be redone (the
                // given model is float32): then iteration 1 alone is redone and tested against the float32 ELBO of
                // iteration 0 if it is within float32 noise of epsilon (fresh = 2).
                ws.active[rec] = 0;
                ws.active64[rec] = 1;
                if (iter == 1 && rp.warm) {
                    ws.fresh[rec] = d >= rp.epsilon + 4.0 * nb ? 1 : 2;
                } else {
                    ws.fresh[rec] = 1;
                    n_iters[rec] = iter - 1;
                }
                return;
            }
        }
        Li[(int64_t)rec * rp.max_iters + iter] = elbo;
        n_iters[rec] = iter + 1;
        int fl = flags[rec];
        if (!isfinite(elbo)) fl |= 1;
        if (iter > 0) {
            if (d < rp.epsilon) {  // VBx/VBx.py:122: stop AFTER this iteration's update
                ws.active[rec] = 0;
                if (iter + 1 < rp.max_iters) fl |= 4;
                if (d < 0.0) fl |= 2;
            }
        }
        ws.prev_elbo[rec] = elbo;
        flags[rec] = fl;
    }
}

// ------------------------------------------------------------------------------------------------
// ELBO trace of the batch: out[i] = sum over recordings of Li[rec][i] (iterations a recording did not run are NaN and
// skipped), out[max_iters + i] = number of recordings that ran iteration i.  One CTA per iteration, fixed summation
// order (deterministic); the caller all-reduces the 2*max_iters doubles over the GPUs (vbx_elbo_trace).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) elbo_trace_kernel(int n_rec, const double *__restrict__ Li, int max_iters, double *out) {
    const int it = blockIdx.x, tid = threadIdx.x;
    double s = 0.0, c = 0.0;
    for (int r = tid; r < n_rec; r += 256) {
        const double v = Li[(int64_t)r * max_iters + it];
        if (v == v) {
            s += v;
            c += 1.0;
        }
    }
    __shared__ double ss[256], cs[256];
    ss[tid] = s;
    cs[tid] = c;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (tid < off) {
            ss[tid] += ss[tid + off];
            cs[tid] += cs[tid + off];
        }
        __syncthreads();
    }
    if (tid == 0) {
        out[it] = ss[0];
        out[max_iters + it] = cs[0];
    }
}
int launch_elbo_trace(const Plan &pl, const double *Li, int max_iters, double *out, cudaStream_t st) {
    elbo_trace_kernel<<<max_iters, 256, 0, st>>>(pl.n_rec, Li, max_iters, out);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_forward_backward(const Plan &pl, const Workspace &ws, const RunParams &rp, float *gamma, float *pi,
                            const int32_t *n_states, double *Li, int32_t *n_iters, int32_t *flags, int iter,
                            int spl, int classic, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    if (pl.split) {
        const int rs = launch_forward_backward_split(pl, ws, rp, gamma, pi, n_states, spl, st);
        if (rs < 0) return rs;
        elbo_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, rp, Li, n_iters, flags, iter);
        return cudaGetLastError() == cudaSuccess ? rs + 1 : -1;
    }
    int rc = -1;
#define VBX_FB(S_, L_) rc = launch_fb_t<S_, L_>(pl, ws, rp, gamma, pi, n_states, classic != 0, st)
    const int S = pl.S;
    if (spl == 0) spl = (S >= 16) ? 2 : 1;
    if (S == 64 && spl < 2) spl = 2;
    if (spl > S) spl = S;
    switch (S) {
        case 4:
            if (spl == 1) VBX_FB(4, 1);
            else if (spl == 2) VBX_FB(4, 2);
            else VBX_FB(4, 4);
            break;
        case 8:
            if (spl == 1) VBX_FB(8, 1);
            else if (spl == 2) VBX_FB(8, 2);
            else VBX_FB(8, 4);
            break;
        case 16:
            if (spl == 1) VBX_FB(16, 1);
            else if (spl == 2) VBX_FB(16, 2);
            else VBX_FB(16, 4);
            break;
        case 32:
            if (spl == 1) VBX_FB(32, 1);
            else if (spl == 2) VBX_FB(32, 2);
            else VBX_FB(32, 4);
            break;
        case 64:
            if (spl == 2) VBX_FB(64, 2);
            else VBX_FB(64, 4);
            break;
        default: return -1;
    }
#undef VBX_FB
    if (rc < 0) return rc;
    const int rl = launch_forward_backward_long(pl, ws, rp, gamma, pi, n_states, st);
    if (rl < 0) return rl;
    elbo_kernel<<<pl.n_rec, 128, 0, st>>>(pl, ws, rp, Li, n_iters, flags, iter);
    return cudaGetLastError() == cudaSuccess ? rc + rl + 1 : -1;
}

}  // namespace vbx
