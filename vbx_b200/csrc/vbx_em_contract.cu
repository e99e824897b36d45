// M-step, speaker model and log-likelihood of one EM iteration in one kernel, so that rho is read from HBM once per
// iteration instead of twice (DESIGN.md section 5.3).  One thread-block cluster per recording of at most
// CL / 4 * kMTile frames; rank k of the cluster is frame slot k % 4 of M-tile k / 4 and holds that slot's 8-frame chunks
// c = slot + 4i of the tile (16 chunks, 64 KB of rho) in shared memory, filled by bulk copies.
//
// The results are bit-identical to mstep_mma_kernel + speaker_model_kernel + loglik_mma_kernel at S <= 16, R = 128:
//   M-step       mstep_mma_kernel at S <= 16 has warp `slot` run, for each of 16 n-tiles, one mma chain over the chunks
//                c = slot + 4i of the tile.  Here warp w of the slot's CTA runs the same chains of n-tiles 4w .. 4w+3 with
//                the same fragments, parks them in the same red[s][r] layout, and the slot sum ((s0 + s1) + s2) + s3 and
//                the float64 sum over tiles are formed in that order over distributed shared memory.
//   speaker      speaker_state / speaker_bias below, the arithmetic of speaker_model_kernel; CTA k owns the
//                states s = k (mod CL), thread = r.
//   log-lik.     every output element of loglik_mma_kernel is its own dot product initialised to -bias, so any 16 held
//                frames form an m-tile; the B fragments are built from the gathered Fa*alpha with the same hi/lo split.
// Rows past the recording's end are zero in shared memory (never copied from past the recording), and their results
// are never stored.
#include <cooperative_groups.h>
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace cg = cooperative_groups;

namespace vbx {

namespace {
constexpr int kSlots = 4;                               // frame slots of an M-tile
constexpr int kRows = 8;                                // frames of a chunk
constexpr int kHeld = kMTile / kRows / kSlots;          // chunks held by one CTA (16)
constexpr int kBars = 4;                                // load mbarriers, kHeld / kBars chunks each
constexpr int kLD = kMaxR + 4;                          // row stride of the parked slot accumulators
constexpr int kRedBytes = 16 * kLD * 4;
constexpr int kRhoBytes = kHeld * kRows * kMaxR * 4;    // 64 KB
// 74 KB in all: three CTAs per SM.  Fa*alpha and the bias take the space of the slot sums once every peer has read them
// (a second cluster barrier).  A separate 8 KB for them saves that barrier but leaves two CTAs per SM, and padding the
// rho rows against bank conflicts costs the same: both measured slower on the headline batch (DESIGN.md section 5.3).
constexpr int kSmemBytes = kRhoBytes + kRedBytes + (kBars + 1) * 8;

__device__ __forceinline__ uint32_t cluster_addr(uint32_t a, uint32_t rank) {   // this CTA's shared address in CTA `rank`
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    return r;
}
// 4 bytes into a peer's shared memory, counted on the peer's mbarrier as transaction bytes
__device__ __forceinline__ void st_async(uint32_t addr, float v, uint32_t bar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(addr),
                 "r"(__float_as_uint(v)), "r"(bar)
                 : "memory");
}

// The per-state arithmetic of speaker_model_body (vbx_kernels.cu) without a prior or given model, statement for
// statement, so that both compute the same invL, alpha, bias and regulariser bit for bit (tests/test_em_contract_gpu.py
// holds them to it).  speaker_model_body keeps its own copy: calling this from it changes the register allocation and so
// the machine code of the speaker-model kernels.  A change to either copy must be made to both.  The thread is column r
// of state s, its warp r / 32; Ns = ws.occ of the state, read by the caller (only for live states); gr = sum over the
// recording's M-tiles of gamma^T rho in tile order (float64).  Returns Fa * alpha and the values alpha_io / invL_io take
// (all 0 in dead columns); the warp's sums of the bias and regulariser terms go to cpart[s][warp] / rpart[s][warp].
__device__ __forceinline__ float speaker_state(int s, int r, int ns, float Ns, float phi, float Fa, float FaFb, double gr,
                                               float &alpha_out, float &invL_out, double (*cpart)[4],
                                               double (*rpart)[4]) {
    const int warp = r >> 5, lane = r & 31;
    const bool dead = s >= ns;   // dead (or padding) column: never wins, never contributes
    float invL = 1.f, alpha = 0.f, Av = 0.f;
    float c = 0.f, reg = 0.f;
    if (!dead) {
        invL = 1.f / (1.f + FaFb * Ns * phi);
        alpha = (float)((double)(FaFb * invL) * gr);
        Av = Fa * alpha;
        const float a2 = alpha * alpha;
        reg = logf(invL) - invL - a2 + 1.f;
        c = (invL + a2) * phi;
    }
    alpha_out = dead ? 0.f : alpha;
    invL_out = dead ? 0.f : invL;
    c = group_sum<32>(c);                             // 32 terms in float, the rest in float64
    reg = group_sum<32>(reg);
    if (lane == 0) {
        cpart[s][warp] = (double)c;
        rpart[s][warp] = (double)reg;
    }
    return Av;
}
// bias (returned) and regulariser (regp) of state s from the four warps' sums of speaker_state; dFa = ws.hp[rec].dFa
__device__ __forceinline__ float speaker_bias(double dFa, int s, int ns, double (*cpart)[4], double (*rpart)[4],
                                              double &regp) {
    const bool dead = s >= ns;
    regp = dead ? 0.0 : (rpart[s][0] + rpart[s][1]) + (rpart[s][2] + rpart[s][3]);
    return dead ? CUDART_INF_F : (float)(dFa * 0.5 * ((cpart[s][0] + cpart[s][1]) + (cpart[s][2] + cpart[s][3])));
}
}  // namespace

template <int S_PAD, int CL>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(128, 3)
    em_contract_kernel(Plan pl, Workspace ws, const float *__restrict__ rho, const float *__restrict__ gamma,
                       const float *__restrict__ Phi, const int32_t *__restrict__ n_states, float *alpha_io,
                       float *invL_io) {
    constexpr int S8 = S_PAD > 8 ? S_PAD : 8;   // states of the speaker model and of the log-likelihood's n-tiles
    constexpr int NT = S8 / 8;
    constexpr int KS = kMaxR / 8;               // k-steps of the log-likelihood
    constexpr int NOWN = (S8 + CL - 1) / CL;    // states owned per CTA
    static_assert(NT * KS * 64 + S8 <= 16 * kLD && kHeld * kRows * S_PAD <= 16 * kLD, "gamma, Fa*alpha and bias must fit in the slot accumulators' space");
    extern __shared__ __align__(128) float4 smem4[];
    float *srho = reinterpret_cast<float *>(smem4);                  // [kHeld][kRows][kMaxR]
    float (*red)[kLD] = reinterpret_cast<float (*)[kLD]>(srho + kHeld * kRows * kMaxR);   // [16][kLD] slot accumulators
    float *sAv = &red[0][0];     // after the speaker model: Fa*alpha [NT][KS][32 lanes][2], the fragment order of loglik_mma
    float *sbias = sAv + NT * KS * 64;                               // [S8]
    const uint32_t bar0 = smem_u32(srho + kHeld * kRows * kMaxR + 16 * kLD);   // kBars load barriers
    const uint32_t avbar = bar0 + 8 * kBars;   // Fa*alpha and bias of every state, sent by the peers with st.async
    __shared__ double cpart[S8][4], rpart[S8][4];

    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank();
    const int rec = blockIdx.x / CL;
    if (!ws.active[rec]) return;   // the same flag for every CTA of the cluster: none leaves while a peer may touch it
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    const int tile = rank / kSlots, fs = rank % kSlots;
    const int64_t r0 = pl.offsets[rec], T = pl.offsets[rec + 1] - r0;
    const int ntiles = (int)((T + kMTile - 1) / kMTile);
    const int64_t f0 = r0 + (int64_t)tile * kMTile;
    const int len = tile < ntiles ? (int)min((int64_t)kMTile, T - (int64_t)tile * kMTile) : 0;
    const int nchunks = (len + kRows - 1) / kRows;
    const int nmine = nchunks > fs ? (nchunks - fs + kSlots - 1) / kSlots : 0;   // held chunks c = fs + 4i, i < nmine
    const int nmt = (nmine + 1) >> 1;                                            // m-tiles of 16 held rows
    // The speaker model's inputs from global memory, read while rho is loading.  Read behind the cluster barrier, as
    // they were, they put up to three dependent L2 round trips between the M-step and the log-likelihood (the
    // occupancies wait for n_states, the bias for a read behind a CTA barrier), and that path holds the CTA's rho slice.
    const int ns = n_states ? n_states[rec] : S_PAD;
    const float phi = Phi[tid];
    const float Fa = ws.hp[rec].Fa, FaFb = ws.hp[rec].FaFb;
    const double dFa = ws.hp[rec].dFa;
    float Ns[NOWN];
#pragma unroll
    for (int k = 0; k < NOWN; ++k) {
        const int s = rank + CL * k;
        Ns[k] = s < ns ? ws.occ[(int64_t)rec * S_PAD + s] : 0.f;
    }

    // ---- load: held chunk i on mbarrier i / 4; rows past the end of the recording (up to the last m-tile) are zero ----
    if (tid == 0) {
        for (int b = 0; b <= kBars; ++b) mbar_init(bar0 + 8 * b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(avbar, (NT * KS * 64 + S_PAD) * 4);
    }
    __syncthreads();
    auto chunk_rows = [&](int i) { return min(kRows, len - kRows * (fs + kSlots * i)); };
    float *sgam = &red[0][0];    // during the M-step: gamma rows of the held chunks [kHeld][kRows][S_PAD]
    if (warp == 0) {
        if (lane < kBars && kHeld / kBars * lane < nmine) {
            uint32_t bytes = 0;
            for (int i = kHeld / kBars * lane; i < min(nmine, kHeld / kBars * (lane + 1)); ++i)
                bytes += chunk_rows(i) * (kMaxR + S_PAD) * 4;
            mbar_expect_tx(bar0 + 8 * lane, bytes);
        }
        __syncwarp();
        if (lane < nmine) {
            const int64_t fr = f0 + kRows * (fs + kSlots * lane);
            const uint32_t bar = bar0 + 8 * (lane / (kHeld / kBars));
            bulk_g2s(smem_u32(srho + lane * kRows * kMaxR), rho + fr * kMaxR, chunk_rows(lane) * kMaxR * 4, bar);
            bulk_g2s(smem_u32(sgam + lane * kRows * S_PAD), gamma + fr * S_PAD, chunk_rows(lane) * S_PAD * 4, bar);
        }
    }
    {
        const int valid = nmine ? kRows * (nmine - 1) + chunk_rows(nmine - 1) : 0;   // held rows with a frame
        float4 *z = reinterpret_cast<float4 *>(srho);
        for (int i = valid * (kMaxR / 4) + tid; i < 2 * nmt * kRows * (kMaxR / 4); i += 128) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();

    // ---- M-step: warp w runs the mma chains of n-tiles 4w .. 4w+3 (columns 32w + 4g + e) over the held chunks ----
    {
        float acc[4][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[e][0] = acc[e][1] = acc[e][2] = acc[e][3] = 0.f;
        const int s0c = min(g, S_PAD - 1), s1c = min(g + 8, S_PAD - 1);
        const bool v0 = g < S_PAD, v1 = g + 8 < S_PAD;
        for (int i = 0; i < nmine; ++i) {
            const int c = fs + kSlots * i;
            const bool va = 8 * c + q < len, vb = 8 * c + q + 4 < len;
            if (i % (kHeld / kBars) == 0) mbar_wait(bar0 + 8 * (i / (kHeld / kBars)), 0);
            // gamma rows past the end are never copied: their values are replaced by 0 before use
            const float *ga = sgam + (i * kRows + q) * S_PAD, *gb = ga + 4 * S_PAD;
            uint32_t ah[4], al[4];
            split_tf32((va && v0) ? ga[s0c] : 0.f, ah[0], al[0]);
            split_tf32((va && v1) ? ga[s1c] : 0.f, ah[1], al[1]);
            split_tf32((vb && v0) ? gb[s0c] : 0.f, ah[2], al[2]);
            split_tf32((vb && v1) ? gb[s1c] : 0.f, ah[3], al[3]);
            const float4 x0 = *reinterpret_cast<const float4 *>(srho + (i * kRows + q) * kMaxR + 32 * warp + 4 * g);
            const float4 x1 = *reinterpret_cast<const float4 *>(srho + (i * kRows + q + 4) * kMaxR + 32 * warp + 4 * g);
            const float b0v[4] = {x0.x, x0.y, x0.z, x0.w};
            const float b1v[4] = {x1.x, x1.y, x1.z, x1.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                uint32_t bh0, bl0, bh1, bl1;
                split_tf32(b0v[e], bh0, bl0);
                split_tf32(b1v[e], bh1, bl1);
                mma_tf32(acc[e], al, bh0, bh1);
                mma_tf32(acc[e], ah, bl0, bl1);
                mma_tf32(acc[e], ah, bh0, bh1);
            }
        }
        __syncthreads();   // every warp is done with the gamma rows the slot accumulators replace
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int c0 = 32 * warp + 8 * q + e, c1 = c0 + 4;   // n = 2q, 2q+1
            red[g][c0] = acc[e][0];
            red[g][c1] = acc[e][1];
            red[g + 8][c0] = acc[e][2];
            red[g + 8][c1] = acc[e][3];
        }
    }
    cluster.sync();   // every slot accumulator of the recording is parked

    // ---- speaker model of the owned states s = rank + CL k; thread = r ----
    // The global stores of the speaker model wait until the slot sums are no longer needed: a cluster barrier's release
    // would otherwise wait for them to drain.
    float avs[NOWN], alphas[NOWN], invLs[NOWN];
    {
        // Every slot accumulator the thread needs, from every CTA of the cluster, is read before any is summed, so that
        // the distributed-shared-memory reads are in flight together.  Read per state, each state's reads would wait
        // behind the previous state's stores to cpart and rpart (the compiler cannot tell the two memories apart).
        // Tiles past the recording's end are read but not summed.
        constexpr int MT = CL / kSlots;   // M-tiles of the cluster
        float red_v[NOWN][MT][kSlots];
#pragma unroll
        for (int k = 0; k < NOWN; ++k) {
            const int s = min(rank + CL * k, S8 - 1);
#pragma unroll
            for (int t = 0; t < MT; ++t)
#pragma unroll
                for (int k2 = 0; k2 < kSlots; ++k2) red_v[k][t][k2] = cluster.map_shared_rank(&red[s][tid], kSlots * t + k2)[0];
        }
#pragma unroll
        for (int k = 0; k < NOWN; ++k) {
            const int s = rank + CL * k;
            avs[k] = 0.f;
            if (s < S8) {
                double gr = 0.0;
                if (s < ns)
#pragma unroll
                    for (int t = 0; t < MT; ++t) {
                        if (t < ntiles) {
                            float v = red_v[k][t][0];
#pragma unroll
                            for (int k2 = 1; k2 < kSlots; ++k2) v += red_v[k][t][k2];
                            gr += (double)v;
                        }
                    }
                avs[k] = speaker_state(s, tid, ns, Ns[k], phi, Fa, FaFb, gr, alphas[k], invLs[k], cpart, rpart);
            }
        }
    }
    __syncthreads();
    float own_bias = 0.f;
    double own_regp = 0.0;
    if (tid < NOWN && rank + CL * tid < S_PAD) own_bias = speaker_bias(dFa, rank + CL * tid, ns, cpart, rpart, own_regp);
    cluster.sync();   // every peer has read the slot sums: their space takes Fa*alpha and the bias
    {
        // column r of state s  ->  fragment element ((i KS + j) 32 + 4 gs + fq) 2 + e of loglik_mma's R = 128 permutation
        const int r = tid, j = 2 * (r >> 4) + ((r >> 1) & 1), fq = (r >> 2) & 3, e = r & 1;
#pragma unroll
        for (int k = 0; k < NOWN; ++k) {
            const int s = rank + CL * k;
            if (s < S8) {
                const uint32_t a = smem_u32(sAv + (((s >> 3) * KS + j) * 32 + 4 * (s & 7) + fq) * 2 + e);
#pragma unroll
                for (int p = 0; p < CL; ++p) st_async(cluster_addr(a, p), avs[k], cluster_addr(avbar, p));
            }
        }
        if (tid < NOWN && rank + CL * tid < S_PAD) {
            const int s = rank + CL * tid;
#pragma unroll
            for (int p = 0; p < CL; ++p) st_async(cluster_addr(smem_u32(sbias + s), p), own_bias, cluster_addr(avbar, p));
            ws.bias[(int64_t)rec * S_PAD + s] = own_bias;
            ws.regp[(int64_t)rec * S_PAD + s] = own_regp;
        }
#pragma unroll
        for (int k = 0; k < NOWN; ++k) {
            const int s = rank + CL * k;
            if (s < S_PAD) {
                const int64_t o = ((int64_t)rec * S_PAD + s) * kMaxR + tid;
                if (alpha_io) alpha_io[o] = alphas[k];
                if (invL_io) invL_io[o] = invLs[k];
            }
        }
    }
    mbar_wait(avbar, 0);   // Fa*alpha and the bias of every state are here

    // ---- log-likelihood over the held rows: m-tile u = held rows 16u + 2g (fragment row g) and 16u + 2g + 1 (row g + 8) ----
    float nb[NT][2];
#pragma unroll
    for (int i = 0; i < NT; ++i) {
        const int s = 8 * i + 2 * q;
        nb[i][0] = s < S_PAD ? -sbias[s] : -CUDART_INF_F;
        nb[i][1] = s + 1 < S_PAD ? -sbias[s + 1] : -CUDART_INF_F;
    }
    // Warp w takes m-tiles w and w + 4 together (twice the independent mma chains).  When w + 4 >= nmt the second
    // m-tile's rows hold no frame of the recording: whatever they compute is never stored.
    const uint2 *sB = reinterpret_cast<const uint2 *>(sAv);
    if (warp < nmt) {
        float D[2][NT][4], E[2][NT][4];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int i = 0; i < NT; ++i) {
                D[m][i][0] = nb[i][0];
                D[m][i][1] = nb[i][1];
                D[m][i][2] = nb[i][0];
                D[m][i][3] = nb[i][1];
                E[m][i][0] = E[m][i][1] = E[m][i][2] = E[m][i][3] = 0.f;
            }
        const float4 *pa[2], *pb[2];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
            pa[m] = reinterpret_cast<const float4 *>(srho + (16 * (warp + 4 * m) + 2 * g) * kMaxR + 4 * q);
            pb[m] = reinterpret_cast<const float4 *>(srho + (16 * (warp + 4 * m) + 2 * g + 1) * kMaxR + 4 * q);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float4 xa[2], xb[2];
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                xa[m] = pa[m][4 * k];
                xb[m] = pb[m][4 * k];
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {   // k-step j = 2k + h: columns 16k + 4q + 2h, +1
                const int j = 2 * k + h;
                uint32_t ah[2][4], al[2][4];
#pragma unroll
                for (int m = 0; m < 2; ++m) {
                    split_tf32(h ? xa[m].z : xa[m].x, ah[m][0], al[m][0]);
                    split_tf32(h ? xb[m].z : xb[m].x, ah[m][1], al[m][1]);
                    split_tf32(h ? xa[m].w : xa[m].y, ah[m][2], al[m][2]);
                    split_tf32(h ? xb[m].w : xb[m].y, ah[m][3], al[m][3]);
                }
#pragma unroll
                for (int i = 0; i < NT; ++i) {
                    const uint2 b = sB[(i * KS + j) * 32 + lane];
                    const uint32_t hx = b.x & 0xffffe000u, hy = b.y & 0xffffe000u;
                    const uint32_t lx = __float_as_uint(__uint_as_float(b.x) - __uint_as_float(hx));
                    const uint32_t ly = __float_as_uint(__uint_as_float(b.y) - __uint_as_float(hy));
#pragma unroll
                    for (int m = 0; m < 2; ++m) {
                        mma_tf32(E[m][i], al[m], hx, hy);
                        mma_tf32(D[m][i], ah[m], hx, hy);
                        mma_tf32(E[m][i], ah[m], lx, ly);
                    }
                }
            }
        }
#pragma unroll
        for (int m = 0; m < 2; ++m) {
#pragma unroll
            for (int i = 0; i < NT; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) D[m][i][e] += E[m][i][e];
            float m0 = fmaxf(D[m][0][0], D[m][0][1]), m1 = fmaxf(D[m][0][2], D[m][0][3]);
#pragma unroll
            for (int i = 1; i < NT; ++i) {
                m0 = fmaxf(m0, fmaxf(D[m][i][0], D[m][i][1]));
                m1 = fmaxf(m1, fmaxf(D[m][i][2], D[m][i][3]));
            }
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            const int u = warp + 4 * m;
            // frames of held rows 16u + 2g and 16u + 2g + 1 in the tile (held row L: chunk fs + 4 (L / 8), row L % 8)
            const int ta = kRows * (fs + kSlots * (2 * u + (g >> 2))) + 2 * (g & 3), tb = ta + 1;
#pragma unroll
            for (int i = 0; i < NT; ++i) {
                const int s = 8 * i + 2 * q;
                if (s < S_PAD) {
                    const float2 va = make_float2(expf(D[m][i][0] - m0), expf(D[m][i][1] - m0));
                    const float2 vb = make_float2(expf(D[m][i][2] - m1), expf(D[m][i][3] - m1));
                    if (ta < len) *reinterpret_cast<float2 *>(ws.p + (f0 + ta) * S_PAD + s) = va;
                    if (tb < len) *reinterpret_cast<float2 *>(ws.p + (f0 + tb) * S_PAD + s) = vb;
                }
            }
            if (q == 0) {
                if (ta < len) ws.rowmax[f0 + ta] = m0;
                if (tb < len) ws.rowmax[f0 + tb] = m1;
            }
        }
    }
}

// CL when the kernel may have its shared memory on the current device and one cluster fits there, else 0 (the three
// kernels run instead; a refusal is not an error).  Called by vbx_plan on the plan's device.
template <int S_PAD, int CL>
static int em_contract_cluster_t() {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CL);
    cfg.blockDim = dim3(128);
    cfg.dynamicSmemBytes = kSmemBytes;
    int n = 0;
    if (!allow_dynamic_smem(em_contract_kernel<S_PAD, CL>, kSmemBytes) ||
        cudaOccupancyMaxActiveClusters(&n, em_contract_kernel<S_PAD, CL>, &cfg) != cudaSuccess)
        return (void)cudaGetLastError(), 0;
    return n >= 1 ? CL : 0;
}

int em_contract_cluster(int S, int R, int64_t max_T, bool split) {
    if (split || R != kMaxR || max_T > 2 * kMTile) return 0;
    const bool two = max_T > kMTile;
    switch (S) {
        case 4: return two ? em_contract_cluster_t<4, 8>() : em_contract_cluster_t<4, 4>();
        case 8: return two ? em_contract_cluster_t<8, 8>() : em_contract_cluster_t<8, 4>();
        case 16: return two ? em_contract_cluster_t<16, 8>() : em_contract_cluster_t<16, 4>();
        default: return 0;
    }
}

int launch_em_contract(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, const float *Phi,
                       const int32_t *n_states, float *alpha_io, float *invL_io, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    const int CL = pl.em_cluster;
#define VBX_EMC(S_, CL_)                                                                                                 \
    em_contract_kernel<S_, CL_><<<pl.n_rec * CL_, 128, kSmemBytes, st>>>(pl, ws, rho, gamma, Phi, n_states, alpha_io, invL_io)
    switch (pl.S * 16 + CL) {
        case 4 * 16 + 4: VBX_EMC(4, 4); break;
        case 4 * 16 + 8: VBX_EMC(4, 8); break;
        case 8 * 16 + 4: VBX_EMC(8, 4); break;
        case 8 * 16 + 8: VBX_EMC(8, 8); break;
        case 16 * 16 + 4: VBX_EMC(16, 4); break;
        case 16 * 16 + 8: VBX_EMC(16, 8); break;
        default: return -1;
    }
#undef VBX_EMC
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace vbx
