// The two skinny in-loop contractions of the EM iteration on the tensor cores, in split-precision
// "3xTF32" (hi*hi + lo*hi + hi*lo, fp32 accumulate), so that results stay at float32 accuracy
// (plain TF32 breaks the 1e-4 parity bar, SURVEY.md section 7 hard part 4):
//
//   mstep_mma   partial[tile][s][r] = sum_{t in tile} gamma[t,s] * rho[t,r]              VBx/VBx.py:96
//   loglik_mma  ll[t,s] = sum_r rho[t,r] * A[s,r] - bias[s]; rowmax; p = exp(ll - rowmax)  VBx/VBx.py:97
//
// Both stream rho exactly once with coalesced 16-byte loads straight into mma.sync fragments (the k / n
// index of the fragment is permuted so that every thread reads contiguous floats), no shared-memory
// staging of rho, and 8-16 KB of loads in flight per warp (ping-pong register sets).
// mma.sync.m16n8k8.tf32 fragment layout (g = lane/4, q = lane%4):
//   A (16x8 row): a0=(g,q) a1=(g+8,q) a2=(g,q+4) a3=(g+8,q+4)    B (8x8 col): b0=(k=q,n=g) b1=(k=q+4,n=g)
//   C/D (16x8):   c0=(g,2q) c1=(g,2q+1) c2=(g+8,2q) c3=(g+8,2q+1)
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {

__device__ __forceinline__ void cp_async16_(void *smem, const void *gmem) {
    unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}

// ------------------------------------------------------------------------------------------------
// M-step accumulation.  D[state][r] (M = 16 states per m-tile, N = 8 r per n-tile, K = 8 frames).
// A = gamma^T chunk (scalar loads, tiny), B = rho chunk.  n-tile j, column n  <->  r = rb + 32*(j/4) + 4*n + j%4,
// so float4 number m of the thread with g = n covers r = rb + 32m + 4g .. +3: the eight g-lanes of a row read one
// full 128-byte line per instruction.  One CTA (4 warps) per <=kMTile-frame tile; warp = (frame slot, r-group);
// the slots are summed through shared memory in fixed order (deterministic).
// ------------------------------------------------------------------------------------------------
// S = 128: two groups of four warps, one per half of the states, each tiled like S = 64; the 67 KB reduction buffer is
// dynamic shared memory.
template <int S_PAD>
__global__ void __launch_bounds__(S_PAD > kMaxS ? 256 : 128, S_PAD > kMaxS ? 2 : 4)
    mstep_mma_kernel(Plan pl, Workspace ws, const float *__restrict__ rho, const float *__restrict__ gamma) {
    constexpr int SH = S_PAD > kMaxS ? S_PAD / kMaxS : 1;  // state blocks, one warp group each
    constexpr int SB = S_PAD / SH;                   // states of one warp group
    constexpr int MT = SB > 16 ? SB / 16 : 1;        // m-tiles of 16 states
    constexpr int NTW = 16 / MT;                     // n-tiles (8 r each) per warp
    constexpr int RW = 8 * NTW;                      // r range of one warp
    constexpr int FS = 4 / MT;                       // frame slots
    constexpr int NQ = NTW / 4;                      // float4 per row per thread
    constexpr int S16 = 16 * MT;
    constexpr int LD = kMaxR + 4;
    __shared__ __align__(16) float red_st[SH > 1 ? 1 : FS][SH > 1 ? 1 : S16][LD];
    extern __shared__ float4 red_dyn[];
    float (*red)[S16 * SH][LD] = SH > 1 ? reinterpret_cast<float (*)[S16 * SH][LD]>(red_dyn) : reinterpret_cast<float (*)[S16 * SH][LD]>(red_st);
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    const int sh = SH > 1 ? warp >> 2 : 0, w4 = SH > 1 ? (warp & 3) : warp;
    const int rg = w4 % MT, fs = w4 / MT;
    const int R = pl.R;
    const int col0 = rg * RW + 4 * g;
    const float *grow = gamma + f0 * S_PAD + sh * SB;

    float acc[MT][NTW][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < NTW; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;

    struct Raw {
        float4 x0[NQ], x1[NQ];
        float ga[MT][4];
    };
    // All loads are unconditional with clamped indices (a predicated load becomes load + select, which waits for
    // the data on the spot): frames past the tile end get gamma = 0 at USE time, columns past R land in
    // accumulators that are never written out.
    auto load_chunk = [&](const int c, Raw &r) {
        const int tac = min(8 * c + q, len - 1), tbc = min(8 * c + q + 4, len - 1);
        const float *xa = rho + (f0 + tac) * R, *xb = rho + (f0 + tbc) * R;
#pragma unroll
        for (int k = 0; k < NQ; ++k) {
            const int col = min(col0 + 32 * k, R - 4);
            r.x0[k] = __ldg(reinterpret_cast<const float4 *>(xa + col));
            r.x1[k] = __ldg(reinterpret_cast<const float4 *>(xb + col));
        }
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const int s0c = min(16 * m + g, S_PAD - 1), s1c = min(16 * m + g + 8, S_PAD - 1);
            r.ga[m][0] = __ldg(grow + (int64_t)tac * S_PAD + s0c);
            r.ga[m][1] = __ldg(grow + (int64_t)tac * S_PAD + s1c);
            r.ga[m][2] = __ldg(grow + (int64_t)tbc * S_PAD + s0c);
            r.ga[m][3] = __ldg(grow + (int64_t)tbc * S_PAD + s1c);
        }
    };
    auto compute = [&](const Raw &r, const int c) {
        const bool va = 8 * c + q < len, vb = 8 * c + q + 4 < len;
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const bool v0 = 16 * m + g < S_PAD, v1 = 16 * m + g + 8 < S_PAD;
            split_tf32((va && v0) ? r.ga[m][0] : 0.f, ah[m][0], al[m][0]);
            split_tf32((va && v1) ? r.ga[m][1] : 0.f, ah[m][1], al[m][1]);
            split_tf32((vb && v0) ? r.ga[m][2] : 0.f, ah[m][2], al[m][2]);
            split_tf32((vb && v1) ? r.ga[m][3] : 0.f, ah[m][3], al[m][3]);
        }
#pragma unroll
        for (int k = 0; k < NQ; ++k) {
            const float b0v[4] = {r.x0[k].x, r.x0[k].y, r.x0[k].z, r.x0[k].w};
            const float b1v[4] = {r.x1[k].x, r.x1[k].y, r.x1[k].z, r.x1[k].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                uint32_t bh0, bl0, bh1, bl1;
                split_tf32(b0v[e], bh0, bl0);
                split_tf32(b1v[e], bh1, bl1);
                const int j = 4 * k + e;
#pragma unroll
                for (int m = 0; m < MT; ++m) {
                    mma_tf32(acc[m][j], al[m], bh0, bh1);
                    mma_tf32(acc[m][j], ah[m], bl0, bl1);
                    mma_tf32(acc[m][j], ah[m], bh0, bh1);
                }
            }
        }
    };
    const int nchunks = (len + 7) >> 3;
    // Load latency is covered by the 16 resident warps per SM (4 CTAs of 4 warps, 2 of 8 at S = 128); the fragment
    // registers are single-buffered to keep the kernel at <= 128 registers.
    Raw ra;
    for (int c = fs; c < nchunks; c += FS) {
        load_chunk(c, ra);
        compute(ra, c);
    }
    // every slot parks its fragment in shared memory, then the CTA sums the slots in fixed order
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < NTW; ++j) {
            const int r0 = rg * RW + 32 * (j >> 2) + 8 * q + (j & 3), r1 = r0 + 4;   // n = 2q, 2q+1
            red[fs][sh * S16 + 16 * m + g][r0] = acc[m][j][0];
            red[fs][sh * S16 + 16 * m + g][r1] = acc[m][j][1];
            red[fs][sh * S16 + 16 * m + g + 8][r0] = acc[m][j][2];
            red[fs][sh * S16 + 16 * m + g + 8][r1] = acc[m][j][3];
        }
    __syncthreads();
    const int R4 = R >> 2;
    float *out = ws.partial + (int64_t)tile * S_PAD * R;
    for (int i = threadIdx.x; i < S_PAD * R4; i += 128 * SH) {
        const int s = i / R4, c4 = i - s * R4;
        float4 v = *reinterpret_cast<const float4 *>(&red[0][s][4 * c4]);
#pragma unroll
        for (int k = 1; k < FS; ++k) {
            const float4 o = *reinterpret_cast<const float4 *>(&red[k][s][4 * c4]);
            v.x += o.x;
            v.y += o.y;
            v.z += o.z;
            v.w += o.w;
        }
        *reinterpret_cast<float4 *>(out + (int64_t)s * R + 4 * c4) = v;
    }
}

int launch_mstep_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *gamma, cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    switch (pl.S) {
        case 4: mstep_mma_kernel<4><<<pl.n_mtiles, 128, 0, st>>>(pl, ws, rho, gamma); break;
        case 8: mstep_mma_kernel<8><<<pl.n_mtiles, 128, 0, st>>>(pl, ws, rho, gamma); break;
        case 16: mstep_mma_kernel<16><<<pl.n_mtiles, 128, 0, st>>>(pl, ws, rho, gamma); break;
        case 32: mstep_mma_kernel<32><<<pl.n_mtiles, 128, 0, st>>>(pl, ws, rho, gamma); break;
        case 64: mstep_mma_kernel<64><<<pl.n_mtiles, 128, 0, st>>>(pl, ws, rho, gamma); break;
        case kMaxSWide: {
            constexpr int smem = kMaxSWide * (kMaxR + 4) * sizeof(float);
            if (!allow_dynamic_smem(mstep_mma_kernel<kMaxSWide>, smem)) return -1;
            mstep_mma_kernel<kMaxSWide><<<pl.n_mtiles, 256, smem, st>>>(pl, ws, rho, gamma);
            break;
        }
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// log-likelihood + row softmax numerator.  D[frame][state] (M = 16 frames, N = 8 states per n-tile, K = 8 r).
// A = rho rows.  R = 128: k-step j, k = q / q+4  <->  column 16*(j/2) + 4q + 2*(j%2) / +1, i.e. float4 number m of a
// thread covers columns 16m + 4q .. +3 and the four lanes of a quad read 64 contiguous bytes of a row per
// instruction.  Other R: column KQ*q + 2j / +1 (KQ = 2*ceil(R/8) contiguous floats per thread).
// B = Fa*alpha, pre-split into hi/lo and stored fragment-major by the speaker-model kernel
// (ws.Afrag_hi/lo: [rec][n-tile][k-step][lane] float2), staged once per CTA in shared memory.
// One CTA (4 warps) per <=256-frame tile, a warp owns every 4th 16-frame m-tile.
// ------------------------------------------------------------------------------------------------
// WITH_C: also emit c_t = sum_j p[t,j] w_j (w = (1-loopP) pi + 1e-8), the reduction the split sweeps take out of their
// recursion (vbx_fb_split.cu).  Costs ~14 % of this kernel's time on bandwidth-bound batches, so only plans that chose the
// split sweeps (small batches) instantiate it.
// S = 128 (split plans only, WITH_C): the staged fragments take 128 KB, one CTA per SM, so the CTA has 8 warps; the lo*hi /
// hi*lo terms accumulate into D itself (16 n-tiles of separate E accumulators would not fit the register file).
template <int S_PAD, bool R128, bool WITH_C>
__global__ void __launch_bounds__(S_PAD > kMaxS ? 256 : 128, S_PAD > kMaxS ? 1 : 3)
    loglik_mma_kernel(Plan pl, Workspace ws, const float *__restrict__ rho, const float *__restrict__ pi,
                      const int32_t *__restrict__ n_states) {
    constexpr int NT = S_PAD > 8 ? S_PAD / 8 : 1;
    constexpr int NW = S_PAD > kMaxS ? 8 : 4;      // warps per CTA
    constexpr bool SPLIT_E = S_PAD <= kMaxS;       // separate accumulators for the small split terms
    extern __shared__ uint2 sfrag[];
    const int R = pl.R;
    const int KS = R128 ? 16 : (R + 7) >> 3;  // k-steps
    const int KQ = 2 * KS;                   // floats per thread per row
    uint2 *sBh = sfrag, *sBl = sfrag + NT * KS * 32;
    const int tile = blockIdx.x;
    const int rec = pl.mtile_rec[tile];
    if (!ws.active[rec]) return;
    const int64_t f0 = pl.mtile_f0[tile];
    const int len = (int)min((int64_t)kMTile, pl.offsets[rec + 1] - f0);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, q = lane & 3;
    {
        const int n16 = NT * KS * 32 / 2;  // 16-byte units per array
        const uint4 *gh = reinterpret_cast<const uint4 *>(ws.Afrag_hi + (int64_t)rec * NT * KS * 64);
        const uint4 *gl = reinterpret_cast<const uint4 *>(ws.Afrag_lo + (int64_t)rec * NT * KS * 64);
        for (int i = tid; i < n16; i += 32 * NW) {
            cp_async16_(reinterpret_cast<uint4 *>(sBh) + i, gh + i);
            cp_async16_(reinterpret_cast<uint4 *>(sBl) + i, gl + i);
        }
        asm volatile("cp.async.commit_group;\n" ::);
    }
    float nb[NT][2], wv[NT][2];      // -bias and the transition weights w = Q pi + 1e-8 of this thread's states
    const int ns = n_states ? n_states[rec] : S_PAD;
    const float Q = WITH_C ? 1.f - ws.hp[rec].loopP : 0.f;
#pragma unroll
    for (int i = 0; i < NT; ++i) {
        const int s = 8 * i + 2 * q;
        nb[i][0] = s < S_PAD ? -ws.bias[(int64_t)rec * S_PAD + s] : -CUDART_INF_F;
        nb[i][1] = s + 1 < S_PAD ? -ws.bias[(int64_t)rec * S_PAD + s + 1] : -CUDART_INF_F;
        wv[i][0] = (WITH_C && s < ns) ? fmaf(Q, pi[(int64_t)rec * S_PAD + s], VBX_EPS_TR) : 0.f;
        wv[i][1] = (WITH_C && s + 1 < ns) ? fmaf(Q, pi[(int64_t)rec * S_PAD + s + 1], VBX_EPS_TR) : 0.f;
    }
    const int n_mt = (len + 15) >> 4;

    auto finish = [&](float (&D)[NT][4], const float (&E)[NT][4], const int mt) {
        if constexpr (SPLIT_E) {
#pragma unroll
            for (int i = 0; i < NT; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) D[i][e] += E[i][e];
        }
        float m0 = fmaxf(D[0][0], D[0][1]), m1 = fmaxf(D[0][2], D[0][3]);
#pragma unroll
        for (int i = 1; i < NT; ++i) {
            m0 = fmaxf(m0, fmaxf(D[i][0], D[i][1]));
            m1 = fmaxf(m1, fmaxf(D[i][2], D[i][3]));
        }
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
        m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
        const int ra = mt * 16 + g, rb = ra + 8;
        float c0 = 0.f, c1 = 0.f;                  // c_t = sum_j p[t,j] w_j for the two rows
#pragma unroll
        for (int i = 0; i < NT; ++i) {
            const int s = 8 * i + 2 * q;
            if (s < S_PAD) {
                const float2 pa = make_float2(expf(D[i][0] - m0), expf(D[i][1] - m0));
                const float2 pb = make_float2(expf(D[i][2] - m1), expf(D[i][3] - m1));
                if (WITH_C) {
                    c0 = fmaf(pa.x, wv[i][0], fmaf(pa.y, wv[i][1], c0));
                    c1 = fmaf(pb.x, wv[i][0], fmaf(pb.y, wv[i][1], c1));
                }
                if (ra < len) *reinterpret_cast<float2 *>(ws.p + (f0 + ra) * S_PAD + s) = pa;
                if (rb < len) *reinterpret_cast<float2 *>(ws.p + (f0 + rb) * S_PAD + s) = pb;
            }
        }
        if (WITH_C) {
            c0 += __shfl_xor_sync(0xffffffffu, c0, 1);
            c1 += __shfl_xor_sync(0xffffffffu, c1, 1);
            c0 += __shfl_xor_sync(0xffffffffu, c0, 2);
            c1 += __shfl_xor_sync(0xffffffffu, c1, 2);
        }
        if (q == 0) {
            if (ra < len) {
                ws.rowmax[f0 + ra] = m0;
                if (WITH_C) ws.cvec[f0 + ra] = c0;
            }
            if (rb < len) {
                ws.rowmax[f0 + rb] = m1;
                if (WITH_C) ws.cvec[f0 + rb] = c1;
            }
        }
    };
    // The split terms go to separate accumulators (E: lo*hi + hi*lo, D: hi*hi) so that consecutive mma of a k-step
    // do not depend on each other; E is folded into D in finish().
    auto kstep = [&](float (&D)[NT][4], float (&E)[NT][4], const int j, const float a0, const float a1, const float a2,
                     const float a3) {
        uint32_t ah[4], al[4];
        split_tf32(a0, ah[0], al[0]);
        split_tf32(a1, ah[1], al[1]);
        split_tf32(a2, ah[2], al[2]);
        split_tf32(a3, ah[3], al[3]);
#pragma unroll
        for (int i = 0; i < NT; ++i) {
            const uint2 bh = sBh[(i * KS + j) * 32 + lane];
            const uint2 bl = sBl[(i * KS + j) * 32 + lane];
            if constexpr (SPLIT_E) {
                mma_tf32(E[i], al, bh.x, bh.y);
                mma_tf32(D[i], ah, bh.x, bh.y);
                mma_tf32(E[i], ah, bl.x, bl.y);
            } else {
                mma_tf32(D[i], al, bh.x, bh.y);
                mma_tf32(D[i], ah, bl.x, bl.y);
                mma_tf32(D[i], ah, bh.x, bh.y);
            }
        }
    };

    if (R128 && SPLIT_E) {   // S = 128 takes the loop below: no room for a register copy of the two rows
        struct Raw {
            float4 xa[8], xb[8];
        };
        auto load_mt = [&](const int mt, Raw &r) {
            // rows past the tile end are clamped (their results are never stored)
            const int ra = min(mt * 16 + g, len - 1), rb = min(mt * 16 + g + 8, len - 1);
            const float4 *pa = reinterpret_cast<const float4 *>(rho + (f0 + ra) * 128 + 4 * q);
            const float4 *pb = reinterpret_cast<const float4 *>(rho + (f0 + rb) * 128 + 4 * q);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                r.xa[k] = __ldg(pa + 4 * k);
                r.xb[k] = __ldg(pb + 4 * k);
            }
        };
        auto compute = [&](const Raw &r, const int mt) {
            float D[NT][4], E[NT][4];
#pragma unroll
            for (int i = 0; i < NT; ++i) {
                D[i][0] = nb[i][0];
                D[i][1] = nb[i][1];
                D[i][2] = nb[i][0];
                D[i][3] = nb[i][1];
                E[i][0] = E[i][1] = E[i][2] = E[i][3] = 0.f;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                kstep(D, E, 2 * k, r.xa[k].x, r.xb[k].x, r.xa[k].y, r.xb[k].y);
                kstep(D, E, 2 * k + 1, r.xa[k].z, r.xb[k].z, r.xa[k].w, r.xb[k].w);
            }
            finish(D, E, mt);
        };
        Raw r0;
        load_mt(warp, r0);
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();
        for (int mt = warp; mt < n_mt; mt += NW) {
            if (mt != warp) load_mt(mt, r0);
            compute(r0, mt);
        }
    } else {
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();
        for (int mt = warp; mt < n_mt; mt += NW) {
            float D[NT][4], E[NT][4];
#pragma unroll
            for (int i = 0; i < NT; ++i) {
                D[i][0] = nb[i][0];
                D[i][1] = nb[i][1];
                D[i][2] = nb[i][0];
                D[i][3] = nb[i][1];
                E[i][0] = E[i][1] = E[i][2] = E[i][3] = 0.f;
            }
            const int ra = min(mt * 16 + g, len - 1), rb = min(mt * 16 + g + 8, len - 1);
            const float *pa = rho + (f0 + ra) * R;
            const float *pb = rho + (f0 + rb) * R;
#pragma unroll 4
            for (int j = 0; j < KS; ++j) {
                // columns of k-step j (R = 128: the coalesced permutation of the branch above)
                const int col = R128 ? 16 * (j >> 1) + 4 * q + 2 * (j & 1) : KQ * q + 2 * j;
                                                          // columns >= R meet zero entries of the alpha fragments,
                const int cc = min(col, R - 2);           // so only the address needs clamping
                const float2 va = __ldg(reinterpret_cast<const float2 *>(pa + cc));
                const float2 vb = __ldg(reinterpret_cast<const float2 *>(pb + cc));
                kstep(D, E, j, va.x, vb.x, va.y, vb.y);
            }
            finish(D, E, mt);
        }
    }
}

static size_t loglik_mma_smem(int S_pad, int R) {
    const int NT = S_pad > 8 ? S_pad / 8 : 1, KS = (R + 7) / 8;
    return (size_t)2 * NT * KS * 32 * sizeof(uint2);
}

template <int S_PAD>
static int launch_loglik_mma_t(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states,
                               cudaStream_t st) {
    const int big = (int)loglik_mma_smem(S_PAD, kMaxR);
    const size_t smem = loglik_mma_smem(S_PAD, pl.R);
    if constexpr (S_PAD > kMaxS) {   // split plans only (vbx_plan): the c_t variants, 8 warps per CTA
        if (!pl.split) return -1;
        auto kernel = pl.R == 128 ? loglik_mma_kernel<S_PAD, true, true> : loglik_mma_kernel<S_PAD, false, true>;
        if (!allow_dynamic_smem(kernel, big)) return -1;
        kernel<<<pl.n_mtiles, 256, smem, st>>>(pl, ws, rho, pi, n_states);
    } else {
        auto kernel = pl.split ? (pl.R == 128 ? loglik_mma_kernel<S_PAD, true, true> : loglik_mma_kernel<S_PAD, false, true>)
                               : (pl.R == 128 ? loglik_mma_kernel<S_PAD, true, false> : loglik_mma_kernel<S_PAD, false, false>);
        if (!allow_dynamic_smem(kernel, big)) return -1;
        kernel<<<pl.n_mtiles, 128, smem, st>>>(pl, ws, rho, pi, n_states);
    }
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_loglik_mma(const Plan &pl, const Workspace &ws, const float *rho, const float *pi, const int32_t *n_states,
                      cudaStream_t st) {
    if (pl.n_mtiles == 0) return 0;
    switch (pl.S) {
        case 4: return launch_loglik_mma_t<4>(pl, ws, rho, pi, n_states, st);
        case 8: return launch_loglik_mma_t<8>(pl, ws, rho, pi, n_states, st);
        case 16: return launch_loglik_mma_t<16>(pl, ws, rho, pi, n_states, st);
        case 32: return launch_loglik_mma_t<32>(pl, ws, rho, pi, n_states, st);
        case 64: return launch_loglik_mma_t<64>(pl, ws, rho, pi, n_states, st);
        case kMaxSWide: return launch_loglik_mma_t<kMaxSWide>(pl, ws, rho, pi, n_states, st);
        default: return -1;
    }
}

}  // namespace vbx
