// Initial responsibilities from speaker turns (DESIGN.md section 5.20): the VB-HMM started from an existing diarization.
// Recording b has the speakers spk_off[b] .. spk_off[b+1]-1 of the packed turn lists; x-vector t of it, segment [lo, hi)
// in ticks, gets
//     c_k = (ticks of [lo, hi) inside speaker k's turns) / (hi - lo)          (0 when hi <= lo)
//     gamma0[t, k] = softmax_k(smoothing_b * c_k) over k < K_b, 0 in the padded columns;  pi0[b, k] = 1 / K_b
//   init_turns_kernel: a group of lanes per x-vector (the plan's S rounded up to a power of two, at most a warp) over the
//   recording's speakers; the first n_rec * S threads of the grid also write pi0.
#include "vbx_internal.cuh"

namespace vbx {

constexpr int kInitThreads = 256;
constexpr int kInitCache = 4;   // logits kept in registers per lane: 4 x 32 lanes cover every float32 plan (S <= 128)

// P(x): the ticks of a speaker's sorted, disjoint turns [lo[i], hi[i]) (i < n) that lie before x, with cum[i] the length
// of turns 0 .. i-1.  Only the last turn that starts before x can reach past x: every earlier one ends before the next
// one starts.
__device__ __forceinline__ int64_t time_before(const int64_t *__restrict__ lo, const int64_t *__restrict__ hi,
                                               const int64_t *__restrict__ cum, int64_t n, int64_t x) {
    int64_t a = 0, b = n;   // binary search for the number of turns with lo < x
    while (a < b) {
        const int64_t m = (a + b) >> 1;
        if (lo[m] < x) a = m + 1;
        else b = m;
    }
    return a == 0 ? 0 : cum[a - 1] + (min(hi[a - 1], x) - lo[a - 1]);
}

// z_k = smoothing * c_k of speaker k (global index) for the segment [lo, hi)
__device__ __forceinline__ double init_logit(const int64_t *__restrict__ turn_off, const int64_t *__restrict__ turn_lo,
                                             const int64_t *__restrict__ turn_hi, const int64_t *__restrict__ turn_cum,
                                             int64_t k, int64_t lo, int64_t hi, double sm) {
    if (hi <= lo) return 0.0;
    const int64_t f = turn_off[k], n = turn_off[k + 1] - f;
    const int64_t covered = time_before(turn_lo + f, turn_hi + f, turn_cum + f, n, hi) -
                            time_before(turn_lo + f, turn_hi + f, turn_cum + f, n, lo);
    return sm * ((double)covered / (double)(hi - lo));
}

template <typename T>
__global__ void __launch_bounds__(kInitThreads) init_turns_kernel(Plan pl, const int64_t *__restrict__ seg,
                                                                  const int64_t *__restrict__ spk_off,
                                                                  const int64_t *__restrict__ turn_off,
                                                                  const int64_t *__restrict__ turn_lo,
                                                                  const int64_t *__restrict__ turn_hi,
                                                                  const int64_t *__restrict__ turn_cum,
                                                                  const double *__restrict__ smoothing,
                                                                  T *__restrict__ gamma, T *__restrict__ pi, int gw) {
    const int64_t gtid = (int64_t)blockIdx.x * kInitThreads + threadIdx.x;
    const int S = pl.S;
    if (gtid < (int64_t)pl.n_rec * S) {
        const int b = (int)(gtid / S), s = (int)(gtid - (int64_t)b * S);
        const int64_t K = spk_off[b + 1] - spk_off[b];
        pi[gtid] = s < K ? (T)(1.0 / (double)K) : (T)0;
    }
    // a group of gw lanes (a power of two <= 32, >= S when S <= 32) per x-vector; every lane of the warp takes part in
    // the shuffles, also the lanes past the last x-vector
    const int64_t t = gtid / gw;
    const int sub = threadIdx.x & (gw - 1);
    const bool live = t < pl.n_frames;
    int64_t k0 = 0, K = 0, lo = 0, hi = 0;
    double sm = 0.0;
    if (live) {
        const int b = find_problem(pl.offsets, pl.n_rec, t);
        k0 = spk_off[b];
        K = spk_off[b + 1] - k0;
        lo = seg[2 * t];
        hi = seg[2 * t + 1];
        sm = smoothing[b];
    }
    // pass 1: the logits of the lane's first kInitCache speakers are kept in registers (every speaker of a plan with
    // S <= 128); an online softmax normaliser per lane (running max m, sum of exp(z - m)), combined over the group
    double zc[kInitCache];
    double m = -INFINITY, z_sum = 0.0;
#pragma unroll
    for (int j = 0; j < kInitCache; ++j) {
        const int64_t k = sub + (int64_t)j * gw;
        zc[j] = k < K ? init_logit(turn_off, turn_lo, turn_hi, turn_cum, k0 + k, lo, hi, sm) : -INFINITY;
    }
    for (int64_t k = sub; k < K; k += gw) {
        const int64_t j = (k - sub) / gw;
        double z = 0.0;
#pragma unroll
        for (int i = 0; i < kInitCache; ++i)
            if (i == j) z = zc[i];
        if (j >= kInitCache) z = init_logit(turn_off, turn_lo, turn_hi, turn_cum, k0 + k, lo, hi, sm);
        if (z > m) {
            z_sum = z_sum * exp(m - z) + 1.0;
            m = z;
        } else {
            z_sum += exp(z - m);
        }
    }
    double M = m;
    for (int o = gw >> 1; o > 0; o >>= 1) M = fmax(M, __shfl_xor_sync(0xffffffffu, M, o, gw));
    double tot = z_sum > 0.0 ? z_sum * exp(m - M) : 0.0;
    for (int o = gw >> 1; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o, gw);
    if (!live) return;
    // pass 2: the row, every column of the plan written once (coalesced across the group)
    T *row = gamma + t * S;
#pragma unroll
    for (int j = 0; j < kInitCache; ++j) {
        const int64_t s = sub + (int64_t)j * gw;
        if (s < S) row[s] = (T)(s < K ? exp(zc[j] - M) / tot : 0.0);
    }
    for (int64_t s = sub + (int64_t)kInitCache * gw; s < S; s += gw)
        row[s] = (T)(s < K ? exp(init_logit(turn_off, turn_lo, turn_hi, turn_cum, k0 + s, lo, hi, sm) - M) / tot : 0.0);
}

// ---- random initialisation (DESIGN.md section 5.22) -------------------------------------------------------------------
// Recording b with N_b live states, x-vector t of it (index inside the recording), state block j = s / 4:
//     (w_0 .. w_3) = Philox4x64-10(counter (t, j, rec_key[b], 0), key (seed[b], 0));  word i belongs to state 4j + i
//     u = ((w >> 11) + 0.5) 2^-53,  e_s = -log u  (a standard exponential),  gamma0[t, s] = e_s / sum_{s' < N_b} e_s'
//     pi0[b, s] = 1 / N_b on the live states; 0 in the padded columns of both
//   init_random_kernel: a group of lanes per x-vector (ceil(S / 4) rounded up to a power of two, at most a warp), lane
//   `sub` owning the blocks sub, sub + gw, ...; the first n_rec * S threads of the grid also write pi0.

constexpr uint64_t kPhiloxM0 = 0xD2E7470EE14C6C93ull, kPhiloxM1 = 0xCA5A826395121157ull;   // Salmon et al. 2011
constexpr uint64_t kPhiloxW0 = 0x9E3779B97F4A7C15ull, kPhiloxW1 = 0xBB67AE8584CAA73Bull;

// Philox4x64-10 (Random123's philox4x64round and key schedule), a pure function of counter and key.
__device__ __forceinline__ void philox4x64(uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3, uint64_t k0, uint64_t k1,
                                           uint64_t w[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += kPhiloxW0;
            k1 += kPhiloxW1;
        }
        const uint64_t hi0 = __umul64hi(kPhiloxM0, c0), lo0 = kPhiloxM0 * c0;
        const uint64_t hi1 = __umul64hi(kPhiloxM1, c2), lo1 = kPhiloxM1 * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
    }
    w[0] = c0;
    w[1] = c1;
    w[2] = c2;
    w[3] = c3;
}

// the four exponentials of block j (0 for the states s >= N)
__device__ __forceinline__ void random_block(int64_t t, int64_t j, uint64_t key, uint64_t seed, int64_t N, double e[4]) {
    uint64_t w[4];
    philox4x64((uint64_t)t, (uint64_t)j, key, 0ull, seed, 0ull, w);
#pragma unroll
    for (int i = 0; i < 4; ++i)
        e[i] = 4 * j + i < N ? -log(((double)(w[i] >> 11) + 0.5) * 0x1p-53) : 0.0;
}

template <typename T>
__device__ __forceinline__ void store_block(T *row, int64_t j, int S, bool vec, const double e[4], double tot) {
    const int64_t s0 = 4 * j;
    if (vec) {                  // S % 4 == 0 and a 16-byte aligned gamma: one (float) or two (double) vector stores
        if constexpr (sizeof(T) == 4) {
            *reinterpret_cast<float4 *>(row + s0) = make_float4((float)(e[0] / tot), (float)(e[1] / tot),
                                                                (float)(e[2] / tot), (float)(e[3] / tot));
        } else {
            reinterpret_cast<double2 *>(row + s0)[0] = make_double2(e[0] / tot, e[1] / tot);
            reinterpret_cast<double2 *>(row + s0)[1] = make_double2(e[2] / tot, e[3] / tot);
        }
        return;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (s0 + i < S) row[s0 + i] = (T)(e[i] / tot);
}

template <typename T>
__global__ void __launch_bounds__(kInitThreads) init_random_kernel(Plan pl, const uint64_t *__restrict__ rec_key,
                                                                   const uint64_t *__restrict__ seed,
                                                                   const int32_t *__restrict__ n_states,
                                                                   T *__restrict__ gamma, T *__restrict__ pi, int gw,
                                                                   bool vec) {
    const int64_t gtid = (int64_t)blockIdx.x * kInitThreads + threadIdx.x;
    const int S = pl.S;
    if (gtid < (int64_t)pl.n_rec * S) {
        const int b = (int)(gtid / S), s = (int)(gtid - (int64_t)b * S);
        const int N = n_states ? min(max(n_states[b], 0), S) : S;
        pi[gtid] = s < N ? (T)(1.0 / (double)N) : (T)0;
    }
    // every lane of the warp takes part in the shuffles, also the lanes past the last x-vector
    const int64_t t = gtid / gw;
    const int sub = threadIdx.x & (gw - 1);
    const bool live = t < pl.n_frames;
    int64_t tl = 0, N = 0;
    uint64_t key = 0, sd = 0;
    if (live) {
        const int b = find_problem(pl.offsets, pl.n_rec, t);
        tl = t - pl.offsets[b];
        N = n_states ? min(max(n_states[b], 0), S) : S;
        key = rec_key[b];
        sd = seed[b];
    }
    const int64_t nblk = (N + 3) >> 2, wblk = (S + 3) >> 2;
    // pass 1: the lane's first block stays in registers (every block of a plan with S <= 128); the lane sums its blocks
    // in order, then the group adds the lane sums by a butterfly.  Lanes without a live block add exact zeros, so the sum,
    // and every bit of the row, depends on N and not on S.
    double e0[4] = {0.0, 0.0, 0.0, 0.0};
    if (sub < nblk) random_block(tl, sub, key, sd, N, e0);
    double tot = (e0[0] + e0[1]) + (e0[2] + e0[3]);
    for (int64_t j = sub + gw; j < nblk; j += gw) {
        double e[4];
        random_block(tl, j, key, sd, N, e);
        tot += (e[0] + e[1]) + (e[2] + e[3]);
    }
    for (int o = gw >> 1; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o, gw);
    if (!live) return;
    // pass 2: the row, every column of the plan written once (coalesced across the group); N = 0 leaves a row of zeros
    if (N == 0) tot = 1.0;
    T *row = gamma + t * S;
    if (sub < wblk) store_block(row, sub, S, vec, e0, tot);
    for (int64_t j = sub + gw; j < wblk; j += gw) {
        double e[4] = {0.0, 0.0, 0.0, 0.0};
        if (j < nblk) random_block(tl, j, key, sd, N, e);
        store_block(row, j, S, vec, e, tot);
    }
}

int launch_init_random(const Plan &pl, const uint64_t *rec_key, const uint64_t *seed, const int32_t *n_states,
                       void *gamma, void *pi, bool f64, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    const int blocks4 = (pl.S + 3) / 4;
    int gw = 1;
    while (gw < 32 && gw < blocks4) gw <<= 1;
    const bool vec = pl.S % 4 == 0 && (reinterpret_cast<uintptr_t>(gamma) & 15) == 0;
    const int64_t threads = max((int64_t)pl.n_frames * gw, (int64_t)pl.n_rec * pl.S);
    const int64_t blocks = (threads + kInitThreads - 1) / kInitThreads;
    if (f64)
        init_random_kernel<double><<<(unsigned)blocks, kInitThreads, 0, st>>>(
            pl, rec_key, seed, n_states, static_cast<double *>(gamma), static_cast<double *>(pi), gw, vec);
    else
        init_random_kernel<float><<<(unsigned)blocks, kInitThreads, 0, st>>>(
            pl, rec_key, seed, n_states, static_cast<float *>(gamma), static_cast<float *>(pi), gw, vec);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_init_turns(const Plan &pl, const int64_t *seg, const int64_t *spk_off, const int64_t *turn_off,
                      const int64_t *turn_lo, const int64_t *turn_hi, const int64_t *turn_cum, const double *smoothing,
                      void *gamma, void *pi, bool f64, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    int gw = 1;
    while (gw < 32 && gw < pl.S) gw <<= 1;
    const int64_t threads = max((int64_t)pl.n_frames * gw, (int64_t)pl.n_rec * pl.S);
    const int64_t blocks = (threads + kInitThreads - 1) / kInitThreads;
    if (f64)
        init_turns_kernel<double><<<(unsigned)blocks, kInitThreads, 0, st>>>(
            pl, seg, spk_off, turn_off, turn_lo, turn_hi, turn_cum, smoothing, static_cast<double *>(gamma),
            static_cast<double *>(pi), gw);
    else
        init_turns_kernel<float><<<(unsigned)blocks, kInitThreads, 0, st>>>(
            pl, seg, spk_off, turn_off, turn_lo, turn_hi, turn_cum, smoothing, static_cast<float *>(gamma),
            static_cast<float *>(pi), gw);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace vbx
