// Adaptive symmetric score normalisation against a cohort (DESIGN.md section 5.17).  Every scored speaker x (archive or
// enrolled speakers, with section 5.15's statistics) is scored against the C cohort speakers with section 5.15's LLR,
// and mu_x, sigma_x are the mean and population standard deviation of its K = min(top_k, C) largest cohort scores.
// vbx_cohort_stats_batch (section 5.19) runs G problems against one cohort, each with its c_g (one set of scored
// speakers is the batch of one): the statistics of the scored speakers of all problems and of the cohort once per
// problem, then
//   enroll_score_kernel  (vbx_enroll.cu, through launch_cohort_scores_batch) the [sum M, C] cohort LLRs of every
//                        problem's rectangle in one launch, unchanged
//   cohort_topk_kernel   one CTA per speaker of all problems: the K-th largest score by a radix select on
//                        order-preserving 64-bit keys (8 passes of 8 bits, histograms in shared memory), then mu and
//                        sigma by fixed-order sums (a row's result depends on the row and C alone)
//   norm_scores_kernel   S(x, y) = 1/2 [ (LLR - mu_x) / sigma_x + (LLR - mu_y) / sigma_y ] in place over the link
//                        distances (d = -S; the diagonal and the cannot-link entries untouched) or the enrolment LLRs,
//                        every problem with its own statistics (NormProblems), for vbx_link_batch and vbx_enroll_batch
#include <algorithm>
#include <cstring>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kTopThreads = 256;
constexpr int kTopWarps = kTopThreads / 32;
constexpr int64_t kNormGrid = 1 << 20;     // CTAs of norm_scores_kernel at most; beyond that they stride

// Sum over the CTA: a fixed butterfly in every warp, then the warps in order (the same bits on every run).
__device__ __forceinline__ double block_sum(double v, double *red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int q = 0; q < kTopWarps; ++q) t += red[q];
    __syncthreads();                                  // red is rewritten by the next call
    return t;
}

// One CTA per scored speaker (row of scores [M, C]).  Pass p = 0 .. 7 histograms byte 7 - p of the keys that match the
// bytes chosen so far and picks the byte of the K-th largest key from the top; after 8 passes `prefix` is that key and
// `k` the rank of the K-th value among its tied copies, so the K largest are the values above it plus k copies of it.
// Every thread sums its strided values in increasing column order and block_sum adds the threads in a fixed order, so
// the result depends on C and the row alone (not on M, the chunk or the launch).
__global__ void __launch_bounds__(kTopThreads) cohort_topk_kernel(const double *__restrict__ scores, int64_t C,
                                                                  int64_t K, double *__restrict__ mean_out,
                                                                  double *__restrict__ std_out) {
    __shared__ unsigned int hist[256];
    __shared__ double red[kTopWarps];
    __shared__ unsigned long long s_prefix;
    __shared__ long long s_k;
    const double *v = scores + (int64_t)blockIdx.x * C;
    unsigned long long prefix = 0, mask = 0;
    long long k = K;
    for (int shift = 56; shift >= 0; shift -= 8) {
        hist[threadIdx.x] = 0u;
        __syncthreads();
        for (int64_t j = threadIdx.x; j < C; j += kTopThreads) {
            const unsigned long long key = order_key(v[j]);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);   // integer counts: order-free
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long above = 0;
            int b = 255;
            for (; b > 0 && above + (long long)hist[b] < k; --b) above += hist[b];
            s_k = k - above;
            s_prefix = prefix | ((unsigned long long)b << shift);
        }
        __syncthreads();
        k = s_k;
        prefix = s_prefix;
        mask |= 255ull << shift;
    }
    const double vk = key_value(prefix);
    double s = 0.0;
    for (int64_t j = threadIdx.x; j < C; j += kTopThreads) {
        const double x = v[j];
        if (order_key(x) > prefix) s += x;
    }
    const double mu = (block_sum(s, red) + (double)k * vk) / (double)K;
    double q = 0.0;
    for (int64_t j = threadIdx.x; j < C; j += kTopThreads) {
        const double x = v[j];
        if (order_key(x) > prefix) q += (x - mu) * (x - mu);
    }
    const double dk = vk - mu;
    const double var = (block_sum(q, red) + (double)k * (dk * dk)) / (double)K;
    if (threadIdx.x == 0) {
        mean_out[blockIdx.x] = mu;
        std_out[blockIdx.x] = sqrt(var);
    }
}

// x [rows, cols] in place: LLR -> S(i, j) with row statistics (mr, sr) and column statistics (mc, sc).  link = 1: x holds
// distances d = -LLR, written back as -S, and the diagonal and the entries equal to `skip` (cannot-link) stay as they
// are.  S is 1/2 (a_i + a_j) with a_i = (LLR - mu_i) / sigma_i: the sum commutes, so d[i][j] and d[j][i] stay the same
// number.  copy_out (optional) receives the result.  Every element takes the statistics of its own problem (q,
// section 5.19), so problem g's entries are those of a call on g alone.  kMode: 1 the rectangle of the problems' rows,
// 2 their square blocks.
template <int kMode>
__global__ void __launch_bounds__(256) norm_scores_kernel(double *__restrict__ x, int64_t rows, int64_t cols,
                                                          const double *__restrict__ mr, const double *__restrict__ sr,
                                                          const double *__restrict__ mc, const double *__restrict__ sc,
                                                          int link, double skip, double *__restrict__ copy_out,
                                                          NormProblems q) {
    const int64_t n = rows * cols, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        int64_t i, j, ri, cj;                             // local row and column; indices of their statistics
        double *xt = x + t;
        if (kMode == 2) {                                 // square blocks: problem g's M x M block
            const int g = find_problem(q.blk, q.G, t);
            const int64_t base = q.off[g], M = q.off[g + 1] - base, lt = t - q.blk[g];
            i = lt / M;
            j = lt - i * M;
            ri = base + i;
            cj = base + j;
            xt = reinterpret_cast<double *>(reinterpret_cast<uint8_t *>(x) + q.x_bytes[g]) + lt;
        } else {                                          // rectangle: rows of every problem against its own columns
            i = ri = t / cols;
            j = t - i * cols;
            cj = (int64_t)find_problem(q.off, q.G, i) * cols + j;
        }
        double d = *xt;
        if (!link || (i != j && d != skip)) {
            const double l = link ? -d : d;
            const double s = as_norm(l, mr, sr, ri, mc, sc, cj);
            d = link ? -s : s;
            *xt = d;
        }
        if (copy_out) copy_out[t] = d;
    }
}

}  // namespace

int launch_norm_scores(double *x, int64_t rows, int64_t cols, const double *mean_r, const double *std_r,
                       const double *mean_c, const double *std_c, bool link, double skip, double *copy_out,
                       cudaStream_t st, const NormProblems &q) {
    const int64_t n = rows * cols;
    if (n == 0) return 0;
    const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, kNormGrid);
    if (q.blk)
        norm_scores_kernel<2><<<grid, 256, 0, st>>>(x, rows, cols, mean_r, std_r, mean_c, std_c, link ? 1 : 0, skip,
                                                    copy_out, q);
    else
        norm_scores_kernel<1><<<grid, 256, 0, st>>>(x, rows, cols, mean_r, std_r, mean_c, std_c, link ? 1 : 0, skip,
                                                    copy_out, q);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

namespace {

// vbx_cohort_stats_batch: the scored speakers of every problem [sum M], the cohort speakers once per problem [G C] with
// their index [G, N_c], the scores [sum M, C] and the problem arrays off, coff (g C), tile_off [G+1] and c [G]
struct CohortBatchWs {
    SpeakerStats a, co;
    int32_t *cspk;
    double *scores;
    int64_t *arrays;
};

CohortBatchWs cohort_batch_layout(uint8_t *ws, int64_t G, int64_t M, int64_t C, int64_t N_c, size_t *total) {
    CohortBatchWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.a = take_stats(take, M);
    w.co = take_stats(take, G * C);
    w.cspk = reinterpret_cast<int32_t *>(take((size_t)G * N_c * 4));
    w.scores = reinterpret_cast<double *>(take((size_t)M * C * 8));
    w.arrays = reinterpret_cast<int64_t *>(take((size_t)(4 * G + 3) * 8));
    if (total) *total = o;
    return w;
}

}  // namespace

size_t cohort_batch_workspace_bytes(int G, const int64_t *M_host, int64_t C, int64_t N_c) {
    int64_t M = 0;
    for (int g = 0; g < G; ++g) M += M_host[g];
    size_t total = 0;
    cohort_batch_layout(nullptr, G, M, C, N_c, &total);
    return total;
}

int launch_cohort_batch(const float *fea, const float *Phi, int64_t N, int R, const int32_t *spk, int G,
                        const int64_t *M_host, const float *cohort_fea, int64_t N_c, const int32_t *cohort_spk,
                        int64_t C, const double *c_host, int64_t top_k, void *workspace, double *mean_out,
                        double *std_out, double *scores_out, cudaStream_t st) {
    std::vector<int64_t> host(4 * (size_t)G + 3, 0);       // off, coff, tile_off [G+1], c [G]: one copy
    int64_t *off = host.data(), *coff = off + (G + 1), *tile = coff + (G + 1);
    for (int g = 0; g < G; ++g) {
        off[g + 1] = off[g] + M_host[g];
        coff[g + 1] = coff[g] + C;
        tile[g + 1] = tile[g] + rect_tiles(M_host[g], C);
    }
    std::memcpy(tile + (G + 1), c_host, (size_t)G * sizeof(double));
    const int64_t M = off[G];
    if (M == 0) return 0;
    const CohortBatchWs w = cohort_batch_layout(reinterpret_cast<uint8_t *>(workspace), G, M, C, N_c, nullptr);
    if (cudaMemcpyAsync(w.arrays, host.data(), host.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st) !=
        cudaSuccess)
        return -1;
    const int64_t *d_off = w.arrays, *d_coff = d_off + (G + 1), *d_tile = d_coff + (G + 1);
    const double *d_c = reinterpret_cast<const double *>(d_tile + (G + 1));
    const int lr = launch_repeat_index(cohort_spk, N_c, G, w.cspk, st);
    const int la = launch_speaker_stats_batch(fea, Phi, spk, N, R, G, d_off, d_c, M, w.a, nullptr, nullptr, st);
    const int lc = launch_speaker_stats_batch(cohort_fea, Phi, w.cspk, N_c, R, G, d_coff, d_c, (int64_t)G * C, w.co,
                                              nullptr, nullptr, st);
    const int ls = launch_cohort_scores_batch(w.a, w.co, Phi, G, d_off, d_tile, d_c, tile[G], C, R, w.scores,
                                              scores_out, st);
    if (lr < 0 || la < 0 || lc < 0 || ls < 0) return -1;
    cohort_topk_kernel<<<(unsigned)M, kTopThreads, 0, st>>>(w.scores, C, std::min(top_k, C), mean_out, std_out);
    return cudaGetLastError() == cudaSuccess ? lr + la + lc + ls + 1 : -1;
}

}  // namespace vbx
