// Streaming diarization (include/vbx_b200.h vbx_stream_window / vbx_stream_commit, DESIGN.md section 5.25): the window
// of a push built from each stream's device-resident state, and the push's result folded back into that state.
//
// A stream's state is a ring of its last min(C, count) projected x-vectors and their final labels, the number K of its
// speakers, and the history statistics n_hist[k], F_hist[k] of the x-vectors that have left the ring, by final label.
//
//   stream_window_kernel  one CTA per pushed stream: [context rows; block rows] into the packed window, the soft initial
//                         responsibilities and the uniform pi over the K + c states, and the history as the priors of the
//                         first K states
//   stream_commit_kernel  one CTA per pushed stream: fresh states renumbered in order of their first block row, the
//                         block's final labels, the evicted rows added to the history in time order (one thread per
//                         feature, so every F_hist element is one sequential float64 sum), then the ring advanced
//
// Enrolled speakers in streams (vbx_stream_enroll, DESIGN.md section 5.29), after a push's commit:
//   stream_enroll_stats_kernel  one CTA per stream with candidates (its unnamed speakers that hold rows of the push):
//                               their whole-stream n, F (history plus ring, the ring read once) and b, e; then one CTA
//                               per enrolled speaker for its b, e
//   enroll_score_kernel         (vbx_enroll.cu) the candidates x enrolled LLRs, through launch_cohort_scores_batch
//   stream_enroll_mask_kernel   -inf for the enrolled speakers a stream has already claimed
//   enroll_assign_kernel        (vbx_enroll.cu) one-to-one per stream at the threshold, through launch_enroll_assign
//   stream_enroll_apply_kernel  the names into the per-slot enrolment state and, with the prior, n_e, F_e into the history
//
// No atomics on floating-point values and no dependence on the rest of the batch: a stream's results are bit-identical
// from run to run, whatever the workspace held and whatever else the push carries.
#include <algorithm>
#include <climits>
#include <cstring>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kThreads = 128;
constexpr int kMaxStates = 128;           // S_max and the tier's S are at most the float32 kernels' 128 states

__global__ void __launch_bounds__(kThreads) stream_window_kernel(
    int C, int R, int S_max, int S, const int32_t *__restrict__ slot, const int64_t *__restrict__ blk_off,
    const int64_t *__restrict__ win_off, const int32_t *__restrict__ blk_lab, const int32_t *__restrict__ n_clusters,
    const float *__restrict__ blk_fea, double smoothing, const float *__restrict__ ctx_fea,
    const int32_t *__restrict__ ctx_lab, const int64_t *__restrict__ count, const int32_t *__restrict__ K,
    const double *__restrict__ n_hist, const double *__restrict__ F_hist, float *__restrict__ fea_out,
    float *__restrict__ gamma_out, float *__restrict__ pi_out, int32_t *__restrict__ n_states_out,
    double *__restrict__ prior_n_out, double *__restrict__ prior_F_out) {
    const int i = blockIdx.x;
    const int64_t s = slot[i], cnt = count[s];
    const int64_t L = cnt < C ? cnt : C;
    const int64_t oldest = C > 0 ? (cnt - L) % C : 0;
    const int k0 = K[s], c = n_clusters[i], ns = k0 + c;
    const int64_t b0 = blk_off[i], h = blk_off[i + 1] - b0, w0 = win_off[i], rows = L + h;
    for (int64_t e = threadIdx.x; e < rows * R; e += blockDim.x) {
        const int64_t q = e / R;
        const int r = (int)(e - q * R);
        fea_out[(w0 + q) * R + r] = q < L ? ctx_fea[(s * C + (oldest + q) % C) * R + r] : blk_fea[(b0 + q - L) * R + r];
    }
    // softmax(smoothing * onehot) over ns states, evaluated in float64 and rounded once; a block row without a cluster
    // of its own (c = 0, the stream is at S_max speakers) starts uniform over the known states
    const double ex = exp(-smoothing), den = 1.0 + (ns - 1) * ex;
    const float hot = (float)(1.0 / den), cold = (float)(ex / den), uni = (float)(1.0 / ns);
    for (int64_t e = threadIdx.x; e < rows * S; e += blockDim.x) {
        const int64_t q = e / S;
        const int k = (int)(e - q * S);
        const int lab = q < L ? ctx_lab[s * C + (oldest + q) % C] : (c > 0 ? k0 + blk_lab[b0 + q - L] : -1);
        gamma_out[(w0 + q) * S + k] = k >= ns ? 0.f : lab < 0 ? uni : k == lab ? hot : cold;
    }
    for (int k = threadIdx.x; k < S; k += blockDim.x) {
        pi_out[(int64_t)i * S + k] = k < ns ? uni : 0.f;
        prior_n_out[(int64_t)i * S + k] = k < k0 ? n_hist[s * S_max + k] : 0.0;
    }
    for (int64_t e = threadIdx.x; e < (int64_t)S * R; e += blockDim.x) {
        const int k = (int)(e / R);
        prior_F_out[(int64_t)i * S * R + e] = k < k0 ? F_hist[(s * S_max + k) * R + (e - (int64_t)k * R)] : 0.0;
    }
    if (threadIdx.x == 0) n_states_out[i] = ns;
}

__global__ void __launch_bounds__(kThreads) stream_commit_kernel(
    int C, int R, int S_max, const int32_t *__restrict__ slot, const int64_t *__restrict__ blk_off,
    const int64_t *__restrict__ win_off, const float *__restrict__ blk_fea, const int32_t *__restrict__ first,
    float *__restrict__ ctx_fea, int32_t *__restrict__ ctx_lab, int64_t *__restrict__ count, int32_t *__restrict__ K,
    double *__restrict__ n_hist, double *__restrict__ F_hist, int32_t *__restrict__ labels_out) {
    __shared__ int first_row[kMaxStates];
    __shared__ int new_id[kMaxStates];
    const int i = blockIdx.x;
    const int64_t s = slot[i], cnt = count[s];
    const int64_t L = cnt < C ? cnt : C;
    const int k0 = K[s];
    const int64_t b0 = blk_off[i], h = blk_off[i + 1] - b0, w0 = win_off[i] + L;
    for (int k = threadIdx.x; k < kMaxStates; k += blockDim.x) first_row[k] = INT_MAX;
    __syncthreads();
    for (int64_t t = threadIdx.x; t < h; t += blockDim.x) {
        const int w = first[w0 + t];
        if (w >= k0 && w < kMaxStates) atomicMin(&first_row[w], (int)t);     // an integer minimum: order-free
    }
    __syncthreads();
    // fresh states that hold block rows become speakers k0, k0 + 1, ... in order of their first row
    int fresh = 0;
#pragma unroll 1
    for (int k = k0; k < kMaxStates; ++k) fresh += first_row[k] != INT_MAX;
    for (int k = threadIdx.x; k < kMaxStates; k += blockDim.x) {
        int rank = 0;
        if (k >= k0 && first_row[k] != INT_MAX)
#pragma unroll 1
            for (int j = k0; j < kMaxStates; ++j) rank += first_row[j] < first_row[k];
        new_id[k] = k0 + rank;
    }
    __syncthreads();
    for (int64_t t = threadIdx.x; t < h; t += blockDim.x) {
        const int w = first[w0 + t];
        labels_out[b0 + t] = w < k0 ? w : new_id[w < kMaxStates ? w : 0];
    }
    __syncthreads();                                       // labels_out is read back below by other threads of the CTA
    // rows leaving the ring, oldest first: the old ring's [cnt - L, cnt - L + n_old), then the block's own rows that do
    // not fit ([cnt, e1) when h > C)
    const int64_t cnt2 = cnt + h, keep = cnt2 < C ? cnt2 : C, e0 = cnt - L, e1 = cnt2 - keep;
    for (int r = threadIdx.x; r < R; r += blockDim.x)
#pragma unroll 1
        for (int64_t g = e0; g < e1; ++g) {
            const bool old = g < cnt;
            const int lab = old ? ctx_lab[s * C + g % C] : labels_out[b0 + g - cnt];
            const float v = old ? ctx_fea[(s * C + g % C) * R + r] : blk_fea[(b0 + g - cnt) * R + r];
            if (lab >= 0 && lab < S_max) F_hist[(s * S_max + lab) * R + r] += (double)v;
        }
    if (threadIdx.x == 0)
#pragma unroll 1
        for (int64_t g = e0; g < e1; ++g) {
            const int lab = g < cnt ? ctx_lab[s * C + g % C] : labels_out[b0 + g - cnt];
            if (lab >= 0 && lab < S_max) n_hist[s * S_max + lab] += 1.0;
        }
    __syncthreads();                                       // the evicted ring rows are read before they are overwritten
    const int64_t g0 = cnt > e1 ? cnt : e1;
    for (int64_t e = threadIdx.x; e < (cnt2 - g0) * R; e += blockDim.x) {
        const int64_t g = g0 + e / R;
        const int r = (int)(e % R);
        ctx_fea[(s * C + g % C) * R + r] = blk_fea[(b0 + g - cnt) * R + r];
    }
    for (int64_t g = g0 + threadIdx.x; g < cnt2; g += blockDim.x) ctx_lab[s * C + g % C] = labels_out[b0 + g - cnt];
    if (threadIdx.x == 0) {
        count[s] = cnt2;
        K[s] = k0 + fresh;
    }
}

// ---- enrolled speakers in streams (DESIGN.md section 5.29) ---------------------------------------------------------
constexpr int kEnrollThreads = 256;       // one thread per feature (R <= 128), the e reduction of link_stats_kernel
constexpr int kEnrollRows = kEnrollThreads;

// The problem arrays of one vbx_stream_enroll call, uploaded in one copy: cand_off [n+1], slot [n], cand_k [M] (the
// candidates of stream i are speakers cand_k[cand_off[i] .. cand_off[i+1]-1] of slot slot[i]), the score problem
// off = {0, M} and tile_off = {0, tiles}, then c and the threshold as doubles.
struct EnrollArrays {
    const int64_t *cand_off, *slot, *cand_k, *off, *tile_off;
    const double *c, *threshold;
};

// The e of one speaker from each thread's term of feature r = threadIdx.x (0 for r >= R): the butterfly of each warp,
// then the warps in order, as link_stats_kernel sums it.  Thread 0 gets the result.
__device__ __forceinline__ double block_e_sum(double e, double *red) {
    for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
    __syncthreads();
    double tot = 0.0;
    if (threadIdx.x == 0)
        for (int q = 0; q < kEnrollThreads / 32; ++q) tot += red[q];
    __syncthreads();                                       // red is rewritten by the next speaker
    return tot;
}

// CTAs 0 .. n-1: stream i's candidates.  Each candidate's n and F start from n_hist, F_hist of its speaker; the ring's
// rows, oldest first, are then added to the candidate that holds their label (one thread per feature, so every F is
// one sequential float64 sum; rows of other speakers are not read).  CTAs n .. n+E-1: enrolled speaker j's b and e from
// n_enroll, F_enroll.  Both write b, e and n with speaker_L_b, speaker_e_term and link_stats_kernel's reduction.
__global__ void __launch_bounds__(kEnrollThreads) stream_enroll_stats_kernel(
    int n, int C, int R, int S_max, EnrollArrays a, const float *__restrict__ Phi, const float *__restrict__ ctx_fea,
    const int32_t *__restrict__ ctx_lab, const int64_t *__restrict__ count, const double *__restrict__ n_hist,
    const double *__restrict__ F_hist, const double *__restrict__ n_enroll, const double *__restrict__ F_enroll,
    SpeakerStats cand, SpeakerStats en, double *__restrict__ n_out, double *__restrict__ F_out) {
    extern __shared__ double acc[];                        // [candidates of the stream][R]
    __shared__ double cnt[kMaxStates];
    __shared__ double red[kEnrollThreads / 32];
    __shared__ int col[kMaxStates];                        // the candidate index of each speaker, -1 for none
    __shared__ int row_col[kEnrollRows];
    __shared__ int64_t row_pos[kEnrollRows];
    const int tid = threadIdx.x;
    const double c = *a.c;
    if ((int)blockIdx.x >= n) {
        const int64_t j = blockIdx.x - n;
        const double nj = n_enroll[j];
        double e = 0.0;
        if (tid < R) {
            double L, b;
            speaker_L_b(c, nj, (double)Phi[tid], F_enroll[j * R + tid], L, b);
            en.b[j * kMaxR + tid] = b;
            e = speaker_e_term(L, b);
        }
        const double tot = block_e_sum(e, red);
        if (tid == 0) {
            en.e[j] = tot;
            en.n[j] = nj;
        }
        return;
    }
    const int i = blockIdx.x;
    const int64_t s = a.slot[i], m0 = a.cand_off[i], nk = a.cand_off[i + 1] - m0;
    for (int k = tid; k < kMaxStates; k += kEnrollThreads) col[k] = -1;
    __syncthreads();
    for (int64_t q = tid; q < nk; q += kEnrollThreads) {
        const int64_t k = a.cand_k[m0 + q];
        col[k] = (int)q;
        cnt[q] = n_hist[s * S_max + k];
    }
    for (int64_t e = tid; e < nk * R; e += kEnrollThreads) {
        const int64_t q = e / R;
        acc[e] = F_hist[(s * S_max + a.cand_k[m0 + q]) * R + (e - q * R)];
    }
    const int64_t cnt_s = count[s], L = cnt_s < C ? cnt_s : C, oldest = C > 0 ? (cnt_s - L) % C : 0;
    for (int64_t q0 = 0; q0 < L; q0 += kEnrollRows) {
        const int rows = (int)(L - q0 < kEnrollRows ? L - q0 : kEnrollRows);
        __syncthreads();                                   // col / acc set up, or the previous chunk's rows consumed
        if (tid < rows) {
            const int64_t pos = (oldest + q0 + tid) % C;
            const int lab = ctx_lab[s * C + pos];
            row_col[tid] = lab >= 0 && lab < kMaxStates ? col[lab] : -1;
            row_pos[tid] = s * C + pos;
        }
        __syncthreads();
        if (tid < R)
#pragma unroll 1
            for (int q = 0; q < rows; ++q) {
                const int j = row_col[q];
                if (j < 0) continue;
                acc[j * R + tid] += (double)ctx_fea[row_pos[q] * R + tid];
                if (tid == 0) cnt[j] += 1.0;
            }
    }
    __syncthreads();
#pragma unroll 1
    for (int64_t q = 0; q < nk; ++q) {
        const int64_t m = m0 + q;
        const double nq = cnt[q];
        double e = 0.0;
        if (tid < R) {
            const double F = acc[q * R + tid];
            double L, b;
            speaker_L_b(c, nq, (double)Phi[tid], F, L, b);
            cand.b[m * kMaxR + tid] = b;
            if (F_out) F_out[m * R + tid] = F;
            e = speaker_e_term(L, b);
        }
        const double tot = block_e_sum(e, red);
        if (tid == 0) {
            cand.e[m] = tot;
            cand.n[m] = nq;
            if (n_out) n_out[m] = nq;
        }
    }
}

// The enrolled speakers already claimed by a stream score -inf against its candidates.
__global__ void __launch_bounds__(kThreads) stream_enroll_mask_kernel(int S_max, int64_t E, EnrollArrays a,
                                                                       const int32_t *__restrict__ named,
                                                                       double *__restrict__ llr) {
    const int i = blockIdx.x;
    const int64_t s = a.slot[i], m0 = a.cand_off[i], nk = a.cand_off[i + 1] - m0;
    for (int64_t e = threadIdx.x; e < nk * S_max; e += blockDim.x) {
        const int64_t q = e / S_max;
        const int32_t x = named[s * S_max + (e - q * S_max)];
        if (x >= 0 && x < E) llr[(m0 + q) * E + x] = -INFINITY;
    }
}

// A candidate assigned to enrolled speaker x takes the name (named = x) and, with the prior, x's statistics join the
// speaker's history.  Every (slot, speaker) belongs to one candidate: no two threads write one element.
__global__ void __launch_bounds__(kThreads) stream_enroll_apply_kernel(int R, int S_max, int prior, EnrollArrays a,
                                                                        const int32_t *__restrict__ assign,
                                                                        const double *__restrict__ n_enroll,
                                                                        const double *__restrict__ F_enroll,
                                                                        int32_t *__restrict__ named,
                                                                        double *__restrict__ n_hist,
                                                                        double *__restrict__ F_hist) {
    const int i = blockIdx.x;
    const int64_t s = a.slot[i], m0 = a.cand_off[i], nk = a.cand_off[i + 1] - m0;
    for (int64_t q = threadIdx.x; q < nk; q += blockDim.x) {
        const int32_t x = assign[m0 + q];
        if (x < 0) continue;
        const int64_t k = a.cand_k[m0 + q];
        named[s * S_max + k] = x;
        if (prior) n_hist[s * S_max + k] += n_enroll[x];
    }
    if (!prior) return;
    for (int64_t e = threadIdx.x; e < nk * R; e += blockDim.x) {
        const int64_t q = e / R;
        const int32_t x = assign[m0 + q];
        if (x >= 0) F_hist[(s * S_max + a.cand_k[m0 + q]) * R + (e - q * R)] += F_enroll[(int64_t)x * R + (e - q * R)];
    }
}

struct StreamEnrollWs {
    int64_t *arrays;
    SpeakerStats cand, en;
    double *llr;
    uint8_t *slices;
};

StreamEnrollWs stream_enroll_layout(uint8_t *ws, int n, int64_t M, int64_t E, int64_t max_k, int sms, size_t *total) {
    StreamEnrollWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.arrays = reinterpret_cast<int64_t *>(take((size_t)(2 * n + M + 7) * 8));
    w.cand = take_stats(take, M);
    w.en = take_stats(take, E);
    w.llr = reinterpret_cast<double *>(take((size_t)M * E * 8));
    w.slices = take(enroll_assign_workspace_bytes(E, max_k, n, sms));
    if (total) *total = o;
    return w;
}

}  // namespace

size_t stream_enroll_workspace_bytes(int n, int64_t M, int64_t E, int64_t max_k, int sms) {
    size_t total = 0;
    stream_enroll_layout(nullptr, n, M, E, max_k, sms, &total);
    return total;
}

int launch_stream_enroll(int n, int C, int R, int S_max, const int32_t *slot_host, const int64_t *cand_off_host,
                         const int32_t *cand_k_host, const float *Phi, double c, const float *ctx_fea,
                         const int32_t *ctx_lab, const int64_t *count, double *n_hist, double *F_hist, int32_t *named,
                         const double *n_enroll, const double *F_enroll, int64_t E, double threshold, int prior,
                         void *workspace, int sms, int32_t *assign_out, double *best_llr_out, double *llr_out,
                         double *n_out, double *F_out, cudaStream_t st) {
    if (n == 0) return 0;
    const int64_t M = cand_off_host[n];
    int64_t max_k = 0;
    for (int i = 0; i < n; ++i) max_k = std::max<int64_t>(max_k, cand_off_host[i + 1] - cand_off_host[i]);
    const StreamEnrollWs w = stream_enroll_layout(reinterpret_cast<uint8_t *>(workspace), n, M, E, max_k, sms, nullptr);
    std::vector<int64_t> host((size_t)(2 * n + M + 7));
    int64_t *p = host.data();
    std::copy(cand_off_host, cand_off_host + n + 1, p);
    std::copy(slot_host, slot_host + n, p + n + 1);
    std::copy(cand_k_host, cand_k_host + M, p + 2 * n + 1);
    int64_t *tail = p + 2 * n + 1 + M;
    tail[0] = 0;
    tail[1] = M;
    tail[2] = 0;
    tail[3] = rect_tiles(M, E);
    std::memcpy(tail + 4, &c, sizeof(double));
    std::memcpy(tail + 5, &threshold, sizeof(double));
    if (cudaMemcpyAsync(w.arrays, host.data(), host.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return -1;
    const int64_t *d = w.arrays;
    const EnrollArrays a{d, d + n + 1, d + 2 * n + 1, d + 2 * n + 1 + M, d + 2 * n + 3 + M,
                         reinterpret_cast<const double *>(d + 2 * n + 5 + M),
                         reinterpret_cast<const double *>(d + 2 * n + 6 + M)};
    const int smem = (int)(max_k * R * sizeof(double));
    if (!allow_dynamic_smem(stream_enroll_stats_kernel, smem)) return -1;
    stream_enroll_stats_kernel<<<(unsigned)(n + E), kEnrollThreads, smem, st>>>(
        n, C, R, S_max, a, Phi, ctx_fea, ctx_lab, count, n_hist, F_hist, n_enroll, F_enroll, w.cand, w.en, n_out, F_out);
    if (cudaGetLastError() != cudaSuccess) return -1;
    const int ls = launch_cohort_scores_batch(w.cand, w.en, Phi, 1, a.off, a.tile_off, a.c, tail[3], E, R, w.llr,
                                              llr_out, st);
    if (ls < 0) return -1;
    stream_enroll_mask_kernel<<<(unsigned)n, kThreads, 0, st>>>(S_max, E, a, named, w.llr);
    const int la = launch_enroll_assign(w.llr, a.cand_off, n, E, max_k, a.threshold, w.slices, sms, assign_out,
                                        best_llr_out, st);
    if (la < 0) return -1;
    stream_enroll_apply_kernel<<<(unsigned)n, kThreads, 0, st>>>(R, S_max, prior, a, assign_out, n_enroll, F_enroll,
                                                                 named, n_hist, F_hist);
    return cudaGetLastError() == cudaSuccess ? 3 + ls + la : -1;
}

int launch_stream_window(int n, int C, int R, int S_max, int S, const int32_t *slot, const int64_t *blk_off,
                         const int64_t *win_off, const int32_t *blk_lab, const int32_t *n_clusters, const float *blk_fea,
                         double smoothing, const float *ctx_fea, const int32_t *ctx_lab, const int64_t *count,
                         const int32_t *K, const double *n_hist, const double *F_hist, float *fea_out, float *gamma_out,
                         float *pi_out, int32_t *n_states_out, double *prior_n_out, double *prior_F_out,
                         cudaStream_t st) {
    if (n == 0) return 0;
    stream_window_kernel<<<n, kThreads, 0, st>>>(C, R, S_max, S, slot, blk_off, win_off, blk_lab, n_clusters, blk_fea,
                                                 smoothing, ctx_fea, ctx_lab, count, K, n_hist, F_hist, fea_out,
                                                 gamma_out, pi_out, n_states_out, prior_n_out, prior_F_out);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_stream_commit(int n, int C, int R, int S_max, const int32_t *slot, const int64_t *blk_off,
                         const int64_t *win_off, const float *blk_fea, const int32_t *first, float *ctx_fea,
                         int32_t *ctx_lab, int64_t *count, int32_t *K, double *n_hist, double *F_hist,
                         int32_t *labels_out, cudaStream_t st) {
    if (n == 0) return 0;
    stream_commit_kernel<<<n, kThreads, 0, st>>>(C, R, S_max, slot, blk_off, win_off, blk_fea, first, ctx_fea, ctx_lab,
                                                 count, K, n_hist, F_hist, labels_out);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace vbx
