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
// No atomics on floating-point values and no dependence on the rest of the batch: a stream's results are bit-identical
// from run to run, whatever the workspace held and whatever else the push carries.
#include <climits>

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

}  // namespace

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
