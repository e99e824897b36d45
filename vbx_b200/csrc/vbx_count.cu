// Output step under a speaker-count bound (DESIGN.md section 5.14): keep the `keep[b]` states of recording b with the
// largest posterior mass N_s = sum_t gamma[t,s] and label every frame by its best (and second best) kept state.
//   state_mass_kernel       -> mass [n_rec,S] float64, one CTA per recording
//   hard_labels_keep_kernel -> first / second [N], tiled like hard_labels_kernel over the 64-frame L-tiles
#include "vbx_internal.cuh"

namespace vbx {

constexpr int kMassThreads = 256;
constexpr int kMassPhases = 32;   // frames t = k, k + 32, k + 64, ... make phase k; phases are added in order 0 .. 31

// N_s of every live state, float64.  Job (k, s) sums the frames of phase k of state s sequentially; the 32 phase sums
// are then added in phase order.  The summation order depends on T alone: not on the plan's padded S, the thread
// count or the other recordings of the batch.  Consecutive jobs are consecutive states of one frame (coalesced rows).
__global__ void __launch_bounds__(kMassThreads) state_mass_kernel(Plan pl, const float *__restrict__ gamma,
                                                                  const int32_t *__restrict__ n_states,
                                                                  double *__restrict__ mass) {
    __shared__ double part[kMassPhases][kMaxSWide];
    const int rec = blockIdx.x;
    const int S = pl.S, ns = n_states ? n_states[rec] : S;
    const int64_t f0 = pl.offsets[rec];
    const int64_t T = pl.offsets[rec + 1] - f0;
    for (int j = threadIdx.x; j < kMassPhases * S; j += kMassThreads) {
        const int k = j / S, s = j - k * S;
        double acc = 0.0;
        if (s < ns)
            for (int64_t t = k; t < T; t += kMassPhases) acc += (double)gamma[(f0 + t) * S + s];
        part[k][s] = acc;
    }
    __syncthreads();
    for (int s = threadIdx.x; s < S; s += kMassThreads) {
        double tot = 0.0;
        for (int k = 0; k < kMassPhases; ++k) tot += part[k][s];
        mass[(int64_t)rec * S + s] = tot;
    }
}

// The kept set of the tile's recording is the keep[rec] live states of largest mass (ties: the lower index), as a
// 128-bit mask; then hard_labels_kernel's top-2 scan over the kept states only.  keep >= n_states keeps every live state
// and the scan is hard_labels_kernel's.
__global__ void __launch_bounds__(kLTile) hard_labels_keep_kernel(Plan pl, const float *__restrict__ gamma,
                                                                  const int32_t *__restrict__ n_states,
                                                                  const int32_t *__restrict__ keep,
                                                                  const double *__restrict__ mass,
                                                                  int32_t *__restrict__ first, int32_t *__restrict__ second) {
    __shared__ double m[kMaxSWide];
    __shared__ uint32_t kept[kMaxSWide / 32];
    const int tile = blockIdx.x;
    const int rec = pl.ltile_rec[tile];
    const int64_t f0 = pl.ltile_f0[tile];
    const int len = (int)min((int64_t)kLTile, pl.offsets[rec + 1] - f0);
    const int S = pl.S, ns = n_states ? n_states[rec] : S;
    const int kp = keep[rec];
    for (int s = threadIdx.x; s < ns; s += kLTile) m[s] = mass[(int64_t)rec * S + s];
    if (threadIdx.x < kMaxSWide / 32) kept[threadIdx.x] = 0u;
    __syncthreads();
    for (int s = threadIdx.x; s < ns; s += kLTile) {
        const double v = m[s];
        int rank = 0;   // live states ahead of s: larger mass, or equal mass and a lower index
        for (int j = 0; j < ns; ++j) rank += (m[j] > v) || (m[j] == v && j < s);
        if (rank < kp) atomicOr(&kept[s >> 5], 1u << (s & 31));
    }
    __syncthreads();
    if ((int)threadIdx.x >= len) return;
    const float4 *row = reinterpret_cast<const float4 *>(gamma + (f0 + threadIdx.x) * S);
    float b1 = -INFINITY, b2 = -INFINITY;
    int i1 = -1, i2 = -1;
    for (int q = 0; q < S / 4; ++q) {
        const float4 v = row[q];
        const float x[4] = {v.x, v.y, v.z, v.w};
        const uint32_t word = kept[q >> 3];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int s = 4 * q + e;
            if (s >= ns) break;
            if (!((word >> (s & 31)) & 1u)) continue;
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

int launch_hard_labels_keep(const Plan &pl, const float *gamma, const int32_t *n_states, const int32_t *keep,
                            int32_t *first, int32_t *second, double *mass, cudaStream_t st) {
    if (pl.n_rec == 0) return 0;
    state_mass_kernel<<<pl.n_rec, kMassThreads, 0, st>>>(pl, gamma, n_states, mass);
    if (pl.n_ltiles) hard_labels_keep_kernel<<<pl.n_ltiles, kLTile, 0, st>>>(pl, gamma, n_states, keep, mass, first, second);
    return cudaGetLastError() == cudaSuccess ? (pl.n_ltiles ? 2 : 1) : -1;
}

}  // namespace vbx
