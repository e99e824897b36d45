// Combination of K diarizations of the same intervals by label mapping and weighted voting (include/vbx_b200.h
// vbx_combine, DESIGN.md section 5.21; DOVER, Stolcke and Yoshioka 2019, with a second label per interval).
//
//   combine_overlap_kernel  one CTA per (recording, unordered pair a < b of hypotheses): O_ab[s, u], the ticks in which
//                           a says s and b says u, in either stream; K more CTAs per recording sum L_a[s], the ticks in
//                           which a says s, and flag a's bad labels.  64-bit integer atomics, in shared memory where the
//                           max_labels x max_labels block fits and in place otherwise, as score_kernel chooses.
//   combine_map_kernel      one CTA per recording: the K (K - 1) / 2 matching totals (one warp per pair), D, the order,
//                           the weights, and the K - 1 sequential assignments against the global labels (warp 0).
//   combine_vote_kernel     one thread per interval of the packed batch: the weighted count vote and the label tallies.
//
// The assignments are shortest augmenting paths (Jonker-Volgenant, the method of scipy's linear_sum_assignment) run by
// one warp: rows are at most 128 labels, so a lane owns the columns j = lane (mod 32) and a Dijkstra step is a strided
// scan and five shuffles, with no CTA barrier.  vbx_enroll.cu's routine is CTA-wide over E + K columns with its state in
// the workspace and its costs read from an LLR row against a threshold; sharing it would put a branch on the caller
// into every step, so this file keeps its own (DESIGN.md section 5.21).  Costs are minus tick counts held in float64:
// every cost, dual and path length is an integer far below 2^53, so the arithmetic is exact.
#include <climits>
#include <cmath>

#include "../../include/vbx_b200.h"
#include "vbx_internal.cuh"

namespace vbx {
namespace {

constexpr int kMaxK = 32;                        // hypotheses
constexpr int kMaxLabels = 128;                  // labels of one hypothesis in one recording
constexpr int kMaxGlobal = 255;                  // global labels of one recording
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCols = 384;                       // kMaxGlobal + kMaxLabels "unmatched" columns, rounded up to 32
constexpr int64_t kSmemCells = 64 * 128;         // 64 KB of int64, the shared block of score_kernel

__host__ __device__ inline int64_t n_pairs(int K) { return (int64_t)K * (K - 1) / 2; }
__host__ __device__ inline int pair_index(int a, int b, int K) { return a * (2 * K - a - 1) / 2 + (b - a - 1); }   // a < b
__host__ __device__ inline int global_stride(int K, int ML) { return K * ML < kMaxGlobal ? K * ML : kMaxGlobal; }

struct CombineWs {
    int32_t *n_labels;     // [n_rec, K]
    int64_t *O, *L;        // [n_rec, P, ML, ML], [n_rec, K, ML] (unused when the caller gives O_out / L_out)
    int64_t *C;            // [n_rec, ML, global_stride]: the cost block of the assignment being solved
    double *w;             // [kMaxK]: hypothesis k's weight, or rank r + 1's default weight
};

CombineWs combine_layout(uint8_t *ws, int64_t n_rec, int K, int ML, size_t *total) {
    CombineWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.n_labels = reinterpret_cast<int32_t *>(take((size_t)n_rec * K * 4));
    w.O = reinterpret_cast<int64_t *>(take((size_t)n_rec * n_pairs(K) * ML * ML * 8));
    w.L = reinterpret_cast<int64_t *>(take((size_t)n_rec * K * ML * 8));
    w.C = reinterpret_cast<int64_t *>(take((size_t)n_rec * ML * global_stride(K, ML) * 8));
    w.w = reinterpret_cast<double *>(take(kMaxK * 8));
    if (total) *total = o;
    return w;
}

// the labels hypothesis k gives interval t: s1, s2 in [-1, n) with s2 only beside a different s1; anything else is a
// bad label (both come back -1)
__device__ __forceinline__ bool read_labels(const int32_t *__restrict__ l1, const int32_t *__restrict__ l2, int64_t at,
                                            int n, int &s1, int &s2) {
    s1 = l1[at];
    s2 = l2[at];
    const bool ok = s1 >= -1 && s1 < n && s2 >= -1 && s2 < n && !(s1 < 0 && s2 >= 0) && !(s1 >= 0 && s2 == s1);
    if (!ok) s1 = s2 = -1;
    return ok;
}

__global__ void __launch_bounds__(kThreads) combine_overlap_kernel(
    const int64_t *__restrict__ offsets, const int64_t *__restrict__ lo, const int64_t *__restrict__ hi, int64_t N,
    int K, const int32_t *__restrict__ labels, const int32_t *__restrict__ labels2,
    const int32_t *__restrict__ n_labels, int ML, int shared_block, int64_t *__restrict__ O_out,
    int64_t *__restrict__ L_out, int32_t *__restrict__ flags) {
    extern __shared__ unsigned long long sO[];
    const int P = (int)n_pairs(K);
    const int64_t rec = blockIdx.x / (P + K);
    const int j = (int)(blockIdx.x - rec * (P + K));
    const bool self = j >= P;                     // the label time of hypothesis j - P
    int a = 0, b = 0;
    if (self) {
        a = b = j - P;
    } else {
        int p = j;
        for (; p >= K - 1 - a; ++a) p -= K - 1 - a;
        b = a + 1 + p;
    }
    const int64_t cells = self ? ML : (int64_t)ML * ML;
    unsigned long long *out = reinterpret_cast<unsigned long long *>(self ? L_out + (rec * K + a) * ML
                                                                          : O_out + (rec * P + j) * cells);
    unsigned long long *acc = shared_block ? sO : out;
    for (int64_t i = threadIdx.x; i < cells; i += kThreads) acc[i] = 0ull;
    __syncthreads();
    const int na = n_labels[rec * K + a], nb = n_labels[rec * K + b];
    const int32_t *a1 = labels + (int64_t)a * N, *a2 = labels2 + (int64_t)a * N;
    const int32_t *b1 = labels + (int64_t)b * N, *b2 = labels2 + (int64_t)b * N;
    bool bad = false;
    for (int64_t t = offsets[rec] + threadIdx.x; t < offsets[rec + 1]; t += kThreads) {
        int s[2], u[2];
        const bool ok = read_labels(a1, a2, t, na, s[0], s[1]);
        const int64_t d = hi[t] - lo[t];
        if (self) {
            bad |= !ok;
            if (d <= 0) continue;
            for (int x = 0; x < 2; ++x)
                if (s[x] >= 0) atomicAdd(&acc[s[x]], (unsigned long long)d);
            continue;
        }
        if (d <= 0 || s[0] < 0) continue;
        read_labels(b1, b2, t, nb, u[0], u[1]);
        for (int x = 0; x < 2; ++x)
            for (int y = 0; y < 2; ++y)
                if (s[x] >= 0 && u[y] >= 0) atomicAdd(&acc[s[x] * ML + u[y]], (unsigned long long)d);
    }
    if (bad) atomicOr(&flags[rec], VBX_COMBINE_BAD_LABEL);
    if (shared_block) {
        __syncthreads();
        for (int64_t i = threadIdx.x; i < cells; i += kThreads) out[i] = sO[i];
    }
}

// One warp's assignment state in shared memory: columns up to kCols, rows up to kMaxLabels.
struct WarpLsap {
    double v[kCols], spc[kCols], u[kMaxLabels];       // column duals, shortest path costs; row duals
    int16_t path[kCols], row4col[kCols], col4row[kMaxLabels];
    uint8_t sc[kCols], sr[kMaxLabels];
};

// Minimum-cost assignment of nr rows to nc >= nr columns by one warp; cost(i, j) finite.  Rows are augmented in index
// order, one Dijkstra over the columns each; a step takes the column of smallest path cost, ties to the lowest column.
// On return st.col4row[i] is row i's column.  Duals and augmentation as scipy's rectangular_lsap.
template <class Cost>
__device__ __forceinline__ void warp_lsap(WarpLsap &st, int nr, int nc, Cost cost) {
    const int lane = threadIdx.x & 31;
    for (int j = lane; j < nc; j += 32) {
        st.v[j] = 0.0;
        st.row4col[j] = -1;
    }
    for (int i = lane; i < nr; i += 32) {
        st.u[i] = 0.0;
        st.col4row[i] = -1;
    }
    __syncwarp();
    for (int cur = 0; cur < nr; ++cur) {
        for (int j = lane; j < nc; j += 32) {
            st.spc[j] = INFINITY;
            st.sc[j] = 0;
        }
        for (int i = lane; i < nr; i += 32) st.sr[i] = 0;
        __syncwarp();
        int i = cur, sink = -1;
        double minVal = 0.0;
        while (sink < 0) {
            const double ui = st.u[i];
            double bv = INFINITY;
            int bj = INT_MAX;
            for (int j = lane; j < nc; j += 32) {
                if (st.sc[j]) continue;
                const double r = minVal + cost(i, j) - ui - st.v[j];
                double p = st.spc[j];
                if (r < p) {
                    st.path[j] = (int16_t)i;
                    st.spc[j] = r;
                    p = r;
                }
                if (p < bv) {                          // increasing j: the lowest column on ties
                    bv = p;
                    bj = j;
                }
            }
            for (int o = 16; o; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
                if (ov < bv || (ov == bv && oj < bj)) {
                    bv = ov;
                    bj = oj;
                }
            }
            if (lane == 0) {
                st.sr[i] = 1;
                st.sc[bj] = 1;
            }
            __syncwarp();
            minVal = bv;
            const int r = st.row4col[bj];
            if (r < 0) sink = bj;
            else i = r;
        }
        for (int k = lane; k < nr; k += 32)
            if (st.sr[k] && k != cur) st.u[k] += minVal - st.spc[st.col4row[k]];
        for (int j = lane; j < nc; j += 32)
            if (st.sc[j]) st.v[j] -= minVal - st.spc[j];
        __syncwarp();
        if (lane == 0) {
            st.u[cur] += minVal;
            int j = sink;
            while (true) {
                const int r = st.path[j];
                st.row4col[j] = (int16_t)r;
                const int prev = st.col4row[r];
                st.col4row[r] = (int16_t)j;
                j = prev;
                if (r == cur) break;
            }
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(kThreads) combine_map_kernel(
    int K, const int32_t *__restrict__ n_labels, int ML, const int64_t *O, const int64_t *L, int64_t *C_all,
    const double *__restrict__ w_in, int w_given, int32_t *__restrict__ order_out, double *__restrict__ weights_out, int64_t *D_out, int32_t *map_out,
    int32_t *__restrict__ n_global_out, int32_t *__restrict__ flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpLsap *states = reinterpret_cast<WarpLsap *>(smem_raw);
    __shared__ int s_n[kMaxK], s_order[kMaxK], s_ng, s_over;
    __shared__ long long s_sumL[kMaxK], s_tot[kMaxK];
    const int64_t rec = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int P = (int)n_pairs(K), Gs = global_stride(K, ML);
    const int64_t *Or = O + rec * P * ML * ML, *Lr = L + rec * K * ML;
    int64_t *D = D_out + rec * K * K, *C = C_all + rec * ML * Gs;
    int32_t *map = map_out + rec * K * kMaxLabels;
    if (tid < K) {
        s_n[tid] = n_labels[rec * K + tid];
        long long sum = 0;
        for (int s = 0; s < s_n[tid]; ++s) sum += Lr[tid * ML + s];
        s_sumL[tid] = sum;
        D[tid * K + tid] = 0;
    }
    for (int i = tid; i < K * kMaxLabels; i += kThreads) map[i] = -1;
    __syncthreads();

    // the matching totals m_ab, one warp per pair; the smaller side gives the rows
    WarpLsap &st = states[warp];
    for (int p = warp, a = 0; p < P; p += kWarps) {
        int q = p;
        for (a = 0; q >= K - 1 - a; ++a) q -= K - 1 - a;
        const int b = a + 1 + q, na = s_n[a], nb = s_n[b];
        const int64_t *blk = Or + (int64_t)p * ML * ML;
        long long m = 0;
        if (na > 0 && nb > 0) {
            const bool flip = na > nb;               // rows are b's labels
            const int nr = flip ? nb : na, nc = flip ? na : nb;
            warp_lsap(st, nr, nc, [=](int i, int j) { return -(double)(flip ? blk[j * ML + i] : blk[i * ML + j]); });
            for (int i = lane; i < nr; i += 32) {
                const int j = st.col4row[i];
                m += flip ? blk[j * ML + i] : blk[i * ML + j];
            }
            for (int o = 16; o; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
            __syncwarp();
        }
        if (lane == 0) D[a * K + b] = D[b * K + a] = s_sumL[a] + s_sumL[b] - 2 * m;
    }
    __syncthreads();

    if (tid < K) {                                   // order by summed disagreement, ties to the lower index
        long long tot = 0;
        for (int b = 0; b < K; ++b) tot += D[tid * K + b];
        s_tot[tid] = tot;
    }
    __syncthreads();
    if (tid < K) {
        int r = 0;                                   // the hypotheses that come before this one
        for (int b = 0; b < K; ++b) r += s_tot[b] < s_tot[tid] || (s_tot[b] == s_tot[tid] && b < tid);
        s_order[r] = tid;
        order_out[rec * K + r] = tid;
        weights_out[rec * K + tid] = w_in[w_given ? tid : r];      // by hypothesis, or the default of rank r + 1
    }
    __syncthreads();
    if (tid == 0) {
        const int anchor = s_order[0];
        int ng = 0;                                  // the anchor's labels that have time, in label order
        for (int s = 0; s < s_n[anchor]; ++s)
            if (Lr[anchor * ML + s] > 0) map[anchor * kMaxLabels + s] = ng++;
        s_ng = ng;                                   // at most kMaxLabels here
        s_over = 0;
    }
    __syncthreads();

    for (int r = 1; r < K && !s_over; ++r) {
        const int h = s_order[r], nh = s_n[h], ng = s_ng;
        // C[s, g] = ticks hypothesis h's label s shares with the labels already mapped to g
        for (int i = tid; i < nh * ng; i += kThreads) C[(i / ng) * Gs + i % ng] = 0;
        __syncthreads();
        for (int q = 0; q < r; ++q) {
            const int b = s_order[q], nb = s_n[b];
            const int64_t *blk = Or + (int64_t)(h < b ? pair_index(h, b, K) : pair_index(b, h, K)) * ML * ML;
            for (int i = tid; i < nh * nb; i += kThreads) {
                const int s = i / nb, u = i % nb, g = map[b * kMaxLabels + u];
                const int64_t o = h < b ? blk[s * ML + u] : blk[u * ML + s];
                if (g >= 0 && o > 0) atomicAdd(reinterpret_cast<unsigned long long *>(&C[s * Gs + g]), (unsigned long long)o);
            }
        }
        __syncthreads();
        if (warp == 0 && nh > 0) {
            // columns g < ng are the global labels, the nh columns after them leave a row unmatched at cost 0
            warp_lsap(states[0], nh, ng + nh, [=](int i, int j) { return j < ng ? -(double)__ldcg(&C[i * Gs + j]) : 0.0; });
            if (lane == 0) {
                int next = ng;
                for (int s = 0; s < nh; ++s) {
                    if (Lr[h * ML + s] <= 0) continue;                     // no time: stays -1
                    const int j = states[0].col4row[s];
                    if (j < ng && __ldcg(&C[s * Gs + j]) > 0) map[h * kMaxLabels + s] = j;
                    else if (next < kMaxGlobal) map[h * kMaxLabels + s] = next++;
                    else s_over = 1;
                }
                s_ng = next;
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        n_global_out[rec] = s_over ? 0 : s_ng;
        if (s_over) atomicOr(&flags[rec], VBX_COMBINE_TOO_MANY_LABELS);
    }
}

// The tally of global label g at interval t: the weights of the hypotheses that say it, added in index order.
__device__ __forceinline__ double tally_of(int g, int64_t t, int64_t N, int K, const int32_t *__restrict__ labels,
                                           const int32_t *__restrict__ labels2, const int32_t *__restrict__ nl,
                                           const int32_t *__restrict__ map, const double *__restrict__ w) {
    double sum = 0.0;
    for (int k = 0; k < K; ++k) {
        int s1, s2;
        read_labels(labels + (int64_t)k * N, labels2 + (int64_t)k * N, t, nl[k], s1, s2);
        const bool says = (s1 >= 0 && map[k * kMaxLabels + s1] == g) || (s2 >= 0 && map[k * kMaxLabels + s2] == g);
        if (says) sum += w[k];
    }
    return sum;
}

// One thread per interval.  No candidate list is kept: each label met is looked up in the two best so far and, when it
// is neither, its tally is summed again over the hypotheses (their labels come from L1), so the kernel's state is two
// (global id, tally) pairs in registers whatever K.
__global__ void __launch_bounds__(kThreads) combine_vote_kernel(
    int64_t n_rec, const int64_t *__restrict__ offsets, int64_t N, int K, const int32_t *__restrict__ labels,
    const int32_t *__restrict__ labels2, const int32_t *__restrict__ n_labels, const int32_t *__restrict__ map_all,
    const double *__restrict__ weights, const int32_t *__restrict__ flags, int32_t *__restrict__ labels_out,
    int32_t *__restrict__ labels2_out) {
    const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (t >= N) return;
    int64_t a = 0, b = n_rec;                        // the last recording that starts at or before t
    while (b - a > 1) {
        const int64_t m = (a + b) >> 1;
        if (offsets[m] <= t) a = m;
        else b = m;
    }
    const int64_t rec = a;
    const int32_t *nl = n_labels + rec * K, *map = map_all + rec * K * kMaxLabels;
    const double *w = weights + rec * K;
    int g1 = -1, g2 = -1;
    double t1 = 0.0, t2 = 0.0;
    double num = 0.0, den = 0.0;
    const bool dead = flags[rec] & VBX_COMBINE_TOO_MANY_LABELS;
    for (int k = 0; k < K && !dead; ++k) {
        int s[2];
        read_labels(labels + (int64_t)k * N, labels2 + (int64_t)k * N, t, nl[k], s[0], s[1]);
        num += w[k] * (double)((s[0] >= 0) + (s[1] >= 0));
        den += w[k];
        for (int x = 0; x < 2; ++x) {
            const int g = s[x] >= 0 ? map[k * kMaxLabels + s[x]] : -1;
            if (g < 0 || g == g1 || g == g2) continue;
            const double tg = tally_of(g, t, N, K, labels, labels2, nl, map, w);
            if (g1 < 0 || tg > t1 || (tg == t1 && g < g1)) {
                g2 = g1;
                t2 = t1;
                g1 = g;
                t1 = tg;
            } else if (g2 < 0 || tg > t2 || (tg == t2 && g < g2)) {
                g2 = g;
                t2 = tg;
            }
        }
    }
    const double n = dead ? 0.0 : floor(0.5 + num / den);
    labels_out[t] = n >= 1.0 ? g1 : -1;
    labels2_out[t] = n >= 2.0 ? g2 : -1;
}

}  // namespace

size_t combine_workspace_bytes(int64_t n_rec, int K, int max_labels) {
    size_t total = 0;
    combine_layout(nullptr, n_rec, K, max_labels, &total);
    return total;
}

int launch_combine(int64_t n_rec, const int64_t *offsets, int64_t N, const int64_t *lo, const int64_t *hi, int K,
                   const int32_t *labels, const int32_t *labels2, const int32_t *n_labels_host, int max_labels,
                   const double *weights_host, void *workspace, int32_t *labels_out,
                   int32_t *labels2_out, int32_t *order_out, double *weights_out, int64_t *D_out, int32_t *map_out,
                   int32_t *n_global_out, int32_t *flags_out, int64_t *O_out, int64_t *L_out, cudaStream_t st) {
    const CombineWs w = combine_layout(reinterpret_cast<uint8_t *>(workspace), n_rec, K, max_labels, nullptr);
    int64_t *O = O_out ? O_out : w.O, *L = L_out ? L_out : w.L;
    // pageable source: staged before the call returns, no wait on the stream
    if (cudaMemcpyAsync(w.n_labels, n_labels_host, (size_t)n_rec * K * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(flags_out, 0, (size_t)n_rec * 4, st) != cudaSuccess)
        return -1;
    const int64_t cells = (int64_t)max_labels * max_labels;
    const int shared_block = cells <= kSmemCells;
    if (!allow_dynamic_smem(combine_overlap_kernel, (int)(kSmemCells * 8)) ||
        !allow_dynamic_smem(combine_map_kernel, (int)(sizeof(WarpLsap) * kWarps)))
        return -1;
    combine_overlap_kernel<<<(unsigned)(n_rec * (n_pairs(K) + K)), kThreads, shared_block ? cells * 8 : 0, st>>>(
        offsets, lo, hi, N, K, labels, labels2, w.n_labels, max_labels, shared_block, O, L, flags_out);
    double wt[kMaxK];
    for (int k = 0; k < K; ++k) {
        volatile double rank = k + 1;                // DOVER's default rank ** -0.1, by the host's pow at run time
        wt[k] = weights_host ? weights_host[k] : std::pow(rank, -0.1);
    }
    if (cudaMemcpyAsync(w.w, wt, (size_t)K * 8, cudaMemcpyHostToDevice, st) != cudaSuccess) return -1;
    combine_map_kernel<<<(unsigned)n_rec, kThreads, sizeof(WarpLsap) * kWarps, st>>>(
        K, w.n_labels, max_labels, O, L, w.C, w.w, weights_host != nullptr, order_out, weights_out, D_out, map_out, n_global_out, flags_out);
    int launches = 2;
    if (N > 0) {
        combine_vote_kernel<<<(unsigned)((N + kThreads - 1) / kThreads), kThreads, 0, st>>>(
            n_rec, offsets, N, K, labels, labels2, w.n_labels, map_out, weights_out, flags_out, labels_out, labels2_out);
        ++launches;
    }
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace vbx
