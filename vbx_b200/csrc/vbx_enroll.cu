// Enrolment against known speakers (DESIGN.md sections 5.16, 5.19).  vbx_enroll_batch runs G problems (e.g. the
// settings of a sweep; one archive is the batch of one) that share fea, Phi and the enrolled set; each has its own
// speakers, c_g and column statistics.  The archive's speakers (section 5.15's table) and the enrolled speakers get
// the statistics n, F, b and e of vbx_link_batch (its span and statistics kernels over all problems at once, through
// launch_speaker_stats_batch), every archive speaker s is scored against every enrolled speaker e with section 5.15's
// LLR, and each recording's speakers are assigned one-to-one to enrolled speakers or to "unknown":
//   enroll_score_kernel   llr [M, E], 32 x 32 tiles of every problem's rectangle, the flat tile index decoded into
//                         (problem, tile); llr[s][e] is bit-identical to -dist[s][e] of vbx_link_batch on the same
//                         speakers (both score through tile_llr_sums and pair_llr)
//   enroll_assign_kernel  per recording b with K_b speakers and threshold h the minimum-cost assignment of the
//                         K_b x (E + K_b) matrix C[k][e] = threshold_h - llr[k][e] (e < E), C[k][E + j] = 0 ("unknown"
//                         columns), by shortest augmenting paths (Jonker-Volgenant, the method of scipy's
//                         linear_sum_assignment): one Dijkstra per row over the columns; a persistent grid, one
//                         (threshold, recording) item per CTA at a time, one output plane per threshold
// With cohort statistics (section 5.17) vbx_cohort.cu's norm_scores_kernel turns llr into S in place between the two.
// launch_cohort_scores_batch runs enroll_score_kernel against a cohort for vbx_cohort_stats_batch.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cstring>
#include <vector>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int64_t kScoreGrid = 1 << 20;     // CTAs of enroll_score_kernel at most; beyond that they stride over the tiles
constexpr int kAssignThreads = 256;
constexpr int kAssignWarps = kAssignThreads / 32;
constexpr int kAssignCtasPerSm = 2;

// one CTA's column and row state in the workspace: columns nc = E + K_b <= E + max_k, rows K_b <= max_k
struct Slice {
    double *v, *spc, *u;                // column duals, shortest path costs; row duals
    int64_t *path, *row4col, *col4row;  // row reaching each column, row of each column, column of each row (-1: none)
    uint8_t *sc, *sr;                   // columns / rows reached in the current Dijkstra
};

__host__ __device__ Slice slice_at(uint8_t *base, int64_t ncm, int64_t km, size_t *total) {
    Slice s;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = base ? base + o : nullptr; o += al(bytes); return p; };
    s.v = reinterpret_cast<double *>(take(ncm * 8));
    s.spc = reinterpret_cast<double *>(take(ncm * 8));
    s.u = reinterpret_cast<double *>(take(km * 8));
    s.path = reinterpret_cast<int64_t *>(take(ncm * 8));
    s.row4col = reinterpret_cast<int64_t *>(take(ncm * 8));
    s.col4row = reinterpret_cast<int64_t *>(take(km * 8));
    s.sc = take(ncm);
    s.sr = take(km);
    if (total) *total = o;
    return s;
}

// The archive speakers of all problems [M], the enrolled speakers once per problem [G E] with their index [G, N_e],
// llr [M, E], the problem arrays (off, eoff = g E, tile_off [G+1], c [G], thresholds [n_thr], recs [at most M + 1]:
// the speaker offsets of the recordings that have speakers) and the slices of CTAs that take n_thr x (recordings with
// speakers) items
struct EnrollWs {
    SpeakerStats a, en;
    int32_t *espk;
    double *llr;
    int64_t *arrays;
    uint8_t *slices;         // ctas x slice_bytes
    size_t slice_bytes;
    int64_t ctas;
};

EnrollWs enroll_layout(uint8_t *ws, int64_t G, int64_t M, int64_t E, int64_t N_e, int64_t max_k, int64_t n_thr, int sms,
                       size_t *total) {
    EnrollWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.a = take_stats(take, M);
    w.en = take_stats(take, G * E);
    w.espk = reinterpret_cast<int32_t *>(take((size_t)G * N_e * 4));
    w.llr = reinterpret_cast<double *>(take((size_t)M * E * 8));
    w.arrays = reinterpret_cast<int64_t *>(take((size_t)(4 * G + 3 + n_thr + M + 1) * 8));
    slice_at(nullptr, E + max_k, max_k, &w.slice_bytes);
    w.ctas = std::min<int64_t>((int64_t)kAssignCtasPerSm * std::max(sms, 1), std::max<int64_t>(M * n_thr, 1));
    w.slices = take(w.slice_bytes * w.ctas);
    if (total) *total = o;
    return w;
}

__global__ void repeat_index_kernel(const int32_t *__restrict__ src, int64_t n, int64_t total,
                                    int32_t *__restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = src[i % n];
}

// The problems of one enroll_score_kernel launch: problem g's rows are off[g] .. off[g+1]-1 of the row statistics and
// of llr, its columns g E .. g E + E - 1 of the column statistics (whose b and e depend on c_g), and its tiles
// tile_off[g] .. tile_off[g+1]-1 of the flat tile index.
struct ScoreProblems {
    int G;
    const int64_t *off, *tile_off;
    const double *c;
};

// Tile (bi, bj) of 32 archive speakers (rows) x 32 enrolled speakers (columns) (tile_llr_sums).  The flat tile index
// runs over the rectangles of all problems (decoded as link_score_kernel does), so the grid stays one-dimensional and
// capped for any G, M_g and E.
__global__ void __launch_bounds__(256) enroll_score_kernel(SpeakerStats A0, SpeakerStats En0, const float *__restrict__ Phi,
                                                           int64_t E, int R, double *__restrict__ llr0,
                                                           double *__restrict__ llr_out0, ScoreProblems pr) {
    __shared__ double a[32][33], bt[32][33], ph[32];
    const int64_t tiles_e = (E + 31) / 32, n_tiles = pr.tile_off[pr.G];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int g = find_problem(pr.tile_off, pr.G, t);
        const int64_t base = pr.off[g], col = (int64_t)g * E, M = pr.off[g + 1] - base, lt = t - pr.tile_off[g];
        const double c = pr.c[g];
        SpeakerStats A = A0, En = En0;
        A.n += base;
        A.e += base;
        A.b += base * kMaxR;
        En.n += col;
        En.e += col;
        En.b += col * kMaxR;
        double *llr = llr0 + base * E, *llr_out = llr_out0 ? llr_out0 + base * E : nullptr;
        const int64_t i0 = (lt / tiles_e) * 32, j0 = (lt % tiles_e) * 32;
        const int64_t j = j0 + tx;
        const double nj = j < E ? En.n[j] : 0.0;
        double cm[4], q[4] = {0, 0, 0, 0}, lg[4] = {0, 0, 0, 0}, prod[4] = {1, 1, 1, 1};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int64_t i = i0 + ty + 8 * u;
            cm[u] = c * ((i < M ? A.n[i] : 0.0) + nj);
        }
        tile_llr_sums(a, bt, ph, A.b, M, En.b, E, Phi, R, i0, j0, cm, q, lg, prod);
        llr_finish<4>(lg, cm, Phi, R);
        if (j >= E) continue;
        const double ej = En.e[j];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int64_t i = i0 + ty + 8 * u;
            if (i >= M) continue;
            const double l = pair_llr(q[u], lg[u], A.n[i], nj, A.e[i], ej);
            llr[i * E + j] = l;
            if (llr_out) llr_out[i * E + j] = l;
        }
    }
}

// (value, column) pairs: the smaller value, on equal values the lower column (-1 only comes with +inf)
__device__ __forceinline__ void take_min(double &bv, int64_t &bj, double ov, int64_t oj) {
    if (ov < bv || (ov == bv && oj < bj)) {
        bv = ov;
        bj = oj;
    }
}

// One CTA per recording at a time.  Per row (speaker) cur = 0 .. K-1 one Dijkstra over the columns: every step scans the
// columns not yet reached, relaxes their path costs from row i (r = minVal + C[i][j] - u[i] - v[j], scipy's order) and
// takes the block argmin; ties go to the lowest column index (so a real column at cost 0 wins over the unknown
// columns).  A reached column that no row holds ends the path; otherwise its row is scanned next.  Then the duals are
// updated and the path augmented as scipy's rectangular_lsap does.  A step that reaches no column (non-finite costs)
// leaves the row unassigned.  Outputs per speaker: its enrolled index or -1, and the LLR of its pair, or for an
// unknown speaker its largest LLR.
// Work items: the recordings with speakers of every problem are one list recs (the problems' speakers are packed one
// after the other, so their offsets run on), and item (h, rec) assigns recording rec at thresholds[h] into plane h of
// the outputs (assign_out + h plane, best_out + h plane): n_thr x n_recs items over the persistent grid, so the slices
// stay CTAs x (E + max_k) and the LLR block is computed once for every threshold.  Bounded for the kAssignCtasPerSm
// CTAs per SM it is launched with, which keeps its state in registers.
__global__ void __launch_bounds__(kAssignThreads, kAssignCtasPerSm) enroll_assign_kernel(
    const double *__restrict__ llr, const int64_t *__restrict__ recs, int64_t n_recs, int64_t E, uint8_t *slices,
    size_t slice_bytes, int64_t max_k, int32_t *__restrict__ assign_all, double *__restrict__ best_all,
    const double *__restrict__ thetas, int64_t n_thr, int64_t plane) {
    __shared__ double wv[kAssignWarps];
    __shared__ int64_t wj[kAssignWarps];
    __shared__ double s_min;
    __shared__ int64_t s_i, s_sink;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const Slice sl = slice_at(slices + (size_t)blockIdx.x * slice_bytes, E + max_k, max_k, nullptr);
    for (int64_t item = blockIdx.x; item < n_recs * n_thr; item += gridDim.x) {
        const int64_t h = item / n_recs, rec = item - h * n_recs;
        const double theta = thetas[h];
        const int64_t s0 = recs[rec], K = recs[rec + 1] - s0, nc = E + K;
        for (int64_t j = tid; j < nc; j += kAssignThreads) {
            sl.v[j] = 0.0;
            sl.row4col[j] = -1;
        }
        for (int64_t k = tid; k < K; k += kAssignThreads) {
            sl.u[k] = 0.0;
            sl.col4row[k] = -1;
        }
        for (int64_t cur = 0; cur < K; ++cur) {
            for (int64_t j = tid; j < nc; j += kAssignThreads) {
                sl.spc[j] = INFINITY;
                sl.sc[j] = 0;
            }
            for (int64_t k = tid; k < K; k += kAssignThreads) sl.sr[k] = 0;
            if (tid == 0) {
                s_i = cur;
                s_sink = -1;
                s_min = 0.0;
            }
            __syncthreads();
            int64_t i = cur, sink = -1;
            double minVal = 0.0;
            for (int64_t step = 0; step < nc && sink == -1; ++step) {
                const double ui = sl.u[i];
                const double *lrow = llr + (s0 + i) * E;
                double bv = INFINITY;
                int64_t bj = -1;
                for (int64_t j = tid; j < nc; j += kAssignThreads) {
                    if (sl.sc[j]) continue;
                    const double cost = j < E ? theta - lrow[j] : 0.0;
                    const double r = minVal + cost - ui - sl.v[j];
                    double p = sl.spc[j];
                    if (r < p) {
                        sl.path[j] = i;
                        sl.spc[j] = r;
                        p = r;
                    }
                    if (p < bv) {                             // strided in increasing j: the lowest column on ties
                        bv = p;
                        bj = j;
                    }
                }
                for (int o = 16; o; o >>= 1)
                    take_min(bv, bj, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bj, o));
                if (lane == 0) {
                    wv[warp] = bv;
                    wj[warp] = bj;
                }
                __syncthreads();
                if (tid == 0) {
                    for (int q = 1; q < kAssignWarps; ++q) take_min(bv, bj, wv[q], wj[q]);
                    sl.sr[i] = 1;
                    if (bj < 0) {
                        s_sink = -2;
                    } else {
                        sl.sc[bj] = 1;
                        s_min = bv;
                        if (sl.row4col[bj] < 0) s_sink = bj;
                        else s_i = sl.row4col[bj];
                    }
                }
                __syncthreads();
                minVal = s_min;
                sink = s_sink;
                i = s_i;
            }
            if (sink >= 0) {                                  // every thread saw the same sink
                for (int64_t k = tid; k < K; k += kAssignThreads)
                    if (sl.sr[k] && k != cur) sl.u[k] += minVal - sl.spc[sl.col4row[k]];
                for (int64_t j = tid; j < nc; j += kAssignThreads)
                    if (sl.sc[j]) sl.v[j] -= minVal - sl.spc[j];
                __syncthreads();
                if (tid == 0) {
                    sl.u[cur] += minVal;
                    int64_t j = sink;
                    while (true) {
                        const int64_t r = sl.path[j];
                        sl.row4col[j] = r;
                        const int64_t prev = sl.col4row[r];
                        sl.col4row[r] = j;
                        j = prev;
                        if (r == cur) break;
                    }
                }
            }
            __syncthreads();                                  // s_* and the slice are read before the next row
        }
        __syncthreads();
        for (int64_t k = warp; k < K; k += kAssignWarps) {
            const int64_t col = sl.col4row[k];
            const double *lrow = llr + (s0 + k) * E;
            const bool named = col >= 0 && col < E;
            double m = -INFINITY;
            if (named) {
                m = lrow[col];
            } else {
                for (int64_t j = lane; j < E; j += 32) m = fmax(m, lrow[j]);
                for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
            }
            if (lane == 0) {
                const int64_t o = h * plane + s0 + k;         // threshold h's plane
                assign_all[o] = named ? (int32_t)col : -1;
                best_all[o] = m;
            }
        }
        __syncthreads();                                      // the next recording rewrites the slice
    }
}

}  // namespace

int64_t rect_tiles(int64_t M, int64_t C) { return ((M + 31) / 32) * ((C + 31) / 32); }

int launch_cohort_scores_batch(const SpeakerStats &a, const SpeakerStats &co, const float *Phi, int G,
                               const int64_t *off, const int64_t *tile_off, const double *c, int64_t n_tiles, int64_t C,
                               int R, double *llr, double *llr_out, cudaStream_t st) {
    if (n_tiles == 0) return 0;
    const ScoreProblems p{G, off, tile_off, c};
    enroll_score_kernel<<<(unsigned)std::min<int64_t>(n_tiles, kScoreGrid), 256, 0, st>>>(a, co, Phi, C, R, llr,
                                                                                         llr_out, p);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

size_t enroll_assign_workspace_bytes(int64_t E, int64_t max_k, int64_t n_recs, int sms) {
    size_t slice = 0;
    slice_at(nullptr, E + max_k, max_k, &slice);
    return slice * (size_t)std::min<int64_t>((int64_t)kAssignCtasPerSm * std::max(sms, 1), std::max<int64_t>(n_recs, 1));
}

int launch_enroll_assign(const double *llr, const int64_t *recs, int64_t n_recs, int64_t E, int64_t max_k,
                         const double *threshold, void *slices, int sms, int32_t *assign_out, double *best_llr_out,
                         cudaStream_t st) {
    if (n_recs == 0) return 0;
    size_t slice = 0;
    slice_at(nullptr, E + max_k, max_k, &slice);
    const int64_t ctas = std::min<int64_t>((int64_t)kAssignCtasPerSm * std::max(sms, 1), n_recs);
    enroll_assign_kernel<<<(unsigned)ctas, kAssignThreads, 0, st>>>(llr, recs, n_recs, E,
                                                                    reinterpret_cast<uint8_t *>(slices), slice, max_k,
                                                                    assign_out, best_llr_out, threshold, 1, 0);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_repeat_index(const int32_t *src, int64_t n, int G, int32_t *dst, cudaStream_t st) {
    const int64_t total = (int64_t)G * n;
    if (total == 0) return 0;
    repeat_index_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 4096), 256, 0, st>>>(src, n, total, dst);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

size_t enroll_batch_workspace_bytes(int G, const int64_t *M_host, int64_t E, int64_t N_e, int64_t max_k, int64_t n_thr,
                                    int sms) {
    int64_t M = 0;
    for (int g = 0; g < G; ++g) M += M_host[g];
    size_t total = 0;
    enroll_layout(nullptr, G, M, E, N_e, max_k, n_thr, sms, &total);
    return total;
}

int launch_enroll_batch(const float *fea, const float *Phi, int64_t N, int R, const int32_t *spk, int G,
                        const int64_t *M_host, const int64_t *rec_off_host, int n_rec, const float *enroll_fea,
                        int64_t N_e, const int32_t *enroll_spk, int64_t E, const double *c_host,
                        const double *thresholds, int64_t n_thr, void *workspace, int sms, int32_t *assign_out,
                        double *best_llr_out, double *llr_out, double *n_out, double *F_out, double *n_enroll_out,
                        double *F_enroll_out, cudaStream_t st, const double *mean, const double *std,
                        const double *enroll_mean, const double *enroll_std) {
    // one upload: off, eoff, tile_off [G+1], c [G], thresholds [n_thr], then the speaker offsets of the recordings
    // with speakers of all problems (problem g's speakers start at off[g], so the list runs on across problems)
    int64_t M_all = 0;
    for (int g = 0; g < G; ++g) M_all += M_host[g];
    std::vector<int64_t> host(4 * (size_t)G + 3 + n_thr, 0);
    host.reserve(host.size() + M_all + 1);            // the recordings below never reallocate: off, eoff, tile stay valid
    int64_t *off = host.data(), *eoff = off + (G + 1), *tile = eoff + (G + 1);
    int64_t max_k = 0;
    for (int g = 0; g < G; ++g) {
        off[g + 1] = off[g] + M_host[g];
        eoff[g + 1] = eoff[g] + E;
        tile[g + 1] = tile[g] + rect_tiles(M_host[g], E);
    }
    std::memcpy(tile + (G + 1), c_host, (size_t)G * sizeof(double));
    std::memcpy(tile + (G + 1) + G, thresholds, (size_t)n_thr * sizeof(double));
    const size_t recs_at = host.size();
    host.push_back(0);
    for (int g = 0; g < G; ++g) {
        const int64_t *ro = rec_off_host + (size_t)g * (n_rec + 1);
        for (int b = 0; b < n_rec; ++b) {
            const int64_t k = ro[b + 1] - ro[b];
            if (k > 0) host.push_back(off[g] + ro[b + 1]);
            max_k = std::max(max_k, k);
        }
    }
    const int64_t M = off[G], n_busy = (int64_t)(host.size() - recs_at) - 1;
    const EnrollWs w = enroll_layout(reinterpret_cast<uint8_t *>(workspace), G, M, E, N_e, max_k, n_thr, sms, nullptr);
    if (cudaMemcpyAsync(w.arrays, host.data(), host.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st) !=
        cudaSuccess)
        return -1;
    const int64_t *d_off = w.arrays, *d_eoff = d_off + (G + 1), *d_tile = d_eoff + (G + 1);
    const double *d_c = reinterpret_cast<const double *>(d_tile + (G + 1)), *d_thr = d_c + G;
    const int64_t *d_recs = w.arrays + recs_at;
    const int lr = launch_repeat_index(enroll_spk, N_e, G, w.espk, st);
    const int la = launch_speaker_stats_batch(fea, Phi, spk, N, R, G, d_off, d_c, M, w.a, n_out, F_out, st);
    const int le = launch_speaker_stats_batch(enroll_fea, Phi, w.espk, N_e, R, G, d_eoff, d_c, (int64_t)G * E, w.en,
                                              n_enroll_out, F_enroll_out, st);
    if (lr < 0 || la < 0 || le < 0) return -1;
    int launches = lr + la + le;
    if (M > 0) {
        const ScoreProblems p{G, d_off, d_tile, d_c};
        enroll_score_kernel<<<(unsigned)std::min<int64_t>(tile[G], kScoreGrid), 256, 0, st>>>(
            w.a, w.en, Phi, E, R, w.llr, mean ? nullptr : llr_out, p);
        ++launches;
        if (mean) {                                   // normalised scores, each problem with its own statistics
            const NormProblems q{G, d_off, nullptr, nullptr};
            const int ln = launch_norm_scores(w.llr, M, E, mean, std, enroll_mean, enroll_std, false, 0.0, llr_out, st,
                                              q);
            if (ln < 0) return -1;
            launches += ln;
        }
    }
    if (n_busy > 0) {
        enroll_assign_kernel<<<(unsigned)std::min<int64_t>(n_busy * n_thr, w.ctas), kAssignThreads, 0, st>>>(
            w.llr, d_recs, n_busy, E, w.slices, w.slice_bytes, max_k, assign_out, best_llr_out, d_thr, n_thr, M);
        ++launches;
    }
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace vbx
