// Speaker linking across the recordings of an archive (DESIGN.md section 5.15).  Every speaker s of the archive (a
// recording's VB-HMM label) has the statistics n_s (its x-vectors) and F_s = sum of their features; with c = Fa / Fb,
// L_s,r = 1 + c n_s Phi_r and b_s,r = c sqrt(Phi_r) F_s,r are the precision and L * alpha of its VB-HMM posterior
// (VBx/VBx.py:95-96).  Two speakers score
//   LLR(s, u) = 1/2 sum_r [ (b_s + b_u)^2 / (L_s + L_u - 1) - log(L_s + L_u - 1) ] - e_s/2 - e_u/2,
//   e_s = sum_r [ b_s,r^2 / L_s,r - log L_s,r ],
// and average linkage runs over d = -LLR (kBig between two speakers of one recording, 0 on the diagonal).
//   link_init_kernel    spans, linkage offsets
//   link_span_kernel    first / last x-vector of every speaker (integer atomics: order-free)
//   link_stats_kernel   n_s, F_s (float64, fixed order), b_s and e_s; one CTA per speaker
//   link_score_kernel   the M x M distances, 32 x 32 tiles of the upper triangle, each written twice
//   norm_scores_kernel  (vbx_cohort.cu) only with cohort statistics (vbx_link_norm): d = -S in place, section 5.17
//   ahc_linkage_kernel  (vbx_ahc.cu) unchanged, over the matrix as one "recording" of M items
#include <algorithm>
#include <climits>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr double kBig = 1.0e30;            // cannot-link distance: finite (scipy and the linkage stop at non-finite ones)
constexpr int kStatsThreads = 256;
constexpr int kStatsPhases = kStatsThreads / 32;   // x-vector t = first + k, first + k + 8, ... makes phase k
constexpr int kLogGroup = 8;
constexpr int64_t kScoreGrid = 1 << 20;    // CTAs of link_score_kernel at most; beyond that they stride over the tiles               // log of a product of 8 denominators: each is 1 + c n Phi, so no overflow

struct LinkWs {
    uint8_t *lk;             // the linkage's region (carve() in vbx_ahc.cu): D [M,M] first
    double *n, *e, *b;       // [M], [M], [M,kMaxR]
    long long *first, *last; // [M]
    int64_t *offs;           // {0, M} and {0, 0}: the linkage's offsets and workspace offsets
};

size_t al(size_t v) { return (v + 255) & ~(size_t)255; }

LinkWs link_layout(uint8_t *ws, int64_t M, size_t *total) {
    LinkWs w;
    size_t o = 0;
    w.lk = ws;
    o += al(linkage_workspace_bytes(M));
    w.n = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * 8);
    w.e = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * 8);
    w.b = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * kMaxR * 8);
    w.first = reinterpret_cast<long long *>(ws + o);
    o += al((size_t)M * 8);
    w.last = reinterpret_cast<long long *>(ws + o);
    o += al((size_t)M * 8);
    w.offs = reinterpret_cast<int64_t *>(ws + o);
    o += al(4 * 8);
    if (total) *total = o;
    return w;
}

__global__ void link_init_kernel(LinkWs w, int64_t M) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < M) {
        w.first[i] = LLONG_MAX;
        w.last[i] = -1;
    }
    if (i == 0) {
        w.offs[0] = 0;
        w.offs[1] = M;
        w.offs[2] = 0;
        w.offs[3] = 0;
    }
}

__global__ void link_span_kernel(LinkWs w, const int32_t *__restrict__ spk, int64_t N, int64_t M) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const int s = spk[t];
    if (s < 0 || s >= M) return;
    atomicMin(&w.first[s], (long long)t);
    atomicMax(&w.last[s], (long long)t);
}

// One CTA per speaker over its span first .. last.  Warp k sums phase k of the span sequentially (lane = feature,
// 4 features per lane), then the 8 phase sums are added in phase order: the order depends on the positions of the
// speaker's x-vectors relative to its first one, not on the batch, the launch or the other speakers.
__global__ void __launch_bounds__(kStatsThreads) link_stats_kernel(LinkWs w, const float *__restrict__ fea,
                                                                   const float *__restrict__ Phi,
                                                                   const int32_t *__restrict__ spk, int R, double c,
                                                                   double *__restrict__ n_out, double *__restrict__ F_out) {
    __shared__ double part[kStatsPhases][kMaxR];
    __shared__ double cnt[kStatsPhases];
    __shared__ double red[kStatsThreads / 32];
    const int s = blockIdx.x;
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long f = w.first[s], l = w.last[s];
    double acc[kMaxR / 32] = {0, 0, 0, 0};
    double m = 0.0;
    if (l >= 0) {
        for (long long t = f + k; t <= l; t += kStatsPhases) {
            if (spk[t] != s) continue;
            m += 1.0;
            const float *x = fea + (int64_t)t * R;
#pragma unroll
            for (int j = 0; j < kMaxR / 32; ++j)
                if (lane + 32 * j < R) acc[j] += (double)x[lane + 32 * j];
        }
    }
#pragma unroll
    for (int j = 0; j < kMaxR / 32; ++j) part[k][lane + 32 * j] = acc[j];
    if (lane == 0) cnt[k] = m;
    __syncthreads();
    double n = 0.0;
    for (int q = 0; q < kStatsPhases; ++q) n += cnt[q];
    double e = 0.0;
    for (int r = threadIdx.x; r < R; r += kStatsThreads) {
        double F = 0.0;
        for (int q = 0; q < kStatsPhases; ++q) F += part[q][r];
        const double ph = (double)Phi[r];
        const double L = 1.0 + c * n * ph, b = c * sqrt(ph) * F;
        w.b[(int64_t)s * kMaxR + r] = b;
        if (F_out) F_out[(int64_t)s * R + r] = F;
        e += b * b / L - log(L);
    }
    for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);   // fixed butterfly, then warps in order
    if (lane == 0) red[k] = e;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int q = 0; q < kStatsThreads / 32; ++q) tot += red[q];
        w.e[s] = tot;
        w.n[s] = n;
        if (n_out) n_out[s] = n;
    }
}

// Tile (bi, bj), bj >= bi, of 32 x 32 speaker pairs: 256 threads, 4 pairs each (rows ty, ty + 8, ..), features in chunks
// of 32 through shared memory.  Every pair sums its features in order r = 0 .. R-1 with operands that commute, so
// d[i][j] and d[j][i] are the same number; the tile is written row-wise and, through shared memory, column-wise.  The
// tiles of the upper triangle are numbered row by row (row bi holds tiles - bi of them) and the CTAs stride over them,
// so the grid stays one-dimensional and within its limit for every M.
__device__ __forceinline__ void score_tile(const LinkWs &w, const float *__restrict__ Phi,
                                           const int32_t *__restrict__ spk_rec, int64_t M, int R, double c,
                                           double *__restrict__ dist_out, int64_t bi, int64_t bj) {
    __shared__ double a[32][33], bt[32][33], ph[32];
    __shared__ double tile[32][33];
    const int64_t i0 = (int64_t)bi * 32, j0 = (int64_t)bj * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t j = j0 + tx;
    const double nj = j < M ? w.n[j] : 0.0;
    double cm[4], q[4] = {0, 0, 0, 0}, lg[4] = {0, 0, 0, 0}, prod[4] = {1, 1, 1, 1};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t i = i0 + ty + 8 * u;
        cm[u] = c * ((i < M ? w.n[i] : 0.0) + nj);
    }
    for (int r0 = 0; r0 < R; r0 += 32) {
        for (int v = ty; v < 32; v += 8) {
            const int r = r0 + tx;
            a[v][tx] = (i0 + v < M && r < R) ? w.b[(i0 + v) * kMaxR + r] : 0.0;
            bt[v][tx] = (j0 + v < M && r < R) ? w.b[(j0 + v) * kMaxR + r] : 0.0;
        }
        if (ty == 0) ph[tx] = r0 + tx < R ? (double)Phi[r0 + tx] : 0.0;
        __syncthreads();
        const int len = min(32, R - r0);
        for (int k = 0; k < len; ++k) {
            const double bj_k = bt[tx][k], p = ph[k];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const double den = fma(cm[u], p, 1.0), x = a[ty + 8 * u][k] + bj_k;
                q[u] += x * x / den;
                prod[u] *= den;
            }
            if (((r0 + k) % kLogGroup) == kLogGroup - 1 || r0 + k == R - 1) {
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    lg[u] += log(prod[u]);
                    prod[u] = 1.0;
                }
            }
        }
        __syncthreads();
    }
    double *D = reinterpret_cast<double *>(w.lk);
    const int rj = j < M ? spk_rec[j] : -1;
    const double ej = j < M ? w.e[j] : 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t i = i0 + ty + 8 * u;
        if (i >= M || j >= M) continue;
        double d;
        if (i == j) d = 0.0;
        else if (spk_rec[i] == rj) d = kBig;
        else if (w.n[i] == 0.0 || nj == 0.0) d = 0.0;
        else d = -0.5 * ((q[u] - lg[u]) - (w.e[i] + ej));
        tile[ty + 8 * u][tx] = d;
        D[i * M + j] = d;
        if (dist_out) dist_out[i * M + j] = d;
    }
    __syncthreads();
    if (bi != bj) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {                 // D[j0 + ty + 8u][i0 + tx] = tile[tx][ty + 8u]
            const int64_t jj = j0 + ty + 8 * u, ii = i0 + tx;
            if (jj >= M || ii >= M) continue;
            D[jj * M + ii] = tile[tx][ty + 8 * u];
            if (dist_out) dist_out[jj * M + ii] = tile[tx][ty + 8 * u];
        }
    }
    __syncthreads();                                  // the CTA's next tile rewrites the shared arrays
}

__global__ void __launch_bounds__(256) link_score_kernel(LinkWs w, const float *__restrict__ Phi,
                                                         const int32_t *__restrict__ spk_rec, int64_t M, int R, double c,
                                                         double *__restrict__ dist_out) {
    const int64_t tiles = (M + 31) / 32, n_tiles = tiles * (tiles + 1) / 2;
    const double tt = 2.0 * (double)tiles + 1.0;
    auto row0 = [tiles](int64_t b) { return b * tiles - b * (b - 1) / 2; };   // first tile of row b
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        int64_t bi = (int64_t)((tt - sqrt(tt * tt - 8.0 * (double)t)) / 2.0);  // row0 inverted, then rounding corrected
        while (bi > 0 && row0(bi) > t) --bi;
        while (bi + 1 < tiles && row0(bi + 1) <= t) ++bi;
        score_tile(w, Phi, spk_rec, M, R, c, dist_out, bi, bi + (t - row0(bi)));
    }
}

}  // namespace

size_t link_workspace_bytes(int64_t M) {
    size_t total = 0;
    link_layout(nullptr, M, &total);
    return total;
}

int launch_link(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, const int32_t *spk_rec,
                int64_t M, double c, void *workspace, double *n_out, double *F_out, double *dist_out, double *Z_out,
                cudaStream_t st, const double *mean, const double *std) {
    if (M == 0) return 0;
    const LinkWs w = link_layout(reinterpret_cast<uint8_t *>(workspace), M, nullptr);
    int launches = 0;
    link_init_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(w, M);
    ++launches;
    if (N > 0) {
        link_span_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(w, spk, N, M);
        ++launches;
    }
    link_stats_kernel<<<(unsigned)M, kStatsThreads, 0, st>>>(w, fea, Phi, spk, R, c, n_out, F_out);
    const int64_t tiles = (M + 31) / 32, n_tiles = tiles * (tiles + 1) / 2;
    link_score_kernel<<<(unsigned)std::min<int64_t>(n_tiles, kScoreGrid), 256, 0, st>>>(w, Phi, spk_rec, M, R, c,
                                                                                        mean ? nullptr : dist_out);
    launches += 2;
    if (mean) {                                       // normalised distances (section 5.17): dist_out gets those
        const int ln = launch_norm_scores(reinterpret_cast<double *>(w.lk), M, M, mean, std, mean, std, true, kBig,
                                          dist_out, st);
        if (ln < 0) return -1;
        launches += ln;
    }
    if (M >= 2) {
        launch_linkage(w.offs, w.offs + 2, w.lk, Z_out, st);
        ++launches;
    }
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

int launch_speaker_stats(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, int64_t M, double c,
                         const SpeakerStats &s, double *n_out, double *F_out, cudaStream_t st) {
    if (M == 0) return 0;
    LinkWs w;
    w.lk = nullptr;
    w.n = s.n;
    w.e = s.e;
    w.b = s.b;
    w.first = s.first;
    w.last = s.last;
    w.offs = s.offs;
    int launches = 2;
    link_init_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(w, M);
    if (N > 0) {
        link_span_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(w, spk, N, M);
        ++launches;
    }
    link_stats_kernel<<<(unsigned)M, kStatsThreads, 0, st>>>(w, fea, Phi, spk, R, c, n_out, F_out);
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace vbx
