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
//   norm_scores_kernel  (vbx_cohort.cu) only with cohort statistics (mean, std): d = -S in place, section 5.17
//   ahc_linkage_kernel  (vbx_ahc.cu) unchanged, over each problem's matrix as one "recording" of M_g items
// vbx_link_batch (sections 5.18, 5.19) runs G independent problems over one fea / Phi, each with its own speaker index
// [G, N], speaker_rec slice and c_g; one archive is the batch of one.  The problems' speakers are packed by the
// offsets off [G+1]; the statistics kernels run one CTA per (problem, speaker), the score kernel's flat tile index runs
// over the upper-triangle tiles of all problems, norm_scores_kernel over every problem's block, and one linkage launch
// has one CTA per problem, so a problem's results do not depend on the others.  vbx_enroll_batch and
// vbx_cohort_stats_batch take the statistics through launch_speaker_stats_batch.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cstring>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr double kBig = 1.0e30;            // cannot-link distance: finite (scipy and the linkage stop at non-finite ones)
constexpr int kStatsThreads = 256;
constexpr int kStatsPhases = kStatsThreads / 32;   // x-vector t = first + k, first + k + 8, ... makes phase k
constexpr int64_t kScoreGrid = 1 << 20;    // CTAs of link_score_kernel at most; beyond that they stride over the tiles

struct LinkWs {
    uint8_t *lk;             // the linkage regions (carve() in vbx_ahc.cu), each D [M_g,M_g] first
    SpeakerStats s;          // M: the speakers of all problems
    int64_t *offs;           // the problem arrays of LinkProblems
};

// The problems of one call (the statistics of vbx_enroll_batch / vbx_cohort_stats_batch leave lk_off, tile_off and
// dist_off null: they launch no score kernel).
struct LinkProblems {
    int G;
    int64_t M, N;            // speakers of all problems; x-vectors (speaker index [G, N])
    const int64_t *off;      // [G+1] speaker offsets (the linkage's offsets)
    const int64_t *lk_off;   // [G+1] byte offsets of the linkage regions in lk (the linkage's workspace offsets)
    const int64_t *tile_off; // [G+1] first flat score tile of each problem
    const int64_t *dist_off; // [G+1] first element of each problem's distances in dist_out
    const double *c;         // [G] Fa_g / Fb_g
};

size_t problem_array_bytes(int64_t G) { return (size_t)(5 * G + 4) * 8; }   // off, lk_off, tile_off, dist_off, c

int64_t score_tiles(int64_t M) {
    const int64_t tiles = (M + 31) / 32;
    return tiles * (tiles + 1) / 2;
}

// lk_bytes: the linkage regions of all problems (each al(linkage_workspace_bytes(M_g))), M: their speakers
LinkWs link_layout(uint8_t *ws, size_t lk_bytes, int64_t M, int64_t G, size_t *total) {
    LinkWs w;
    size_t o = 0;
    w.lk = ws;
    o += lk_bytes;
    w.s.n = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * 8);
    w.s.e = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * 8);
    w.s.b = reinterpret_cast<double *>(ws + o);
    o += al((size_t)M * kMaxR * 8);
    w.s.first = reinterpret_cast<long long *>(ws + o);
    o += al((size_t)M * 8);
    w.s.last = reinterpret_cast<long long *>(ws + o);
    o += al((size_t)M * 8);
    w.offs = reinterpret_cast<int64_t *>(ws + o);
    o += al(problem_array_bytes(G));
    if (total) *total = o;
    return w;
}

__global__ void link_init_kernel(LinkWs w, LinkProblems p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.M) {
        w.s.first[i] = LLONG_MAX;
        w.s.last[i] = -1;
    }
}

// One thread per (problem, x-vector); speaker[g, t] is a local index of problem g.
__global__ void link_span_kernel(LinkWs w, LinkProblems p, const int32_t *__restrict__ spk) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)p.G * p.N) return;
    const int s = spk[i];
    const int64_t g = i / p.N, t = i - g * p.N, base = p.off[g], M = p.off[g + 1] - base;
    if (s < 0 || s >= M) return;
    atomicMin(&w.s.first[base + s], (long long)t);
    atomicMax(&w.s.last[base + s], (long long)t);
}

// One CTA per speaker over its span first .. last.  Warp k sums phase k of the span sequentially (lane = feature,
// 4 features per lane), then the 8 phase sums are added in phase order: the order depends on the positions of the
// speaker's x-vectors relative to its first one, not on the batch, the launch, the problem or the other speakers.
// CTA s is speaker s of all problems: local speaker s - off[g] of problem g.
__global__ void __launch_bounds__(kStatsThreads) link_stats_kernel(LinkWs w, LinkProblems p, const float *__restrict__ fea,
                                                                   const float *__restrict__ Phi,
                                                                   const int32_t *__restrict__ spk, int R,
                                                                   double *__restrict__ n_out, double *__restrict__ F_out) {
    __shared__ double part[kStatsPhases][kMaxR];
    __shared__ double cnt[kStatsPhases];
    __shared__ double red[kStatsThreads / 32];
    const int s = blockIdx.x;
    const int g = find_problem(p.off, p.G, s);
    const int ls = s - (int)p.off[g];
    const double c = p.c[g];
    spk += (int64_t)g * p.N;
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long f = w.s.first[s], l = w.s.last[s];
    double acc[kMaxR / 32] = {0, 0, 0, 0};
    double m = 0.0;
    if (l >= 0) {
        for (long long t = f + k; t <= l; t += kStatsPhases) {
            if (spk[t] != ls) continue;
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
        double L, b;
        speaker_L_b(c, n, (double)Phi[r], F, L, b);
        w.s.b[(int64_t)s * kMaxR + r] = b;
        if (F_out) F_out[(int64_t)s * R + r] = F;
        e += speaker_e_term(L, b);
    }
    for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);   // fixed butterfly, then warps in order
    if (lane == 0) red[k] = e;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int q = 0; q < kStatsThreads / 32; ++q) tot += red[q];
        w.s.e[s] = tot;
        w.s.n[s] = n;
        if (n_out) n_out[s] = n;
    }
}

// Tile (bi, bj), bj >= bi, of 32 x 32 speaker pairs (tile_llr_sums).  Every pair sums its features in order
// r = 0 .. R-1 with operands that commute, so d[i][j] and d[j][i] are the same number; the tile is written row-wise
// and, through shared memory, column-wise.  The tiles of the upper triangle are numbered row by row (row bi holds
// tiles - bi of them) and the CTAs stride over them, so the grid stays one-dimensional and within its limit for any M.
__device__ __forceinline__ void score_tile(const LinkWs &w, const float *__restrict__ Phi,
                                           const int32_t *__restrict__ spk_rec, int64_t M, int R, double c,
                                           double *__restrict__ dist_out, int64_t bi, int64_t bj) {
    __shared__ double a[32][33], bt[32][33], ph[32];
    __shared__ double tile[32][33];
    const int64_t i0 = (int64_t)bi * 32, j0 = (int64_t)bj * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t j = j0 + tx;
    const double nj = j < M ? w.s.n[j] : 0.0;
    double cm[4], q[4] = {0, 0, 0, 0}, lg[4] = {0, 0, 0, 0}, prod[4] = {1, 1, 1, 1};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t i = i0 + ty + 8 * u;
        cm[u] = c * ((i < M ? w.s.n[i] : 0.0) + nj);
    }
    tile_llr_sums(a, bt, ph, w.s.b, M, w.s.b, M, Phi, R, i0, j0, cm, q, lg, prod);
    llr_finish<4>(lg, cm, Phi, R);
    double *D = reinterpret_cast<double *>(w.lk);
    const int rj = j < M ? spk_rec[j] : -1;
    const double ej = j < M ? w.s.e[j] : 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t i = i0 + ty + 8 * u;
        if (i >= M || j >= M) continue;
        double d;
        if (i == j) d = 0.0;
        else if (spk_rec[i] == rj) d = kBig;
        else d = pair_llr(q[u], lg[u], w.s.n[i], nj, w.s.e[i], ej, -0.5);
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

// The flat tile index t runs over the tiles of all problems, tile_off[g] .. tile_off[g+1] - 1 being problem g's, so the
// grid stays one-dimensional and capped for any G and M_g.
__global__ void __launch_bounds__(256) link_score_kernel(LinkWs w, LinkProblems p, const float *__restrict__ Phi,
                                                         const int32_t *__restrict__ spk_rec, int R,
                                                         double *__restrict__ dist_out) {
    for (int64_t t = blockIdx.x; t < p.tile_off[p.G]; t += gridDim.x) {
        const int g = find_problem(p.tile_off, p.G, t);
        const int64_t base = p.off[g], M = p.off[g + 1] - base, lt = t - p.tile_off[g];
        LinkWs wg = w;
        wg.lk += p.lk_off[g];
        wg.s.n += base;
        wg.s.e += base;
        wg.s.b += base * kMaxR;
        double *dist = dist_out ? dist_out + p.dist_off[g] : nullptr;
        const int64_t tiles = (M + 31) / 32;
        const double tt = 2.0 * (double)tiles + 1.0;
        auto row0 = [tiles](int64_t b) { return b * tiles - b * (b - 1) / 2; };   // first tile of row b
        int64_t bi = (int64_t)((tt - sqrt(tt * tt - 8.0 * (double)lt)) / 2.0);   // row0 inverted, then rounding corrected
        while (bi > 0 && row0(bi) > lt) --bi;
        while (bi + 1 < tiles && row0(bi + 1) <= lt) ++bi;
        score_tile(wg, Phi, spk_rec + base, M, R, p.c[g], dist, bi, bi + (lt - row0(bi)));
    }
}

}  // namespace

size_t link_batch_workspace_bytes(int G, const int64_t *M_host, std::vector<int64_t> *lk_off) {
    size_t lk = 0, total = 0;
    int64_t M = 0;
    if (lk_off) lk_off->assign(G + 1, 0);
    for (int g = 0; g < G; ++g) {
        if (lk_off) (*lk_off)[g] = (int64_t)lk;
        lk += al(linkage_workspace_bytes(M_host[g]));
        M += M_host[g];
    }
    if (lk_off) (*lk_off)[G] = (int64_t)lk;
    link_layout(nullptr, lk, M, G, &total);
    return total;
}

namespace {

// The statistics (and, with n_tiles > 0 score tiles, the distances) of the problems p over the workspace w.
int launch_problems(const LinkWs &w, const LinkProblems &p, int64_t n_tiles, const float *fea, const float *Phi,
                    const int32_t *spk, int R, const int32_t *spk_rec, double *n_out, double *F_out, double *dist_out,
                    cudaStream_t st) {
    int launches = 2;
    link_init_kernel<<<(unsigned)((p.M + 255) / 256), 256, 0, st>>>(w, p);
    if (p.N > 0) {
        link_span_kernel<<<(unsigned)(((int64_t)p.G * p.N + 255) / 256), 256, 0, st>>>(w, p, spk);
        ++launches;
    }
    link_stats_kernel<<<(unsigned)p.M, kStatsThreads, 0, st>>>(w, p, fea, Phi, spk, R, n_out, F_out);
    if (n_tiles > 0) {
        link_score_kernel<<<(unsigned)std::min<int64_t>(n_tiles, kScoreGrid), 256, 0, st>>>(w, p, Phi, spk_rec, R,
                                                                                           dist_out);
        ++launches;
    }
    return launches;
}

}  // namespace

int launch_link_batch(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, const int32_t *spk_rec,
                      int G, const int64_t *M_host, const double *c_host, void *workspace, double *n_out,
                      double *F_out, double *dist_out, double *Z_out, cudaStream_t st, const double *mean,
                      const double *std) {
    std::vector<int64_t> lk_off;
    link_batch_workspace_bytes(G, M_host, &lk_off);
    // the problem arrays: off, lk_off, tile_off, dist_off [G+1] and c [G], uploaded in one copy
    std::vector<int64_t> host(5 * (size_t)G + 4, 0);
    int64_t *off = host.data(), *tile = off + 2 * (G + 1), *dist = off + 3 * (G + 1);
    bool linkage = false;
    for (int g = 0; g < G; ++g) {
        off[g + 1] = off[g] + M_host[g];
        tile[g + 1] = tile[g] + score_tiles(M_host[g]);
        dist[g + 1] = dist[g] + M_host[g] * M_host[g];
        linkage = linkage || M_host[g] >= 2;
    }
    std::copy(lk_off.begin(), lk_off.end(), host.begin() + (G + 1));
    std::memcpy(host.data() + 4 * (G + 1), c_host, (size_t)G * sizeof(double));
    const int64_t M = off[G];
    if (M == 0) return 0;
    const LinkWs w = link_layout(reinterpret_cast<uint8_t *>(workspace), (size_t)lk_off[G], M, G, nullptr);
    if (cudaMemcpyAsync(w.offs, host.data(), host.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return -1;
    LinkProblems p;
    p.G = G;
    p.M = M;
    p.N = N;
    p.off = w.offs;
    p.lk_off = w.offs + (G + 1);
    p.tile_off = w.offs + 2 * (G + 1);
    p.dist_off = w.offs + 3 * (G + 1);
    p.c = reinterpret_cast<const double *>(w.offs + 4 * (G + 1));
    int launches = launch_problems(w, p, tile[G], fea, Phi, spk, R, spk_rec, n_out, F_out, mean ? nullptr : dist_out,
                                   st);
    if (mean) {                                       // normalised distances (section 5.17): dist_out gets those
        const NormProblems q{G, p.off, p.dist_off, p.lk_off};
        const int ln = launch_norm_scores(reinterpret_cast<double *>(w.lk), dist[G], 1, mean, std, mean, std, true,
                                          kBig, dist_out, st, q);
        if (ln < 0) return -1;
        launches += ln;
    }
    if (linkage) {
        launch_linkage(p.off, p.lk_off, G, w.lk, Z_out, st);
        ++launches;
    }
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

int launch_speaker_stats_batch(const float *fea, const float *Phi, const int32_t *spk, int64_t N, int R, int G,
                               const int64_t *off, const double *c, int64_t M, const SpeakerStats &s, double *n_out,
                               double *F_out, cudaStream_t st) {
    if (M == 0) return 0;
    const LinkWs w{nullptr, s, nullptr};
    LinkProblems p;
    p.G = G;
    p.M = M;
    p.N = N;
    p.off = off;
    p.lk_off = p.tile_off = p.dist_off = nullptr;
    p.c = c;
    const int launches = launch_problems(w, p, 0, fea, Phi, spk, R, nullptr, n_out, F_out, nullptr, st);
    return cudaGetLastError() == cudaSuccess ? launches : -1;
}

}  // namespace vbx
