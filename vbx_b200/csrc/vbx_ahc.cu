// AHC initialisation on the device (SURVEY.md 8f.3): the step that gives VBx() its `gamma` init and speaker count.
//   VBx/vbhmm.py:135      scr_mx = cos_similarity(x)                  (VBx/diarization_lib.py:190-213)
//   VBx/vbhmm.py:137      thr, _ = twoGMMcalib_lin(scr_mx.ravel())    (VBx/diarization_lib.py:13-31)
//   VBx/vbhmm.py:139-141  average-linkage clustering of -scr_mx       (fastcluster.linkage(method='average'))
// Everything is float64, like the reference.  Per recording: the T x T matrix of NEGATED cosine similarities lives
// in the caller's workspace (the clustering works on distances d = -similarity, the calibration on s = -d).
// The linkage comes back in the scipy / fastcluster layout Z [T-1, 4]; cutting it at -(thr + bias)
// (VBx/vbhmm.py:144-146) is an O(T) traversal done by the host mirror (vbx_b200/ahc.py).
//
// Kernels
//   ahc_cosine_kernel    32 x 32 output tile per CTA, rows normalised on the fly, DFMA over the feature dimension.
//   ahc_gmm_*            two-Gaussian shared-variance EM on all T^2 scores: one accumulation launch (64 chunks per
//                        recording, fixed-order reduction => deterministic) + one parameter update per iteration.
//   ahc_linkage_kernel   one 1024-thread CTA per recording.  Nearest-neighbour arrays (nn, nnd) make one merge
//                        O(T) work: block argmin over nnd, Lance-Williams update of one row/column, and a warp-per-row
//                        recomputation of the few rows whose nearest neighbour was merged away.
#include <cfloat>
#include <climits>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kGmmChunks = 64;
constexpr int kGmmIters = 20;        // twoGMMcalib_lin(niters=20)
constexpr int kLinkThreads = 1024;

struct AhcRec {                      // carved out of the workspace for each recording
    double *D;                       // [T,T]  negated cosine similarity / current cluster distances
    double *nnd;                     // [T]    distance to the nearest active cluster
    int32_t *nn;                     // [T]    its slot
    int32_t *cid;                    // [T]    scipy cluster id held by the slot (leaf i, or T + merge index)
    int32_t *csize;                  // [T]
    int32_t *todo;                   // [T]    slots whose nearest neighbour must be recomputed
    uint8_t *alive;                  // [T]
};

__device__ __forceinline__ AhcRec carve(const int64_t *offsets, const int64_t *d_off, uint8_t *ws, int rec, int &T) {
    T = (int)(offsets[rec + 1] - offsets[rec]);
    AhcRec r;
    uint8_t *p = ws + d_off[rec];
    r.D = reinterpret_cast<double *>(p);
    p += (size_t)T * T * 8;
    r.nnd = reinterpret_cast<double *>(p);
    p += (size_t)T * 8;
    r.nn = reinterpret_cast<int32_t *>(p);
    p += (size_t)T * 4;
    r.cid = reinterpret_cast<int32_t *>(p);
    p += (size_t)T * 4;
    r.csize = reinterpret_cast<int32_t *>(p);
    p += (size_t)T * 4;
    r.todo = reinterpret_cast<int32_t *>(p);
    p += (size_t)T * 4;
    r.alive = p;
    return r;
}

// ---- cosine similarity (negated) --------------------------------------------------------------------------
template <typename XT>
__global__ void __launch_bounds__(256) ahc_cosine_kernel(const int64_t *__restrict__ offsets, const int64_t *__restrict__ d_off,
                                                         uint8_t *ws, const XT *__restrict__ x, int dim) {
    const int rec = blockIdx.z;
    int T;
    const AhcRec r = carve(offsets, d_off, ws, rec, T);
    const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
    if (i0 >= T || j0 >= T) return;
    __shared__ double a[32][33], b[32][33], na[32], nb[32];
    const XT *xr = x + offsets[rec] * dim;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8 threads, 4 outputs each
    double acc[4] = {0, 0, 0, 0};
    double sa = 0, sb = 0;                                        // row norms, accumulated by ty == 0 / ty == 1
    for (int k0 = 0; k0 < dim; k0 += 32) {
        for (int q = ty; q < 32; q += 8) {
            const int k = k0 + tx;
            a[q][tx] = (i0 + q < T && k < dim) ? (double)xr[(int64_t)(i0 + q) * dim + k] : 0.0;
            b[q][tx] = (j0 + q < T && k < dim) ? (double)xr[(int64_t)(j0 + q) * dim + k] : 0.0;
        }
        __syncthreads();
        if (ty == 0)
            for (int k = 0; k < 32; ++k) sa += a[tx][k] * a[tx][k];
        if (ty == 1)
            for (int k = 0; k < 32; ++k) sb += b[tx][k] * b[tx][k];
#pragma unroll 8
        for (int k = 0; k < 32; ++k) {
            const double bv = b[tx][k];
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] += a[ty + 8 * q][k] * bv;
        }
        __syncthreads();
    }
    if (ty == 0) na[tx] = sqrt(sa) + 1.0e-32;                    // x / (sqrt(sum x^2) + 1e-32), diarization_lib.py:201
    if (ty == 1) nb[tx] = sqrt(sb) + 1.0e-32;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int i = i0 + ty + 8 * q, j = j0 + tx;
        if (i < T && j < T) r.D[(int64_t)i * T + j] = -(acc[q] / (na[ty + 8 * q] * nb[tx]));
    }
}

// ---- two-Gaussian calibration ------------------------------------------------------------------------------
// params[rec][8] = {w0, w1, m0, m1, var, thr, -, -};  partial[rec][chunk][6]
__device__ __forceinline__ double block_sum(double v, double *red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    double t = 0;
    for (int i = 0; i < nw; ++i) t += red[i];                   // fixed order
    return t;
}

__global__ void __launch_bounds__(256) ahc_gmm_accum_kernel(const int64_t *__restrict__ offsets, const int64_t *__restrict__ d_off,
                                                            uint8_t *ws, const double *__restrict__ params,
                                                            double *__restrict__ partial, int first) {
    const int rec = blockIdx.y, chunk = blockIdx.x;
    int T;
    const AhcRec r = carve(offsets, d_off, ws, rec, T);
    __shared__ double red[8];
    const int64_t n = (int64_t)T * T;
    const int64_t L = (n + kGmmChunks - 1) / kGmmChunks;
    const int64_t e0 = chunk * L, e1 = min(n, e0 + L);
    double s[6] = {0, 0, 0, 0, 0, 0};
    if (first) {                                                // moments for the initial parameters
        for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
            const double v = -r.D[e];
            s[0] += v;
            s[1] += v * v;
        }
    } else {
        const double *p = params + rec * 8;
        const double lw0 = log(p[0]), lw1 = log(p[1]), m0 = p[2], m1 = p[3], var = p[4];
        const double c = -0.5 * log(var), hv = 0.5 / var;
        for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
            const double v = -r.D[e];
            const double l0 = lw0 + c - (v - m0) * (v - m0) * hv;        // diarization_lib.py:24
            const double l1 = lw1 + c - (v - m1) * (v - m1) * hv;
            const double mx = fmax(l0, l1);
            const double e0x = exp(l0 - mx), e1x = exp(l1 - mx);
            const double g0 = e0x / (e0x + e1x), g1 = e1x / (e0x + e1x);  // softmax(lls, axis=1)
            s[0] += g0;
            s[1] += g1;
            s[2] += v * g0;
            s[3] += v * g1;
            s[4] += v * v * g0;
            s[5] += v * v * g1;
        }
    }
    for (int q = 0; q < 6; ++q) {
        const double t = block_sum(s[q], red);
        if (threadIdx.x == 0) partial[((int64_t)rec * kGmmChunks + chunk) * 6 + q] = t;
    }
}

__global__ void ahc_gmm_update_kernel(const int64_t *__restrict__ offsets, double *__restrict__ params,
                                      const double *__restrict__ partial, int first, int n_rec, double *__restrict__ thr_out) {
    const int rec = blockIdx.x * blockDim.x + threadIdx.x;
    if (rec >= n_rec) return;
    const double T = (double)(offsets[rec + 1] - offsets[rec]);
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (int c = 0; c < kGmmChunks; ++c)
        for (int q = 0; q < 6; ++q) s[q] += partial[((int64_t)rec * kGmmChunks + c) * 6 + q];
    double *p = params + rec * 8;
    if (first) {                                                // diarization_lib.py:19-22
        const double n = T * T, mean = s[0] / n, var = s[1] / n - mean * mean, sd = sqrt(var);
        p[0] = 0.5;
        p[1] = 0.5;
        p[2] = mean - sd;
        p[3] = mean + sd;
        p[4] = var;
        p[5] = INFINITY;
    } else {                                                    // diarization_lib.py:26-30
        const double c0 = s[0], c1 = s[1];
        const double w0 = c0 / (c0 + c1), w1 = c1 / (c0 + c1);
        const double m0 = s[2] / c0, m1 = s[3] / c1;
        const double var = (s[4] / c0 - m0 * m0) * w0 + (s[5] / c1 - m1 * m1) * w1;
        const double num = (log(w0 * w0 / var) - m0 * m0 / var) - (log(w1 * w1 / var) - m1 * m1 / var);
        const double den = m0 / var - m1 / var;
        p[0] = w0;
        p[1] = w1;
        p[2] = m0;
        p[3] = m1;
        p[4] = var;
        p[5] = -0.5 * num / den;
    }
    if (thr_out) thr_out[rec] = p[5];
}

// ---- average linkage ------------------------------------------------------------------------------------------
struct MinPair {
    double d;
    int i;
};
__device__ __forceinline__ MinPair min_pair(MinPair a, MinPair b) { return (b.d < a.d || (b.d == a.d && b.i < a.i)) ? b : a; }
__device__ __forceinline__ MinPair warp_min(MinPair v) {
    for (int o = 16; o; o >>= 1) {
        MinPair w;
        w.d = __shfl_xor_sync(0xffffffffu, v.d, o);
        w.i = __shfl_xor_sync(0xffffffffu, v.i, o);
        v = min_pair(v, w);
    }
    return v;
}
// nearest active neighbour of slot `row` (warp-wide; lanes stride the row, ties -> lowest slot)
__device__ __forceinline__ void recompute_row(const AhcRec &r, int T, int row, int lane) {
    MinPair best{DBL_MAX, INT_MAX};
    const double *d = r.D + (int64_t)row * T;
    for (int k = lane; k < T; k += 32)
        if (k != row && r.alive[k]) best = min_pair(best, MinPair{d[k], k});
    best = warp_min(best);
    if (lane == 0) {
        r.nn[row] = best.i;
        r.nnd[row] = best.d;
    }
}

__global__ void __launch_bounds__(kLinkThreads) ahc_linkage_kernel(const int64_t *__restrict__ offsets,
                                                                   const int64_t *__restrict__ d_off, uint8_t *ws,
                                                                   double *__restrict__ Z_out) {
    const int rec = blockIdx.x;
    int T;
    const AhcRec r = carve(offsets, d_off, ws, rec, T);
    if (T < 2) return;
    double *Z = Z_out + offsets[rec] * 4;                      // T_b - 1 of the recording's T_b rows are used
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, n_warps = kLinkThreads / 32;
    __shared__ MinPair s_red[kLinkThreads / 32];
    __shared__ MinPair s_best;
    __shared__ int s_todo;

    for (int i = tid; i < T; i += kLinkThreads) {
        r.alive[i] = 1;
        r.cid[i] = i;
        r.csize[i] = 1;
    }
    __syncthreads();
    for (int row = warp; row < T; row += n_warps) recompute_row(r, T, row, lane);
    __syncthreads();

    for (int step = 0; step < T - 1; ++step) {
        // 1. the closest pair of clusters
        MinPair best{DBL_MAX, INT_MAX};
        for (int i = tid; i < T; i += kLinkThreads)
            if (r.alive[i]) best = min_pair(best, MinPair{r.nnd[i], i});
        best = warp_min(best);
        if (lane == 0) s_red[warp] = best;
        __syncthreads();
        if (warp == 0) {
            MinPair v = lane < n_warps ? s_red[lane] : MinPair{DBL_MAX, INT_MAX};
            v = warp_min(v);
            if (lane == 0) {
                s_best = v;
                s_todo = 0;
            }
        }
        __syncthreads();
        if (s_best.i == INT_MAX || !(s_best.d < DBL_MAX)) {
            // no finite distance left (NaN x-vectors): there is nothing to merge by; mark the rest of the linkage and stop
            for (int k = step * 4 + tid; k < (T - 1) * 4; k += kLinkThreads) Z[k] = nan("");
            return;                                               // block-uniform: s_best lives in shared memory
        }
        const int p = s_best.i, q = r.nn[p];
        const int a = min(p, q), b = max(p, q);                  // slot a keeps the merged cluster, slot b dies
        const double dist = s_best.d;
        const int na = r.csize[a], nb = r.csize[b];
        const double wa = (double)na / (double)(na + nb), wb = (double)nb / (double)(na + nb);
        __syncthreads();                                          // everyone has read nn[p], csize before they change
        // 2. Lance-Williams update of row / column a, collect the slots that lost their nearest neighbour
        double *da = r.D + (int64_t)a * T;
        const double *db = r.D + (int64_t)b * T;
        for (int k = tid; k < T; k += kLinkThreads) {
            if (!r.alive[k] || k == a || k == b) continue;
            const double dn = wa * da[k] + wb * db[k];
            da[k] = dn;
            r.D[(int64_t)k * T + a] = dn;
            const int nk = r.nn[k];
            if (nk == a || nk == b) {
                r.todo[atomicAdd(&s_todo, 1)] = k;
            } else if (dn < r.nnd[k]) {
                r.nn[k] = a;
                r.nnd[k] = dn;
            }
        }
        if (tid == 0) {
            const int ca = r.cid[a], cb = r.cid[b];
            Z[step * 4 + 0] = (double)min(ca, cb);
            Z[step * 4 + 1] = (double)max(ca, cb);
            Z[step * 4 + 2] = dist;
            Z[step * 4 + 3] = (double)(na + nb);
            r.alive[b] = 0;
            r.cid[a] = T + step;
            r.csize[a] = na + nb;
        }
        __syncthreads();
        // 3. nearest neighbours of the merged cluster and of the slots that pointed at a or b
        const int n_todo = s_todo;
        if (step < T - 2) {
            for (int w = warp; w <= n_todo; w += n_warps) recompute_row(r, T, w == n_todo ? a : r.todo[w], lane);
        }
        __syncthreads();
    }
}

}  // namespace

size_t ahc_workspace_bytes(const int64_t *offsets_host, int n_rec, std::vector<int64_t> *d_off_host) {
    size_t total = 0;
    if (d_off_host) d_off_host->assign(n_rec + 1, 0);
    for (int b = 0; b < n_rec; ++b) {
        const size_t T = (size_t)(offsets_host[b + 1] - offsets_host[b]);
        if (d_off_host) (*d_off_host)[b] = (int64_t)total;
        size_t bytes = T * T * 8 + T * (8 + 4 + 4 + 4 + 4) + T;
        total += (bytes + 255) & ~(size_t)255;
    }
    if (d_off_host) (*d_off_host)[n_rec] = (int64_t)total;
    // + per-recording offsets, GMM parameters and partial sums
    total += ((size_t)(n_rec + 1) * 8 + 255) & ~(size_t)255;
    total += ((size_t)n_rec * 8 * 8 + 255) & ~(size_t)255;
    total += ((size_t)n_rec * kGmmChunks * 6 * 8 + 255) & ~(size_t)255;
    return total;
}

// d_off (filled by ahc_workspace_bytes) must stay alive until the copy below has been staged: the caller owns it.
int launch_ahc(const Plan &pl, const std::vector<int64_t> &d_off, const void *x, int x_is_f64, int dim, void *workspace,
               size_t workspace_bytes, double *Z_out, double *thr_out, cudaStream_t st, std::string *err) {
    if (pl.n_rec == 0) return 0;
    if ((int)d_off.size() != pl.n_rec + 1) {
        if (err) *err = "AHC: workspace layout missing";
        return -1;
    }
    if (pl.n_rec > 65535) {
        if (err) *err = "AHC: more than 65535 recordings per call";
        return -1;
    }
    const int64_t max_T = pl.max_T;
    {
        size_t need = (size_t)d_off[pl.n_rec];
        need += ((size_t)(pl.n_rec + 1) * 8 + 255) & ~(size_t)255;
        need += ((size_t)pl.n_rec * 8 * 8 + 255) & ~(size_t)255;
        need += ((size_t)pl.n_rec * kGmmChunks * 6 * 8 + 255) & ~(size_t)255;
        if (workspace_bytes < need) {
            if (err) *err = "AHC workspace too small";
            return -1;
        }
    }
    uint8_t *ws = reinterpret_cast<uint8_t *>(workspace);
    size_t tail = (size_t)d_off[pl.n_rec];
    int64_t *d_off_dev = reinterpret_cast<int64_t *>(ws + tail);
    tail += ((size_t)(pl.n_rec + 1) * 8 + 255) & ~(size_t)255;
    double *params = reinterpret_cast<double *>(ws + tail);
    tail += ((size_t)pl.n_rec * 8 * 8 + 255) & ~(size_t)255;
    double *partial = reinterpret_cast<double *>(ws + tail);
    if (cudaMemcpyAsync(d_off_dev, d_off.data(), (size_t)(pl.n_rec + 1) * 8, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        if (err) *err = "AHC: copying the workspace offsets failed";
        return -1;
    }
    int launches = 0;
    const int tiles = (int)((max_T + 31) / 32);
    if (tiles > 0) {
        const dim3 grid(tiles, tiles, pl.n_rec);             // blockIdx.z carries the recording
        if (x_is_f64)
            ahc_cosine_kernel<double><<<grid, 256, 0, st>>>(pl.offsets, d_off_dev, ws, reinterpret_cast<const double *>(x), dim);
        else
            ahc_cosine_kernel<float><<<grid, 256, 0, st>>>(pl.offsets, d_off_dev, ws, reinterpret_cast<const float *>(x), dim);
        ++launches;
    }
    const dim3 ggrid(kGmmChunks, pl.n_rec);
    for (int it = 0; it <= kGmmIters; ++it) {
        ahc_gmm_accum_kernel<<<ggrid, 256, 0, st>>>(pl.offsets, d_off_dev, ws, params, partial, it == 0);
        ahc_gmm_update_kernel<<<(pl.n_rec + 127) / 128, 128, 0, st>>>(pl.offsets, params, partial, it == 0, pl.n_rec, thr_out);
        launches += 2;
    }
    ahc_linkage_kernel<<<pl.n_rec, kLinkThreads, 0, st>>>(pl.offsets, d_off_dev, ws, Z_out);
    ++launches;
    if (cudaGetLastError() != cudaSuccess) {
        if (err) *err = "AHC kernel launch failed";
        return -1;
    }
    return launches;
}

size_t linkage_workspace_bytes(int64_t T) { return (size_t)T * T * 8 + (size_t)T * (8 + 4 + 4 + 4 + 4) + (size_t)T; }

void launch_linkage(const int64_t *offsets, const int64_t *d_off, int n, void *ws, double *Z_out, cudaStream_t st) {
    ahc_linkage_kernel<<<n, kLinkThreads, 0, st>>>(offsets, d_off, reinterpret_cast<uint8_t *>(ws), Z_out);
}

}  // namespace vbx
