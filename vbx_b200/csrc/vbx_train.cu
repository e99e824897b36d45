// Class statistics of labelled x-vectors for back-end training (include/vbx_b200.h vbx_class_scatter, DESIGN.md
// section 5.24): the float64 class means and the within-class scatter sum_rows (x - m_class)(x - m_class)^T of a float32
// [N, D] array whose rows are packed by class.
//
//   train_row_class_kernel  one thread per row: its class, by binary search on the offsets (the scatter kernel reads it
//                           for every tile pair, so it is found once)
//   train_class_mean_kernel one CTA per (class, 32 columns): 8 row phases summed in row order, then in phase order
//   train_scatter_kernel    one CTA per (row split, 64 x 64 output tile on or above the diagonal): 32-row chunks
//                           centred by their class mean in float64 into shared memory, then 4 warps of 32 x 32 outputs
//                           on the FP64 tensor cores (mma.sync m8n8k4 f64, DMMA.8x8x4), the partial tile to the
//                           workspace
//   train_scatter_sum_kernel one thread per element of the upper tiles: the splits' partials in split order, written to
//                           both triangles (the mirror is the same double)
//
// Rows are centred before the products: S = G - n m m^T would cancel catastrophically on uncentred x-vectors.  The split
// count depends on N and D only and every sum has a fixed order, so a call is bit-identical from run to run whatever the
// device and whatever the workspace held.
#include <algorithm>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kTile = 64;                 // output tile edge
constexpr int kRows = 32;                 // rows per shared-memory chunk
constexpr int kPitch = kTile + 8;         // doubles per shared row: the 8 x 4 fragment loads take the minimum 2 wavefronts
constexpr int kThreads = 128;             // 4 warps, 2 x 2 of 32 x 32 outputs
constexpr int kTargetCtas = 1024;         // tile pairs x splits aimed at (several waves on 132 SMs)

__host__ __device__ size_t al(size_t v) { return (v + 255) & ~(size_t)255; }

int64_t tile_count(int D) { return (D + kTile - 1) / kTile; }
int64_t pair_count(int D) { const int64_t T = tile_count(D); return T * (T + 1) / 2; }

// Rows per split, a multiple of kRows; the splits = ceil(N / rows) then cover [0, N) in order.
int64_t split_rows(int64_t N, int D) {
    const int64_t want = std::max<int64_t>(1, (kTargetCtas + pair_count(D) - 1) / pair_count(D));
    const int64_t rows = (N + want - 1) / want;
    return std::max<int64_t>(kRows, (rows + kRows - 1) / kRows * kRows);
}
int64_t split_count(int64_t N, int D) { return std::max<int64_t>(1, (N + split_rows(N, D) - 1) / split_rows(N, D)); }

struct ScatterWs {
    int64_t *offsets;   // [K + 1]
    int32_t *cls;       // [N]
    double *partial;    // [splits, pairs, 64, 64]
};

ScatterWs scatter_layout(uint8_t *ws, int64_t N, int D, int64_t K, size_t *total) {
    ScatterWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.offsets = reinterpret_cast<int64_t *>(take((size_t)(K + 1) * 8));
    w.cls = reinterpret_cast<int32_t *>(take((size_t)N * 4));
    w.partial = reinterpret_cast<double *>(take((size_t)split_count(N, D) * pair_count(D) * kTile * kTile * 8));
    if (total) *total = o;
    return w;
}

__global__ void __launch_bounds__(256) train_row_class_kernel(const int64_t *__restrict__ off, int64_t K, int64_t N,
                                                              int32_t *__restrict__ cls) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    int64_t lo = 0, hi = K;                      // the class c with off[c] <= r < off[c + 1] (empty classes skipped)
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= r) lo = mid; else hi = mid;
    }
    cls[r] = (int32_t)lo;
}

__global__ void __launch_bounds__(256) train_class_mean_kernel(const float *__restrict__ X, int D,
                                                               const int64_t *__restrict__ off,
                                                               double *__restrict__ means) {
    __shared__ double part[8][33];
    const int64_t c = blockIdx.x;
    const int col = blockIdx.y * 32 + threadIdx.x;
    const int64_t lo = off[c], hi = off[c + 1];
    double s = 0.0;
    if (col < D)
        for (int64_t r = lo + threadIdx.y; r < hi; r += 8) s += (double)X[r * D + col];
    part[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && col < D) {
        double t = 0.0;
        for (int q = 0; q < 8; ++q) t += part[q][threadIdx.x];
        means[c * D + col] = hi > lo ? t / (double)(hi - lo) : 0.0;
    }
}

__device__ __forceinline__ void dmma_884(double (&d)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

// The centred rows [r0, r0 + kRows) of columns [c0, c0 + 64) into s (zero past N, past `end` and past D).
__device__ __forceinline__ void load_centred(double (*s)[kPitch], const float *__restrict__ X, int D,
                                             const int32_t *__restrict__ cls, const double *__restrict__ means,
                                             int64_t r0, int64_t end, int c0) {
    const int col = threadIdx.x & (kTile - 1), c = c0 + col;
    for (int q = threadIdx.x >> 6; q < kRows; q += kThreads / kTile) {
        const int64_t r = r0 + q;
        double v = 0.0;
        if (r < end && c < D) v = (double)X[r * D + c] - means[(int64_t)cls[r] * D + c];
        s[q][col] = v;
    }
}

__global__ void __launch_bounds__(kThreads) train_scatter_kernel(const float *__restrict__ X, int64_t N, int D,
                                                                 const int32_t *__restrict__ cls,
                                                                 const double *__restrict__ means, int64_t rows_per,
                                                                 int64_t n_pairs, double *__restrict__ partial) {
    __shared__ __align__(16) double sa[kRows][kPitch];
    __shared__ __align__(16) double sb[kRows][kPitch];
    const int64_t p = blockIdx.x, split = blockIdx.y;
    int bi = 0, rem = (int)p, T = (D + kTile - 1) / kTile;
    while (rem >= T - bi) { rem -= T - bi; ++bi; }     // pair p = (bi, bj), bi <= bj, row-major over the upper tiles
    const int bj = bi + rem;
    const bool diag = bi == bj;
    const int64_t begin = split * rows_per, end = min(N, begin + rows_per);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    double acc[4][4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    double (*sbp)[kPitch] = diag ? sa : sb;
    for (int64_t r0 = begin; r0 < end; r0 += kRows) {
        __syncthreads();                                  // the previous chunk's fragments are read
        load_centred(sa, X, D, cls, means, r0, end, bi * kTile);
        if (!diag) load_centred(sb, X, D, cls, means, r0, end, bj * kTile);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kRows; k += 4) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = sa[k + t][wm + 8 * i + g];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = sbp[k + t][wn + 8 * j + g];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dmma_884(acc[i][j], a[i], b[j]);
        }
    }
    double *out = partial + (split * n_pairs + p) * (kTile * kTile);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<double2 *>(out + (wm + 8 * i + g) * kTile + wn + 8 * j + 2 * t) =
                make_double2(acc[i][j][0], acc[i][j][1]);
}

__global__ void __launch_bounds__(256) train_scatter_sum_kernel(const double *__restrict__ partial, int64_t n_split,
                                                                int64_t n_pairs, int D, double *__restrict__ S) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_pairs * kTile * kTile) return;
    const int64_t p = e / (kTile * kTile);
    const int a = (int)(e % (kTile * kTile)) / kTile, b = (int)(e % kTile);
    int bi = 0, rem = (int)p, T = (D + kTile - 1) / kTile;
    while (rem >= T - bi) { rem -= T - bi; ++bi; }
    const int bj = bi + rem;
    const int i = bi * kTile + a, j = bj * kTile + b;
    if (i >= D || j >= D || (bi == bj && a > b)) return;   // a diagonal tile's lower half is its upper half's mirror
    double s = 0.0;
    for (int64_t q = 0; q < n_split; ++q) s += partial[(q * n_pairs + p) * (kTile * kTile) + a * kTile + b];
    S[(int64_t)i * D + j] = s;
    S[(int64_t)j * D + i] = s;
}

}  // namespace

size_t class_scatter_workspace_bytes(int64_t N, int D, int64_t K) {
    size_t total = 0;
    scatter_layout(nullptr, N, D, K, &total);
    return total;
}

int launch_class_scatter(const float *X, int64_t N, int D, int64_t K, const int64_t *offsets_host, void *workspace,
                         double *means_out, double *scatter_out, cudaStream_t st) {
    const ScatterWs w = scatter_layout(reinterpret_cast<uint8_t *>(workspace), N, D, K, nullptr);
    if (cudaMemcpyAsync(w.offsets, offsets_host, (size_t)(K + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st) !=
        cudaSuccess)
        return -1;
    int n = 0;
    if (N > 0) {
        train_row_class_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(w.offsets, K, N, w.cls);
        ++n;
    }
    train_class_mean_kernel<<<dim3((unsigned)K, (unsigned)((D + 31) / 32)), dim3(32, 8), 0, st>>>(X, D, w.offsets,
                                                                                                  means_out);
    const int64_t pairs = pair_count(D), splits = split_count(N, D);
    train_scatter_kernel<<<dim3((unsigned)pairs, (unsigned)splits), kThreads, 0, st>>>(X, N, D, w.cls, means_out,
                                                                                       split_rows(N, D), pairs,
                                                                                       w.partial);
    const int64_t elems = pairs * kTile * kTile;
    train_scatter_sum_kernel<<<(unsigned)((elems + 255) / 256), 256, 0, st>>>(w.partial, splits, pairs, D,
                                                                              scatter_out);
    return cudaGetLastError() == cudaSuccess ? n + 3 : -1;
}

}  // namespace vbx
