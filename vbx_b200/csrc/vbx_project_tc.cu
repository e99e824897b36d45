// Projection  rho[N,128] = X[N,D] . V[D,128]  on the Hopper tensor cores (wgmma, sm_90a), in split-precision 3xTF32
// (x_lo*v_hi + x_hi*v_lo + x_hi*v_hi, fp32 accumulation in registers) because plain TF32 breaks the 1e-4 parity bar of
// the EM loop (SURVEY.md section 7, hard part 4).
// Reference: the caller-side projection VBx/vbhmm.py:129,153 folded with the scale VBx/VBx.py:88-89 (SURVEY 8d).
//
// The same kernel, templated on MODE, also runs the real-data front end (x-vector transform and PLDA projection,
// VBx/vbhmm.py:125-129,153; launch_xvector_chain_wgmma below).
//
// One persistent CTA per SM, 12 warps, tiles of 256 frames:
//   warps 0-7   two consumer warpgroups, 128 frames each as two wgmma M=64 row sets.  Each thread ld.shared's its A
//               fragments from the raw fp32 X block, splits them into TF32 parts in registers and issues
//               wgmma.mma_async m64n128k8 tf32 with A from registers and B (V) by shared-memory descriptor, into
//               2 x 64 fp32 accumulator registers (4 k-steps x NS(NS+1)/2 split terms x 2 row sets per 32-column block).
//               One commit group per k-step; a stage is released to the producer when its last group has retired.
//               The epilogue works on the register accumulators: the per-frame constant G_t (quad shuffles) and
//               float2 stores of rho.
//   warps 8-11  producer: one thread issues, per 32-column block, the TMA tile copy of the raw 256-frame x 32-column X
//               block (128-byte swizzle; rows past N are zero-filled by the copy and never stored) and the bulk-async
//               copy (cp.async.bulk) of the pre-split V images, both completing on the stage's full barrier.
// Shared memory: NS = 2: 3 stages x (X 32 KB + V hi/lo 32 KB) = 192 KB; NS = 3: 2 stages x (X 32 KB + V 48 KB).
// X is read from shared memory once (by the thread whose fragment it is) and V once per wgmma M=64 row set, so the 256-frame
// tile halves the V bytes streamed from L2 per frame against a 128-frame tile.
//
// NS = 3 (the real-data front end): operands are split three ways, x = x1 + x2 + x3 exactly (3 x 11 mantissa bits), and
// six products are accumulated (x3 v1, x1 v3, x2 v2, x2 v1, x1 v2, x1 v1): the dropped terms are below 2^-33, i.e. the
// GEMM is at fp32-accumulate accuracy.  The shipped LDA matrix is badly conditioned (sum |a_k lda_kn| ~ 1e3 |sum|), so
// the 2^-21 relative error per product of the two-way split is visible on real data.
#include <cuda.h>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kTileM = 256;                 // frames per CTA tile: two warpgroups x two wgmma M=64 row sets
constexpr int kKB = 32;                     // columns of X per pipeline block (= one 128-byte swizzle row)
constexpr int kVBytes = 128 * 128;          // one image of V^T: 128 rows x 128 bytes
constexpr int kXBytes = kTileM * 128;       // the raw fp32 X block of a tile: 256 rows x 128 bytes
constexpr int kConsumerThreads = 256;       // two warpgroups
constexpr int kThreads = kConsumerThreads + 128;  // + the producer warpgroup (one thread of it issues the copies)

template <int NS> struct Pipe {
    static constexpr int kStages = NS == 2 ? 3 : 2;
    static constexpr int kStageBytes = kXBytes + NS * kVBytes;   // raw X block, NS images of V^T
    // 1 KB alignment slack, stages, barriers (128 B), 1/Phi or e_off (512 B)
    static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + 128 + 512;
};

// TMA copy of the box at (column c0, row c1) of a 2-D tensor map into shared memory
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, dense 8-row groups (SBO = 1024 B, LBO unused = 1).
// Advancing along K inside the 128-byte swizzle row only adds to the start address (bits 0-13, in 16-byte units), so
// the consumers add small integers to one descriptor per stage.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    const uint32_t lo = ((smem_addr >> 4) & 0x3fffu) | (1u << 16);
    const uint32_t hi = (1024u >> 4) | (1u << 30);                 // SBO, layout type 1 = SWIZZLE_128B
    return ((uint64_t)hi << 32) | lo;
}
// D[64 x 128] (+)= A[registers, 64 x 8] * B[smem, 128 x 8]^T, tf32, fp32 accumulators in registers.  A fragment of the
// thread (warp w of the warpgroup, g = lane / 4, t = lane % 4): a0 = A[16w + g][t], a1 = A[16w + g + 8][t],
// a2 = A[16w + g][t + 4], a3 = A[16w + g + 8][t + 4].
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching the accumulators across the asynchronous MMAs
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void split_rn(const float x, float &hi, float &lo) {
    const uint32_t h = (__float_as_uint(x) + 0x1000u) & 0xffffe000u;
    hi = __uint_as_float(h);
    lo = __uint_as_float((__float_as_uint(x - hi) + 0x1000u) & 0xffffe000u);
}

// x = x1 + x2 + x3 exactly: 11 + 11 + <= 2 mantissa bits, each part a TF32 number
__device__ __forceinline__ void split3_rn(const float x, float &x1, float &x2, float &x3) {
    x1 = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
    const float r1 = x - x1;                                   // exact
    x2 = __uint_as_float((__float_as_uint(r1) + 0x1000u) & 0xffffe000u);
    x3 = r1 - x2;                                              // exact, fits TF32
}

// ---- setup: V [D,128] -> per 32-row block of V the swizzled K-major images of V^T, NS parts of 16 KB each ----
template <int NS>
__global__ void build_v_images_kernel(const float *__restrict__ V, int D, float *__restrict__ img) {
    const int kb = blockIdx.x;                       // k-block
    for (int i = threadIdx.x; i < 128 * 32; i += blockDim.x) {
        const int n = i >> 5, kk = i & 31;           // row n of V^T, column kk inside the block
        const float v = V[(int64_t)(kb * kKB + kk) * 128 + n];
        const int c = kk >> 2, e = kk & 3;
        const int off = n * 32 + (((c ^ (n & 7)) << 2) | e);   // float index inside the 16 KB image
        float *dst = img + (int64_t)kb * NS * 4096 + off;
        if (NS == 2) {
            float hi, lo;
            split_rn(v, hi, lo);
            dst[0] = hi;
            dst[4096] = lo;
        } else {
            float v1, v2, v3;
            split3_rn(v, v1, v2, v3);
            dst[0] = v1;
            dst[4096] = v2;
            dst[2 * 4096] = v3;
        }
    }
}

// MODE 0  rho = X . V, G_t from rho and Phi                                   (the projection of SURVEY 8d)
// MODE 2  rho = (X - a_off) . V, G_t as above                                  (PLDA stage, VBx/vbhmm.py:153)
// MODE 1  out = l2norm(l2norm(X - a_off) . V - e_off)                          (x-vector transform, VBx/vbhmm.py:125-129)
//         the consumers also accumulate ||x - a_off||^2 of their rows from the A fragments, summed over the quad
// xmap: TMA map of X [N rows, D columns] fp32, box 32 columns x kTileM rows, 128-byte swizzle.
// Registers are allocated per warpgroup: the CTA starts at 168 per thread (3 x 128 x 168 <= 64K), then the producer
// warpgroup gives up all but 40 and the consumers take 232, which the register-A wgmma pipeline needs without spills.
template <int MODE, int NS>
__global__ void __launch_bounds__(kThreads, 1)
project_wgmma_kernel(const __grid_constant__ CUtensorMap xmap, const float *__restrict__ vimg, float *__restrict__ rho,
                     int64_t N, int D, const float *__restrict__ Phi, float *__restrict__ gframe,
                     const float *__restrict__ a_off, const float *__restrict__ e_off) {
    constexpr int kStages = Pipe<NS>::kStages, kStageBytes = Pipe<NS>::kStageBytes;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // the stage buffers must be 1024-byte aligned (128-byte swizzle)
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + kStages * kStageBytes);
    float *s_inv_phi = reinterpret_cast<float *>(bars + 16);   // 128 floats: 1/Phi (MODE 0, 2) or e_off (MODE 1)
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t bar_base = smem_u32(bars);
    auto full = [&](int s) { return bar_base + 8u * s; };
    auto empty = [&](int s) { return bar_base + 8u * (kStages + s); };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_kb = D / kKB;
    const int64_t n_tiles = (N + kTileM - 1) / kTileM;

    if (tid < 128) s_inv_phi[tid] = MODE == 1 ? e_off[tid] : 1.f / Phi[tid];
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full(s), 1);
            mbar_init(empty(s), kConsumerThreads);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid >= kConsumerThreads) {
        // ======================= producer =======================
        // Blocks of this CTA in order: b -> (tile = blockIdx.x + (b / n_kb) * gridDim.x, kb = b % n_kb).
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (tid == kConsumerThreads) {
            const int64_t my_tiles = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
            const int64_t n_blocks = my_tiles * n_kb;
            for (int64_t b = 0; b < n_blocks; ++b) {
                const int s = (int)(b % kStages);
                const uint32_t ph = (uint32_t)((b / kStages) & 1);
                const int64_t tile = blockIdx.x + (b / n_kb) * gridDim.x;
                const int kb = (int)(b % n_kb);
                mbar_wait(empty(s), ph ^ 1);               // the consumers are done with this stage
                const uint32_t stage = smem_base + s * kStageBytes;
                mbar_expect_tx(full(s), kXBytes + NS * kVBytes);   // a box past the last row still counts in full
                tma_load_2d(stage, &xmap, kb * kKB, (int)(tile * kTileM), full(s));
                bulk_g2s(stage + kXBytes, vimg + (int64_t)kb * NS * 4096, NS * kVBytes, full(s));
            }
        }
    } else {
        // ======================= consumers: split, MMA, epilogue =======================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int wg = tid >> 7;                       // warpgroup: frames 128 wg .. 128 wg + 127 of the tile
        const int g = lane >> 2, t = lane & 3;
        const int rq = 16 * (warp & 3) + g;            // accumulator rows rq and rq + 8 of each 64-row set
        const int cq = 2 * t;                          // accumulator columns 8 j + cq, + 1
        // this thread's A elements inside a stage: row 128 wg + 64 m + rq (+ 8), column 8 ks + t (+ 4) of the
        // 128-byte swizzled block, i.e. 16-byte chunk (2 ks (+ 1)) ^ (row & 7) = (2 ks (+ 1)) ^ g, word t
        const float *a_rows = reinterpret_cast<const float *>(smem) + (128 * wg + rq) * 32 + t;
        float d0[64], d1[64];
        float ss[2][2];                                // MODE 1: ||x - a_off||^2 partial of rows (set m, +0 / +8)
        int s = 0, last = 0;
        uint32_t ph = 0;
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
#pragma unroll
            for (int m = 0; m < 2; ++m) ss[m][0] = ss[m][1] = 0.f;
            for (int kb = 0; kb < n_kb; ++kb) {
                float ao[8];                           // a_off of columns 8 ks + t, 8 ks + t + 4
#pragma unroll
                for (int i = 0; i < 8; ++i) ao[i] = MODE != 0 ? __ldg(a_off + kb * kKB + 4 * i + t) : 0.f;
                mbar_wait(full(s), ph);
                const float *xs = a_rows + s * (kStageBytes / 4);
                const uint64_t b0 = make_desc(smem_base + s * kStageBytes + kXBytes);
                constexpr uint64_t kImg = kVBytes >> 4;        // one V image, in 16-byte descriptor units
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const int o0 = ((2 * ks) ^ g) << 2, o1 = ((2 * ks + 1) ^ g) << 2;   // float offsets of the chunks
                    uint32_t p1[2][4], p2[2][4], p3[2][4];     // split parts (hi, lo[, lo2]) of the two row sets
#pragma unroll
                    for (int m = 0; m < 2; ++m) {
                        float x[4] = {xs[m * 64 * 32 + o0], xs[m * 64 * 32 + 8 * 32 + o0], xs[m * 64 * 32 + o1],
                                      xs[m * 64 * 32 + 8 * 32 + o1]};
                        if (MODE != 0) {
                            x[0] -= ao[2 * ks];
                            x[1] -= ao[2 * ks];
                            x[2] -= ao[2 * ks + 1];
                            x[3] -= ao[2 * ks + 1];
                        }
                        if (MODE == 1) {
                            ss[m][0] = fmaf(x[2], x[2], fmaf(x[0], x[0], ss[m][0]));
                            ss[m][1] = fmaf(x[3], x[3], fmaf(x[1], x[1], ss[m][1]));
                        }
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            float h, l, l2 = 0.f;
                            if (NS == 2) split_rn(x[j], h, l);
                            else split3_rn(x[j], h, l, l2);
                            p1[m][j] = __float_as_uint(h);
                            p2[m][j] = __float_as_uint(l);
                            p3[m][j] = __float_as_uint(l2);
                        }
                    }
                    const uint64_t k = ks * 2;             // 8 tf32 = 32 bytes inside the swizzle row (16-byte units)
                    const uint32_t first = (kb == 0 && ks == 0) ? 0u : 1u;
                    wgmma_fence();                         // the A registers were just written
                    if (NS == 2) {                         // lo*hi + hi*lo + hi*hi
                        wgmma_tf32(d0, p2[0], b0 + k, first);
                        wgmma_tf32(d0, p1[0], b0 + kImg + k, 1u);
                        wgmma_tf32(d0, p1[0], b0 + k, 1u);
                        wgmma_tf32(d1, p2[1], b0 + k, first);
                        wgmma_tf32(d1, p1[1], b0 + kImg + k, 1u);
                        wgmma_tf32(d1, p1[1], b0 + k, 1u);
                    } else {                               // smallest terms first: x3 v1, x1 v3, x2 v2, x2 v1, x1 v2, x1 v1
                        wgmma_tf32(d0, p3[0], b0 + k, first);
                        wgmma_tf32(d0, p1[0], b0 + 2 * kImg + k, 1u);
                        wgmma_tf32(d0, p2[0], b0 + kImg + k, 1u);
                        wgmma_tf32(d0, p2[0], b0 + k, 1u);
                        wgmma_tf32(d0, p1[0], b0 + kImg + k, 1u);
                        wgmma_tf32(d0, p1[0], b0 + k, 1u);
                        wgmma_tf32(d1, p3[1], b0 + k, first);
                        wgmma_tf32(d1, p1[1], b0 + 2 * kImg + k, 1u);
                        wgmma_tf32(d1, p2[1], b0 + kImg + k, 1u);
                        wgmma_tf32(d1, p2[1], b0 + k, 1u);
                        wgmma_tf32(d1, p1[1], b0 + kImg + k, 1u);
                        wgmma_tf32(d1, p1[1], b0 + k, 1u);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                       // the previous k-step's MMAs have retired
                    if (ks == 0 && kb > 0) mbar_arrive(empty(last));   // ... and with them the previous block's stage
                }
                last = s;
                if (++s == kStages) {
                    s = 0;
                    ph ^= 1;
                }
            }
            wgmma_wait<0>();
            fence_operands(d0);
            fence_operands(d1);
            mbar_arrive(empty(last));
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                float(&d)[64] = m == 0 ? d0 : d1;
                const int64_t ra = tile * kTileM + 128 * wg + 64 * m + rq, rb = ra + 8;
                float na = 0.f, nb = 0.f;
                if (MODE == 1) {
                    // y = acc / ||x - mean1|| - mean2 ; out = y / ||y||
                    float n1a = ss[m][0], n1b = ss[m][1];
                    n1a += __shfl_xor_sync(0xffffffffu, n1a, 1);
                    n1a += __shfl_xor_sync(0xffffffffu, n1a, 2);
                    n1b += __shfl_xor_sync(0xffffffffu, n1b, 1);
                    n1b += __shfl_xor_sync(0xffffffffu, n1b, 2);
                    const float ia = 1.f / sqrtf(n1a), ib = 1.f / sqrtf(n1b);
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const float2 e = *reinterpret_cast<const float2 *>(s_inv_phi + 8 * j + cq);
                        d[4 * j] = fmaf(d[4 * j], ia, -e.x);
                        d[4 * j + 1] = fmaf(d[4 * j + 1], ia, -e.y);
                        d[4 * j + 2] = fmaf(d[4 * j + 2], ib, -e.x);
                        d[4 * j + 3] = fmaf(d[4 * j + 3], ib, -e.y);
                        na = fmaf(d[4 * j], d[4 * j], fmaf(d[4 * j + 1], d[4 * j + 1], na));
                        nb = fmaf(d[4 * j + 2], d[4 * j + 2], fmaf(d[4 * j + 3], d[4 * j + 3], nb));
                    }
                    na += __shfl_xor_sync(0xffffffffu, na, 1);
                    na += __shfl_xor_sync(0xffffffffu, na, 2);
                    nb += __shfl_xor_sync(0xffffffffu, nb, 1);
                    nb += __shfl_xor_sync(0xffffffffu, nb, 2);
                    const float sa = 1.f / sqrtf(na), sb = 1.f / sqrtf(nb);
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (ra < N) *reinterpret_cast<float2 *>(rho + ra * 128 + 8 * j + cq) = make_float2(d[4 * j] * sa, d[4 * j + 1] * sa);
                        if (rb < N) *reinterpret_cast<float2 *>(rho + rb * 128 + 8 * j + cq) = make_float2(d[4 * j + 2] * sb, d[4 * j + 3] * sb);
                    }
                } else {
                    // ||fea||^2 = sum_r rho^2 / Phi_r   (VBx/VBx.py:87); a row's 128 columns are spread over a quad of lanes
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const float2 ip = *reinterpret_cast<const float2 *>(s_inv_phi + 8 * j + cq);
                        na = fmaf(d[4 * j] * d[4 * j], ip.x, fmaf(d[4 * j + 1] * d[4 * j + 1], ip.y, na));
                        nb = fmaf(d[4 * j + 2] * d[4 * j + 2], ip.x, fmaf(d[4 * j + 3] * d[4 * j + 3], ip.y, nb));
                        if (ra < N) *reinterpret_cast<float2 *>(rho + ra * 128 + 8 * j + cq) = make_float2(d[4 * j], d[4 * j + 1]);
                        if (rb < N) *reinterpret_cast<float2 *>(rho + rb * 128 + 8 * j + cq) = make_float2(d[4 * j + 2], d[4 * j + 3]);
                    }
                    na += __shfl_xor_sync(0xffffffffu, na, 1);
                    na += __shfl_xor_sync(0xffffffffu, na, 2);
                    nb += __shfl_xor_sync(0xffffffffu, nb, 1);
                    nb += __shfl_xor_sync(0xffffffffu, nb, 2);
                    if (t == 0) {                          // G_t, R = 128
                        if (ra < N) gframe[ra] = -0.5f * (na + 128.f * 1.8378770664093453f);
                        if (rb < N) gframe[rb] = -0.5f * (nb + 128.f * 1.8378770664093453f);
                    }
                }
            }
        }
    }
}

// V2[k,n] = tr[n,k] * sqrt(psi[n]): the PLDA projection (x - mu) . tr^T (VBx/vbhmm.py:153) folded with the
// scale rho = fea * sqrt(Phi) (VBx/VBx.py:89)
__global__ void build_plda_v_kernel(const float *__restrict__ tr, const float *__restrict__ psi, float *__restrict__ V2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 128 * 128) {
        const int k = i >> 7, n = i & 127;
        V2[i] = tr[n * 128 + k] * sqrtf(psi[n]);
    }
}

using EncodeTiledFn = CUresult (*)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                   const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// the driver's tensor-map encoder through the runtime, so that the library does not link against libcuda itself
EncodeTiledFn encode_tiled() {
    static const EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}

// TMA map of X [N, D] fp32 row-major: boxes of 32 columns x kTileM rows, 128-byte swizzle (the wgmma K-major layout),
// rows past N read as zeros.  False, with the reason, when TMA cannot address X.
bool encode_x_map(CUtensorMap *map, const float *X, int64_t N, int D, std::string *err) {
    if (reinterpret_cast<uintptr_t>(X) & 15) {
        if (err) *err = "the tensor-core projection needs X 16-byte aligned (TMA)";
        return false;
    }
    if (N > INT32_MAX - kTileM) {
        if (err) *err = "the tensor-core projection needs fewer than 2^31 - 256 frames (TMA row coordinate)";
        return false;
    }
    const EncodeTiledFn encode = encode_tiled();
    if (!encode) {
        if (err) *err = "cuTensorMapEncodeTiled is not available from the driver";
        return false;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)D * sizeof(float)};
    const cuuint32_t box[2] = {kKB, kTileM};
    const cuuint32_t elem_strides[2] = {1, 1};
    const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(X), dims, strides, box, elem_strides,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        if (err) *err = "cuTensorMapEncodeTiled failed for X (error " + std::to_string((int)r) + ")";
        return false;
    }
    return true;
}

// one GEMM pass [N,D] x [D,128] of the given MODE; V is row-major [D,128] in device memory
template <int MODE, int NS>
int launch_gemm_tc(float *vimg, int64_t N, const float *X, int D, const float *V, const float *Phi, float *out, float *gframe,
                   const float *a_off, const float *e_off, cudaStream_t st, std::string *err) {
    CUtensorMap xmap;
    if (!encode_x_map(&xmap, X, N, D, err)) return -1;
    if (!allow_dynamic_smem(project_wgmma_kernel<MODE, NS>, Pipe<NS>::kSmemBytes)) {
        if (err) *err = "the device refused the wgmma projection's shared-memory size";
        return -1;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
        if (err) *err = "cudaDeviceGetAttribute(multiprocessor count) failed";
        return -1;
    }
    build_v_images_kernel<NS><<<D / kKB, 256, 0, st>>>(V, D, vimg);
    const int64_t n_tiles = (N + kTileM - 1) / kTileM;
    const int grid = (int)std::min<int64_t>(n_tiles, sms);
    project_wgmma_kernel<MODE, NS><<<grid, kThreads, Pipe<NS>::kSmemBytes, st>>>(xmap, vimg, out, N, D, Phi, gframe, a_off, e_off);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        if (err) *err = std::string("wgmma projection launch failed: ") + cudaGetErrorString(e);
        return -1;
    }
    return 2;
}

}  // namespace

// Scratch of the tensor-core front end inside the caller's workspace: the swizzled hi/lo images of V (2 x 16 KB per
// 32 rows of V) for D up to kTcMaxD, and the folded PLDA matrix of the x-vector chain.
size_t tc_scratch_floats() { return (size_t)(kTcMaxD / kKB) * 3 * 4096 + 128 * 128; }

int launch_project_wgmma(const Plan &pl, float *tc_scratch, const float *X, int D, const float *V, const float *Phi, float *rho,
                         float *gframe, cudaStream_t st, std::string *err) {
    if (pl.R != 128) {
        if (err) *err = "the tensor-core projection needs R == 128";
        return -1;
    }
    if (D % kKB != 0 || D < kKB) {
        if (err) *err = "the tensor-core projection needs D to be a multiple of 32";
        return -1;
    }
    if (D > kTcMaxD || !tc_scratch) {
        if (err) *err = "the tensor-core projection needs D <= 2048 and a plan with R == 128";
        return -1;
    }
    if (pl.n_frames == 0) return 0;
    return launch_gemm_tc<0, 2>(tc_scratch, pl.n_frames, X, D, V, Phi, rho, gframe, nullptr, nullptr, st, err);
}

// The caller-side chain of VBx/vbhmm.py:125-129,153 plus the scale of VBx/VBx.py:88-89 as two tensor-core passes:
//   x_norm = l2norm(l2norm(x_raw - mean1) . lda - mean2)             [N,128]
//   rho    = (x_norm - plda_mu) . (plda_tr^T * sqrt(psi))            [N,128], with G_t per frame
int launch_xvector_chain_wgmma(const Plan &pl, float *tc_scratch, const float *x_raw, int Dx, const float *mean1, const float *lda,
                               const float *mean2, const float *plda_mu, const float *plda_tr, const float *psi,
                               float *x_norm, float *rho, float *gframe, cudaStream_t st, std::string *err) {
    if (pl.R != 128) {
        if (err) *err = "the x-vector chain needs R == 128";
        return -1;
    }
    if (Dx % kKB != 0 || Dx < kKB) {
        if (err) *err = "the x-vector chain needs the x-vector dimension to be a multiple of 32";
        return -1;
    }
    if (Dx > kTcMaxD || !tc_scratch) {
        if (err) *err = "the x-vector chain needs an x-vector dimension <= 2048";
        return -1;
    }
    if (pl.n_frames == 0) return 0;
    float *v2 = tc_scratch + (size_t)(kTcMaxD / kKB) * 3 * 4096;
    int n = launch_gemm_tc<1, 3>(tc_scratch, pl.n_frames, x_raw, Dx, lda, nullptr, x_norm, nullptr, mean1, mean2, st, err);
    if (n < 0) return -1;
    build_plda_v_kernel<<<64, 256, 0, st>>>(plda_tr, psi, v2);
    int m = launch_gemm_tc<2, 3>(tc_scratch, pl.n_frames, x_norm, 128, v2, psi, rho, gframe, plda_mu, nullptr, st, err);
    if (m < 0) return -1;
    return n + m + 1;
}

}  // namespace vbx
