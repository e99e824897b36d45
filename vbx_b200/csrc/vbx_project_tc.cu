// Projection  rho[N,128] = X[N,D] . V[D,128]  on the Hopper tensor cores (wgmma, sm_90a), in split-precision 3xTF32
// (x_lo*v_hi + x_hi*v_lo + x_hi*v_hi, fp32 accumulation in registers) because plain TF32 breaks the 1e-4 parity bar of
// the EM loop (SURVEY.md section 7, hard part 4).
// Reference: the caller-side projection VBx/vbhmm.py:129,153 folded with the scale VBx/VBx.py:88-89 (SURVEY 8d).
//
// The same kernel, templated on MODE, also runs the real-data front end (x-vector transform and PLDA projection,
// VBx/vbhmm.py:125-129,153; launch_xvector_chain_wgmma below).
//
// One persistent CTA per SM, 16 warps, tiles of 128 frames:
//   warps 0-7   producers: coalesced LDG of a 128-frame x 32-column block of X (prefetched one block ahead in
//               registers), split into TF32 parts, stored into the 128B-swizzled K-major wgmma layout;
//               thread 0 also issues the bulk-async (TMA, cp.async.bulk) copies of the pre-split V block.
//   warps 8-15  two consumer warpgroups, 64 frames each: wgmma.mma_async m64n128k8 tf32 from shared memory into
//               64 fp32 registers per thread (4 k-steps x NS(NS+1)/2 split terms per 32-column block); a stage is
//               released to the producers one block later (wgmma.wait_group 1).  The epilogue works on the register
//               accumulators: the per-frame constant G_t (quad shuffles) and float2 stores of rho.
// Shared memory: NS = 2: 3 stages x (A hi/lo 32 KB + B hi/lo 32 KB) = 192 KB; NS = 3: 2 stages x (A 48 KB + B 48 KB).
//
// NS = 3 (the real-data front end): operands are split three ways, x = x1 + x2 + x3 exactly (3 x 11 mantissa bits), and
// six products are accumulated (x3 v1, x1 v3, x2 v2, x2 v1, x1 v2, x1 v1): the dropped terms are below 2^-33, i.e. the
// GEMM is at fp32-accumulate accuracy.  The shipped LDA matrix is badly conditioned (sum |a_k lda_kn| ~ 1e3 |sum|), so
// the 2^-21 relative error per product of the two-way split is visible on real data.
#include <cuda.h>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kTileM = 128;                 // frames per CTA tile: two wgmma M=64 tiles
constexpr int kKB = 32;                     // columns of X per pipeline block (= one 128-byte swizzle row)
constexpr int kABytes = 128 * 128;          // one 128-row x 128-byte operand image
constexpr int kProducerThreads = 256;
constexpr int kConsumerThreads = 256;       // two warpgroups
constexpr int kThreads = kProducerThreads + kConsumerThreads;

template <int NS> struct Pipe {
    static constexpr int kStages = NS == 2 ? 3 : 2;
    static constexpr int kStageBytes = 2 * NS * kABytes;   // A: NS images of 128 frames, B: NS images of V^T
    // 1 KB alignment slack, stages, barriers (128 B), 1/Phi or e_off (512 B), row norms [2][128] (1 KB)
    static constexpr int kSmemBytes = 1024 + kStages * kStageBytes + 128 + 512 + 2 * kTileM * 4;
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory matrix descriptor: K-major, 128-byte swizzle, dense 8-row groups (SBO = 1024 B, LBO unused = 1).
// Advancing along K inside the 128-byte swizzle row, or by whole 1024-byte row groups, only adds to the start address
// (bits 0-13, in 16-byte units), so the consumers add small integers to one descriptor per stage.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    const uint32_t lo = ((smem_addr >> 4) & 0x3fffu) | (1u << 16);
    const uint32_t hi = (1024u >> 4) | (1u << 30);                 // SBO, layout type 1 = SWIZZLE_128B
    return ((uint64_t)hi << 32) | lo;
}
// D[64 x 128] (+)= A[smem, 64 x 8] * B[smem, 128 x 8]^T, tf32, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching the accumulators across the asynchronous MMAs
__device__ __forceinline__ void fence_operands(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// streaming 16-byte load that does not allocate in L1: with ~195 KB of shared memory only ~30 KB of L1 remain, and
// allocating loads would cap the bytes in flight at that size
__device__ __forceinline__ float4 ldg_stream(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, const float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
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
//         the producers also accumulate ||x - a_off||^2 per row and hand it to the epilogue through shared memory
template <int MODE, int NS>
__global__ void __launch_bounds__(kThreads, 1)
project_wgmma_kernel(const float *__restrict__ X, const float *__restrict__ vimg, float *__restrict__ rho, int64_t N,
                     int D, const float *__restrict__ Phi, float *__restrict__ gframe,
                     const float *__restrict__ a_off, const float *__restrict__ e_off) {
    constexpr int kStages = Pipe<NS>::kStages, kStageBytes = Pipe<NS>::kStageBytes;
    constexpr int ROWS_PT = kTileM / 32;         // rows per producer thread
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // the stage buffers must be 1024-byte aligned (128-byte swizzle)
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + kStages * kStageBytes);
    float *s_inv_phi = reinterpret_cast<float *>(bars + 16);   // 128 floats: 1/Phi (MODE 0, 2) or e_off (MODE 1)
    float *s_n1 = s_inv_phi + 128;                             // [2][kTileM] row norms (MODE 1), by tile parity
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t bar_base = smem_u32(bars);
    auto full_a = [&](int s) { return bar_base + 8u * s; };
    auto full_b = [&](int s) { return bar_base + 8u * (kStages + s); };
    auto empty = [&](int s) { return bar_base + 8u * (2 * kStages + s); };

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_kb = D / kKB;
    const int64_t n_tiles = (N + kTileM - 1) / kTileM;

    if (tid < 128) s_inv_phi[tid] = MODE == 1 ? e_off[tid] : 1.f / Phi[tid];
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(full_a(s), kProducerThreads);
            mbar_init(full_b(s), 1);
            mbar_init(empty(s), kConsumerThreads);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 8) {
        // ======================= producers =======================
        // Blocks of this CTA in order: b -> (tile = blockIdx.x + (b / n_kb) * gridDim.x, kb = b % n_kb).  Two
        // ping-pong register sets keep the loads of the next block in flight while one is split and stored.
        const int c = tid & 7;            // 16-byte chunk inside the 128-byte row
        const int r0 = tid >> 3;          // rows r0 + 32 i
        const int64_t my_tiles = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        const int64_t n_blocks = my_tiles * n_kb;
        float4 bufA[ROWS_PT], bufB[ROWS_PT];
        float ss[ROWS_PT];                // MODE 1: running ||x - a_off||^2 of this thread's rows (its 4 columns)
#pragma unroll
        for (int i = 0; i < ROWS_PT; ++i) ss[i] = 0.f;
        auto issue = [&](const int64_t b, float4(&buf)[ROWS_PT]) {
            if (b >= n_blocks) return;
            const int64_t tile = blockIdx.x + (b / n_kb) * gridDim.x;
            const int kb = (int)(b % n_kb);
            const int64_t row_base = tile * kTileM;
#pragma unroll
            for (int i = 0; i < ROWS_PT; ++i) {
                const int64_t row = min(row_base + r0 + 32 * i, N - 1);
                buf[i] = ldg_stream(reinterpret_cast<const float4 *>(X + row * D + kb * kKB) + c);
            }
        };
        auto process = [&](const int64_t b, const float4(&buf)[ROWS_PT]) {
            const int s = (int)(b % kStages);
            const uint32_t ph = (uint32_t)((b / kStages) & 1);
            const int kb = (int)(b % n_kb);
            float4 aoff = make_float4(0.f, 0.f, 0.f, 0.f);
            if (MODE != 0) aoff = __ldg(reinterpret_cast<const float4 *>(a_off + kb * kKB) + c);
            mbar_wait(empty(s), ph ^ 1);               // the MMAs that read this stage have completed
            const uint32_t stage = smem_base + s * kStageBytes;
            if (tid == 0) {
                mbar_expect_tx(full_b(s), NS * kABytes);
                bulk_g2s(stage + NS * kABytes, vimg + (int64_t)kb * NS * 4096, NS * kABytes, full_b(s));
            }
#pragma unroll
            for (int i = 0; i < ROWS_PT; ++i) {
                const int m = r0 + 32 * i;             // 0..kTileM-1
                float4 hi, lo, x = buf[i];
                if (MODE != 0) {
                    x.x -= aoff.x;
                    x.y -= aoff.y;
                    x.z -= aoff.z;
                    x.w -= aoff.w;
                }
                if (MODE == 1) ss[i] = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, ss[i]))));
                const uint32_t off = (uint32_t)(m * 128 + ((c ^ (m & 7)) << 4));
                if (NS == 2) {
                    split_rn(x.x, hi.x, lo.x);
                    split_rn(x.y, hi.y, lo.y);
                    split_rn(x.z, hi.z, lo.z);
                    split_rn(x.w, hi.w, lo.w);
                    st_shared_v4(stage + 0 * kABytes + off, hi);
                    st_shared_v4(stage + 1 * kABytes + off, lo);
                } else {
                    float4 lo2;
                    split3_rn(x.x, hi.x, lo.x, lo2.x);
                    split3_rn(x.y, hi.y, lo.y, lo2.y);
                    split3_rn(x.z, hi.z, lo.z, lo2.z);
                    split3_rn(x.w, hi.w, lo.w, lo2.w);
                    st_shared_v4(stage + 0 * kABytes + off, hi);
                    st_shared_v4(stage + 1 * kABytes + off, lo);
                    st_shared_v4(stage + 2 * kABytes + off, lo2);
                }
            }
            if (MODE == 1 && kb == n_kb - 1) {
                // row norms of the finished tile: the 8 lanes that share a row are adjacent
                float *dst = s_n1 + ((b / n_kb) & 1) * kTileM;
#pragma unroll
                for (int i = 0; i < ROWS_PT; ++i) {
                    float v = ss[i];
                    v += __shfl_xor_sync(0xffffffffu, v, 1);
                    v += __shfl_xor_sync(0xffffffffu, v, 2);
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    if (c == 0) dst[r0 + 32 * i] = v;
                    ss[i] = 0.f;
                }
            }
            fence_proxy_async_smem();                  // make the generic-proxy stores visible to the tensor core
            mbar_arrive(full_a(s));
        };
        issue(0, bufA);
        for (int64_t b = 0; b < n_blocks; b += 2) {
            issue(b + 1, bufB);
            process(b, bufA);
            if (b + 1 < n_blocks) {
                issue(b + 2, bufA);
                process(b + 1, bufB);
            }
        }
    } else {
        // ======================= consumers: MMA + epilogue =======================
        const int ct = tid - kProducerThreads;
        const int wg = ct >> 7;                        // warpgroup: frames 64 wg .. 64 wg + 63 of the tile
        const int rq = 16 * ((ct >> 5) & 3) + (lane >> 2);   // accumulator rows rq and rq + 8 of the warpgroup
        const int cq = 2 * (lane & 3);                 // accumulator columns 8 j + cq, + 1
        constexpr uint64_t kImg = kABytes >> 4;        // one operand image, in 16-byte descriptor units
        float d[64];
        int s = 0, last = 0;
        uint32_t ph = 0;
        int it = 0;
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
            for (int kb = 0; kb < n_kb; ++kb) {
                mbar_wait(full_a(s), ph);
                mbar_wait(full_b(s), ph);
                const uint32_t stage = smem_base + s * kStageBytes;
                const uint64_t a0 = make_desc(stage + wg * 64 * 128);     // this warpgroup's 64 rows of the A images
                const uint64_t b0 = make_desc(stage + NS * kABytes);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const uint64_t k = ks * 2;         // 8 tf32 = 32 bytes inside the swizzle row (16-byte units)
                    const uint32_t first = (kb == 0 && ks == 0) ? 0u : 1u;
                    if (NS == 2) {                      // lo*hi + hi*lo + hi*hi
                        wgmma_tf32(d, a0 + kImg + k, b0 + k, first);
                        wgmma_tf32(d, a0 + k, b0 + kImg + k, 1u);
                        wgmma_tf32(d, a0 + k, b0 + k, 1u);
                    } else {                            // smallest terms first: x3 v1, x1 v3, x2 v2, x2 v1, x1 v2, x1 v1
                        wgmma_tf32(d, a0 + 2 * kImg + k, b0 + k, first);
                        wgmma_tf32(d, a0 + k, b0 + 2 * kImg + k, 1u);
                        wgmma_tf32(d, a0 + kImg + k, b0 + kImg + k, 1u);
                        wgmma_tf32(d, a0 + kImg + k, b0 + k, 1u);
                        wgmma_tf32(d, a0 + k, b0 + kImg + k, 1u);
                        wgmma_tf32(d, a0 + k, b0 + k, 1u);
                    }
                }
                wgmma_commit();
                if (kb > 0) {                          // the previous block's MMAs have retired: release its stage
                    wgmma_wait<1>();
                    mbar_arrive(empty(last));
                }
                last = s;
                if (++s == kStages) {
                    s = 0;
                    ph ^= 1;
                }
            }
            wgmma_wait<0>();
            fence_operands(d);
            const int64_t ra = tile * kTileM + wg * 64 + rq, rb = ra + 8;
            float n1a = 0.f, n1b = 0.f;
            if (MODE == 1) {                           // read before the release: the producers reuse this slot two tiles on
                n1a = s_n1[(it & 1) * kTileM + wg * 64 + rq];
                n1b = s_n1[(it & 1) * kTileM + wg * 64 + rq + 8];
            }
            mbar_arrive(empty(last));
            float na = 0.f, nb = 0.f;
            if (MODE == 1) {
                // y = acc / ||x - mean1|| - mean2 ; out = y / ||y||
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
                if ((lane & 3) == 0) {                 // G_t, R = 128
                    if (ra < N) gframe[ra] = -0.5f * (na + 128.f * 1.8378770664093453f);
                    if (rb < N) gframe[rb] = -0.5f * (nb + 128.f * 1.8378770664093453f);
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

// cudaFuncSetAttribute is per device; everything else the launches need comes from the caller's workspace
bool g_configured[64][3][2] = {};

// one GEMM pass [N,D] x [D,128] of the given MODE; V is row-major [D,128] in device memory
template <int MODE, int NS>
int launch_gemm_tc(float *vimg, int64_t N, const float *X, int D, const float *V, const float *Phi, float *out, float *gframe,
                   const float *a_off, const float *e_off, cudaStream_t st, std::string *err) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) {
        if (err) *err = "device index out of range";
        return -1;
    }
    if (!g_configured[dev][MODE][NS - 2]) {
        if (cudaFuncSetAttribute(project_wgmma_kernel<MODE, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, Pipe<NS>::kSmemBytes) !=
            cudaSuccess) {
            if (err) *err = "cudaFuncSetAttribute(smem) failed";
            return -1;
        }
        g_configured[dev][MODE][NS - 2] = true;
    }
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
        if (err) *err = "cudaDeviceGetAttribute(multiprocessor count) failed";
        return -1;
    }
    build_v_images_kernel<NS><<<D / kKB, 256, 0, st>>>(V, D, vimg);
    const int64_t n_tiles = (N + kTileM - 1) / kTileM;
    const int grid = (int)std::min<int64_t>(n_tiles, sms);
    project_wgmma_kernel<MODE, NS><<<grid, kThreads, Pipe<NS>::kSmemBytes, st>>>(X, vimg, out, N, D, Phi, gframe, a_off, e_off);
    if (cudaGetLastError() != cudaSuccess) {
        if (err) *err = "wgmma projection launch failed";
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
