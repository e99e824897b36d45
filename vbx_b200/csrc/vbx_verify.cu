// Speaker-verification trials scored with the back end (DESIGN.md section 5.27).  A trial compares an enrolment item with
// a test item (a speaker's x-vectors, or one x-vector); both sides get the statistics n, F, b, e of section 5.15 through
// launch_speaker_stats_batch (one problem per side, c = Fa / Fb), and
//   verify_score_kernel   one warp per 32 trials (i, j): the b rows of the two sides staged through shared memory in
//                         32-feature chunks with coalesced loads, each lane summing its own trial in order r = 0 .. R-1
//                         with vbx_link's score_tile operations in the same order, so a trial's LLR is bit-identical to
//                         the enrolment and cohort LLR of the same pair; with cohort statistics the AS-norm score S of
//                         norm_scores_kernel's expression (enrolment item = row, test item = column)
// The error rates of a scored list (target / nontarget labels) run on the device in a fixed order, without atomics on
// floating-point values:
//   verify_keys_kernel    order-preserving 64-bit keys (-0.0 folded into +0.0), labels as 0 / 1, non-finite scores
//                         counted (integer atomics)
//   cub::DeviceRadixSort  (key, label) pairs ascending
//   verify_tar_kernel     the sorted labels as int64, then cub::DeviceScan: tar[s] = targets before sorted position s
//   verify_sweep_kernel   every candidate threshold (the first position of each group of equal scores, and +inf at
//                         position T): P_miss = tar / N_tar, P_fa = (N_non - nontargets before) / N_non; slot 0 reduces the
//                         EER bracket (the last candidate with P_miss < P_fa, the first with P_miss >= P_fa) and scatters
//                         the Cllr terms by rank within their class, slot 1 + o the least cost of operating point o and
//                         its lowest position; per-CTA partials by exact min / max
//   verify_cllr_kernel    the two Cllr sums over the class-ranked terms on a fixed grid (per-thread strides, a fixed
//                         butterfly, warps in order)
//   verify_final_kernel   one thread: the partials reduced, EER by linear interpolation, minDCF and its threshold, actDCF at
//                         the Bayes threshold by binary search, Cllr
// Everything a call computes depends on the scores and labels alone (not on their order, the grid or earlier calls).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr int kLogGroup = 8;                // as vbx_link: log of a product of 8 denominators, overflowed_log_sum
constexpr int kScoreWarps = 2;              // warps per CTA of verify_score_kernel (33.8 KB of staging)
constexpr int64_t kScoreGrid = 1 << 20;     // CTAs of verify_score_kernel at most; beyond that they stride
constexpr int kSweepThreads = 256;
constexpr int kSweepGrid = 1024;            // CTAs per slot of verify_sweep_kernel at most
constexpr int kCllrThreads = 256;
constexpr int kCllrCtas = 256;              // the fixed partition of the Cllr sums

__host__ __device__ size_t al(size_t v) { return (v + 255) & ~(size_t)255; }

// As vbx_link: the log term sum_r log(fma(cm, Phi_r, 1)) of a pair whose sum of group logs came out +inf: some product of
// kLogGroup denominators overflowed (each denominator is finite, but any finite positive Fa / Fb is accepted, so c can
// be large).  The same groups in the same order, each multiply that would overflow first flushing the product so far
// into the sum; a group that did not overflow gives the same log as in the scoring loop.  Out of line and reached only
// from that case, so the loop's registers and instructions stay those of plain groups.
__device__ __noinline__ double overflowed_log_sum(double cm, const float *__restrict__ Phi, int R) {
    double lg = 0.0, prod = 1.0;
    for (int r = 0; r < R; ++r) {
        const double den = fma(cm, (double)Phi[r], 1.0), pd = prod * den;
        if (pd > DBL_MAX) {
            lg += log(prod);
            prod = den;
        } else {
            prod = pd;
        }
        if ((r % kLogGroup) == kLogGroup - 1 || r == R - 1) {
            lg += log(prod);
            prod = 1.0;
        }
    }
    return lg;
}

// ---------------------------------------------------------------------------------------------------------------- scores

struct VerifyScoreWs {
    SpeakerStats e, t;
    int64_t *arrays;         // off_e [2], off_t [2], c [1]
};

VerifyScoreWs score_layout(uint8_t *ws, int64_t M_e, int64_t M_t, size_t *total) {
    VerifyScoreWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.e = take_stats(take, M_e);
    w.t = take_stats(take, M_t);
    w.arrays = reinterpret_cast<int64_t *>(take(5 * 8));
    if (total) *total = o;
    return w;
}

// Warp w of the grid takes trials 32 w .. 32 w + 31, lane l trial 32 w + l.  Per chunk of 32 features the warp loads
// the b rows of its 32 enrolment and 32 test items (row v: lane = feature, 256 contiguous bytes) into its own shared
// tiles, then each lane runs over the chunk for its trial with score_tile's operations: den = fma(cm, Phi_r, 1),
// x = b_i + b_j, q += x x / den, prod *= den and lg += log(prod) after every kLogGroup features and the last (an lg of
// +inf recomputed by overflowed_log_sum).  A trial whose index lies outside its side loads nothing and writes NaN.
__global__ void __launch_bounds__(kScoreWarps * 32) verify_score_kernel(
    SpeakerStats En, SpeakerStats Te, int64_t M_e, int64_t M_t, const float *__restrict__ Phi, int R, double c,
    const int32_t *__restrict__ ti, const int32_t *__restrict__ tj, int64_t T, const double *__restrict__ mean_e,
    const double *__restrict__ std_e, const double *__restrict__ mean_t, const double *__restrict__ std_t,
    double *__restrict__ score_out) {
    __shared__ double a[kScoreWarps][32][33], bt[kScoreWarps][32][33], ph[kScoreWarps][32];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int64_t n_warps = (T + 31) / 32, stride = (int64_t)gridDim.x * kScoreWarps;
    for (int64_t w = (int64_t)blockIdx.x * kScoreWarps + wl; w < n_warps; w += stride) {
        const int64_t t = w * 32 + lane;
        const int64_t i = t < T ? (int64_t)ti[t] : -1, j = t < T ? (int64_t)tj[t] : -1;
        const bool ok = i >= 0 && i < M_e && j >= 0 && j < M_t;
        const double ni = ok ? En.n[i] : 0.0, nj = ok ? Te.n[j] : 0.0;
        const double cm = c * (ni + nj);
        double q = 0.0, lg = 0.0, prod = 1.0;
        for (int r0 = 0; r0 < R; r0 += 32) {
            const int r = r0 + lane;
            for (int v = 0; v < 32; ++v) {
                const int iv = __shfl_sync(0xffffffffu, (int)(ok ? i : -1), v);
                const int jv = __shfl_sync(0xffffffffu, (int)(ok ? j : -1), v);
                a[wl][v][lane] = (iv >= 0 && r < R) ? En.b[(int64_t)iv * kMaxR + r] : 0.0;
                bt[wl][v][lane] = (jv >= 0 && r < R) ? Te.b[(int64_t)jv * kMaxR + r] : 0.0;
            }
            ph[wl][lane] = r < R ? (double)Phi[r] : 0.0;
            __syncwarp();
            const int len = min(32, R - r0);
            for (int k = 0; k < len; ++k) {
                const double p = ph[wl][k];
                const double den = fma(cm, p, 1.0), x = a[wl][lane][k] + bt[wl][lane][k];
                q += x * x / den;
                prod *= den;
                if (((r0 + k) % kLogGroup) == kLogGroup - 1 || r0 + k == R - 1) {
                    lg += log(prod);
                    prod = 1.0;
                }
            }
            __syncwarp();                             // the next chunk rewrites the tiles
        }
        if (lg > DBL_MAX) lg = overflowed_log_sum(cm, Phi, R);
        if (t >= T) continue;
        double s = NAN;
        if (ok) {
            const double l = (ni == 0.0 || nj == 0.0) ? 0.0 : 0.5 * ((q - lg) - (En.e[i] + Te.e[j]));
            s = mean_e ? 0.5 * ((l - mean_e[i]) / std_e[i] + (l - mean_t[j]) / std_t[j]) : l;
        }
        score_out[t] = s;
    }
}

// ------------------------------------------------------------------------------------------------------------- metrics

// Doubles ordered as their keys are ordered (as unsigned integers): negative values bit-inverted, the others with the
// sign bit set (vbx_cohort's order_key), after -0.0 is folded into +0.0 so that the two are one value.
__device__ __forceinline__ unsigned long long score_key(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

__device__ __forceinline__ double key_score(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// log(1 + exp(x)) as max(x, 0) + log1p(exp(-|x|))
__device__ __forceinline__ double softplus(double x) { return __dadd_rn(fmax(x, 0.0), log1p(exp(-fabs(x)))); }

struct SweepPart {
    double cost;             // slot 1 + o: least cost; slot 0: unused
    long long lo, hi;        // slot 1 + o: its lowest position; slot 0: last failing / first passing candidate
};

struct VerifyMetricsWs {
    unsigned long long *key_in, *key;
    uint8_t *lab_in, *lab;
    long long *tar;          // [T] targets before each sorted position
    double *terms;           // [T] Cllr terms: targets at their class rank, nontargets at N_tar + their class rank
    SweepPart *part;         // [(n_op + 1), kSweepGrid]
    double *cllr_part;       // [2, kCllrCtas]
    unsigned long long *nonfinite;
    double *ops;             // [n_op, 4]: C_miss p, C_fa (1 - p), their min, the Bayes threshold
    void *cub_tmp;
    size_t cub_bytes;
};

size_t cub_temp_bytes(int64_t T) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                    (const uint8_t *)nullptr, (uint8_t *)nullptr, T);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (long long *)nullptr, T);
    return std::max(a, b);
}

VerifyMetricsWs metrics_layout(uint8_t *ws, int64_t T, int n_op, size_t cub_bytes, size_t *total) {
    VerifyMetricsWs w;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = ws ? ws + o : nullptr; o += al(bytes); return p; };
    w.key_in = reinterpret_cast<unsigned long long *>(take((size_t)T * 8));
    w.key = reinterpret_cast<unsigned long long *>(take((size_t)T * 8));
    w.lab_in = take((size_t)T);
    w.lab = take((size_t)T);
    w.tar = reinterpret_cast<long long *>(take((size_t)T * 8));
    w.terms = reinterpret_cast<double *>(take((size_t)T * 8));
    w.part = reinterpret_cast<SweepPart *>(take((size_t)(n_op + 1) * kSweepGrid * sizeof(SweepPart)));
    w.cllr_part = reinterpret_cast<double *>(take(2 * kCllrCtas * 8));
    w.nonfinite = reinterpret_cast<unsigned long long *>(take(8));
    w.ops = reinterpret_cast<double *>(take((size_t)n_op * 4 * 8));
    w.cub_tmp = take(cub_bytes);
    w.cub_bytes = cub_bytes;
    if (total) *total = o;
    return w;
}

__global__ void verify_keys_kernel(const double *__restrict__ scores, const uint8_t *__restrict__ is_target, int64_t T,
                                   unsigned long long *__restrict__ key, uint8_t *__restrict__ lab,
                                   unsigned long long *__restrict__ nonfinite) {
    unsigned int bad = 0;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (int64_t)gridDim.x * blockDim.x) {
        const double v = scores[t];
        bad += isfinite(v) ? 0u : 1u;
        key[t] = score_key(v);
        lab[t] = is_target[t] ? 1 : 0;
    }
    for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(nonfinite, (unsigned long long)bad);   // integer counts: order-free
}

__global__ void verify_tar_kernel(const uint8_t *__restrict__ lab, int64_t T, long long *__restrict__ tar) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (int64_t)gridDim.x * blockDim.x)
        tar[t] = lab[t];
}

// The counts at sorted position s (0 .. T): targets below s and nontargets at or above s.
struct Counts {
    long long n_tar, n_non;
    __device__ __forceinline__ void at(const long long *tar, int64_t T, int64_t s, long long &miss, long long &fa) const {
        miss = s < T ? tar[s] : n_tar;
        fa = n_non - (s - miss);
    }
};

__device__ __forceinline__ Counts class_counts(const long long *tar, const uint8_t *lab, int64_t T) {
    Counts c;
    c.n_tar = tar[T - 1] + lab[T - 1];
    c.n_non = T - c.n_tar;
    return c;
}

__device__ __forceinline__ bool is_candidate(const unsigned long long *key, int64_t T, int64_t s) {
    return s == 0 || s == T || key[s] != key[s - 1];
}

// (cost, position) pairs: the smaller cost, on equal costs the lower position
__device__ __forceinline__ void take_min(double &bc, long long &bs, double oc, long long os) {
    if (oc < bc || (oc == bc && os < bs)) {
        bc = oc;
        bs = os;
    }
}

__device__ void block_reduce_part(SweepPart &p, bool eer) {
    __shared__ SweepPart red[kSweepThreads / 32];
    for (int o = 16; o; o >>= 1) {
        const double oc = __shfl_xor_sync(0xffffffffu, p.cost, o);
        const long long olo = __shfl_xor_sync(0xffffffffu, p.lo, o), ohi = __shfl_xor_sync(0xffffffffu, p.hi, o);
        if (eer) {
            p.lo = max(p.lo, olo);
            p.hi = min(p.hi, ohi);
        } else {
            take_min(p.cost, p.lo, oc, olo);
        }
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = p;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int q = 1; q < kSweepThreads / 32; ++q) {
            if (eer) {
                p.lo = max(p.lo, red[q].lo);
                p.hi = min(p.hi, red[q].hi);
            } else {
                take_min(p.cost, p.lo, red[q].cost, red[q].lo);
            }
        }
    }
    __syncthreads();
}

__device__ __forceinline__ double ratio(long long a, long long b) { return __ddiv_rn((double)a, (double)b); }

// (C_miss p) P_miss + (C_fa (1 - p)) P_fa, normalised by min(C_miss p, C_fa (1 - p)); no contraction into fma
__device__ __forceinline__ double dcf(const double *op, double pm, double pf) {
    return __ddiv_rn(__dadd_rn(__dmul_rn(op[0], pm), __dmul_rn(op[1], pf)), op[2]);
}

// grid (x, n_op + 1): slot y = blockIdx.y.  Positions s = 0 .. T over the CTAs of the slot.
__global__ void __launch_bounds__(kSweepThreads) verify_sweep_kernel(const unsigned long long *__restrict__ key,
                                                                      const uint8_t *__restrict__ lab,
                                                                      const long long *__restrict__ tar, int64_t T,
                                                                      const double *__restrict__ ops,
                                                                      double *__restrict__ terms,
                                                                      SweepPart *__restrict__ part) {
    const Counts cnt = class_counts(tar, lab, T);
    const int slot = blockIdx.y;
    const bool eer = slot == 0;
    const double *op = ops + 4 * (slot - 1);
    SweepPart p{INFINITY, eer ? -1ll : (long long)LLONG_MAX, (long long)T};
    for (int64_t s = (int64_t)blockIdx.x * kSweepThreads + threadIdx.x; s <= T; s += (int64_t)gridDim.x * kSweepThreads) {
        if (eer && s < T) {                           // the Cllr term of this trial at its rank within its class
            const double v = key_score(key[s]);
            const long long tb = tar[s];
            if (lab[s]) terms[tb] = softplus(-v);
            else terms[cnt.n_tar + (s - tb)] = softplus(v);
        }
        if (!is_candidate(key, T, s)) continue;
        long long miss, fa;
        cnt.at(tar, T, s, miss, fa);
        const double pm = ratio(miss, cnt.n_tar), pf = ratio(fa, cnt.n_non);
        if (eer) {
            if (pm >= pf) p.hi = min(p.hi, (long long)s);
            else p.lo = max(p.lo, (long long)s);
        } else {
            take_min(p.cost, p.lo, dcf(op, pm, pf), (long long)s);
        }
    }
    block_reduce_part(p, eer);
    if (threadIdx.x == 0) part[(int64_t)slot * gridDim.x + blockIdx.x] = p;
}

// Sum over the CTA: a fixed butterfly in every warp, then the warps in order.
__device__ __forceinline__ double cllr_block_sum(double v) {
    __shared__ double red[kCllrThreads / 32];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int q = 0; q < kCllrThreads / 32; ++q) t += red[q];
    __syncthreads();
    return t;
}

// grid (kCllrCtas, 2): y = 0 the target terms [0, N_tar), y = 1 the nontarget terms [N_tar, T); thread k of the grid
// sums ranks k, k + kCllrCtas x kCllrThreads, ... in order
__global__ void __launch_bounds__(kCllrThreads) verify_cllr_kernel(const double *__restrict__ terms,
                                                                    const uint8_t *__restrict__ lab,
                                                                    const long long *__restrict__ tar, int64_t T,
                                                                    double *__restrict__ cllr_part) {
    const Counts cnt = class_counts(tar, lab, T);
    const int64_t base = blockIdx.y ? cnt.n_tar : 0, n = blockIdx.y ? cnt.n_non : cnt.n_tar;
    double s = 0.0;
    for (int64_t k = (int64_t)blockIdx.x * kCllrThreads + threadIdx.x; k < n; k += (int64_t)kCllrCtas * kCllrThreads)
        s += terms[base + k];
    s = cllr_block_sum(s);
    if (threadIdx.x == 0) cllr_part[blockIdx.y * kCllrCtas + blockIdx.x] = s;
}

// One thread: each slot's grid_x partials reduced in order (exact min / max: any order gives the same result), then the
// metrics.
__global__ void verify_final_kernel(const unsigned long long *__restrict__ key, const uint8_t *__restrict__ lab,
                                    const long long *__restrict__ tar, int64_t T, const double *__restrict__ ops,
                                    int n_op, const SweepPart *__restrict__ part, int grid_x,
                                    const double *__restrict__ cllr_part, const unsigned long long *__restrict__ nonfinite,
                                    long long *__restrict__ counts_out, double *__restrict__ eer_out,
                                    double *__restrict__ cllr_out, double *__restrict__ min_dcf_out,
                                    double *__restrict__ threshold_out, double *__restrict__ act_dcf_out) {
    const Counts cnt = class_counts(tar, lab, T);
    counts_out[0] = cnt.n_tar;
    counts_out[1] = cnt.n_non;
    counts_out[2] = (long long)*nonfinite;
    auto value = [&](long long s) { return s < T ? key_score(key[s]) : (double)INFINITY; };
    // EER: the segment between the last candidate with P_miss < P_fa and the first with P_miss >= P_fa
    long long lo = -1, hi = T;
    for (int b = 0; b < grid_x; ++b) {
        lo = max(lo, part[b].lo);
        hi = min(hi, part[b].hi);
    }
    double eer = NAN;
    if (lo >= 0) {
        long long m0, f0, m1, f1;
        cnt.at(tar, T, lo, m0, f0);
        cnt.at(tar, T, hi, m1, f1);
        const double pm0 = ratio(m0, cnt.n_tar), pf0 = ratio(f0, cnt.n_non);
        const double pm1 = ratio(m1, cnt.n_tar), pf1 = ratio(f1, cnt.n_non);
        const double a = __dsub_rn(pm0, pf0), b = __dsub_rn(pm1, pf1);
        const double lam = __ddiv_rn(a, __dsub_rn(a, b));
        eer = __dadd_rn(pf0, __dmul_rn(lam, __dsub_rn(pf1, pf0)));
    }
    *eer_out = eer;
    for (int o = 0; o < n_op; ++o) {
        const SweepPart *po = part + (int64_t)(o + 1) * grid_x;
        double bc = INFINITY;
        long long bs = LLONG_MAX;
        for (int b = 0; b < grid_x; ++b) take_min(bc, bs, po[b].cost, po[b].lo);
        const double *op = ops + 4 * o;
        min_dcf_out[o] = bc;
        threshold_out[o] = value(bs);
        // actDCF: accepted where score >= theta; s = the first sorted position whose score is >= theta
        const double theta = op[3];
        long long l = 0, r = T;
        while (l < r) {
            const long long m = l + (r - l) / 2;
            if (key_score(key[m]) < theta) l = m + 1;
            else r = m;
        }
        long long miss, fa;
        cnt.at(tar, T, l, miss, fa);
        act_dcf_out[o] = dcf(op, ratio(miss, cnt.n_tar), ratio(fa, cnt.n_non));
    }
    double st = 0.0, sn = 0.0;
    for (int b = 0; b < kCllrCtas; ++b) {
        st += cllr_part[b];
        sn += cllr_part[kCllrCtas + b];
    }
    *cllr_out = (st / (double)cnt.n_tar + sn / (double)cnt.n_non) / (2.0 * log(2.0));
}

}  // namespace

size_t verify_score_workspace_bytes(int64_t M_e, int64_t M_t) {
    size_t total = 0;
    score_layout(nullptr, M_e, M_t, &total);
    return total;
}

int launch_verify_score(const float *enroll_fea, int64_t N_e, const int32_t *enroll_item, int64_t M_e,
                        const float *test_fea, int64_t N_t, const int32_t *test_item, int64_t M_t, int R,
                        const float *Phi, double c, const int32_t *ti, const int32_t *tj, int64_t T,
                        const double *mean_e, const double *std_e, const double *mean_t, const double *std_t,
                        void *workspace, double *score_out, cudaStream_t st) {
    const VerifyScoreWs w = score_layout(reinterpret_cast<uint8_t *>(workspace), M_e, M_t, nullptr);
    int64_t host[5] = {0, M_e, 0, M_t, 0};
    std::memcpy(&host[4], &c, sizeof(double));
    if (cudaMemcpyAsync(w.arrays, host, sizeof(host), cudaMemcpyHostToDevice, st) != cudaSuccess) return -1;
    const double *d_c = reinterpret_cast<const double *>(w.arrays + 4);
    const int le = launch_speaker_stats_batch(enroll_fea, Phi, enroll_item, N_e, R, 1, w.arrays, d_c, M_e, w.e, nullptr,
                                              nullptr, st);
    const int lt = launch_speaker_stats_batch(test_fea, Phi, test_item, N_t, R, 1, w.arrays + 2, d_c, M_t, w.t, nullptr,
                                              nullptr, st);
    if (le < 0 || lt < 0) return -1;
    if (T == 0) return le + lt;
    const int64_t ctas = std::min<int64_t>(((T + 31) / 32 + kScoreWarps - 1) / kScoreWarps, kScoreGrid);
    verify_score_kernel<<<(unsigned)ctas, kScoreWarps * 32, 0, st>>>(w.e, w.t, M_e, M_t, Phi, R, c, ti, tj, T, mean_e,
                                                                     std_e, mean_t, std_t, score_out);
    return cudaGetLastError() == cudaSuccess ? le + lt + 1 : -1;
}

size_t verify_metrics_workspace_bytes(int64_t T, int n_op) {
    size_t total = 0;
    metrics_layout(nullptr, T, n_op, cub_temp_bytes(T), &total);
    return total;
}

int launch_verify_metrics(const double *scores, const uint8_t *is_target, int64_t T, const double *ops_host, int n_op,
                          void *workspace, long long *counts_out, double *eer_out, double *cllr_out,
                          double *min_dcf_out, double *threshold_out, double *act_dcf_out, cudaStream_t st) {
    const VerifyMetricsWs w = metrics_layout(reinterpret_cast<uint8_t *>(workspace), T, n_op, cub_temp_bytes(T), nullptr);
    if (cudaMemsetAsync(w.nonfinite, 0, 8, st) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(w.ops, ops_host, (size_t)n_op * 4 * sizeof(double), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return -1;
    const unsigned grid = (unsigned)std::min<int64_t>((T + 255) / 256, 4096);
    verify_keys_kernel<<<grid, 256, 0, st>>>(scores, is_target, T, w.key_in, w.lab_in, w.nonfinite);
    size_t bytes = w.cub_bytes;
    if (cub::DeviceRadixSort::SortPairs(w.cub_tmp, bytes, w.key_in, w.key, w.lab_in, w.lab, T, 0, 64, st) !=
        cudaSuccess)
        return -1;
    verify_tar_kernel<<<grid, 256, 0, st>>>(w.lab, T, w.tar);
    bytes = w.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(w.cub_tmp, bytes, w.tar, T, st) != cudaSuccess) return -1;
    const int gx = (int)std::min<int64_t>((T + kSweepThreads) / kSweepThreads, kSweepGrid);   // T + 1 positions
    verify_sweep_kernel<<<dim3(gx, n_op + 1), kSweepThreads, 0, st>>>(w.key, w.lab, w.tar, T, w.ops, w.terms, w.part);
    verify_cllr_kernel<<<dim3(kCllrCtas, 2), kCllrThreads, 0, st>>>(w.terms, w.lab, w.tar, T, w.cllr_part);
    verify_final_kernel<<<1, 1, 0, st>>>(w.key, w.lab, w.tar, T, w.ops, n_op, w.part, gx, w.cllr_part, w.nonfinite,
                                          counts_out, eer_out, cllr_out, min_dcf_out, threshold_out, act_dcf_out);
    // keys, sort (its kernels counted as one), labels, scan (counted as one), sweep, Cllr, final
    return cudaGetLastError() == cudaSuccess ? 7 : -1;
}

}  // namespace vbx
