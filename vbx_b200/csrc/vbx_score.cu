// Diarization error rate accumulation (include/vbx_b200.h vbx_score, DESIGN.md section 5.11; with a second label per
// interval inside overlap regions, vbx_score_overlap, section 5.12).
//
// One CTA per (setting, recording) entry.  The entry's system output is one owned time interval per x-vector with one
// label each.  An interval whose successor has the same label extends to its `join_hi` instead of its `hi`: that
// bridges the short pauses that pipeline.merge_adjacent_labels treats as touching (np.isclose), so the entry scores
// exactly the RTTM segments the project writes.  The recording's scored time is a sorted list of disjoint regions, each
// with the bitmask of the reference speakers active in it (0 = scored non-speech).  Threads stride over the intervals;
// each binary-searches the first region that ends after the interval's start and walks regions until its end, adding
// the overlap (integer microseconds) to
//   covered  (system speaks over reference speech), fa (system speaks over scored non-speech),
//   O[r, s]  for every active reference speaker r and the interval's label s.
// All sums are 64-bit integer atomics, so results do not depend on the order of the additions: bit-reproducible across
// runs, batch compositions and launch shapes.  Each entry's O [n_ref x n_labels] sits in shared memory when it fits the
// launch's shared block and is accumulated directly in its global block otherwise; either way one CTA owns it.
// With label time (vbx_score_jer, section 5.13) each entry also sums, per label, the scored time in which the system says
// it (S [n_labels]); that block follows the same shared-or-global policy.
#include "../../include/vbx_b200.h"
#include "vbx_internal.cuh"

namespace vbx {
namespace {

constexpr int kScoreThreads = 256;
constexpr int64_t kScoreSmemCells = 64 * 128;      // 64 KB of int64: 64 reference speakers x 128 labels
constexpr int64_t kScoreSmemLabels = 128;          // 1 KB of int64 label time after the O cells (label-time launches)

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Adds v to T[key] once per group of lanes in `act` with the same key (key < 0: nothing).  Consecutive intervals mostly
// share a label, so one atomic usually serves the whole warp.  The group's sum is a tree over its lanes in rank order
// (each round, every lane adds the value of the next remaining lane of its group; odd ranks drop out), which ends at
// the group's lowest lane.  Integer sums: the result does not depend on the grouping.
__device__ __forceinline__ void add_label_time(unsigned long long *T, int key, unsigned long long v) {
    const unsigned act = __activemask();
    const unsigned peers = __match_any_sync(act, key);
    const unsigned lane = threadIdx.x & 31u;
    unsigned rank = __popc(peers & ((1u << lane) - 1u));
    unsigned rest = peers & ~((2u << lane) - 1u);       // lanes of my group above me (2u << 31 wraps to 0: none)
    while (__any_sync(act, rest)) {
        const int next = __ffs(rest);
        const unsigned long long o = __shfl_sync(act, v, next ? next - 1 : (int)lane);
        if (next) v += o;
        rest &= __ballot_sync(act, !(rank & 1u));
        rank >>= 1;
    }
    if (key >= 0 && v && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&T[key], v);
}

// kSecond (vbx_score_overlap): interval t also says labels2[t] (-1 = nothing) inside the regions whose ovl flag is set,
// up to its own end (join_hi where the next interval has the same second label).  Both streams start at lo, so a region
// piece [a, b) carries stream 1 for its first d1 = clamp(end1 - a) ticks and stream 2 for its first d2; over that piece
// min(d1, d2) ticks have two system labels and |d1 - d2| one, which is all the md-eval counting needs:
//   both += min(N_ref, N_sys) d,  fa += max(0, N_sys - N_ref) d,  O[r, s] += d for every active r and s,
// i.e. with d1 + d2 label-ticks in the piece: all of them covered when N_ref >= 2, all false alarm when N_ref = 0, and
// for N_ref = 1 the min(d1, d2) ticks of the second label are a false alarm.  `covered` then holds `both`.
// kLabelTime (vbx_score_jer): also S[s] += d1 and S[s2] += d2 over every scored region piece, non-speech included, summed
// per interval in registers and added once per interval (add_label_time).  S [n_labels] of entry e sits after the O cells
// in shared memory when n_labels <= kScoreSmemLabels, else it is accumulated in place at T_out + t_off[e].  The extra
// parameters come last, so the other instantiations keep their parameter layout.
template <bool kSecond, bool kLabelTime>
__global__ void __launch_bounds__(kScoreThreads) score_kernel(
    int32_t n_rec, const int64_t *__restrict__ sys_off, const int64_t *__restrict__ sys_lo,
    const int64_t *__restrict__ sys_hi, const int64_t *__restrict__ sys_join_hi, const int64_t *__restrict__ reg_off, const int64_t *__restrict__ reg_lo,
    const int64_t *__restrict__ reg_hi, const uint64_t *__restrict__ reg_mask, const uint8_t *__restrict__ reg_ovl,
    const int32_t *__restrict__ n_ref, const int32_t *__restrict__ entry_rec, const int64_t *__restrict__ label_off,
    const int32_t *__restrict__ labels, const int32_t *__restrict__ labels2,
    const int32_t *__restrict__ n_labels, const int64_t *__restrict__ o_off, int64_t max_cells, int64_t smem_cells,
    int64_t *__restrict__ covered_out, int64_t *__restrict__ fa_out, int64_t *__restrict__ O_out,
    int32_t *__restrict__ flags_out, const int64_t *__restrict__ t_off, int64_t *__restrict__ T_out) {
    extern __shared__ unsigned long long sO[];
    __shared__ unsigned long long s_cov, s_fa;
    __shared__ int s_flags;
    const int e = blockIdx.x;
    const int rec = entry_rec[e];
    const int K = (rec >= 0 && rec < n_rec) ? n_ref[rec] : 0;
    const int L = n_labels[e];
    const int64_t cells = (K > 0 && L > 0) ? (int64_t)K * L : 0;
    if (rec < 0 || rec >= n_rec || K > 64 || cells > max_cells) {    // uniform over the CTA: the entry is not counted
        if (threadIdx.x == 0) {
            covered_out[e] = 0;
            fa_out[e] = 0;
            flags_out[e] = VBX_SCORE_BAD_RECORDING;
        }
        return;
    }
    const bool shared_block = cells <= smem_cells;
    unsigned long long *O = shared_block ? sO : reinterpret_cast<unsigned long long *>(O_out + o_off[e]);
    for (int64_t i = threadIdx.x; i < cells; i += blockDim.x) O[i] = 0ull;
    unsigned long long *S = nullptr;
    if constexpr (kLabelTime) {
        S = L <= kScoreSmemLabels ? sO + smem_cells : reinterpret_cast<unsigned long long *>(T_out + t_off[e]);
        for (int i = threadIdx.x; i < L; i += blockDim.x) S[i] = 0ull;
    }
    if (threadIdx.x == 0) {
        s_cov = 0ull;
        s_fa = 0ull;
        s_flags = 0;
    }
    __syncthreads();

    const int64_t t0 = sys_off[rec], t1 = sys_off[rec + 1];
    const int64_t r0 = reg_off[rec], r1 = reg_off[rec + 1];
    const int32_t *lab = labels + label_off[e];
    const int32_t *lab2 = kSecond ? labels2 + label_off[e] : nullptr;
    const uint64_t live = K >= 64 ? ~0ull : ((1ull << (K < 0 ? 0 : K)) - 1ull);
    unsigned long long cov = 0ull, fa = 0ull;
    int flags = 0;
    for (int64_t t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
        const int s = lab[t - t0];
        if (s < 0 || s >= L) {
            flags |= VBX_SCORE_BAD_LABEL;
            continue;
        }
        const int64_t lo = sys_lo[t];
        const int64_t hi = (t + 1 < t1 && lab[t + 1 - t0] == s) ? sys_join_hi[t] : sys_hi[t];
        if constexpr (kSecond) {
            const int s2 = lab2[t - t0];
            if (s2 < -1 || s2 >= L || s2 == s) {
                flags |= VBX_SCORE_BAD_LABEL;
                continue;
            }
            const int64_t hi2 = s2 < 0 ? lo : (t + 1 < t1 && lab2[t + 1 - t0] == s2) ? sys_join_hi[t] : sys_hi[t];
            const int64_t end = max(hi, hi2);
            if (end <= lo) continue;
            int64_t a = r0, b = r1;            // first region that ends after lo
            while (a < b) {
                const int64_t m = (a + b) >> 1;
                if (reg_hi[m] <= lo) a = m + 1;
                else b = m;
            }
            unsigned long long v1 = 0ull, v2 = 0ull;            // label time of this interval (kLabelTime)
            for (int64_t r = a; r < r1; ++r) {
                const int64_t rs = reg_lo[r];
                if (rs >= end) break;
                const int64_t p0 = max(lo, rs), re = reg_hi[r];
                const int64_t d1 = max((int64_t)0, min(hi, re) - p0);
                const int64_t d2 = reg_ovl[r] ? max((int64_t)0, min(hi2, re) - p0) : 0;
                if (d1 + d2 == 0) continue;
                if constexpr (kLabelTime) {
                    v1 += (unsigned long long)d1;
                    v2 += (unsigned long long)d2;
                }
                uint64_t msk = reg_mask[r];
                if (msk & ~live) {
                    flags |= VBX_SCORE_BAD_REGION;
                    continue;
                }
                const unsigned long long two = (unsigned long long)min(d1, d2), all = (unsigned long long)(d1 + d2);
                if (msk == 0ull) fa += all;                         // N_ref = 0: every system label is a false alarm
                else if (msk & (msk - 1ull)) cov += all;            // N_ref >= 2: every system label is covered
                else {                                              // N_ref = 1: the second of two is a false alarm
                    cov += all - two;
                    fa += two;
                }
                while (msk) {
                    const int k = __ffsll((long long)msk) - 1;
                    msk &= msk - 1ull;
                    if (d1) atomicAdd(&O[(int64_t)k * L + s], (unsigned long long)d1);
                    if (d2) atomicAdd(&O[(int64_t)k * L + s2], (unsigned long long)d2);
                }
            }
            if constexpr (kLabelTime) {
                add_label_time(S, s, v1);
                add_label_time(S, s2, v2);
            }
        } else {
            if (hi <= lo) continue;
            int64_t a = r0, b = r1;            // first region that ends after lo
            while (a < b) {
                const int64_t m = (a + b) >> 1;
                if (reg_hi[m] <= lo) a = m + 1;
                else b = m;
            }
            unsigned long long v1 = 0ull;                       // label time of this interval (kLabelTime)
            for (int64_t r = a; r < r1; ++r) {
                const int64_t rs = reg_lo[r];
                if (rs >= hi) break;
                const int64_t d = min(hi, reg_hi[r]) - max(lo, rs);
                if (d <= 0) continue;
                if constexpr (kLabelTime) v1 += (unsigned long long)d;
                uint64_t msk = reg_mask[r];
                if (msk & ~live) {
                    flags |= VBX_SCORE_BAD_REGION;
                    continue;
                }
                if (msk == 0ull) {
                    fa += (unsigned long long)d;
                    continue;
                }
                cov += (unsigned long long)d;
                while (msk) {
                    const int k = __ffsll((long long)msk) - 1;
                    msk &= msk - 1ull;
                    atomicAdd(&O[(int64_t)k * L + s], (unsigned long long)d);
                }
            }
            if constexpr (kLabelTime) add_label_time(S, s, v1);
        }
    }
    cov = warp_sum(cov);
    fa = warp_sum(fa);
    flags = __reduce_or_sync(0xffffffffu, flags);
    if ((threadIdx.x & 31) == 0) {
        if (cov) atomicAdd(&s_cov, cov);
        if (fa) atomicAdd(&s_fa, fa);
        if (flags) atomicOr(&s_flags, flags);
    }
    __syncthreads();
    if (shared_block) {
        int64_t *dst = O_out + o_off[e];
        for (int64_t i = threadIdx.x; i < cells; i += blockDim.x) dst[i] = (int64_t)sO[i];
    }
    if constexpr (kLabelTime) {
        if (L <= kScoreSmemLabels) {
            int64_t *dst = T_out + t_off[e];
            for (int i = threadIdx.x; i < L; i += blockDim.x) dst[i] = (int64_t)S[i];
        }
    }
    if (threadIdx.x == 0) {
        covered_out[e] = (int64_t)s_cov;
        fa_out[e] = (int64_t)s_fa;
        flags_out[e] = s_flags;
    }
}

}  // namespace

int launch_score(int n_rec, const int64_t *sys_off, const int64_t *sys_lo, const int64_t *sys_hi, const int64_t *sys_join_hi,
                 const int64_t *reg_off,
                 const int64_t *reg_lo, const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_ovl,
                 const int32_t *n_ref, int n_entries, const int32_t *entry_rec, const int64_t *label_off,
                 const int32_t *labels, const int32_t *labels2,
                 const int32_t *n_labels, const int64_t *o_off, int64_t max_cells, int64_t *covered_out,
                 int64_t *fa_out, int64_t *O_out, int32_t *flags_out, const int64_t *t_off, int64_t *T_out,
                 cudaStream_t st) {
    if (n_entries == 0) return 0;
    const bool second = labels2 != nullptr, label_time = T_out != nullptr;
    auto kernel = label_time ? (second ? score_kernel<true, true> : score_kernel<false, true>)
                             : (second ? score_kernel<true, false> : score_kernel<false, false>);
    const int64_t smem_cells = max_cells < kScoreSmemCells ? max_cells : kScoreSmemCells;
    // label-time launches add 1 KB after the O cells: 65 KB at most, still three CTAs per SM where O alone fits three
    const int64_t smem_words = smem_cells + (label_time ? kScoreSmemLabels : 0);
    const int64_t max_words = kScoreSmemCells + (label_time ? kScoreSmemLabels : 0);
    const size_t smem = (size_t)smem_words * sizeof(unsigned long long);
    if (smem > 48 * 1024 && !allow_dynamic_smem(kernel, (int)(max_words * sizeof(unsigned long long)))) return -1;
    kernel<<<n_entries, kScoreThreads, smem, st>>>(n_rec, sys_off, sys_lo, sys_hi, sys_join_hi, reg_off, reg_lo, reg_hi, reg_mask,
                                                   reg_ovl, n_ref, entry_rec, label_off, labels, labels2, n_labels, o_off,
                                                   max_cells, smem_cells, covered_out, fa_out, O_out, flags_out, t_off, T_out);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace vbx
