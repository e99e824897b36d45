// forward_backward(lls, tr, ip) of the reference module for an ARBITRARY transition matrix      VBx/VBx.py:146-175
//
// The EM loop only ever calls it with tr = loopP*I + (1-loopP)*1*pi^T, which the hot-path kernels exploit (O(S) per
// frame, vbx_kernels.cu).  The module-level function is public API of VBx.py, so the shadow module offers it too:
// float64, log domain, dense S x S log-sum-exp per frame exactly as the reference computes it.  One CTA, thread = state;
// log(tr + 1e-8) and its transpose sit in shared memory (rows padded by one) when they fit, else they are recomputed.
#include <math_constants.h>

#include "vbx_internal.cuh"

namespace vbx {

namespace {

constexpr double kEps = 1e-8;   // VBx/VBx.py:158

template <bool SMEM_TR>
__global__ void __launch_bounds__(1024) fb_dense_kernel(const double *__restrict__ lls, const double *__restrict__ tr,
                                                        const double *__restrict__ ip, int T, int S, double *post,
                                                        double *tll_out, double *lfw, double *lbw) {
    extern __shared__ double sm[];
    double *va = sm;            // [S] vector of the previous step
    double *vb = sm + S;        // [S]
    double *ltr = sm + 2 * S;   // [S][S+1] log(tr + eps) (row i = from-state), when SMEM_TR
    const int j = threadIdx.x;
    const int LD = S + 1;
    if (SMEM_TR) {
        for (int i = j; i < S * S; i += blockDim.x) ltr[(i / S) * LD + i % S] = log(tr[i] + kEps);
    }
    auto L = [&](int from, int to) { return SMEM_TR ? ltr[from * LD + to] : log(tr[(int64_t)from * S + to] + kEps); };
    // forward: lfw[0] = lls[0] + log(ip + eps);  lfw[t, j] = lls[t, j] + logsumexp_i(lfw[t-1, i] + ltr[i, j])
    double cur = -CUDART_INF;
    if (j < S) {
        cur = lls[j] + log(ip[j] + kEps);
        lfw[j] = cur;
        va[j] = cur;
    }
    __syncthreads();
    double *prev = va, *next = vb;
    for (int t = 1; t < T; ++t) {
        if (j < S) {
            double m = -CUDART_INF;
            for (int i = 0; i < S; ++i) m = fmax(m, prev[i] + L(i, j));
            double s = 0.0;
            for (int i = 0; i < S; ++i) s += exp(prev[i] + L(i, j) - m);
            cur = lls[(int64_t)t * S + j] + (m + log(s));
            lfw[(int64_t)t * S + j] = cur;
            next[j] = cur;
        }
        __syncthreads();
        double *tmp = prev;
        prev = next;
        next = tmp;
    }
    // tll = logsumexp(lfw[T-1])
    double tll;
    {
        double m = -CUDART_INF;
        for (int i = 0; i < S; ++i) m = fmax(m, prev[i]);
        double s = 0.0;
        for (int i = 0; i < S; ++i) s += exp(prev[i] - m);
        tll = m + log(s);
    }
    if (j == 0) *tll_out = tll;
    __syncthreads();
    // backward: lbw[T-1] = 0;  lbw[t, i] = logsumexp_j(ltr[i, j] + lls[t+1, j] + lbw[t+1, j])
    if (j < S) {
        lbw[(int64_t)(T - 1) * S + j] = 0.0;
        post[(int64_t)(T - 1) * S + j] = exp(lfw[(int64_t)(T - 1) * S + j] - tll);
        prev[j] = lls[(int64_t)(T - 1) * S + j];          // lls[t+1] + lbw[t+1]
    }
    __syncthreads();
    for (int t = T - 2; t >= 0; --t) {
        if (j < S) {
            double m = -CUDART_INF;
            for (int k = 0; k < S; ++k) m = fmax(m, L(j, k) + prev[k]);
            double s = 0.0;
            for (int k = 0; k < S; ++k) s += exp(L(j, k) + prev[k] - m);
            const double b = m + log(s);
            lbw[(int64_t)t * S + j] = b;
            post[(int64_t)t * S + j] = exp(lfw[(int64_t)t * S + j] + b - tll);
            next[j] = lls[(int64_t)t * S + j] + b;
        }
        __syncthreads();
        double *tmp = prev;
        prev = next;
        next = tmp;
    }
}

}  // namespace

int launch_fb_dense(const double *lls, const double *tr, const double *ip, int T, int S, double *post, double *tll,
                    double *lfw, double *lbw, cudaStream_t st) {
    const int threads = ((S + 31) / 32) * 32;
    const size_t small = (size_t)2 * S * sizeof(double);
    const size_t full = small + (size_t)S * (S + 1) * sizeof(double);
    if (full <= 200 * 1024) {
        if (!allow_dynamic_smem(fb_dense_kernel<true>, 200 * 1024)) return -1;
        fb_dense_kernel<true><<<1, threads, full, st>>>(lls, tr, ip, T, S, post, tll, lfw, lbw);
    } else {
        fb_dense_kernel<false><<<1, threads, small, st>>>(lls, tr, ip, T, S, post, tll, lfw, lbw);
    }
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace vbx
