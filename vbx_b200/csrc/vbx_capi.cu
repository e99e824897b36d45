// C ABI of vbx_b200 (include/vbx_b200.h): handle, batch plan, workspace carving, EM-loop driver.
#include <dlfcn.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <map>
#include <mutex>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

#include "../../include/vbx_b200.h"
#include "vbx_internal.cuh"

bool vbx::allow_dynamic_smem(const void *kernel, int bytes) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, int> allowed;   // (kernel, device) -> bytes set
    std::lock_guard<std::mutex> lock(mu);
    int &have = allowed[{kernel, dev}];
    if (have >= bytes) return true;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return false;
    have = bytes;
    return true;
}

struct vbx_handle_s {
    int device = 0;
    int sms = 0;                 // multiprocessors of the device
    std::string err;
    vbx::Plan plan;
    vbx::Workspace ws;
    bool planned = false, bound = false, prepared = false;
    bool f64_only = false;       // the plan came from vbx_plan_f64: any S / R, float64 entry points only
    size_t ws_need = 0;
    void *plan_mem = nullptr;  // one device allocation backing all plan arrays
    int opt_fb_spl = 0;
    int opt_fb_classic = 0;  // 1 = the normalise-every-frame sweep, 0 = one-step look-ahead
    int opt_fb_ring = 1;     // look-ahead sweep fed from shared-memory rings (1) or from register bursts (0)
    int opt_projection = 0;
    int opt_timing = 0;
    int opt_gemm = 0;  // 0 = mma.sync 3xTF32, 1 = FFMA
    int opt_debug_sync = 0;      // 1 = synchronise after every launch group and name it on stderr (debugging aid)
    int opt_fb_split = 0;        // 0 = auto (few recordings: sweeps on separate warps), 1 = always, 2 = never
    int opt_exact_stop = 1;      // 1 = finish recordings in float64 once the ELBO step nears epsilon (vbx_exact64.cu)
    int64_t launches = 0;
    // The forward-backward sweep of a large batch is latency bound (a tenth of the warps an SM can hold).  When two
    // sub-batches run on two streams (vbx_b200/parts.py) it should interleave with the other sub-batch's bandwidth-bound
    // contractions, but the block scheduler hands out the CTAs of the grid that was launched first until none are left.
    // The fused sweep of a batch of >= 1024 recordings therefore runs on a high-priority side stream of this handle
    // (ordered against `stream` by two events): its CTAs take the next free SM slots ahead of the queued contraction CTAs
    // of the other sub-batch (measured faster on the headline batch and ragged config 3, DESIGN.md section 5.6).
    cudaStream_t hi_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // CUDA graph of a whole vbx_run (small batches are launch bound: a run is 41 rounds x up to 12 launches).  The second
    // call with identical arguments is captured on graph_stream; later identical calls replay the graph with one launch.
    int opt_graph = 0;           // 0 = auto (plans on the split schedule, i.e. small batches), 1 = always, 2 = never
    cudaStream_t graph_stream = nullptr;
    cudaEvent_t ev_g0 = nullptr, ev_g1 = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    uint64_t graph_key = 0, seen_key = 0;
    int64_t graph_launches = 0;
    bool graph_broken = false;
    // NCCL communicator owned by the caller (vbx_attach_comm); ncclAllReduce is resolved from the libnccl the process
    // already uses, so the library has no link-time dependency on NCCL
    void *nccl_comm = nullptr;
    int nccl_ranks = 1;
    int (*nccl_allreduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    std::vector<int64_t> offsets_host;  // kept for the AHC workspace layout
    std::vector<int64_t> ahc_d_off;
    size_t ahc_need = 0;
    // per-kernel-class CUDA-event timing (opt_timing): events are recorded on the launching stream
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_used = 0;
    std::vector<int> ev_class;  // class of the (2i, 2i+1) event pair
    double t_ms[VBX_N_KERNEL_CLASSES] = {0};
    int64_t t_cnt[VBX_N_KERNEL_CLASSES] = {0};
};

namespace {

int fail(vbx_handle_t h, int code, const std::string &msg) {
    if (h) h->err = msg;
    return code;
}
int cuda_fail(vbx_handle_t h, cudaError_t e, const char *what) {
    return fail(h, VBX_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// The kernels read and write these arrays with 16-byte vector accesses (float4 rows, the sweeps' bulk copies): a pointer
// off that grid must be refused before anything is launched.  Null pointers are left to the null checks.
int misaligned16(vbx_handle_t h, const std::string &who, std::initializer_list<std::pair<const void *, const char *>> arrays) {
    for (const auto &a : arrays)
        if (reinterpret_cast<uintptr_t>(a.first) & 15)
            return fail(h, VBX_ERR_ARG, who + ": " + a.second + " must be 16-byte aligned");
    return VBX_OK;
}

// NVTX range around an entry point (visible in nsys / ncu --nvtx timelines; no cost without a tool attached)
struct Range {
    explicit Range(const char *name) { nvtxRangePushA(name); }
    ~Range() { nvtxRangePop(); }
};

// Every entry point runs on the handle's device and leaves the caller's current device as it found it.
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != device) err = cudaSetDevice(device);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
};

struct Carver {
    char *base;
    size_t off = 0;
    explicit Carver(void *b) : base(static_cast<char *>(b)) {}
    template <typename T>
    T *take(size_t n) {
        T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
        off += align_up(n * sizeof(T));
        return p;
    }
};

// a captured run is only valid for the plan, workspace and options it was captured with
void drop_graph(vbx_handle_t h) {
    if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
    h->graph_exec = nullptr;
    h->graph_key = h->seen_key = 0;
}

size_t carve(const vbx::Plan &pl, void *base, vbx::Workspace *ws) {
    Carver c(base);
    const size_t N = (size_t)pl.n_frames, S = (size_t)pl.S, R = (size_t)pl.R, B = (size_t)pl.n_rec;
    vbx::Workspace w;
    w.p = c.take<float>(N * S);
    w.rowmax = c.take<float>(N);
    w.rsigma = c.take<float>(N);
    w.cvec = c.take<float>(N);
    w.partial = c.take<float>((size_t)pl.n_mtiles * S * R);
    w.A = c.take<float>(B * S * R);
    {
        const size_t NT = S > 8 ? S / 8 : 1, KS = (R + 7) / 8;
        w.Afrag_hi = c.take<float>(B * NT * KS * 64);
        w.Afrag_lo = c.take<float>(B * NT * KS * 64);
    }
    w.bias = c.take<float>(B * S);
    w.occ = c.take<float>(B * S);
    w.regp = c.take<double>(B * S);
    w.gsum = c.take<double>(B);
    w.gpart = c.take<double>((size_t)pl.n_mtiles);
    w.prev_elbo = c.take<double>(B);
    w.active = c.take<int32_t>(B);
    w.scratch = c.take<float>(2 * std::max<size_t>(S, vbx::kMaxS));
    if (pl.R == 128) w.tc_scratch = c.take<float>(vbx::tc_scratch_floats());
    if (pl.split) {
        w.ahat = c.take<float>(N * S);
        w.bhat = c.take<float>(N * S);
        w.socc = c.take<float>((size_t)pl.n_mtiles * S);
        w.sent = c.take<float>((size_t)pl.n_mtiles * S);
    }
    {
        const size_t LC = (size_t)pl.n_lchunks;
        w.fa_u = c.take<float>(LC * S * S);
        w.fa_lam = c.take<float>(LC * S);
        w.fa_exp = c.take<float>(LC * S);
        w.astart = c.take<float>(LC * S);
        w.bb_v = c.take<float>(LC * S * S);
        w.bb_mu = c.take<float>(LC * S);
        w.bb_exp = c.take<float>(LC * S);
        w.beta = c.take<float>(LC * S);
        w.occp = c.take<float>(LC * S);
        w.entp = c.take<float>(LC * S);
    }
    if (pl.exact) {
        w.active64 = c.take<int32_t>(B);
        w.fresh = c.take<int32_t>(B);
        w.gamma_snap = c.take<float>(2 * N * S);
        w.pi_snap = c.take<float>(2 * B * S);
        w.p64 = c.take<double>(N * S);
        w.rowmax64 = c.take<double>(N);
        w.rsig64 = c.take<double>(N);
        w.partial64 = c.take<double>((size_t)pl.n_mtiles * S * R);
        w.occp64 = c.take<double>((size_t)pl.n_mtiles * S);
        w.alpha64 = c.take<double>(B * S * R);
        w.bias64 = c.take<double>(B * S);
        w.reg64 = c.take<double>(B);
        w.pi64 = c.take<double>(B * S);
    }
    w.hp = c.take<vbx::RecParams>(B);
    if (ws) *ws = w;
    return c.off + 256;
}

}  // namespace

extern "C" {

const char *vbx_version(void) { return "vbx_b200 0.2 (sm_90a)"; }

int32_t vbx_padded_states(int32_t n) {
    if (n < 1 || n > vbx::kMaxS) return -1;
    int32_t s = 4;
    while (s < n) s <<= 1;
    return s;
}

int32_t vbx_padded_states_wide(int32_t n) {
    if (n > vbx::kMaxS && n <= vbx::kMaxSWide) return vbx::kMaxSWide;
    return vbx_padded_states(n);
}

int vbx_create(int32_t device, vbx_handle_t *out) {
    if (!out) return VBX_ERR_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0 || device < 0 || device >= count)
        return VBX_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return VBX_ERR_CUDA;
    if (prop.major != 9 || prop.minor != 0) return VBX_ERR_NO_DEVICE;  // kernels are built for sm_90a only
    vbx_handle_t h = new vbx_handle_s();
    h->device = device;
    h->sms = prop.multiProcessorCount;
    {
        DeviceGuard guard(device);
        int lo = 0, hi = 0;
        if (guard.err != cudaSuccess || cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess ||
            cudaStreamCreateWithPriority(&h->hi_stream, cudaStreamNonBlocking, hi) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess ||
            cudaStreamCreateWithFlags(&h->graph_stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_g0, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&h->ev_g1, cudaEventDisableTiming) != cudaSuccess) {
            vbx_destroy(h);   // releases whatever was created (null members are skipped)
            return VBX_ERR_CUDA;
        }
    }
    *out = h;
    return VBX_OK;
}

int vbx_destroy(vbx_handle_t h) {
    if (!h) return VBX_ERR_ARG;
    DeviceGuard guard(h->device);
    if (h->plan_mem) cudaFree(h->plan_mem);
    if (h->hi_stream) cudaStreamDestroy(h->hi_stream);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
    if (h->graph_stream) cudaStreamDestroy(h->graph_stream);
    if (h->ev_g0) cudaEventDestroy(h->ev_g0);
    if (h->ev_g1) cudaEventDestroy(h->ev_g1);
    for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
    delete h;
    return VBX_OK;
}

const char *vbx_last_error(vbx_handle_t h) { return h ? h->err.c_str() : "null handle"; }

int vbx_set_option(vbx_handle_t h, const char *name, int32_t value) {
    if (!h || !name) return VBX_ERR_ARG;
    drop_graph(h);
    if (!strcmp(name, "graph")) {
        if (value < 0 || value > 2) return fail(h, VBX_ERR_ARG, "graph must be 0 (auto), 1 (always) or 2 (never)");
        h->opt_graph = value;
        return VBX_OK;
    }
    if (!strcmp(name, "fb_states_per_lane")) {
        if (value != 0 && value != 1 && value != 2 && value != 4) return fail(h, VBX_ERR_ARG, "fb_states_per_lane must be 0,1,2,4");
        h->opt_fb_spl = value;
        return VBX_OK;
    }
    if (!strcmp(name, "fb_classic")) {
        h->opt_fb_classic = value ? 1 : 0;
        return VBX_OK;
    }
    if (!strcmp(name, "fb_ring")) {
        h->opt_fb_ring = value ? 1 : 0;
        return VBX_OK;
    }
    if (!strcmp(name, "gemm")) {
        if (value != 0 && value != 1) return fail(h, VBX_ERR_ARG, "gemm must be 0 (mma 3xTF32) or 1 (FFMA)");
        h->opt_gemm = value;
        return VBX_OK;
    }
    if (!strcmp(name, "debug_sync")) {
        h->opt_debug_sync = value ? 1 : 0;
        return VBX_OK;
    }
    if (!strcmp(name, "fb_split")) {   // takes effect at the next vbx_plan
        if (value < 0 || value > 2) return fail(h, VBX_ERR_ARG, "fb_split must be 0 (auto), 1 (always) or 2 (never)");
        h->opt_fb_split = value;
        return VBX_OK;
    }
    if (!strcmp(name, "exact_stop")) {   // takes effect at the next vbx_plan (workspace layout)
        h->opt_exact_stop = value ? 1 : 0;
        return VBX_OK;
    }
    if (!strcmp(name, "timing")) {
        h->opt_timing = value ? 1 : 0;
        return VBX_OK;
    }
    if (!strcmp(name, "projection")) {
        if (value < 0 || value > 2) return fail(h, VBX_ERR_ARG, "projection must be 0,1,2");
        h->opt_projection = value;
        return VBX_OK;
    }
    return fail(h, VBX_ERR_ARG, std::string("unknown option ") + name);
}

int vbx_plan(vbx_handle_t h, const int64_t *offsets_host, int32_t n_rec, int32_t R, int32_t S,
             size_t *workspace_bytes_out) {
    if (!h || !offsets_host || n_rec < 0) return fail(h, VBX_ERR_ARG, "vbx_plan: null argument");
    if (R < 4 || R > vbx::kMaxR || (R & 3)) return fail(h, VBX_ERR_ARG, "vbx_plan: R must be a multiple of 4 in [4,128]");
    if (S != 4 && S != 8 && S != 16 && S != 32 && S != 64 && S != vbx::kMaxSWide)
        return fail(h, VBX_ERR_ARG, "vbx_plan: S must come from vbx_padded_states() or vbx_padded_states_wide()");
    if (S == vbx::kMaxSWide && h->opt_fb_split == 2)
        return fail(h, VBX_ERR_ARG, "vbx_plan: S = 128 plans always take the split forward-backward schedule (there is no fused "
                                    "sweep at 128 states), so option fb_split = 2 (never) cannot be honoured");
    if (n_rec > 0 && offsets_host[0] != 0) return fail(h, VBX_ERR_ARG, "vbx_plan: offsets[0] must be 0");
    for (int b = 0; b < n_rec; ++b) {
        const int64_t T = offsets_host[b + 1] - offsets_host[b];
        if (T < 0) return fail(h, VBX_ERR_ARG, "vbx_plan: offsets must be non-decreasing");
        if (T > (int64_t)1 << 30) return fail(h, VBX_ERR_ARG, "vbx_plan: recording longer than 2^30 frames");
    }
    DeviceGuard guard(h->device);
    cudaError_t e = guard.err;
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaSetDevice");

    std::vector<int32_t> order(n_rec);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) {
        return offsets_host[a + 1] - offsets_host[a] > offsets_host[b + 1] - offsets_host[b];
    });
    std::vector<int32_t> lrec, mrec, mbegin(n_rec + 1, 0);
    std::vector<int64_t> lf0, mf0;
    int64_t maxT = 0;
    for (int b = 0; b < n_rec; ++b) {
        const int64_t lo = offsets_host[b], hi = offsets_host[b + 1];
        maxT = std::max(maxT, hi - lo);
        for (int64_t f = lo; f < hi; f += vbx::kLTile) {
            lrec.push_back(b);
            lf0.push_back(f);
        }
        mbegin[b] = (int32_t)mrec.size();
        for (int64_t f = lo; f < hi; f += vbx::kMTile) {
            mrec.push_back(b);
            mf0.push_back(f);
        }
    }
    mbegin[n_rec] = (int32_t)mrec.size();
    // Few recordings cannot fill the GPU with one warp-group each: run the forward and the backward sweep of every
    // recording concurrently on separate warps (vbx_fb_split.cu).  Auto: when the sweeps of the fused kernel would occupy
    // at most two warps per SM.  S = 128 always splits (the fused sweep and the chunked scan stop at 64 states).
    bool split = h->opt_fb_split == 1 || S == vbx::kMaxSWide;
    if (h->opt_fb_split == 0 && !split) {
        const int spl = S >= 16 ? 2 : 1, rpw = 32 / (S / spl);
        const int warps = (n_rec + rpw - 1) / rpw;
        split = warps <= 2 * h->sms;
    }
    // long recordings -> chunk lists of the chunked-scan forward-backward (not needed by the split sweeps)
    std::vector<int32_t> lrec_list, lrec_first(std::max(n_rec, 1), 0), lrec_nchunks(std::max(n_rec, 1), 0), lchunk_rec, lchunk_idx;
    for (int b = 0; b < n_rec && !split; ++b) {
        const int64_t T = offsets_host[b + 1] - offsets_host[b];
        if (T >= vbx::kLongT) {
            const int K = (int)((T + vbx::kChunk - 1) / vbx::kChunk);
            lrec_list.push_back(b);
            lrec_first[b] = (int32_t)lchunk_rec.size();
            lrec_nchunks[b] = K;
            for (int k = 0; k < K; ++k) {
                lchunk_rec.push_back(b);
                lchunk_idx.push_back(k);
            }
        }
    }

    // one device blob for all plan arrays
    size_t off = 0;
    auto reserve = [&](size_t bytes) {
        size_t o = off;
        off += align_up(bytes);
        return o;
    };
    const size_t o_off = reserve(sizeof(int64_t) * (n_rec + 1));
    const size_t o_ord = reserve(sizeof(int32_t) * std::max(n_rec, 1));
    const size_t o_lrec = reserve(sizeof(int32_t) * std::max<size_t>(lrec.size(), 1));
    const size_t o_lf0 = reserve(sizeof(int64_t) * std::max<size_t>(lf0.size(), 1));
    const size_t o_mrec = reserve(sizeof(int32_t) * std::max<size_t>(mrec.size(), 1));
    const size_t o_mf0 = reserve(sizeof(int64_t) * std::max<size_t>(mf0.size(), 1));
    const size_t o_mb = reserve(sizeof(int32_t) * (n_rec + 1));
    const size_t o_ll = reserve(sizeof(int32_t) * std::max<size_t>(lrec_list.size(), 1));
    const size_t o_lf = reserve(sizeof(int32_t) * lrec_first.size());
    const size_t o_ln = reserve(sizeof(int32_t) * lrec_nchunks.size());
    const size_t o_lcr = reserve(sizeof(int32_t) * std::max<size_t>(lchunk_rec.size(), 1));
    const size_t o_lci = reserve(sizeof(int32_t) * std::max<size_t>(lchunk_idx.size(), 1));
    if (h->plan_mem) {
        cudaFree(h->plan_mem);
        h->plan_mem = nullptr;
    }
    h->planned = h->bound = h->prepared = false;
    h->f64_only = false;
    drop_graph(h);
    e = cudaMalloc(&h->plan_mem, off);
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc(plan)");
    char *base = static_cast<char *>(h->plan_mem);
    auto up = [&](size_t o, const void *src, size_t bytes) {
        return bytes ? cudaMemcpy(base + o, src, bytes, cudaMemcpyHostToDevice) : cudaSuccess;
    };
    if ((e = up(o_off, offsets_host, sizeof(int64_t) * (n_rec + 1))) != cudaSuccess ||
        (e = up(o_ord, order.data(), sizeof(int32_t) * n_rec)) != cudaSuccess ||
        (e = up(o_lrec, lrec.data(), sizeof(int32_t) * lrec.size())) != cudaSuccess ||
        (e = up(o_lf0, lf0.data(), sizeof(int64_t) * lf0.size())) != cudaSuccess ||
        (e = up(o_mrec, mrec.data(), sizeof(int32_t) * mrec.size())) != cudaSuccess ||
        (e = up(o_mf0, mf0.data(), sizeof(int64_t) * mf0.size())) != cudaSuccess ||
        (e = up(o_mb, mbegin.data(), sizeof(int32_t) * (n_rec + 1))) != cudaSuccess ||
        (e = up(o_ll, lrec_list.data(), sizeof(int32_t) * lrec_list.size())) != cudaSuccess ||
        (e = up(o_lf, lrec_first.data(), sizeof(int32_t) * lrec_first.size())) != cudaSuccess ||
        (e = up(o_ln, lrec_nchunks.data(), sizeof(int32_t) * lrec_nchunks.size())) != cudaSuccess ||
        (e = up(o_lcr, lchunk_rec.data(), sizeof(int32_t) * lchunk_rec.size())) != cudaSuccess ||
        (e = up(o_lci, lchunk_idx.data(), sizeof(int32_t) * lchunk_idx.size())) != cudaSuccess)
        return cuda_fail(h, e, "cudaMemcpy(plan)");

    vbx::Plan &pl = h->plan;
    pl.n_rec = n_rec;
    pl.R = R;
    pl.S = S;
    pl.exact = h->opt_exact_stop;
    pl.split = split ? 1 : 0;
    pl.em_cluster = vbx::em_contract_cluster(S, R, maxT, split);
    pl.n_frames = n_rec ? offsets_host[n_rec] : 0;
    pl.n_ltiles = (int32_t)lrec.size();
    pl.n_mtiles = (int32_t)mrec.size();
    pl.max_T = maxT;
    pl.offsets = reinterpret_cast<const int64_t *>(base + o_off);
    pl.order = reinterpret_cast<const int32_t *>(base + o_ord);
    pl.ltile_rec = reinterpret_cast<const int32_t *>(base + o_lrec);
    pl.ltile_f0 = reinterpret_cast<const int64_t *>(base + o_lf0);
    pl.mtile_rec = reinterpret_cast<const int32_t *>(base + o_mrec);
    pl.mtile_f0 = reinterpret_cast<const int64_t *>(base + o_mf0);
    pl.mtile_begin = reinterpret_cast<const int32_t *>(base + o_mb);
    pl.n_lrec = (int32_t)lrec_list.size();
    pl.n_lchunks = (int32_t)lchunk_rec.size();
    pl.lrec_list = reinterpret_cast<const int32_t *>(base + o_ll);
    pl.lrec_first = reinterpret_cast<const int32_t *>(base + o_lf);
    pl.lrec_nchunks = reinterpret_cast<const int32_t *>(base + o_ln);
    pl.lchunk_rec = reinterpret_cast<const int32_t *>(base + o_lcr);
    pl.lchunk_idx = reinterpret_cast<const int32_t *>(base + o_lci);
    h->ws_need = carve(pl, nullptr, nullptr);
    h->offsets_host.assign(offsets_host, offsets_host + (n_rec ? n_rec + 1 : 0));
    if (n_rec == 0) h->offsets_host.assign(1, 0);
    h->ahc_need = vbx::ahc_workspace_bytes(h->offsets_host.data(), n_rec, &h->ahc_d_off);
    h->planned = true;
    if (workspace_bytes_out) *workspace_bytes_out = h->ws_need;
    return VBX_OK;
}

int vbx_plan_f64(vbx_handle_t h, const int64_t *offsets_host, int32_t n_rec, int32_t R, int32_t S) {
    if (!h || !offsets_host || n_rec < 0) return fail(h, VBX_ERR_ARG, "vbx_plan_f64: null argument");
    if (R < 1 || S < 1 || S > 3600) return fail(h, VBX_ERR_ARG, "vbx_plan_f64: need R >= 1 and 1 <= S <= 3600");
    if (n_rec > 0 && offsets_host[0] != 0) return fail(h, VBX_ERR_ARG, "vbx_plan_f64: offsets[0] must be 0");
    for (int b = 0; b < n_rec; ++b) {
        const int64_t T = offsets_host[b + 1] - offsets_host[b];
        if (T < 0 || T > (int64_t)1 << 30) return fail(h, VBX_ERR_ARG, "vbx_plan_f64: bad recording length");
    }
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (h->plan_mem) {
        cudaFree(h->plan_mem);
        h->plan_mem = nullptr;
    }
    h->planned = h->bound = h->prepared = false;
    cudaError_t e = cudaMalloc(&h->plan_mem, sizeof(int64_t) * (n_rec + 1));
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc(plan)");
    e = cudaMemcpy(h->plan_mem, offsets_host, sizeof(int64_t) * (n_rec + 1), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return cuda_fail(h, e, "cudaMemcpy(plan)");
    h->plan = vbx::Plan();
    h->plan.n_rec = n_rec;
    h->plan.R = R;
    h->plan.S = S;
    h->plan.n_frames = n_rec ? offsets_host[n_rec] : 0;
    h->plan.offsets = static_cast<const int64_t *>(h->plan_mem);
    h->offsets_host.assign(offsets_host, offsets_host + n_rec + 1);
    h->ahc_need = 0;
    h->planned = true;
    h->f64_only = true;
    return VBX_OK;
}

int vbx_bind_workspace(vbx_handle_t h, void *workspace, size_t bytes) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_bind_workspace: call vbx_plan first");
    if (h->f64_only) return fail(h, VBX_ERR_STATE, "vbx_bind_workspace: the plan came from vbx_plan_f64 (float64 entry points only)");
    if (!workspace || bytes < h->ws_need) return fail(h, VBX_ERR_STATE, "vbx_bind_workspace: workspace too small");
    const size_t mis = reinterpret_cast<uintptr_t>(workspace) & 255;
    char *base = static_cast<char *>(workspace) + (mis ? 256 - mis : 0);
    carve(h->plan, base, &h->ws);
    drop_graph(h);
    h->bound = true;
    h->prepared = false;
    return VBX_OK;
}

static int check_ready(vbx_handle_t h, const char *who) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned || !h->bound) return fail(h, VBX_ERR_STATE, std::string(who) + ": plan and bind a workspace first");
    return VBX_OK;
}
static int counted(vbx_handle_t h, int n, const char *what) {
    if (n < 0) return cuda_fail(h, cudaGetLastError(), what);
    h->launches += n;
    if (h->opt_debug_sync) {
        fprintf(stderr, "[vbx_b200] %s: %d launch(es) ...", what, n);
        fflush(stderr);
        const cudaError_t e = cudaDeviceSynchronize();
        fprintf(stderr, " %s\n", cudaGetErrorString(e));
        fflush(stderr);
        if (e != cudaSuccess) return cuda_fail(h, e, what);
    }
    return VBX_OK;
}
// Brackets one kernel class with a pair of events on `st` when timing is enabled.
struct Timed {
    vbx_handle_t h;
    cudaStream_t st;
    bool on;
    Timed(vbx_handle_t h_, cudaStream_t st_, int cls) : h(h_), st(st_), on(h_->opt_timing != 0) {
        if (!on) return;
        while (h->ev_pool.size() < h->ev_used + 2) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
            h->ev_pool.push_back(e);
        }
        h->ev_class.push_back(cls);
        cudaEventRecord(h->ev_pool[h->ev_used], st);
    }
    ~Timed() {
        if (!on) return;
        cudaEventRecord(h->ev_pool[h->ev_used + 1], st);
        h->ev_used += 2;
    }
};

int vbx_prepare_scale(vbx_handle_t h, const float *fea, const float *Phi, float *rho_out, void *stream) {
    Range nvtx_range("vbx_prepare_scale");
    int rc = check_ready(h, "vbx_prepare_scale");
    if (rc) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (h->plan.n_frames && (!fea || !Phi || !rho_out)) return fail(h, VBX_ERR_ARG, "vbx_prepare_scale: null pointer");
    if ((rc = misaligned16(h, "vbx_prepare_scale", {{fea, "fea"}, {Phi, "Phi"}, {rho_out, "rho_out"}}))) return rc;
    {
        Timed t(h, (cudaStream_t)stream, VBX_K_PREPARE);
        rc = counted(h, vbx::launch_prepare_scale(h->plan, h->ws, fea, Phi, rho_out, (cudaStream_t)stream), "prepare_scale");
    }
    if (rc) return rc;
    h->prepared = true;
    return VBX_OK;
}

int vbx_prepare_project(vbx_handle_t h, const float *X, int32_t D, const float *V, const float *Phi, float *rho_out,
                        void *stream) {
    Range nvtx_range("vbx_prepare_project");
    int rc = check_ready(h, "vbx_prepare_project");
    if (rc) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (h->plan.n_frames && (!X || !V || !Phi || !rho_out)) return fail(h, VBX_ERR_ARG, "vbx_prepare_project: null pointer");
    if (D < 32 || (D & 31)) return fail(h, VBX_ERR_ARG, "vbx_prepare_project: D must be a multiple of 32");
    if ((rc = misaligned16(h, "vbx_prepare_project", {{X, "X"}, {V, "V"}, {rho_out, "rho_out"}}))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    bool done = false, fused_g = false;
    Timed *tp = new Timed(h, st, VBX_K_PROJECT);
    if (h->opt_projection != 1) {   // auto: wgmma when the shape allows it (R == 128, D % 32 == 0), else FFMA tiles
        std::string why;
        // the wgmma epilogue also emits G_t per frame into the (not yet used) rowmax scratch array
        int n = vbx::launch_project_wgmma(h->plan, h->ws.tc_scratch, X, D, V, Phi, rho_out, h->ws.rowmax, st, &why);
        if (n >= 0) {
            h->launches += n;
            done = true;
            fused_g = true;
        } else if (h->opt_projection == 2) {
            delete tp;
            return fail(h, VBX_ERR_ARG, "vbx_prepare_project: wgmma path unavailable: " + why);
        }
    }
    if (!done) rc = counted(h, vbx::launch_project_ffma(h->plan, X, D, V, rho_out, st), "project_ffma");
    delete tp;
    if (rc) return rc;
    {
        Timed t(h, st, VBX_K_PREPARE);
        rc = counted(h, fused_g ? vbx::launch_gsum_from_frames(h->plan, h->ws, h->ws.rowmax, st)
                                : vbx::launch_g_from_rho(h->plan, h->ws, rho_out, Phi, st), "g_from_rho");
    }
    if (rc) return rc;
    h->prepared = true;
    return VBX_OK;
}

int vbx_prepare_xvectors(vbx_handle_t h, const float *x_raw, int32_t Dx, const float *mean1, const float *lda,
                         const float *mean2, const float *plda_mu, const float *plda_tr, const float *plda_psi,
                         float *x_norm_out, float *rho_out, void *stream) {
    Range nvtx_range("vbx_prepare_xvectors");
    int rc = check_ready(h, "vbx_prepare_xvectors");
    if (rc) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (!mean1 || !lda || !mean2 || !plda_mu || !plda_tr || !plda_psi)
        return fail(h, VBX_ERR_ARG, "vbx_prepare_xvectors: null model pointer");
    if (h->plan.n_frames && (!x_raw || !x_norm_out || !rho_out)) return fail(h, VBX_ERR_ARG, "vbx_prepare_xvectors: null pointer");
    if (x_norm_out && x_norm_out == rho_out) return fail(h, VBX_ERR_ARG, "vbx_prepare_xvectors: x_norm_out and rho_out must not alias");
    if (Dx < 32 || (Dx & 31)) return fail(h, VBX_ERR_ARG, "vbx_prepare_xvectors: Dx must be a multiple of 32");
    if (h->plan.R != 128) return fail(h, VBX_ERR_ARG, "vbx_prepare_xvectors: the plan must have R == 128");
    cudaStream_t st = (cudaStream_t)stream;
    {
        Timed t(h, st, VBX_K_PROJECT);
        std::string why;
        int n = vbx::launch_xvector_chain_wgmma(h->plan, h->ws.tc_scratch, x_raw, Dx, mean1, lda, mean2, plda_mu, plda_tr, plda_psi,
                                                x_norm_out, rho_out, h->ws.rowmax, st, &why);
        if (n < 0) return fail(h, VBX_ERR_CUDA, "vbx_prepare_xvectors: " + why);
        h->launches += n;
    }
    {
        Timed t(h, st, VBX_K_PREPARE);
        rc = counted(h, vbx::launch_gsum_from_frames(h->plan, h->ws, h->ws.rowmax, st), "gsum_from_frames");
    }
    if (rc) return rc;
    h->prepared = true;
    return VBX_OK;
}

}  // extern "C"

// vbx_run (per_rec = false: the scalars Fa, Fb, loop_prob hold for every recording) and vbx_run_per_recording (per_rec:
// device arrays Fa_v, Fb_v, loopP_v [n_rec]); run_init_kernel turns either into the per-recording table the kernels read.
static int run_impl(vbx_handle_t h, const char *who, bool per_rec, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
                    const int32_t *n_states, double Fa, double Fb, double loop_prob, const double *Fa_v, const double *Fb_v,
                    const double *loopP_v, int32_t max_iters, double epsilon, float *alpha_io, float *invL_io,
                    int32_t warm_start, double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream,
                    const double *prior_n = nullptr, const double *prior_F = nullptr) {
    Range nvtx_range(who);
    const std::string w(who);
    int rc = check_ready(h, who);
    if (rc) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (!h->prepared) return fail(h, VBX_ERR_STATE, w + ": call vbx_prepare_scale/project first (G is part of the ELBO)");
    if (max_iters < 0) return fail(h, VBX_ERR_ARG, w + ": max_iters < 0");
    if (!per_rec && !(Fb != 0.0)) return fail(h, VBX_ERR_ARG, w + ": Fb must be non-zero");
    if (per_rec && (!Fa_v || !Fb_v || !loopP_v)) return fail(h, VBX_ERR_ARG, w + ": Fa, Fb and loop_prob must be device arrays [n_rec]");
    if (warm_start && (!alpha_io || !invL_io)) return fail(h, VBX_ERR_ARG, w + ": warm_start needs alpha_io and invL_io");
    const vbx::Plan &pl = h->plan;
    if (pl.n_rec == 0) return VBX_OK;
    if (!Li_out || !n_iters_out || !flags_out || !pi_io) return fail(h, VBX_ERR_ARG, w + ": null output pointer");
    if (pl.n_frames && (!rho || !Phi || !gamma_io)) return fail(h, VBX_ERR_ARG, w + ": null pointer");
    if ((rc = misaligned16(h, w, {{rho, "rho"}, {gamma_io, "gamma_io"}}))) return rc;
    vbx::RunParams rp;
    rp.epsilon = epsilon;
    rp.max_iters = max_iters;
    // epsilon = -inf (fixed iteration count) and NaN never stop: nothing to decide, everything stays float32
    rp.hybrid = (pl.exact && epsilon > -1e300 && epsilon < 1e300 && max_iters > 1) ? 1 : 0;
    rp.warm = warm_start ? 1 : 0;

    // ---- the launch sequence of one run, on stream `st` (directly, or under stream capture) ----
    auto enqueue = [&](cudaStream_t st) -> int {
    int rc = 0;
    {
        Timed t(h, st, VBX_K_RUN_INIT);
        rc = counted(h, vbx::launch_run_init(pl, h->ws, gamma_io, n_states, Li_out, n_iters_out, flags_out, max_iters, Fa, Fb,
                                             loop_prob, Fa_v, Fb_v, loopP_v, st), "run_init");
    }
    if (rc) return rc;
    // With the float64 finishing phase a recording that switched lags one round behind (it redoes two iterations):
    // one extra round, in which only the float64 kernels run.
    const int rounds = max_iters + (rp.hybrid ? 1 : 0);
    const bool fb_hi = !pl.split && pl.n_rec >= 1024;
    for (int it = 0; it < rounds; ++it) {
        Range nvtx_iter("vbx_em_iteration");
        const bool given = it == 0 && warm_start;
        if (it < max_iters) {
            if (rp.hybrid) {   // state entering this iteration, for recordings that switch to float64 later
                Timed t(h, st, VBX_K_EXACT64);
                rc = counted(h, vbx::launch_snapshot(pl, h->ws, gamma_io, pi_io, it, st), "snapshot");
                if (rc) return rc;
            }
            if (pl.em_cluster && !h->opt_gemm && !given && !prior_n) {
                Timed t(h, st, VBX_K_EM_CONTRACT);
                rc = counted(h, vbx::launch_em_contract(pl, h->ws, rho, gamma_io, Phi, n_states, alpha_io, invL_io, st),
                             "em_contract");
                if (rc) return rc;
            } else {   // the three kernels: split plans, S > 16, T > 1024, warm starts and priors
                if (!given) {
                    Timed t(h, st, VBX_K_MSTEP);
                    rc = counted(h, h->opt_gemm ? vbx::launch_mstep_partial(pl, h->ws, rho, gamma_io, st)
                                                : vbx::launch_mstep_mma(pl, h->ws, rho, gamma_io, st), "mstep_partial");
                }
                if (rc) return rc;
                {
                    Timed t(h, st, VBX_K_SPEAKER_MODEL);
                    rc = counted(h, vbx::launch_speaker_model(pl, h->ws, Phi, n_states, alpha_io, invL_io, given, st, prior_n,
                                                              prior_F), "speaker_model");
                }
                if (rc) return rc;
                {
                    Timed t(h, st, VBX_K_LOGLIK);
                    rc = counted(h, h->opt_gemm ? vbx::launch_loglik(pl, h->ws, rho, pi_io, n_states, st) : vbx::launch_loglik_mma(pl, h->ws, rho, pi_io, n_states, st), "loglik");
                }
                if (rc) return rc;
            }
            if (fb_hi) {   // the sweep on the high-priority side stream, ordered after the log-likelihoods and before the next M-step
                cudaEventRecord(h->ev_fork, st);
                cudaStreamWaitEvent(h->hi_stream, h->ev_fork, 0);
            }
            {
                cudaStream_t fs = fb_hi ? h->hi_stream : st;
                Timed t(h, fs, VBX_K_FWDBWD);
                rc = counted(h, vbx::launch_forward_backward(pl, h->ws, rp, gamma_io, pi_io, n_states, Li_out, n_iters_out, flags_out, it, h->opt_fb_spl, h->opt_fb_classic, h->opt_fb_ring, fs), "forward_backward");
            }
            if (fb_hi) {
                cudaEventRecord(h->ev_join, h->hi_stream);
                cudaStreamWaitEvent(st, h->ev_join, 0);
            }
            if (rc) return rc;
        }
        if (rp.hybrid && it > 0) {   // one float64 iteration for the recordings in the finishing phase (none at it == 0)
            Timed t(h, st, VBX_K_EXACT64);
            rc = counted(h, vbx::launch_exact64_round(pl, h->ws, rp, rho, Phi, gamma_io, pi_io, n_states, alpha_io, invL_io, Li_out,
                                                      n_iters_out, flags_out, st, prior_n, prior_F), "exact64");
            if (rc) return rc;
        }
    }
    return VBX_OK;
    };   // enqueue

    cudaStream_t user = (cudaStream_t)stream;
    const bool want_graph = (h->opt_graph == 1 || (h->opt_graph == 0 && pl.split)) && !h->opt_timing && !h->opt_debug_sync &&
                            !h->graph_broken;
    if (!want_graph) return enqueue(user);
    // identity of this call: every argument that ends up inside a kernel parameter
    uint64_t key = 1469598103934665603ull;
    auto mix = [&](uint64_t v) { key = (key ^ v) * 1099511628211ull; };
    auto bits = [](double d) { uint64_t u; memcpy(&u, &d, 8); return u; };
    for (const void *p : {(const void *)rho, (const void *)Phi, (const void *)gamma_io, (const void *)pi_io, (const void *)n_states,
                          (const void *)alpha_io, (const void *)invL_io, (const void *)Li_out, (const void *)n_iters_out,
                          (const void *)flags_out, (const void *)h->ws.p, (const void *)Fa_v, (const void *)Fb_v,
                          (const void *)loopP_v, (const void *)prior_n, (const void *)prior_F})
        mix((uint64_t)(uintptr_t)p);
    mix(bits(Fa)); mix(bits(Fb)); mix(bits(loop_prob)); mix(bits(epsilon)); mix((uint64_t)max_iters); mix((uint64_t)warm_start);
    if (key == 0) key = 1;
    auto replay = [&]() -> int {
        cudaEventRecord(h->ev_g0, user);
        cudaStreamWaitEvent(h->graph_stream, h->ev_g0, 0);
        const cudaError_t e = cudaGraphLaunch(h->graph_exec, h->graph_stream);
        cudaEventRecord(h->ev_g1, h->graph_stream);
        cudaStreamWaitEvent(user, h->ev_g1, 0);
        if (e != cudaSuccess) return cuda_fail(h, e, "cudaGraphLaunch");
        return VBX_OK;
    };
    if (h->graph_exec && key == h->graph_key) {
        h->launches += h->graph_launches;
        return replay();
    }
    if (key != h->seen_key) {          // first call with these arguments: run directly, capture if they come again
        h->seen_key = key;
        return enqueue(user);
    }
    // second identical call: capture the launch sequence (relaxed mode: other threads' CUDA calls are not affected)
    drop_graph(h);
    h->seen_key = key;
    const int64_t before = h->launches;
    if (cudaStreamBeginCapture(h->graph_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
        cudaGetLastError();
        h->graph_broken = true;
        return enqueue(user);
    }
    const int crc = enqueue(h->graph_stream);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(h->graph_stream, &graph);
    cudaGraphExec_t exec = nullptr;
    if (crc != VBX_OK || ce != cudaSuccess || !graph || cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
        cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        h->launches = before;
        h->graph_broken = true;           // this handle keeps launching directly
        return enqueue(user);
    }
    cudaGraphDestroy(graph);
    h->graph_exec = exec;
    h->graph_key = key;
    h->graph_launches = h->launches - before;
    return replay();
}

extern "C" {

int vbx_run(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
            const int32_t *n_states, double Fa, double Fb, double loop_prob, int32_t max_iters, double epsilon,
            float *alpha_io, float *invL_io, int32_t warm_start, double *Li_out, int32_t *n_iters_out,
            int32_t *flags_out, void *stream) {
    return run_impl(h, "vbx_run", false, rho, Phi, gamma_io, pi_io, n_states, Fa, Fb, loop_prob, nullptr, nullptr, nullptr, max_iters,
                    epsilon, alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, stream);
}

int vbx_run_per_recording(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
                          const int32_t *n_states, const double *Fa, const double *Fb, const double *loop_prob,
                          int32_t max_iters, double epsilon, float *alpha_io, float *invL_io, int32_t warm_start,
                          double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream) {
    return run_impl(h, "vbx_run_per_recording", true, rho, Phi, gamma_io, pi_io, n_states, 0.0, 1.0, 0.0, Fa, Fb, loop_prob, max_iters,
                    epsilon, alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, stream);
}

int vbx_run_prior(vbx_handle_t h, const float *rho, const float *Phi, float *gamma_io, float *pi_io,
                  const int32_t *n_states, const double *Fa, const double *Fb, const double *loop_prob,
                  int32_t max_iters, double epsilon, float *alpha_io, float *invL_io, int32_t warm_start,
                  double *Li_out, int32_t *n_iters_out, int32_t *flags_out, const double *prior_n,
                  const double *prior_F, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!prior_n || !prior_F) return fail(h, VBX_ERR_ARG, "vbx_run_prior: prior_n and prior_F must be device arrays");
    return run_impl(h, "vbx_run_prior", true, rho, Phi, gamma_io, pi_io, n_states, 0.0, 1.0, 0.0, Fa, Fb, loop_prob, max_iters,
                    epsilon, alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, stream, prior_n, prior_F);
}

int vbx_hard_labels(vbx_handle_t h, const float *gamma, const int32_t *n_states, int32_t *first_out,
                    int32_t *second_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned || h->f64_only) return fail(h, VBX_ERR_STATE, "vbx_hard_labels: call vbx_plan first");
    if (h->plan.n_frames && (!gamma || !first_out)) return fail(h, VBX_ERR_ARG, "vbx_hard_labels: null pointer");
    if (const int rc = misaligned16(h, "vbx_hard_labels", {{gamma, "gamma"}})) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_hard_labels(h->plan, gamma, n_states, first_out, second_out, (cudaStream_t)stream), "hard_labels");
}

int vbx_hard_labels_keep(vbx_handle_t h, const float *gamma, const int32_t *n_states, const int32_t *keep,
                         int32_t *first_out, int32_t *second_out, double *mass_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned || h->f64_only) return fail(h, VBX_ERR_STATE, "vbx_hard_labels_keep: call vbx_plan first");
    if (h->plan.n_rec == 0) return VBX_OK;
    if (!keep || !mass_out || (h->plan.n_frames && (!gamma || !first_out)))
        return fail(h, VBX_ERR_ARG, "vbx_hard_labels_keep: null pointer");
    if (const int rc = misaligned16(h, "vbx_hard_labels_keep", {{gamma, "gamma"}})) return rc;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    // keep lives on the device: read it back once to refuse counts below 1 (the labels leave the device next anyway)
    std::vector<int32_t> kh(h->plan.n_rec);
    cudaError_t e = cudaMemcpyAsync(kh.data(), keep, kh.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(h, e, "vbx_hard_labels_keep: reading keep");
    for (int b = 0; b < h->plan.n_rec; ++b)
        if (kh[b] < 1) return fail(h, VBX_ERR_ARG, "vbx_hard_labels_keep: keep[" + std::to_string(b) + "] < 1");
    return counted(h, vbx::launch_hard_labels_keep(h->plan, gamma, n_states, keep, first_out, second_out, mass_out,
                                                   (cudaStream_t)stream), "hard_labels_keep");
}

int vbx_init_turns(vbx_handle_t h, const int64_t *seg, const int64_t *spk_off, const int64_t *turn_off,
                   const int64_t *turn_lo, const int64_t *turn_hi, const int64_t *turn_cum, const double *smoothing,
                   void *gamma_out, void *pi_out, int32_t out_is_f64, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_init_turns: call vbx_plan or vbx_plan_f64 first");
    const vbx::Plan &pl = h->plan;
    if (pl.n_rec == 0) return VBX_OK;
    if (!spk_off || !turn_off || !smoothing || !pi_out || (pl.n_frames && (!seg || !gamma_out)))
        return fail(h, VBX_ERR_ARG, "vbx_init_turns: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    // the speaker and turn offsets live on the device: read them back once to refuse negative counts and K_b > S
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int64_t> so(pl.n_rec + 1);
    cudaError_t e = cudaMemcpyAsync(so.data(), spk_off, so.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(h, e, "vbx_init_turns: reading spk_off");
    if (so[0] != 0) return fail(h, VBX_ERR_ARG, "vbx_init_turns: spk_off[0] must be 0");
    for (int b = 0; b < pl.n_rec; ++b) {
        const int64_t K = so[b + 1] - so[b];
        if (K < 0) return fail(h, VBX_ERR_ARG, "vbx_init_turns: recording " + std::to_string(b) + " has a negative speaker count");
        if (K > pl.S)
            return fail(h, VBX_ERR_ARG, "vbx_init_turns: recording " + std::to_string(b) + " has " + std::to_string(K) +
                                            " speakers, more than the plan's S = " + std::to_string(pl.S));
    }
    std::vector<int64_t> to(so[pl.n_rec] + 1);
    e = cudaMemcpyAsync(to.data(), turn_off, to.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(h, e, "vbx_init_turns: reading turn_off");
    if (to[0] != 0) return fail(h, VBX_ERR_ARG, "vbx_init_turns: turn_off[0] must be 0");
    for (size_t k = 0; k + 1 < to.size(); ++k)
        if (to[k + 1] < to[k])
            return fail(h, VBX_ERR_ARG, "vbx_init_turns: speaker " + std::to_string(k) + " has a negative turn count");
    if (to.back() > 0 && (!turn_lo || !turn_hi || !turn_cum)) return fail(h, VBX_ERR_ARG, "vbx_init_turns: null pointer");
    return counted(h, vbx::launch_init_turns(pl, seg, spk_off, turn_off, turn_lo, turn_hi, turn_cum, smoothing, gamma_out,
                                             pi_out, out_is_f64 != 0, st), "init_turns");
}

int vbx_init_random(vbx_handle_t h, const uint64_t *rec_key, const uint64_t *seed, const int32_t *n_states,
                    void *gamma_out, void *pi_out, int32_t out_is_f64, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_init_random: call vbx_plan or vbx_plan_f64 first");
    const vbx::Plan &pl = h->plan;
    if (pl.n_rec == 0) return VBX_OK;
    if (!rec_key || !seed || !pi_out || (pl.n_frames && !gamma_out))
        return fail(h, VBX_ERR_ARG, "vbx_init_random: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_init_random(pl, rec_key, seed, n_states, gamma_out, pi_out, out_is_f64 != 0,
                                              (cudaStream_t)stream), "init_random");
}

int vbx_ahc_workspace_bytes(vbx_handle_t h, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    if (!h->planned || h->f64_only) return fail(h, VBX_ERR_STATE, "vbx_ahc_workspace_bytes: call vbx_plan first");
    *bytes_out = h->ahc_need;
    return VBX_OK;
}

int vbx_ahc(vbx_handle_t h, const void *x, int32_t x_is_f64, int32_t dim, void *workspace, size_t workspace_bytes,
            double *Z_out, double *thr_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_ahc");
    if (!h->planned || h->f64_only) return fail(h, VBX_ERR_STATE, "vbx_ahc: call vbx_plan first");
    if (dim < 1) return fail(h, VBX_ERR_ARG, "vbx_ahc: dim < 1");
    if (h->plan.n_rec == 0) return VBX_OK;
    if (!workspace || !thr_out || (h->plan.n_frames && (!x || !Z_out))) return fail(h, VBX_ERR_ARG, "vbx_ahc: null pointer");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VBX_ERR_ARG, "vbx_ahc: workspace must be 256-byte aligned");
    if (workspace_bytes < h->ahc_need) return fail(h, VBX_ERR_ARG, "vbx_ahc: workspace smaller than vbx_ahc_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    std::string why;
    int n = vbx::launch_ahc(h->plan, h->ahc_d_off, x, x_is_f64, dim, workspace, workspace_bytes, Z_out, thr_out,
                            (cudaStream_t)stream, &why);
    if (n < 0) return fail(h, VBX_ERR_CUDA, "vbx_ahc: " + why);
    h->launches += n;
    return VBX_OK;
}

// the sizes M [G] of vbx_link_batch's problems: each in [0, VBX_LINK_MAX_SPEAKERS], their sum within one launch's grid
static int check_problem_sizes(vbx_handle_t h, const std::string &who, int32_t G, const int64_t *M) {
    if (G < 0) return fail(h, VBX_ERR_ARG, who + ": G < 0");
    if (G > 0 && !M) return fail(h, VBX_ERR_ARG, who + ": null pointer");
    int64_t total = 0;
    for (int32_t g = 0; g < G; ++g) {
        if (M[g] < 0 || M[g] > VBX_LINK_MAX_SPEAKERS)
            return fail(h, VBX_ERR_ARG, who + ": M[" + std::to_string(g) + "] must lie in [0, VBX_LINK_MAX_SPEAKERS]");
        total += M[g];
        if (total > INT32_MAX) return fail(h, VBX_ERR_ARG, who + ": more than 2^31 - 1 speakers in all");
    }
    return VBX_OK;
}

int vbx_link_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    const int rc = check_problem_sizes(h, "vbx_link_batch_workspace_bytes", G, M);
    if (rc != VBX_OK) return rc;
    *bytes_out = vbx::link_batch_workspace_bytes(G, M);
    return VBX_OK;
}

// c [G] = Fa[g] / Fb[g], each finite and >= 0
static int problem_scalars(vbx_handle_t h, const std::string &who, int32_t G, const double *Fa, const double *Fb,
                           std::vector<double> *c) {
    if (G > 0 && (!Fa || !Fb)) return fail(h, VBX_ERR_ARG, who + ": null pointer");
    c->assign(G, 0.0);
    for (int32_t g = 0; g < G; ++g) {
        (*c)[g] = Fa[g] / Fb[g];
        if (!((*c)[g] >= 0.0) || (*c)[g] == INFINITY)
            return fail(h, VBX_ERR_ARG, who + ": Fa[" + std::to_string(g) + "] / Fb[" + std::to_string(g) +
                                            "] must be finite and >= 0");
    }
    return VBX_OK;
}

int vbx_link_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                   const int32_t *speaker, const int64_t *M, const int32_t *speaker_rec, const double *Fa,
                   const double *Fb, void *workspace, size_t workspace_bytes, double *n_out, double *F_out,
                   double *dist_out, double *Z_out, const double *mean, const double *std, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_link_batch");
    const std::string who("vbx_link_batch");
    int rc = check_problem_sizes(h, who, G, M);
    if (rc != VBX_OK) return rc;
    if (N < 0) return fail(h, VBX_ERR_ARG, who + ": N < 0");
    if (R < 1 || R > vbx::kMaxR) return fail(h, VBX_ERR_ARG, who + ": R must lie in [1, 128]");
    std::vector<double> c;
    rc = problem_scalars(h, who, G, Fa, Fb, &c);
    if (rc != VBX_OK) return rc;
    if (!mean != !std) return fail(h, VBX_ERR_ARG, who + ": give both of mean and std, or neither");
    int64_t total = 0, largest = 0;
    for (int32_t g = 0; g < G; ++g) {
        total += M[g];
        largest = std::max(largest, M[g]);
    }
    if (total == 0) return VBX_OK;
    if (!Phi || !speaker_rec || !workspace || (N > 0 && (!fea || !speaker)) || (largest >= 2 && !Z_out))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::link_batch_workspace_bytes(G, M))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_link_batch_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_link_batch(fea, Phi, speaker, N, R, speaker_rec, G, M, c.data(), workspace, n_out,
                                             F_out, dist_out, Z_out, (cudaStream_t)stream, mean, std), "link_batch");
}

int vbx_enroll_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, int64_t E, int64_t N_e,
                                     int64_t max_k, int32_t n_thr, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    const std::string who("vbx_enroll_batch_workspace_bytes");
    const int rc = check_problem_sizes(h, who, G, M);
    if (rc != VBX_OK) return rc;
    if (E < 1 || N_e < 1 || max_k < 0 || n_thr < 1)
        return fail(h, VBX_ERR_ARG, who + ": need E, N_e, n_thr >= 1 and max_k >= 0");
    *bytes_out = vbx::enroll_batch_workspace_bytes(G, M, E, N_e, max_k, n_thr, h->sms);
    return VBX_OK;
}

int vbx_enroll_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                     const int32_t *speaker, const int64_t *M, const int64_t *speaker_rec_offsets, int32_t n_rec,
                     const float *enroll_fea, int64_t N_e, const int32_t *enroll_speaker, int64_t E, const double *Fa,
                     const double *Fb, const double *thresholds, int32_t n_thr, void *workspace,
                     size_t workspace_bytes, int32_t *assign_out, double *best_llr_out, double *llr_out, double *n_out,
                     double *F_out, double *n_enroll_out, double *F_enroll_out, const double *mean, const double *std,
                     const double *enroll_mean, const double *enroll_std, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_enroll_batch");
    const std::string who("vbx_enroll_batch");
    int rc = check_problem_sizes(h, who, G, M);
    if (rc != VBX_OK) return rc;
    if (N < 0 || n_rec < 0 || N_e < 1 || E < 1 || n_thr < 1)
        return fail(h, VBX_ERR_ARG, who + ": need N, n_rec >= 0 and N_e, E, n_thr >= 1");
    if (R < 1 || R > vbx::kMaxR) return fail(h, VBX_ERR_ARG, who + ": R must lie in [1, 128]");
    std::vector<double> c;
    rc = problem_scalars(h, who, G, Fa, Fb, &c);
    if (rc != VBX_OK) return rc;
    if (!thresholds) return fail(h, VBX_ERR_ARG, who + ": null pointer");
    for (int32_t k = 0; k < n_thr; ++k)
        if (!(std::fabs(thresholds[k]) <= 1e15))
            return fail(h, VBX_ERR_ARG, who + ": |thresholds[" + std::to_string(k) + "]| must be <= 1e15");
    int64_t total = 0;
    for (int32_t g = 0; g < G; ++g) total += M[g];
    const bool norm = mean || std || enroll_mean || enroll_std;
    if (norm && !(enroll_mean && enroll_std && ((mean && std) || total == 0)))
        return fail(h, VBX_ERR_ARG, who + ": give all four of mean, std, enroll_mean and enroll_std, or none");
    if (!Phi || !workspace || !enroll_fea || !enroll_speaker || (G > 0 && !speaker_rec_offsets) ||
        (N > 0 && (!fea || !speaker)) || (total > 0 && (!assign_out || !best_llr_out)))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    int64_t max_k = 0;
    for (int32_t g = 0; g < G; ++g) {
        const int64_t *ro = speaker_rec_offsets + (size_t)g * (n_rec + 1);
        if (ro[0] != 0 || ro[n_rec] != M[g])
            return fail(h, VBX_ERR_ARG, who + ": speaker_rec_offsets row " + std::to_string(g) + " must run from 0 to M[" +
                                            std::to_string(g) + "]");
        for (int32_t b = 0; b < n_rec; ++b) {
            const int64_t k = ro[b + 1] - ro[b];
            if (k < 0) return fail(h, VBX_ERR_ARG, who + ": speakers are not packed by recording (offsets decrease)");
            max_k = std::max(max_k, k);
        }
    }
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::enroll_batch_workspace_bytes(G, M, E, N_e, max_k, n_thr, h->sms))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_enroll_batch_workspace_bytes()");
    if (G == 0) return VBX_OK;
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_enroll_batch(fea, Phi, N, R, speaker, G, M, speaker_rec_offsets, n_rec, enroll_fea,
                                               N_e, enroll_speaker, E, c.data(), thresholds, n_thr, workspace, h->sms,
                                               assign_out, best_llr_out, llr_out, n_out, F_out, n_enroll_out,
                                               F_enroll_out, (cudaStream_t)stream, mean, std, enroll_mean, enroll_std),
                   "enroll_batch");
}

int vbx_cohort_stats_batch_workspace_bytes(vbx_handle_t h, int32_t G, const int64_t *M, int64_t C, int64_t N_c,
                                           size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    const std::string who("vbx_cohort_stats_batch_workspace_bytes");
    const int rc = check_problem_sizes(h, who, G, M);
    if (rc != VBX_OK) return rc;
    if (C < 2 || N_c < 1) return fail(h, VBX_ERR_ARG, who + ": need C >= 2 and N_c >= 1");
    *bytes_out = vbx::cohort_batch_workspace_bytes(G, M, C, N_c);
    return VBX_OK;
}

int vbx_cohort_stats_batch(vbx_handle_t h, const float *fea, const float *Phi, int64_t N, int32_t R, int32_t G,
                           const int32_t *speaker, const int64_t *M, const float *cohort_fea, int64_t N_c,
                           const int32_t *cohort_speaker, int64_t C, const double *Fa, const double *Fb, int32_t top_k,
                           void *workspace, size_t workspace_bytes, double *mean_out, double *std_out,
                           double *scores_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_cohort_stats_batch");
    const std::string who("vbx_cohort_stats_batch");
    int rc = check_problem_sizes(h, who, G, M);
    if (rc != VBX_OK) return rc;
    if (N < 0 || N_c < 1 || C < 2) return fail(h, VBX_ERR_ARG, who + ": need N >= 0, N_c >= 1 and C >= 2");
    if (top_k < 2) return fail(h, VBX_ERR_ARG, who + ": top_k must be >= 2");
    if (R < 1 || R > vbx::kMaxR) return fail(h, VBX_ERR_ARG, who + ": R must lie in [1, 128]");
    std::vector<double> c;
    rc = problem_scalars(h, who, G, Fa, Fb, &c);
    if (rc != VBX_OK) return rc;
    int64_t total = 0;
    for (int32_t g = 0; g < G; ++g) total += M[g];
    if (total == 0) return VBX_OK;
    if (!Phi || !workspace || !cohort_fea || !cohort_speaker || !mean_out || !std_out || (N > 0 && (!fea || !speaker)))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::cohort_batch_workspace_bytes(G, M, C, N_c))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_cohort_stats_batch_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_cohort_batch(fea, Phi, N, R, speaker, G, M, cohort_fea, N_c, cohort_speaker, C,
                                               c.data(), top_k, workspace, mean_out, std_out, scores_out,
                                               (cudaStream_t)stream),
                   "cohort_batch");
}

int vbx_verify_score_workspace_bytes(vbx_handle_t h, int32_t M_e, int32_t M_t, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    if (M_e < 1 || M_t < 1) return fail(h, VBX_ERR_ARG, "vbx_verify_score_workspace_bytes: need M_e, M_t >= 1");
    *bytes_out = vbx::verify_score_workspace_bytes(M_e, M_t);
    return VBX_OK;
}

int vbx_verify_score(vbx_handle_t h, const float *enroll_fea, int64_t N_e, const int32_t *enroll_item, int32_t M_e,
                     const float *test_fea, int64_t N_t, const int32_t *test_item, int32_t M_t, int32_t R,
                     const float *Phi, double Fa, double Fb, const int32_t *trial_enroll, const int32_t *trial_test,
                     int64_t T, const double *enroll_mean, const double *enroll_std, const double *test_mean,
                     const double *test_std, void *workspace, size_t workspace_bytes, double *score_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_verify_score");
    const std::string who("vbx_verify_score");
    if (M_e < 1 || M_t < 1 || N_e < 1 || N_t < 1 || T < 0)
        return fail(h, VBX_ERR_ARG, who + ": need M_e, M_t, N_e, N_t >= 1 and T >= 0");
    if (R < 1 || R > vbx::kMaxR) return fail(h, VBX_ERR_ARG, who + ": R must lie in [1, 128]");
    if (!(std::isfinite(Fa) && Fa > 0.0 && std::isfinite(Fb) && Fb > 0.0))
        return fail(h, VBX_ERR_ARG, who + ": Fa and Fb must be finite and > 0");
    const double c = Fa / Fb;
    if (!(c > 0.0) || c == INFINITY) return fail(h, VBX_ERR_ARG, who + ": Fa / Fb must be finite and > 0");
    const int n_norm = !!enroll_mean + !!enroll_std + !!test_mean + !!test_std;
    if (n_norm != 0 && n_norm != 4)
        return fail(h, VBX_ERR_ARG, who + ": give all four of enroll_mean, enroll_std, test_mean and test_std, or none");
    if (!enroll_fea || !enroll_item || !test_fea || !test_item || !Phi || !workspace ||
        (T > 0 && (!trial_enroll || !trial_test || !score_out)))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::verify_score_workspace_bytes(M_e, M_t))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_verify_score_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_verify_score(enroll_fea, N_e, enroll_item, M_e, test_fea, N_t, test_item, M_t, R, Phi,
                                               c, trial_enroll, trial_test, T, enroll_mean, enroll_std, test_mean,
                                               test_std, workspace, score_out, (cudaStream_t)stream),
                   "verify_score");
}

int vbx_verify_metrics_workspace_bytes(vbx_handle_t h, int64_t T, int32_t n_op, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    if (T < 1 || n_op < 1 || n_op > VBX_VERIFY_MAX_OPS)
        return fail(h, VBX_ERR_ARG, "vbx_verify_metrics_workspace_bytes: need T >= 1 and n_op in [1, VBX_VERIFY_MAX_OPS]");
    DeviceGuard guard(h->device);         // the sort's temporary storage is sized for the handle's device
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    *bytes_out = vbx::verify_metrics_workspace_bytes(T, n_op);
    return VBX_OK;
}

int vbx_verify_metrics(vbx_handle_t h, const double *scores, const uint8_t *is_target, int64_t T, int32_t n_op,
                       const double *p_target, double c_miss, double c_fa, void *workspace, size_t workspace_bytes,
                       int64_t *counts_out, double *eer_out, double *cllr_out, double *min_dcf_out,
                       double *threshold_out, double *act_dcf_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_verify_metrics");
    const std::string who("vbx_verify_metrics");
    if (T < 1 || n_op < 1 || n_op > VBX_VERIFY_MAX_OPS)
        return fail(h, VBX_ERR_ARG, who + ": need T >= 1 and n_op in [1, VBX_VERIFY_MAX_OPS]");
    if (!(std::isfinite(c_miss) && c_miss > 0.0 && std::isfinite(c_fa) && c_fa > 0.0))
        return fail(h, VBX_ERR_ARG, who + ": c_miss and c_fa must be finite and > 0");
    if (!scores || !is_target || !p_target || !workspace || !counts_out || !eer_out || !cllr_out || !min_dcf_out ||
        !threshold_out || !act_dcf_out)
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    std::vector<double> ops(4 * (size_t)n_op);
    for (int32_t o = 0; o < n_op; ++o) {
        const double p = p_target[o];
        if (!(p > 0.0 && p < 1.0))
            return fail(h, VBX_ERR_ARG, who + ": p_target[" + std::to_string(o) + "] must lie in (0, 1)");
        ops[4 * o] = c_miss * p;
        ops[4 * o + 1] = c_fa * (1.0 - p);
        ops[4 * o + 2] = std::min(ops[4 * o], ops[4 * o + 1]);
        ops[4 * o + 3] = std::log(ops[4 * o + 1] / ops[4 * o]);
        if (!(ops[4 * o + 2] > 0.0) || !std::isfinite(ops[4 * o + 3]))
            return fail(h, VBX_ERR_ARG, who + ": the costs of p_target[" + std::to_string(o) + "] are out of range");
    }
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (workspace_bytes < vbx::verify_metrics_workspace_bytes(T, n_op))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_verify_metrics_workspace_bytes()");
    return counted(h, vbx::launch_verify_metrics(scores, is_target, T, ops.data(), n_op, workspace,
                                                 reinterpret_cast<long long *>(counts_out), eer_out, cllr_out,
                                                 min_dcf_out, threshold_out, act_dcf_out, (cudaStream_t)stream),
                   "verify_metrics");
}

int vbx_verify_calibrate_workspace_bytes(vbx_handle_t h, int64_t T, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    if (T < 1) return fail(h, VBX_ERR_ARG, "vbx_verify_calibrate_workspace_bytes: need T >= 1");
    DeviceGuard guard(h->device);         // the sort's temporary storage is sized for the handle's device
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    *bytes_out = vbx::verify_calibrate_workspace_bytes(T);
    return VBX_OK;
}

int vbx_verify_calibrate(vbx_handle_t h, const double *scores, const uint8_t *is_target, int64_t T, double prior,
                         void *workspace, size_t workspace_bytes, int64_t *info_out, double *out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_verify_calibrate");
    const std::string who("vbx_verify_calibrate");
    if (T < 1) return fail(h, VBX_ERR_ARG, who + ": need T >= 1");
    if (!(prior > 0.0 && prior < 1.0)) return fail(h, VBX_ERR_ARG, who + ": prior must lie in (0, 1)");
    if (!std::isfinite(std::log(prior / (1.0 - prior))))
        return fail(h, VBX_ERR_ARG, who + ": the log odds of prior are out of range");
    if (!scores || !is_target || !workspace || !info_out || !out) return fail(h, VBX_ERR_ARG, who + ": null pointer");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    if (workspace_bytes < vbx::verify_calibrate_workspace_bytes(T))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_verify_calibrate_workspace_bytes()");
    return counted(h, vbx::launch_verify_calibrate(scores, is_target, T, prior, workspace,
                                                   reinterpret_cast<long long *>(info_out), out, (cudaStream_t)stream),
                   "verify_calibrate");
}

int vbx_f64_workspace_bytes(vbx_handle_t h, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_f64_workspace_bytes: call vbx_plan first");
    *bytes_out = vbx::f64_workspace_bytes(h->plan);
    return VBX_OK;
}

}  // extern "C"

static int run_f64_impl(vbx_handle_t h, void *workspace, size_t workspace_bytes, const double *fea, const double *Phi,
                        double *gamma_io, double *pi_io, const int32_t *n_states, double Fa, double Fb, double loop_prob,
                        int32_t max_iters, double epsilon, double *alpha_io, double *invL_io, int32_t warm_start,
                        double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream,
                        const double *prior_n = nullptr, const double *prior_F = nullptr) {
    Range nvtx_range("vbx_run_f64");
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_run_f64: call vbx_plan first");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    const vbx::Plan &pl = h->plan;
    if (pl.n_rec == 0) return VBX_OK;
    if (!workspace || workspace_bytes < vbx::f64_workspace_bytes(pl)) return fail(h, VBX_ERR_STATE, "vbx_run_f64: workspace too small");
    if (max_iters < 0 || !(Fb != 0.0)) return fail(h, VBX_ERR_ARG, "vbx_run_f64: bad max_iters / Fb");
    if (!Li_out || !n_iters_out || !flags_out || !pi_io || (pl.n_frames && (!fea || !Phi || !gamma_io)))
        return fail(h, VBX_ERR_ARG, "vbx_run_f64: null pointer");
    if (warm_start && (!alpha_io || !invL_io)) return fail(h, VBX_ERR_ARG, "vbx_run_f64: warm_start needs alpha_io and invL_io");
    return counted(h, vbx::launch_run_f64(pl, workspace, fea, Phi, gamma_io, pi_io, n_states, Fa, Fb, loop_prob, max_iters, epsilon,
                                          alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, (cudaStream_t)stream,
                                          prior_n, prior_F),
                   "run_f64");
}

extern "C" {

int vbx_run_f64(vbx_handle_t h, void *workspace, size_t workspace_bytes, const double *fea, const double *Phi,
                double *gamma_io, double *pi_io, const int32_t *n_states, double Fa, double Fb, double loop_prob,
                int32_t max_iters, double epsilon, double *alpha_io, double *invL_io, int32_t warm_start,
                double *Li_out, int32_t *n_iters_out, int32_t *flags_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    return run_f64_impl(h, workspace, workspace_bytes, fea, Phi, gamma_io, pi_io, n_states, Fa, Fb, loop_prob, max_iters,
                        epsilon, alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, stream);
}

int vbx_run_f64_prior(vbx_handle_t h, void *workspace, size_t workspace_bytes, const double *fea, const double *Phi,
                      double *gamma_io, double *pi_io, const int32_t *n_states, double Fa, double Fb, double loop_prob,
                      int32_t max_iters, double epsilon, double *alpha_io, double *invL_io, int32_t warm_start,
                      double *Li_out, int32_t *n_iters_out, int32_t *flags_out, const double *prior_n,
                      const double *prior_F, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!prior_n || !prior_F) return fail(h, VBX_ERR_ARG, "vbx_run_f64_prior: prior_n and prior_F must be device arrays");
    return run_f64_impl(h, workspace, workspace_bytes, fea, Phi, gamma_io, pi_io, n_states, Fa, Fb, loop_prob, max_iters,
                        epsilon, alpha_io, invL_io, warm_start, Li_out, n_iters_out, flags_out, stream, prior_n, prior_F);
}

int vbx_forward_backward(vbx_handle_t h, const double *lls, const double *tr, const double *ip, int32_t T, int32_t S,
                         double *post_out, double *tll_out, double *lfw_out, double *lbw_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (T < 1 || S < 1 || S > 1024) return fail(h, VBX_ERR_ARG, "vbx_forward_backward: need T >= 1 and 1 <= S <= 1024");
    if (!lls || !tr || !ip || !post_out || !tll_out || !lfw_out || !lbw_out) return fail(h, VBX_ERR_ARG, "vbx_forward_backward: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_fb_dense(lls, tr, ip, T, S, post_out, tll_out, lfw_out, lbw_out, (cudaStream_t)stream), "fb_dense");
}

int vbx_score(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo, const int64_t *sys_hi,
              const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo, const int64_t *reg_hi, const uint64_t *reg_mask,
              const int32_t *n_ref, int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets,
              const int32_t *labels, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
              int64_t *covered_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_score");
    if (n_rec < 0 || n_entries < 0 || max_cells < 0) return fail(h, VBX_ERR_ARG, "vbx_score: negative count");
    if (n_entries == 0) return VBX_OK;
    if (n_rec == 0) return fail(h, VBX_ERR_ARG, "vbx_score: entries need at least one recording");
    if (!sys_offsets || !sys_lo || !sys_hi || !sys_join_hi || !reg_offsets || !reg_lo || !reg_hi || !reg_mask || !n_ref || !entry_rec ||
        !label_offsets || !labels || !n_labels || !o_offsets || !covered_out || !fa_out || !flags_out ||
        (max_cells > 0 && !O_out))
        return fail(h, VBX_ERR_ARG, "vbx_score: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_score(n_rec, sys_offsets, sys_lo, sys_hi, sys_join_hi, reg_offsets, reg_lo, reg_hi, reg_mask,
                                        nullptr, n_ref, n_entries, entry_rec, label_offsets, labels, nullptr, n_labels,
                                        o_offsets, max_cells, covered_out, fa_out, O_out, flags_out, nullptr, nullptr,
                                        (cudaStream_t)stream),
                   "score");
}

int vbx_score_overlap(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo,
                      const int64_t *sys_hi, const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo,
                      const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_overlap, const int32_t *n_ref,
                      int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets, const int32_t *labels,
                      const int32_t *labels2, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
                      int64_t *both_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_score_overlap");
    if (n_rec < 0 || n_entries < 0 || max_cells < 0) return fail(h, VBX_ERR_ARG, "vbx_score_overlap: negative count");
    if (n_entries == 0) return VBX_OK;
    if (n_rec == 0) return fail(h, VBX_ERR_ARG, "vbx_score_overlap: entries need at least one recording");
    if (!sys_offsets || !sys_lo || !sys_hi || !sys_join_hi || !reg_offsets || !reg_lo || !reg_hi || !reg_mask ||
        !reg_overlap || !n_ref || !entry_rec || !label_offsets || !labels || !labels2 || !n_labels || !o_offsets ||
        !both_out || !fa_out || !flags_out || (max_cells > 0 && !O_out))
        return fail(h, VBX_ERR_ARG, "vbx_score_overlap: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_score(n_rec, sys_offsets, sys_lo, sys_hi, sys_join_hi, reg_offsets, reg_lo, reg_hi, reg_mask,
                                        reg_overlap, n_ref, n_entries, entry_rec, label_offsets, labels, labels2, n_labels,
                                        o_offsets, max_cells, both_out, fa_out, O_out, flags_out, nullptr, nullptr,
                                        (cudaStream_t)stream),
                   "score_overlap");
}

int vbx_score_jer(vbx_handle_t h, int32_t n_rec, const int64_t *sys_offsets, const int64_t *sys_lo,
                  const int64_t *sys_hi, const int64_t *sys_join_hi, const int64_t *reg_offsets, const int64_t *reg_lo,
                  const int64_t *reg_hi, const uint64_t *reg_mask, const uint8_t *reg_overlap, const int32_t *n_ref,
                  int32_t n_entries, const int32_t *entry_rec, const int64_t *label_offsets, const int32_t *labels,
                  const int32_t *labels2, const int32_t *n_labels, const int64_t *o_offsets, int64_t max_cells,
                  int64_t *both_out, int64_t *fa_out, int64_t *O_out, int32_t *flags_out, const int64_t *t_offsets,
                  int64_t *label_time_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_score_jer");
    if (n_rec < 0 || n_entries < 0 || max_cells < 0) return fail(h, VBX_ERR_ARG, "vbx_score_jer: negative count");
    if (n_entries == 0) return VBX_OK;
    if (n_rec == 0) return fail(h, VBX_ERR_ARG, "vbx_score_jer: entries need at least one recording");
    if (!sys_offsets || !sys_lo || !sys_hi || !sys_join_hi || !reg_offsets || !reg_lo || !reg_hi || !reg_mask || !n_ref ||
        !entry_rec || !label_offsets || !labels || !n_labels || !o_offsets || !t_offsets || !label_time_out || !both_out ||
        !fa_out || !flags_out || (max_cells > 0 && !O_out))
        return fail(h, VBX_ERR_ARG, "vbx_score_jer: null pointer");
    if (!reg_overlap != !labels2)
        return fail(h, VBX_ERR_ARG, "vbx_score_jer: reg_overlap and labels2 must both be given or both be NULL");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_score(n_rec, sys_offsets, sys_lo, sys_hi, sys_join_hi, reg_offsets, reg_lo, reg_hi, reg_mask,
                                        reg_overlap, n_ref, n_entries, entry_rec, label_offsets, labels, labels2, n_labels,
                                        o_offsets, max_cells, both_out, fa_out, O_out, flags_out, t_offsets,
                                        label_time_out, (cudaStream_t)stream),
                   labels2 ? "score_jer_overlap" : "score_jer");
}

static int check_combine_sizes(vbx_handle_t h, const std::string &who, int32_t n_rec, int32_t K, int32_t max_labels) {
    if (n_rec < 0) return fail(h, VBX_ERR_ARG, who + ": negative count");
    if (K < 2 || K > 32) return fail(h, VBX_ERR_ARG, who + ": K must lie in [2, 32]");
    if (max_labels < 1 || max_labels > 128) return fail(h, VBX_ERR_ARG, who + ": max_labels must lie in [1, 128]");
    if ((int64_t)n_rec * (K * (K - 1) / 2 + K) > INT32_MAX)
        return fail(h, VBX_ERR_ARG, who + ": n_rec (K (K - 1) / 2 + K) must stay below 2^31");
    return VBX_OK;
}

int vbx_combine_workspace_bytes(vbx_handle_t h, int32_t n_rec, int32_t K, int32_t max_labels, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    const int rc = check_combine_sizes(h, "vbx_combine_workspace_bytes", n_rec, K, max_labels);
    if (rc != VBX_OK) return rc;
    *bytes_out = vbx::combine_workspace_bytes(n_rec, K, max_labels);
    return VBX_OK;
}

int vbx_combine(vbx_handle_t h, int32_t n_rec, const int64_t *offsets, int64_t N, const int64_t *lo, const int64_t *hi,
                int32_t K, const int32_t *labels, const int32_t *labels2, const int32_t *n_labels, int32_t max_labels,
                const double *weights, void *workspace, size_t workspace_bytes, int32_t *labels_out,
                int32_t *labels2_out, int32_t *order_out, double *weights_out, int64_t *D_out, int32_t *map_out,
                int32_t *n_global_out, int32_t *flags_out, int64_t *O_out, int64_t *L_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_combine");
    const std::string who("vbx_combine");
    const int rc = check_combine_sizes(h, who, n_rec, K, max_labels);
    if (rc != VBX_OK) return rc;
    if (N < 0) return fail(h, VBX_ERR_ARG, who + ": negative count");
    if (weights)
        for (int32_t k = 0; k < K; ++k)
            if (!(std::isfinite(weights[k]) && weights[k] > 0.0))
                return fail(h, VBX_ERR_ARG, who + ": weights[" + std::to_string(k) + "] must be finite and > 0");
    if (n_rec == 0) {
        if (N != 0) return fail(h, VBX_ERR_ARG, who + ": intervals need at least one recording");
        return VBX_OK;
    }
    if (!offsets || !n_labels || !workspace || !order_out || !weights_out || !D_out || !map_out || !n_global_out ||
        !flags_out || (N > 0 && (!lo || !hi || !labels || !labels2 || !labels_out || !labels2_out)))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    for (int64_t i = 0; i < (int64_t)n_rec * K; ++i)
        if (n_labels[i] < 0 || n_labels[i] > max_labels)
            return fail(h, VBX_ERR_ARG, who + ": n_labels[" + std::to_string(i / K) + ", " + std::to_string(i % K) +
                                            "] must lie in [0, max_labels]");
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::combine_workspace_bytes(n_rec, K, max_labels))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_combine_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_combine(n_rec, offsets, N, lo, hi, K, labels, labels2, n_labels, max_labels, weights,
                                          workspace, labels_out, labels2_out, order_out, weights_out, D_out, map_out,
                                          n_global_out, flags_out, O_out, L_out, (cudaStream_t)stream),
                   "combine");
}

static int check_scatter_sizes(vbx_handle_t h, const std::string &who, int64_t N, int32_t D, int32_t K) {
    if (N < 0 || K < 1) return fail(h, VBX_ERR_ARG, who + ": N must be >= 0 and K >= 1");
    if (D < 1 || D > 1024) return fail(h, VBX_ERR_ARG, who + ": D must lie in [1, 1024]");
    return VBX_OK;
}

int vbx_class_scatter_workspace_bytes(vbx_handle_t h, int64_t N, int32_t D, int32_t K, size_t *bytes_out) {
    if (!h || !bytes_out) return VBX_ERR_ARG;
    const int rc = check_scatter_sizes(h, "vbx_class_scatter_workspace_bytes", N, D, K);
    if (rc != VBX_OK) return rc;
    *bytes_out = vbx::class_scatter_workspace_bytes(N, D, K);
    return VBX_OK;
}

int vbx_class_scatter(vbx_handle_t h, const float *X, int64_t N, int32_t D, int32_t K, const int64_t *offsets,
                      void *workspace, size_t workspace_bytes, double *means_out, double *scatter_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_class_scatter");
    const std::string who("vbx_class_scatter");
    const int rc = check_scatter_sizes(h, who, N, D, K);
    if (rc != VBX_OK) return rc;
    if ((N > 0 && !X) || !offsets || !workspace || !means_out || !scatter_out)
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    if (misaligned16(h, who, {{X, "X"}}) != VBX_OK) return VBX_ERR_ARG;
    if (offsets[0] != 0 || offsets[K] != N) return fail(h, VBX_ERR_ARG, who + ": offsets must run from 0 to N");
    for (int32_t i = 0; i < K; ++i)
        if (offsets[i + 1] < offsets[i])
            return fail(h, VBX_ERR_ARG, who + ": offsets decrease at class " + std::to_string(i));
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0)
        return fail(h, VBX_ERR_ARG, who + ": workspace must be 256-byte aligned");
    if (workspace_bytes < vbx::class_scatter_workspace_bytes(N, D, K))
        return fail(h, VBX_ERR_ARG, who + ": workspace smaller than vbx_class_scatter_workspace_bytes()");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_class_scatter(X, N, D, K, offsets, workspace, means_out, scatter_out,
                                                (cudaStream_t)stream),
                   "class_scatter");
}

static int check_stream_sizes(vbx_handle_t h, const std::string &who, int32_t n, int32_t C, int32_t R, int32_t S_max,
                              int32_t S) {
    if (n < 0 || C < 0) return fail(h, VBX_ERR_ARG, who + ": n and C must be >= 0");
    if (R < 1 || R > vbx::kMaxR) return fail(h, VBX_ERR_ARG, who + ": R must lie in [1, 128]");
    if (S_max < 1 || S_max > 128 || S < 1 || S > 128) return fail(h, VBX_ERR_ARG, who + ": S_max and S must lie in [1, 128]");
    return VBX_OK;
}

int vbx_stream_window(vbx_handle_t h, int32_t n, int32_t C, int32_t R, int32_t S_max, int32_t S, const int32_t *slot,
                      const int64_t *blk_off, const int64_t *win_off, const int32_t *blk_lab, const int32_t *n_clusters,
                      const float *blk_fea, double smoothing, const float *ctx_fea, const int32_t *ctx_lab,
                      const int64_t *count, const int32_t *K, const double *n_hist, const double *F_hist, float *fea_out,
                      float *gamma_out, float *pi_out, int32_t *n_states_out, double *prior_n_out, double *prior_F_out,
                      void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_stream_window");
    const std::string who("vbx_stream_window");
    const int rc = check_stream_sizes(h, who, n, C, R, S_max, S);
    if (rc != VBX_OK) return rc;
    if (!std::isfinite(smoothing)) return fail(h, VBX_ERR_ARG, who + ": smoothing must be finite");
    if (n > 0 && (!slot || !blk_off || !win_off || !blk_lab || !n_clusters || !blk_fea || (C > 0 && (!ctx_fea || !ctx_lab)) ||
                  !count || !K || !n_hist || !F_hist || !fea_out || !gamma_out || !pi_out || !n_states_out ||
                  !prior_n_out || !prior_F_out))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_stream_window(n, C, R, S_max, S, slot, blk_off, win_off, blk_lab, n_clusters, blk_fea,
                                                smoothing, ctx_fea, ctx_lab, count, K, n_hist, F_hist, fea_out, gamma_out,
                                                pi_out, n_states_out, prior_n_out, prior_F_out, (cudaStream_t)stream),
                   "stream_window");
}

int vbx_stream_commit(vbx_handle_t h, int32_t n, int32_t C, int32_t R, int32_t S_max, const int32_t *slot,
                      const int64_t *blk_off, const int64_t *win_off, const float *blk_fea, const int32_t *first,
                      float *ctx_fea, int32_t *ctx_lab, int64_t *count, int32_t *K, double *n_hist, double *F_hist,
                      int32_t *labels_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    Range nvtx_range("vbx_stream_commit");
    const std::string who("vbx_stream_commit");
    const int rc = check_stream_sizes(h, who, n, C, R, S_max, S_max);
    if (rc != VBX_OK) return rc;
    if (n > 0 && (!slot || !blk_off || !win_off || !blk_fea || !first || (C > 0 && (!ctx_fea || !ctx_lab)) || !count ||
                  !K || !n_hist || !F_hist || !labels_out))
        return fail(h, VBX_ERR_ARG, who + ": null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    return counted(h, vbx::launch_stream_commit(n, C, R, S_max, slot, blk_off, win_off, blk_fea, first, ctx_fea, ctx_lab,
                                                count, K, n_hist, F_hist, labels_out, (cudaStream_t)stream),
                   "stream_commit");
}

int vbx_attach_comm(vbx_handle_t h, void *nccl_comm, int32_t n_ranks, const char *libnccl_path) {
    if (!h) return VBX_ERR_ARG;
    if (!nccl_comm) {   // detach
        h->nccl_comm = nullptr;
        h->nccl_ranks = 1;
        return VBX_OK;
    }
    if (n_ranks < 1) return fail(h, VBX_ERR_ARG, "vbx_attach_comm: n_ranks < 1");
    if (!h->nccl_allreduce) {
        // the NCCL this process already talks through (torch's): find it without loading a second copy
        void *lib = nullptr;
        if (libnccl_path && *libnccl_path) lib = dlopen(libnccl_path, RTLD_NOW | RTLD_NOLOAD);
        if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!lib && libnccl_path && *libnccl_path) lib = dlopen(libnccl_path, RTLD_NOW);
        if (!lib) return fail(h, VBX_ERR_STATE, "vbx_attach_comm: libnccl.so.2 is not loaded in this process and no usable path was given");
        void *sym = dlsym(lib, "ncclAllReduce");
        if (!sym) return fail(h, VBX_ERR_STATE, "vbx_attach_comm: ncclAllReduce not found");
        h->nccl_allreduce = reinterpret_cast<int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t)>(sym);
    }
    h->nccl_comm = nccl_comm;
    h->nccl_ranks = n_ranks;
    return VBX_OK;
}

int vbx_elbo_trace(vbx_handle_t h, const double *Li, int32_t max_iters, double *trace_out, void *stream) {
    Range nvtx_range("vbx_elbo_trace");
    if (!h) return VBX_ERR_ARG;
    if (!h->planned) return fail(h, VBX_ERR_STATE, "vbx_elbo_trace: call vbx_plan first");
    if (max_iters < 1 || !trace_out || (h->plan.n_rec && !Li)) return fail(h, VBX_ERR_ARG, "vbx_elbo_trace: bad argument");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = counted(h, vbx::launch_elbo_trace(h->plan, Li, max_iters, trace_out, st), "elbo_trace");
    if (rc) return rc;
    if (h->nccl_comm && h->nccl_ranks > 1) {
        // the one collective of the path (SURVEY 8e): per-iteration ELBO sums and active counts over all GPUs
        const int nrc = h->nccl_allreduce(trace_out, trace_out, (size_t)2 * max_iters, /*ncclFloat64*/ 8, /*ncclSum*/ 0, h->nccl_comm, st);
        if (nrc != 0) return fail(h, VBX_ERR_CUDA, "vbx_elbo_trace: ncclAllReduce failed with code " + std::to_string(nrc));
    }
    return VBX_OK;
}

int vbx_get_gsum(vbx_handle_t h, double *gsum_out, void *stream) {
    if (!h) return VBX_ERR_ARG;
    if (!h->planned || !h->bound || !h->prepared) return fail(h, VBX_ERR_STATE, "vbx_get_gsum: call vbx_prepare_* first");
    if (h->plan.n_rec == 0) return VBX_OK;
    if (!gsum_out) return fail(h, VBX_ERR_ARG, "vbx_get_gsum: null pointer");
    DeviceGuard guard(h->device);
    if (guard.err != cudaSuccess) return cuda_fail(h, guard.err, "cudaSetDevice");
    const cudaError_t e = cudaMemcpyAsync(gsum_out, h->ws.gsum, sizeof(double) * h->plan.n_rec, cudaMemcpyDeviceToDevice,
                                          (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(h, e, "vbx_get_gsum");
    return VBX_OK;
}

int64_t vbx_launch_count(vbx_handle_t h) { return h ? h->launches : -1; }

int vbx_get_timings(vbx_handle_t h, double *ms_out, int64_t *count_out, int32_t reset) {
    if (!h) return VBX_ERR_ARG;
    DeviceGuard guard(h->device);
    for (size_t i = 0; i + 1 < h->ev_used; i += 2) {
        cudaError_t e = cudaEventSynchronize(h->ev_pool[i + 1]);
        if (e != cudaSuccess) return cuda_fail(h, e, "cudaEventSynchronize");
        float ms = 0.f;
        e = cudaEventElapsedTime(&ms, h->ev_pool[i], h->ev_pool[i + 1]);
        if (e != cudaSuccess) return cuda_fail(h, e, "cudaEventElapsedTime");
        const int cls = h->ev_class[i / 2];
        h->t_ms[cls] += ms;
        h->t_cnt[cls] += 1;
    }
    h->ev_used = 0;
    h->ev_class.clear();
    for (int c = 0; c < VBX_N_KERNEL_CLASSES; ++c) {
        if (ms_out) ms_out[c] = h->t_ms[c];
        if (count_out) count_out[c] = h->t_cnt[c];
        if (reset) {
            h->t_ms[c] = 0.0;
            h->t_cnt[c] = 0;
        }
    }
    return VBX_OK;
}

}  // extern "C"
