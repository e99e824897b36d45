"""Times back-end training (DESIGN.md section 5.24).

1. vbx_class_scatter on float32 rows at N in {1e5, 1e6, 4e6} x D in {128, 256, 512}, K = N / 150 classes of equal
   size: kernel time from CUDA events over --reps launches after a warm-up, alternating --rounds times with the obvious
   torch float64 route (class means by index_add_, a float64 centred copy, Xc^T Xc) timed the same way.  Achieved FLOP/s
   count N D (D + 1), the symmetric half; the share of peak is the larger of FLOPs / 67 TFLOP/s (FP64 tensor cores, H100
   SXM data sheet) and the N D 4 input bytes / 3.35 TB/s, over the kernel time, naming the bound.  Both routes' outputs
   are compared.
2. Whole train_backend calls on a synthetic set of 1 M x 256 x-vectors of 6 000 speakers (lda_dim 128, 10 EM
   iterations), against the float64 oracle (oracle/train_oracle.py) on the host cores.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_train.py --out profiles/h100_train.json
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from vbx_b200 import _lib, train  # noqa: E402

PEAK_DMMA = 67e12      # FP64 tensor-core FLOP/s, H100 SXM data sheet
PEAK_HBM = 3.35e12     # bytes/s


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def scatter_case(N, D, reps, rounds, dev, lib, h):
    K = max(1, N // 150)
    off = np.linspace(0, N, K + 1).astype(np.int64)
    gen = torch.Generator(device=dev).manual_seed(N + D)
    X = torch.randn((N, D), generator=gen, device=dev) + torch.randn((K, D), generator=gen, device=dev).repeat_interleave(
        torch.from_numpy(np.diff(off)).to(dev), dim=0)
    need = ctypes.c_size_t()
    assert lib.vbx_class_scatter_workspace_bytes(h, N, D, K, ctypes.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    means = torch.empty((K, D), dtype=torch.float64, device=dev)
    S = torch.empty((D, D), dtype=torch.float64, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    offp = off.ctypes.data_as(ctypes.c_void_p)

    def kernel():
        rc = lib.vbx_class_scatter(h, p(X), N, D, K, offp, p(ws), ws.numel(), p(means), p(S), st)
        assert rc == 0, lib.vbx_last_error(h)
    cls = torch.repeat_interleave(torch.arange(K, device=dev), torch.from_numpy(np.diff(off)).to(dev))
    n = torch.from_numpy(np.diff(off).astype(np.float64)).to(dev)
    out = {}

    def torch_route():
        Xd = X.double()
        m = torch.zeros((K, D), dtype=torch.float64, device=dev).index_add_(0, cls, Xd) / n[:, None]
        Xc = Xd - m[cls]
        out['S'] = Xc.T @ Xc
    kernel()
    torch_route()
    torch.cuda.synchronize()
    diff = float(((S - out['S']).abs().max() / out['S'].diagonal().abs().max()).item())
    tk, tt = [], []
    for _ in range(rounds):
        tk.append(timed(kernel, reps))
        tt.append(timed(torch_route, reps))
    k_s, t_s = float(np.median(tk)), float(np.median(tt))
    flops, nbytes = N * D * (D + 1), N * D * 4
    bound = max(flops / PEAK_DMMA, nbytes / PEAK_HBM)
    return dict(N=N, D=D, K=K, kernel_ms=round(k_s * 1e3, 4), kernel_ms_min=round(min(tk) * 1e3, 4),
                torch_ms=round(t_s * 1e3, 4), torch_ms_min=round(min(tt) * 1e3, 4), speedup=round(t_s / k_s, 3),
                tflops=round(flops / k_s / 1e12, 2), share_of_bound=round(bound / k_s, 4),
                bound='fp64_tensor' if flops / PEAK_DMMA >= nbytes / PEAK_HBM else 'hbm',
                max_rel_diff_vs_torch=diff)


def synthetic_set(N, K, Dx, seed):
    rng = np.random.default_rng(seed)
    sizes = rng.multinomial(N - 2 * K, np.ones(K) / K) + 2
    centres = (rng.standard_normal((K, Dx)) * np.exp(np.linspace(0.5, -1.5, Dx))[None, :]).astype(np.float32)
    q, _ = np.linalg.qr(rng.standard_normal((Dx, Dx)))
    within = (q * np.exp(np.linspace(0, -2, Dx))[None, :]).astype(np.float32)
    x = np.repeat(centres, sizes, 0) + rng.standard_normal((N, Dx), dtype=np.float32) @ within.T + 3.0
    off = np.concatenate([[0], np.cumsum(sizes)])
    return {f's{k}': x[off[k]:off[k + 1]] for k in range(K)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--sizes', default='100000x128,100000x256,100000x512,1000000x128,1000000x256,1000000x512,'
                                      '4000000x128,4000000x256,4000000x512')
    ap.add_argument('--train-n', type=int, default=1_000_000)
    ap.add_argument('--train-k', type=int, default=6000)
    ap.add_argument('--no-oracle', action='store_true', help='skip the host oracle of part 2')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train.py needs a CUDA device')
    dev = torch.device('cuda:0')
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    scatter = []
    try:
        for size in args.sizes.split(','):
            N, D = (int(v) for v in size.split('x'))
            scatter.append(scatter_case(N, D, args.reps, args.rounds, dev, lib, h))
            print(json.dumps(scatter[-1]), file=sys.stderr)
            torch.cuda.empty_cache()
    finally:
        lib.vbx_destroy(h)
    sets = synthetic_set(args.train_n, args.train_k, 256, 7)
    train.train_backend(sets, lda_dim=128, em_iters=10, device=dev)          # warm-up
    walls = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        tf, pl, rep = train.train_backend(sets, lda_dim=128, em_iters=10, device=dev)
        walls.append(time.perf_counter() - t0)
    whole = dict(N=rep['N'], K=rep['K'], Dx=256, lda_dim=128, em_iters=10, seconds=round(float(np.median(walls)), 3),
                 seconds_min=round(min(walls), 3), stages={k: round(v, 4) for k, v in rep['seconds'].items()})
    if not args.no_oracle:
        from oracle import train_oracle
        t0 = time.perf_counter()
        ref = train_oracle.train(sets, lda_dim=128, em_iters=10)
        whole['oracle_host_seconds'] = round(time.perf_counter() - t0, 3)
        whole['host_cores'] = os.cpu_count()
        W = np.linalg.inv(pl[1].T @ pl[1])
        whole['rel_diff_W'] = float(np.linalg.norm(W - ref['W']) / np.linalg.norm(ref['W']))
        whole['rel_diff_trace'] = float(np.max(np.abs(np.array(rep['objective']) - ref['trace']) / np.abs(ref['trace'])))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    line = dict(gpu=q[0] if q else torch.cuda.get_device_name(0), class_scatter=scatter, train_backend=whole)
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
