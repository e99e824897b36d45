"""Device time of the fused EM contraction alone (em_contract_kernel, vbx_em_contract.cu), against the HBM bytes its shapes
must move, on the headline shape: 4096 recordings x 1000 frames, S = 16, R = 128, 10 iterations (one launch each).
--frames / --recordings time other shapes: recordings of at most 512 frames take clusters of 4 CTAs instead of 8 (e.g.
--frames 500 --recordings 8192).

bytes per launch:  rho read once (4 R), gamma read (4 S), p and rowmax written (4 S + 4) per frame, plus alpha and invL
                   written (2 x 4 S R) per recording
Kernel times come from torch.profiler (CUDA activity) over --runs calls of vbx_run after a warm-up; the achieved bandwidth
is those bytes over the kernel's device time, also as a fraction of 3.35 TB/s (H100 SXM data sheet).

    python tools/bench_em_contract.py [--runs 5] [--frames 1000] [--recordings 4096] [--out result.json]
"""
import argparse
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench_project import gpu_info  # noqa: E402
from vbx_b200 import synth  # noqa: E402
from vbx_b200.batch import VbxBatch  # noqa: E402

HBM = 3.35e12
R, S, ITERS = 128, 16, 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=5)
    ap.add_argument('--frames', type=int, default=1000, help='frames per recording (at most 1024)')
    ap.add_argument('--recordings', type=int, default=4096, help='a multiple of 8')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    B, T = a.recordings, a.frames
    if not 0 < T <= 1024 or B <= 0 or B % 8:
        raise SystemExit('--frames must be 1 .. 1024 and --recordings a positive multiple of 8')
    if not torch.cuda.is_available():
        raise SystemExit('bench_em_contract.py needs a CUDA device')
    dev = torch.device('cuda:0')
    N = B * T
    d = synth.make_batch([T] * 8, R=R, S=S, seed=0)         # one 8-recording pattern tiled over the batch
    fea = torch.from_numpy(d['fea']).to(dev).repeat(B // 8, 1)
    g0 = torch.from_numpy(d['gamma0'].astype('float32')).to(dev).repeat(B // 8, 1)
    vb = VbxBatch([T] * B, R, S, device=dev, exact_stop=False)
    vb.prepare_scale(fea, torch.from_numpy(d['Phi']).to(dev))
    gamma, pi = torch.empty((N, S), device=dev), torch.empty((B, S), device=dev)
    alpha, invL = torch.empty((B, S, R), device=dev), torch.empty((B, S, R), device=dev)

    def call():
        gamma.copy_(g0)
        pi.fill_(1.0 / S)
        vb.run(gamma, pi, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=ITERS, epsilon=-float('inf'), alpha=alpha, invL=invL,
               return_model=True)

    for _ in range(2):
        call()
    torch.cuda.synchronize()
    info = gpu_info()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.runs):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        us = getattr(e, 'device_time_total', None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0 or e.count == 0:
            continue
        m = re.search(r'(\w+)(<[^<>]*>)?\(', e.key)
        kernels[m.group(1) + (m.group(2) or '') if m else e.key] = dict(ms=us / 1e3, launches=e.count)
    fused = {k: v for k, v in kernels.items() if 'em_contract_kernel' in k}
    if not fused:
        raise SystemExit('em_contract_kernel did not run: ' + ', '.join(sorted(kernels)))
    ms = sum(v['ms'] for v in fused.values()) / sum(v['launches'] for v in fused.values())
    nbytes = N * (4 * R + 4 * S + 4 * S + 4) + B * 2 * 4 * S * R
    res = dict(gpu=info, recordings=B, frames_per_recording=T, S=S, R=R, iterations=ITERS, runs=a.runs,
               kernel=sorted(fused), ms_per_launch=ms, bytes_per_launch=nbytes, achieved_gbs=nbytes / (ms * 1e-3) / 1e9,
               fraction_of_3_35TBps=nbytes / (ms * 1e-3) / HBM, floor_ms_at_3_35TBps=nbytes / HBM * 1e3,
               other_kernels_ms_per_run={k: v['ms'] / a.runs for k, v in kernels.items() if k not in fused},
               gpu_after=gpu_info())
    vb.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(txt + '\n')


if __name__ == '__main__':
    main()
