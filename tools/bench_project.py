"""Device time of the tensor-core front end alone (vbx_project_tc.cu), against the HBM bytes its shapes must move.

Two workloads, each on 4096 recordings x 1000 frames (N = 4 096 000):
  projection      vbx_prepare_project, D = 256 -> R = 128 (the headline step's projection, project_wgmma_kernel<0,2>)
                  bytes: X read, rho and G_t written                         N * (4 D + 4 R + 4)
  xvector_chain   vbx_prepare_xvectors, Dx = 256 (x-vector transform <1,3> then PLDA projection <2,3>)
                  bytes: x_raw read, x_norm written and read, rho and G_t written   N * (4 Dx + 3 * 4 R + 4)
Kernel times come from torch.profiler (CUDA activity) over --launches calls after a warm-up; per call the table lists
every kernel the call launched, and the achieved bandwidth of the wgmma kernels' bytes over their device time as a
fraction of 3.35 TB/s (H100 SXM data sheet).

    python tools/bench_project.py [--launches 20] [--out result.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vbx_b200.batch import VbxBatch  # noqa: E402

HBM = 3.35e12
B, T, R, D = 4096, 1000, 128, 256


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    name, plim, sm, smax = [v.strip() for v in q[0].split(',')]
    return dict(name=name, power_limit=plim, sm_clock=sm, sm_clock_max=smax)


def profile(call, launches):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(launches):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        us = getattr(e, 'device_time_total', None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0 or e.count == 0:
            continue
        m = re.search(r'(\w+)(<[^<>]*>)?\(', e.key)             # "void ns::kernel<0, 2>(args)" -> "kernel<0, 2>"
        kernels[m.group(1) + (m.group(2) or '') if m else e.key] = dict(ms_per_call=us / 1e3 / launches, launches_per_call=e.count / launches)
    return kernels


def summarise(kernels, bytes_per_call):
    wg = sum(v['ms_per_call'] for k, v in kernels.items() if 'project_wgmma_kernel' in k)
    total = sum(v['ms_per_call'] for v in kernels.values())
    return dict(kernels=kernels, bytes_per_call=bytes_per_call, wgmma_ms_per_call=wg, all_kernels_ms_per_call=total,
                achieved_gbs=bytes_per_call / (wg * 1e-3) / 1e9, fraction_of_3_35TBps=bytes_per_call / (wg * 1e-3) / HBM,
                floor_ms_at_3_35TBps=bytes_per_call / HBM * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if a.launches < 20:
        ap.error('--launches must be at least 20')
    if not torch.cuda.is_available():
        raise SystemExit('bench_project.py needs a CUDA device')
    dev = torch.device('cuda:0')
    N = B * T
    gen = torch.Generator(device=dev).manual_seed(0)
    vb = VbxBatch([T] * B, R, 16, device=dev, exact_stop=False)
    X = torch.randn((N, D), generator=gen, device=dev)
    V = torch.randn((D, R), generator=gen, device=dev) / D ** 0.5
    Phi = 0.5 + torch.rand(R, generator=gen, device=dev) * 5.0
    rho = torch.empty((N, R), device=dev)
    res = dict(gpu=gpu_info(), recordings=B, frames_per_recording=T, N=N, launches=a.launches)
    res['projection'] = dict(D=D, **summarise(profile(lambda: vb.prepare_project(X, V, Phi, out=rho), a.launches),
                                               N * (4 * D + 4 * R + 4)))
    q, _ = torch.linalg.qr(torch.randn((R, R), generator=gen, device=dev))
    model = (torch.randn(D, generator=gen, device=dev) * 0.5, torch.randn((D, R), generator=gen, device=dev) / D ** 0.5,
             torch.randn(R, generator=gen, device=dev) * 0.05, torch.randn(R, generator=gen, device=dev) * 0.02,
             q.contiguous(), Phi)
    res['xvector_chain'] = dict(Dx=D, **summarise(profile(lambda: vb.prepare_xvectors(X, *model, out=rho), a.launches),
                                                   N * (4 * D + 3 * 4 * R + 4)))
    res['gpu_after'] = gpu_info()
    vb.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(txt + '\n')


if __name__ == '__main__':
    main()
