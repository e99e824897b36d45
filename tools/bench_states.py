"""Cost of the S = 128 state tier against S = 64, per kernel class, on one GPU.

Batch: 4096 recordings x 1000 frames, R = 128, 10 EM iterations at epsilon = -inf (no float64 finish), all plans on the
split forward-backward schedule (S = 64 is forced onto it so that the comparison is like for like).  Configurations:
S = 64 with 64 live states, S = 128 with 128 and with 100 live states.  For each: the device time of every kernel class
(vbx_get_timings, a separate run with option "timing"), the algorithmic bytes of the class computed from the shapes
below as a fraction of 3.35 TB/s (H100 SXM data sheet), and the time of one vbx_run (CUDA events, timing off).

Per-frame floors (bytes every iteration must move; R = 128):
  M-step          rho + gamma                        4R + 4S
  log-likelihood  rho + p + rowmax + c_t              4R + 4S + 8
  sweeps+combine  p twice, ahat/bhat written and read, gamma written: 8 arrays of S floats, + c twice, rsigma
                                                      32S + 16
The speaker model reads the per-tile partial sums (n_tiles x S x R floats) and writes A and its fragment images.

Also: ES2005a at --threshold 0.15 (108 AHC clusters) through diarize_batch (S = 128 tier) end to end, and the VB step of
that recording on the S = 128 float32 kernels against the float64 kernels the drop-in VBx() uses.

    python tools/bench_states.py [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vbx_b200 import pipeline                # noqa: E402
from vbx_b200.batch import VbxBatch, run_f64  # noqa: E402

HBM = 3.35e12
B, T, R, ITERS = 4096, 1000, 128, 10
HP = dict(Fa=0.3, Fb=17.0, loopProb=0.99)


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    name, plim, sm, smax = [v.strip() for v in q[0].split(',')]
    return dict(name=name, power_limit=plim, sm_clock=sm, sm_clock_max=smax)


def class_bytes(S, n_mtiles):
    N = B * T
    return {
        'mstep_partial': N * (4 * R + 4 * S) + n_mtiles * S * R * 4,
        'speaker_model': n_mtiles * S * R * 4 + B * S * R * 4 * 3,
        'loglik': N * (4 * R + 4 * S + 8),
        'forward_backward': N * (32 * S + 16),
    }


def one_config(S_pad, live, dev, rng):
    N = B * T
    lens = np.full(B, T)
    vb = VbxBatch(lens, R, live, device=dev, exact_stop=False, fb_split=1, S_pad=S_pad)
    assert vb.S == S_pad
    torch.manual_seed(int(rng.integers(1 << 30)))
    fea = torch.randn((N, R), device=dev)
    Phi = torch.from_numpy(np.exp(np.linspace(np.log(5.6), np.log(0.53), R)).astype(np.float32)).to(dev)
    g0 = torch.zeros((N, S_pad), device=dev)
    g0[:, :live] = torch.softmax(3.0 * torch.randn((N, live), device=dev), dim=1)
    p0 = torch.zeros((B, S_pad), device=dev)
    p0[:, :live] = 1.0 / live
    vb.prepare_scale(fea, Phi)
    g, p = g0.clone(), p0.clone()
    bufs = vb.output_buffers(ITERS)

    def run():
        g.copy_(g0)
        p.copy_(p0)
        return vb.run(g, p, maxIters=ITERS, epsilon=-np.inf, buffers=bufs, **HP)

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = []
    for _ in range(5):
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        steps.append(e0.elapsed_time(e1))
    vb.set_option('timing', 1)
    vb.timings(reset=True)
    run()
    torch.cuda.synchronize()
    tm = vb.timings(reset=True)
    vb.set_option('timing', 0)
    n_mtiles = int(np.sum((lens + 511) // 512))
    by = class_bytes(S_pad, n_mtiles)
    kernels = {}
    for k, (ms, cnt) in tm.items():
        if cnt == 0:
            continue
        row = dict(ms_per_iter=ms / ITERS, launches=int(cnt))
        if k in by:
            row['bytes_per_iter'] = by[k]
            row['fraction_of_3.35TBps'] = by[k] / (ms / ITERS * 1e-3) / HBM
        kernels[k] = row
    gam = g[:, :live].double()
    assert torch.isfinite(gam).all()
    floor = sum(by[k] for k in ('mstep_partial', 'loglik', 'forward_backward'))
    vb.close()
    return dict(S=S_pad, live_states=live, step_ms=dict(median=float(np.median(steps)), min=float(np.min(steps)),
                                                         max=float(np.max(steps))),
                step_ms_per_iter=float(np.median(steps)) / ITERS, kernels=kernels,
                floor_bytes_per_iter=floor, floor_ms_per_iter_at_3_35TBps=floor / HBM * 1e3)


def es2005a(dev):
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'es2005a.npz'))
    m = np.load(os.path.join(ROOT, 'tests', 'golden', 'es2005a_model.npz'))
    rec = {'ES2005a': (z['x_raw'], z['seg_times'])}
    args = ((m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi']), float(z['Fa']), float(z['Fb']),
            float(z['loopProb']))
    kw = dict(threshold=0.15, smoothing=float(z['smoothing']), device=dev)
    pipeline.diarize_batch(rec, *args, **kw)                      # warm-up (module loads, plans)
    torch.cuda.synchronize()
    e2e = []
    for _ in range(3):
        t0 = time.perf_counter()
        res = pipeline.diarize_batch(rec, *args, **kw)['ES2005a']
        torch.cuda.synchronize()
        e2e.append((time.perf_counter() - t0) * 1e3)
    # the VB step alone from the same AHC initialisation: S = 128 float32 tier vs float64 kernels (drop-in route)
    from oracle.ahc_oracle import ahc_labels
    lab = ahc_labels(z['x_lda'], 0.15)[0]
    S = int(lab.max()) + 1
    Tn = len(lab)
    q = np.exp(np.eye(S)[lab] * float(z['smoothing']))
    q /= q.sum(1, keepdims=True)
    vbkw = dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopProb=float(z['loopProb']), maxIters=40, epsilon=1e-6)
    times = {}
    for route in ('float32_S128', 'float64'):
        f64 = route == 'float64'
        dt = torch.float64 if f64 else torch.float32
        vb = VbxBatch([Tn], 128, S, device=dev, f64_only=f64)
        fea = torch.from_numpy(z['fea']).to(dev).to(dt).contiguous()
        Phi = torch.from_numpy(z['Phi']).to(dev).to(dt).contiguous()
        if not f64:
            vb.prepare_scale(fea, Phi)
        samples = []
        for rep in range(4):
            g = torch.zeros((Tn, vb.S), dtype=dt, device=dev)
            g[:, :S] = torch.from_numpy(q).to(dev).to(dt)
            p = torch.zeros((1, vb.S), dtype=dt, device=dev)
            p[0, :S] = 1.0 / S
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run_f64(vb, fea, Phi, g, p, **vbkw) if f64 else vb.run(g, p, **vbkw)
            torch.cuda.synchronize()
            if rep:
                samples.append((time.perf_counter() - t0) * 1e3)
        times[route] = dict(ms=float(np.median(samples)), iterations=int(out['n_iters'][0]))
        vb.close()
    return dict(clusters=S, diarize_batch_ms=dict(median=float(np.median(e2e)), min=float(np.min(e2e))),
                diarize_batch_iterations=res['iterations'], vb_step=times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_states.py needs a CUDA device')
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(0)
    info_before = gpu_info()
    res = dict(gpu=info_before, batch=dict(recordings=B, frames=T, R=R, iterations=ITERS, epsilon='-inf', schedule='split'))
    res['configs'] = [one_config(64, 64, dev, rng), one_config(128, 128, dev, rng), one_config(128, 100, dev, rng)]
    res['es2005a_threshold_0.15'] = es2005a(dev)
    res['gpu_after'] = gpu_info()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(txt + '\n')


if __name__ == '__main__':
    main()
