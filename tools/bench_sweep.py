"""Times a hyperparameter sweep (vbx_b200/sweep.py) against the same settings run one after another with scalar
parameters, and ES2005a under 216 settings.  Prints one JSON line; --out also writes it there.

The archive is synthetic and seeded, shaped like AMI dev: 17 recordings of 2 000 .. 8 000 x-vectors (so recordings of
at least 4 096 frames take the chunked scan), built from the shipped ES2005a x-vectors and model.  The grid has 64
settings of Fa, Fb and loopP at the example threshold and smoothing.  The sequential runs reuse the sweep's front end
and AHC output, so the comparison is of the VB-HMM step alone; the front end is timed separately.

    python tools/bench_sweep.py --out profiles/h100_sweep.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from vbx_b200 import pipeline, sweep  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden')
GRID64 = dict(Fa=[0.2, 0.3, 0.4, 0.5], Fb=[6.0, 17.0, 40.0, 64.0], loopP=[0.35, 0.65, 0.9, 0.99], threshold=[-0.015],
              smoothing=[5.0])
GRID216 = dict(Fa=[0.1, 0.2, 0.3, 0.4, 0.5, 0.6], Fb=[4.0, 6.0, 11.0, 17.0, 32.0, 64.0],
               loopP=[0.35, 0.5, 0.65, 0.8, 0.9, 0.99], threshold=[-0.015], smoothing=[5.0])


def synthetic_archive(x_es, seed=0):
    """17 recordings of 2 000 .. 8 000 x-vectors: sticky speaker turns over 2 .. 8 speakers, each speaker a random
    ES2005a x-vector plus noise of the spread ES2005a shows."""
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    recs = {}
    for r in range(17):
        T = int(rng.integers(2000, 8001))
        K = int(rng.integers(2, 9))
        centers = x_es[rng.choice(len(x_es), K, replace=False)]
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(K)
        x = centers[spk] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        recs[f'syn{r:02d}'] = (x, seg)
    return recs


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def sequential(recs, transform, plda, grid, dev):
    """The settings one after another, each one scalar-parameter batch per state tier, on ONE front end and AHC output."""
    names = list(recs)
    lens = np.array([recs[n][0].shape[0] for n in names], dtype=np.int64)
    (fea, Phi, _, th, Zs), t_front = timed(lambda: pipeline._front_end(recs, names, lens, transform, plda, 128, 'auto', dev, 0.0))
    fea, Phi = pipeline._pad_features(fea, Phi)

    def vb_all():
        from vbx_b200 import ahc
        from vbx_b200.batch import VbxBatch
        for s in sweep.grid_settings(grid):
            labels = ahc.cut(Zs, th, lens, s.threshold)
            lab_d = torch.from_numpy(np.concatenate(labels)).to(dev)
            pipeline._vb_stage([(s.Fa, s.Fb, s.loopP, s.smoothing)], [labels], [lab_d], Zs, lens, fea, Phi, None,
                               'AHC+VB', dev, VbxBatch, None, maxIters=40, epsilon=1e-6)
    _, t_vb = timed(vb_all)
    return t_front, t_vb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_sweep.py needs a CUDA device')
    dev = torch.device('cuda:0')
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs = synthetic_archive(z['x_raw'])
    es = {'ES2005a': (z['x_raw'], z['seg_times'])}
    sweep.sweep_batch(es, transform, plda, dict(GRID64, Fa=[0.3], Fb=[17.0], loopP=[0.99]), device=dev)    # warm-up
    out_sweep, t_sweep = timed(lambda: sweep.sweep_batch(recs, transform, plda, GRID64, device=dev))
    t_front, t_seq = sequential(recs, transform, plda, GRID64, dev)
    _, t_es = timed(lambda: sweep.sweep_batch(es, transform, plda, GRID216, device=dev))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='hyperparameter sweep', gpu=q.stdout.strip(),
        archive=f'synthetic, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all',
        settings=len(sweep.grid_settings(GRID64)), max_iters=40, epsilon=1e-6,
        sweep_s=round(t_sweep, 3), front_end_and_ahc_s=round(t_front, 3),
        sweep_vb_s=round(t_sweep - t_front, 3), sequential_scalar_vb_s=round(t_seq, 3),
        speedup_vb=round(t_seq / max(t_sweep - t_front, 1e-9), 2),
        speakers=sorted(set(v['n_speakers'] for per in out_sweep.values() for v in per.values())),
        es2005a_216_settings_s=round(t_es, 3))
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
