"""Times diarize_batch under speaker-count constraints (DESIGN.md section 5.14) on the synthetic archive of
tools/bench_sweep.py (17 recordings of 2 000 .. 8 000 x-vectors, 2 .. 8 speakers each) three ways: unconstrained,
max_speakers=1 (every recording takes rule 2: one vbx_hard_labels_keep call per state tier) and min_speakers=16 (every
recording takes rule 3: a VB-HMM re-run per state tier).  Whole calls alternate in one process (medians); the device time of
the new kernels comes from torch.profiler in a run of its own.  Prints one JSON line; --out also writes it there.

    python tools/bench_count.py --out profiles/h100_count.json
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_sweep import GOLD, synthetic_archive  # noqa: E402
from vbx_b200 import pipeline  # noqa: E402

MODES = {'unconstrained': {}, 'max_speakers=1': dict(max_speakers=1), 'min_speakers=16': dict(min_speakers=16)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_count.py needs a CUDA device')
    dev = torch.device('cuda:0')
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs = synthetic_archive(z['x_raw'])
    kw = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=40, epsilon=1e-6, device=dev)

    def call(mode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipeline.diarize_batch(recs, transform, plda, **kw, **MODES[mode])
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    rules = {}
    for mode in MODES:                                  # warm-up, and the rule every recording took
        out, _ = call(mode)
        rules[mode] = sorted(set(it.get('count_rule', '-') for it in out.values()))
    times = {mode: [] for mode in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            times[mode].append(call(mode)[1])
    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    for mode in ('unconstrained', 'max_speakers=1'):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(mode)
        for e in prof.key_averages():
            for k in ('state_mass_kernel', 'hard_labels_keep_kernel', 'hard_labels_kernel'):
                if k in e.key and not (k == 'hard_labels_kernel' and 'keep' in e.key):
                    us = getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0))
                    kernels[f'{mode}: {k}'] = dict(us=round(us, 1), launches=int(e.count))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='speaker-count constraints', gpu=q.stdout.strip(),
        archive=f'synthetic, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all',
        rounds=args.rounds, rules=rules,
        median_s={mode: round(float(np.median(t)), 4) for mode, t in times.items()},
        min_s={mode: round(float(np.min(t)), 4) for mode, t in times.items()},
        kernels_device=kernels)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
