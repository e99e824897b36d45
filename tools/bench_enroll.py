"""Times enrolment against known speakers (DESIGN.md section 5.16).

1. enroll_speakers (vbx_enroll_batch) on synthetic archives of (M, E) = (1 000, 100), (16 000, 1 000) and
   (100 000, 1 000) speakers (4 per recording, 1 .. 15 x-vectors each; enrolled speakers 1 .. 15 x-vectors each;
   R = 128): device time of every kernel from torch.profiler over --rounds calls after one warm-up call, next to the
   pairs and bytes the score kernel needs.  The statistics row sums the span and statistics kernels of both speaker sets
   and the copy of the enrolled speaker index.
2. Whole diarize_batch calls on the synthetic archive of tools/bench_sweep.py (17 recordings) without and with an
   enrolment of 10 speakers (20 x-vectors each), alternating in one process (medians, minima, maxima).
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_enroll.py --out profiles/h100_enroll.json
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
from bench_link import speakers  # noqa: E402
from bench_sweep import GOLD, synthetic_archive  # noqa: E402
from vbx_b200 import enroll, pipeline  # noqa: E402

KERNELS = {'statistics': ('link_init_kernel', 'link_span_kernel', 'link_stats_kernel', 'repeat_index_kernel'),
           'score': ('enroll_score_kernel',), 'assignment': ('enroll_assign_kernel',)}


def enrolled(E, R=128, seed=1, device='cuda'):
    rng = np.random.default_rng(seed)
    espk = np.repeat(np.arange(E), rng.integers(1, 16, E))
    efea = torch.randn((len(espk), R), generator=torch.Generator().manual_seed(seed)).to(device)
    return efea, espk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--sizes', default='1000x100,16000x1000,100000x1000')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_enroll.py needs a CUDA device')
    from torch.profiler import ProfilerActivity, profile
    sizes = {}
    for size in args.sizes.split(','):
        M, E = (int(v) for v in size.split('x'))
        fea, Phi, offs, labels = speakers(M)
        efea, espk = enrolled(E)
        run = lambda: enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 0.0)
        res = run()                                                         # warm-up: module load
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.rounds):
            run()
        wall = (time.perf_counter() - t0) / args.rounds
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.rounds):
                run()
        kern = {k: 0.0 for k in KERNELS}
        for e in prof.key_averages():
            for k, names in KERNELS.items():
                if any(n in e.key for n in names):
                    kern[k] += getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)) / args.rounds
        sizes[size] = dict(M=M, E=E, N=int(fea.shape[0]), N_e=len(espk), recordings=len(labels),
                           whole_call_s=round(wall, 4), kernels_us={k: round(v, 1) for k, v in kern.items()},
                           named=int((res.assign >= 0).sum()),
                           score=dict(pairs=M * E, llr_bytes_written=8 * M * E, fp64_div=M * E * 128,
                                      fp64_log=M * E * 16))
        del fea, efea
        torch.cuda.empty_cache()

    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs = synthetic_archive(z['x_raw'])
    rng = np.random.default_rng(5)
    x = z['x_raw']
    known = {f'spk{k}': x[rng.choice(len(x), 20, replace=False)] for k in range(10)}
    kw = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=40, epsilon=1e-6,
              device=torch.device('cuda:0'))
    modes = {'without': {}, 'enroll': dict(enroll=known, enroll_threshold=0.0)}

    def call(mode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipeline.diarize_batch(recs, transform, plda, **kw, **modes[mode])
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    for mode in modes:
        out, _ = call(mode)
    named = sum(not v.startswith('unknown-') for it in out.values() for v in it['speaker_names'].values())
    n_spk = sum(len(it['speaker_names']) for it in out.values())
    times = {mode: [] for mode in modes}
    for _ in range(args.rounds):
        for mode in modes:
            times[mode].append(call(mode)[1])
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='enrolment against known speakers', gpu=q.stdout.strip(), synthetic=sizes,
        archive=f'synthetic, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all; '
                f'{n_spk} speakers, {named} named at threshold 0 by 10 enrolled speakers',
        rounds=args.rounds, median_s={k: round(float(np.median(t)), 4) for k, t in times.items()},
        min_s={k: round(float(np.min(t)), 4) for k, t in times.items()},
        max_s={k: round(float(np.max(t)), 4) for k, t in times.items()})
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
