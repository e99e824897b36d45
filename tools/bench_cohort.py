"""Times score normalisation against a cohort (DESIGN.md section 5.17).

1. cohort_stats (vbx_cohort_stats_batch) on synthetic archives of M = 16 000 speakers (4 per recording, 1 .. 15
   x-vectors each, R = 128) against C = 1 000 and 10 000 cohort speakers (1 .. 15 x-vectors each) at top_k = 200: device
   time of every kernel from torch.profiler over --rounds calls after one warm-up call, next to the pairs and bytes the
   score kernel needs. The statistics row sums the span and statistics kernels of both speaker sets and the copy of the
   cohort speaker index.  Also the normalisation kernel inside link_speakers(norm=) at M = 4 000 (the linkage dominates
   that call).
2. Whole diarize_batch calls on the synthetic archive of tools/bench_sweep.py (17 recordings) with linking and an
   enrolment of 10 speakers, without and with a cohort of 200 speakers (20 x-vectors each), alternating in one process
   (medians, minima, maxima).
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_cohort.py --out profiles/h100_cohort.json
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
from bench_enroll import enrolled  # noqa: E402
from bench_link import speakers  # noqa: E402
from bench_sweep import GOLD, synthetic_archive  # noqa: E402
from vbx_b200 import cohort, link, pipeline  # noqa: E402

KERNELS = {'statistics': ('link_init_kernel', 'link_span_kernel', 'link_stats_kernel', 'repeat_index_kernel'),
           'score': ('enroll_score_kernel',), 'top_k': ('cohort_topk_kernel',), 'normalise': ('norm_scores_kernel',)}


def profiled(run, rounds):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            run()
    kern = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        for k, names in KERNELS.items():
            if any(n in e.key for n in names):
                kern[k] += getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)) / rounds
    return {k: round(v, 1) for k, v in kern.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--sizes', default='16000x1000,16000x10000')
    ap.add_argument('--top-k', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cohort.py needs a CUDA device')
    sizes = {}
    for size in args.sizes.split(','):
        M, C = (int(v) for v in size.split('x'))
        fea, Phi, offs, labels = speakers(M)
        cfea, cspk = enrolled(C, seed=2)
        run = lambda: cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=args.top_k)
        st = run()                                                          # warm-up: module load
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.rounds):
            run()
        wall = (time.perf_counter() - t0) / args.rounds
        sizes[size] = dict(M=M, C=C, top_k=args.top_k, N=int(fea.shape[0]), N_c=len(cspk),
                           whole_call_s=round(wall, 4), kernels_us=profiled(run, args.rounds),
                           sigma_range=[round(float(st.std.min()), 3), round(float(st.std.max()), 3)],
                           score=dict(pairs=M * C, llr_bytes_written=8 * M * C, fp64_div=M * C * 128,
                                      fp64_log=M * C * 16),
                           top_k_bytes_read=10 * 8 * M * C)
        del fea, cfea
        torch.cuda.empty_cache()
    # the normalisation kernel inside link_speakers(norm=)
    M = 4000
    fea, Phi, offs, labels = speakers(M)
    cfea, cspk = enrolled(1000, seed=2)
    st = cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=args.top_k)
    run = lambda: link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, norm=(st.mean, st.std))
    run()
    link_norm = dict(M=M, kernels_us=profiled(run, 1), bytes=16 * M * M)
    del fea, cfea
    torch.cuda.empty_cache()

    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs = synthetic_archive(z['x_raw'])
    rng = np.random.default_rng(5)
    x = z['x_raw']
    known = {f'spk{k}': x[rng.choice(len(x), 20, replace=False)] for k in range(10)}
    sd = x.std(0)
    crowd = {f'c{k}': x.mean(0) + 2.0 * sd * rng.standard_normal(x.shape[1]) + 0.5 * sd * rng.standard_normal((20, x.shape[1]))
             for k in range(200)}
    kw = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=40, epsilon=1e-6,
              device=torch.device('cuda:0'))
    modes = {'without': dict(link_threshold=0.0, enroll=known, enroll_threshold=0.0),
             'cohort': dict(link_threshold=0.0, enroll=known, enroll_threshold=0.0, cohort=crowd)}

    def call(mode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipeline.diarize_batch(recs, transform, plda, **kw, **modes[mode])
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    for mode in modes:
        out, _ = call(mode)
    n_spk = sum(len(it['speaker_names']) for it in out.values())
    times = {mode: [] for mode in modes}
    for _ in range(args.rounds):
        for mode in modes:
            times[mode].append(call(mode)[1])
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='score normalisation against a cohort', gpu=q.stdout.strip(), synthetic=sizes, link_norm=link_norm,
        archive=f'synthetic, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all; '
                f'{n_spk} speakers, linked at 0 and named at 0 by 10 enrolled speakers; cohort of 200 speakers',
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
