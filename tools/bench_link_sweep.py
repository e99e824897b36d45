"""Times speaker linking inside the sweep (DESIGN.md section 5.18).

(a) G linking problems of M speakers each (tools/bench_link.py's synthetic speakers, 4 per recording, R = 128; problem g
    with the Fa / Fb of setting g of tools/bench_sweep.py's 64-setting grid, cycled): G link_speakers calls one after
    another against one link.link_many call (vbx_link_batch), for G in {1, 64, 216} x M in {43, 1 000} and once G = 64 x
    M = 4 000.  Whole-call time is a host clock around work that ends in a readback; device time is the sum of the
    kernels' times from torch.profiler in a separate run (not taken for M = 4 000, whose sequential run alone takes
    minutes).
(b) The 64-setting sweep of tools/bench_sweep.py on a seeded multi-session archive of AMI-dev shape (17 recordings of
    2 000 .. 8 000 x-vectors, 3 .. 5 speakers each from a pool of 40, synth.multi_session_archive) with its reference,
    without linking and with 8 link thresholds, alternating, medians of 5; the host scoring across files
    (sweep.summarize_across_files) is timed on its own.
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it there.

    python tools/bench_link_sweep.py --out profiles/h100_link_sweep.json
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
from bench_link import KERNELS, speakers  # noqa: E402
from bench_sweep import GOLD, GRID64  # noqa: E402
from vbx_b200 import link, sweep, synth  # noqa: E402

THRESHOLDS = [-20.0, -10.0, 0.0, 10.0, 20.0, 30.0, 48.0, 64.0]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def device_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return round(sum(getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0))
                     for e in prof.key_averages() if any(k in e.key for k in KERNELS)) / 1e3, 3)


def problems(G, M, profiled):
    fea, Phi, offs, labels = speakers(M)
    settings = sweep.grid_settings(GRID64)
    Fa = [settings[g % len(settings)].Fa for g in range(G)]
    Fb = [settings[g % len(settings)].Fb for g in range(G)]
    seq = lambda: [link.link_speakers(fea, Phi, offs, labels, Fa[g], Fb[g]) for g in range(G)]
    bat = lambda: link.link_many(fea, Phi, offs, [labels] * G, Fa, Fb)
    bat()                                                         # warm-up: allocator, module
    got, t_bat = timed(bat)
    want, t_seq = timed(seq)
    same = all(all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])) for a, b in zip(got, want))
    row = dict(G=G, M=M, N=int(fea.shape[0]), bit_identical=same, sequential_s=round(t_seq, 4),
               batched_s=round(t_bat, 4), whole_call_ratio=round(t_seq / t_bat, 2))
    if profiled:
        d_seq, d_bat = device_ms(seq), device_ms(bat)
        row.update(sequential_device_ms=d_seq, batched_device_ms=d_bat, device_ratio=round(d_seq / d_bat, 2))
    del fea
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-4000', action='store_true', help='leave out G = 64 x M = 4 000')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_link_sweep.py needs a CUDA device')
    dev = torch.device('cuda:0')
    rows = [problems(G, M, True) for M in (43, 1000) for G in (1, 64, 216)]
    if not args.skip_4000:
        rows.append(problems(64, 4000, False))

    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs, ref, _ = synth.multi_session_archive(z['x_raw'], n_rec=17, pool=40, lengths=(2000, 8000), speakers=(3, 5),
                                               seed=0)
    modes = {'without': {}, 'link_8_thresholds': dict(link_thresholds=THRESHOLDS)}
    run = lambda mode: sweep.sweep_batch(recs, transform, plda, GRID64, device=dev, ref_rttm=ref, **modes[mode])
    es = {'ES2005a': (z['x_raw'], z['seg_times'])}
    sweep.sweep_batch(es, transform, plda, dict(GRID64, Fa=[0.3], Fb=[17.0], loopP=[0.99]), device=dev,
                      link_thresholds=[0.0])                                                     # warm-up
    times = {mode: [] for mode in modes}
    host = []
    for _ in range(args.rounds):
        for mode in modes:
            out, t = timed(lambda: run(mode))
            times[mode].append(t)
            if mode != 'without':
                t0 = time.perf_counter()
                tot, ranking = sweep.summarize_across_files(out)
                host.append(time.perf_counter() - t0)
    best = ranking['full'][0]
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    med = {k: round(float(np.median(t)), 3) for k, t in times.items()}
    line = dict(
        bench='speaker linking inside the sweep', gpu=q.stdout.strip(), problems=rows,
        archive=f'synthetic multi-session, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, '
                f'{sum(lens)} in all, speakers from a pool of 40',
        settings=len(sweep.grid_settings(GRID64)), link_thresholds=THRESHOLDS, rounds=args.rounds,
        sweep_median_s=med, sweep_min_s={k: round(float(np.min(t)), 3) for k, t in times.items()},
        sweep_max_s={k: round(float(np.max(t)), 3) for k, t in times.items()},
        linking_cost_s=round(med['link_8_thresholds'] - med['without'], 3),
        across_files_host_median_s=round(float(np.median(host)), 3),
        best_across_files=dict(name=best, der=tot[best]['full']['der']))
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
