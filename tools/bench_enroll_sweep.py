"""Times enrolment and cohort normalisation inside the sweep (DESIGN.md section 5.19).

(a) G enrolment problems of M archive speakers each (tools/bench_link.py's synthetic speakers, 4 per recording, R = 128;
    problem g with the Fa / Fb of setting g of tools/bench_sweep.py's 64-setting grid, cycled) against E enrolled
    speakers at 8 thresholds: 8 G enroll_speakers calls one after another (one per problem and threshold, what the
    single entry offers) against one enroll.enroll_many call (vbx_enroll_batch), for G in {1, 64, 216} x M in {43,
    1 000} x E in {10, 1 000}, and G = 64 x M = 16 000 x E = 1 000 (whole call only).  Whole-call time is a host clock
    around work that ends in a readback; device time is the sum of the kernels' times from the kernel events of a
    torch.profiler capture (the sequential calls once, the batched call 3 times) in a separate run (None when the
    capture holds none).
(b) The 64-setting sweep of tools/bench_sweep.py on tools/bench_link_sweep.py's seeded multi-session archive with its
    reference: without enrolment, with the 40 pool speakers enrolled (20 held-out x-vectors each) at 8 thresholds, and
    the same with a cohort of 200 other speakers; alternating, medians of 5.  summarize_by_name is timed on its own.
(c) The worked case of DESIGN.md section 5.19: synth.multi_session_archive with its defaults (seed 13), its pool of 10
    speakers enrolled with 20 held-out x-vectors each, a 3 x 3 grid of Fa x Fb, and DER by name (full protocol) of
    every setting at WORKED_T.
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it there.

    python tools/bench_enroll_sweep.py --out profiles/h100_enroll_sweep.json
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
from bench_sweep import GOLD, GRID64  # noqa: E402
from vbx_b200 import enroll, sweep, synth  # noqa: E402

THRESHOLDS = [-20.0, -10.0, 0.0, 10.0, 20.0, 30.0, 40.0, 60.0]
WORKED_T = [-40.0, -20.0, -10.0, 0.0, 10.0, 20.0, 40.0, 80.0]
WORKED_GRID = dict(Fa=[0.1, 0.3, 0.5], Fb=[6.0, 17.0, 64.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
KERNELS = ('link_init_kernel', 'link_span_kernel', 'link_stats_kernel', 'enroll_score_kernel', 'enroll_assign_kernel',
           'repeat_index_kernel', 'norm_scores_kernel')


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def device_ms(fn, repeats=3):
    """Mean summed device time (ms) of the enrolment kernels over `repeats` calls of fn, from the kernel events of one
    torch.profiler capture; None when the capture holds no such kernel (the profiler dropped them)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(repeats):
            fn()
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events()
          if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in KERNELS)]
    return round(sum(us) / repeats / 1e3, 3) if us else None


def problems(G, M, E, profiled):
    fea, Phi, offs, labels = speakers(M)
    rng = np.random.default_rng(E)
    espk = np.concatenate([np.arange(E), rng.integers(0, E, 2 * E)])
    efea = torch.randn((len(espk), fea.shape[1]), generator=torch.Generator().manual_seed(E)).to(fea.device)
    settings = sweep.grid_settings(GRID64)
    Fa = [settings[g % len(settings)].Fa for g in range(G)]
    Fb = [settings[g % len(settings)].Fb for g in range(G)]
    seq = lambda: [[enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, Fa[g], Fb[g], t) for t in THRESHOLDS]
                   for g in range(G)]
    bat = lambda: enroll.enroll_many(fea, Phi, offs, [labels] * G, efea, espk, Fa, Fb, THRESHOLDS)
    bat()                                                         # warm-up: allocator, module
    got, t_bat = timed(bat)
    want, t_seq = timed(seq)
    same = all(np.array_equal(got[g].assign[h], want[g][h].assign) and
               np.array_equal(got[g].best_llr[h], want[g][h].best_llr)
               for g in range(G) for h in range(len(THRESHOLDS)))
    row = dict(G=G, M=M, E=E, thresholds=len(THRESHOLDS), N=int(fea.shape[0]), bit_identical=same,
               sequential_s=round(t_seq, 4), batched_s=round(t_bat, 4), whole_call_ratio=round(t_seq / t_bat, 2))
    if profiled:
        d_seq, d_bat = device_ms(seq, 1), device_ms(bat, 3)
        row.update(sequential_device_ms=d_seq, batched_device_ms=d_bat,     # None: the profiler recorded no kernels
                   device_ratio=round(d_seq / d_bat, 2) if d_seq and d_bat else None)
    del fea, efea
    torch.cuda.empty_cache()
    return row


def pool_speakers(x_ref, seed, pool, n, offset=1000):
    """n x-vectors of each of `pool` speakers whose centres synth.multi_session_archive(seed=seed, pool=pool) draws."""
    x = np.asarray(x_ref, dtype=np.float64)
    sd = x.std(0)
    centres = x.mean(0) + 2.0 * sd * np.random.default_rng(seed).standard_normal((pool, x.shape[1]))
    rng = np.random.default_rng(seed + offset)
    return {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((n, x.shape[1])) for k in range(pool)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-16000', action='store_true', help='leave out G = 64 x M = 16 000')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_enroll_sweep.py needs a CUDA device')
    dev = torch.device('cuda:0')
    rows = [problems(G, M, E, True) for E in (10, 1000) for M in (43, 1000) for G in (1, 64, 216)]
    if not args.skip_16000:
        rows.append(problems(64, 16000, 1000, False))

    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs, ref, _ = synth.multi_session_archive(z['x_raw'], n_rec=17, pool=40, lengths=(2000, 8000), speakers=(3, 5),
                                               seed=0)
    held = pool_speakers(z['x_raw'], 0, 40, 20)
    coh = {f'c{k}': v for k, v in pool_speakers(z['x_raw'], 77, 200, 5).items()}
    modes = {'without': {}, 'enroll_8_thresholds': dict(enroll=held, enroll_thresholds=THRESHOLDS),
             'enroll_8_thresholds_cohort_200': dict(enroll=held, enroll_thresholds=THRESHOLDS, cohort=coh)}
    run = lambda mode: sweep.sweep_batch(recs, transform, plda, GRID64, device=dev, ref_rttm=ref, **modes[mode])
    es = {'ES2005a': (z['x_raw'], z['seg_times'])}
    sweep.sweep_batch(es, transform, plda, dict(GRID64, Fa=[0.3], Fb=[17.0], loopP=[0.99]), device=dev, enroll=held,
                      enroll_thresholds=[0.0], cohort=coh)                                        # warm-up
    times = {mode: [] for mode in modes}
    host = []
    best = {}
    for _ in range(args.rounds):
        for mode in modes:
            out, t = timed(lambda: run(mode))
            times[mode].append(t)
            if mode != 'without':
                t0 = time.perf_counter()
                tot, ranking = sweep.summarize_by_name(out)
                host.append(time.perf_counter() - t0)
                best[mode] = dict(name=ranking['full'][0], der_by_name=tot[ranking['full'][0]]['full']['der'])
    wrecs, wref, _ = synth.multi_session_archive(z['x_raw'])
    wout = sweep.sweep_batch(wrecs, transform, plda, WORKED_GRID, device=dev, ref_rttm=wref,
                             enroll=pool_speakers(z['x_raw'], 13, 10, 20), enroll_thresholds=WORKED_T)
    wtot, wrank = sweep.summarize_by_name(wout)
    worked = dict(thresholds=WORKED_T, best=wrank['full'][0],
                  der_by_name={s.name: [round(wtot[sweep.enroll_key(s, t)]['full']['der'], 4) for t in WORKED_T]
                               for s in wout})
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    med = {k: round(float(np.median(t)), 3) for k, t in times.items()}
    line = dict(
        bench='enrolment and cohort normalisation inside the sweep', gpu=q.stdout.strip(), problems=rows,
        archive=f'synthetic multi-session, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, '
                f'{sum(lens)} in all, speakers from a pool of 40, all 40 enrolled with 20 held-out x-vectors each; '
                f'cohort: 200 other speakers, 5 x-vectors each',
        settings=len(sweep.grid_settings(GRID64)), enroll_thresholds=THRESHOLDS, rounds=args.rounds,
        sweep_median_s=med, sweep_min_s={k: round(float(np.min(t)), 3) for k, t in times.items()},
        sweep_max_s={k: round(float(np.max(t)), 3) for k, t in times.items()},
        enrolment_cost_s=round(med['enroll_8_thresholds'] - med['without'], 3),
        cohort_cost_s=round(med['enroll_8_thresholds_cohort_200'] - med['enroll_8_thresholds'], 3),
        by_name_host_median_s=round(float(np.median(host)), 3), best_by_name=best, worked_case=worked)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
