"""Device time of the score calibration (DESIGN.md section 5.28), and calibration on a held-out list.

Workloads: the two trial lists of tools/bench_verify.py without a cohort, scored on the device at R = 128, Fa = 0.3,
Fb = 17 (vox1o: 37 720 trials; large: 10 000 000 trials).  Per workload:
  - kernel times from torch.profiler in a run of its own: the sort prefix (keys, radix sort, labels, scan), the class
    split and init, every Newton evaluation and update launch (those after convergence return at once; the ones that
    ran are the first `passes`), the hull levels, the minCllr segments and final kernel;
  - the whole verify.calibrate call by host clock around a synchronised call, median of 5, profiler off;
  - the float64 oracle on the host cores (the whole vox1o list; the first 1 000 000 trials of large);
  - the byte model of one Newton evaluation: 8 bytes per trial (its class-split score), over the kernel's time;
  - held out: the same workload drawn again with another seed, calibrated on the first list and evaluated on the second
    (actDCF and Cllr of a s + b against minDCF and minCllr of the held-out list).
The card's name, power limit and SM clock limit are read in the same call.

    python tools/bench_calibrate.py --out profiles/h100_calibrate.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_verify import FA, FB, R, card, workload  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
P_TARGETS = (0.01, 0.001)


def profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    groups = dict(sort_prefix=[], split_init=[], newton_eval=[], newton_update=[], hull_chunk=[], hull_merge=[],
                  min_cllr=[])
    keys = (('calibrate_eval', 'newton_eval'), ('calibrate_update', 'newton_update'),
            ('calibrate_hull_chunk', 'hull_chunk'), ('calibrate_hull_merge', 'hull_merge'),
            ('calibrate_segments', 'min_cllr'), ('calibrate_final', 'min_cllr'), ('calibrate_split', 'split_init'),
            ('calibrate_init', 'split_init'), ('verify_keys', 'sort_prefix'), ('verify_tar', 'sort_prefix'),
            ('Radix', 'sort_prefix'), ('Onesweep', 'sort_prefix'), ('onesweep', 'sort_prefix'),
            ('DeviceScan', 'sort_prefix'))
    events = sorted((e for e in p.events() if e.device_type.name == 'CUDA'), key=lambda e: e.time_range.start)
    for e in events:
        if 'emcpy' in e.name or 'emset' in e.name:
            continue
        us = e.device_time if hasattr(e, 'device_time') else e.cuda_time
        for k, g in keys:
            if k in e.name:
                groups[g].append(us / 1e3)
                break
    return groups


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_calibrate.json'))
    ap.add_argument('--workloads', default='vox1o,large')
    args = ap.parse_args()
    import torch
    from oracle import calibrate_oracle as O
    from vbx_b200 import synth, verify
    dev = torch.device('cuda:0')
    Phi = synth.plda_phi(R).astype(np.float32)
    res = dict(card=card(), R=R, Fa=FA, Fb=FB, hbm_bytes_per_s=HBM_BYTES_PER_S, workloads={})
    for name in args.workloads.split(','):
        lists = []
        for seed in (7, 8):
            fe, ie, ft, it, tr, y = workload(name, np.random.default_rng(seed), Phi)
            s = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=FA, Fb=FB, device=dev)
            lists.append((torch.from_numpy(s).to(dev), s, y))
        sd, s, y = lists[0]
        T = len(s)
        call = lambda: verify.calibrate(sd, y, device=dev)
        fit = call()                                               # warm-up
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        kern = profile(call)
        active = kern['newton_eval'][:fit['passes']]
        eval_bytes = 8 * T
        row = dict(trials=T, n_target=fit['n_target'], passes=fit['passes'], hull_vertices=fit['hull_vertices'],
                   a=fit['a'], b=fit['b'], cllr_prior=fit['cllr_prior'], min_cllr=fit['min_cllr'],
                   whole_call_ms_median=1e3 * float(np.median(walls)), whole_call_ms=[1e3 * w for w in walls],
                   kernels_ms={g: float(np.sum(v)) for g, v in kern.items()},
                   launches={g: len(v) for g, v in kern.items()},
                   newton_eval_ms_per_active_pass=float(np.mean(active)) if active else None,
                   newton_eval_ms_after_convergence=float(np.mean(kern['newton_eval'][fit['passes']:]))
                   if len(kern['newton_eval']) > fit['passes'] else None,
                   hull_merge_ms_per_level=kern['hull_merge'], newton_eval_bytes=eval_bytes)
        if active:
            row['newton_eval_fraction_of_hbm'] = eval_bytes / (np.mean(active) * 1e-3) / HBM_BYTES_PER_S
        n = min(T, 1000000)
        t0 = time.perf_counter()
        ref = O.calibrate(s[:n], y[:n])
        row['oracle_host_s'] = time.perf_counter() - t0
        row['oracle_trials'] = n
        if n == T:
            row['oracle_rel_err'] = {k: abs(fit[k] - ref[k]) / abs(ref[k]) for k in ('a', 'b', 'cllr_prior', 'min_cllr')}
            row['oracle_hull_vertices_equal'] = fit['hull_vertices'] == ref['hull_vertices']
        # held out: calibrate on list 0, evaluate on list 1
        _, s1, y1 = lists[1]
        held = verify.calibrate(s1, y1, device=dev)
        raw = verify.error_rates(s1, y1, P_TARGETS, device=dev)
        cal = verify.error_rates(fit['a'] * s1 + fit['b'], y1, P_TARGETS, device=dev)
        row['held_out'] = dict(p_target=list(P_TARGETS), min_dcf=raw['min_dcf'], min_cllr=held['min_cllr'],
                               raw=dict(cllr=raw['cllr'], act_dcf=raw['act_dcf']),
                               calibrated=dict(cllr=cal['cllr'], act_dcf=cal['act_dcf']),
                               self_calibrated_cllr=held['cllr_prior'])
        res['workloads'][name] = row
        print(name, json.dumps({k: row[k] for k in ('whole_call_ms_median', 'passes', 'hull_vertices',
                                                      'newton_eval_ms_per_active_pass')}),
              json.dumps(row['kernels_ms']), json.dumps(row['held_out']), flush=True)
    res['host_cores'] = os.cpu_count()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
