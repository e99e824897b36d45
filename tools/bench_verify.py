"""Device time of speaker-verification trial scoring and its error rates (DESIGN.md section 5.27).

Workloads, all at R = 128 with Fa = 0.3, Fb = 17, each with and without a 1 000-speaker cohort (3 x-vectors each):
  vox1o  a VoxCeleb1-O-shaped list: 4 874 single-x-vector items of 40 speakers on both sides, 37 720 trials
  large  100 000 enrolment items of 3 x-vectors, 1 000 000 single-x-vector test items, 10 000 000 trials
Reports per kernel group (statistics, scores, normalisation-free sort, sweep) the device time from torch.profiler in a
run of its own, the whole score_trials + error_rates call by host clock around a synchronised call (median of 5, profiler
off), and the float64 oracle on the host cores (the whole vox1o list; the first 1 000 000 trials of large).  Byte model of
the score kernel: every trial reads its two b rows, 2 x 128 x 8 bytes, and writes 8 bytes; items' statistics read their
x-vectors once.  The card's name, power limit and SM clock limit are read in the same call.

    python tools/bench_verify.py --out profiles/h100_verify.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R = 128
FA, FB = 0.3, 17.0


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def speakers(n_spk, rng, Phi):
    return rng.standard_normal((n_spk, R)).astype(np.float32) * np.sqrt(Phi)


def workload(name, rng, Phi):
    if name == 'vox1o':
        K, N, T = 40, 4874, 37720
        y = speakers(K, rng, Phi)
        who = rng.integers(0, K, N)
        fea = (y[who] + rng.standard_normal((N, R)).astype(np.float32))
        i = rng.integers(0, N, T)
        same = rng.random(T) < 0.5                                   # half of the trials are target trials
        j = np.where(same, 0, rng.integers(0, N, T))
        for k in np.nonzero(same)[0]:
            pool = np.nonzero(who == who[i[k]])[0]
            j[k] = pool[rng.integers(0, len(pool))]
        return fea, np.arange(N), fea, np.arange(N), np.stack([i, j], 1), who[i] == who[j]
    K, M_e, N_t, T = 20000, 100000, 1000000, 10000000
    y = speakers(K, rng, Phi)
    we, wt = rng.integers(0, K, M_e), rng.integers(0, K, N_t)
    ie = np.repeat(np.arange(M_e), 3)
    fe = y[we][ie] + rng.standard_normal((3 * M_e, R)).astype(np.float32)
    ft = y[wt] + rng.standard_normal((N_t, R)).astype(np.float32)
    tr = np.stack([rng.integers(0, M_e, T), rng.integers(0, N_t, T)], 1)
    return fe, ie, ft, np.arange(N_t), tr, we[tr[:, 0]] == wt[tr[:, 1]]


GROUPS = (('statistics', ('link_span', 'link_stats', 'link_init')), ('scores', ('verify_score',)),
          ('sort', ('RadixSort', 'Onesweep', 'onesweep')),
          ('sweep', ('verify_keys', 'verify_tar', 'DeviceScan', 'verify_sweep', 'verify_cllr', 'verify_final')),
          ('cohort', ('enroll_score', 'cohort_topk', 'repeat_index')))


def profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    out = {g: 0.0 for g, _ in GROUPS}
    other = {}
    for e in p.events():
        if e.device_type.name != 'CUDA' or 'emcpy' in e.name or 'emset' in e.name:
            continue
        us = e.device_time if hasattr(e, 'device_time') else e.cuda_time
        for g, keys in GROUPS:
            if any(k in e.name for k in keys):
                out[g] += us / 1e3
                break
        else:
            other[e.name[:60]] = other.get(e.name[:60], 0.0) + us / 1e3
    out['other'] = other
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_verify.json'))
    ap.add_argument('--workloads', default='vox1o,large')
    args = ap.parse_args()
    import torch
    from oracle import verify_oracle as O
    from vbx_b200 import synth, verify
    dev = torch.device('cuda:0')
    Phi = synth.plda_phi(R).astype(np.float32)
    res = dict(card=card(), R=R, Fa=FA, Fb=FB, workloads={})
    for name in args.workloads.split(','):
        rng = np.random.default_rng(7)
        fe, ie, ft, it, tr, y = workload(name, rng, Phi)
        fc = (speakers(1000, rng, Phi)[np.repeat(np.arange(1000), 3)] +
              rng.standard_normal((3000, R)).astype(np.float32))
        ic = np.repeat(np.arange(1000), 3)
        for with_cohort in (False, True):
            def call():
                norm = verify.trial_norm(fe, ie, ft, it, Phi, fc, ic, FA, FB, top_k=200, device=dev) \
                    if with_cohort else None
                s = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=FA, Fb=FB, norm=norm, device=dev)
                return s, verify.error_rates(s, y, (0.01, 0.001), device=dev)
            s, m = call()                                         # warm-up: module load, every shape
            torch.cuda.synchronize()
            walls = []
            for _ in range(5):
                t0 = time.perf_counter()
                call()
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
            kern = profile(call)
            T = len(tr)
            score_bytes = T * (2 * R * 8 + 8 + 8)
            row = dict(trials=T, enroll_items=int(ie.max()) + 1, test_items=int(it.max()) + 1,
                       enroll_xvectors=len(fe), test_xvectors=len(ft), cohort_speakers=1000 if with_cohort else 0,
                       kernels_ms=kern, whole_call_ms_median=1e3 * float(np.median(walls)),
                       whole_call_ms=[1e3 * w for w in walls], score_kernel_bytes=score_bytes,
                       score_kernel_GBps=score_bytes / (kern['scores'] * 1e-3) / 1e9 if kern['scores'] else None,
                       eer=m['eer'], min_dcf=m['min_dcf'], cllr=m['cllr'])
            if not with_cohort:
                n = min(T, 1000000)
                t0 = time.perf_counter()
                ne, Fe = O.statistics(fe.astype(np.float64), ie, int(ie.max()) + 1)
                nt, Ft = O.statistics(ft.astype(np.float64), it, int(it.max()) + 1)
                ref = O.llr_trials(ne, Fe, nt, Ft, Phi.astype(np.float64), FA / FB, tr[:n, 0], tr[:n, 1])
                om = O.error_rates(ref, y[:n], (0.01, 0.001))
                row['oracle_host_s'] = time.perf_counter() - t0
                row['oracle_trials'] = n
                row['oracle_max_rel_err'] = float(np.max(np.abs(s[:n] - ref) / np.maximum(np.abs(ref), 1.0)))
                if n == T:
                    row['oracle_metrics_equal'] = bool(om['eer'] == m['eer'] and om['min_dcf'] == m['min_dcf'])
            res['workloads'][f'{name}{"_cohort" if with_cohort else ""}'] = row
            print(name, 'cohort' if with_cohort else 'plain', json.dumps({k: row[k] for k in
                  ('whole_call_ms_median', 'eer', 'cllr')}), json.dumps(kern), flush=True)
    res['host_cores'] = os.cpu_count()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
