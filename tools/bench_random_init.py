"""Times random starts of the VB-HMM, init='RANDOM+VB' (DESIGN.md section 5.22), and measures what they do to DER.

(a) vbx_init_random alone at B = 4 096 recordings x T = 1 000 x-vectors with N = S = 16 and N = S = 128, float32 output.
    kernel_ms: the mean device time of init_random_kernel from the kernel events of a torch.profiler capture of
    `launches` calls; fill_ms: the same for a torch fill of the same gamma (a store-only kernel of the same bytes, the
    stores' achieved floor on this card).  bytes: the gamma and pi writes; model_ms: bytes at the data sheet's 3.35 TB/s.
    philox_blocks: Philox4x64-10 evaluations (N / 4 per x-vector), each 40 64-bit multiplies (20 high, 20 low halves).
(b) Long recordings: whole diarize_batch calls on one synthetic recording (synth.multi_session_archive(n_rec=1,
    lengths=(T, T)) from the ES2005a x-vectors) at T = 4 000, 8 000 and 16 000 with init='AHC+VB' and with
    init='RANDOM+VB', N = 10, R = 1 and R = 8; T = 30 000 with RANDOM+VB only.  Alternating, medians of --rounds (host
    clock around calls that end in a readback).  AHC+VB runs at a T only while the previous T's median, times 8 (the
    AHC's cost grows at least as T^2, its linkage near T^3), stays under --ahc-limit seconds; a size it skips is
    reported as skipped with that estimate.
(c) Accuracy: DER (full protocol) of AHC+VB and of RANDOM+VB with N = 10 at R = 1 and R = 8 on
    synth.multi_session_archive's default archive (seed 13) and on the T = 8 000 recording of (b).
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it there (after each
part, so that a partial run still leaves its numbers).

    python tools/bench_random_init.py --out profiles/h100_random_init.json
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
from vbx_b200 import pipeline, score, synth  # noqa: E402
from vbx_b200.batch import VbxBatch, _ptr  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden')
KW = dict(Fa=0.3, Fb=17.0, loopP=0.99, smoothing=5.0, threshold=-0.015, max_iters=40, epsilon=1e-6)
N_STATES = 10


def kernel_case(B, T, N, launches):
    """(a) for one shape."""
    dev = torch.device('cuda:0')
    vb = VbxBatch([T] * B, 128, N, device=dev, allocate=False)
    g = torch.empty((vb.N, vb.S), device=dev)
    p = torch.empty((B, vb.S), device=dev)
    keys = torch.arange(B, dtype=torch.int64, device=dev) * 7919 + 11
    seeds = torch.full((B,), 3, dtype=torch.int64, device=dev)
    stream = vb._stream()
    call = lambda: vb._check(vb.lib.vbx_init_random(vb._h, _ptr(keys), _ptr(seeds), None, _ptr(g), _ptr(p), 0, stream))
    for _ in range(3):
        call()
        g.fill_(0.5)
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(launches):
            call()
            g.fill_(0.5)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    us = [e.device_time for e in ev if 'init_random_kernel' in e.name]
    fill = [e.device_time for e in ev if 'fill' in e.name.lower() or 'FillFunctor' in e.name]
    call()
    assert bool(torch.allclose(g.view(B, T, vb.S).sum(2), torch.ones((B, T), device=dev)))
    nbytes = 4 * vb.N * vb.S + 4 * B * vb.S
    kms = float(np.mean(us)) / 1e3 if us else None
    fms = float(np.mean(fill)) / 1e3 if fill else None
    vb.close()
    del g
    torch.cuda.empty_cache()
    return dict(B=B, T=T, N=N, S=N, launches=launches, kernel_ms=round(kms, 4) if kms else None,
                kernel_events=len(us), fill_ms=round(fms, 4) if fms else None, bytes=int(nbytes),
                model_ms_at_3_35_TBps=round(nbytes / 3.35e12 * 1e3, 4),
                achieved_TBps=round(nbytes / (kms * 1e-3) / 1e12, 3) if kms else None,
                philox_blocks=B * T * (N // 4))


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def sys_rows(lines):
    return [(l.split()[1], float(l.split()[3]), float(l.split()[4]), l.split()[7]) for l in lines]


def full_der(ref, out):
    rows = [r for it in out.values() for r in sys_rows(it['rttm'])]
    return round(float(score.score_rttm(ref, rows, 0.0, False)[1]['der']), 4)


MODES = {'AHC+VB': dict(init='AHC+VB'),
         'RANDOM+VB R=1': dict(init='RANDOM+VB', init_states=N_STATES, restarts=1),
         'RANDOM+VB R=8': dict(init='RANDOM+VB', init_states=N_STATES, restarts=8)}


def long_recordings(transform, plda, z, rounds, ahc_limit, keep):
    out, ahc_est = [], 0.0
    for T in (4000, 8000, 16000, 30000):
        recs, ref, _ = synth.multi_session_archive(z['x_raw'], n_rec=1, lengths=(T, T))
        modes = [m for m in MODES if m != 'AHC+VB' or (T <= 16000 and ahc_est < ahc_limit)]
        row = dict(T=T, speakers=len({r[3] for r in ref}))
        if T <= 16000 and 'AHC+VB' not in modes:
            row['AHC+VB'] = f'skipped: about {ahc_est:.0f} s per call expected (8 x the median at T = {T // 2})'
        results = {}
        for m in modes:                                # an untimed warm-up, whose outputs are the ones scored in (c)
            results[m] = pipeline.diarize_batch(recs, transform, plda, **KW, **MODES[m])
        times = {m: [] for m in modes}
        for _ in range(rounds):
            for m in modes:
                times[m].append(timed(lambda: pipeline.diarize_batch(recs, transform, plda, **KW, **MODES[m]))[1])
        for m in modes:
            row[m] = dict(median_s=round(float(np.median(times[m])), 3),
                          all_s=[round(t, 3) for t in times[m]])
            if T == 8000:
                row[m]['der_full'] = full_der(ref, results[m])
            it = next(iter(results[m].values()))
            row[m].update(n_speakers=it['n_speakers'], iterations=it['iterations'])
            if 'restart' in it:
                row[m].update(restart=it['restart'], restart_elbos=[round(v, 2) for v in it['restart_elbos']])
        if 'AHC+VB' in modes:
            ahc_est = 8 * row['AHC+VB']['median_s']
        out.append(row)
        keep(out)
    return out


def accuracy(transform, plda, z):
    recs, ref, _ = synth.multi_session_archive(z['x_raw'])
    out = dict(archive=f'synth.multi_session_archive defaults (seed 13): {len(recs)} recordings', params=KW,
               init_states=N_STATES)
    for m, kw in MODES.items():
        res = pipeline.diarize_batch(recs, transform, plda, **KW, **kw)
        out[m] = dict(der_full=full_der(ref, res), speakers=sum(it['n_speakers'] for it in res.values()))
    out['reference_speakers'] = sum(len({r[3] for r in ref if r[0] == n}) for n in recs)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--ahc-limit', type=float, default=60.0, help='skip AHC+VB calls expected to take longer (s)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_random_init.py needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    line = dict(bench='random starts: vbx_init_random and diarize_batch(init=RANDOM+VB)', gpu=q.stdout.strip(),
                params=KW, init_states=N_STATES, rounds=args.rounds)

    def keep(part=None, key=None):
        if key is not None:
            line[key] = part
        if args.out:
            with open(args.out, 'w') as fp:
                fp.write(json.dumps(line) + '\n')

    keep(line['gpu'], 'gpu')
    keep([kernel_case(4096, 1000, N, args.launches) for N in (16, 128)], 'kernel')
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    keep(accuracy(transform, plda, z), 'accuracy')
    long_recordings(transform, plda, z, args.rounds, args.ahc_limit, lambda rows: keep(rows, 'long_recordings'))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
