"""Times enrolled speakers as state priors of the VB-HMM (DESIGN.md section 5.23).

1. The speaker-model kernel with and without a prior: 4 096 recordings x 1 000 x-vectors, R = 128, S = 16 and
   S = 128, --launches EM iterations at a fixed iteration count, with the library's per-class timing (CUDA events
   around every launch): speaker_model_kernel against speaker_model_prior_kernel on the same batch.
2. The EM iteration of the headline batch (bench.py's: 4 096 x 1 000, S = 16, 10 iterations, as one batch) with
   vbx_run against vbx_run_prior with an all-zero prior, the C entries called directly (no host-side checks in the
   timed window), alternating in one process (medians of --rounds), outputs compared.
3. Whole diarize_batch calls on the synthetic multi-session archive of tests/test_enroll_prior_gpu.py (8 recordings,
   10 pool speakers, 20 enrolment x-vectors each) with post-hoc enrolment and with enroll_prior, alternating (medians
   of --rounds), with DER per file and by name (collar 0.25, overlaps scored) at both pool spreads.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_enroll_prior.py --out profiles/h100_enroll_prior.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from bench import WORKLOADS, make_device_batch  # noqa: E402
from vbx_b200 import pipeline, score  # noqa: E402
from vbx_b200.batch import VbxBatch  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')


def speaker_model(S, launches, dev):
    """Device ms per launch of the speaker-model kernel without and with a prior (half the states enrolled)."""
    lens = np.full(4096, 1000, dtype=np.int64)
    d = make_device_batch(lens, S, 17, dev)
    vb = VbxBatch(lens, 128, S, device=dev, exact_stop=False)
    vb.prepare_project(d['X'], d['V'], d['Phi'])
    rng = np.random.default_rng(0)
    pn = np.zeros((4096, vb.S))
    pn[:, ::2] = rng.integers(1, 300, (4096, (vb.S + 1) // 2))
    pF = rng.normal(0, 3.0, (4096, vb.S, 128)) * pn[:, :, None] ** 0.5
    prior = (torch.from_numpy(pn).to(dev), torch.from_numpy(pF).to(dev))
    out = {}
    vb.set_option('timing', 1)
    for mode in ('plain', 'prior', 'plain', 'prior'):       # second pass is the measured one
        g = d['gamma0'].clone()
        p = torch.full((4096, vb.S), 1.0 / S, device=dev)
        vb.timings(reset=True)
        vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=launches, epsilon=-np.inf,
               prior=prior if mode == 'prior' else None)
        torch.cuda.synchronize()
        ms, n = vb.timings(reset=True)['speaker_model']
        out[mode] = round(1e3 * ms / max(n, 1), 2)
    vb.close()
    del d
    torch.cuda.empty_cache()
    return {'us_per_launch': out, 'launches': launches}


def em_step(rounds, dev):
    """The headline batch's EM iteration through vbx_run and through vbx_run_prior with an all-zero prior, alternating.
    One VbxBatch (no sub-batches) and the C entries called directly, so that the host-side checks of VbxBatch.run (a
    device-to-host copy of the per-recording values and of the prior) stay out of the timed window."""
    import ctypes
    w = WORKLOADS['headline']
    lens = np.full(w['B'], w['T'], dtype=np.int64)
    d = make_device_batch(lens, w['S'], 1234, dev)
    vb = VbxBatch(lens, 128, w['S'], device=dev)
    vb.prepare_project(d['X'], d['V'], d['Phi'])
    hyper = vb._hyper(w['Fa'], w['Fb'], w['loopP'], arrays=True)
    zero = (torch.zeros((w['B'], vb.S), dtype=torch.float64, device=dev),
            torch.zeros((w['B'], vb.S, 128), dtype=torch.float64, device=dev))
    g = torch.empty_like(d['gamma0'])
    p = torch.empty((w['B'], vb.S), device=dev)
    bufs = vb.output_buffers(w['iters'])
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    common = lambda: (vb._h, P(vb.rho), P(vb.Phi), P(g), P(p), P(vb.n_states))
    tail = (int(w['iters']), float(-np.inf), None, None, 0, P(bufs['Li']), P(bufs['n_iters']), P(bufs['flags']))

    def once(prior):
        g.copy_(d['gamma0'])
        p.fill_(1.0 / w['S'])
        torch.cuda.synchronize()
        st = vb._stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if prior is None:
            rc = vb.lib.vbx_run(*common(), float(w['Fa']), float(w['Fb']), float(w['loopP']), *tail, st)
        else:
            rc = vb.lib.vbx_run_prior(*common(), *(P(t) for t in hyper), *tail, P(prior[0]), P(prior[1]), st)
        e1.record()
        torch.cuda.synchronize()
        assert rc == 0, vb.lib.vbx_last_error(vb._h)
        return e0.elapsed_time(e1) / w['iters'], (g.clone(), p.clone(), bufs['Li'].clone())

    once(None)
    once(zero)
    times = {'vbx_run': [], 'vbx_run_prior_zero': []}
    same = True
    for _ in range(rounds):
        a, ra = once(None)
        b, rb = once(zero)
        times['vbx_run'].append(a)
        times['vbx_run_prior_zero'].append(b)
        same = same and all(torch.equal(x, y) for x, y in zip(ra, rb))
    vb.close()
    del d
    torch.cuda.empty_cache()
    return dict(ms_per_iteration_median={k: round(float(np.median(v)), 3) for k, v in times.items()},
                ms_per_iteration_min={k: round(float(np.min(v)), 3) for k, v in times.items()},
                ms_per_iteration_max={k: round(float(np.max(v)), 3) for k, v in times.items()},
                bit_identical=bool(same), rounds=rounds, batch='one VbxBatch, C entries called directly')


def sessions(x_es, seed=13, n_rec=8, pool=10, spread=2.0):
    """tests/test_enroll_prior_gpu.py's synthetic archive: (recordings, reference rows, enrolment)."""
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + spread * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, rows = {}, []
    for r in range(n_rec):
        T = int(rng.integers(300, 601))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        recs[f'ses{r:02d}'] = (x, seg)
        rows += [(f'ses{r:02d}', round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    return recs, rows, held


def der(rows, items):
    sys_rows = [(line.split()[1], float(line.split()[3]), float(line.split()[4]), line.split()[7])
                for it in items.values() for line in it['rttm_named']]
    per, tot = score.score_rttm(rows, sys_rows, 0.25, False, by_name=True)
    return dict(per_file={n: round(100 * v['der'], 2) for n, v in per.items()}, overall=round(100 * tot['der'], 2),
                by_name=round(100 * tot['by_name']['der'], 2))


def pipeline_calls(rounds, threshold, dev):
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    kw = dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']),
              threshold=-0.015, max_iters=40, epsilon=1e-6, device=dev)
    out = {}
    for spread in (2.0, 0.7):
        recs, rows, held = sessions(z['x_raw'], spread=spread)
        modes = {'post_hoc': dict(enroll=held, enroll_threshold=threshold),
                 'enroll_prior': dict(enroll=held, enroll_threshold=threshold, enroll_prior=True)}

        def call(mode):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = pipeline.diarize_batch(recs, transform, plda, **kw, **modes[mode])
            torch.cuda.synchronize()
            return res, time.perf_counter() - t0

        res = {mode: call(mode)[0] for mode in modes}
        times = {mode: [] for mode in modes}
        for _ in range(rounds):
            for mode in modes:
                times[mode].append(call(mode)[1])
        out[f'spread_{spread}'] = dict(
            median_s={k: round(float(np.median(t)), 4) for k, t in times.items()},
            min_s={k: round(float(np.min(t)), 4) for k, t in times.items()},
            max_s={k: round(float(np.max(t)), 4) for k, t in times.items()},
            der={k: der(rows, r) for k, r in res.items()},
            priors_attached=sum(len(it['prior_speakers']) for it in res['enroll_prior'].values()),
            speakers={k: sum(len(it['speaker_names']) for it in r.values()) for k, r in res.items()})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--threshold', type=float, default=20.0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_enroll_prior.py needs a CUDA device')
    dev = torch.device('cuda', torch.cuda.current_device())
    line = dict(bench='enrolled speakers as state priors of the VB-HMM')
    line['speaker_model_4096x1000'] = {f'S{S}': speaker_model(S, args.launches, dev) for S in (16, 128)}
    line['headline_em_step'] = em_step(args.rounds, dev)
    line['diarize_batch'] = dict(pipeline_calls(args.rounds, args.threshold, dev), rounds=args.rounds,
                                 enroll_threshold=args.threshold,
                                 archive='synthetic, seeded: 8 recordings of 300 .. 600 x-vectors, 2 .. 5 of 10 pool '
                                         'speakers each, 20 enrolment x-vectors per pool speaker')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    line['gpu'] = q.stdout.strip()
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
