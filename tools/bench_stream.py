"""Times streaming diarization (DESIGN.md section 5.25) and measures its quality against offline AHC + VB.

1. Speed.  1 024 and 4 096 concurrent synthetic streams (pool speakers around ES2005a's mean x-vector, 2 .. 5 per
   stream, sticky turns), pushes of 40 x-vectors (10 s at the 0.25 s shift) to every stream, C = 240.  The first
   ceil(C / 40) + 1 pushes bring every stream past its first C x-vectors and are not timed; the next --pushes are.  Per
   push: the wall time (host clock around the push, which ends with its labels on the host, so the device is
   synchronised) and the stages StreamDiarizer.push times: the front end and the VB-HMM (prepare, run, hard labels) as
   CUDA-event intervals, which also hold host work (the PLDA diagonalisation and the block's upload; run()'s host
   checks of the prior); the device AHC with the linkage's copy to the host (events); the host cut of every block
   (host clock); the window and commit kernels alone (events right around their launches).  rest_share is the wall
   time outside all of these: plans, the wrappers' host checks and uploads, label readback.  The real-time factor is
   stream-seconds of audio per second of wall time.  The bytes window and commit must move (window_commit_bytes, from
   the push's tier shapes) over their kernel time give their achieved bandwidth.
2. Quality.  The synthetic archive of test_enroll_gpu.py (8 recordings, 2 .. 5 pool speakers at 2 sd) streamed with
   5 / 10 / 30 s blocks and C = 120 and 240, scored (collar 0.25) against the reference and against offline AHC + VB.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_stream.py --out profiles/h100_stream.json

With --enroll-speakers E1,E2,... it measures enrolled speakers in streams (DESIGN.md section 5.29) instead:
3. Speed, per E: the streams of 1. (--streams, C = 240, 10 s pushes) run by two StreamDiarizers fed the same blocks,
   one with E enrolled speakers (20 x-vectors each; the first min(E, 200) are the pool speakers the streams draw from,
   the rest speakers no stream has), threshold 0, and one without; after the warm-up pushes the two alternate which
   pushes first.  Per push the wall time of each (medians), the naming step's interval (timing['enroll']), the
   candidates it scored and their LLR pairs (candidates x E), and a byte model of the statistics kernel.  One more push
   runs under torch.profiler for the device time of each new kernel.
4. Quality: the archive of the enrolment tests (8 recordings, 10 pool speakers, 20 held-out x-vectors of each enrolled)
   streamed with 5 and 10 s blocks (C = 240), with and without enroll_prior, scored by name (collar 0.25) against the
   reference, beside offline diarize_batch(enroll=[, enroll_prior]) at the same threshold; and the share of stream
   speakers named at their first push.

    python tools/bench_stream.py --streams 4096 --enroll-speakers 100,1000 --out profiles/h100_stream_enroll.json
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
from vbx_b200.stream import StreamDiarizer, block_schedule  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
H, SHIFT = 40, 0.25


def model():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'es2005a.npz'))
    m = np.load(os.path.join(ROOT, 'tests', 'golden', 'es2005a_model.npz'))
    kw = dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']))
    return z['x_raw'], (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi']), kw


class Streams:
    """n synthetic live streams: each push draws the next H x-vectors of every stream."""

    def __init__(self, x_ref, n, seed):
        self.rng = np.random.default_rng(seed)
        sd = x_ref.std(0)
        self.sd, self.mean = sd.astype(np.float32), x_ref.mean(0).astype(np.float32)
        self.centres = (self.mean + 2.0 * sd * self.rng.standard_normal((200, x_ref.shape[1]))).astype(np.float32)
        self.who = [self.rng.choice(200, int(self.rng.integers(2, 6)), replace=False) for _ in range(n)]
        self.cur = np.zeros(n, dtype=np.int64)
        self.t = 0

    def block(self):
        out = {}
        seg = np.stack([np.arange(self.t, self.t + H) * SHIFT, np.arange(self.t, self.t + H) * SHIFT + 1.5], 1)
        for i, who in enumerate(self.who):
            spk = np.empty(H, dtype=np.int64)
            c = self.cur[i]
            for t in range(H):
                if self.rng.random() >= 0.97:
                    c = self.rng.integers(len(who))
                spk[t] = c
            self.cur[i] = c
            x = self.centres[who[spk]] + 0.5 * self.sd * self.rng.standard_normal((H, len(self.sd)), dtype=np.float32)
            out[f's{i:05d}'] = (x, seg)
        self.t += H
        return out


def window_commit_bytes(tiers, R):
    """Bytes the window and commit kernels must move in one push, from the shapes of its state tiers (the push's
    timing record).  Window: reads the context rows (features and labels), the block (features and AHC labels) and the
    K known speakers' history (n and F), writes the window's features and gamma0, pi0 and the prior at the tier's S.
    Commit: reads the window labels of the block rows, the evicted rows (features and labels) and the block's features,
    adds every evicted row to the history (read and write of n and F), writes the block into the ring (features and
    labels) and its final labels."""
    window = commit = 0
    for t in tiers:
        n, S, L, h, e, K = t['streams'], t['S'], t['context_rows'], t['block_rows'], t['evicted_rows'], t['known_speakers']
        window += L * (R * 4 + 4) + h * (R * 4 + 4) + K * (R + 1) * 8 + (L + h) * (R + S) * 4 + n * S * 4 \
            + n * S * (R + 1) * 8
        commit += h * 4 + e * (R * 4 + 4) + h * R * 4 + 2 * e * (R + 1) * 8 + h * (R * 4 + 4) + h * 4
    return window, commit


def speed(n, pushes, x_ref, transform, plda, kw, dev):
    src = Streams(x_ref, n, seed=n)
    sd = StreamDiarizer(transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'], context=240,
                        device=dev)
    for _ in range(240 // H + 1):
        sd.push(src.block())
    sd.timing = []
    walls = []
    for _ in range(pushes):
        blk = src.block()
        t0 = time.perf_counter()
        sd.push(blk)
        walls.append(time.perf_counter() - t0)
    T = sd.timing
    K = np.array([st.K for st in sd.streams.values()])
    med = lambda v: float(np.median(v))
    wall = med(walls)
    stages = {k: med([t[k] for t in T]) for k in ('front_end', 'ahc_linkage', 'ahc_host_cut', 'window', 'vb', 'commit')}
    wb, cb = (med([window_commit_bytes(t['tiers'], sd.R)[i] for t in T]) for i in range(2))
    return dict(streams=n, block_xvectors=H, context=240, pushes_timed=pushes, wall_ms=round(wall * 1e3, 2),
                wall_ms_min=round(min(walls) * 1e3, 2),
                stage_ms={k: round(v * 1e3, 3) for k, v in stages.items()},
                stage_share={k: round(v / wall, 4) for k, v in stages.items()},
                rest_share=round(1.0 - sum(stages.values()) / wall, 4),
                tiers=T[-1]['tiers'], real_time_factor=round(n * H * SHIFT / wall, 1),
                speakers_mean=round(float(K.mean()), 2),
                window_bytes=int(wb), window_kernel_GBps=round(wb / stages['window'] / 1e9, 1),
                commit_bytes=int(cb), commit_kernel_GBps=round(cb / stages['commit'] / 1e9, 1))


def quality(x_ref, transform, plda, kw, dev):
    recs, rows, _ = synth.multi_session_archive(x_ref, n_rec=8, seed=13)
    opts = dict(threshold=-0.015, max_iters=40, epsilon=1e-6)
    off = pipeline.diarize_batch(recs, transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'],
                                 init='AHC+VB', **opts)
    turns = lambda lines: [(l.split()[1], float(l.split()[3]), float(l.split()[4]), l.split()[7]) for l in lines]
    off_rows = [r for n in recs for r in turns(off[n]['rttm'])]
    der = lambda ref, sys_rows: round(100 * score.score_rttm(ref, sys_rows, 0.25, False)[1]['der'], 2)
    out = dict(offline_der_vs_reference=der(rows, off_rows), runs=[])
    for C in (120, 240):
        for B in (5.0, 10.0, 30.0):
            sd = StreamDiarizer(transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'], context=C,
                                device=dev, **opts)
            for push in block_schedule(recs, B):
                if push:
                    sd.push({n: (recs[n][0][r], recs[n][1][r]) for n, r in push.items()})
            sys_rows = [r for n in recs for r in turns(sd.rttm(n))]
            out['runs'].append(dict(block_seconds=B, context=C, der_vs_reference=der(rows, sys_rows),
                                    der_vs_offline=der(off_rows, sys_rows)))
    return out


ENROLL_KERNELS = ('stream_enroll_stats_kernel', 'enroll_score_kernel', 'stream_enroll_mask_kernel',
                  'enroll_assign_kernel', 'stream_enroll_apply_kernel')


def enrolled_speakers(src, E, dim, seed):
    """E enrolled speakers of 20 x-vectors: the first min(E, 200) around the pool centres of src, the rest around new
    centres no stream draws from."""
    rng = np.random.default_rng(seed)
    extra = src.mean + 2.0 * src.sd * rng.standard_normal((max(E - len(src.centres), 0), dim))
    centres = np.concatenate([src.centres, extra.astype(np.float32)])[:E]
    return {f'e{j:04d}': c + 0.5 * src.sd * rng.standard_normal((20, dim)) for j, c in enumerate(centres)}


def stats_bytes(timing, C, R, E):
    """Bytes stream_enroll_stats_kernel moves at most in one push: per stream with candidates the ring's labels and
    every ring row (C (R + 1) 4; only the candidates' rows are read), per candidate its history read and its b, e, n
    written ((R + 1) 8 each way), per enrolled speaker n_e, F_e read and b, e, n written."""
    return timing['enroll_streams'] * C * (R + 1) * 4 + timing['enroll_candidates'] * (R + 1) * 16 + E * (R + 1) * 16


def enroll_speed(n, E, pushes, x_ref, transform, plda, kw, dev):
    src = Streams(x_ref, n, seed=n)
    enr = enrolled_speakers(src, E, x_ref.shape[1], seed=E)
    mk = lambda **e: StreamDiarizer(transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'],
                                    context=240, device=dev, **e)
    sd_e, sd_0 = mk(enroll=enr, enroll_threshold=0.0), mk()
    for _ in range(240 // H + 1):
        blk = src.block()
        sd_e.push(blk)
        sd_0.push(blk)
    sd_e.timing = []
    walls = {'with': [], 'without': []}
    for i in range(pushes):
        blk = src.block()
        for which in (('with', 'without') if i % 2 == 0 else ('without', 'with')):
            sd = sd_e if which == 'with' else sd_0
            t0 = time.perf_counter()
            sd.push(blk)
            walls[which].append(time.perf_counter() - t0)
    T = sd_e.timing
    blk = src.block()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        sd_e.push(blk)
        torch.cuda.synchronize(dev)
    dev_us = {}
    for ev in prof.key_averages():
        for k in ENROLL_KERNELS:
            if k in ev.key:
                dev_us[k] = dev_us.get(k, 0.0) + ev.device_time_total
    med = lambda v: float(np.median(v))
    cand = med([t['enroll_candidates'] for t in T])
    sb = med([stats_bytes(t, 240, sd_e.R, E) for t in T])
    stats_ms = dev_us.get('stream_enroll_stats_kernel', float('nan')) * 1e-3
    named = [len(st.names) for st in sd_e.streams.values()]
    return dict(streams=n, enrolled=E, block_xvectors=H, context=240, pushes_timed=pushes,
                wall_ms_with=round(med(walls['with']) * 1e3, 2), wall_ms_without=round(med(walls['without']) * 1e3, 2),
                wall_ms_added=round((med(walls['with']) - med(walls['without'])) * 1e3, 2),
                enroll_step_ms=round(med([t['enroll'] for t in T]) * 1e3, 3),
                candidates_per_push=cand, streams_with_candidates=med([t['enroll_streams'] for t in T]),
                llr_pairs_per_push=int(cand * E),
                kernel_ms_profiled_push={k: round(v * 1e-3, 4) for k, v in dev_us.items()},
                stats_bytes_bound=int(sb), stats_kernel_GBps_bound=round(sb / (stats_ms * 1e-3) / 1e9, 1),
                named_speakers_mean=round(float(np.mean(named)), 2))


def sessions(x_es, seed=13, n_rec=8, pool=10):
    """The multi-session archive of the enrolment tests: pool speakers at 2 sd around ES2005a's mean x-vector, 2 .. 5
    per recording with sticky turns, reference rows naming them p<index>, and 20 held-out x-vectors of each."""
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + 2.0 * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, rows = {}, []
    for r in range(n_rec):
        T = int(rng.integers(300, 601))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        name = f'ses{r:02d}'
        recs[name] = (x, seg)
        rows += [(name, round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    return recs, rows, held


def enroll_quality(x_ref, transform, plda, kw, dev, threshold=0.0):
    recs, rows, held = sessions(x_ref)
    opts = dict(threshold=-0.015, max_iters=40, epsilon=1e-6)
    turns = lambda lines: [(l.split()[1], float(l.split()[3]), float(l.split()[4]), l.split()[7]) for l in lines]
    der = lambda sys_rows: round(100 * score.score_rttm(rows, sys_rows, 0.25, False, by_name=True)[1]['by_name']['der'], 2)
    out = dict(threshold=threshold, offline=[], streamed=[])
    for prior in (False, True):
        off = pipeline.diarize_batch(recs, transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'],
                                     init='AHC+VB', enroll=held, enroll_threshold=threshold, enroll_prior=prior, **opts)
        out['offline'].append(dict(enroll_prior=prior,
                                   der_by_name=der([r for n in recs for r in turns(off[n]['rttm_named'])])))
    for B in (5.0, 10.0):
        for prior in (False, True):
            sd = StreamDiarizer(transform, plda, kw['Fa'], kw['Fb'], kw['loopP'], smoothing=kw['smoothing'], context=240,
                                device=dev, enroll=held, enroll_threshold=threshold, enroll_prior=prior, **opts)
            first, at_first = {}, 0
            for push in block_schedule(recs, B):
                if not push:
                    continue
                got = sd.push({n: (recs[n][0][r], recs[n][1][r]) for n, r in push.items()})
                for n, res in got.items():
                    for k in np.unique(res['labels']).tolist():
                        if (n, k) not in first:
                            first[(n, k)] = True
                            at_first += k in res['named']
            named = sum(len(st.names) for st in sd.streams.values())
            out['streamed'].append(dict(block_seconds=B, enroll_prior=prior,
                                        der_by_name=der([r for n in recs for r in turns(sd.rttm(n))]),
                                        speakers=len(first), named=named, named_at_first_push=at_first,
                                        share_named_at_first_push=round(at_first / max(len(first), 1), 4)))
    return out


def enroll_main(args, x_ref, transform, plda, kw, dev):
    runs = []
    for n in (int(v) for v in args.streams.split(',')):
        for E in (int(v) for v in args.enroll_speakers.split(',')):
            runs.append(enroll_speed(n, E, args.pushes, x_ref, transform, plda, kw, dev))
            print(json.dumps(runs[-1]), file=sys.stderr)
            torch.cuda.empty_cache()
    q = enroll_quality(x_ref, transform, plda, kw, dev)
    print(json.dumps(q), file=sys.stderr)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    line = dict(gpu=smi[0] if smi else torch.cuda.get_device_name(0), speed=runs, quality=q)
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(s + '\n')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='1024,4096')
    ap.add_argument('--pushes', type=int, default=10)
    ap.add_argument('--enroll-speakers', default=None,
                    help='E1,E2,...: measure enrolled speakers in streams (DESIGN.md section 5.29) instead')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_stream.py needs a CUDA device')
    dev = torch.device('cuda:0')
    x_ref, transform, plda, kw = model()
    if args.enroll_speakers is not None:
        return enroll_main(args, x_ref, transform, plda, kw, dev)
    runs = []
    for n in (int(v) for v in args.streams.split(',')):
        runs.append(speed(n, args.pushes, x_ref, transform, plda, kw, dev))
        print(json.dumps(runs[-1]), file=sys.stderr)
        torch.cuda.empty_cache()
    q = quality(x_ref, transform, plda, kw, dev)
    print(json.dumps(q), file=sys.stderr)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    line = dict(gpu=smi[0] if smi else torch.cuda.get_device_name(0), speed=runs, quality=q)
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
