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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--streams', default='1024,4096')
    ap.add_argument('--pushes', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_stream.py needs a CUDA device')
    dev = torch.device('cuda:0')
    x_ref, transform, plda, kw = model()
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
