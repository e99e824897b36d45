"""Times VB resegmentation, init='RTTM+VB' (DESIGN.md section 5.20), and measures what it does to DER.

(a) vbx_init_turns alone at B = 4 096 recordings x T = 1 000 x-vectors (1.5 s segments every 0.24 s) with K = 16
    speakers (S = 16) and K = 128 (S = 128), float32 output, each recording's 240 s cut into 200 turns of random
    speakers.  kernel_ms: the mean device time of init_turns_kernel from the kernel events of a torch.profiler capture
    of `launches` calls; call_ms: CUDA events around each whole call (the entry reads spk_off and turn_off back before
    it launches), median.  bytes: the gamma and pi writes plus the segment reads; model_ms: bytes at the data sheet's
    3.35 TB/s.
(b) diarize_batch on the 17-recording synthetic multi-session archive of tools/bench_enroll_sweep.py with init='AHC+VB'
    and with init='RTTM+VB' from the archive's reference, alternating, medians of 5 (host clock around calls that end
    in a readback).
(c) Usefulness: synth.multi_session_archive with its defaults (seed 13) and its reference rows; DER (full protocol) of
    the input RTTM, of init='RTTM+VB' from it and of init='AHC+VB', for an input with 30 % of the reference turns given
    another speaker of the recording, and for an input with only the first 20 % of each recording's reference turns.
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it there.

    python tools/bench_init.py --out profiles/h100_init_rttm.json
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
from vbx_b200 import pipeline, resegment, score, synth  # noqa: E402
from vbx_b200.batch import VbxBatch, _ptr  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden')
KW = dict(Fa=0.3, Fb=17.0, loopP=0.99, smoothing=5.0, threshold=-0.015, max_iters=40, epsilon=1e-6)


def synthetic_pack(B, T, K, seed=0):
    """B recordings of T x-vectors, 240 s each cut into 200 turns of random speakers of K, packed with numpy (every
    speaker's turns sorted; turns of one speaker may touch)."""
    rng = np.random.default_rng(seed)
    n_turns = 200
    step = 240_000_000 // n_turns
    spk = rng.integers(0, K, (B, n_turns))
    rec = np.repeat(np.arange(B), n_turns)
    lo = np.tile(np.arange(n_turns, dtype=np.int64) * step, B)
    order = np.lexsort((lo, spk.reshape(-1), rec))            # by recording, speaker, time
    lo = lo[order]
    hi = lo + step
    key = rec[order] * K + spk.reshape(-1)[order]
    counts = np.bincount(key, minlength=B * K)
    turn_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    c = np.concatenate([[0], np.cumsum(hi - lo)])
    turn_cum = (c[:-1] - np.repeat(c[turn_off[:-1]], counts)).astype(np.int64)
    t0 = np.arange(T, dtype=np.int64) * 240_000
    seg = np.tile(np.stack([t0, t0 + 1_500_000], 1), (B, 1))
    return resegment.TurnPack(seg=seg, spk_off=np.arange(B + 1, dtype=np.int64) * K, turn_off=turn_off, turn_lo=lo,
                              turn_hi=hi, turn_cum=turn_cum)


def kernel_case(B, T, K, launches):
    """(a) for one shape."""
    pack = synthetic_pack(B, T, K)
    n_turns = int(pack.turn_off[-1]) // B
    dev = torch.device('cuda:0')
    vb = VbxBatch([T] * B, 128, K, device=dev, allocate=False)
    g = torch.empty((vb.N, vb.S), device=dev)
    p = torch.empty((B, vb.S), device=dev)
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in pack] + [torch.full((B,), 5.0, dtype=torch.float64,
                                                                                         device=dev)]
    stream = vb._stream()
    call = lambda: vb._check(vb.lib.vbx_init_turns(vb._h, *(_ptr(a) for a in d), _ptr(g), _ptr(p), 0, stream))
    for _ in range(3):
        call()
    ms = []
    for _ in range(launches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(launches):
            call()
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events()
          if e.device_type == torch.autograd.DeviceType.CUDA and 'init_turns_kernel' in e.name]
    assert bool(torch.allclose(g.view(B, T, vb.S).sum(2), torch.ones((B, T), device=dev)))
    nbytes = 4 * vb.N * vb.S + 4 * B * vb.S + 16 * vb.N
    kms = float(np.mean(us)) / 1e3 if us else None
    vb.close()
    del g, d
    torch.cuda.empty_cache()
    return dict(B=B, T=T, K=K, S=K, turns_per_recording=n_turns, launches=launches,
                kernel_ms=round(kms, 4) if kms else None, kernel_events=len(us),
                call_median_ms=round(float(np.median(ms)), 4), bytes=int(nbytes),
                model_ms_at_3_35_TBps=round(nbytes / 3.35e12 * 1e3, 4),
                achieved_TBps=round(nbytes / (kms * 1e-3) / 1e12, 3) if kms else None)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def turns_of(rows):
    """Reference rows (one per x-vector) -> turns: runs of one speaker merged, per recording in time order."""
    out = []
    for rec in dict.fromkeys(r[0] for r in rows):
        cur = None
        for r in (r for r in rows if r[0] == rec):
            if cur is not None and cur[3] == r[3] and abs(cur[1] + cur[2] - r[1]) < 1e-6:
                cur = (rec, cur[1], round(r[1] + r[2] - cur[1], 6), cur[3])
                continue
            if cur is not None:
                out.append(cur)
            cur = r
        out.append(cur)
    return out


def sys_rows(lines):
    return [(l.split()[1], float(l.split()[3]), float(l.split()[4]), l.split()[7]) for l in lines]


def full_der(ref, rows):
    return round(float(score.score_rttm(ref, rows, 0.0, False)[1]['der']), 4)


def usefulness(transform, plda, z):
    recs, ref, _ = synth.multi_session_archive(z['x_raw'])
    turns = turns_of(ref)
    rng = np.random.default_rng(5)
    spk = {rec: sorted({t[3] for t in turns if t[0] == rec}) for rec in recs}
    wrong = []
    for t in turns:
        if rng.random() < 0.3:
            t = t[:3] + (str(rng.choice([k for k in spk[t[0]] if k != t[3]])),)
        wrong.append(t)
    partial = []
    for rec in recs:
        mine = [t for t in turns if t[0] == rec]
        partial += mine[:max(1, int(round(0.2 * len(mine))))]
    ahc = pipeline.diarize_batch(recs, transform, plda, init='AHC+VB', **KW)
    ahc_der = full_der(ref, [r for it in ahc.values() for r in sys_rows(it['rttm'])])
    out = dict(archive=f'synth.multi_session_archive defaults (seed 13): {len(recs)} recordings, {len(turns)} reference '
                       f'turns', params=KW, ahc_vb_der=ahc_der)
    for name, rows in (('wrong_speaker_30pct', wrong), ('first_20pct_of_turns', partial)):
        res = pipeline.diarize_batch(recs, transform, plda, init='RTTM+VB', init_rttm=rows, **KW)
        out[name] = dict(turns=len(rows), input_der=full_der(ref, rows),
                         rttm_vb_der=full_der(ref, [r for it in res.values() for r in sys_rows(it['rttm_init'])]),
                         speakers_in=sum(len(set(r[3] for r in rows if r[0] == n)) for n in recs),
                         speakers_out=sum(it['n_speakers'] for it in res.values()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_init.py needs a CUDA device')
    kernel = [kernel_case(4096, 1000, K, args.launches) for K in (16, 128)]
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs, ref, _ = synth.multi_session_archive(z['x_raw'], n_rec=17, pool=40, lengths=(2000, 8000), speakers=(3, 5),
                                               seed=0)
    modes = {'AHC+VB': dict(init='AHC+VB'), 'RTTM+VB': dict(init='RTTM+VB', init_rttm=ref)}
    for mode in modes:                                                                  # warm-up
        pipeline.diarize_batch(recs, transform, plda, **KW, **modes[mode])
    times = {mode: [] for mode in modes}
    for _ in range(args.rounds):
        for mode in modes:
            times[mode].append(timed(lambda: pipeline.diarize_batch(recs, transform, plda, **KW, **modes[mode]))[1])
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='VB resegmentation: vbx_init_turns and diarize_batch(init=RTTM+VB)', gpu=q.stdout.strip(), kernel=kernel,
        archive=f'synthetic multi-session, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, '
                f'{sum(lens)} in all; RTTM+VB from its reference',
        rounds=args.rounds, diarize_median_s={k: round(float(np.median(t)), 3) for k, t in times.items()},
        diarize_min_s={k: round(float(np.min(t)), 3) for k, t in times.items()},
        diarize_max_s={k: round(float(np.max(t)), 3) for k, t in times.items()},
        usefulness=usefulness(transform, plda, z))
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
