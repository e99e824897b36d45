"""Times DER scoring of a 216-setting sweep (vbx_b200/score.py, kernel vbx_score) on a seeded synthetic archive, and the
pure-Python line-sweep oracle (oracle/der_oracle.py) on a subset.  Prints one JSON line; --out also writes it there.

The archive is shaped like tools/bench_sweep.py's: 17 recordings of 2 000 .. 8 000 x-vectors (1.5 s every 0.24 s, a few
pauses), 2 .. 8 speakers, ground-truth labels whose merged segments are the reference RTTM.  Each of the 216 settings
gets its own system labelling per recording: the truth under a random relabelling with a setting-dependent share of
x-vectors reassigned, so every entry has misses, false alarms and confusion to count.  All three AMI protocols are scored.

    python tools/bench_score.py --out profiles/h100_score.json

--overlap times overlap-aware scoring (vbx_score_overlap, DESIGN.md section 5.12) against vbx_score on the same entries in
the same process, alternating the two: every entry also gets a second label per x-vector (different from the first), and
each recording seeded overlap regions covering about 15 % of its reference speech time.

    python tools/bench_score.py --overlap --out profiles/h100_score_overlap.json

--jer times label-time accumulation for the Jaccard error rate (vbx_score_jer, DESIGN.md section 5.13) on the same
archive and second labels: the kernel of each launch kind (vbx_score, vbx_score_overlap, vbx_score_jer single-label and
two-stream) on the `full` regions, alternating, and whole score_entries calls with and without jer='full', broken down
into uploads, kernels, readback, DER matchings and JER matchings.

    python tools/bench_score.py --jer --out profiles/h100_score_jer.json
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
from oracle import der_oracle  # noqa: E402
from vbx_b200 import pipeline, score, synth  # noqa: E402

N_SETTINGS = 216


def archive(seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.integers(2000, 8001, 17)
    arch = synth.make_scoring_archive(lens, seed=seed, gap_prob=0.02)
    rows = []
    for n, (seg, lab) in arch.items():
        s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
        rows += [(n, float(a), float(z - a), f'spk{k}') for a, z, k in zip(s, e, l)]
    turns = score.reference_turns(rows)
    names = list(arch)
    t0 = time.perf_counter()
    recs = [score.prepare_recording(n, turns[n], score.owned_intervals(arch[n][0])) for n in names]
    t_prep = time.perf_counter() - t0
    entries = []
    for k in range(N_SETTINGS):
        flip = 0.01 + 0.2 * k / N_SETTINGS
        for b, n in enumerate(names):
            lab = arch[n][1]
            perm = rng.permutation(int(lab.max()) + 2)
            sysl = perm[lab]
            sel = rng.random(len(lab)) < flip
            sysl[sel] = rng.integers(0, len(perm), int(sel.sum()))
            entries.append((b, sysl))
    return arch, names, rows, recs, entries, t_prep


def overlap_inputs(arch, names, recs_turns, entries, seed=1):
    """Seeded overlap regions (about OVERLAP_SHARE of each recording's speech time) and second labels for `entries`;
    its own generator, so the single-label entries are those of the plain benchmark."""
    rng = np.random.default_rng(seed)
    ovl = []
    for n in names:
        lo, hi = score.merge_turns(np.concatenate([t[0] for t in recs_turns[n]]), np.concatenate([t[1] for t in recs_turns[n]]))
        speech = int(np.sum(hi - lo))
        span = int(arch[n][0][-1, 1] * 1e6)
        k = int(np.ceil(OVERLAP_SHARE * speech / 1.75e6))
        a = rng.integers(0, span, k)
        ovl.append(score.merge_turns(a, a + rng.integers(500_000, 3_000_001, k)))
    entries2 = []
    for b, lab in entries:
        L = int(lab.max()) + 1
        entries2.append((b, lab, (lab + rng.integers(1, max(L, 2), len(lab))) % max(L, 2)))
    return ovl, entries2


OVERLAP_SHARE = 0.15


def main_overlap(args, dev):
    arch, names, rows, recs, entries, _ = archive()
    turns = score.reference_turns(rows)
    ovl, entries2 = overlap_inputs(arch, names, turns, entries)
    t0 = time.perf_counter()
    recs = [score.prepare_recording(n, turns[n], score.owned_intervals(arch[n][0]), overlap=o) for n, o in zip(names, ovl)]
    t_prep = time.perf_counter() - t0
    speech = sum(r.regions['full'][3] for r in recs)
    share = sum(int(np.sum(o[1] - o[0])) for o in ovl)
    n_int = sum(len(recs[b].sys_lo) for b, _ in entries)
    score.score_entries(recs, entries[:17], device=dev)                # warm-up of both instantiations
    score.score_entries(recs, entries2[:17], device=dev)
    times = {'vbx_score': [], 'vbx_score_overlap': []}
    for _ in range(args.reps):                                         # alternating, same entries
        for key, ent in (('vbx_score', entries), ('vbx_score_overlap', entries2)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = score.score_entries(recs, ent, device=dev)
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
            if key == 'vbx_score':
                res1 = r
            else:
                res2 = r
    from torch.profiler import ProfilerActivity, profile
    kern = {'vbx_score': [], 'vbx_score_overlap': []}
    for _ in range(args.reps):
        for key, ent in (('vbx_score', entries), ('vbx_score_overlap', entries2)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                score.score_entries(recs, ent, device=dev)
                torch.cuda.synchronize()
            kern[key] += [e.time_range.elapsed_us() / 1000.0 for e in prof.events() if 'score_kernel' in e.name]
    sub = entries2[:args.oracle_entries]
    mismatches = 0
    for i, (b, lab, lab2) in enumerate(sub):
        seg = arch[names[b]][0]
        s, e, l = pipeline.overlap_segments(seg, lab, lab2, ovl[b])
        ref = [(int(score.to_ticks(r[1])), int(score.to_ticks(r[1] + r[2])), r[3]) for r in rows if r[0] == names[b]]
        sysseg = list(zip(score.to_ticks(s).tolist(), score.to_ticks(e).tolist(), l.tolist()))
        for p, c, io in score.PROTOCOLS:
            mismatches += der_oracle.der_ticks(ref, sysseg, int(score.to_ticks(c)), io) != res2[i][p]['ticks']
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    lens = [len(a[0]) for a in arch.values()]
    stat = lambda v: dict(median=round(float(np.median(v)), 4), min=round(min(v), 4), max=round(max(v), 4), n=len(v))
    line = dict(
        bench='overlap-aware DER scoring of a hyperparameter sweep, against single-label scoring', gpu=q.stdout.strip(),
        archive=f'synthetic, seeded: {len(lens)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all',
        settings=N_SETTINGS, entries=len(entries), intervals_per_protocol=int(n_int), protocols=len(score.PROTOCOLS),
        overlap_share_of_speech=round(share / speech, 4),
        score_entries_s={k: stat(v) for k, v in times.items()},
        kernel_ms_per_protocol={k: stat(v) for k, v in kern.items()},
        host_region_prep_s=round(t_prep, 4),
        oracle_entries=len(sub), oracle_mismatches=int(mismatches),
        overall_der={k: {p: score.overall([x[p] for x in r])['der'] for p, _, _ in score.PROTOCOLS}
                     for k, r in (('vbx_score', res1), ('vbx_score_overlap', res2))})
    return line


def timed(fn, acc):
    def wrapper(*a, **k):
        t0 = time.perf_counter()
        try:
            return fn(*a, **k)
        finally:
            acc.append(time.perf_counter() - t0)
    return wrapper


def main_jer(args, dev):
    from torch.profiler import ProfilerActivity, profile
    arch, names, rows, recs, entries, _ = archive()
    turns = score.reference_turns(rows)
    ovl, entries2 = overlap_inputs(arch, names, turns, entries)
    full = (('full', 0.0, False),)
    one = [score.prepare_recording(n, turns[n], score.owned_intervals(arch[n][0]), protocols=full, overlap=o)
           for n, o in zip(names, ovl)]
    calls = {'vbx_score': lambda: score.score_entries(one, entries, device=dev),
             'vbx_score_overlap': lambda: score.score_entries(one, entries2, device=dev),
             'vbx_score_jer': lambda: score.score_entries(one, entries, device=dev, jer='full'),
             'vbx_score_jer (two-stream)': lambda: score.score_entries(one, entries2, device=dev, jer='full')}
    for f in calls.values():                                           # warm-up of every instantiation
        f()
    kern, kname = {k: [] for k in calls}, {}
    for _ in range(args.launches):                                     # alternating, one launch per call
        for key, f in calls.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                f()
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if 'score_kernel' in e.name]
            kern[key] += [e.time_range.elapsed_us() / 1000.0 for e in ev]
            kname[key] = sorted({'score_kernel' + e.name.split('score_kernel')[1].split('(')[0] for e in ev})
    # whole score_entries calls over the three protocols, with and without jer, alternating
    recs = [score.prepare_recording(n, turns[n], score.owned_intervals(arch[n][0])) for n in names]
    whole = {'without jer': [], 'with jer': []}
    res = {}
    for _ in range(args.reps):
        for key, jer in (('without jer', None), ('with jer', 'full')):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[key] = score.score_entries(recs, entries, device=dev, jer=jer)
            torch.cuda.synchronize()
            whole[key].append(time.perf_counter() - t0)
    # breakdown of one call each: host time in the matchings (wrapped), device time of kernels and copies (profiler)
    parts = {}
    real = (score.finish, score.jer_finish, score.reference_time)
    for key, jer in (('without jer', None), ('with jer', 'full')):
        der_t, jer_t = [], []
        score.finish, score.jer_finish, score.reference_time = (timed(real[0], der_t), timed(real[1], jer_t),
                                                                timed(real[2], jer_t))
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                score.score_entries(recs, entries, device=dev, jer=jer)
                torch.cuda.synchronize()
                total = time.perf_counter() - t0
        finally:
            score.finish, score.jer_finish, score.reference_time = real
        ev = list(prof.events())
        dev_ms = lambda pat: round(sum(e.time_range.elapsed_us() for e in ev if pat in e.name) / 1000.0, 3)
        parts[key] = dict(total_s_profiled=round(total, 4), kernels_ms=dev_ms('score_kernel'),
                          uploads_ms_device=dev_ms('HtoD'), readback_ms_device=dev_ms('DtoH'),
                          der_matchings_s=round(sum(der_t), 4), der_matchings=len(der_t),
                          jer_matchings_s=round(sum(jer_t), 4),
                          rest_s=round(total - sum(der_t) - sum(jer_t), 4))
    same_der = all({p: r[p] for p, _, _ in score.PROTOCOLS} == q for r, q in zip(res['with jer'], res['without jer']))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    lens = [len(a[0]) for a in arch.values()]
    stat = lambda v: dict(median=round(float(np.median(v)), 4), min=round(min(v), 4), max=round(max(v), 4), n=len(v))
    return dict(
        bench='JER label-time scoring of a hyperparameter sweep, against the DER launches', gpu=q.stdout.strip(),
        archive=f'synthetic, seeded: {len(lens)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all',
        settings=N_SETTINGS, entries=len(entries), intervals_per_launch=int(sum(len(recs[b].sys_lo) for b, _ in entries)),
        kernel_ms_full_regions={k: stat(v) for k, v in kern.items()}, kernel_names=kname,
        score_entries_s={k: stat(v) for k, v in whole.items()},
        breakdown=parts, der_unchanged_with_jer=bool(same_der),
        overall_jer=score.overall_jer([r['jer'] for r in res['with jer']])['jer'],
        overall_der={p: score.overall([r[p] for r in res['with jer']])['der'] for p, _, _ in score.PROTOCOLS})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', default=5, type=int)
    ap.add_argument('--oracle-entries', default=17, type=int)
    ap.add_argument('--overlap', action='store_true', help='time vbx_score_overlap against vbx_score')
    ap.add_argument('--jer', action='store_true', help='time vbx_score_jer against vbx_score and vbx_score_overlap')
    ap.add_argument('--launches', default=15, type=int, help='--jer: profiled launches of each kind')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_score.py needs a CUDA device')
    dev = torch.device('cuda:0')
    if args.overlap or args.jer:
        s = json.dumps(main_jer(args, dev) if args.jer else main_overlap(args, dev))
        print(s)
        if args.out:
            with open(args.out, 'w') as fp:
                fp.write(s + '\n')
        return
    arch, names, rows, recs, entries, t_prep = archive()
    n_int = sum(len(recs[b].sys_lo) for b, _ in entries)
    score.score_entries(recs, entries[:17], device=dev)                # warm-up: module load, allocator
    times = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = score.score_entries(recs, entries, device=dev)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    # kernel time per protocol launch, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        score.score_entries(recs, entries, device=dev)
        torch.cuda.synchronize()
    kern = [e.time_range.elapsed_us() for e in prof.events() if "score_kernel" in e.name]
    # the oracle on a subset: the first setting over all recordings
    sub = entries[:args.oracle_entries]
    t0 = time.perf_counter()
    mismatches = 0
    for i, (b, lab) in enumerate(sub):
        seg = arch[names[b]][0]
        s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
        ref = [(int(score.to_ticks(r[1])), int(score.to_ticks(r[1] + r[2])), r[3]) for r in rows if r[0] == names[b]]
        sysseg = list(zip(score.to_ticks(s).tolist(), score.to_ticks(e).tolist(), l.tolist()))
        for p, c, io in score.PROTOCOLS:
            mismatches += der_oracle.der_ticks(ref, sysseg, int(score.to_ticks(c)), io) != res[i][p]['ticks']
    t_oracle = time.perf_counter() - t0
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    lens = [len(a[0]) for a in arch.values()]
    ders = {p: score.overall([r[p] for r in res])['der'] for p, _, _ in score.PROTOCOLS}
    line = dict(
        bench='DER scoring of a hyperparameter sweep', gpu=q.stdout.strip(),
        archive=f'synthetic, seeded: {len(lens)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all',
        settings=N_SETTINGS, entries=len(entries), intervals_per_protocol=int(n_int), protocols=len(score.PROTOCOLS),
        score_entries_s=dict(median=round(float(np.median(times)), 4), min=round(min(times), 4), max=round(max(times), 4),
                             reps=len(times)),
        kernel_ms_per_protocol=[round(k / 1000.0, 3) for k in kern],
        host_region_prep_s=round(t_prep, 4),
        oracle_s=round(t_oracle, 3), oracle_entries=len(sub), oracle_mismatches=int(mismatches),
        overall_der=ders)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
