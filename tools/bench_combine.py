"""Times the combination of diarizations (vbx_b200/combine.py, vbx_combine, DESIGN.md section 5.21) and reports the DER of
the combination beside the DER of each input.  Prints one JSON line; --out also writes it there.  Needs a GPU.

Sizes: the seeded synthetic archive of tools/bench_score.py (17 recordings of 2 000 .. 8 000 x-vectors, about 85 k in
all, the x-vectors' owned intervals) with K = 2, 8 and 32 hypotheses, as a sweep's settings give them, and 4 096
recordings of 1 000 intervals with K = 8.  A hypothesis is the truth under a random relabelling with a share of its
x-vectors (1 % .. 21 %, growing with k) reassigned, as bench_score.py makes a setting's labels.

Per size: whole combine_labels calls (host clock around a call that ends with its results on the host, so uploads,
the three kernels and the readback), and the device time of each kernel from torch.profiler in runs of their own; all
after a warm-up call of the same shape.  The DER of every input and of the combination is score.score_entries' under
the three AMI protocols against the archive's truth.
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
from vbx_b200 import combine, pipeline, score, synth  # noqa: E402

KERNELS = ('combine_overlap_kernel', 'combine_map_kernel', 'combine_vote_kernel')


def hypotheses(truth, K, rng):
    hyps = []
    for k in range(K):
        flip = 0.01 + 0.2 * k / K
        per = []
        for lab in truth:
            perm = rng.permutation(int(lab.max()) + 2)
            sysl = perm[lab]
            sel = rng.random(len(lab)) < flip
            sysl[sel] = rng.integers(0, len(perm), int(sel.sum()))
            per.append((sysl, None))
        hyps.append(per)
    return hyps


def stat(v):
    return dict(median=round(float(np.median(v)), 4), min=round(float(min(v)), 4), max=round(float(max(v)), 4), n=len(v))


def measure(intervals, hyps, dev, reps):
    from torch.profiler import ProfilerActivity, profile
    combine.combine_labels(intervals, hyps, device=dev)                # warm-up: module load, allocator
    whole = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = combine.combine_labels(intervals, hyps, device=dev)
        torch.cuda.synchronize()
        whole.append((time.perf_counter() - t0) * 1e3)
    kern = {k: [] for k in KERNELS}
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            combine.combine_labels(intervals, hyps, device=dev)
            torch.cuda.synchronize()
        for e in prof.events():
            for k in KERNELS:
                if k in e.name:
                    kern[k].append(e.time_range.elapsed_us() / 1000.0)
    n = int(sum(len(iv[0]) for iv in intervals))
    return res, dict(recordings=len(intervals), intervals=n, K=len(hyps), label_bytes=8 * len(hyps) * n,
                     combine_labels_ms=stat(whole), kernel_ms={k: stat(v) for k, v in kern.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', default=5, type=int)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_combine.py needs a CUDA device')
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(0)
    lens = rng.integers(2000, 8001, 17)
    arch = synth.make_scoring_archive(lens, seed=0, gap_prob=0.02)
    names = list(arch)
    rows = []
    for n, (seg, lab) in arch.items():
        s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
        rows += [(n, float(a), float(z - a), f'spk{k}') for a, z, k in zip(s, e, l)]
    turns = score.reference_turns(rows)
    recs = [score.prepare_recording(n, turns[n], score.owned_intervals(arch[n][0])) for n in names]
    intervals = [(r.sys_lo, r.sys_hi) for r in recs]
    sizes, der = [], {}
    for K in (2, 8, 32):
        hyps = hypotheses([arch[n][1] for n in names], K, rng)
        res, m = measure(intervals, hyps, dev, args.reps)
        entries = [(b, hyps[k][b][0]) for k in range(K) for b in range(len(names))]
        entries += [(b, res[b]['labels']) for b in range(len(names))]
        sc = score.score_entries(recs, entries, device=dev)
        overall = lambda part: {p: score.overall([x[p] for x in part])['der'] for p, _, _ in score.PROTOCOLS}
        inputs = [overall(sc[k * len(names):(k + 1) * len(names)]) for k in range(K)]
        der[f'K={K}'] = dict(inputs=inputs, best_input={p: min(i[p] for i in inputs) for p, _, _ in score.PROTOCOLS},
                             combined=overall(sc[K * len(names):]),
                             anchors=sorted({r['order'][0] for r in res}))
        sizes.append(dict(m, archive='synthetic, seeded: 17 recordings'))
    T, B, K = 1000, 4096, 8
    truth = [np.repeat(rng.integers(0, 4, T // 10), 10) for _ in range(B)]
    lo = np.arange(T, dtype=np.int64) * 240_000
    _, m = measure([(lo, lo + 240_000)] * B, hypotheses(truth, K, rng), dev, args.reps)
    sizes.append(dict(m, archive='synthetic, seeded: 4 096 recordings of 1 000 intervals'))
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    line = dict(bench='combination of diarizations: label mapping and weighted voting', gpu=q.stdout.strip(), sizes=sizes,
                der=der, note='kernel_ms: device time per launch (torch.profiler); combine_labels_ms: host clock around '
                              'the whole call, uploads and readback included')
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
