"""Times speaker linking across recordings (DESIGN.md section 5.15).

1. link_speakers (vbx_link_batch) on synthetic archives of M = 1 000, 4 000 and 16 000 speakers (4 per recording,
   1 .. 15 x-vectors each, R = 128): device time of every kernel from torch.profiler (one warm-up call first), next to
   the bytes and operations the statistics and score kernels need, computed from the shapes.  The linkage is one CTA
   doing M - 1 dependent merges.
2. Whole diarize_batch calls on the synthetic archive of tools/bench_sweep.py (17 recordings) without and with
   link_threshold, alternating in one process (medians, minima, maxima), and the time of each linking step inside
   linked calls (link_speakers, link_cut, linked_lines).
The card's name and power limit are read in the same run.  Prints one JSON line; --out also writes it there.

    python tools/bench_link.py --out profiles/h100_link.json

--replay 1000,4000 needs no GPU: it replays the linkage kernel's nearest-neighbour bookkeeping (ahc_linkage_kernel in
vbx_ahc.cu: the pair of lowest nearest-neighbour distance merges, the Lance-Williams update of its row, and a full
re-scan of every row whose nearest neighbour was merged away) in numpy on the float64 distances of the same synthetic
speakers (oracle/link_oracle.py) and counts the re-scanned rows per merge.
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
from bench_sweep import GOLD, synthetic_archive  # noqa: E402
from vbx_b200 import link, pipeline  # noqa: E402

KERNELS = ('link_init_kernel', 'link_span_kernel', 'link_stats_kernel', 'link_score_kernel', 'ahc_linkage_kernel')


def speakers(M, R=128, seed=0, device='cuda'):
    """fea [N,R] float32 on `device`, Phi [R], offsets and labels of M speakers, 4 per recording."""
    rng = np.random.default_rng(seed)
    per = rng.integers(1, 16, M)
    labels, lens = [], []
    for b in range(0, M, 4):
        lab = np.repeat(np.arange(len(per[b:b + 4])), per[b:b + 4])
        rng.shuffle(lab)
        labels.append(lab)
        lens.append(len(lab))
    N = int(sum(lens))
    fea = torch.randn((N, R), generator=torch.Generator().manual_seed(seed)).to(device)
    Phi = torch.from_numpy(np.sort(rng.uniform(0.2, 6.0, R))[::-1].astype(np.float32).copy()).to(device)
    return fea, Phi, np.concatenate([[0], np.cumsum(lens)]), labels


def replay(M):
    """Rows re-scanned by the linkage kernel's bookkeeping over the float64 distances of speakers(M)."""
    from oracle import link_oracle
    fea, Phi, offs, labels = speakers(M, device='cpu')
    table = link.speaker_table(labels)
    spk = np.concatenate([l + np.searchsorted(table.rec, b) for b, l in enumerate(labels)])
    n, F = link_oracle.statistics(fea.double().numpy(), spk, M)
    D = link_oracle.distances(n, F, Phi.double().numpy(), 0.3 / 17, table.rec)
    alive = np.ones(M, dtype=bool)
    size = np.ones(M)
    idx = np.arange(M)

    def nearest(rows):
        sub = D[rows].copy()
        sub[:, ~alive] = np.inf
        sub[np.arange(len(rows)), rows] = np.inf
        k = np.argmin(sub, axis=1)                      # ties: the lowest slot, as the kernel's warp reduction
        return k, sub[np.arange(len(rows)), k]

    nn, nnd = nearest(idx)
    todo_per_merge = []
    for step in range(M - 1):
        live = idx[alive]
        p = live[np.argmin(nnd[live])]
        a, b = min(p, nn[p]), max(p, nn[p])
        wa, wb = size[a] / (size[a] + size[b]), size[b] / (size[a] + size[b])
        ks = live[(live != a) & (live != b)]
        dn = wa * D[a, ks] + wb * D[b, ks]
        D[a, ks] = dn
        D[ks, a] = dn
        lost = (nn[ks] == a) | (nn[ks] == b)
        closer = ~lost & (dn < nnd[ks])
        nn[ks[closer]], nnd[ks[closer]] = a, dn[closer]
        alive[b] = False
        size[a] += size[b]
        todo = np.concatenate([ks[lost], [a]])
        todo_per_merge.append(len(todo) - 1)
        if step < M - 2:
            nn[todo], nnd[todo] = nearest(todo)
    t = np.array(todo_per_merge)
    return dict(merges=M - 1, rescanned_rows=int(t.sum()) + M - 2, mean_per_merge=round(float(t.mean()) + 1, 1),
                max_per_merge=int(t.max()) + 1, slots_scanned=int(((t + 1) * (M - np.arange(M - 1))).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--sizes', default='1000,4000,16000')
    ap.add_argument('--replay', default=None, help='comma-separated M: count the linkage\'s re-scanned rows on the host')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if args.replay:
        s = json.dumps(dict(bench='linkage bookkeeping replayed on the host (float64 oracle distances)',
                            speakers={m: replay(int(m)) for m in args.replay.split(',')}))
        print(s)
        if args.out:
            with open(args.out, 'w') as fp:
                fp.write(s + '\n')
        return
    if not torch.cuda.is_available():
        raise SystemExit('bench_link.py needs a CUDA device')
    from torch.profiler import ProfilerActivity, profile
    R = 128
    sizes = {}
    fea, Phi, offs, labels = speakers(1000)
    link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0)               # warm-up: module load
    for M in (int(m) for m in args.sizes.split(',')):
        fea, Phi, offs, labels = speakers(M)
        N = int(fea.shape[0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0)
        wall = time.perf_counter() - t0
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0)
        kern = {}
        for e in prof.key_averages():
            for k in KERNELS:
                if k in e.key:
                    kern[k] = round(getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0)), 1)
        pairs = M * (M + 1) // 2
        spans = sum(int(offs[b + 1] - offs[b]) * min(4, M - 4 * b) for b in range(len(labels)))
        sizes[str(M)] = dict(
            N=N, R=R, whole_call_s=round(wall, 4), kernels_us=kern,
            stats=dict(bytes=N * R * 4 + spans * 4, flops=N * R,
                       note='features read once per speaker (a recording\'s speakers share its span in L2), speaker '
                            'index read once per speaker per x-vector of its span'),
            score=dict(pairs=pairs, bytes_written=8 * M * M, fp64_div=pairs * R, fp64_log=pairs * (R // 8),
                       fp64_other=pairs * R * 5, note='upper triangle computed, both halves written'),
            linkage=dict(merges=M - 1, matrix_bytes=8 * M * M,
                         note='one 1024-thread CTA; every merge scans the M nearest-neighbour distances and updates '
                              'one row and column of the matrix'))
        del fea
        torch.cuda.empty_cache()

    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs = synthetic_archive(z['x_raw'])
    kw = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=40, epsilon=1e-6,
              device=torch.device('cuda:0'))
    modes = {'without': {}, 'link_threshold=0': dict(link_threshold=0.0)}

    def call(mode):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipeline.diarize_batch(recs, transform, plda, **kw, **modes[mode])
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    for mode in modes:
        out, _ = call(mode)
    n_global = len({g for it in out.values() for g in it['global_speakers'].values()})
    n_local = sum(len(it['global_speakers']) for it in out.values())
    times = {mode: [] for mode in modes}
    for _ in range(args.rounds):
        for mode in modes:
            times[mode].append(call(mode)[1])
    # where a linked call spends its extra time: each linking step timed inside the calls (host clock around work that
    # ends in a readback, so device work is included)
    steps = {'link_speakers': [], 'link_cut': [], 'linked_lines': []}

    def timed(fn, key):
        def run(*a, **k):
            t0 = time.perf_counter()
            r = fn(*a, **k)
            steps[key][-1] += time.perf_counter() - t0
            return r
        return run
    real = link.link_speakers, link.link_cut, pipeline.linked_lines
    link.link_speakers, link.link_cut = timed(real[0], 'link_speakers'), timed(real[1], 'link_cut')
    pipeline.linked_lines = timed(real[2], 'linked_lines')
    for _ in range(args.rounds):
        for v in steps.values():
            v.append(0.0)
        call('link_threshold=0')
    link.link_speakers, link.link_cut, pipeline.linked_lines = real
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    lens = [r[0].shape[0] for r in recs.values()]
    line = dict(
        bench='speaker linking across recordings', gpu=q.stdout.strip(), synthetic_speakers=sizes,
        archive=f'synthetic, seeded: {len(recs)} recordings, {min(lens)} .. {max(lens)} x-vectors, {sum(lens)} in all; '
                f'{n_local} speakers linked into {n_global}',
        rounds=args.rounds, median_s={k: round(float(np.median(t)), 4) for k, t in times.items()},
        min_s={k: round(float(np.min(t)), 4) for k, t in times.items()},
        max_s={k: round(float(np.max(t)), 4) for k, t in times.items()},
        linking_steps_median_ms={k: round(1e3 * float(np.median(v)), 2) for k, v in steps.items()})
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, 'w') as fp:
            fp.write(s + '\n')


if __name__ == '__main__':
    main()
