"""Times and scores PLDA adaptation to the archive (DESIGN.md section 5.26).

Speed:
1. The archive statistics at the headline size, 4 096 recordings x 1 000 x-vectors: vbx_class_scatter on the first-pass
   rows z [4 096 000, 128] float32 as one class, kernel time from CUDA events over --reps launches; the front end's
   first pass (adapt.project_archive, Dx = 256) that produces z, from a host clock around a synchronised call.
2. Whole adapt.adapt_backend calls on that archive (Dx = 256, chain tcgen05), host clock, medians of --rounds, with the
   seconds of each stage.
3. diarize_batch on the 17-recording synthetic archive of tools/bench_sweep.py with the shipped model, and the same
   with adapt_backend first (what `cli --adapt` runs), alternating, medians of --rounds.

Accuracy, on a synthetic domain shift: synth.multi_session_archive around ES2005a's x-vectors (12 recordings, pool of
40 speakers, seed 2024), every x-vector then moved by one seeded offset (1.0 x ES2005a's per-dimension spread times
N(0, 1) per dimension, seed 7) and given extra noise along 8 seeded orthonormal directions of the raw space (N(0, 1) x
3 x the mean per-dimension spread along each).  DER (collar 0.25, overlaps scored) through diarize_batch at ES2005a's
settings (threshold -0.015, Fa 0.3, Fb 17, loopP 0.99) for the shipped model, --adapt, --adapt --recentre, and the
PLDA interpolated at alpha in {0.25, 0.5, 0.75} between the shipped one and a PLDA trained (train_backend with the
shipped transform) on a labelled slice of the same shifted domain: 60 other recordings (seed 2025, pool of 300 other
speakers, 145 of them present; a PLDA in the d = 128 space needs more than 128 speakers to have a non-singular
between-speaker covariance, which the diarization's diagonalisation needs).  The distortion is as written above and
was not tuned.

The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; --out also writes it.

    python tools/bench_adapt.py --out profiles/h100_adapt.json
"""
import argparse
import ctypes
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
from vbx_b200 import _lib, adapt, pipeline, score, synth, train  # noqa: E402

HYPER = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=40, epsilon=1e-6)


def shipped():
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])


def sync_clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def stats_kernel(z, reps, dev):
    """CUDA-event time of one vbx_class_scatter launch on z as one class."""
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(dev.index, ctypes.byref(h)) == 0
    N, D = int(z.shape[0]), int(z.shape[1])
    off = np.array([0, N], dtype=np.int64)
    need = ctypes.c_size_t()
    assert lib.vbx_class_scatter_workspace_bytes(h, N, D, 1, ctypes.byref(need)) == 0
    ws = torch.empty(max(need.value, 1), dtype=torch.uint8, device=dev)
    means = torch.empty((1, D), dtype=torch.float64, device=dev)
    S = torch.empty((D, D), dtype=torch.float64, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def launch():
        assert lib.vbx_class_scatter(h, p(z), N, D, 1, off.ctypes.data_as(ctypes.c_void_p), p(ws), ws.numel(),
                                     p(means), p(S), st) == 0
    launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    b.synchronize()
    lib.vbx_destroy(h)
    ms = a.elapsed_time(b) / reps
    flops, nbytes = N * D * (D + 1), N * D * 4
    return dict(N=N, D=D, ms=ms, tflops=flops / ms * 1e-9, tbytes_per_s=nbytes / ms * 1e-9,
                share_fp64_tc=flops / 67e12 / (ms * 1e-3), share_hbm=nbytes / 3.35e12 / (ms * 1e-3))


def speed(rounds, reps, dev):
    transform, plda = shipped()
    x_es = np.load(os.path.join(GOLD, 'es2005a.npz'))['x_raw']
    rng = np.random.default_rng(0)
    B, T = 4096, 1000
    lens = np.full(B, T, dtype=np.int64)
    x = (x_es.mean(0) + x_es.std(0) * rng.standard_normal((B * T, x_es.shape[1]), dtype=np.float32)).astype(np.float64)
    z, t_proj = sync_clock(lambda: adapt.project_archive(x, lens, transform, plda, 128, 'auto', dev))
    z, t_proj = sync_clock(lambda: adapt.project_archive(x, lens, transform, plda, 128, 'auto', dev))
    out = dict(stats_kernel=stats_kernel(z, reps, dev), first_pass_seconds=t_proj)
    del z
    recs = {f'r{b:04d}': (x[b * T:(b + 1) * T], None) for b in range(B)}
    runs = []
    for r in range(rounds + 1):
        (_, _, rep), t = sync_clock(lambda: adapt.adapt_backend(recs, transform, plda, device=dev))
        if r:
            runs.append(dict(seconds=t, stages=rep['seconds']))
    out['adapt_backend'] = dict(B=B, T=T, Dx=int(x.shape[1]), chain=rep['chain'],
                                median_seconds=float(np.median([r['seconds'] for r in runs])), runs=runs)
    del recs, x
    arch = synthetic_archive(x_es)
    n = sum(len(v[0]) for v in arch.values())
    plain, adapted = [], []

    def with_adapt():
        t2, p2, _ = adapt.adapt_backend(arch, transform, plda, device=dev)
        return pipeline.diarize_batch(arch, t2, p2, device=dev, **HYPER)
    sync_clock(lambda: pipeline.diarize_batch(arch, transform, plda, device=dev, **HYPER))
    sync_clock(with_adapt)
    for _ in range(rounds):
        plain.append(sync_clock(lambda: pipeline.diarize_batch(arch, transform, plda, device=dev, **HYPER))[1])
        adapted.append(sync_clock(with_adapt)[1])
    out['diarize_batch'] = dict(recordings=len(arch), xvectors=n, shipped_seconds=plain, adapt_seconds=adapted,
                                shipped_median=float(np.median(plain)), adapt_median=float(np.median(adapted)))
    return out


def shift(recs, x_es, seed=7, dirs=8):
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    off = 1.0 * sd * rng.standard_normal(x_es.shape[1])
    Q, _ = np.linalg.qr(rng.standard_normal((x_es.shape[1], dirs)))
    out = {}
    for i, (name, (x, seg)) in enumerate(recs.items()):
        g = np.random.default_rng([seed, i]).standard_normal((len(x), dirs)) * 3.0 * sd.mean()
        out[name] = (x + off[None, :] + g @ Q.T, seg)
    return out


def der(recs, rows, transform, plda, dev):
    out = pipeline.diarize_batch(recs, transform, plda, device=dev, **HYPER)
    sys_rows = [r for item in out.values() for r in
                ((l.split()[1], float(l.split()[3]), float(l.split()[4]), l.split()[7]) for l in item['rttm'])]
    _, tot = score.score_rttm([(r[0], r[1], r[2], r[3]) for r in rows], sys_rows, 0.25, False, device=dev)
    return float(tot['der'])


def accuracy(dev):
    transform, plda = shipped()
    x_es = np.load(os.path.join(GOLD, 'es2005a.npz'))['x_raw']
    recs, rows, _ = synth.multi_session_archive(x_es, n_rec=12, pool=40, seed=2024)
    recs = shift(recs, x_es)
    res = dict(archive=dict(recordings=len(recs), xvectors=sum(len(v[0]) for v in recs.values())))
    res['shipped'] = der(recs, rows, transform, plda, dev)
    t2, p2, rep = adapt.adapt_backend(recs, transform, plda, device=dev)
    res['adapt'] = der(recs, rows, t2, p2, dev)
    res['adapt_report'] = dict(delta_norm=rep['delta_norm'], inflated=rep['inflated'],
                               largest_eigenvalues=rep['eigenvalues'][:5])
    t3, p3, rep3 = adapt.adapt_backend(recs, transform, plda, device=dev, recentre=True)
    res['adapt_recentre'] = der(recs, rows, t3, p3, dev)
    res['adapt_recentre_report'] = dict(delta_norm=rep3['delta_norm'], inflated=rep3['inflated'])
    lab, _, truth = synth.multi_session_archive(x_es, n_rec=60, pool=300, seed=2025)
    lab = shift(lab, x_es)
    classes = {}
    for name, (x, _) in lab.items():
        for t, k in enumerate(truth[name]):
            classes.setdefault(f'p{k}', []).append(x[t])
    classes = {k: np.stack(v) for k, v in classes.items()}
    _, p_in, rep_in = train.train_backend(classes, device=dev, transform=transform)
    res['slice'] = dict(recordings=len(lab), speakers=rep_in['K'], xvectors=rep_in['N'])
    res['in_domain_only'] = der(recs, rows, transform, p_in, dev)
    res['interpolate'] = {f'{a:g}': der(recs, rows, transform, adapt.interpolate_plda(p_in, plda, a), dev)
                          for a in (0.25, 0.5, 0.75)}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    line = dict(gpu=q[0] if q else torch.cuda.get_device_name(0), accuracy=accuracy(dev),
                speed=speed(args.rounds, args.reps, dev))
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
