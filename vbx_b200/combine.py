"""Combine several diarizations of an archive into one by label mapping and weighted voting (DESIGN.md section 5.21;
DOVER, Stolcke and Yoshioka 2019, with up to two simultaneous speakers per hypothesis), on the GPU (vbx_combine).

    python -m vbx_b200.combine --sys-rttm A B C [--weights 1,0.9,0.8] --out-rttm-dir OUT [--json]

Each of A, B, C is an RTTM file or a directory of *.rttm: one hypothesis.  A recording that a hypothesis lacks counts as
silent there.  Every hypothesis may have two speakers at once; three or more raise an error naming the file and time.
Per recording the hypotheses are ordered by how much they disagree with the others, the labels of each are mapped to
those of the ones before it, and every stretch of time keeps the speakers most hypotheses (by weight) agree on.  Without
--weights a hypothesis weighs rank ** -0.1 (rank 1 = the one that disagrees least).  OUT/<recording>.rttm holds the
result with speakers numbered by global label; --json prints the order, weights and disagreement matrix per recording.
Not compared with dover-lap: the rule is the one DESIGN.md states, mapped anchor-first as DOVER does.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

MAX_HYPOTHESES = 32
MAX_LABELS = 128


def check_weights(weights, K):
    """None, or K finite weights > 0 as a float64 array (ValueError otherwise)."""
    if weights is None:
        return None
    w = np.asarray(weights, dtype=np.float64).reshape(-1)
    if len(w) != K:
        raise ValueError(f'{len(w)} weights for {K} hypotheses')
    if not np.all(np.isfinite(w) & (w > 0)):
        raise ValueError(f'weights must be finite and > 0, got {w.tolist()}')
    return np.ascontiguousarray(w)


def combine_labels(intervals, hypotheses, weights=None, device=None, strict=True, blocks=False):
    """One vbx_combine call over many recordings.
    intervals: per recording (lo, hi), int64 ticks (score.to_ticks), sorted and disjoint.
    hypotheses: K in 2 .. 32 entries, each a list with per recording (labels, labels2): int arrays over the recording's
    intervals, -1 = none; labels2 may be None.  Labels lie in [-1, 128).
    weights: None (rank ** -0.1 per recording) or K finite weights > 0.
    Returns per recording dict(labels, labels2 (int64, global ids, -1 = none), order (hypotheses by rank), weights [K],
    D [K, K] int64 ticks, map (per hypothesis an int64 array: its label -> global id, -1 = a label without time),
    n_global, flags); blocks=True adds O ({(a, b): ticks a's label s shares with b's label u} for a < b) and L (per
    hypothesis the ticks of each label).
    strict: a second label without a first or equal to it, or more than 255 global labels in a recording, raise VbxError
    naming the recording's index; strict=False returns them as flags (_lib.COMBINE_*) instead."""
    import torch
    from . import _lib
    from ._lib import VbxError
    K, B = len(hypotheses), len(intervals)
    if not 2 <= K <= MAX_HYPOTHESES:
        raise ValueError(f'{K} hypotheses: combination takes 2 .. {MAX_HYPOTHESES}')
    w = check_weights(weights, K)
    if any(len(h) != B for h in hypotheses):
        raise ValueError(f'every hypothesis needs labels for all {B} recordings')
    lo = [np.asarray(iv[0], dtype=np.int64).reshape(-1) for iv in intervals]
    hi = [np.asarray(iv[1], dtype=np.int64).reshape(-1) for iv in intervals]
    lens = np.array([len(a) for a in lo], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    N = int(offsets[-1])
    l1, l2 = np.full((K, N), -1, dtype=np.int32), np.full((K, N), -1, dtype=np.int32)
    n_labels = np.zeros((B, K), dtype=np.int32)
    for k, hyp in enumerate(hypotheses):
        for b, (a1, a2) in enumerate(hyp):
            a1 = np.asarray(a1, dtype=np.int64).reshape(-1)
            a2 = np.full(len(a1), -1, dtype=np.int64) if a2 is None else np.asarray(a2, dtype=np.int64).reshape(-1)
            if len(a1) != lens[b] or len(a2) != lens[b] or len(hi[b]) != lens[b]:
                raise ValueError(f'hypothesis {k}, recording {b}: {len(a1)} labels for {lens[b]} intervals')
            top = int(max(a1.max(initial=-1), a2.max(initial=-1)))
            if top >= MAX_LABELS or min(a1.min(initial=-1), a2.min(initial=-1)) < -1:
                raise ValueError(f'hypothesis {k}, recording {b}: labels must lie in [-1, {MAX_LABELS})')
            n_labels[b, k] = top + 1
            l1[k, offsets[b]:offsets[b + 1]] = a1
            l2[k, offsets[b]:offsets[b + 1]] = a2
    if B == 0:
        return []
    if not torch.cuda.is_available():
        raise VbxError('combine_labels(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    ML, P = max(int(n_labels.max()), 1), K * (K - 1) // 2
    lib = _lib.load()
    d = lambda a: torch.from_numpy(np.concatenate([a.reshape(-1), np.zeros(1, a.dtype)])).to(dev)   # never empty
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    try:
        need = ctypes.c_size_t()
        if lib.vbx_combine_workspace_bytes(h, B, K, ML, ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_combine_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        with torch.cuda.device(dev):
            ins = [d(offsets), d(np.concatenate(lo)), d(np.concatenate(hi)), d(l1), d(l2)]
            ws = torch.empty(max(int(need.value), 1), dtype=torch.uint8, device=dev)
            new = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
            out1, out2 = new(N + 1, torch.int32), new(N + 1, torch.int32)
            order, wout = new((B, K), torch.int32), new((B, K), torch.float64)
            D, gmap = new((B, K, K), torch.int64), new((B, K, MAX_LABELS), torch.int32)
            ng, flags = new(B, torch.int32), new(B, torch.int32)
            O = new((B, P, ML, ML), torch.int64) if blocks else None
            L = new((B, K, ML), torch.int64) if blocks else None
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            rc = lib.vbx_combine(h, B, p(ins[0]), N, p(ins[1]), p(ins[2]), K, p(ins[3]), p(ins[4]),
                                 n_labels.ctypes.data_as(ctypes.c_void_p), ML,
                                 w.ctypes.data_as(ctypes.c_void_p) if w is not None else None, p(ws), ws.numel(),
                                 p(out1), p(out2), p(order), p(wout), p(D), p(gmap), p(ng), p(flags), p(O), p(L), stream)
            if rc != 0:
                raise VbxError(f'vbx_combine failed ({rc}): {lib.vbx_last_error(h).decode()}')
            host = [t.cpu().numpy() if t is not None else None for t in (out1, out2, order, wout, D, gmap, ng, flags, O, L)]
    finally:
        lib.vbx_destroy(h)
    out1, out2, order, wout, D, gmap, ng, flags, O, L = host
    if strict and flags.any():
        b = int(np.nonzero(flags)[0][0])
        why = 'more than 255 global labels' if flags[b] & _lib.COMBINE_TOO_MANY_LABELS else \
            'a second label without a first one, or equal to it'
        raise VbxError(f'vbx_combine: recording {b} flags {int(flags[b])}: {why}')
    res = []
    pairs = [(a, c) for a in range(K) for c in range(a + 1, K)]
    for b in range(B):
        s = slice(int(offsets[b]), int(offsets[b + 1]))
        item = dict(labels=out1[s].astype(np.int64), labels2=out2[s].astype(np.int64), order=order[b].tolist(),
                    weights=wout[b].copy(), D=D[b].copy(), n_global=int(ng[b]), flags=int(flags[b]),
                    map=[gmap[b, k, :n_labels[b, k]].astype(np.int64) for k in range(K)])
        if blocks:
            item['O'] = {pr: O[b, i, :n_labels[b, pr[0]], :n_labels[b, pr[1]]].copy() for i, pr in enumerate(pairs)}
            item['L'] = [L[b, k, :n_labels[b, k]].copy() for k in range(K)]
        res.append(item)
    return res


def common_timeline(rows_per_hypothesis):
    """Hypotheses with their own turn boundaries -> one set of atomic intervals per recording.
    rows_per_hypothesis: K lists of formats.read_rttm rows (recording, onset, duration, speaker).  Per recording (the
    sorted union of all recordings; one a hypothesis lacks is silent there) the boundaries of every hypothesis's turns
    (score.system_stretches, in ticks) cut the time into intervals on which no hypothesis changes; intervals on which
    all are silent are dropped.  Three or more simultaneous speakers in a hypothesis raise ValueError naming the
    recording and the time.  Returns (names, intervals, hypotheses) as combine_labels takes them: labels are numbered
    by speaker name within a hypothesis and recording."""
    from . import score
    by = [score._rows_by_recording(rows) for rows in rows_per_hypothesis]
    names = sorted(set().union(*by)) if by else []
    intervals, hyps = [], [[] for _ in by]
    for n in names:
        st = [score.system_stretches(b.get(n, []), n) for b in by]
        cuts = np.unique(np.concatenate([a for s in st for a in s[:2]] + [np.zeros(0, dtype=np.int64)]))
        lo, hi = cuts[:-1], cuts[1:]
        labs = []
        for slo, shi, s1, s2 in st:
            j = np.searchsorted(slo, lo, 'right') - 1
            inside = (j >= 0) & (shi[np.maximum(j, 0)] > lo) if len(slo) else np.zeros(len(lo), dtype=bool)
            jj = np.maximum(j, 0)
            labs.append((np.where(inside, s1[jj] if len(slo) else -1, -1).astype(np.int64),
                         np.where(inside, s2[jj] if len(slo) else -1, -1).astype(np.int64)))
        keep = np.zeros(len(lo), dtype=bool)
        for a1, _ in labs:
            keep |= a1 >= 0
        intervals.append((lo[keep], hi[keep]))
        for k, (a1, a2) in enumerate(labs):
            hyps[k].append((a1[keep], a2[keep]))
    return names, intervals, hyps


def combined_lines(name, lo, hi, labels, labels2):
    """RTTM lines of one recording from combined labels over intervals [lo, hi) in ticks: the merged segments of the
    first labels, then those of the second (pipeline.merge_adjacent_labels; silent intervals dropped), speakers numbered
    global id + 1."""
    from .pipeline import merge_adjacent_labels, rttm_lines
    s, e = np.asarray(lo, dtype=np.int64) / 1e6, np.asarray(hi, dtype=np.int64) / 1e6
    lines = []
    for lab in (labels, labels2):
        lab = np.asarray(lab)
        on = lab >= 0
        lines += rttm_lines(name, *merge_adjacent_labels(s[on], e[on], lab[on]))
    return lines


def combine_rttm(paths, weights=None, device=None):
    """Combine K hypotheses given as RTTM paths (files or directories of *.rttm) or as lists of formats.read_rttm rows.
    Returns {recording: dict(rttm (lines), lo, hi, and combine_labels' fields)}."""
    from . import score
    rows = [score.read_rttm_path(x) if isinstance(x, (str, os.PathLike)) else list(x) for x in paths]
    if not 2 <= len(rows) <= MAX_HYPOTHESES:
        raise ValueError(f'{len(rows)} hypotheses: combination takes 2 .. {MAX_HYPOTHESES}')
    check_weights(weights, len(rows))
    names, intervals, hyps = common_timeline(rows)
    res = combine_labels(intervals, hyps, weights, device)
    out = {}
    for n, (lo, hi), item in zip(names, intervals, res):
        out[n] = dict(item, lo=lo, hi=hi, rttm=combined_lines(n, lo, hi, item['labels'], item['labels2']))
    return out


def summary(item):
    """The JSON form of one recording's order, weights and disagreement matrix (seconds)."""
    return dict(order=list(item['order']), weights=[float(x) for x in item['weights']],
                D=(np.asarray(item['D']) * 1e-6).tolist(), n_global=int(item['n_global']))


def parse_weights(text):
    try:
        out = [float(t) for t in str(text).split(',') if t.strip()]
    except ValueError:
        raise argparse.ArgumentTypeError(f'expected comma-separated numbers, got {text!r}')
    if not out:
        raise argparse.ArgumentTypeError(f'expected comma-separated numbers, got {text!r}')
    return out


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--sys-rttm', required=True, nargs='+', help='2 .. 32 hypotheses: RTTM files or directories of *.rttm')
    ap.add_argument('--weights', default=None, type=parse_weights,
                    help='one weight > 0 per hypothesis, comma-separated (default: rank ** -0.1 per recording)')
    ap.add_argument('--out-rttm-dir', required=True, help='directory for one <recording>.rttm each')
    ap.add_argument('--device', default=None, help='CUDA device, e.g. cuda:0 (default: the current device)')
    ap.add_argument('--json', action='store_true', help='print order, weights and disagreement matrix per recording')
    return ap


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if not 2 <= len(args.sys_rttm) <= MAX_HYPOTHESES:
        ap.error(f'--sys-rttm takes 2 .. {MAX_HYPOTHESES} hypotheses')
    if args.weights is not None and len(args.weights) != len(args.sys_rttm):
        ap.error('--weights needs one weight per hypothesis')
    out = combine_rttm(args.sys_rttm, args.weights, args.device)
    os.makedirs(args.out_rttm_dir, exist_ok=True)
    for n, item in out.items():
        with open(os.path.join(args.out_rttm_dir, f'{n}.rttm'), 'w') as fp:
            fp.write(''.join(line + os.linesep for line in item['rttm']))
    if args.json:
        print(json.dumps({n: summary(item) for n, item in out.items()}, sort_keys=True))
    return 0


if __name__ == '__main__':
    sys.exit(main())
