"""Diarization error rate restated as a line sweep over integer ticks (test infrastructure; product code never imports it).

It starts from RTTM-level segments -- reference turns and the system's merged segments (pipeline.merge_adjacent_labels
output or a parsed system RTTM) -- not from the owned x-vector intervals or the scored regions the device scores, and
counts errors the md-eval way per stretch of constant state:  miss += max(0, N_ref - N_sys) d,
fa += max(0, N_sys - N_ref) d,  conf = sum min(N_ref, N_sys) d - (best one-to-one speaker mapping of the overlaps).
Explicit sets of active reference and system speakers are kept at every boundary event.
"""
from collections import defaultdict

import numpy as np


def merge_speaker_turns(turns):
    """[(start, end, speaker)] -> the same with each speaker's overlapping or touching turns merged, empty ones dropped."""
    by = defaultdict(list)
    for s, e, k in turns:
        if e > s:
            by[k].append((int(s), int(e)))
    out = []
    for k, ts in by.items():
        ts.sort()
        cs, ce = ts[0]
        for s, e in ts[1:]:
            if s <= ce:
                ce = max(ce, e)
            else:
                out.append((cs, ce, k))
                cs, ce = s, e
        out.append((cs, ce, k))
    return out


def der_ticks(ref_turns, sys_segments, collar=0, ignore_overlaps=False, uem=None):
    """ref_turns: [(start, end, speaker)] ticks; sys_segments: [(start, end, label)] ticks; collar: ticks; uem: None (all
    time scored) or [(onset, offset)] ticks.  Returns dict(miss, fa, conf, scored) in ticks (Python ints)."""
    from scipy.optimize import linear_sum_assignment
    ref = merge_speaker_turns(ref_turns)
    ev = defaultdict(list)               # time -> [(kind, key, +1 / -1)]
    for s, e, k in ref:
        ev[s].append(('ref', k, 1))
        ev[e].append(('ref', k, -1))
        if collar > 0:
            for x in (s, e):
                ev[x - collar].append(('collar', None, 1))
                ev[x + collar].append(('collar', None, -1))
    for s, e, l in sys_segments:
        if e > s:
            ev[int(s)].append(('sys', l, 1))
            ev[int(e)].append(('sys', l, -1))
    for s, e in uem or []:
        if e > s:
            ev[int(s)].append(('uem', None, 1))
            ev[int(e)].append(('uem', None, -1))
    cnt = {'ref': defaultdict(int), 'sys': defaultdict(int), 'collar': defaultdict(int), 'uem': defaultdict(int)}
    miss = fa = both = scored = 0
    overlap = defaultdict(int)           # (ref speaker, sys label) -> ticks
    times = sorted(ev)
    for t, t_next in zip(times, times[1:] + [None]):
        for kind, key, step in ev[t]:
            cnt[kind][key] += step
        if t_next is None:
            break
        d = t_next - t
        ref_on = {k for k, c in cnt['ref'].items() if c > 0}
        sys_on = {k for k, c in cnt['sys'].items() if c > 0}
        if uem is not None and cnt['uem'][None] <= 0:
            continue
        if cnt['collar'][None] > 0 or (ignore_overlaps and len(ref_on) >= 2):
            continue
        nr, ns = len(ref_on), len(sys_on)
        scored += nr * d
        miss += max(0, nr - ns) * d
        fa += max(0, ns - nr) * d
        both += min(nr, ns) * d
        for r in ref_on:
            for s in sys_on:
                overlap[(r, s)] += d
    matched = 0
    if overlap:
        rs = sorted({r for r, _ in overlap}, key=str)
        ss = sorted({s for _, s in overlap}, key=str)
        M = np.array([[overlap.get((r, s), 0) for s in ss] for r in rs], dtype=np.int64)
        i, j = linear_sum_assignment(M, maximize=True)
        matched = int(sum(int(M[a, b]) for a, b in zip(i, j)))
    return dict(miss=miss, fa=fa, conf=both - matched, scored=scored)
