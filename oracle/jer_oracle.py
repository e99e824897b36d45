"""The tick counts behind the Jaccard error rate, restated as a line sweep (test infrastructure; product code never
imports it).  Kept beside der_oracle.py, whose DER sweep it mirrors, so that the DER oracle stays as it is.

It starts from RTTM-level segments -- reference turns and the system's segments (pipeline.merge_adjacent_labels output,
pipeline.overlap_segments output or a parsed system RTTM) -- not from the owned x-vector intervals or the scored regions
the device scores.  Scored time is the UEM (all time without one), with no collar and overlaps scored.  Explicit sets of
active reference and system speakers are kept at every boundary event, as der_oracle.der_ticks keeps them.
"""
from collections import defaultdict

from .der_oracle import merge_speaker_turns


def jer_ticks(ref_turns, sys_segments, uem=None):
    """ref_turns: [(start, end, speaker)] ticks; sys_segments: [(start, end, label)] ticks; uem: None (all time scored)
    or [(onset, offset)] ticks.  Returns dict(R={speaker: scored ticks}, S={label: scored ticks}, I={(speaker, label):
    ticks both are active}) of Python ints, speakers, labels and pairs with no scored time left out."""
    ev = defaultdict(list)               # time -> [(kind, key, +1 / -1)]
    for s, e, k in merge_speaker_turns(ref_turns):
        ev[s].append(('ref', k, 1))
        ev[e].append(('ref', k, -1))
    for s, e, l in sys_segments:
        if e > s:
            ev[int(s)].append(('sys', l, 1))
            ev[int(e)].append(('sys', l, -1))
    for s, e in uem or []:
        if e > s:
            ev[int(s)].append(('uem', None, 1))
            ev[int(e)].append(('uem', None, -1))
    cnt = {'ref': defaultdict(int), 'sys': defaultdict(int), 'uem': defaultdict(int)}
    R, S, I = defaultdict(int), defaultdict(int), defaultdict(int)
    times = sorted(ev)
    for t, t_next in zip(times, times[1:] + [None]):
        for kind, key, step in ev[t]:
            cnt[kind][key] += step
        if t_next is None:
            break
        if uem is not None and cnt['uem'][None] <= 0:
            continue
        d = t_next - t
        ref_on = {k for k, c in cnt['ref'].items() if c > 0}
        sys_on = {k for k, c in cnt['sys'].items() if c > 0}
        for r in ref_on:
            R[r] += d
        for s in sys_on:
            S[s] += d
        for r in ref_on:
            for s in sys_on:
                I[(r, s)] += d
    return dict(R=dict(R), S=dict(S), I=dict(I))
