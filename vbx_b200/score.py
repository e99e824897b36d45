"""Diarization error rate (DER) of system output against reference RTTMs, accumulated on the GPU.

The scoring contract (DESIGN.md section 5.11): every boundary is converted once to int64 microseconds ("ticks"); reference
turns of one speaker that overlap or touch are merged; a collar c removes [x - c, x + c] around every merged reference
onset and offset, `ignore_overlaps` removes time with two or more reference speakers, a UEM restricts the scored time.
Over the scored time, with N_ref reference speakers active and the system silent or saying one label s,
    covered += d if the system speaks and N_ref >= 1,   fa += d if it speaks and N_ref = 0,   O[r, s] += d for active r,
    miss = ref_total - covered,  conf = covered - max one-to-one matching of O,  DER = (miss + fa + conf) / ref_total,
with ref_total the scored reference speaker time.  The kernel (vbx_score) accumulates covered, fa and O for many
(setting, recording) entries in one launch; the reference regions, ref_total and the matching are host work.

Overlap-aware output (DESIGN.md section 5.12) adds a second label per interval, said only inside overlap regions (an
overlapped-speech detector's RTTM, or the reference's own overlaps).  With N_sys in {0, 1, 2} system labels the counts
become  both += min(N_ref, N_sys) d,  fa += max(0, N_sys - N_ref) d,  O[r, s] += d for every active r and s;
miss = ref_total - both, conf = both - matching (vbx_score_overlap).

Jaccard error rate (DESIGN.md section 5.13), dscore's second metric: per recording the mean over reference speakers of
1 - |ref and sys| / |ref or sys| (scored time) after the one-to-one mapping that minimises it, without a collar and with overlaps scored.
vbx_score_jer adds each system label's scored time to the DER counts; R per speaker and the mapping are host work.

    python -m vbx_b200.score --ref-rttm ref/ --sys-rttm out/ [--uem all.uem] [--collar 0.25] [--ignore-overlaps]
        [--overlapping-system] [--jer] [--json]

PATH is an RTTM file or a directory of *.rttm.  Every reference recording is scored (one without system output counts as
all missed); system output for a recording the reference lacks is an error.  A system RTTM with overlapping speakers
needs --overlapping-system (at most two at a time).
"""
import argparse
import ctypes
import glob
import json
import os
import sys
from collections import namedtuple

import numpy as np

MAX_REF_SPEAKERS = 64
# the three protocols of the AMI recipe (AMI-diarization-setup): (name, collar seconds, ignore overlaps)
PROTOCOLS = (('forgiving', 0.25, True), ('fair', 0.25, False), ('full', 0.0, False))

# One recording prepared for scoring: the system's owned intervals [sys_lo, sys_hi) in ticks with their joined ends
# (sys_join_hi, see owned_intervals), the number of reference speakers and, per protocol name, the scored regions
# (lo, hi, mask, ref_total); overlap_regions: None, or per protocol name the scored regions split at the boundaries of
# the recording's overlap regions, (lo, hi, mask, ovl) with ovl = uint8 1 inside them (see split_regions);
# protocols: None, or per protocol name (collar ticks, ignore_overlaps), which decides where JER may be taken.
ScoredRecording = namedtuple('ScoredRecording', 'name sys_lo sys_hi sys_join_hi n_ref regions overlap_regions protocols',
                             defaults=(None, None))


def to_ticks(seconds):
    """Seconds -> int64 microseconds, np.rint(seconds * 1e6)."""
    return np.rint(np.asarray(seconds, dtype=np.float64) * 1e6).astype(np.int64)


def merge_turns(starts, ends):
    """Turns [start, end) in ticks -> sorted, disjoint turns: empty ones dropped, overlapping or touching ones merged."""
    s, e = np.asarray(starts, dtype=np.int64).reshape(-1), np.asarray(ends, dtype=np.int64).reshape(-1)
    keep = e > s
    s, e = s[keep], e[keep]
    o = np.argsort(s, kind='stable')
    s, e = s[o], e[o]
    if len(s) == 0:
        return s, e
    run = np.maximum.accumulate(e)
    first = np.nonzero(np.concatenate([[True], s[1:] > run[:-1]]))[0]
    return s[first], np.maximum.reduceat(e, first)


def reference_turns(rows):
    """formats.read_rttm rows -> {recording: [(starts, ends) merged ticks, one pair per speaker, speakers by name]}.
    Speakers whose turns are all empty are dropped; more than 64 speakers in a recording raise ValueError."""
    return {rec: [t for _, t in spk] for rec, spk in named_reference_turns(rows).items()}


def named_reference_turns(rows):
    """reference_turns() with each speaker's RTTM name kept: {recording: [(name, (starts, ends))]}, same order."""
    out = named_turns(rows)
    for rec, turns in out.items():
        if len(turns) > MAX_REF_SPEAKERS:
            raise ValueError(f'recording {rec!r}: {len(turns)} reference speakers, at most {MAX_REF_SPEAKERS} are supported')
    return out


def named_turns(rows):
    """named_reference_turns() without its cap on the number of speakers (which belongs to the score kernel)."""
    per = {}
    for rec, start, dur, spk in rows:
        per.setdefault(rec, {}).setdefault(spk, []).append((start, start + dur))
    out = {}
    for rec, spks in per.items():
        turns = []
        for spk in sorted(spks):
            t = to_ticks(np.array(spks[spk], dtype=np.float64))
            s, e = merge_turns(t[:, 0], t[:, 1])
            if len(s):
                turns.append((spk, (s, e)))
        out[rec] = turns
    return out


def reference_speaker_counts(turns, uem=None):
    """The oracle speaker count of every recording: {recording: number of speakers of reference_turns() `turns` with
    positive scored time}.  uem: None (all time is scored) or {recording: [(onset, offset)] seconds} (formats.read_uem),
    which then holds every recording of `turns`; a speaker who talks only outside it does not count."""
    out = {}
    for rec, spk in turns.items():
        if uem is None:
            out[rec] = len(spk)        # reference_turns keeps speakers with at least one non-empty turn only
            continue
        u = to_ticks(np.asarray(uem[rec], dtype=np.float64).reshape(-1, 2))
        ulo, uhi = merge_turns(u[:, 0], u[:, 1])
        n = 0
        for s, e in spk:
            # time of the speaker's disjoint turns inside the disjoint scored intervals
            inside = np.minimum(e[:, None], uhi[None, :]) - np.maximum(s[:, None], ulo[None, :])
            n += bool((inside > 0).any())
        out[rec] = n
    return out


def overlap_ticks(intervals):
    """Overlap regions [(onset, offset)] seconds (None = none) -> (lo, hi) int64 ticks, sorted and disjoint: the union
    of the intervals (merge_turns)."""
    t = to_ticks(np.asarray(intervals if intervals is not None else [], dtype=np.float64).reshape(-1, 2))
    return merge_turns(t[:, 0], t[:, 1])


def overlaps_from_rows(rows):
    """formats.read_rttm rows (an overlapped-speech detector's output; the speaker field is ignored) -> {recording:
    [(onset, offset)] seconds}, each recording's turns unioned.  A recording without rows has no overlap regions."""
    per = {}
    for rec, start, dur, _ in rows:
        per.setdefault(rec, []).append((start, start + dur))
    out = {}
    for rec, iv in per.items():
        lo, hi = overlap_ticks(iv)
        out[rec] = [(a / 1e6, b / 1e6) for a, b in zip(lo.tolist(), hi.tolist())]
    return out


def oracle_overlaps(turns):
    """reference_turns()[name] -> (lo, hi) ticks: the time in which two or more (merged) reference turns are active."""
    if not turns:
        z = np.zeros(0, dtype=np.int64)
        return z, z
    x = np.concatenate([a for t in turns for a in t])
    step = np.concatenate([np.full(len(t[0]), k, dtype=np.int64) for t in turns for k in (1, -1)])
    o = np.argsort(x, kind='stable')
    x, n = x[o], np.cumsum(step[o])
    on = n[:-1] >= 2                    # n[i] speakers on [x[i], x[i+1]); empty pieces at equal times are dropped
    return merge_turns(x[:-1][on], x[1:][on])


def split_regions(regions, overlap):
    """Scored regions (lo, hi, mask, ...) split at the boundaries of the overlap regions overlap = (lo, hi) ticks ->
    (lo, hi, mask, ovl): the same scored time and masks, ovl = uint8 1 where the piece lies inside an overlap region;
    neighbours with equal mask and flag joined (so with no overlap regions the regions come back unchanged)."""
    lo, hi, mask = (np.asarray(a) for a in regions[:3])
    olo, ohi = (np.asarray(a, dtype=np.int64) for a in overlap)
    if len(lo) == 0:
        return lo, hi, mask, np.zeros(0, dtype=np.uint8)
    b = np.unique(np.concatenate([lo, hi, olo, ohi]))
    plo, phi = b[:-1], b[1:]
    j = np.searchsorted(lo, plo, 'right') - 1
    keep = (j >= 0) & (hi[np.maximum(j, 0)] > plo)
    plo, phi, j = plo[keep], phi[keep], j[keep]
    pmask = mask[j]
    if len(olo):
        k = np.searchsorted(olo, plo, 'right') - 1
        ovl = ((k >= 0) & (ohi[np.maximum(k, 0)] > plo)).astype(np.uint8)
    else:
        ovl = np.zeros(len(plo), dtype=np.uint8)
    first = np.nonzero(np.concatenate([[True], (plo[1:] != phi[:-1]) | (pmask[1:] != pmask[:-1])
                                       | (ovl[1:] != ovl[:-1])]))[0]
    return plo[first], np.concatenate([phi[first[1:] - 1], phi[-1:]]), pmask[first], ovl[first]


def owned_intervals(seg_times):
    """x-vector segment times (T x 2 seconds) -> (lo, hi, join_hi) in ticks.  Segment t owns [lo_t, hi_t), where
    lo_t = (e_{t-1} + s_t) // 2 if s_t < e_{t-1} else s_t, and hi_t = (e_t + s_{t+1}) // 2 if s_{t+1} < e_t else e_t
    (s, e in ticks).  pipeline.merge_adjacent_labels also joins equal labels across a pause it takes for touching
    (np.isclose(e_t, s_{t+1}): up to about 1e-5 of the time, 10 ms at 1000 s); join_hi_t = lo_{t+1} there and hi_t
    elsewhere, and an interval followed by one of the same label ends at join_hi_t.  Runs of equal labels over these
    intervals are then exactly the segments merge_adjacent_labels writes to the RTTM."""
    seg = np.asarray(seg_times, dtype=np.float64).reshape(-1, 2)
    st = to_ticks(seg)
    lo, hi = st[:, 0].copy(), st[:, 1].copy()
    join_hi = hi.copy()
    if len(seg) > 1:
        over = st[1:, 0] < st[:-1, 1]
        mid = (st[:-1, 1] + st[1:, 0]) // 2
        lo[1:][over] = mid[over]
        hi[:-1][over] = mid[over]
        touching = np.isclose(seg[:-1, 1], seg[1:, 0])        # the test of pipeline.merge_adjacent_labels
        join_hi = hi.copy()
        join_hi[:-1] = np.where(touching, lo[1:], hi[:-1])
    return lo, hi, join_hi


def effective_hi(timeline, labels):
    """Where each owned interval ends for a labelling: join_hi where the next interval has the same label, else hi."""
    lo, hi, join_hi = timeline
    labels = np.asarray(labels).reshape(-1)
    out = np.asarray(hi, dtype=np.int64).copy()
    if len(labels) > 1:
        same = labels[1:] == labels[:-1]
        out[:-1][same] = np.asarray(join_hi)[:-1][same]
    return out


def scored_regions(turns, collar, ignore_overlaps, scored):
    """Scored time of one recording under one protocol.  turns: merged per-speaker (starts, ends) ticks; collar: ticks;
    scored: (lo, hi) sorted disjoint ticks (the UEM, or one interval spanning everything).  Returns (lo, hi, mask,
    ref_total): sorted disjoint regions, mask = uint64 bits of the active reference speakers (0 = scored non-speech),
    neighbours with equal masks joined, and ref_total = sum of N_ref * duration (Python int)."""
    slo, shi = (np.asarray(a, dtype=np.int64) for a in scored)
    c = int(collar)
    pts = [slo, shi]
    for s, e in turns:
        pts += [s, e] + ([s - c, s + c, e - c, e + c] if c else [])
    b = np.unique(np.concatenate(pts))
    lo, hi = b[:-1], b[1:]                           # elementary stretches: nothing changes inside one
    mask = np.zeros(len(lo), dtype=np.uint64)
    n = np.zeros(len(lo), dtype=np.int64)
    for k, (s, e) in enumerate(turns):
        j = np.searchsorted(s, lo, 'right') - 1
        act = (j >= 0) & (e[np.maximum(j, 0)] > lo)
        mask |= act.astype(np.uint64) << np.uint64(k)
        n += act
    if len(slo):
        j = np.searchsorted(slo, lo, 'right') - 1
        keep = (j >= 0) & (shi[np.maximum(j, 0)] > lo)
    else:
        keep = np.zeros(len(lo), dtype=bool)
    if c and turns:
        x = np.concatenate([np.concatenate([s, e]) for s, e in turns])
        zs, ze = np.sort(x - c), np.sort(x + c)
        keep &= np.searchsorted(zs, lo, 'right') - np.searchsorted(ze, lo, 'right') == 0
    if ignore_overlaps:
        keep &= n < 2
    lo, hi, mask, n = lo[keep], hi[keep], mask[keep], n[keep]
    ref_total = int(np.sum(n * (hi - lo)))
    if len(lo):
        first = np.nonzero(np.concatenate([[True], (lo[1:] != hi[:-1]) | (mask[1:] != mask[:-1])]))[0]
        hi = np.concatenate([hi[first[1:] - 1], hi[-1:]])
        lo, mask = lo[first], mask[first]
    return lo, hi, mask, ref_total


def collar_ticks(collar):
    if not collar >= 0:
        raise ValueError(f'collar must be >= 0 seconds, got {collar}')
    return int(to_ticks(collar))


def prepare_recording(name, turns, timeline, uem=None, protocols=PROTOCOLS, overlap=None):
    """A ScoredRecording.  turns: reference_turns()[name]; timeline: the system's intervals in ticks as (lo, hi,
    join_hi): owned_intervals() of the x-vectors, or (lo, hi, hi) for the turns of a system RTTM; uem: None (all time is
    scored) or [(onset, offset)] seconds; protocols: (name, collar seconds, ignore_overlaps) triples; overlap: None, or
    the overlap regions as sorted disjoint (lo, hi) ticks (overlap_ticks, oracle_overlaps) for overlap-aware entries."""
    if len(turns) > MAX_REF_SPEAKERS:
        raise ValueError(f'recording {name!r}: {len(turns)} reference speakers, at most {MAX_REF_SPEAKERS} are supported')
    sys_lo, sys_hi, sys_join_hi = (np.asarray(a, dtype=np.int64) for a in timeline)
    if uem is None:      # nothing speaks outside the span of all turns: scoring all time = scoring that span
        cat = np.concatenate([sys_lo, sys_hi, sys_join_hi] + [a for t in turns for a in t])
        scored = (np.array([cat.min()]), np.array([cat.max()])) if len(cat) else (cat, cat)
    else:
        u = to_ticks(np.asarray(uem, dtype=np.float64).reshape(-1, 2))
        scored = merge_turns(u[:, 0], u[:, 1])
    regions = {p: scored_regions(turns, collar_ticks(c), io, scored) for p, c, io in protocols}
    split = None if overlap is None else {p: split_regions(g, overlap) for p, g in regions.items()}
    return ScoredRecording(name, sys_lo, sys_hi, sys_join_hi, len(turns), regions, split,
                           {p: (collar_ticks(c), bool(io)) for p, c, io in protocols})


def result(miss, fa, conf, scored):
    """Error dict from tick counts: der (None without scored reference speech) and seconds, plus the exact ticks."""
    miss, fa, conf, scored = int(miss), int(fa), int(conf), int(scored)
    return dict(der=(miss + fa + conf) / scored if scored else None, miss=miss * 1e-6, fa=fa * 1e-6, conf=conf * 1e-6,
                scored=scored * 1e-6, ticks=dict(miss=miss, fa=fa, conf=conf, scored=scored))


def overall(results):
    """Sum of the numerators over the sum of the denominators of several result() dicts."""
    t = [r['ticks'] for r in results]
    return result(*(sum(x[k] for x in t) for k in ('miss', 'fa', 'conf', 'scored')))


def finish(covered, fa, O, ref_total):
    """result() from the accumulated covered (overlap-aware: both) / fa ticks and the overlap matrix O [n_ref x n_labels]
    (int64)."""
    from scipy.optimize import linear_sum_assignment
    O = np.asarray(O, dtype=np.int64)
    matched = 0
    if O.size:
        r, c = linear_sum_assignment(O, maximize=True)
        matched = int(O[r, c].sum())
    covered = int(covered)
    return result(int(ref_total) - covered, fa, covered - matched, ref_total)


def rank(per_setting, key='der'):
    """{name: result dict} -> names by result[key] ascending, 'der' (result, overall) or 'jer' (jer_finish, overall_jer);
    stable in the given order, settings without a value last."""
    names = list(per_setting)
    return sorted(names, key=lambda n: (per_setting[n][key] is None, per_setting[n][key] or 0.0))


def reference_time(regions, n_ref):
    """Scored time of each reference speaker (list of n_ref Python ints) over a region set (lo, hi, mask, ...)."""
    lo, hi = (np.asarray(a, dtype=np.int64) for a in regions[:2])
    mask = np.asarray(regions[2], dtype=np.uint64)
    return [int(np.sum((hi - lo)[((mask >> np.uint64(k)) & np.uint64(1)) == 1])) for k in range(n_ref)]


def speaker_jer(t):
    """One counted reference speaker's Jaccard error from its ticks (an element of jer_finish()['ticks']): 1 unmapped,
    else 1 - I / (R + S - I)."""
    if t['label'] is None:
        return 1.0
    u = t['R'] + t['S'] - t['I']
    return (u - t['I']) / u


def _jer_value(ticks):
    return sum(speaker_jer(t) for t in ticks) / len(ticks) if ticks else None


def jer_finish(R, S, O):
    """Jaccard error rate of one recording (DESIGN.md section 5.13) from exact ticks under scored time without a collar
    and with overlaps scored: R [K] reference speakers' scored time, S [L] the system labels' scored time, O [K x L]
    their intersections.  Speakers with R = 0 and labels with S = 0 are not counted; the one-to-one mapping minimises
    the summed cost c = (R + S - 2 I) / (R + S - I) (scipy.optimize.linear_sum_assignment); a mapped speaker's error is
    its c, an unmapped one's 1.  Returns dict(jer=mean over counted speakers or None without one, speakers=their number,
    ticks=[dict(ref=k, R, label=s or None, S, I) per counted speaker, by k]); jer is a pure function of ticks."""
    from scipy.optimize import linear_sum_assignment
    R = np.asarray(R, dtype=np.int64).reshape(-1)
    S = np.asarray(S, dtype=np.int64).reshape(-1)
    O = np.asarray(O, dtype=np.int64).reshape(len(R), len(S))
    ks, ls = np.nonzero(R > 0)[0], np.nonzero(S > 0)[0]
    label = {}
    if len(ks) and len(ls):
        Rk, Sl, I = R[ks][:, None], S[ls][None, :], O[np.ix_(ks, ls)]
        cost = (Rk + Sl - 2 * I).astype(np.float64) / (Rk + Sl - I).astype(np.float64)
        rows, cols = linear_sum_assignment(cost)
        label = {int(ks[r]): int(ls[c]) for r, c in zip(rows, cols)}
    ticks = []
    for k in ks.tolist():
        s = label.get(k)
        ticks.append(dict(ref=k, R=int(R[k]), label=s, S=None if s is None else int(S[s]),
                          I=None if s is None else int(O[k, s])))
    return dict(jer=_jer_value(ticks), speakers=len(ticks), ticks=ticks)


def overall_jer(results):
    """JER of several recordings from their jer_finish() dicts: the mean over all their counted reference speakers, so
    every speaker weighs the same whatever its recording.  dict(jer, speakers); jer None without any speaker."""
    ticks = [t for r in results for t in r['ticks']]
    return dict(jer=_jer_value(ticks), speakers=len(ticks))


def _overlap_split(rec, proto):
    if rec.overlap_regions is not None:
        return rec.overlap_regions[proto]
    lo, hi, mask, _ = rec.regions[proto]
    return lo, hi, mask, np.zeros(len(lo), dtype=np.uint8)


def score_entries(recordings, entries, device=None, jer=None, blocks=False):
    """Score many (recording, labels) entries in one vbx_score launch per protocol.
    recordings: list of ScoredRecording (all with the same protocols); entries: [(recording index, labels)], labels int
    [len(sys_lo)] in [0, n) (n = max label + 1).  Returns [{protocol: result dict}] in entry order.  A label outside
    that range raises VbxError.
    Overlap-aware entries (recording index, labels, labels2) go to one vbx_score_overlap launch per protocol instead:
    labels2 (None = no second speaker, or int with -1 = none) is said inside the recording's overlap regions
    (prepare_recording(overlap=); none when it was not given).  A call takes one kind of entry only.
    jer: None, or the name of a protocol with collar 0 and overlaps scored (DESIGN.md section 5.13).  That protocol's
    launch goes to vbx_score_jer, which also sums each label's scored time, and every entry's dict gains
    'jer': jer_finish() (replacing the DER of a protocol that is itself named 'jer').  Any other protocol raises
    ValueError.
    blocks: every entry's dict also gains 'O': {protocol: its n_ref x n labels overlap block, int64 ticks}."""
    import torch
    from . import _lib
    from ._lib import VbxError
    if jer is not None:
        for r in recordings:
            if (r.protocols or {}).get(jer) != (0, False):
                raise ValueError(f'jer={jer!r}: the Jaccard error rate needs a protocol of these recordings with collar '
                                 '0 and overlaps scored')
    if not entries:
        return []
    if not torch.cuda.is_available():
        raise VbxError('score_entries(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    lens = np.array([len(r.sys_lo) for r in recordings], dtype=np.int64)
    sys_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n_ref = np.array([r.n_ref for r in recordings], dtype=np.int32)
    second = len(entries[0]) == 3
    if any(len(e) != len(entries[0]) or len(e) not in (2, 3) for e in entries):
        raise ValueError('entries must all be (recording, labels) or all (recording, labels, labels2)')
    rec_idx = np.array([e[0] for e in entries], dtype=np.int32)
    labs = [np.asarray(e[1]).reshape(-1) for e in entries]
    labs2 = [np.full(len(l), -1, dtype=np.int64) if e[2] is None else np.asarray(e[2]).reshape(-1)
             for e, l in zip(entries, labs)] if second else []
    for i, (b, l) in enumerate(zip(rec_idx, labs)):
        if not 0 <= b < len(recordings):
            raise ValueError(f'entry {i}: recording index {b} out of range')
        if len(l) != lens[b] or (second and len(labs2[i]) != lens[b]):
            raise ValueError(f'entry {i}: {len(l)} labels for {lens[b]} intervals of {recordings[b].name!r}')
    n_labels = np.array([max(int(l.max()) + 1, 1) if len(l) else 1 for l in labs], dtype=np.int32)
    if second:
        n_labels = np.maximum(n_labels, [int(l.max()) + 1 if len(l) else 1 for l in labs2]).astype(np.int32)
    label_off = np.concatenate([[0], np.cumsum([len(l) for l in labs])[:-1]]).astype(np.int64)
    cells = n_ref[rec_idx].astype(np.int64) * n_labels
    o_off = np.concatenate([[0], np.cumsum(cells)[:-1]]).astype(np.int64)
    protocols = list(recordings[0].regions)
    lib = _lib.load()
    # one unused trailing element: an empty array still gets a device pointer
    d = lambda a: torch.from_numpy(np.concatenate([a, np.zeros(1, a.dtype)])).to(dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    common = [d(sys_off)] + [d(np.concatenate([getattr(r, f) for r in recordings])) for f in ('sys_lo', 'sys_hi', 'sys_join_hi')]
    ent = [d(rec_idx), d(label_off), d(np.concatenate(labs).astype(np.int32))]
    ent += [d(np.concatenate(labs2).astype(np.int32))] if second else []
    ent += [d(n_labels), d(o_off)]
    nref_d = d(n_ref)
    if jer is not None:
        t_off = np.concatenate([[0], np.cumsum(n_labels.astype(np.int64))[:-1]]).astype(np.int64)
        t_off_d = d(t_off)
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    outs = {}
    try:
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            for proto in protocols:
                regs = [_overlap_split(r, proto) if second else r.regions[proto] for r in recordings]
                reg_off = np.concatenate([[0], np.cumsum([len(g[0]) for g in regs])]).astype(np.int64)
                rd = [d(reg_off)] + [d(np.concatenate([g[i] for g in regs]).view(np.int64)) for i in range(3)]
                rd += [d(np.concatenate([g[3] for g in regs]).astype(np.uint8))] if second else []
                cov = torch.empty(len(entries), dtype=torch.int64, device=dev)
                fa = torch.empty_like(cov)
                O = torch.empty(max(int(cells.sum()), 1), dtype=torch.int64, device=dev)
                flags = torch.empty(len(entries), dtype=torch.int32, device=dev)
                if proto == jer:
                    fn = lib.vbx_score_jer
                    T = torch.empty(max(int(n_labels.sum()), 1), dtype=torch.int64, device=dev)
                    # single-label entries pass NULL for reg_overlap and labels2
                    args = [*map(p, rd), None] if not second else list(map(p, rd))
                    args += [p(nref_d), len(entries)] + list(map(p, ent[:3])) + ([] if second else [None])
                    args += list(map(p, ent[3:])) + [int(cells.max()), p(cov), p(fa), p(O), p(flags), p(t_off_d), p(T)]
                    rc = fn(h, len(recordings), *map(p, common), *args, stream)
                    outs[proto] = (cov, fa, O, flags, T, rd)
                else:
                    fn = lib.vbx_score_overlap if second else lib.vbx_score
                    rc = fn(h, len(recordings), *map(p, common), *map(p, rd), p(nref_d), len(entries), *map(p, ent),
                            int(cells.max()), p(cov), p(fa), p(O), p(flags), stream)
                    outs[proto] = (cov, fa, O, flags, rd)      # rd stays referenced until the results are read
                if rc != 0:
                    raise VbxError(f'{fn.__name__} failed ({rc}): {lib.vbx_last_error(h).decode()}')
            host = {k: tuple(t.cpu().numpy() for t in v[:-1]) for k, v in outs.items()}
    finally:
        lib.vbx_destroy(h)
    res = [{} for _ in entries]
    for proto in protocols:
        cov, fa, O, flags = host[proto][:4]
        bad = np.nonzero(flags)[0]
        if len(bad):
            i = int(bad[0])
            why = f'labels must lie in [0, {int(n_labels[i])})' if flags[i] & _lib.SCORE_BAD_LABEL else 'bad input'
            if second and flags[i] & _lib.SCORE_BAD_LABEL:
                why += ', second labels in [-1, n) and different from the first'
            name = 'vbx_score_jer' if proto == jer else 'vbx_score_overlap' if second else 'vbx_score'
            raise VbxError(f'{name}: entry {i} ({recordings[rec_idx[i]].name!r}) flags {int(flags[i])}: {why}')
        for i, b in enumerate(rec_idx):
            blk = O[o_off[i]:o_off[i] + cells[i]].reshape(int(n_ref[b]), int(n_labels[i]))
            res[i][proto] = finish(cov[i], fa[i], blk, recordings[b].regions[proto][3])
            if blocks:
                res[i].setdefault('O', {})[proto] = blk
    if jer is not None:
        O, T = host[jer][2], host[jer][4]
        R = [reference_time(r.regions[jer], r.n_ref) for r in recordings]
        for i, b in enumerate(rec_idx):
            blk = O[o_off[i]:o_off[i] + cells[i]].reshape(int(n_ref[b]), int(n_labels[i]))
            res[i]['jer'] = jer_finish(R[b], T[t_off[i]:t_off[i] + n_labels[i]], blk)
    return res


def _rows_by_recording(rows):
    out = {}
    for row in rows:
        out.setdefault(row[0], []).append(row)
    return out


def system_turns(rows, recording=''):
    """System RTTM rows of one recording -> (lo, hi, labels): turns in ticks sorted by start, turns of the same label
    merged, labels numbered by name.  Overlapping turns of different labels raise ValueError (single-speaker output
    only)."""
    names = sorted(set(r[3] for r in rows))
    lo, hi, lab = [], [], []
    for k, spk in enumerate(names):
        t = to_ticks(np.array([(r[1], r[1] + r[2]) for r in rows if r[3] == spk], dtype=np.float64))
        s, e = merge_turns(t[:, 0], t[:, 1])
        lo.append(s)
        hi.append(e)
        lab.append(np.full(len(s), k, dtype=np.int32))
    if not names:
        z = np.zeros(0, dtype=np.int64)
        return z, z, np.zeros(0, dtype=np.int32)
    lo, hi, lab = np.concatenate(lo), np.concatenate(hi), np.concatenate(lab)
    o = np.argsort(lo, kind='stable')
    lo, hi, lab = lo[o], hi[o], lab[o]
    if len(lo) > 1 and np.any(lo[1:] < np.maximum.accumulate(hi)[:-1]):
        raise ValueError(f'recording {recording!r}: the system RTTM has overlapping turns of different speakers; '
                         'only single-speaker system output can be scored')
    return lo, hi, lab


def system_stretches(rows, recording=''):
    """System RTTM rows of one recording whose speakers may overlap -> (lo, hi, labels, labels2): sorted disjoint
    stretches in ticks in which one or two labels speak (labels numbered by name, turns of one label merged; labels2 =
    -1 where one speaks, else the larger number).  Three or more simultaneous speakers raise ValueError."""
    names = sorted(set(r[3] for r in rows))
    turns = []
    for spk in names:
        t = to_ticks(np.array([(r[1], r[1] + r[2]) for r in rows if r[3] == spk], dtype=np.float64))
        turns.append(merge_turns(t[:, 0], t[:, 1]))
    b = np.unique(np.concatenate([a for t in turns for a in t] + [np.zeros(0, dtype=np.int64)]))
    lo, hi = b[:-1], b[1:]
    l1, l2 = np.full(len(lo), -1, dtype=np.int32), np.full(len(lo), -1, dtype=np.int32)
    n = np.zeros(len(lo), dtype=np.int64)
    for k, (s, e) in enumerate(turns):
        if len(s) == 0:                 # a speaker whose turns are all empty says nothing
            continue
        j = np.searchsorted(s, lo, 'right') - 1
        act = (j >= 0) & (e[np.maximum(j, 0)] > lo)
        l2 = np.where(act & (l1 >= 0), k, l2)
        l1 = np.where(act & (l1 < 0), k, l1)
        n += act
    if np.any(n > 2):
        i = int(np.argmax(n > 2))
        raise ValueError(f'recording {recording!r}: {int(n[i])} system speakers at {lo[i] / 1e6:.6f} s; '
                         'at most two simultaneous system speakers can be scored')
    keep = n > 0
    return lo[keep], hi[keep], l1[keep], l2[keep]


def score_rttm(ref_turns, sys_turns, collar, ignore_overlaps, uem=None, device=None, overlapping=False, jer=False,
               across_files=False, by_name=False):
    """DER of system RTTM rows against reference RTTM rows (both as formats.read_rttm returns them).
    uem: None or {recording: [(onset, offset)]} (formats.read_uem).  overlapping: the system may have two speakers at
    once (system_stretches, scored by vbx_score_overlap); otherwise overlapping system turns raise ValueError.  Returns
    ({recording: result dict}, overall result dict) over the reference's recordings.
    jer: also the Jaccard error rate (DESIGN.md section 5.13; no collar, overlaps scored, whatever the DER uses): every
    result dict gains jer (None without a counted reference speaker) and each recording's also jer_ticks
    (jer_finish()['ticks']).
    across_files: speakers are one speaker in every file where they have the same RTTM name, in the reference and in
    the system (DESIGN.md section 5.15); the overall dict gains across_files, a result dict with the overall miss and fa
    and conf = sum of covered - max one-to-one matching of the overlaps summed over all files by name.
    by_name: a system speaker is right only where its RTTM name is the reference speaker's (DESIGN.md section 5.16): the
    overall dict gains by_name, a result dict with the overall miss and fa and conf = sum of covered - the overlaps of
    equal names summed over all files (so by_name conf >= across_files conf)."""
    c = collar_ticks(collar)
    # JER is taken without a collar and with overlaps: from the DER's own launch when that is the protocol, else from
    # one more region set
    jer_proto = None if not jer else 'score' if c == 0 and not ignore_overlaps else 'jer'
    named = named_reference_turns(ref_turns)
    ref = {rec: [t for _, t in spk] for rec, spk in named.items()}
    sys_by = _rows_by_recording(sys_turns)
    extra = sorted(set(sys_by) - set(ref))
    if extra:
        raise ValueError(f'system output for recordings the reference lacks: {extra}')
    names = sorted(ref)
    recs, entries = [], []
    for b, n in enumerate(names):
        if uem is not None and n not in uem:
            raise ValueError(f'recording {n!r} is missing from the UEM')
        proto = (('score', collar, bool(ignore_overlaps)),) + ((('jer', 0.0, False),) if jer_proto == 'jer' else ())
        u = None if uem is None else uem[n]
        if overlapping:                 # stream 2 is said wherever the system has a second speaker: no clipping
            lo, hi, lab, lab2 = system_stretches(sys_by.get(n, []), n)
            recs.append(prepare_recording(n, ref[n], (lo, hi, hi), u, proto, overlap=(lo[:1], hi[-1:])))
            entries.append((b, lab, lab2))
            continue
        lo, hi, lab = system_turns(sys_by.get(n, []), n)
        recs.append(prepare_recording(n, ref[n], (lo, hi, hi), u, proto))
        entries.append((b, lab))
    res = score_entries(recs, entries, device, jer=jer_proto, blocks=across_files or by_name)
    per = {n: r['score'] for n, r in zip(names, res)}
    tot = overall(list(per.values()))
    if across_files or by_name:
        sys_names = {n: sorted(set(r[3] for r in sys_by.get(n, []))) for n in names}
        args = (tot, [[k for k, _ in named[n]] for n in names], [sys_names[n] for n in names],
                [r['O']['score'] for r in res])
        if across_files:
            tot['across_files'] = across_files_result(*args)
        if by_name:
            tot['by_name'] = by_name_result(*args)
    if jer:
        for n, r in zip(names, res):
            per[n] = dict(per[n], jer=r['jer']['jer'], jer_ticks=r['jer']['ticks'])
        tot['jer'] = overall_jer([r['jer'] for r in res])['jer']
    return per, tot


def across_files_result(tot, ref_names, sys_names, blocks):
    """DER across files (DESIGN.md section 5.15) from overall() `tot` of the per-file results and, per file, the names
    of its reference speakers (block rows), of its system labels (sorted, as system_turns numbers them) and its overlap
    block: the blocks are summed by name and matched once.  A block has a column for every label up to the last one with
    a non-empty turn, so names past it (speakers whose turns are all empty) and a file without system names add nothing."""
    from scipy.optimize import linear_sum_assignment
    _, _, O = _blocks_by_name(ref_names, sys_names, blocks)
    matched = 0
    if O.size:
        r, c = linear_sum_assignment(O, maximize=True)
        matched = int(O[r, c].sum())
    t = tot['ticks']
    covered = t['scored'] - t['miss']
    return result(t['miss'], t['fa'], covered - matched, t['scored'])


def by_name_result(tot, ref_names, sys_names, blocks):
    """Name-level DER (DESIGN.md section 5.16), arguments as across_files_result: the overlap blocks summed by name,
    and only the cells whose reference and system names are equal count as matched."""
    rows, cols, O = _blocks_by_name(ref_names, sys_names, blocks)
    matched = sum(int(O[i, cols[k]]) for k, i in rows.items() if k in cols)
    t = tot['ticks']
    covered = t['scored'] - t['miss']
    return result(t['miss'], t['fa'], covered - matched, t['scored'])


def _blocks_by_name(ref_names, sys_names, blocks):
    """The per-file overlap blocks summed by name: ({ref name: row}, {system name: column}, O [rows, columns])."""
    rows = {k: i for i, k in enumerate(sorted({k for ks in ref_names for k in ks}))}
    cols = {k: i for i, k in enumerate(sorted({k for ks in sys_names for k in ks}))}
    O = np.zeros((len(rows), len(cols)), dtype=np.int64)
    for rk, sk, blk in zip(ref_names, sys_names, blocks):
        blk = np.asarray(blk)
        w = min(blk.shape[1], len(sk))
        if rk and w:
            np.add.at(O, np.ix_([rows[k] for k in rk], [cols[k] for k in sk[:w]]), blk[:, :w])
    return rows, cols, O


def read_rttm_path(path):
    """formats.read_rttm rows of an RTTM file, or of every *.rttm in a directory (sorted by name)."""
    from . import formats
    files = sorted(glob.glob(os.path.join(path, '*.rttm'))) if os.path.isdir(path) else [path]
    if not files:
        raise ValueError(f'{path}: no *.rttm files')
    return [row for f in files for row in formats.read_rttm(f)]


def read_overlaps(path):
    """Overlap regions from an RTTM file or directory (overlaps_from_rows): {recording: [(onset, offset)] seconds}."""
    return overlaps_from_rows(read_rttm_path(path))


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--ref-rttm', required=True, help='reference RTTM file or directory of *.rttm')
    ap.add_argument('--sys-rttm', required=True, help='system RTTM file or directory of *.rttm')
    ap.add_argument('--uem', default=None, help='UEM file (default: all time is scored)')
    ap.add_argument('--collar', default=0.25, type=float, help='seconds removed either side of every reference boundary')
    ap.add_argument('--ignore-overlaps', action='store_true', help='do not score time with 2 or more reference speakers')
    ap.add_argument('--overlapping-system', action='store_true',
                    help='the system RTTM may have two speakers at once (overlap-aware output)')
    ap.add_argument('--json', action='store_true', help='print one JSON object instead of the table')
    ap.add_argument('--jer', action='store_true',
                    help='also the Jaccard error rate (no collar, overlaps scored, whatever the DER options)')
    ap.add_argument('--across-files', action='store_true',
                    help='also the DER with each speaker name one speaker in every file (ACROSS FILES row)')
    ap.add_argument('--by-name', action='store_true',
                    help='also the DER with system speakers right only under the reference name (BY NAME row)')
    return ap


def main(argv=None):
    args = build_parser().parse_args(argv)
    from . import formats
    uem = formats.read_uem(args.uem) if args.uem else None
    per, tot = score_rttm(read_rttm_path(args.ref_rttm), read_rttm_path(args.sys_rttm), args.collar,
                          args.ignore_overlaps, uem, overlapping=args.overlapping_system, jer=args.jer,
                          across_files=args.across_files, by_name=args.by_name)
    if args.json:
        print(json.dumps(dict(collar=args.collar, ignore_overlaps=args.ignore_overlaps, files=per, overall=tot),
                         sort_keys=True))
        return 0
    rows = list(per.items()) + [('OVERALL', tot)] + ([('ACROSS FILES', tot['across_files'])] if args.across_files else []) \
        + ([('BY NAME', tot['by_name'])] if args.by_name else [])
    w = max(len(n) for n, _ in rows)
    jer_head = f'  {"JER %":>7}' if args.jer else ''
    print(f'{"file":<{w}}  {"DER %":>7}  {"miss %":>7}  {"FA %":>7}  {"conf %":>7}  {"scored s":>10}{jer_head}')
    for n, r in rows:
        pct = [100.0 * r[k] / r['scored'] if r['scored'] else float('nan') for k in ('miss', 'fa', 'conf')]
        der = 100.0 * r['der'] if r['der'] is not None else float('nan')
        jer = r.get('jer') if n not in ('ACROSS FILES', 'BY NAME') else None
        jer_col = (f'  {100.0 * jer if jer is not None else float("nan"):7.2f}') if args.jer else ''
        print(f'{n:<{w}}  {der:7.2f}  {pct[0]:7.2f}  {pct[1]:7.2f}  {pct[2]:7.2f}  {r["scored"]:10.2f}{jer_col}')
    return 0


if __name__ == '__main__':
    sys.exit(main())
