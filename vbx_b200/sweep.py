"""Hyperparameter sweep: a whole grid of VBx settings over an archive as few large batches.

Every VBx recipe tunes Fa, Fb, loopP, the AHC threshold and the init smoothing per dataset, by grid search on a dev set.
Here the front end and the AHC linkage run once per archive; each threshold only repeats the host cut of the stored
linkage (ahc.cut).  Every (recording, setting) pair is one entry of a batch with per-recording Fa, Fb and loopP
(vbx_run_per_recording; a one-setting grid passes numbers to vbx_run, with bit-identical results), so a grid is a
handful of large batches instead of one small batch per setting.

    python -m vbx_b200.sweep --out-dir sweep --xvec-ark-file exp/ES2005a.ark --segments-file exp/ES2005a.seg \\
        --xvec-transform transform.h5 --plda-file plda --lda-dim 128 \\
        --Fa 0.2,0.3,0.4 --Fb 6,17,64 --loopP 0.35,0.65,0.99 --threshold=-0.015,0.1 --init-smoothing 5

(a list that starts with '-' needs the --option=list form) writes OUT/<setting>/<recording>.rttm and OUT/summary.json (speakers, iterations and flags per setting and recording).
With --ref-rttm (a file or a directory of *.rttm; optionally --uem) every entry is also scored on the GPU (vbx_b200/score.py)
under the three AMI protocols: summary.json then holds the DER per recording and setting, the overall DER per setting, and
`ranking`: per protocol, the setting names by overall DER.
With --overlap-rttm PATH (an overlapped-speech detector's RTTM) or --oracle-overlaps (the reference's own overlaps; needs
--ref-rttm) every setting also writes OUT/<setting>/overlap/<recording>.rttm, the overlap-aware output (DESIGN.md section
5.12); with a reference it is scored too, and summary.json gains der_overlap and ranking_overlap next to der and ranking.
With --jer (needs --ref-rttm) the `full` launch also gives the Jaccard error rate (DESIGN.md section 5.13): summary.json
gains jer per recording and setting and ranking_jer (with overlaps also jer_overlap and ranking_jer_overlap).
With --num-speakers (an integer, a 'recording count' file, or oracle: the reference's speaker count, needs --ref-rttm) or
--min-speakers / --max-speakers, every setting holds each recording to that speaker count (DESIGN.md section 5.14):
summary.json gains count_rule and speakers_vb per recording and setting, and count_rules per setting (how many
recordings took each rule).
With --link-threshold LIST (comma-separated LLR thresholds, the --option=list form when the list starts with '-') the
speakers of every setting are linked across the archive (DESIGN.md sections 5.15 and 5.18): all settings in one batched
vbx_link_batch call, every threshold a host cut of the setting's linkage.  summary.json then gains linked = {threshold:
global_speakers per recording[, der_across_files][, der_across_files_overlap]} per setting and, with a reference,
ranking_across_files (and ranking_across_files_overlap): per protocol, the names <setting>_link<threshold> by DER across
files.  No linked RTTM files are written: the maps and cli --link-threshold at the chosen setting reproduce them.
With --enroll-ark FILE --enroll-utt2spk FILE (both or neither) and --enroll-threshold LIST the speakers of every setting
are named by the enrolled speakers at every threshold (DESIGN.md sections 5.16 and 5.19): all settings in one batched
vbx_enroll_batch call.  summary.json then gains named = {threshold: speaker_names per recording[, der_by_name]
[, der_by_name_overlap]} per setting and, with a reference, ranking_by_name (and ranking_by_name_overlap): per protocol,
the names <setting>_enroll<threshold> by DER by name.  With --cohort-ark FILE --cohort-utt2spk FILE (both or neither;
--cohort-top, default 200) both link and enrolment thresholds are on the normalised score of section 5.17.  No named
RTTM files are written: cli with --enroll-threshold at the chosen setting reproduces them.
With --init RTTM+VB --init-rttm PATH every setting resegments that diarization instead of starting from AHC (DESIGN.md
section 5.20); --threshold must then hold one value.  The RTTM files keep their numbered speakers: cli with --init
RTTM+VB at the chosen setting writes them with the input's speaker names.
With --init RANDOM+VB --init-states N [--restarts R] [--seed S] every setting starts from random responsibilities
instead of AHC (DESIGN.md section 5.22), the same draws for every setting; --threshold and --init-smoothing must then
hold one value each.
With --combine N (the N best settings of ranking['full']; needs --ref-rttm) or --combine all, those settings' outputs are
combined into one by label mapping and weighted voting (DESIGN.md section 5.21): OUT/combined/<recording>.rttm, and
summary.json gains combined = {hypotheses, recordings: {name: order, weights, speakers}[, der][, jer]}, scored under
the same protocols.  Every other key of summary.json is as without --combine.
With --adapt [--recentre] [--adapt-within-scale ...] the back end is adapted to the archive once (DESIGN.md section
5.26), as cli --adapt adapts it, and every setting runs with the adapted model.
"""
import argparse
import itertools
import json
import os
import sys
from collections import namedtuple

import numpy as np

GRID_KEYS = ('Fa', 'Fb', 'loopP', 'threshold', 'smoothing')
BUDGET_FRACTION = 0.5          # default max_batch_bytes: this share of the device memory free at the start


def _fmt(v):
    return f'{float(v):g}'


class Setting(namedtuple('Setting', GRID_KEYS)):
    """One point of the grid."""

    @property
    def name(self):
        """Stable directory name, e.g. Fa0.3_Fb17_loopP0.99_thr-0.015_sm5."""
        return f'Fa{_fmt(self.Fa)}_Fb{_fmt(self.Fb)}_loopP{_fmt(self.loopP)}_thr{_fmt(self.threshold)}_sm{_fmt(self.smoothing)}'


def grid_settings(grid):
    """grid: {'Fa': [...], 'Fb': [...], 'loopP': [...], 'threshold': [...], 'smoothing': [...]} -> list of Setting, the
    product in that key order.  Missing keys, empty lists, Fb = 0, loopP outside [0, 1] or unknown keys raise ValueError."""
    unknown = set(grid) - set(GRID_KEYS)
    if unknown:
        raise ValueError(f'unknown grid keys {sorted(unknown)}; expected {list(GRID_KEYS)}')
    vals = []
    for k in GRID_KEYS:
        v = [float(x) for x in grid.get(k, [])]
        if not v:
            raise ValueError(f'grid[{k!r}] needs at least one value')
        if not all(np.isfinite(v)):
            raise ValueError(f'grid[{k!r}]: values must be finite')
        vals.append(list(dict.fromkeys(v)))         # duplicates would only repeat work
    if any(x == 0 for x in vals[1]):
        raise ValueError('Fb must be non-zero')
    if any(x < 0 or x > 1 for x in vals[2]):
        raise ValueError('loopP must lie in [0, 1]')
    return [Setting(*p) for p in itertools.product(*vals)]


def parse_list(text):
    """'0.3,0.4' -> [0.3, 0.4] (the command line's comma-separated lists)."""
    try:
        out = [float(t) for t in str(text).split(',') if t.strip()]
    except ValueError:
        raise ValueError(f'expected comma-separated numbers, got {text!r}')
    if not out:
        raise ValueError(f'expected comma-separated numbers, got {text!r}')
    return out


def pack(sizes, budget):
    """Entries with byte sizes `sizes`, in order, into consecutive batches whose summed size stays within `budget`.
    Returns a list of lists of entry indices (every entry in exactly one batch).  An entry larger than the budget on its
    own raises ValueError."""
    batches, cur, used = [], [], 0
    for i, sz in enumerate(sizes):
        if sz > budget:
            raise ValueError(f'one entry needs {int(sz)} bytes, more than max_batch_bytes = {int(budget)}')
        if cur and used + sz > budget:
            batches.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += sz
    if cur:
        batches.append(cur)
    return batches


def pack_by(n, size_of, budget):
    """Entries 0 .. n-1, in order, into consecutive batches whose size_of(list of entries) stays within `budget` (for
    workspaces that are not a plain sum of per-entry sizes).  None: one batch.  An entry larger than the budget on its
    own raises ValueError."""
    if budget is None:
        return [list(range(n))] if n else []
    batches, cur = [], []
    for i in range(n):
        if cur and size_of(cur + [i]) <= budget:
            cur.append(i)
            continue
        if size_of([i]) > budget:
            raise ValueError(f'one entry needs {int(size_of([i]))} bytes, more than max_batch_bytes = {int(budget)}')
        if cur:
            batches.append(cur)
        cur = [i]
    if cur:
        batches.append(cur)
    return batches


def entry_bytes(T, n_states, R, device):
    """Device bytes one (recording, setting) entry adds to a float32 batch: its share of the plan's workspace (the larger
    of the split and the fused-sweep plans of the recording alone, which bounds what it adds to any batch), plus its
    replicated rho rows and gamma rows."""
    from .batch import VbxBatch
    from .pipeline import _tier
    ws = 0
    for fb_split in (1, 2) if _tier(n_states) == 0 else (1,):
        vb = VbxBatch([T], R, n_states, device=device, allocate=False, fb_split=fb_split)
        ws = max(ws, vb.workspace_bytes)
        S = vb.S
        vb.close()
    return ws + 4 * T * (R + S)


def packer(lens, R, device, budget):
    """The split of pipeline._vb_stage for a sweep: split(entries, ns) packs a float32 tier's (setting, recording)
    entries with ns[e] states, in order, into consecutive batches of at most `budget` bytes (pack, entry_bytes)."""
    from ._lib import padded_states
    size_cache = {}

    def split(entries, ns):
        sizes = []
        for e in entries:                                     # (setting, recording[, restart])
            key = (int(lens[e[1]]), padded_states(ns[e]))         # the size depends on T and the padded S only
            if key not in size_cache:
                size_cache[key] = entry_bytes(key[0], key[1], R, device)
            sizes.append(size_cache[key])
        return [[entries[i] for i in idx] for idx in pack(sizes, budget)]
    return split


def sweep_batch(recordings, transform, plda, grid, lda_dim=128, max_iters=40, epsilon=1e-6, init='AHC+VB', chain='auto',
                device=None, max_batch_bytes=None, output_2nd=False, ref_rttm=None, uem=None, overlaps=None,
                oracle_overlaps=False, jer=False, num_speakers=None, min_speakers=None, max_speakers=None,
                link_thresholds=None, enroll=None, enroll_thresholds=None, cohort=None, cohort_top=200, init_rttm=None,
                init_states=None, restarts=None, seed=None):
    """Every setting of `grid` (see grid_settings) for every recording, with the front end and AHC run once.

    recordings, transform, plda, lda_dim, max_iters, epsilon, init, chain, output_2nd: as for pipeline.diarize_batch.
    Entries (recording, setting) are grouped into diarize_batch's state tiers (<= 64, 65 .. 128 AHC clusters: float32
    batches with per-recording Fa / Fb / loopP, numbers when the grid has one setting, packed into as few batches as fit
    max_batch_bytes, default half of the free device memory; more than 128: one float64 run per setting), all in
    pipeline._vb_stage.
    ref_rttm: None, or the reference as an RTTM path (file or directory of *.rttm) or formats.read_rttm rows; uem: None,
    a UEM path or formats.read_uem's dict.  With a reference every (setting, recording) entry is scored after all batches
    have run, in one vbx_score launch per protocol (score.PROTOCOLS), and each recording's dict gains
    der = {protocol: score.result dict}.  A recording that the reference (or the UEM) lacks raises ValueError before any
    work; reference recordings that `recordings` lacks are ignored.
    overlaps: None or {recording: [(onset, offset)] seconds} (score.read_overlaps); oracle_overlaps: use the time in which
    the reference has two or more speakers instead (needs ref_rttm).  Either makes each recording's dict also hold
    rttm_overlap and overlap_seconds as diarize_batch(overlaps=) does and, with a reference, der_overlap = {protocol:
    score.result dict} of that output, scored in one more vbx_score_overlap launch per protocol.  Needs init='AHC+VB'.
    jer: also the Jaccard error rate, from the `full` protocol's launch (no extra launch): items gain jer (and with
    overlaps jer_overlap) = score.jer_finish dict.  Needs ref_rttm.
    num_speakers / min_speakers / max_speakers: a known or bounded speaker count per recording, as for
    pipeline.diarize_batch, the same for every setting; num_speakers='oracle' takes each recording's number of reference
    speakers with scored time (needs ref_rttm; inside the UEM when one is given).  Every (recording, setting) entry then
    follows the rules of DESIGN.md section 5.14 and its dict gains count_rule, n_speakers_vb and count.  The re-runs of
    rule 3 of all settings are packed into batches per state tier like the first pass.
    link_thresholds: None, or LLR thresholds for speaker linking across the archive (DESIGN.md sections 5.15 and 5.18;
    each checked by link.check_threshold before any device work, duplicates dropped).  The final first labels of every
    setting are linked in one link.link_many call within max_batch_bytes, and each threshold is a host cut of the
    setting's linkage (link.link_cut, second labels as diarize_batch handles them).  Each recording's dict gains
    global_speakers = {threshold: {label: global id}}, equal to diarize_batch(link_threshold=threshold)'s with that
    setting's scalars; with a reference also ref_speakers (the reference speaker names, in the rows of the blocks) and
    der_blocks = {protocol: overlap block} (with overlaps der_overlap_blocks too), what summarize_across_files needs.
    enroll, enroll_thresholds: None, or known speakers {name: raw x-vectors [n, Dx]} as for diarize_batch and a list of
    LLR thresholds (DESIGN.md sections 5.16 and 5.19; each checked by enroll.check_threshold before any device work,
    duplicates dropped; there is no default).  The enrolled x-vectors go through the front end once; the final first
    labels of every setting are scored against them in one enroll.enroll_many call within max_batch_bytes, each
    setting's LLR block assigned at every threshold.  Each recording's dict gains speaker_names = {threshold: {label:
    name}} and speaker_llr = {threshold: {label: llr}}, equal to diarize_batch(enroll_threshold=threshold)'s with that
    setting's scalars (unknown speakers are unknown-<recording>-<label + 1>: with link_thresholds as well, linking and
    enrolment are each what diarize_batch gives with that option alone), and with a reference ref_speakers and
    der_blocks as for linking (what summarize_by_name needs).
    cohort, cohort_top: None, or a cohort {name: raw x-vectors [n, Dx]} as for diarize_batch (section 5.17; needs
    link_thresholds or enroll).  Its statistics for every setting's speakers (and enrolled speakers) come from batched
    cohort.cohort_stats_many calls; a speaker without spread raises ValueError naming the setting and the speaker before
    any linking or enrolment kernel runs.  link_thresholds and enroll_thresholds are then on the normalised score S,
    every dict gains score_norm, and with enroll speaker_score replaces speaker_llr.
    init='RTTM+VB', init_rttm: VB resegmentation as for diarize_batch (DESIGN.md section 5.20).  The init turns are read
    and checked once and packed for every batch; each entry starts from its recording's turns with its setting's
    smoothing.  The grid's threshold axis has no effect then and must hold exactly one value (ValueError otherwise).
    Each dict gains init_speakers and rttm_init; the written RTTM files keep their numbered speakers.
    init='RANDOM+VB', init_states, restarts, seed: random starts as for diarize_batch (DESIGN.md section 5.22), the same
    for every setting: every (setting, recording, restart) is one entry of the tiers and packing, and each (setting,
    recording) keeps its restart of largest final ELBO.  The grid's threshold and smoothing axes have no effect then and
    must each hold exactly one value (ValueError otherwise).  Each dict gains restart, init_seed, elbo and restart_elbos.
    Returns {Setting: {recording: dict(rttm, labels, labels2nd, n_speakers, iterations, flags[, der][, rttm_overlap,
    overlap_seconds][, der_overlap][, count_rule, n_speakers_vb, count][, global_speakers][, speaker_names, speaker_llr
    or speaker_score][, score_norm][, ref_speakers, der_blocks[, der_overlap_blocks]])}}; each recording's dict is the
    one diarize_batch returns with that setting's scalars."""
    import torch
    from . import ahc as _ahc
    from ._lib import VbxError
    from .parts import make_batch
    from .pipeline import (_check_init, _count_fields, _front_end, _pad_features, _result, _side_features, _vb_stage,
                           count_bounds, init_fields, restart_fields)
    settings = grid_settings(grid)
    links = check_link_thresholds(link_thresholds)
    dims = {int(np.asarray(r[0]).shape[1]) for r in recordings.values()}
    dim = next(iter(dims)) if len(dims) == 1 else -1
    enrolled, enroll_thr = check_enroll_options(enroll, enroll_thresholds, dim)
    cohort_set = None
    if cohort is not None:
        from . import cohort as _cohort
        if links is None and enrolled is None:
            raise ValueError('a cohort normalises the linking and enrolment scores: it needs link_thresholds or enroll')
        _cohort.check_top_k(cohort_top)
        cohort_set = _cohort.check_cohort(cohort, dim)
    with_overlap = oracle_overlaps or overlaps is not None
    random = _check_init(init, with_overlap, init_rttm, init_states, restarts, seed)
    if random is not None:
        for axis in ('threshold', 'smoothing'):
            if len({getattr(s, axis) for s in settings}) != 1:
                raise ValueError(f"init='RANDOM+VB' runs no AHC threshold cut and no smoothed init: the grid's {axis} "
                                 'axis must hold one value')
    init_from = None                                         # (seg_times, init speakers) per recording
    if init == 'RTTM+VB':
        from .resegment import load_init
        if len({s.threshold for s in settings}) != 1:
            raise ValueError("init='RTTM+VB' runs no AHC threshold cut: the grid's threshold axis must hold one value")
        init_turns = load_init(init_rttm, list(recordings))
        init_from = [(recordings[n][1], init_turns[n]) for n in recordings]
    if oracle_overlaps and ref_rttm is None:
        raise ValueError('oracle_overlaps are the overlaps of the reference: they need ref_rttm')
    if oracle_overlaps and overlaps is not None:
        raise ValueError('give overlaps or oracle_overlaps, not both')
    if jer and ref_rttm is None:
        raise ValueError('jer scores against the reference: it needs ref_rttm')
    oracle_count = isinstance(num_speakers, str)
    if oracle_count and num_speakers != 'oracle':
        raise ValueError(f"num_speakers: expected an int, a dict or 'oracle', got {num_speakers!r}")
    if oracle_count and ref_rttm is None:
        raise ValueError("num_speakers='oracle' counts the reference's speakers: it needs ref_rttm")
    if oracle_count and (min_speakers is not None or max_speakers is not None):
        raise ValueError('give num_speakers or min_speakers / max_speakers, not both')
    bounds = None if oracle_count else count_bounds(list(recordings), num_speakers, min_speakers, max_speakers)
    if not torch.cuda.is_available():
        raise VbxError('sweep_batch(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    names = list(recordings)
    if uem is not None and ref_rttm is None:
        raise ValueError('uem restricts the scored time: it needs ref_rttm')
    ref = _load_reference(names, ref_rttm, uem) if ref_rttm is not None else None
    if oracle_count:
        from .score import reference_speaker_counts
        num_speakers = reference_speaker_counts({n: ref[0][n] for n in names}, ref[1])
        empty = [n for n in names if num_speakers[n] < 1]
        if empty:
            raise ValueError(f'recordings without scored reference speech have no oracle speaker count: {empty}')
        bounds = count_bounds(names, num_speakers, min_speakers, max_speakers)
    if not names:
        return {s: {} for s in settings}
    lens = np.array([np.asarray(recordings[n][0]).shape[0] for n in names], dtype=np.int64)
    with_ahc = init in ('AHC', 'AHC+VB') or bounds is not None     # other inits: the AHC linkage serves rule 3 only
    fea, Phi, _, th, Zs = _front_end(recordings, names, lens, transform, plda, lda_dim, chain, dev, 0.0, ahc=with_ahc)
    fea, Phi = _pad_features(fea, Phi)
    thresholds = list(dict.fromkeys(s.threshold for s in settings))
    ahc_labels = lab_d = {t: None for t in thresholds}
    if init in ('AHC', 'AHC+VB'):
        ahc_labels = {t: _ahc.cut(Zs, th, lens, t) for t in thresholds}              # VBx/vbhmm.py:144-146, host only
        lab_d = {t: torch.from_numpy(np.concatenate(ahc_labels[t])).to(dev) for t in thresholds}
    if max_batch_bytes is None:
        max_batch_bytes = int(torch.cuda.mem_get_info(dev)[0] * BUDGET_FRACTION)
    if random is not None:
        from .random_init import name_key
        random = random._replace(keys=[name_key(n) for n in names])
    # per (setting, recording): labels, labels2nd, iterations, flags[, unconstrained count, rule]
    res = _vb_stage([(s.Fa, s.Fb, s.loopP, s.smoothing) for s in settings], [ahc_labels[s.threshold] for s in settings],
                    [lab_d[s.threshold] for s in settings], Zs, lens, fea, Phi, bounds, init, dev, make_batch,
                    packer(lens, int(fea.shape[1]), dev, max_batch_bytes), turns=init_from, random=random,
                    maxIters=max_iters, epsilon=epsilon)
    maps = named = norm = None
    if links is not None or enrolled is not None:
        offs = np.concatenate([[0], np.cumsum(lens)])
        labels = [[res[(k, b)][0] for b in range(len(names))] for k in range(len(settings))]
        Fa, Fb = [s.Fa for s in settings], [s.Fb for s in settings]
        side = lambda sets: _side_features(sets, recordings, names, transform, plda, lda_dim, chain, dev, fea, Phi)
        enrolled_fea = side(enrolled) if enrolled is not None else None
        if cohort_set is not None:
            norm = _cohort_norm_many(side(cohort_set), cohort_top, settings, enrolled, enrolled_fea, names, fea, Phi,
                                     offs, labels, dev, max_batch_bytes)
    if links is not None:
        from . import link
        linked = link.link_many(fea, Phi, offs, labels, Fa, Fb, dev, max_batch_bytes,
                                norm=None if norm is None else [st[:2] for st in norm['archive']])
        maps = [{t: link.link_cut(Z, table, t, [res[(k, b)][1] for b in range(len(names))]) for t in links}
                for k, (table, _, _, Z) in enumerate(linked)]
    if enrolled is not None:
        from . import enroll as _enroll
        en_norm = None if norm is None else [tuple(a[:2]) + tuple(e[:2]) for a, e in zip(norm['archive'],
                                                                                          norm['enrolled'])]
        en = _enroll.enroll_many(fea, Phi, offs, labels, enrolled_fea[0], enrolled_fea[1], Fa, Fb, enroll_thr, dev,
                                 max_bytes=max_batch_bytes, norm=en_norm)
        enrolled_names = [k for k, _ in enrolled]
        named = [{t: _enroll.enroll_names(r.table, r.assign[h], r.best_llr[h], enrolled_names, names,
                                          [res[(k, b)][1] for b in range(len(names))])
                  for h, t in enumerate(enroll_thr)} for k, r in enumerate(en)]
    from . import score
    ovl = [None] * len(names)
    if with_overlap:
        ovl = [score.oracle_overlaps(ref[0][n]) if oracle_overlaps else score.overlap_ticks(overlaps.get(n))
               for n in names]
    der = der_ovl = None
    if ref is not None:
        turns, uem_map = ref[:2]
        scored = []
        for n, o in zip(names, ovl):
            timeline = score.owned_intervals(recordings[n][1])
            scored.append(score.prepare_recording(n, turns[n], timeline, None if uem_map is None else uem_map[n],
                                                  overlap=o))
        keys = [(k, b) for k in range(len(settings)) for b in range(len(names))]
        jp = 'full' if jer else None
        blk = maps is not None or named is not None
        der = dict(zip(keys, score.score_entries(scored, [(b, res[(k, b)][0]) for k, b in keys], device=dev, jer=jp,
                                                 blocks=blk)))
        if with_overlap:
            der_ovl = dict(zip(keys, score.score_entries(scored, [(b, res[(k, b)][0], res[(k, b)][1]) for k, b in keys],
                                                         device=dev, jer=jp, blocks=blk)))
    out = {}
    for k, s in enumerate(settings):
        out[s] = {}
        for b, n in enumerate(names):
            l1, l2, it, fl = res[(k, b)][:4]
            item = _result(n, recordings[n][1], l1, l2, it, output_2nd, ovl[b])
            item['flags'] = int(fl)
            if bounds is not None:
                _count_fields(item, *res[(k, b)][4:6], bounds[0][b], bounds[1][b])
            if der is not None:
                item['der'] = {p: v for p, v in der[(k, b)].items() if p not in ('jer', 'O')}
                if jer:
                    item['jer'] = der[(k, b)]['jer']
            if der_ovl is not None:
                item['der_overlap'] = {p: v for p, v in der_ovl[(k, b)].items() if p not in ('jer', 'O')}
                if jer:
                    item['jer_overlap'] = der_ovl[(k, b)]['jer']
            if maps is not None:
                item['global_speakers'] = {t: maps[k][t][b] for t in links}
            if named is not None:
                item['speaker_names'] = {t: named[k][t][0][b] for t in enroll_thr}
                item['speaker_llr' if norm is None else 'speaker_score'] = {t: named[k][t][1][b] for t in enroll_thr}
            if norm is not None:
                item['score_norm'] = {'top_k': norm['K'], 'cohort_speakers': norm['C']}
            if init_from is not None:
                init_fields(item, n, recordings[n][1], l1, l2, init_from[b][1],
                            None if bounds is None else res[(k, b)][5], ovl[b])
            if random is not None:
                restart_fields(item, random.seed, *res[(k, b)][-1])
            if (maps is not None or named is not None) and der is not None:
                item['ref_speakers'] = ref[2][n]
                item['der_blocks'] = der[(k, b)]['O']
                if der_ovl is not None:
                    item['der_overlap_blocks'] = der_ovl[(k, b)]['O']
            out[s][n] = item
    return out


def check_link_thresholds(thresholds):
    """None, or the link thresholds as floats without duplicates (first occurrence kept).  A threshold that
    link.check_threshold refuses, or an empty list, raises ValueError."""
    if thresholds is None:
        return None
    from .link import check_threshold
    out = list(dict.fromkeys(check_threshold(t) for t in thresholds))
    if not out:
        raise ValueError('link_thresholds needs at least one value')
    return out


def check_enroll_options(enroll, thresholds, dim):
    """(enroll.check_enrolment's list or None, the enrolment thresholds or None) of sweep_batch's enroll and
    enroll_thresholds: both or neither; the thresholds as enroll.check_thresholds takes them (duplicates dropped), and
    no two with the same name f'{t:g}' (enroll_key), which would share one entry of the rankings."""
    if enroll is None and thresholds is None:
        return None, None
    if enroll is None:
        raise ValueError('enroll_thresholds without enroll')
    if thresholds is None:
        raise ValueError('enroll needs enroll_thresholds: the LLR is not calibrated, so there is no default')
    from . import enroll as _enroll
    thr = _enroll.check_thresholds(thresholds)
    names = {}
    for t in thr:                                     # their name in enroll_key and summary.json
        if names.setdefault(f'{t:g}', t) != t:
            raise ValueError(f'enrolment thresholds {names[f"{t:g}"]!r} and {t!r} have the same name {t:g} in the '
                             'rankings and summary.json: give thresholds that differ in their first 6 significant digits')
    return _enroll.check_enrolment(enroll, dim), thr


def _cohort_norm_many(cohort_fea, top_k, settings, enrolled, enrolled_fea, names, fea, Phi, offs, labels, dev,
                      max_bytes):
    """DESIGN.md sections 5.17 and 5.19 for sweep_batch: the cohort statistics of every setting's speakers and of the
    enrolled speakers under every setting's scalars, in batched cohort.cohort_stats_many calls, each checked for spread
    per setting (ValueError naming the setting and the speaker, before any linking or enrolment kernel).  Returns
    dict(archive: [CohortStats] per setting, enrolled: [CohortStats] per setting or None, K, C)."""
    from . import cohort as _cohort
    from .link import speaker_table
    fea_c, spk_c = cohort_fea
    Fa, Fb = [s.Fa for s in settings], [s.Fb for s in settings]
    arch = _cohort.cohort_stats_many(fea, Phi, offs, labels, fea_c, spk_c, Fa, Fb, top_k, dev, max_bytes)
    for s, st, l1 in zip(settings, arch, labels):
        t = speaker_table(l1)
        _cohort.check_spread(st.std, [f'setting {s.name}: {names[b]} speaker {l + 1}'
                                      for b, l in zip(t.rec.tolist(), t.label.tolist())])
    enr = None
    if enrolled is not None:
        enr = _cohort.cohort_stats_many(enrolled_fea[0], Phi, None, [enrolled_fea[1]] * len(settings), fea_c, spk_c,
                                        Fa, Fb, top_k, dev, max_bytes)
        for s, st in zip(settings, enr):
            _cohort.check_spread(st.std, [f'setting {s.name}: enrolled {k}' for k, _ in enrolled])
    return dict(archive=arch, enrolled=enr, K=min(top_k, int(spk_c.max()) + 1), C=int(spk_c.max()) + 1)


def _load_reference(names, ref_rttm, uem):
    """-> (score.reference_turns of the recordings `names`, {recording: UEM intervals} or None, {recording: the
    reference speaker names in the order of the turns}), checked up front."""
    from . import formats, score
    rows = score.read_rttm_path(ref_rttm) if isinstance(ref_rttm, (str, os.PathLike)) else list(ref_rttm)
    wanted = set(names)
    named = score.named_reference_turns([r for r in rows if r[0] in wanted])
    turns = {rec: [t for _, t in spk] for rec, spk in named.items()}
    missing = [n for n in names if n not in turns]
    if missing:
        raise ValueError(f'recordings missing from the reference RTTM: {missing}')
    if isinstance(uem, (str, os.PathLike)):
        uem = formats.read_uem(uem)
    if uem is not None:
        missing = [n for n in names if n not in uem]
        if missing:
            raise ValueError(f'recordings missing from the UEM: {missing}')
    return turns, uem, {rec: [k for k, _ in spk] for rec, spk in named.items()}


def summarize_der(out, key='der'):
    """sweep_batch output with `key` ('der' or 'der_overlap') -> ({setting name: {protocol: overall result dict}},
    {protocol: setting names by overall DER, stable in grid order})."""
    from . import score
    tot = {s.name: {p: score.overall([item[key][p] for item in per_rec.values()]) for p, _, _ in score.PROTOCOLS}
           for s, per_rec in out.items()}
    ranking = {p: score.rank({n: tot[n][p] for n in tot}) for p, _, _ in score.PROTOCOLS}
    return tot, ranking


def link_key(setting, threshold):
    """The ranking name of a setting linked at a threshold, e.g. Fa0.3_Fb17_loopP0.99_thr-0.015_sm5_link48."""
    return f'{setting.name}_link{threshold:g}'


def across_files_by_id(tot, ref_names, blocks, maps):
    """DER across files (DESIGN.md section 5.15) of linked output: tot, an overall() result of the files; per file the
    reference names of its block rows, its overlap block [n_ref, labels] and its {label: global id} map.  The blocks'
    columns are summed by global id (a label the map lacks has no turns, so its column is empty) and matched once,
    as score.across_files_result does with RTTM names."""
    from scipy.optimize import linear_sum_assignment
    from . import score
    rows = {k: i for i, k in enumerate(sorted({k for ks in ref_names for k in ks}))}
    n_ids = 1 + max((g for m in maps for g in m.values()), default=-1)
    O = np.zeros((len(rows), n_ids), dtype=np.int64)
    for rk, blk, m in zip(ref_names, blocks, maps):
        blk = np.asarray(blk, dtype=np.int64)
        cols = [l for l in range(blk.shape[1]) if l in m]
        if rk and cols:
            np.add.at(O, np.ix_([rows[k] for k in rk], [m[l] for l in cols]), blk[:, cols])
    matched = 0
    if O.size:
        r, c = linear_sum_assignment(O, maximize=True)
        matched = int(O[r, c].sum())
    t = tot['ticks']
    return score.result(t['miss'], t['fa'], t['scored'] - t['miss'] - matched, t['scored'])


def summarize_across_files(out, key='der'):
    """sweep_batch(link_thresholds=, ref_rttm=) output with `key` ('der' or 'der_overlap') -> ({link_key(setting,
    threshold): {protocol: DER across files}}, {protocol: those names by DER across files, stable in grid order, then
    threshold order}).  Per (setting, threshold) the per-file blocks are summed by global id and matched once
    (across_files_by_id)."""
    from . import score
    tot = {}
    for s, per_rec in out.items():
        items = list(per_rec.values())
        if not items:
            continue
        for t in items[0]['global_speakers']:
            tot[link_key(s, t)] = {
                p: across_files_by_id(score.overall([it[key][p] for it in items]), [it['ref_speakers'] for it in items],
                                      [it[key + '_blocks'][p] for it in items], [it['global_speakers'][t] for it in items])
                for p, _, _ in score.PROTOCOLS}
    ranking = {p: score.rank({n: tot[n][p] for n in tot}) for p, _, _ in score.PROTOCOLS}
    return tot, ranking


def enroll_key(setting, threshold):
    """The ranking name of a setting named at an enrolment threshold, e.g. Fa0.3_Fb17_loopP0.99_thr-0.015_sm5_enroll20."""
    return f'{setting.name}_enroll{threshold:g}'


def summarize_by_name(out, key='der'):
    """sweep_batch(enroll=, enroll_thresholds=, ref_rttm=) output with `key` ('der' or 'der_overlap') -> ({enroll_key(
    setting, threshold): {protocol: DER by name}}, {protocol: those names by DER by name, stable in grid order, then
    threshold order}).  Per (setting, threshold) each file's block columns (one per label) take the labels' names and
    score.by_name_result sums them by name: host work only, no assignment is solved."""
    from . import score
    from .enroll import UNKNOWN
    tot = {}
    for s, per_rec in out.items():
        if not per_rec:
            continue
        items = list(per_rec.values())
        for t in items[0]['speaker_names']:
            cols = []
            for rec, it in per_rec.items():
                m = it['speaker_names'][t]
                n_cols = max((np.asarray(it[key + '_blocks'][p]).shape[1] for p, _, _ in score.PROTOCOLS), default=0)
                cols.append([m.get(l, f'{UNKNOWN}{rec}-{l + 1}') for l in range(n_cols)])    # a label without turns
            tot[enroll_key(s, t)] = {
                p: score.by_name_result(score.overall([it[key][p] for it in items]), [it['ref_speakers'] for it in items],
                                        cols, [it[key + '_blocks'][p] for it in items])
                for p, _, _ in score.PROTOCOLS}
    ranking = {p: score.rank({n: tot[n][p] for n in tot}) for p, _, _ in score.PROTOCOLS}
    return tot, ranking


def summarize_jer(out, key='jer'):
    """sweep_batch(jer=True) output with `key` ('jer' or 'jer_overlap') -> ({setting name: score.overall_jer dict},
    setting names by overall JER, stable in grid order, settings without a JER last)."""
    from . import score
    tot = {s.name: score.overall_jer([item[key] for item in per_rec.values()]) for s, per_rec in out.items()}
    return tot, score.rank(tot, key='jer')


def combine_settings(out, recordings, settings=None, weights=None, device=None):
    """Combine the outputs of several settings of sweep_batch's return value `out` into one diarization per recording
    (DESIGN.md section 5.21), in one vbx_combine call over all recordings.  recordings: the dict sweep_batch was given
    (its segment times are the shared intervals, score.owned_intervals, so no timeline union is needed); settings: the
    Settings to combine, in the order that breaks ties (None: all, in grid order), 2 .. 32 of them; weights: None (rank
    ** -0.1 per recording) or one per setting.  Each setting votes with its first labels: labels2nd is its second most
    likely speaker of every x-vector, not a claim that two people speak, and as a second label it would vote for a second
    speaker everywhere.  Returns {recording: dict(rttm, labels, n_speakers, order (indices into settings), weights, D,
    map, n_global)}."""
    from . import combine, score
    from .pipeline import merge_adjacent_labels, rttm_lines
    settings = list(out) if settings is None else list(settings)
    missing = [s for s in settings if s not in out]
    if missing:
        raise ValueError(f'settings the sweep did not run: {[getattr(s, "name", s) for s in missing]}')
    if not 2 <= len(settings) <= combine.MAX_HYPOTHESES:
        raise ValueError(f'{len(settings)} settings: combination takes 2 .. {combine.MAX_HYPOTHESES}')
    names = list(out[settings[0]])
    intervals = [score.owned_intervals(recordings[n][1])[:2] for n in names]
    hyps = [[(out[s][n]['labels'], None) for n in names] for s in settings]
    res = combine.combine_labels(intervals, hyps, weights, device)
    comb = {}
    for n, item in zip(names, res):
        seg = np.asarray(recordings[n][1], dtype=np.float64).reshape(-1, 2)
        lines = rttm_lines(n, *merge_adjacent_labels(seg[:, 0], seg[:, 1], item['labels']))
        comb[n] = dict(rttm=lines, labels=item['labels'], n_speakers=int(len(set(item['labels'].tolist()))),
                       order=item['order'], weights=item['weights'], D=item['D'], map=item['map'],
                       n_global=item['n_global'])
    return comb


def score_combined(comb, recordings, ref_rttm, uem=None, jer=False, device=None):
    """The DER (and JER) of combine_settings' output under score.PROTOCOLS, as sweep_batch scores a setting: ({protocol:
    overall result dict}, overall JER dict or None)."""
    from . import score
    names = list(comb)
    turns, uem_map, _ = _load_reference(names, ref_rttm, uem)
    scored = [score.prepare_recording(n, turns[n], score.owned_intervals(recordings[n][1]),
                                      None if uem_map is None else uem_map[n]) for n in names]
    res = score.score_entries(scored, [(b, comb[n]['labels']) for b, n in enumerate(names)], device=device,
                              jer='full' if jer else None)
    der = {p: score.overall([r[p] for r in res]) for p, _, _ in score.PROTOCOLS}
    return der, score.overall_jer([r['jer'] for r in res]) if jer else None


def parse_combine(text):
    """--combine: 'all' or an integer >= 2."""
    if str(text) == 'all':
        return 'all'
    try:
        n = int(text)
    except ValueError:
        n = 0
    if n < 2:
        raise argparse.ArgumentTypeError(f"expected 'all' or an integer >= 2, got {text!r}")
    return n


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--combine', default=None, type=parse_combine,
                    help="combine the N best settings (needs --ref-rttm), or 'all', into OUT/combined/*.rttm")
    ap.add_argument('--init', default='AHC+VB', choices=['AHC', 'AHC+VB', 'RTTM+VB', 'RANDOM+VB'])
    ap.add_argument('--init-rttm', default=None,
                    help='with --init RTTM+VB: the diarization (RTTM file or directory of *.rttm) the VB-HMM starts from')
    ap.add_argument('--out-dir', required=True, type=str)
    ap.add_argument('--xvec-ark-file', required=True, type=str)
    ap.add_argument('--segments-file', required=True, type=str)
    ap.add_argument('--xvec-transform', required=True, type=str)
    ap.add_argument('--plda-file', required=True, type=str)
    ap.add_argument('--lda-dim', required=True, type=int)
    ap.add_argument('--Fa', required=True, type=parse_list, help='comma-separated values')
    ap.add_argument('--Fb', required=True, type=parse_list, help='comma-separated values')
    ap.add_argument('--loopP', required=True, type=parse_list, help='comma-separated values')
    ap.add_argument('--threshold', required=True, type=parse_list, help='comma-separated values')
    ap.add_argument('--init-smoothing', default=[5.0], type=parse_list, help='comma-separated values')
    ap.add_argument('--max-iters', default=40, type=int)
    ap.add_argument('--epsilon', default=1e-6, type=float)
    ap.add_argument('--chain', default='auto', choices=['auto', 'tcgen05', 'float64'])
    ap.add_argument('--device', default=None, help='CUDA device, e.g. cuda:0 (default: the current device)')
    ap.add_argument('--max-batch-bytes', default=None, type=int)
    ap.add_argument('--ref-rttm', default=None, help='reference RTTM file or directory of *.rttm: score every setting')
    ap.add_argument('--uem', default=None, help='UEM file restricting the scored time (with --ref-rttm)')
    ap.add_argument('--overlap-rttm', default=None,
                    help='overlap regions (RTTM file or directory): also write and score overlap-aware output')
    ap.add_argument('--oracle-overlaps', action='store_true',
                    help="use the reference's overlaps (with --ref-rttm) as the overlap regions")
    ap.add_argument('--jer', action='store_true', help='also score and rank by Jaccard error rate (with --ref-rttm)')
    ap.add_argument('--link-threshold', default=None, type=parse_list,
                    help='comma-separated LLR thresholds: link every setting\'s speakers across the archive')
    ap.add_argument('--enroll-ark', default=None, help='x-vectors of known speakers (Kaldi ark) to name speakers by')
    ap.add_argument('--enroll-utt2spk', default=None, help='the speaker of each x-vector of --enroll-ark (utt2spk)')
    ap.add_argument('--enroll-threshold', default=None, type=parse_list,
                    help='comma-separated LLR thresholds at which a speaker takes an enrolled name')
    ap.add_argument('--cohort-ark', default=None,
                    help='x-vectors of cohort speakers (Kaldi ark), none of them in the archive, to normalise the '
                         'linking and enrolment scores by')
    ap.add_argument('--cohort-utt2spk', default=None, help='the speaker of each x-vector of --cohort-ark (utt2spk)')
    ap.add_argument('--cohort-top', default=200, type=int,
                    help="how many of each speaker's largest cohort scores set its mean and spread (default 200)")
    from .cli import add_adapt_options, add_count_options, add_random_options
    add_count_options(ap, allow_oracle=True)
    add_random_options(ap)
    add_adapt_options(ap)
    return ap


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if (args.enroll_ark is None) != (args.enroll_utt2spk is None):
        ap.error('--enroll-ark and --enroll-utt2spk go together')
    if (args.cohort_ark is None) != (args.cohort_utt2spk is None):
        ap.error('--cohort-ark and --cohort-utt2spk go together')
    if (args.init == 'RTTM+VB') != (args.init_rttm is not None):
        ap.error('--init RTTM+VB and --init-rttm go together')
    from .cli import check_adapt_options, check_random_options
    check_random_options(ap, args)
    scales = check_adapt_options(ap, args)
    if isinstance(args.combine, int) and args.ref_rttm is None:
        ap.error('--combine N takes the N best settings by DER: it needs --ref-rttm (or --combine all)')
    from . import formats
    segs = formats.read_segments(args.segments_file)
    plda = formats.read_kaldi_plda(args.plda_file)
    transform = formats.read_xvec_transform(args.xvec_transform)
    recs = {}
    for name, (keys, x) in formats.read_xvectors_by_recording(args.xvec_ark_file).items():
        seg_names, times = segs[name]
        assert np.all(np.array(seg_names) == np.array(keys))
        recs[name] = (x, times)
    if scales is not None:      # adapted once; every setting runs with the adapted model
        from .adapt import adapt_backend
        transform, plda, _ = adapt_backend(recs, transform, plda, lda_dim=args.lda_dim, chain=args.chain,
                                           device=args.device, recentre=args.recentre, **scales)
    from .score import read_overlaps
    overlaps = read_overlaps(args.overlap_rttm) if args.overlap_rttm is not None else None
    grid = dict(Fa=args.Fa, Fb=args.Fb, loopP=args.loopP, threshold=args.threshold, smoothing=args.init_smoothing)
    out = sweep_batch(recs, transform, plda, grid, lda_dim=args.lda_dim, max_iters=args.max_iters, epsilon=args.epsilon,
                      init=args.init, chain=args.chain, device=args.device, max_batch_bytes=args.max_batch_bytes,
                      ref_rttm=args.ref_rttm, uem=args.uem, overlaps=overlaps, oracle_overlaps=args.oracle_overlaps,
                      jer=args.jer, num_speakers=args.num_speakers, min_speakers=args.min_speakers,
                      max_speakers=args.max_speakers, link_thresholds=args.link_threshold,
                      enroll=formats.read_enrolment(args.enroll_ark, args.enroll_utt2spk) if args.enroll_ark else None,
                      enroll_thresholds=args.enroll_threshold,
                      cohort=formats.read_enrolment(args.cohort_ark, args.cohort_utt2spk) if args.cohort_ark else None,
                      cohort_top=args.cohort_top, init_rttm=args.init_rttm, init_states=args.init_states,
                      restarts=args.restarts, seed=args.seed)
    summary = {}
    for s, per_rec in out.items():
        d = os.path.join(args.out_dir, s.name)
        os.makedirs(d, exist_ok=True)
        summary[s.name] = dict(setting=s._asdict(), recordings={})
        for name, item in per_rec.items():
            with open(os.path.join(d, f'{name}.rttm'), 'w') as fp:
                fp.write(''.join(line + os.linesep for line in item['rttm']))
            summary[s.name]['recordings'][name] = dict(speakers=item['n_speakers'], iterations=item['iterations'],
                                                       flags=item['flags'])
            for key in ('der', 'der_overlap', 'overlap_seconds', 'jer', 'jer_overlap', 'count_rule', 'restart',
                        'init_seed'):
                if key in item:
                    summary[s.name]['recordings'][name][key] = item[key]
            if 'count_rule' in item:
                summary[s.name]['recordings'][name]['speakers_vb'] = item['n_speakers_vb']
                rules = summary[s.name].setdefault('count_rules', {})
                rules[item['count_rule']] = rules.get(item['count_rule'], 0) + 1
            if 'rttm_overlap' in item:
                os.makedirs(os.path.join(d, 'overlap'), exist_ok=True)
                with open(os.path.join(d, 'overlap', f'{name}.rttm'), 'w') as fp:
                    fp.write(''.join(line + os.linesep for line in item['rttm_overlap']))
    if args.ref_rttm is not None:
        tot, summary['ranking'] = summarize_der(out)
        for name, d in tot.items():
            summary[name]['der'] = d
        if overlaps is not None or args.oracle_overlaps:
            tot, summary['ranking_overlap'] = summarize_der(out, 'der_overlap')
            for name, d in tot.items():
                summary[name]['der_overlap'] = d
        if args.jer:
            for key in ('jer', 'jer_overlap') if overlaps is not None or args.oracle_overlaps else ('jer',):
                tot, summary['ranking_' + key] = summarize_jer(out, key)
                for name, d in tot.items():
                    summary[name][key] = d
    if args.link_threshold is not None:
        ovl = overlaps is not None or args.oracle_overlaps
        for s, per_rec in out.items():
            linked = summary[s.name]['linked'] = {}
            for t in check_link_thresholds(args.link_threshold):
                linked[f'{t:g}'] = dict(global_speakers={n: it['global_speakers'][t] for n, it in per_rec.items()})
        if args.ref_rttm is not None:
            for key in ('der', 'der_overlap') if ovl else ('der',):
                tot, summary['ranking_across_files' + key[3:]] = summarize_across_files(out, key)
                for s in out:
                    for t in check_link_thresholds(args.link_threshold):
                        summary[s.name]['linked'][f'{t:g}']['der_across_files' + key[3:]] = tot[link_key(s, t)]
    if args.enroll_threshold is not None:
        ovl = overlaps is not None or args.oracle_overlaps
        thr = list(dict.fromkeys(args.enroll_threshold))
        for s, per_rec in out.items():
            summary[s.name]['named'] = {f'{t:g}': dict(speaker_names={n: it['speaker_names'][t]
                                                                        for n, it in per_rec.items()}) for t in thr}
        if args.ref_rttm is not None:
            for key in ('der', 'der_overlap') if ovl else ('der',):
                tot, summary['ranking_by_name' + key[3:]] = summarize_by_name(out, key)
                for s in out:
                    for t in thr:
                        summary[s.name]['named'][f'{t:g}']['der_by_name' + key[3:]] = tot[enroll_key(s, t)]
    if args.combine is not None:
        by_name = {s.name: s for s in out}
        chosen = list(out) if args.combine == 'all' else [by_name[n] for n in summary['ranking']['full'][:args.combine]]
        comb = combine_settings(out, recs, chosen, device=args.device)
        os.makedirs(os.path.join(args.out_dir, 'combined'), exist_ok=True)
        block = summary['combined'] = dict(hypotheses=[s.name for s in chosen], recordings={})
        for name, item in comb.items():
            with open(os.path.join(args.out_dir, 'combined', f'{name}.rttm'), 'w') as fp:
                fp.write(''.join(line + os.linesep for line in item['rttm']))
            block['recordings'][name] = dict(order=item['order'], weights=[float(w) for w in item['weights']],
                                             speakers=item['n_speakers'])
        if args.ref_rttm is not None:
            block['der'], jer_tot = score_combined(comb, recs, args.ref_rttm, args.uem, args.jer, args.device)
            if args.jer:
                block['jer'] = jer_tot
    with open(os.path.join(args.out_dir, 'summary.json'), 'w') as fp:
        json.dump(summary, fp, indent=1, sort_keys=True)
    return 0


if __name__ == '__main__':
    sys.exit(main())
