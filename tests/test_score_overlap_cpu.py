"""Overlap-aware output and its scoring (DESIGN.md section 5.12) on the host: the overlap regions, the split scored
regions, the combined RTTM segments and the two-stream counting, checked in exact ticks against the worked case and the
line-sweep oracle (oracle/der_oracle.py).  The device accumulation (vbx_score_overlap) is restated here as a loop over
intervals, regions and the stretches between the two stream ends."""
import os

import numpy as np
import pytest

from oracle import der_oracle
from vbx_b200 import pipeline, score, synth

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
S = 1_000_000        # ticks per second


def accumulate2(rec, labels, labels2, proto):
    """What vbx_score_overlap computes for one entry, stretch by stretch; then the host's finish()."""
    lo, hi, mask, ovl = score._overlap_split(rec, proto)
    ref_total = rec.regions[proto][3]
    timeline = (rec.sys_lo, rec.sys_hi, rec.sys_join_hi)
    labels = np.asarray(labels)
    L = max([int(labels.max()) + 1 if len(labels) else 1] + ([int(labels2.max()) + 1] if labels2 is not None and len(labels2) else []))
    e1 = score.effective_hi(timeline, labels)
    e2 = rec.sys_lo if labels2 is None else np.where(np.asarray(labels2) < 0, rec.sys_lo,    # -1: no second label
                                                     score.effective_hi(timeline, labels2))
    O = np.zeros((rec.n_ref, L), dtype=np.int64)
    both = fa = 0
    for t, a in enumerate(rec.sys_lo.tolist()):
        end1, end2 = int(e1[t]), int(e2[t])
        for rl, rh, m, f in zip(lo.tolist(), hi.tolist(), mask.tolist(), ovl.tolist()):
            x0 = max(a, rl)
            if x0 >= rh:
                continue
            cuts = sorted({x0, rh} | {c for c in (end1, end2) if x0 < c < rh})
            for x, y in zip(cuts, cuts[1:]):
                if y <= x:
                    continue
                sys_on = ([int(labels[t])] if x < end1 else []) + \
                         ([int(labels2[t])] if labels2 is not None and f and x < end2 else [])
                ref_on = [k for k in range(rec.n_ref) if m >> k & 1]
                d = y - x
                both += min(len(ref_on), len(sys_on)) * d
                fa += max(0, len(sys_on) - len(ref_on)) * d
                for r in ref_on:
                    for s in sys_on:
                        O[r, s] += d
    return score.finish(both, fa, O, ref_total)


def oracle_entry(ref_rows, seg, labels, labels2, overlap, uem, collar, ignore):
    """The oracle on the segments overlap_segments writes."""
    t = score.to_ticks
    s, e, l = pipeline.overlap_segments(seg, labels, labels2, overlap)
    ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows]
    return der_oracle.der_ticks(ref, list(zip(t(s).tolist(), t(e).tolist(), l.tolist())), int(t(collar)), ignore,
                                None if uem is None else [(int(t(a)), int(t(b))) for a, b in uem])


def ref_layers(rng, span_cs, K, layers):
    """Reference turns (start s, duration s, speaker) over [0, span_cs) centiseconds: `layers` independent sequences of
    turns, so at most that many speakers overlap."""
    turns, spk = [], 0
    for _ in range(layers):
        t = int(rng.integers(0, 200))
        while t < span_cs:
            d = int(rng.integers(10, 300))
            turns.append((t / 100.0, d / 100.0, f'spk{spk % K}'))
            spk += int(rng.integers(1, K + 1))
            t += d + int(rng.integers(0, 150))
    return turns


def second_labels(rng, labels, L):
    """A second label per interval, different from the first."""
    return (labels + rng.integers(1, L, len(labels))) % L


def random_case(seed):
    rng = np.random.default_rng(seed)
    T = int(rng.integers(1, 50))
    seg, _ = synth.make_scoring_archive([T], seed=seed, gap_prob=0.1)['syn00']
    span = int(round(seg[:, 1].max() * 100)) + 200
    K, layers = int(rng.integers(1, 6)), int(rng.integers(1, 5))
    ref_rows = [('r',) + x for x in ref_layers(rng, span, K, layers)]
    turns = score.reference_turns(ref_rows).get('r', [])
    L = int(rng.integers(1, 6))
    labels = np.zeros(T, dtype=np.int64)
    labels[0] = rng.integers(L)
    for i in range(1, T):
        labels[i] = labels[i - 1] if rng.random() < 0.8 else rng.integers(L)
    labels2 = None if L == 1 or rng.random() < 0.15 else second_labels(rng, labels, L)
    oracle = bool(seed % 2)
    if oracle:
        overlap = score.oracle_overlaps(turns)
    else:
        cut = np.sort(rng.integers(0, span, 2 * int(rng.integers(0, 6)))) / 100.0
        overlap = score.overlap_ticks(cut.reshape(-1, 2).tolist())
    uem = [(0.5, span / 200.0), (span / 200.0 + 1.0, span / 100.0)] if rng.random() < 0.5 else None
    rec = score.prepare_recording('r', turns, score.owned_intervals(seg), uem, overlap=overlap)
    return ref_rows, seg, rec, labels, labels2, overlap, uem, oracle


@pytest.mark.parametrize('seed', range(40))
def test_two_stream_accumulation_equals_the_oracle(seed):
    ref_rows, seg, rec, labels, labels2, overlap, uem, _ = random_case(seed)
    for p, c, io in score.PROTOCOLS:
        got = accumulate2(rec, labels, labels2, p)
        assert got['ticks'] == oracle_entry(ref_rows, seg, labels, labels2, overlap, uem, c, io), p


@pytest.mark.parametrize('seed', range(1, 40, 2))
def test_oracle_overlaps_never_increase_der(seed):
    """Stream 2 adds time only where N_ref >= 2, and a maximum matching cannot shrink when cells of O grow."""
    ref_rows, seg, rec, labels, labels2, overlap, uem, oracle = random_case(seed)
    assert oracle
    if labels2 is None:
        labels2 = second_labels(np.random.default_rng(seed), labels, max(int(labels.max()) + 2, 2))
    for p, _, _ in score.PROTOCOLS:
        one, two = accumulate2(rec, labels, None, p)['ticks'], accumulate2(rec, labels, labels2, p)['ticks']
        if p == 'forgiving':
            assert two == one
        else:
            assert two['fa'] == one['fa'] and two['scored'] == one['scored']
            assert two['miss'] + two['conf'] <= one['miss'] + one['conf']


def worked(overlap):
    ref_rows = [('r', 0.0, 10.0, 'a'), ('r', 6.0, 4.0, 'b')]
    seg = np.array([[0.0, 10.0]])
    rec = score.prepare_recording('r', score.reference_turns(ref_rows)['r'], score.owned_intervals(seg),
                                  overlap=score.overlap_ticks(overlap))
    got = accumulate2(rec, np.array([0]), np.array([1]), 'full')
    assert got['ticks'] == oracle_entry(ref_rows, seg, np.array([0]), np.array([1]), score.overlap_ticks(overlap),
                                        None, 0.0, False)
    return got


def test_worked_case():
    assert worked([(6.0, 10.0)])['ticks'] == dict(miss=0, fa=0, conf=0, scored=14 * S)
    got = worked([])
    assert got['ticks'] == dict(miss=4 * S, fa=0, conf=0, scored=14 * S) and got['der'] == 4 / 14
    got = worked([(4.0, 10.0)])
    assert got['ticks'] == dict(miss=0, fa=2 * S, conf=0, scored=14 * S) and got['der'] == 2 / 14


def stream_runs(timeline, labels, clip=None):
    """Runs of equal labels over the owned intervals (joined ends), optionally cut to regions (lo, hi) ticks."""
    runs = []
    for a, b, x in zip(timeline[0].tolist(), score.effective_hi(timeline, labels).tolist(), labels.tolist()):
        if runs and runs[-1][2] == x and runs[-1][1] == a:
            runs[-1] = (runs[-1][0], b, x)
        elif b > a:
            runs.append((a, b, x))
    if clip is None:
        return runs
    return [(max(a, c), min(b, d), x) for a, b, x in runs for c, d in zip(*(v.tolist() for v in clip))
            if min(b, d) > max(a, c)]


def check_written_segments(seg, rng, n):
    timeline = score.owned_intervals(seg)
    span = float(seg[:, 1].max())
    for _ in range(n):
        L = int(rng.integers(2, 6))
        lab = rng.integers(0, L, len(seg))
        lab2 = second_labels(rng, lab, L)
        cut = np.sort(rng.uniform(float(seg[0, 0]), span, 2 * int(rng.integers(1, 8))))
        overlap = score.overlap_ticks(cut.reshape(-1, 2).tolist())
        s, e, l = pipeline.overlap_segments(seg, lab, lab2, overlap)
        got = list(zip(score.to_ticks(s).tolist(), score.to_ticks(e).tolist(), l.tolist()))
        want = stream_runs(timeline, lab) + stream_runs(timeline, lab2, overlap)
        assert got == want
        lines = pipeline.rttm_lines('r', s, e, l)
        parsed = [(float(x.split()[3]), float(x.split()[4]), int(x.split()[7]) - 1) for x in lines]
        for (a, d, k), (wa, wb, wk) in zip(parsed, want):                   # each written number is rounded to 1 us
            assert k == wk and abs(int(score.to_ticks(a)) - wa) <= 1 and abs(int(score.to_ticks(a + d)) - wb) <= 2
        assert len(parsed) == len(want)
        assert pipeline.overlap_segments(seg, lab, None, overlap)[0].tolist() == s[:len(stream_runs(timeline, lab))].tolist()


def test_written_segments_are_the_two_streams_on_es2005a():
    check_written_segments(np.load(os.path.join(GOLD, 'es2005a.npz'))['seg_times'], np.random.default_rng(0), 40)


def test_written_segments_are_the_two_streams_late_in_long_recordings():
    """Past 1000 s and 2000 s merge_adjacent_labels bridges 10 to 20 ms pauses; both streams must follow it."""
    rng = np.random.default_rng(2)
    for t0 in (1000.0, 2000.0, 3600.0):
        starts, t = [], t0
        for _ in range(300):
            starts.append(t)
            r = rng.random()
            step = 0.24 if r > 0.15 else (1.5 + 0.01 * int(rng.integers(1, 3)) if r > 0.05 else 1.5 + 0.01 * int(rng.integers(3, 300)))
            t = round(t + step, 2)
        seg = np.stack([np.array(starts), np.array(starts) + 1.5], 1)
        lo, hi, join_hi = score.owned_intervals(seg)
        if t0 >= 2000.0:
            assert np.sum(join_hi > hi) > 5
        check_written_segments(seg, rng, 15)


def test_no_overlap_regions_is_the_single_speaker_output():
    rng = np.random.default_rng(4)
    for seed in range(12):
        ref_rows, seg, _, labels, labels2, _, uem, _ = random_case(seed)
        L = int(labels.max()) + 2
        labels2 = second_labels(rng, labels, L)
        none = score.overlap_ticks([])
        turns = score.reference_turns(ref_rows).get('r', [])
        rec = score.prepare_recording('r', turns, score.owned_intervals(seg), uem, overlap=none)
        for p, c, io in score.PROTOCOLS:
            assert all(np.array_equal(a, b) for a, b in zip(rec.overlap_regions[p][:3], rec.regions[p][:3]))
            assert not rec.overlap_regions[p][3].any()
            want = oracle_entry(ref_rows, seg, labels, None, none, uem, c, io)
            assert accumulate2(rec, labels, labels2, p)['ticks'] == want
            assert accumulate2(rec, labels, None, p)['ticks'] == want
        item = pipeline._result('r', seg, labels, labels2, 3, False, none)
        assert item['rttm_overlap'] == item['rttm'] and item['overlap_seconds'] == 0.0
        assert set(pipeline._result('r', seg, labels, labels2, 3, False)) == \
            {'rttm', 'labels', 'labels2nd', 'iterations', 'n_speakers', 'rttm2nd'}


def test_overlap_regions_from_rttm_rows_ignore_speakers_and_union():
    rows = [('a', 1.0, 2.0, 'x'), ('a', 2.5, 1.0, 'y'), ('a', 5.0, 1.0, 'x'), ('b', 0.0, 0.0, 'x'), ('c', 3.0, 1.0, 'z')]
    assert score.overlaps_from_rows(rows) == {'a': [(1.0, 3.5), (5.0, 6.0)], 'b': [], 'c': [(3.0, 4.0)]}


def test_oracle_overlaps_are_two_or_more_reference_speakers():
    rows = [('r', 0.0, 4.0, 'a'), ('r', 3.0, 3.0, 'b'), ('r', 5.0, 2.0, 'c'), ('r', 7.0, 1.0, 'a'), ('r', 8.0, 1.0, 'b')]
    lo, hi = score.oracle_overlaps(score.reference_turns(rows)['r'])
    assert lo.tolist() == [3 * S, 5 * S] and hi.tolist() == [4 * S, 6 * S]           # touching turns do not overlap
    assert [a.tolist() for a in score.oracle_overlaps([])] == [[], []]


def system_host(ref, sys, protocols=score.PROTOCOLS):
    """Overlapping system turns scored through system_stretches and the two-stream loop, against the oracle."""
    rr = [('r', float(s), float(e) - float(s), k) for s, e, k in ref]
    turns = score.reference_turns(rr)['r']
    lo, hi, l1, l2 = score.system_stretches([('r', float(s), float(e) - float(s), k) for s, e, k in sys], 'r')
    rec = score.prepare_recording('r', turns, (lo, hi, hi), None, protocols, overlap=(lo[:1], hi[-1:]))
    t = lambda x: int(score.to_ticks(x))
    for p, c, io in protocols:
        got = accumulate2(rec, l1, l2, p)['ticks']
        want = der_oracle.der_ticks([(t(s), t(e), k) for s, e, k in ref], [(t(s), t(e), k) for s, e, k in sys], t(c), io)
        assert got == want, p


def test_overlapping_system_rttm_scores_equal_the_oracle():
    system_host([(0, 10, 'a'), (6, 10, 'b')], [(0, 10, '0'), (6, 10, '1')])
    system_host([(0, 10, 'a'), (6, 10, 'b')], [(0, 10, '0'), (4, 10, '1')])
    rng = np.random.default_rng(11)
    for _ in range(30):
        ref, sys = [], []
        for k in range(int(rng.integers(1, 5))):
            t = float(rng.integers(0, 20))
            for _ in range(int(rng.integers(1, 5))):
                d = float(rng.integers(1, 40)) / 4
                ref.append((t, t + d, f's{k}'))
                t += d + float(rng.integers(0, 12)) / 4
        for layer in range(2):                  # two layers of system turns: at most two at a time
            cuts = np.unique(rng.integers(0, 240, 10)) / 4.0
            sys += [(a, b, str(2 * int(rng.integers(0, 3)) + layer)) for a, b in zip(cuts[:-1], cuts[1:]) if rng.random() < 0.6]
        system_host(ref, sys)


def test_three_system_speakers_are_an_error():
    rows = [('r', 0.0, 5.0, '0'), ('r', 1.0, 5.0, '1'), ('r', 2.0, 1.0, '2')]
    with pytest.raises(ValueError, match=r"'r'.*3 system speakers at 2\.000000 s"):
        score.system_stretches(rows, 'r')
    with pytest.raises(ValueError, match='3 system speakers'):
        score.score_rttm([('r', 0.0, 1.0, 'a')], rows, 0.25, False, overlapping=True)
    with pytest.raises(ValueError, match='overlapping'):
        score.score_rttm([('r', 0.0, 1.0, 'a')], rows[:2], 0.25, False)


def test_overlap_options_need_the_vb_hmm():
    with pytest.raises(ValueError, match='AHC'):
        pipeline.diarize_batch({}, None, None, 0.3, 17, 0.99, init='AHC', overlaps={})
    from vbx_b200 import sweep
    grid = dict(Fa=[0.3], Fb=[17], loopP=[0.99], threshold=[0.0], smoothing=[5.0])
    with pytest.raises(ValueError, match='AHC'):
        sweep.sweep_batch({}, None, None, grid, init='AHC', overlaps={})
    with pytest.raises(ValueError, match='ref_rttm'):
        sweep.sweep_batch({}, None, None, grid, oracle_overlaps=True)
