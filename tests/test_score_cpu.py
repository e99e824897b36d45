"""DER scoring (vbx_b200/score.py) on the host: the scored regions, the owned-interval timeline, the error algebra and the
readers, checked in exact ticks against the worked cases of DESIGN.md section 5.11 and the line-sweep oracle
(oracle/der_oracle.py).  The device accumulation is restated here as a plain loop over intervals and regions."""
import os

import numpy as np
import pytest

from oracle import der_oracle
from vbx_b200 import formats, pipeline, score

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
S = 1_000_000        # ticks per second


def accumulate(rec, labels, proto):
    """What vbx_score computes for one entry, as a loop; then the host's finish()."""
    lo, hi, mask, ref_total = rec.regions[proto]
    L = max(int(np.max(labels)) + 1, 1) if len(labels) else 1
    O = np.zeros((rec.n_ref, L), dtype=np.int64)
    cov = fa = 0
    ends = score.effective_hi((rec.sys_lo, rec.sys_hi, rec.sys_join_hi), labels)
    for a, b, s in zip(rec.sys_lo.tolist(), ends.tolist(), np.asarray(labels).tolist()):
        for rl, rh, m in zip(lo.tolist(), hi.tolist(), mask.tolist()):
            d = min(b, rh) - max(a, rl)
            if d <= 0:
                continue
            if m == 0:
                fa += d
                continue
            cov += d
            for k in range(rec.n_ref):
                if m >> k & 1:
                    O[k, s] += d
    return score.finish(cov, fa, O, ref_total)


def rows(rec, turns):
    """[(start s, end s, speaker)] -> formats.read_rttm rows."""
    return [(rec, float(s), float(e) - float(s), str(k)) for s, e, k in turns]


def score_host(ref, sys, uem=None, protocols=score.PROTOCOLS):
    """ref / sys: [(start s, end s, speaker)] of one recording -> ({protocol: result}, {protocol: oracle ticks})."""
    turns = score.reference_turns(rows('r', ref))['r'] if ref else []
    lo, hi, lab = score.system_turns(rows('r', sys), 'r')
    rec = score.prepare_recording('r', turns, (lo, hi, hi), uem, protocols)
    got = {p: accumulate(rec, lab, p) for p, _, _ in protocols}
    t = lambda x: int(score.to_ticks(x))
    want = {p: der_oracle.der_ticks([(t(s), t(e), k) for s, e, k in ref], [(t(s), t(e), k) for s, e, k in sys],
                                    t(c), io, None if uem is None else [(t(a), t(b)) for a, b in uem])
            for p, c, io in protocols}
    for p in want:
        assert got[p]['ticks'] == want[p], p
    return got


def ticks(r):
    return r['ticks']


def test_case_a():
    got = score_host([(0, 10, 'a'), (10, 20, 'b')], [(0, 9, '0'), (9, 20, '1')])
    assert ticks(got['full']) == dict(miss=0, fa=0, conf=1 * S, scored=20 * S)
    assert got['full']['der'] == 0.05
    for p in ('fair', 'forgiving'):
        assert ticks(got[p]) == dict(miss=0, fa=0, conf=750_000, scored=19 * S)
        assert got[p]['der'] == 0.75 / 19


def test_case_b():
    got = score_host([(0, 6, 'a'), (4, 10, 'b')], [(0, 5, '0'), (5, 12, '1')])
    assert ticks(got['full']) == dict(miss=2 * S, fa=2 * S, conf=0, scored=12 * S)
    assert ticks(got['fair']) == dict(miss=1_500_000, fa=1_750_000, conf=0, scored=10 * S)
    assert ticks(got['forgiving']) == dict(miss=0, fa=1_750_000, conf=0, scored=7 * S)
    assert got['fair']['der'] == 0.325 and got['forgiving']['der'] == 0.25


def test_perfect_system_with_permuted_labels_scores_zero():
    ref = [(0, 3, 'a'), (3, 7.5, 'b'), (8, 9, 'c'), (9, 12, 'a')]
    got = score_host(ref, [(s, e, {'a': '2', 'b': '0', 'c': '1'}[k]) for s, e, k in ref])
    for p in got:
        assert got[p]['der'] == 0.0


def test_silent_system_is_all_miss():
    got = score_host([(0, 3, 'a'), (2, 7, 'b')], [])
    for p in got:
        t = ticks(got[p])
        assert t['miss'] == t['scored'] > 0 and t['fa'] == t['conf'] == 0 and got[p]['der'] == 1.0


def test_system_over_non_speech_is_pure_false_alarm():
    got = score_host([(0, 3, 'a'), (10, 12, 'b')], [(4, 9, '0')])
    for p in got:
        t = ticks(got[p])
        assert t['fa'] == 5 * S and t['conf'] == 0 and t['miss'] == t['scored']
    assert ticks(got['full'])['scored'] == 5 * S


def test_touching_turns_of_one_speaker_make_no_collar():
    joined = score.reference_turns(rows('r', [(0, 4, 'a'), (4, 9, 'a')]))['r']
    assert len(joined) == 1 and joined[0][0].tolist() == [0] and joined[0][1].tolist() == [9 * S]
    got = score_host([(0, 4, 'a'), (4, 9, 'a')], [(0, 9, '0')])
    assert ticks(got['fair'])['scored'] == 8_500_000        # collars only at 0 and 9


def test_zero_length_turns_are_dropped():
    got = score_host([(0, 4, 'a'), (6, 6, 'b'), (2, 2, 'a')], [(0, 4, '0')])
    assert score.reference_turns(rows('r', [(6, 6, 'b')]))['r'] == []
    assert ticks(got['fair']) == dict(miss=0, fa=0, conf=0, scored=3_500_000)


def test_uem_restricts_the_scored_time():
    got = score_host([(0, 10, 'a')], [(0, 4, '0'), (12, 14, '1')], uem=[(2, 6), (11, 13)])
    assert ticks(got['full']) == dict(miss=2 * S, fa=1 * S, conf=0, scored=4 * S)


def test_recording_without_reference_speech_has_no_der():
    got = score_host([], [(0, 2, '0')])
    for p in got:
        assert got[p]['der'] is None and ticks(got[p])['fa'] == 2 * S


def test_overall_sums_numerators_and_denominators():
    a = score.result(1, 2, 3, 10)
    b = score.result(0, 0, 0, 30)
    assert score.overall([a, b])['der'] == 6 / 40
    assert score.overall([score.result(0, 1, 0, 0)])['der'] is None


def timeline_equals_merged_segments(seg, rng, n=200):
    timeline = score.owned_intervals(seg)
    lo = timeline[0]
    for _ in range(n):
        lab = rng.integers(0, int(rng.integers(1, 6)), len(seg))
        s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
        want = list(zip(score.to_ticks(s).tolist(), score.to_ticks(e).tolist(), l.tolist()))
        got = []                                   # join runs of equal labels over touching owned intervals
        for a, b, x in zip(lo.tolist(), score.effective_hi(timeline, lab).tolist(), lab.tolist()):
            if got and got[-1][2] == x and got[-1][1] == a:
                got[-1] = (got[-1][0], b, x)
            else:
                got.append((a, b, x))
        assert got == want


def test_owned_intervals_equal_merge_adjacent_labels_on_es2005a():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    timeline_equals_merged_segments(z['seg_times'], np.random.default_rng(0))


def test_owned_intervals_equal_merge_adjacent_labels_with_gaps():
    rng = np.random.default_rng(1)
    starts, t = [], 0.0
    for i in range(400):
        starts.append(t)
        t = round(t + (0.24 if rng.random() > 0.05 else 1.5 + 0.01 * int(rng.integers(1, 300))), 2)
    seg = np.stack([np.array(starts), np.array(starts) + 1.5], 1)
    assert np.sum(seg[1:, 0] > seg[:-1, 1]) > 5
    timeline_equals_merged_segments(seg, rng)


def test_owned_intervals_bridge_the_pauses_the_rttm_writer_joins():
    """Past 1000 s merge_adjacent_labels takes pauses of up to ~1e-5 of the time for touching and joins equal labels
    across them; the owned timeline must end the first interval at the next one's start there, and only there."""
    seg = np.array([[1998.0, 1999.5], [1999.51, 2001.01]])
    lo, hi, join_hi = score.owned_intervals(seg)
    assert hi.tolist() == [1999_500_000, 2001_010_000] and join_hi.tolist() == [1999_510_000, 2001_010_000]
    s, e, _ = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], np.array([3, 3]))
    assert score.to_ticks(s).tolist() == [1998_000_000] and score.to_ticks(e).tolist() == [2001_010_000]
    assert score.effective_hi((lo, hi, join_hi), [3, 3]).tolist() == [1999_510_000, 2001_010_000]
    assert score.effective_hi((lo, hi, join_hi), [3, 4]).tolist() == [1999_500_000, 2001_010_000]
    far = np.array([[10.0, 11.5], [11.51, 13.01]])                      # at 10 s the same pause is a pause
    assert score.owned_intervals(far)[2].tolist() == [11_500_000, 13_010_000]


def test_owned_intervals_equal_merge_adjacent_labels_late_in_long_recordings():
    """Segment times past 1000 s and 2000 s with pauses of 10 to 20 ms (joined there) and longer ones."""
    rng = np.random.default_rng(2)
    for t0 in (1000.0, 1500.0, 2000.0, 3600.0):
        starts, t = [], t0
        for i in range(400):
            starts.append(t)
            r = rng.random()
            step = 0.24 if r > 0.15 else (1.5 + 0.01 * int(rng.integers(1, 3)) if r > 0.05 else 1.5 + 0.01 * int(rng.integers(3, 300)))
            t = round(t + step, 2)
        seg = np.stack([np.array(starts), np.array(starts) + 1.5], 1)
        gaps = seg[1:, 0] - seg[:-1, 1]
        assert np.sum((gaps > 0.005) & (gaps < 0.025)) > 5
        lo, hi, join_hi = score.owned_intervals(seg)
        if t0 >= 2000.0:
            assert np.sum(join_hi > hi) > 5                 # the pauses are bridged for equal labels
        timeline_equals_merged_segments(seg, rng, n=50)


def test_read_uem(tmp_path):
    p = tmp_path / 'a.uem'
    p.write_text(';; comment\nES2005a 1 0.000 10.5\n\nES2005a 1 12 20\nIS1009a 1 3.25 9\n')
    assert formats.read_uem(str(p)) == {'ES2005a': [(0.0, 10.5), (12.0, 20.0)], 'IS1009a': [(3.25, 9.0)]}
    p.write_text('ES2005a 1 0\n')
    with pytest.raises(ValueError):
        formats.read_uem(str(p))


def test_read_rttm_directory(tmp_path):
    (tmp_path / 'b.rttm').write_text('SPEAKER b 1 1.000000 2.000000 <NA> <NA> x <NA> <NA>\n')
    (tmp_path / 'a.rttm').write_text('SPEAKER a 1 0.500000 1.000000 <NA> <NA> y <NA> <NA>\n')
    (tmp_path / 'notes.txt').write_text('SPEAKER c 1 0 1 <NA> <NA> z <NA> <NA>\n')
    assert score.read_rttm_path(str(tmp_path)) == [('a', 0.5, 1.0, 'y'), ('b', 1.0, 2.0, 'x')]
    assert score.read_rttm_path(str(tmp_path / 'b.rttm')) == [('b', 1.0, 2.0, 'x')]


def test_ranking_is_stable_on_ties():
    r = lambda der: dict(der=der)
    per = {'s1': r(0.2), 's2': r(0.1), 's3': r(0.2), 's4': r(None), 's5': r(0.1)}
    assert score.rank(per) == ['s2', 's5', 's1', 's3', 's4']


def test_more_than_64_reference_speakers_is_an_error():
    ref = rows('big', [(i, i + 1, f'spk{i}') for i in range(65)])
    with pytest.raises(ValueError, match='big'):
        score.reference_turns(ref)
    assert len(score.reference_turns(ref[:64])['big']) == 64


def test_missing_reference_recording_is_an_error():
    with pytest.raises(ValueError, match='lacks'):
        score.score_rttm(rows('a', [(0, 1, 'x')]), rows('b', [(0, 1, '0')]), 0.25, False)


def test_missing_uem_recording_is_an_error():
    with pytest.raises(ValueError, match='UEM'):
        score.score_rttm(rows('a', [(0, 1, 'x')]), rows('a', [(0, 1, '0')]), 0.25, False, uem={'b': [(0, 1)]})


def test_overlapping_system_speakers_are_an_error():
    with pytest.raises(ValueError, match='overlapping'):
        score.system_turns(rows('r', [(0, 5, '0'), (4, 6, '1')]), 'r')
    lo, hi, lab = score.system_turns(rows('r', [(0, 5, '0'), (4, 6, '0'), (6, 7, '1')]), 'r')
    assert lo.tolist() == [0, 6 * S] and hi.tolist() == [6 * S, 7 * S] and lab.tolist() == [0, 1]


def test_negative_collar_is_an_error():
    with pytest.raises(ValueError, match='collar'):
        score.score_rttm(rows('a', [(0, 1, 'x')]), rows('a', [(0, 1, '0')]), -0.1, False)
    with pytest.raises(ValueError, match='collar'):
        score.prepare_recording('a', [], ([0], [1], [1]), protocols=(('p', -1.0, False),))


def test_random_recordings_match_the_oracle():
    """Ragged random references (up to 4 overlapping speakers) and systems: host regions + accumulation == oracle."""
    rng = np.random.default_rng(7)
    for _ in range(30):
        K = int(rng.integers(1, 7))
        ref = []
        for k in range(K):
            t = float(rng.integers(0, 20))
            for _ in range(int(rng.integers(1, 5))):
                d = float(rng.integers(1, 40)) / 4
                ref.append((t, t + d, f's{k}'))
                t += d + float(rng.integers(0, 12)) / 4
        cuts = np.unique(rng.integers(0, 240, 12)) / 4.0
        sys = [(a, b, str(int(rng.integers(0, 4)))) for a, b in zip(cuts[:-1], cuts[1:]) if rng.random() < 0.8]
        uem = [(1.0, 20.5), (25.0, 50.0)] if rng.random() < 0.5 else None
        score_host(ref, sys, uem=uem)
