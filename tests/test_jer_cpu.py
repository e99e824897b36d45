"""Jaccard error rate host side (DESIGN.md section 5.13): jer_finish against a brute force over all one-to-one mappings,
the worked case, who counts, speaker-weighted overall JER, ranking by JER and the argument errors.  No GPU needed."""
import itertools

import numpy as np
import pytest

from oracle import der_oracle
from oracle.jer_oracle import jer_ticks
from vbx_b200 import score, sweep


def brute_jer(R, S, O):
    """Mean over speakers with R > 0 of the best injective mapping onto labels with S > 0 (unmapped: 1)."""
    ks = [k for k in range(len(R)) if R[k] > 0]
    ls = [s for s in range(len(S)) if S[s] > 0]
    if not ks:
        return None
    c = {(k, s): (R[k] + S[s] - 2 * O[k][s]) / (R[k] + S[s] - O[k][s]) for k in ks for s in ls}
    best = float('inf')
    m = min(len(ks), len(ls))
    for sub in itertools.combinations(ks, m):
        for perm in itertools.permutations(ls, m):
            total = sum(c[(k, s)] for k, s in zip(sub, perm)) + (len(ks) - m)
            best = min(best, total)
    return best / len(ks)


def random_case(rng, K, L, ties):
    """R, S, O consistent with one timeline: every intersection at most either side's time."""
    R = rng.integers(0, 50, K) * (rng.random(K) > 0.2)
    S = rng.integers(0, 50, L) * (rng.random(L) > 0.2)
    if ties:
        R[:] = np.where(R > 0, 20, 0)
        S[:] = np.where(S > 0, 20, 0)
    O = np.zeros((K, L), dtype=np.int64)
    for k in range(K):
        for s in range(L):
            hi = min(R[k], S[s])
            O[k, s] = rng.integers(0, hi + 1) if hi and rng.random() < 0.6 else 0
            if ties and hi:
                O[k, s] = 10 * (rng.random() < 0.5)
    return R, S, O


@pytest.mark.parametrize('K,L', [(1, 1), (3, 3), (5, 2), (2, 5), (4, 6), (6, 4), (0, 3), (3, 0)])
@pytest.mark.parametrize('ties', [False, True])
def test_jer_finish_equals_brute_force(K, L, ties):
    rng = np.random.default_rng(100 * K + L + ties)
    for _ in range(40):
        R, S, O = random_case(rng, K, L, ties)
        got = score.jer_finish(R, S, O)
        want = brute_jer(R.tolist(), S.tolist(), O.tolist())
        if want is None:
            assert got['jer'] is None and got['speakers'] == 0
            continue
        assert got['jer'] == pytest.approx(want, abs=1e-12)
        assert got['speakers'] == int(np.sum(R > 0))
        assert got['jer'] == sum(score.speaker_jer(t) for t in got['ticks']) / len(got['ticks'])
        labels = [t['label'] for t in got['ticks'] if t['label'] is not None]
        assert len(labels) == len(set(labels)) and all(S[s] > 0 for s in labels)
        for t in got['ticks']:
            assert t['R'] == R[t['ref']]
            if t['label'] is not None:
                assert (t['S'], t['I']) == (S[t['label']], O[t['ref'], t['label']])


def test_zero_rows_and_columns_are_not_counted():
    R, S = [10, 0, 4], [0, 10, 0, 0]
    O = [[0, 10, 0, 0], [0, 0, 0, 0], [0, 4, 0, 0]]
    got = score.jer_finish(R, S, O)
    assert [t['ref'] for t in got['ticks']] == [0, 2]
    assert got['ticks'][0] == dict(ref=0, R=10, label=1, S=10, I=10)
    assert got['ticks'][1] == dict(ref=2, R=4, label=None, S=None, I=None)
    assert got['jer'] == 0.5


def test_no_reference_speaker_gives_none_even_when_the_system_speaks():
    assert score.jer_finish([], [5, 7], np.zeros((0, 2))) == dict(jer=None, speakers=0, ticks=[])
    assert score.jer_finish([0, 0], [5, 7], np.zeros((2, 2)))['jer'] is None


S_ = 1_000_000


def worked(regions2):
    """The worked case of DESIGN.md section 5.13 through the oracle: reference a [0, 10) s, b [6, 10) s; the system says
    0 on [0, 10) s and, with regions2 = (lo, hi) seconds, 1 there."""
    ref = [(0, 10 * S_, 'a'), (6 * S_, 10 * S_, 'b')]
    sysseg = [(0, 10 * S_, 0)] + ([(regions2[0] * S_, regions2[1] * S_, 1)] if regions2 else [])
    t = jer_ticks(ref, sysseg)
    R = [t['R'].get(k, 0) for k in 'ab']
    S = [t['S'].get(s, 0) for s in (0, 1)]
    O = [[t['I'].get((k, s), 0) for s in (0, 1)] for k in 'ab']
    return score.jer_finish(R, S, O), der_oracle.der_ticks(ref, sysseg)


def test_worked_case():
    got, der = worked(None)
    assert got['jer'] == 0.5
    assert got['ticks'] == [dict(ref=0, R=10 * S_, label=0, S=10 * S_, I=10 * S_), dict(ref=1, R=4 * S_, label=None,
                                                                                        S=None, I=None)]
    assert (der['miss'] + der['fa'] + der['conf']) / der['scored'] == 4 / 14
    assert worked((6, 10))[0]['jer'] == 0.0
    got, _ = worked((4, 10))
    assert got['ticks'][1] == dict(ref=1, R=4 * S_, label=1, S=6 * S_, I=4 * S_)
    assert got['jer'] == pytest.approx(1 / 6, abs=1e-15)


def test_reference_time_and_uem_exclusion():
    """A speaker entirely outside the UEM has R = 0 and is not counted; R is each speaker's scored time."""
    rows = [('r', 0.0, 10.0, 'a'), ('r', 6.0, 4.0, 'b'), ('r', 20.0, 5.0, 'c')]
    turns = score.reference_turns(rows)['r']
    lo = score.to_ticks(np.array([0.0, 5.0]))
    timeline = (lo, lo + 5 * S_, lo + 5 * S_)
    rec = score.prepare_recording('r', turns, timeline, uem=[(0.0, 12.0)], protocols=(('full', 0.0, False),))
    R = score.reference_time(rec.regions['full'], rec.n_ref)
    assert R == [10 * S_, 4 * S_, 0]
    t = jer_ticks([(0, 10 * S_, 'a'), (6 * S_, 10 * S_, 'b'), (20 * S_, 25 * S_, 'c')], [], uem=[(0, 12 * S_)])
    assert t['R'] == {'a': 10 * S_, 'b': 4 * S_}
    O = np.array([[10 * S_, 0], [4 * S_, 0], [0, 0]])
    got = score.jer_finish(R, [10 * S_, 0], O)
    assert got['speakers'] == 2 and got['jer'] == 0.5
    # with no UEM the same speaker counts, and is missed
    rec = score.prepare_recording('r', turns, timeline, protocols=(('full', 0.0, False),))
    assert score.reference_time(rec.regions['full'], rec.n_ref)[2] == 5 * S_


def test_overall_jer_weights_speakers():
    a = score.jer_finish([10, 10, 10], [10], [[10], [0], [0]])          # 0, 1, 1
    b = score.jer_finish([4], [4], [[4]])                               # 0
    none = score.jer_finish([], [3], np.zeros((0, 1)))
    assert a['jer'] == pytest.approx(2 / 3) and b['jer'] == 0.0
    tot = score.overall_jer([a, b, none])
    assert tot == dict(jer=0.5, speakers=4)                             # not the mean of recordings (1 / 3)
    assert score.overall_jer([none]) == dict(jer=None, speakers=0)


def test_rank_by_jer():
    per = {'x': dict(jer=0.3), 'y': dict(jer=None), 'z': dict(jer=0.1), 'w': dict(jer=0.3)}
    assert score.rank(per, key='jer') == ['z', 'x', 'w', 'y']
    assert score.rank({'a': dict(der=0.2), 'b': dict(der=0.1)}) == ['b', 'a']


def test_jer_needs_a_protocol_without_collar_that_scores_overlaps():
    rows = [('r', 0.0, 10.0, 'a')]
    turns = score.reference_turns(rows)['r']
    lo = score.to_ticks(np.array([0.0, 5.0]))
    rec = score.prepare_recording('r', turns, (lo, lo + 5 * S_, lo + 5 * S_))
    for p in ('forgiving', 'fair', 'nonexistent'):
        with pytest.raises(ValueError, match='collar'):
            score.score_entries([rec], [(0, np.zeros(2, dtype=np.int64))], jer=p)
    assert rec.protocols['full'] == (0, False)


def test_sweep_jer_needs_a_reference():
    grid = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[0.0], smoothing=[5.0])
    with pytest.raises(ValueError, match='ref_rttm'):
        sweep.sweep_batch({}, None, None, grid, jer=True)
    assert '--jer' in sweep.build_parser().format_help()
    assert '--jer' in score.build_parser().format_help()
