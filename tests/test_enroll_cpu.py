"""Enrolment against known speakers (DESIGN.md section 5.16) on the host: the rectangular LLR against explicit Gaussian
marginals, the assignment oracle against exhaustive search, the naming rule and its composition with linking, the
enrolment readers, argument errors, and the name-level DER against a line sweep over the recordings laid end to end.
The device accumulation of the DER is restated here as a loop over intervals and regions, so score_rttm's host work
runs without a GPU."""
import itertools
from collections import defaultdict

import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import enroll_oracle
from vbx_b200 import enroll, formats, link, score


# ---- the score and the assignment ----------------------------------------------------------------------------------

def _log_marginal(X, Phi):
    n = X.shape[0]
    return sum(multivariate_normal(np.zeros(n), np.eye(n) + Phi[r] * np.ones((n, n))).logpdf(X[:, r])
               for r in range(X.shape[1]))


@pytest.mark.parametrize('c', [1.0, 0.3 / 17])
@pytest.mark.parametrize('seed', range(4))
def test_llr_is_the_log_ratio_of_gaussian_marginals(c, seed):
    rng = np.random.default_rng(seed)
    R = int(rng.integers(1, 5))
    Phi = rng.uniform(0.1, 4.0, R)
    Xs = [rng.standard_normal((int(rng.integers(1, 5)), R)) * 2 for _ in range(2)]
    Xe = [rng.standard_normal((int(rng.integers(1, 5)), R)) * 2 for _ in range(3)]
    got = enroll_oracle.llr(np.array([len(x) for x in Xs], dtype=np.float64), np.array([x.sum(0) for x in Xs]),
                            np.array([len(x) for x in Xe], dtype=np.float64), np.array([x.sum(0) for x in Xe]), Phi, c)
    assert got.shape == (2, 3)
    P = Phi * c
    for i, a in enumerate(Xs):
        for j, b in enumerate(Xe):
            A, B = a * np.sqrt(c), b * np.sqrt(c)
            want = _log_marginal(np.vstack([A, B]), P) - _log_marginal(A, P) - _log_marginal(B, P)
            assert abs(got[i, j] - want) <= 1e-10 * max(1.0, abs(want)), (got[i, j], want)


@pytest.mark.parametrize('seed', range(5))
def test_assignment_oracle_is_the_exhaustive_optimum(seed):
    rng = np.random.default_rng(seed)
    K, E = int(rng.integers(1, 5)), int(rng.integers(1, 5))
    L = rng.standard_normal((K, E)) * 20
    for t in (-100.0, 0.0, 10.0, 100.0):
        a, obj = enroll_oracle.assign(L, np.array([0, K]), t)
        best = 0.0
        for k in range(0, min(K, E) + 1):             # every one-to-one naming of k speakers
            for rows in itertools.combinations(range(K), k):
                for cols in itertools.permutations(range(E), k):
                    best = min(best, sum(t - L[r, e] for r, e in zip(rows, cols)))
        assert abs(obj[0] - best) <= 1e-9 * max(1.0, abs(best))
        named = a >= 0
        assert (L[named, a[named]] >= t).all() and len(set(a[named].tolist())) == int(named.sum())


# ---- names -----------------------------------------------------------------------------------------------------------

def test_names_unknowns_and_second_only_labels():
    table = link.speaker_table([np.array([0, 2, 2]), np.zeros(0, dtype=np.int64), np.array([1, 0])])
    # speakers: (0,0) (0,2) (2,0) (2,1)
    names, llrs = enroll.enroll_names(table, [1, -1, -1, 0], [5.0, -3.0, 1.5, 9.0], ['alice', 'bob'], ['a', 'b', 'c'],
                                      labels2=[np.array([3, -1, 0]), None, np.array([0, 4])])
    assert names == [{0: 'bob', 2: 'unknown-a-3', 3: 'unknown-a-4'}, {}, {0: 'unknown-c-1', 1: 'alice', 4: 'unknown-c-5'}]
    assert llrs == [{0: 5.0, 2: -3.0}, {}, {0: 1.5, 1: 9.0}]
    want = enroll_oracle.names(table.rec, table.label, [1, -1, -1, 0], ['alice', 'bob'], ['a', 'b', 'c'],
                               labels2=[np.array([3, -1, 0]), None, np.array([0, 4])])
    assert names == want


def test_names_with_linked_unknowns():
    labels = [np.array([0, 1, 1]), np.array([0, 1]), np.array([0])]
    labels2 = [np.array([2, 0, 0]), None, None]
    table = link.speaker_table(labels)
    assign = [0, -1, -1, 1, -1]               # (0,0) -> e0, (1,1) -> e1; (0,1), (1,0), (2,0) unknown
    first, _ = enroll.enroll_names(table, assign, np.zeros(5), ['e0', 'e1'], ['r0', 'r1', 'r2'], labels2)
    l1 = [enroll.mask_named(l, m) for l, m in zip(labels, first)]
    l2 = [enroll.mask_named(l, m) for l, m in zip(labels2, first)]
    assert [x.tolist() for x in l1] == [[-1, 1, 1], [0, -1], [0]]
    assert l2[0].tolist() == [2, -1, -1] and l2[1] is None
    # the unknowns (0,1), (1,0), (2,0): (0,1) ~ (2,0), (1,0) apart; label 2 of recording 0 only occurs as a second label
    ut = link.speaker_table(l1)
    assert ut.rec.tolist() == [0, 1, 2] and ut.label.tolist() == [1, 0, 0]
    from oracle import link_oracle
    d = np.array([[0.0, 50.0, -20.0], [50.0, 0.0, 50.0], [-20.0, 50.0, 0.0]])
    lk = link.link_cut(link_oracle.link(d), ut, 0.0, l2)
    names, _ = enroll.enroll_names(table, assign, np.zeros(5), ['e0', 'e1'], ['r0', 'r1', 'r2'], labels2, link=lk)
    assert names == [{0: 'e0', 1: 'unknown-1', 2: 'unknown-3'}, {0: 'unknown-2', 1: 'e1'}, {0: 'unknown-1'}]


# ---- readers and argument errors ----------------------------------------------------------------------------------

def test_enrolment_readers(tmp_path):
    rng = np.random.default_rng(0)
    keys = ['b-1', 'a-1', 'b-2', 'c-1']
    x = rng.standard_normal((4, 6)).astype(np.float32)
    formats.write_vec_flt_ark(str(tmp_path / 'e.ark'), keys, x)
    (tmp_path / 'u').write_text('a-1 A\n\nb-1 B\nb-2 B\nc-1 C\nd-1 D2\n')
    assert formats.read_utt2spk(str(tmp_path / 'u')) == {'a-1': 'A', 'b-1': 'B', 'b-2': 'B', 'c-1': 'C', 'd-1': 'D2'}
    with pytest.raises(ValueError, match='speakers without x-vectors'):
        formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'u'))
    (tmp_path / 'u').write_text('a-1 A\nb-1 B\nb-2 B\nc-1 C\nz-9 B\n')
    got = formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'u'))
    assert list(got) == ['B', 'A', 'C']
    assert np.array_equal(got['B'], x[[0, 2]]) and np.array_equal(got['A'], x[[1]]) and got['C'].dtype == np.float64
    (tmp_path / 'u2').write_text('a-1 A\nb-1 B\nb-2 B\n')
    with pytest.raises(ValueError, match="'c-1' has no speaker"):
        formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'u2'))
    (tmp_path / 'u3').write_text('a-1 A\na-1 B\n')
    with pytest.raises(ValueError, match='listed twice'):
        formats.read_utt2spk(str(tmp_path / 'u3'))
    (tmp_path / 'u4').write_text('a-1 A extra\n')
    with pytest.raises(ValueError, match='expected'):
        formats.read_utt2spk(str(tmp_path / 'u4'))


def test_argument_errors_come_before_device_work(monkeypatch):
    from vbx_b200 import pipeline
    import torch
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: (_ for _ in ()).throw(AssertionError('device touched')))
    recs = {'r': (np.zeros((3, 8)), np.zeros((3, 2)))}
    ok = {'alice': np.ones((2, 8))}
    bad = [({'': np.ones((1, 8))}, 0.0, 'non-empty'), ({'a b': np.ones((1, 8))}, 0.0, 'whitespace'),
           ({'unknown-x': np.ones((1, 8))}, 0.0, 'reserved'), ({'a': np.ones((0, 8))}, 0.0, 'at least one'),
           ({'a': np.ones((2, 7))}, 0.0, 'dimension 7'), (ok, None, 'no default'), (ok, 2e15, 'must lie'),
           (ok, float('nan'), 'must lie'), (None, 1.0, 'without enroll'), ({}, 1.0, 'non-empty')]
    for e, t, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pipeline.diarize_batch(recs, None, None, 0.3, 17.0, 0.99, enroll=e, enroll_threshold=t)
    with pytest.raises(ValueError, match='every enrolled speaker'):
        enroll.enroll_speakers(np.zeros((2, 4)), np.ones(4), [0, 2], [np.zeros(2)], np.zeros((2, 4)), [0, 2], 0.3, 17.0,
                               0.0)
    with pytest.raises(ValueError, match='must lie'):
        enroll.enroll_speakers(np.zeros((2, 4)), np.ones(4), [0, 2], [np.zeros(2)], np.zeros((1, 4)), [0], 0.3, 17.0,
                               -1e16)


def test_cli_enrolment_options_go_together(capsys):
    from vbx_b200 import cli
    base = ['--init', 'AHC+VB', '--out-rttm-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform',
            't', '--plda-file', 'p', '--threshold', '0', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']
    for extra in (['--enroll-ark', 'e'], ['--enroll-threshold', '3'], ['--enroll-ark', 'e', '--enroll-utt2spk', 'u']):
        with pytest.raises(SystemExit):
            cli.main(base + extra)
        assert 'go together' in capsys.readouterr().err


# ---- name-level DER --------------------------------------------------------------------------------------------------

def _host_score_entries(recordings, entries, device=None, jer=None, blocks=False):
    """score.score_entries with the device accumulation restated on the host (score_rttm's entries: no joined ends)."""
    out = []
    for e in entries:
        rec = recordings[e[0]]
        l1 = np.asarray(e[1])
        l2 = np.asarray(e[2]) if len(e) == 3 and e[2] is not None else np.full(len(l1), -1)
        L = max([int(l1.max()) + 1 if len(l1) else 1, int(l2.max()) + 1 if len(l2) else 1])
        res = {}
        for proto in rec.regions:
            lo, hi, mask, ovl = score._overlap_split(rec, proto)
            O = np.zeros((rec.n_ref, L), dtype=np.int64)
            both = fa = 0
            for a, z, s1, s2 in zip(rec.sys_lo.tolist(), rec.sys_hi.tolist(), l1.tolist(), l2.tolist()):
                for rl, rh, m, f in zip(lo.tolist(), hi.tolist(), mask.tolist(), ovl.tolist()):
                    d = min(z, rh) - max(a, rl)
                    if d <= 0:
                        continue
                    sys_on = [s1] + ([s2] if s2 >= 0 and f else [])
                    ref_on = [k for k in range(rec.n_ref) if m >> k & 1]
                    both += min(len(ref_on), len(sys_on)) * d
                    fa += max(0, len(sys_on) - len(ref_on)) * d
                    for r in ref_on:
                        for s in sys_on:
                            O[r, s] += d
            res[proto] = score.finish(both, fa, O, rec.regions[proto][3])
            if blocks:
                res.setdefault('O', {})[proto] = O
        out.append(res)
    return out


def _archive(rng, n_files, pool, two_speaker):
    """Reference and system rows of n_files recordings; system names are drawn from the reference's names (and one
    name the reference never uses), by layer parity under two_speaker so that two layers never share a name."""
    ref, sys = [], []
    layers = 2 if two_speaker else 1
    for f in range(n_files):
        name = f'rec{f}'
        spk = rng.choice(pool, int(rng.integers(1, 4)), replace=False)
        t = float(rng.integers(0, 8))
        for _ in range(int(rng.integers(3, 9))):
            k = spk[int(rng.integers(len(spk)))]
            d = float(rng.integers(1, 40)) / 4
            ref.append((name, t, d, str(k)))
            if rng.random() < 0.3:
                ref.append((name, t + d / 2, d, str(spk[int(rng.integers(len(spk)))])))
            t += d + float(rng.integers(0, 8)) / 4
        for layer in range(layers):
            cuts = np.unique(rng.integers(0, int(4 * t) + 8, 8)) / 4.0
            sys += [(name, float(a), float(b - a), str(int(rng.integers(0, (len(pool) + 1) // layers + 1)) * layers + layer))
                    for a, b in zip(cuts[:-1], cuts[1:]) if rng.random() < 0.7]
    return ref, sys


def _concatenated(ref, sys, uem, collar):
    t = lambda x: int(score.to_ticks(x))
    names = sorted({r[0] for r in ref})
    shift, off = {}, 0
    for n in names:
        shift[n] = off
        ends = [t(r[1] + r[2]) for r in ref + sys if r[0] == n] + [t(b) for a, b in (uem or {}).get(n, [])]
        off += max(ends) + 2 * t(collar) + 1
    R = [(t(r[1]) + shift[r[0]], t(r[1] + r[2]) + shift[r[0]], r[3]) for r in ref]
    S = [(t(r[1]) + shift[r[0]], t(r[1] + r[2]) + shift[r[0]], r[3]) for r in sys]
    U = None if uem is None else [(t(a) + shift[n], t(b) + shift[n]) for n in names for a, b in uem[n]]
    return R, S, U


def _by_name_sweep(ref, sys, collar, ignore_overlaps, uem):
    """A line sweep over ticks counting the md-eval errors with speakers matched only by equal names."""
    from oracle.der_oracle import merge_speaker_turns
    ev = defaultdict(list)
    for s, e, k in merge_speaker_turns(ref):
        ev[s].append(('ref', k, 1))
        ev[e].append(('ref', k, -1))
        if collar > 0:
            for x in (s, e):
                ev[x - collar].append(('collar', None, 1))
                ev[x + collar].append(('collar', None, -1))
    for s, e, k in sys:
        if e > s:
            ev[s].append(('sys', k, 1))
            ev[e].append(('sys', k, -1))
    for s, e in uem or []:
        if e > s:
            ev[s].append(('uem', None, 1))
            ev[e].append(('uem', None, -1))
    cnt = defaultdict(lambda: defaultdict(int))
    miss = fa = conf = scored = 0
    times = sorted(ev)
    for t, t_next in zip(times, times[1:]):
        for kind, key, step in ev[t]:
            cnt[kind][key] += step
        d = t_next - t
        ref_on = {k for k, c in cnt['ref'].items() if c > 0}
        sys_on = {k for k, c in cnt['sys'].items() if c > 0}
        if (uem is not None and cnt['uem'][None] <= 0) or cnt['collar'][None] > 0 or \
                (ignore_overlaps and len(ref_on) >= 2):
            continue
        scored += len(ref_on) * d
        miss += max(0, len(ref_on) - len(sys_on)) * d
        fa += max(0, len(sys_on) - len(ref_on)) * d
        conf += (min(len(ref_on), len(sys_on)) - len(ref_on & sys_on)) * d
    return dict(miss=miss, fa=fa, conf=conf, scored=scored)


@pytest.mark.parametrize('two_speaker', [False, True])
@pytest.mark.parametrize('with_uem', [False, True])
@pytest.mark.parametrize('proto', score.PROTOCOLS, ids=[p[0] for p in score.PROTOCOLS])
def test_by_name_equals_the_sweep_on_the_concatenation(monkeypatch, proto, with_uem, two_speaker):
    monkeypatch.setattr(score, 'score_entries', _host_score_entries)
    _, collar, ignore = proto
    rng = np.random.default_rng(29 + 2 * with_uem + two_speaker)
    for _ in range(6):
        ref, sys = _archive(rng, int(rng.integers(1, 5)), np.arange(5), two_speaker)
        names = sorted({r[0] for r in ref})
        uem = {n: [(1.0, 9.0), (12.5, 60.0)] for n in names} if with_uem else None
        per, tot = score.score_rttm(ref, sys, collar, ignore, uem, overlapping=two_speaker, by_name=True,
                                    across_files=True)
        R, S, U = _concatenated(ref, sys, uem, collar)
        want = _by_name_sweep(R, S, int(score.to_ticks(collar)), ignore, U)
        assert tot['by_name']['ticks'] == want
        assert tot['by_name']['ticks']['conf'] >= tot['across_files']['ticks']['conf']
        plain_per, plain_tot = score.score_rttm(ref, sys, collar, ignore, uem, overlapping=two_speaker)
        assert plain_per == per and plain_tot == {k: v for k, v in tot.items() if k not in ('by_name', 'across_files')}


def test_by_name_with_the_reference_names_and_with_a_swap(monkeypatch):
    monkeypatch.setattr(score, 'score_entries', _host_score_entries)
    # file b is the longer one, so with its names swapped the best mapping across files is the swap
    ref = [('a', 0.0, 5.0, 'x'), ('a', 5.0, 3.0, 'y'), ('a', 9.0, 2.0, 'x'), ('b', 0.0, 20.0, 'y'), ('b', 20.0, 20.0, 'x')]
    sys = [('a', 0.0, 5.5, 'x'), ('a', 5.5, 3.0, 'y'), ('a', 9.0, 2.0, 'x'), ('b', 0.0, 20.0, 'y'), ('b', 20.0, 20.0, 'x')]
    for proto in score.PROTOCOLS:
        _, tot = score.score_rttm(ref, sys, proto[1], proto[2], by_name=True, across_files=True)
        assert tot['by_name'] == tot['across_files'], proto
        swapped = [r[:3] + ({'x': 'y', 'y': 'x'}[r[3]],) if r[0] == 'b' else r for r in sys]
        _, tot2 = score.score_rttm(ref, swapped, proto[1], proto[2], by_name=True, across_files=True)
        assert tot2['by_name']['der'] > tot2['across_files']['der'], proto
        assert tot2['der'] == tot['der'], proto
