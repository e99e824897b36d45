"""Speaker linking across recordings (DESIGN.md section 5.15) on the host: the closed-form LLR against explicit Gaussian
marginals, the speaker table and the cut, and the DER across files against the line-sweep oracle on the recordings
laid end to end on one time axis.  The device accumulation is restated here as a loop over intervals and regions, so
score_rttm's host work runs without a GPU."""
import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import der_oracle, link_oracle
from vbx_b200 import link, score


# ---- the score ---------------------------------------------------------------------------------------------------------

def _log_marginal(X, Phi):
    """log p(X) of the stacked x-vectors X [n,R] of one latent speaker, prior N(0, I): per feature r the column is
    N(0, I + Phi_r 11^T)."""
    n = X.shape[0]
    return sum(multivariate_normal(np.zeros(n), np.eye(n) + Phi[r] * np.ones((n, n))).logpdf(X[:, r])
               for r in range(X.shape[1]))


@pytest.mark.parametrize('c', [1.0, 0.3 / 17])
@pytest.mark.parametrize('seed', range(6))
def test_llr_is_the_log_ratio_of_gaussian_marginals(c, seed):
    rng = np.random.default_rng(seed)
    R = int(rng.integers(1, 6))
    ns, nu = int(rng.integers(1, 6)), int(rng.integers(1, 6))
    Phi = rng.uniform(0.1, 4.0, R)
    Phi[0] = 0.0 if R > 1 else Phi[0]                 # a padded feature contributes nothing
    Xs, Xu = rng.standard_normal((ns, R)) * 2, rng.standard_normal((nu, R)) * 2
    # the score under c equals the c = 1 score of fea * sqrt(c) with Phi * c (same L and b)
    Ys, Yu, P = Xs * np.sqrt(c), Xu * np.sqrt(c), Phi * c
    want = _log_marginal(np.vstack([Ys, Yu]), P) - _log_marginal(Ys, P) - _log_marginal(Yu, P)
    got = link_oracle.llr([ns, nu], [Xs.sum(0), Xu.sum(0)], Phi, c)
    assert abs(got[0, 1] - want) <= 1e-10 * max(1.0, abs(want)), (got[0, 1], want)
    assert got[0, 1] == got[1, 0] or abs(got[0, 1] - got[1, 0]) <= 1e-12 * abs(want)


def test_llr_is_symmetric_and_zero_without_x_vectors():
    rng = np.random.default_rng(3)
    n = np.array([0, 3, 1, 7, 0, 2], dtype=np.float64)
    F = rng.standard_normal((6, 8)) * n[:, None]
    Phi = rng.uniform(0, 3, 8)
    L = link_oracle.llr(n, F, Phi, 0.3 / 17)
    np.testing.assert_allclose(L, L.T, rtol=1e-13, atol=1e-13)
    assert not L[[0, 4]].any() and not L[:, [0, 4]].any()
    d = link_oracle.distances(n, F, Phi, 0.3 / 17, np.array([0, 0, 1, 1, 2, 3]))
    assert d[0, 1] == link.BIG and d[2, 3] == link.BIG and not np.diag(d).any()


# ---- the table and the cut -----------------------------------------------------------------------------------------

def test_speaker_table_order():
    t = link.speaker_table([np.array([2, 0, 2]), np.zeros(0, dtype=np.int64), np.array([5, 1, 1, 5, 3]), np.array([0])])
    assert t.rec.tolist() == [0, 0, 2, 2, 2, 3] and t.label.tolist() == [0, 2, 1, 3, 5, 0] and t.n_recordings == 4


def test_cut_numbering_and_second_only_labels():
    table = link.speaker_table([np.array([0, 1]), np.array([0, 1]), np.array([0])])
    # speakers 0..4 = (0,0) (0,1) (1,0) (1,1) (2,0); (0,1)~(1,0) at LLR 10, (0,0)~(2,0) at LLR 5, the rest far apart
    llr = np.full((5, 5), -50.0)
    for a, b, v in ((1, 2, 10.0), (0, 4, 5.0)):
        llr[a, b] = llr[b, a] = v
    d = -llr
    for a, b in ((0, 1), (2, 3)):
        d[a, b] = d[b, a] = link.BIG
    np.fill_diagonal(d, 0)
    Z = link_oracle.link(d)
    maps = link.link_cut(Z, table, 0.0, labels2=[np.array([1, 3]), None, np.array([-1])])
    # first appearance over the table: (0,0) -> 0, (0,1) -> 1, (1,0) -> 1, (1,1) -> 2, (2,0) -> 0; label 3 of
    # recording 0 occurs only as a second label and comes after all linked ids
    assert maps == [{0: 0, 1: 1, 3: 3}, {0: 1, 1: 2}, {0: 0}]
    assert link.link_cut(Z, table, 7.0) == [{0: 0, 1: 1}, {0: 1, 1: 2}, {0: 3}]
    assert link.link_cut(Z, table, 20.0) == [{0: 0, 1: 1}, {0: 2, 1: 3}, {0: 4}]
    assert link.link_cut(Z, table, -1e6)[0] == {0: 0, 1: 1}           # cannot-link pairs stay apart
    for bad in (1.1e15, -2e15, float('nan'), float('inf')):
        with pytest.raises(ValueError):
            link.link_cut(Z, table, bad)


def test_raising_the_threshold_only_splits():
    rng = np.random.default_rng(5)
    recs = [rng.integers(0, 4, 20) for _ in range(8)]
    table = link.speaker_table(recs)
    M = len(table.rec)
    n = rng.integers(1, 30, M).astype(np.float64)
    centers = rng.standard_normal((5, 16)) * 3
    F = (centers[rng.integers(0, 5, M)] + 0.3 * rng.standard_normal((M, 16))) * n[:, None]
    d = link_oracle.distances(n, F, np.full(16, 2.0), 0.3 / 17, table.rec)
    Z = link_oracle.link(d)
    prev = None
    for t in np.concatenate([[-1e6], np.linspace(-200, 200, 41), [1e6]]):
        maps = link.link_cut(Z, table, t)
        g = np.array([maps[b][l] for b, l in zip(table.rec.tolist(), table.label.tolist())])
        for b in range(len(recs)):
            assert len(set(g[table.rec == b])) == int(np.sum(table.rec == b))
        if prev is not None:           # every new cluster lies inside one old cluster
            for k in np.unique(g):
                assert len(set(prev[g == k])) == 1
        prev = g


# ---- DER across files ------------------------------------------------------------------------------------------------

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
    """Reference and system rows of n_files recordings drawn from a pool of speakers (names shared across files)."""
    ref, sys = [], []
    for f in range(n_files):
        name = f'rec{f}'
        spk = rng.choice(pool, int(rng.integers(1, 4)), replace=False)
        t = float(rng.integers(0, 8))
        for _ in range(int(rng.integers(3, 9))):
            k = spk[int(rng.integers(len(spk)))]
            d = float(rng.integers(1, 40)) / 4
            ref.append((name, t, d, str(k)))
            if rng.random() < 0.3:                         # a second reference speaker overlapping
                ref.append((name, t + d / 2, d, str(spk[int(rng.integers(len(spk)))])))
            t += d + float(rng.integers(0, 8)) / 4
        layers = 2 if two_speaker else 1
        for layer in range(layers):
            cuts = np.unique(rng.integers(0, int(4 * t) + 8, 8)) / 4.0
            sys += [(name, float(a), float(b - a), f'g{int(rng.integers(0, len(pool) + 1)) * layers + layer}')
                    for a, b in zip(cuts[:-1], cuts[1:]) if rng.random() < 0.7]
    return ref, sys


def _concatenated(ref, sys, uem, collar):
    """The recordings laid end to end: each shifted past the previous one's last boundary plus two collars."""
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


@pytest.mark.parametrize('two_speaker', [False, True])
@pytest.mark.parametrize('with_uem', [False, True])
@pytest.mark.parametrize('proto', score.PROTOCOLS, ids=[p[0] for p in score.PROTOCOLS])
def test_der_across_files_equals_the_oracle_on_the_concatenation(monkeypatch, proto, with_uem, two_speaker):
    monkeypatch.setattr(score, 'score_entries', _host_score_entries)
    _, collar, ignore = proto
    rng = np.random.default_rng(17 + 2 * with_uem + two_speaker)
    for _ in range(6):
        ref, sys = _archive(rng, int(rng.integers(1, 5)), np.arange(5), two_speaker)
        names = sorted({r[0] for r in ref})
        uem = {n: [(1.0, 9.0), (12.5, 60.0)] for n in names} if with_uem else None
        per, tot = score.score_rttm(ref, sys, collar, ignore, uem, overlapping=two_speaker, across_files=True)
        R, S, U = _concatenated(ref, sys, uem, collar)
        want = der_oracle.der_ticks(R, S, int(score.to_ticks(collar)), ignore, U)
        assert tot['across_files']['ticks'] == want
        assert {k: tot['ticks'][k] for k in ('miss', 'fa', 'scored')} == {k: want[k] for k in ('miss', 'fa', 'scored')}
        assert tot['across_files']['ticks']['conf'] >= tot['ticks']['conf']
        if len(names) == 1:
            assert tot['across_files'] == per[names[0]]
        plain_per, plain_tot = score.score_rttm(ref, sys, collar, ignore, uem, overlapping=two_speaker)
        assert plain_per == per and plain_tot == {k: v for k, v in tot.items() if k != 'across_files'}


def test_one_file_across_files_is_the_file(monkeypatch):
    monkeypatch.setattr(score, 'score_entries', _host_score_entries)
    ref = [('a', 0.0, 5.0, 'x'), ('a', 5.0, 3.0, 'y'), ('a', 9.0, 2.0, 'x')]
    sys = [('a', 0.0, 6.0, '1'), ('a', 6.0, 5.0, '2')]
    per, tot = score.score_rttm(ref, sys, 0.25, False, across_files=True)
    assert tot['across_files'] == per['a'] == {k: v for k, v in tot.items() if k != 'across_files'}


@pytest.mark.parametrize('two_speaker', [False, True])
def test_across_files_with_empty_system_turns(monkeypatch, two_speaker):
    """System speakers whose turns all have zero length (here named last in their file, so the overlap block has no
    column for them) and a file whose every system turn is empty: the DER across files still equals the oracle."""
    monkeypatch.setattr(score, 'score_entries', _host_score_entries)
    ref = [('a', 0.0, 5.0, 'x'), ('a', 5.0, 3.0, 'y'), ('b', 1.0, 4.0, 'x'), ('c', 0.0, 2.0, 'y')]
    sys = [('a', 0.0, 6.0, '1'), ('a', 6.0, 2.0, '2'), ('a', 9.0, 0.0, '9'), ('a', 3.0, 0.0000004, 'z'),
           ('b', 1.0, 4.0, '2'), ('b', 2.0, 0.0, '9'), ('c', 0.5, 0.0, '1'), ('c', 1.0, 0.0, '3')]
    if two_speaker:
        sys.append(('a', 4.0, 2.0, '2'))
    for proto in score.PROTOCOLS:
        per, tot = score.score_rttm(ref, sys, proto[1], proto[2], overlapping=two_speaker, across_files=True)
        R, S, _ = _concatenated(ref, sys, None, proto[1])
        assert tot['across_files']['ticks'] == der_oracle.der_ticks(R, S, int(score.to_ticks(proto[1])), proto[2]), proto


def test_named_reference_turns_keep_reference_turns():
    rows = [('a', 1.0, 2.0, 'z'), ('a', 0.0, 1.0, 'b'), ('a', 3.0, 0.0, 'e'), ('b', 0.0, 1.0, 'q')]
    named = score.named_reference_turns(rows)
    plain = score.reference_turns(rows)
    assert [k for k, _ in named['a']] == ['b', 'z'] and [k for k, _ in named['b']] == ['q']
    for rec in plain:
        assert len(plain[rec]) == len(named[rec])
        for (s, e), (_, (s2, e2)) in zip(plain[rec], named[rec]):
            assert np.array_equal(s, s2) and np.array_equal(e, e2)
