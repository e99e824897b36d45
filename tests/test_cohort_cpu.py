"""Score normalisation against a cohort (DESIGN.md section 5.17) without a GPU: the oracle (oracle/norm_oracle.py)
against explicit definitions, ties at the K-th value and top_k >= C, the worked case of DESIGN.md, the argument errors
(all before any device work) and the pairing of the command-line options."""
import numpy as np
import pytest

from oracle import link_oracle, norm_oracle
from vbx_b200 import cohort


def _explicit(row, top_k):
    """mu and sigma from the definition: the K largest values one at a time, a tie at the K-th value taking copies."""
    vals = sorted((float(v) for v in row), reverse=True)[:min(top_k, len(row))]
    mu = sum(vals) / len(vals)
    return mu, (sum((v - mu) ** 2 for v in vals) / len(vals)) ** 0.5


@pytest.mark.parametrize('top_k', [2, 3, 5, 9, 10, 15])
def test_top_stats_equal_the_definition(top_k):
    rng = np.random.default_rng(top_k)
    S = np.round(rng.standard_normal((7, 10)) * 4)          # integers: ties at the K-th value are common
    S[0] = 3.0                                             # every value tied
    S[1, :4] = S[1].max()                                  # the largest value four times
    mu, sd = norm_oracle.top_stats(S, top_k)
    for i, row in enumerate(S):
        m, s = _explicit(row, top_k)
        assert mu[i] == pytest.approx(m, rel=1e-15, abs=1e-15) and sd[i] == pytest.approx(s, rel=1e-13, abs=1e-15)
    assert sd[0] == 0.0
    if top_k >= 10:                                        # top_k >= C: every cohort score (plain S-norm)
        np.testing.assert_array_equal(mu, S.mean(axis=1))
        np.testing.assert_allclose(sd, S.std(axis=1), rtol=1e-15)


def test_normalised_score_is_symmetric_and_explicit():
    rng = np.random.default_rng(1)
    M, R, c = 6, 5, 0.3 / 17
    n = rng.integers(1, 9, M).astype(np.float64)
    F = rng.standard_normal((M, R)) * n[:, None]
    Phi = rng.uniform(0.5, 3, R)
    L = link_oracle.llr(n, F, Phi, c)
    mu, sd = rng.standard_normal(M) * 5, rng.uniform(0.5, 4, M)
    S = norm_oracle.normalise(L, mu, sd, mu, sd)
    Ls = 0.5 * (L + L.T)                                   # the oracle's LLR is symmetric to rounding; this one exactly
    np.testing.assert_array_equal(norm_oracle.normalise(Ls, mu, sd, mu, sd), norm_oracle.normalise(Ls, mu, sd, mu, sd).T)
    for i in range(M):
        for j in range(M):
            assert S[i, j] == pytest.approx(0.5 * ((L[i, j] - mu[i]) / sd[i] + (L[i, j] - mu[j]) / sd[j]), rel=1e-14)
    rec = np.array([0, 0, 1, 1, 2, 3])
    d = norm_oracle.link_distances(n, F, Phi, c, rec, mu, sd)
    assert (np.diag(d) == 0).all() and d[0, 1] == d[2, 3] == link_oracle.BIG
    assert d[0, 2] == -S[0, 2]


def test_cohort_llr_is_the_enrolment_llr():
    rng = np.random.default_rng(2)
    n, nc = rng.integers(1, 5, 4).astype(float), rng.integers(1, 5, 3).astype(float)
    F, Fc, Phi = rng.standard_normal((4, 6)), rng.standard_normal((3, 6)), rng.uniform(0.2, 2, 6)
    full = link_oracle.llr(np.concatenate([n, nc]), np.vstack([F, Fc]), Phi, 0.1)
    np.testing.assert_array_equal(norm_oracle.cohort_llr(n, F, nc, Fc, Phi, 0.1), full[:4, 4:])


def test_worked_case():
    """DESIGN.md section 5.17: x scores (10, 6, 4, 2) and y (3, 1, 1, -5) against four cohort speakers; at top_k = 2,
    mu_x = 8, sigma_x = 2, mu_y = 2, sigma_y = 1, and LLR(x, y) = 12 normalises to 1/2 (4/2 + 10/1) = 6.  At top_k = 3
    y's third score ties with its second: mu_y = 5/3, sigma_y = sqrt(8/9).  At top_k >= 4 (S-norm) all four count."""
    co = np.array([[10.0, 6.0, 4.0, 2.0], [3.0, 1.0, 1.0, -5.0]])
    mu, sd = norm_oracle.top_stats(co, 2)
    assert mu.tolist() == [8.0, 2.0] and sd.tolist() == [2.0, 1.0]
    S = norm_oracle.normalise(np.array([[12.0]]), mu[:1], sd[:1], mu[1:], sd[1:])
    assert S.tolist() == [[6.0]]
    mu3, sd3 = norm_oracle.top_stats(co, 3)
    assert mu3[1] == pytest.approx(5 / 3) and sd3[1] == pytest.approx((8 / 9) ** 0.5)
    mu4, sd4 = norm_oracle.top_stats(co, 4)
    assert mu4.tolist() == [5.5, 0.0] and sd4[1] == 3.0
    assert norm_oracle.top_stats(co, 100)[0].tolist() == mu4.tolist()


def test_normalised_assignment_oracle():
    S = np.array([[2.0, 0.5], [1.5, -1.0]])
    a, obj = norm_oracle.assign(S, np.array([0, 2]), 1.0)
    # C = [[-1, 0.5, 0, 0], [-0.5, 2, 0, 0]]: k0 -> 0 with k1 unknown costs -1, k0 -> 1 with k1 -> 0 costs 0, k1 -> 0
    # alone -0.5
    assert a.tolist() == [0, -1] and obj.tolist() == [-1.0]


def test_argument_errors_come_before_device_work(monkeypatch):
    from vbx_b200 import pipeline
    import torch
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: (_ for _ in ()).throw(AssertionError('device touched')))
    recs = {'r': (np.zeros((3, 8)), np.zeros((3, 2)))}
    ok = {'a': np.ones((2, 8)), 'b': np.ones((1, 8))}
    enr = dict(enroll={'alice': np.ones((2, 8))}, enroll_threshold=0.0)
    bad = [(dict(cohort={}, link_threshold=0.0), 'non-empty'),
           (dict(cohort={'a': np.ones((3, 8))}, link_threshold=0.0), 'at least 2'),
           (dict(cohort={'a': np.ones((3, 8)), 'b': np.ones((0, 8))}, **enr), 'at least one'),
           (dict(cohort={'a': np.ones((3, 8)), 'b': np.ones((2, 7))}, link_threshold=0.0), 'dimension 7'),
           (dict(cohort=ok), 'needs link_threshold or enroll'),
           (dict(cohort=ok, cohort_top=1, link_threshold=0.0), 'top_k'),
           (dict(cohort=ok, cohort_top=2.5, **enr), 'top_k'),
           (dict(cohort=[np.ones((2, 8))], link_threshold=0.0), 'dict')]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pipeline.diarize_batch(recs, None, None, 0.3, 17.0, 0.99, **kw)
    fea, Phi = np.zeros((3, 4)), np.ones(4)
    with pytest.raises(ValueError, match='at least 2'):
        cohort.cohort_stats(fea, Phi, [0, 3], [np.zeros(3)], np.zeros((2, 4)), [0, 0], 0.3, 17.0)
    with pytest.raises(ValueError, match='every cohort speaker'):
        cohort.cohort_stats(fea, Phi, [0, 3], [np.zeros(3)], np.zeros((2, 4)), [0, 2], 0.3, 17.0)
    with pytest.raises(ValueError, match='top_k'):
        cohort.cohort_stats(fea, Phi, [0, 3], [np.zeros(3)], np.zeros((2, 4)), [0, 1], 0.3, 17.0, top_k=1)
    with pytest.raises(ValueError, match='every scored speaker'):
        cohort.cohort_stats(fea, Phi, None, [0, 2, 2], np.zeros((2, 4)), [0, 1], 0.3, 17.0)


def test_spread_check_names_the_speakers():
    cohort.check_spread([1.0, 3.0], ['a', 'b'])
    for std, who in (([1.0, 0.0], 'b'), ([np.nan, 1.0], 'a'), ([1.0, np.inf], 'b'), ([1e-7, 2.0], 'a')):
        with pytest.raises(ValueError, match=f'{who} '):
            cohort.check_spread(std, ['a', 'b'])


def test_cli_cohort_options_go_together(capsys):
    from vbx_b200 import cli
    base = ['--init', 'AHC+VB', '--out-rttm-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform',
            't', '--plda-file', 'p', '--threshold', '0', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']
    cases = [(['--cohort-ark', 'c', '--link-threshold', '0'], 'go together'),
             (['--cohort-utt2spk', 'u', '--link-threshold', '0'], 'go together'),
             (['--cohort-top', '50', '--link-threshold', '0'], 'needs --cohort-ark'),
             (['--cohort-ark', 'c', '--cohort-utt2spk', 'u'], 'give --link-threshold or the enrolment'),
             (['--cohort-ark', 'c', '--cohort-utt2spk', 'u', '--cohort-top', '1', '--link-threshold', '0'], '>= 2')]
    for extra, msg in cases:
        with pytest.raises(SystemExit):
            cli.main(base + extra)
        assert msg in capsys.readouterr().err, extra
