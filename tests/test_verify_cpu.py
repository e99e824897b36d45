"""Speaker-verification trials (DESIGN.md section 5.27) on the host: the oracle's metrics on the worked case, its LLR
against explicit Gaussian marginals, the metrics' invariances, the trial-list reader and the command line's usage
errors."""
import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import verify_oracle as O
from vbx_b200 import formats, verify


def _log_marginal(X, Phi):
    """log p(X) of the stacked x-vectors X [n,R] of one latent speaker, prior N(0, I): per feature r the column is
    N(0, I + Phi_r 11^T)."""
    n = X.shape[0]
    return sum(multivariate_normal(np.zeros(n), np.eye(n) + Phi[r] * np.ones((n, n))).logpdf(X[:, r])
               for r in range(X.shape[1]))


def worked_case():
    return np.array([3.0, 1.0, 1.0, 2.0, 1.0, 0.0, -1.0]), np.array([1, 1, 1, 0, 0, 0, 0], dtype=bool)


def test_worked_case():
    s, y = worked_case()
    m = O.error_rates(s, y, p_targets=(0.5, 0.25))
    assert m['candidates'].tolist() == [-1.0, 0.0, 1.0, 2.0, 3.0, np.inf]
    assert np.allclose(m['p_miss'], [0, 0, 0, 2 / 3, 2 / 3, 1], rtol=0, atol=1e-16)
    assert np.allclose(m['p_fa'], [1, 3 / 4, 1 / 2, 1 / 4, 0, 0], rtol=0, atol=1e-16)
    assert abs(m['eer'] - 4 / 11) <= 1e-15
    assert abs(m['min_dcf'][0] - 0.5) <= 1e-15 and m['threshold'][0] == 1.0
    assert abs(m['act_dcf'][0] - 0.75) <= 1e-15
    assert abs(m['min_dcf'][1] - 2 / 3) <= 1e-15 and m['threshold'][1] == 3.0
    assert abs(m['act_dcf'][1] - 17 / 12) <= 1e-15
    assert (m['n_target'], m['n_nontarget']) == (3, 4)


@pytest.mark.parametrize('c', [1.0, 0.3 / 17])
@pytest.mark.parametrize('seed', range(4))
def test_llr_is_the_log_ratio_of_gaussian_marginals(c, seed):
    rng = np.random.default_rng(100 + seed)
    R = int(rng.integers(1, 6))
    ne, nt = int(rng.integers(1, 5)), int(rng.integers(1, 5))
    Phi = rng.uniform(0.1, 4.0, R)
    Xe, Xt = rng.standard_normal((ne, R)) * 2, rng.standard_normal((nt, R)) * 2
    Ye, Yt, P = Xe * np.sqrt(c), Xt * np.sqrt(c), Phi * c
    want = _log_marginal(np.vstack([Ye, Yt]), P) - _log_marginal(Ye, P) - _log_marginal(Yt, P)
    ve, Fe = O.statistics(Xe, np.zeros(ne, dtype=int), 1)
    vt, Ft = O.statistics(Xt, np.zeros(nt, dtype=int), 1)
    got = O.llr_trials(ve, Fe, vt, Ft, Phi, c, [0], [0])[0]
    assert abs(got - want) <= 1e-10 * max(1.0, abs(want)), (got, want)


def random_trials(T, seed, ties=False):
    rng = np.random.default_rng(seed)
    y = rng.random(T) < 0.3
    s = np.where(y, 2.0, 0.0) + rng.standard_normal(T) * 1.5
    if ties:
        s = np.round(s)
    y[0], y[1] = True, False
    return s, y


def same_metrics(a, b):
    for k in ('eer', 'min_dcf', 'threshold', 'act_dcf', 'n_target', 'n_nontarget'):
        assert a[k] == b[k], k
    assert abs(a['cllr'] - b['cllr']) <= 1e-12 * abs(b['cllr'])


@pytest.mark.parametrize('ties', [False, True])
def test_metrics_ignore_the_order_of_the_trials(ties):
    s, y = random_trials(5000, 3, ties)
    p = np.random.default_rng(4).permutation(len(s))
    same_metrics(O.error_rates(s[p], y[p], (0.01, 0.3)), O.error_rates(s, y, (0.01, 0.3)))


def test_a_constant_shift_moves_the_thresholds_only():
    s, y = random_trials(3000, 5, ties=True)
    a, b = O.error_rates(s, y, (0.01, 0.2, 0.5)), O.error_rates(s + 4.0, y, (0.01, 0.2, 0.5))
    assert a['eer'] == b['eer'] and a['min_dcf'] == b['min_dcf']
    assert np.array_equal(np.array(a['threshold']) + 4.0, b['threshold'])


def test_signed_zeros_are_one_value():
    s = np.array([-0.0, 0.0, 1.0, -1.0])
    y = np.array([1, 0, 1, 0], dtype=bool)
    m = O.error_rates(s, y, (0.5,))
    assert m['candidates'].tolist() == [-1.0, 0.0, 1.0, np.inf]


# ---- trial lists --------------------------------------------------------------------------------------------------------

def write(tmp_path, text, name='trials'):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_read_trials(tmp_path):
    e, t, y = formats.read_trials(write(tmp_path, 'a x target\n\nb y nontarget\na x target\n'))
    assert e == ['a', 'b', 'a'] and t == ['x', 'y', 'x'] and y.tolist() == [True, False, True]
    e, t, y = formats.read_trials(write(tmp_path, 'a x\nb y\n'), ['a', 'b'], ['x', 'y'])
    assert e == ['a', 'b'] and t == ['x', 'y'] and y is None


@pytest.mark.parametrize('text, match', [
    ('a x target\nb y\n', 'mixed'),
    ('a x maybe\n', 'neither'),
    ('a x target extra\n', 'expected'),
    ('a\n', 'expected'),
    ('\n\n', 'no trials'),
    ('a x target\nc y nontarget\n', r':2: .*enrolment'),
    ('a x target\nb z nontarget\n', r':2: .*test'),
])
def test_read_trials_refusals(tmp_path, text, match):
    with pytest.raises(ValueError, match=match):
        formats.read_trials(write(tmp_path, text), ['a', 'b'], ['x', 'y'])


def test_check_p_targets():
    assert verify.check_p_targets([0.5, 0.01]) == [0.5, 0.01] and verify.check_p_targets(0.25) == [0.25]
    for bad in ([0.0], [1.0], [-0.1], [np.nan], []):
        with pytest.raises(ValueError):
            verify.check_p_targets(bad)


@pytest.mark.parametrize('extra', [
    ['--cohort-ark', 'c.ark'],
    ['--cohort-top', '10'],
    ['--cohort-ark', 'c.ark', '--cohort-utt2spk', 'u', '--cohort-top', '1'],
    ['--p-target', '0.5,1.5'],
    ['--p-target', 'x'],
    ['--c-miss', '0'],
    ['--c-fa', 'inf'],
    ['--Fa', '-1'],
    ['--Fb', 'nan'],
    ['--chain', 'fp16'],
])
def test_usage_errors_exit_2(extra, capsys):
    base = ['--trials', 't', '--enroll-ark', 'e.ark', '--test-ark', 't.ark', '--xvec-transform', 'x.npz',
            '--plda-file', 'plda']
    with pytest.raises(SystemExit) as e:
        verify.main(base + extra)
    assert e.value.code == 2


def test_metrics_need_both_classes_before_any_device_work():
    with pytest.raises(ValueError, match='target and nontarget'):
        verify.error_rates(np.zeros(4), np.ones(4, dtype=bool))
    with pytest.raises(ValueError, match='p_target'):
        verify.error_rates(np.zeros(4), np.array([1, 0, 0, 0]), p_targets=(2.0,))
    with pytest.raises(ValueError, match='c_miss'):
        verify.error_rates(np.zeros(4), np.array([1, 0, 0, 0]), c_miss=0.0)


def test_score_checks_before_any_device_work():
    fea, item, Phi = np.ones((3, 4)), np.array([0, 1, 1]), np.ones(4)
    with pytest.raises(ValueError, match='outside'):
        verify.score_trials(fea, item, fea, item, Phi, [[0, 2]])
    with pytest.raises(ValueError, match='non-finite'):
        verify.score_trials(np.full((3, 4), np.nan), item, fea, item, Phi, [[0, 1]])
    with pytest.raises(ValueError, match='dimension'):
        verify.score_trials(np.ones((3, 5)), item, fea, item, Phi, [[0, 1]])
    with pytest.raises(ValueError, match='Fa'):
        verify.score_trials(fea, item, fea, item, Phi, [[0, 1]], Fa=0.0)
    with pytest.raises(ValueError, match='Fb'):
        verify.score_trials(fea, item, fea, item, Phi, [[0, 1]], Fb=np.inf)
