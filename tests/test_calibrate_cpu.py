"""Score calibration (DESIGN.md section 5.28) on the host: the oracle's fit and minCllr on the worked case, its Newton
state machine against scipy, PAV as sequential pooling against the ROC hull, the invariances of minCllr, separable
lists, calibration files and the usage errors of both command lines."""
import json
import math

import numpy as np
import pytest
from scipy.optimize import minimize

from oracle import calibrate_oracle as O
from vbx_b200 import cli, verify


def worked_case():
    return np.array([3.0, 1.0, 1.0, 2.0, 1.0, 0.0, -1.0]), np.array([1, 1, 1, 0, 0, 0, 0], dtype=bool)


def rel(got, want):
    return abs(got - want) / max(abs(want), 1e-300)


def test_worked_case():
    s, y = worked_case()
    assert O.roc_hull(s, y) == [(4, 3), (2, 3), (0, 1), (0, 0)]          # from (N_non, N_tar) to (0, 0)
    assert O.pav_blocks(s, y) == [(0, 2), (2, 2), (1, 0)]
    want = (2 / 3 * math.log(7 / 4) + 0.5 * math.log(7 / 3)) / (2 * math.log(2))
    assert rel(want, 0.5747164126866467) <= 1e-15
    assert rel(O.min_cllr(s, y), want) <= 1e-15
    f = O.fit(s, y, 0.5)
    assert f['status'] == 0
    assert rel(f['a'], 1.0775784972559423) <= 1e-10 and rel(f['b'], -1.1648381046978393) <= 1e-10
    assert rel(f['cllr_prior'], 0.8034306752311062) <= 1e-12
    f = O.fit(s, y, 0.01)
    assert f['status'] == 0
    assert rel(f['a'], 1.2683733645220252) <= 1e-10 and rel(f['b'], -1.4891900440709454) <= 1e-10


def random_list(seed, T=400, ties=False):
    rng = np.random.default_rng(seed)
    y = rng.random(T) < 0.3
    y[:2] = [True, False]
    s = rng.standard_normal(T) + 1.5 * y
    if ties:
        s = np.round(s * 3) / 3
    return s, y


def objective(w, s, y, prior):
    a, b = w
    z = a * s + b + math.log(prior / (1 - prior))
    return (prior * np.mean(O.softplus(-z[y])) + (1 - prior) * np.mean(O.softplus(z[~y]))) / math.log(2)


def gradient(w, s, y, prior):
    """The gradient of objective, by scipy's logistic function."""
    from scipy.special import expit
    a, b = w
    z = a * s + b + math.log(prior / (1 - prior))
    r = np.where(y, -expit(-z), expit(z)) * np.where(y, prior / y.sum(), (1 - prior) / (~y).sum())
    return np.array([np.sum(r * s), np.sum(r)]) / math.log(2)


@pytest.mark.parametrize('prior', [0.5, 0.01, 0.9])
@pytest.mark.parametrize('seed', range(3))
def test_fit_agrees_with_scipy(prior, seed):
    s, y = random_list(seed)
    f = O.fit(s, y, prior)
    assert f['status'] == 0 and f['passes'] < O.MAX_PASSES
    r = minimize(objective, [0.0, 0.0], args=(s, y, prior), jac=gradient, method='BFGS', options=dict(gtol=1e-15))
    assert abs(f['a'] - r.x[0]) <= 1e-9 * max(1.0, abs(r.x[0]))
    assert abs(f['b'] - r.x[1]) <= 1e-9 * max(1.0, abs(r.x[1]))
    assert f['cllr_prior'] <= r.fun * (1 + 1e-14)
    assert rel(f['cllr_prior'], objective([f['a'], f['b']], s, y, prior)) <= 1e-12


@pytest.mark.parametrize('seed', range(6))
def test_pav_blocks_are_the_hull_segments(seed):
    s, y = random_list(seed, T=300, ties=True)
    blocks = O.pav_blocks(s, y)
    assert O.hull_segments(O.roc_hull(s, y)) == blocks
    frac = [t / (t + n) for t, n in blocks]
    assert all(a < b for a, b in zip(frac, frac[1:]))                   # strictly increasing after pooling


@pytest.mark.parametrize('seed', range(4))
def test_min_cllr_ignores_strictly_increasing_maps(seed):
    s, y = random_list(seed, ties=seed % 2 == 1)
    m = O.min_cllr(s, y)
    for g in (lambda v: 3.0 * v - 7.0, np.exp, lambda v: v ** 3 + v):
        assert rel(O.min_cllr(g(s), y), m) <= 1e-13
    assert O.roc_hull(np.exp(s), y) == O.roc_hull(s, y)


@pytest.mark.parametrize('seed', range(4))
def test_min_cllr_is_at_most_the_calibrated_cllr(seed):
    s, y = random_list(seed, ties=seed % 2 == 1)
    assert O.min_cllr(s, y) <= O.fit(s, y, 0.5)['cllr_prior'] + 1e-15


def test_separable_lists():
    y = np.array([1, 1, 0, 0, 0], dtype=bool)
    s = np.array([2.0, 1.0, 1.0, 0.0, -1.0])                           # targets at or above every nontarget
    assert O.separable(s, y) == 'above'
    c = O.calibrate(s, y)
    assert c['status'] == 1 and math.isnan(c['a']) and 0.0 < c['min_cllr'] < 1.0     # one tie across the classes
    assert O.min_cllr(np.array([2.0, 1.5, 1.0, 0.0, -1.0]), y) == 0.0  # strictly separated: exactly 0
    assert O.separable(-s, y) == 'below'
    assert O.calibrate(-s, y)['status'] == 1
    # the optimal monotone transform cannot reverse the order: every trial pools into one block, minCllr = 1
    assert rel(O.min_cllr(np.array([-2.0, -1.5, 1.0, 2.0, 3.0]), y), 1.0) <= 1e-15


def test_calibrate_checks_before_any_device_work():
    with pytest.raises(ValueError, match='no trials'):
        verify.calibrate(np.zeros(0), np.zeros(0))
    with pytest.raises(ValueError, match='target and nontarget'):
        verify.calibrate(np.zeros(4), np.ones(4, dtype=bool))
    with pytest.raises(ValueError, match='labels'):
        verify.calibrate(np.zeros(4), np.ones(3, dtype=bool))
    with pytest.raises(ValueError, match='prior'):
        verify.calibrate(np.zeros(2), np.array([1, 0]), prior=1.0)


# ---- calibration files -------------------------------------------------------------------------------------------------

def model_files(tmp_path):
    tf, plda = tmp_path / 'transform.npz', tmp_path / 'plda'
    tf.write_bytes(b'transform bytes')
    plda.write_bytes(b'plda bytes')
    return str(tf), str(plda)


def write_cal(tmp_path, kind='llr', Fa=0.3, Fb=17.0, lda_dim=128, top=None, a=1.5, b=-2.0, prior=0.5):
    tf, plda = model_files(tmp_path)
    path = str(tmp_path / 'cal.json')
    fit = dict(a=a, b=b, prior=prior, n_target=10, n_nontarget=90)
    verify.write_calibration(path, fit, kind, Fa, Fb, lda_dim, top, tf, plda)
    return path, tf, plda


def test_calibration_file_round_trip(tmp_path):
    path, tf, plda = write_cal(tmp_path, kind='as-norm', top=50, a=1.0775784972559423, b=-1.1648381046978393)
    cal = verify.read_calibration(path)
    assert cal['a'] == 1.0775784972559423 and cal['b'] == -1.1648381046978393
    assert (cal['score_kind'], cal['Fa'], cal['Fb'], cal['lda_dim'], cal['cohort_top']) == ('as-norm', 0.3, 17.0, 128, 50)
    assert (cal['n_target'], cal['n_nontarget'], cal['prior']) == (10, 90, 0.5)
    assert cal['xvec_transform_sha256'] == verify.file_sha256(tf)
    assert verify.calibration_mismatch(cal, 'as-norm', 0.3, 17.0, 128, 50, tf, plda) is None
    assert verify.raw_threshold(cal, 0.0) == (0.0 - cal['b']) / cal['a']
    path, _, _ = write_cal(tmp_path)
    assert verify.read_calibration(path)['cohort_top'] is None


@pytest.mark.parametrize('edit, match', [
    (dict(version=2), 'version'),
    (dict(version=None), 'version'),
    (dict(a=None), 'a must be a finite number'),
    (dict(b='x'), 'b must be a finite number'),
    (dict(prior=1.0), 'prior'),
    (dict(Fa=0.0), 'Fa and Fb'),
    (dict(score_kind='plda'), 'score_kind'),
    (dict(lda_dim=0), 'lda_dim'),
    (dict(n_target=1.5), 'n_target'),
    (dict(cohort_top=10), 'cohort_top'),
    (dict(plda_file_sha256='abc'), 'SHA-256'),
])
def test_calibration_file_refusals(tmp_path, edit, match):
    path, _, _ = write_cal(tmp_path)
    doc = json.load(open(path))
    doc.update(edit)
    with open(path, 'w') as f:
        json.dump(doc, f)
    with pytest.raises(ValueError, match=match):
        verify.read_calibration(path)


@pytest.mark.parametrize('key', verify.CALIBRATION_KEYS)
def test_calibration_file_refuses_missing_keys(tmp_path, key):
    path, _, _ = write_cal(tmp_path)
    doc = json.load(open(path))
    del doc[key]
    with open(path, 'w') as f:
        json.dump(doc, f)
    with pytest.raises(ValueError, match='version' if key == 'version' else 'missing'):
        verify.read_calibration(path)


def test_calibration_file_refuses_non_finite_values_and_other_files(tmp_path):
    path, _, _ = write_cal(tmp_path)
    text = open(path).read().replace('"a": 1.5', '"a": NaN')
    open(path, 'w').write(text)
    with pytest.raises(ValueError, match='finite'):
        verify.read_calibration(path)
    open(path, 'w').write('[1, 2]')
    with pytest.raises(ValueError, match='not a calibration file'):
        verify.read_calibration(path)
    open(path, 'w').write('{')
    with pytest.raises(ValueError, match='not a calibration file'):
        verify.read_calibration(path)


def test_raw_threshold_refuses_a_slope_that_is_not_positive():
    assert verify.raw_threshold(dict(a=2.0, b=1.0), 5.0) == 2.0
    for a in (0.0, -1.0):
        with pytest.raises(ValueError, match='not positive'):
            verify.raw_threshold(dict(a=a, b=0.0), 0.0)


def test_mismatches(tmp_path):
    path, tf, plda = write_cal(tmp_path)
    cal = verify.read_calibration(path)
    ok = ['llr', 0.3, 17.0, 128, None, tf, plda]
    assert verify.calibration_mismatch(cal, *ok) is None
    for k, v in ((0, 'as-norm'), (1, 0.4), (2, 16.0), (3, 64)):
        a = list(ok)
        a[k] = v
        if k == 0:
            a[4] = 200
        assert verify.calibration_mismatch(cal, *a) is not None, k
    other = tmp_path / 'other'
    other.write_bytes(b'another plda')
    assert 'plda' in verify.calibration_mismatch(cal, *ok[:6], str(other))
    assert 'xvec-transform' in verify.calibration_mismatch(cal, *ok[:5], str(other), plda)


# ---- command lines -----------------------------------------------------------------------------------------------------

VERIFY_BASE = ['--trials', 't', '--enroll-ark', 'e.ark', '--test-ark', 't.ark']


@pytest.mark.parametrize('extra', [
    ['--calibrate-out', 'c.json', '--calibration', 'd.json'],
    ['--calibration-prior', '0.3'],
    ['--calibrate-out', 'c.json', '--calibration-prior', '0'],
    ['--calibrate-out', 'c.json', '--calibration-prior', '1'],
    ['--calibration', 'missing.json'],
])
def test_verify_usage_errors_exit_2(tmp_path, extra):
    tf, plda = model_files(tmp_path)
    with pytest.raises(SystemExit) as e:
        verify.main(VERIFY_BASE + ['--xvec-transform', tf, '--plda-file', plda] + extra)
    assert e.value.code == 2


@pytest.mark.parametrize('extra', [
    ['--Fa', '0.5'],
    ['--Fb', '2'],
    ['--lda-dim', '64'],
    ['--cohort-ark', 'c.ark', '--cohort-utt2spk', 'c.u'],
])
def test_verify_refuses_a_calibration_of_another_run(tmp_path, extra):
    path, tf, plda = write_cal(tmp_path, Fa=1.0, Fb=1.0)
    base = VERIFY_BASE + ['--xvec-transform', tf, '--plda-file', plda, '--calibration', path]
    with pytest.raises(SystemExit) as e:
        verify.main(base + extra)
    assert e.value.code == 2
    other = tmp_path / 'plda2'
    other.write_bytes(b'x')
    with pytest.raises(SystemExit) as e:
        verify.main(VERIFY_BASE + ['--xvec-transform', tf, '--plda-file', str(other), '--calibration', path])
    assert e.value.code == 2


def cli_base(tf, plda):
    return ['--init', 'AHC+VB', '--out-rttm-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 's',
            '--xvec-transform', tf, '--plda-file', plda, '--threshold', '0', '--lda-dim', '128', '--Fa', '0.3', '--Fb',
            '17', '--loopP', '0.99']


@pytest.mark.parametrize('extra, kind', [
    ([], 'llr'),                                                                       # neither linking nor enrolment
    (['--link-threshold', '0', '--adapt'], 'llr'),
    (['--enroll-threshold', '0'], 'llr'),                                              # without the enrolment files
    (['--link-threshold', '0', '--Fa', '0.4'], 'llr'),
    (['--link-threshold', '0', '--lda-dim', '64'], 'llr'),
    (['--link-threshold', '0', '--cohort-ark', 'c.ark', '--cohort-utt2spk', 'c.u'], 'llr'),
    (['--link-threshold', '0'], 'as-norm'),
    (['--link-threshold', '0', '--cohort-ark', 'c.ark', '--cohort-utt2spk', 'c.u', '--cohort-top', '20'], 'as-norm'),
])
def test_cli_usage_errors_exit_2(tmp_path, extra, kind):
    path, tf, plda = write_cal(tmp_path, kind=kind, top=None if kind == 'llr' else 200)
    args = cli_base(tf, plda) + ['--calibration', path] + extra
    with pytest.raises(SystemExit) as e:
        cli.main(args)
    assert e.value.code == 2


def test_cli_refuses_a_calibration_that_reverses_the_order_and_other_models(tmp_path):
    path, tf, plda = write_cal(tmp_path, a=-1.0)
    with pytest.raises(SystemExit) as e:
        cli.main(cli_base(tf, plda) + ['--calibration', path, '--link-threshold', '0'])
    assert e.value.code == 2
    path, tf, plda = write_cal(tmp_path)
    other = tmp_path / 'plda2'
    other.write_bytes(b'x')
    with pytest.raises(SystemExit) as e:
        cli.main(cli_base(tf, str(other)) + ['--calibration', path, '--link-threshold', '0'])
    assert e.value.code == 2


def test_cli_enrolment_threshold_still_required_without_a_calibration(tmp_path):
    tf, plda = model_files(tmp_path)
    with pytest.raises(SystemExit) as e:
        cli.main(cli_base(tf, plda) + ['--enroll-ark', 'e.ark', '--enroll-utt2spk', 'e.u'])
    assert e.value.code == 2


def test_cli_thresholds_are_mapped_before_diarizing(tmp_path):
    """With --calibration the cli hands diarize_batch the raw thresholds (t - b) / a, an omitted --enroll-threshold
    being 0."""
    path, tf, plda = write_cal(tmp_path, a=1.5, b=-2.0)
    ap = cli.build_parser()
    args = ap.parse_args(cli_base(tf, plda) + ['--calibration', path, '--link-threshold', '1', '--enroll-ark', 'e.ark',
                                               '--enroll-utt2spk', 'e.u'])
    assert cli.calibrated_thresholds(ap, args) == ((1.0 + 2.0) / 1.5, (0.0 + 2.0) / 1.5)
    args = ap.parse_args(cli_base(tf, plda) + ['--calibration', path, '--enroll-threshold', '-1', '--enroll-ark',
                                               'e.ark', '--enroll-utt2spk', 'e.u'])
    assert cli.calibrated_thresholds(ap, args) == (None, (-1.0 + 2.0) / 1.5)
