"""PLDA adaptation, interpolation and re-centring on the host (DESIGN.md section 5.26): adapt_plda against the float64
oracle on given statistics, the two properties of the definition, the scales, interpolation, the Kaldi-form round trip
of the shipped model, recentre_transform against numpy, and every refusal in the functions and the three parsers."""
import os
import re

import numpy as np
import pytest

from oracle import adapt_oracle as O
from vbx_b200 import adapt, cli, sweep, train

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


def spd(d, rng, lo, hi):
    q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    return (q * np.exp(rng.uniform(np.log(lo), np.log(hi), d))[None, :]) @ q.T


def model(d=12, seed=0):
    """A Kaldi-form PLDA (as train_backend writes it) and its covariances."""
    rng = np.random.default_rng(seed)
    W, B = spd(d, rng, 0.2, 2.0), spd(d, rng, 0.05, 5.0)
    mu = rng.standard_normal(d)
    plda = adapt.plda_from_covariances(mu, W, B)
    return plda, adapt.plda_covariances(plda)


def archive(d, seed, scale=1.5, shift=0.7):
    rng = np.random.default_rng(seed)
    m = shift * rng.standard_normal(d)
    C = spd(d, rng, 0.1, 4.0) * scale
    return m, C


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


@pytest.mark.parametrize('scales', [{}, dict(within_scale=0.5, between_scale=0.2, mean_scale=0.0),
                                    dict(within_scale=2.0, between_scale=1.0, mean_scale=3.0)])
@pytest.mark.parametrize('d', [1, 12, 128])
def test_adapt_plda_matches_the_oracle(d, scales):
    plda, (mu, W, B) = model(d, d)
    m, C = archive(d, d + 1)
    got, rep = adapt.adapt_plda(plda, m, C, **scales)
    s = adapt.check_scales(**scales)
    want = O.adapt(mu, *O.covariances(plda[1], plda[2]), m, C, s['within_scale'], s['between_scale'],
                   s['mean_scale'])
    mu2, W2, B2 = adapt.plda_covariances(got)
    assert np.array_equal(mu2, m)
    assert rel(W2, want[1]) <= 1e-10 and rel(B2, want[2]) <= 1e-10
    assert np.allclose(rep['eigenvalues'], want[3][::-1], rtol=1e-10, atol=1e-12)
    assert rep['inflated'] == int((want[3] > 1).sum()) and rep['scales'] == s
    assert rep['delta_norm'] == pytest.approx(np.linalg.norm(m - mu), rel=1e-15)
    assert np.all(np.diff(got[2]) <= 0)                     # psi descending, as train_backend writes it


def test_no_excess_variance_leaves_the_covariances_bit_for_bit():
    plda, (mu, W, B) = model(16, 3)
    Sigma = W + B
    for m, C in ((mu, 0.5 * Sigma), (mu + 1e-3, 0.3 * W), (mu, Sigma * 0.999)):
        mu2, W2, B2, lam, _ = adapt.adapt_covariances(mu, W, B, m, C, 0.3, 0.7, 1.0)
        assert lam.max() <= 1.0
        assert np.array_equal(W2, W) and np.array_equal(B2, B) and np.array_equal(mu2, m)


@pytest.mark.parametrize('w', [0.0, 0.3, 0.5, 1.0])
def test_unit_total_scale_lifts_every_direction_to_max_lambda_one(w):
    plda, (mu, W, B) = model(20, 4)
    m, C = archive(20, 5, scale=1.0)
    _, W2, B2, lam, V = adapt.adapt_covariances(mu, W, B, m, C, w, 1.0 - w, 1.0)
    assert 0 < (lam > 1).sum() < len(lam)                   # some directions inflated, some not
    assert np.abs(V.T @ (W2 + B2) @ V - np.diag(np.maximum(lam, 1.0))).max() <= 1e-10


def test_zero_within_and_between_scales_move_only_the_mean():
    plda, (mu, W, B) = model(10, 6)
    m, C = archive(10, 7, scale=3.0)
    mu2, W2, B2, lam, _ = adapt.adapt_covariances(mu, W, B, m, C, 0.0, 0.0, 1.0)
    assert lam.max() > 1
    assert np.array_equal(W2, W) and np.array_equal(B2, B) and np.array_equal(mu2, m)


def test_excess_is_linear_in_each_scale():
    plda, (mu, W, B) = model(10, 8)
    m, C = archive(10, 9, scale=3.0)
    _, W1, B1, lam1, _ = adapt.adapt_covariances(mu, W, B, m, C, 1.0, 1.0, 1.0)
    E = W1 - W
    assert rel(B1 - B, E) <= 1e-12
    for w, b in ((0.3, 0.7), (2.5, 0.1), (0.0, 4.0)):
        _, W2, B2, lam2, _ = adapt.adapt_covariances(mu, W, B, m, C, w, b, 1.0)
        assert np.array_equal(lam1, lam2)                   # E depends on neither scale
        assert np.abs((W2 - W) - w * E).max() <= 1e-12 * np.abs(E).max()
        assert np.abs((B2 - B) - b * E).max() <= 1e-12 * np.abs(E).max()


def test_mean_scale_adds_the_mean_shift():
    """mean_scale = 0 ignores the shift: the result equals adapting to a set already centred on mu."""
    plda, (mu, W, B) = model(8, 10)
    m, C = archive(8, 11, shift=3.0)
    a = adapt.adapt_covariances(mu, W, B, m, C, 0.3, 0.7, 0.0)
    b = adapt.adapt_covariances(mu, W, B, mu, C, 0.3, 0.7, 1.0)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    c = adapt.adapt_covariances(mu, W, B, m, C, 0.3, 0.7, 1.0)
    assert c[3].max() > a[3].max()


@pytest.mark.parametrize('alpha', [0.0, 1.0, 0.25])
def test_interpolation(alpha):
    p_in, c_in = model(14, 12)
    p_out, c_out = model(14, 13)
    got = adapt.interpolate_plda(p_in, p_out, alpha)
    if alpha in (0.0, 1.0):
        want = p_in if alpha == 1.0 else p_out
        for g, w in zip(got, want):
            assert np.abs(g - w).max() <= 1e-12 * max(np.abs(w).max(), 1.0)
    cov = adapt.plda_covariances(got)
    for g, a, b in zip(cov, c_in, c_out):
        assert rel(g, alpha * a + (1 - alpha) * b) <= 1e-11


def test_shipped_model_round_trips_through_the_covariance_form():
    """T up to each row's sign: the shipped (Kaldi-written) model does not fix row signs, train_backend writes each row's
    largest-magnitude entry positive."""
    z = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    plda = (z['plda_mu'], z['plda_tr'], z['plda_psi'])
    mu, T, psi = adapt.plda_from_covariances(*adapt.plda_covariances(plda))
    assert np.array_equal(mu, plda[0])
    assert np.abs(psi - plda[2]).max() <= 1e-10 * np.abs(plda[2]).max()
    sign = np.sign(np.sum(T * plda[1], 1))
    assert np.abs(T * sign[:, None] - plda[1]).max() <= 1e-10 * np.abs(plda[1]).max()


def test_recentre_transform_matches_numpy():
    rng = np.random.default_rng(14)
    Dx, d = 24, 6
    transform = (rng.standard_normal(Dx), rng.standard_normal(d), rng.standard_normal((Dx, d)))
    x = 3.0 + rng.standard_normal((500, Dx))
    m1 = x.mean(0)
    y = x - m1
    y /= np.linalg.norm(y, axis=1, keepdims=True)
    want = (m1, y.mean(0) @ transform[2], transform[2])
    got = adapt.recentre_transform(transform, x, device='cpu')
    for g, w in zip(got, want):
        assert np.abs(g - w).max() <= 1e-13 * max(np.abs(w).max(), 1.0)


def test_refusals_of_the_functions():
    plda, _ = model(6, 15)
    m, C = archive(6, 16)
    cases = [
        (lambda: adapt.adapt_plda(plda, m, C, within_scale=-0.1), 'within_scale must be a finite number >= 0, got -0.1'),
        (lambda: adapt.adapt_plda(plda, m, C, mean_scale=float('nan')), 'mean_scale must be a finite number'),
        (lambda: adapt.adapt_plda(plda, m, C, between_scale=float('inf')), 'between_scale must be a finite number'),
        (lambda: adapt.interpolate_plda(plda, plda, 1.5), 'alpha must lie in [0, 1], got 1.5'),
        (lambda: adapt.interpolate_plda(plda, plda, -0.1), 'alpha must lie in [0, 1], got -0.1'),
        (lambda: adapt.interpolate_plda(plda, model(5, 1)[0], 0.5), 'd = 6 and d = 5'),
        (lambda: adapt.adapt_plda((plda[0], plda[1], np.r_[plda[2][:-1], -0.5]), m, C), 'psi < 0'),
        (lambda: adapt.adapt_plda((plda[0], np.diag([1.0, 1, 1, 1, 1, 0]), plda[2]), m, C), 'singular'),
        (lambda: adapt.adapt_plda(plda, m[:5], C), 'd = 6'),
        (lambda: adapt.adapt_plda(plda, m, np.full_like(C, np.nan)), 'non-finite'),
    ]
    for fn, match in cases:
        with pytest.raises(ValueError, match=re.escape(match)):
            fn()


def backend_case(n=(5, 4), Dx=8, d=4, seed=17):
    rng = np.random.default_rng(seed)
    recs = {f'r{i}': (rng.standard_normal((k, Dx)), None) for i, k in enumerate(n)}
    transform = (rng.standard_normal(Dx), rng.standard_normal(d), rng.standard_normal((Dx, d)))
    return recs, transform, model(d, seed)[0]


@pytest.mark.parametrize('change, match', [
    (dict(recs={'a': (np.ones((1, 8)), None)}), 'at least 2 x-vectors, the archive has 1'),
    (dict(recs={'a': (np.r_[np.ones((3, 8)), np.full((1, 8), np.nan)], None)}), '1 non-finite x-vector'),
    (dict(plda=model(5, 2)[0]), 'maps to d = 4, the PLDA has d = 5'),
    (dict(within_scale=-1.0), 'within_scale must be a finite number >= 0'),
    (dict(adapt=False, mean_scale=0.5), "adaptation scales ['mean_scale'] without adapt"),
    (dict(bogus_scale=1.0), "unknown adaptation scale(s) ['bogus_scale']"),
    (dict(transform_dx=9), 'takes Dx = 9, the x-vectors have Dx = 8'),
])
def test_refusals_of_adapt_backend(change, match):
    """Every refusal comes before any device work: these run without a GPU."""
    recs, transform, plda = backend_case()
    recs = change.pop('recs', recs)
    plda = change.pop('plda', plda)
    if 'transform_dx' in change:
        n = change.pop('transform_dx')
        transform = (np.zeros(n), transform[1], np.zeros((n, 4)))
    with pytest.raises(ValueError, match=re.escape(match)):
        adapt.adapt_backend(recs, transform, plda, device='cpu', **change)


def test_fixed_transform_refusals_of_train_backend():
    rng = np.random.default_rng(18)
    sets = {f's{i}': rng.standard_normal((3, 6)) for i in range(3)}
    with pytest.raises(ValueError, match=re.escape('N - K = 9 - 3 = 6 is below d = 7')):
        train.train_backend(sets, transform=(np.zeros(6), np.zeros(7), np.ones((6, 7))))
    with pytest.raises(ValueError, match=re.escape('takes Dx = 5, the x-vectors have Dx = 6')):
        train.train_backend(sets, transform=(np.zeros(5), np.zeros(2), np.ones((5, 2))))
    with pytest.raises(ValueError, match=re.escape('inconsistent x-vector transform')):
        train.train_backend(sets, transform=(np.zeros(6), np.zeros(3), np.ones((6, 2))))


CLI = ['--init', 'AHC+VB', '--out-rttm-dir', 'o', '--xvec-ark-file', 'a', '--segments-file', 's', '--xvec-transform',
       't', '--plda-file', 'p', '--threshold', '0', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']
SWEEP = ['--out-dir', 'o', '--xvec-ark-file', 'a', '--segments-file', 's', '--xvec-transform', 't', '--plda-file', 'p',
         '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99', '--threshold', '0']
SCALE_ERRORS = [['--recentre'], ['--adapt-within-scale', '0.5'], ['--adapt-mean-scale', '1'],
                ['--adapt', '--adapt-within-scale=-0.1'], ['--adapt', '--adapt-between-scale', 'nan'],
                ['--adapt', '--adapt-mean-scale', 'inf']]


@pytest.mark.parametrize('extra', SCALE_ERRORS)
@pytest.mark.parametrize('mod, base', [(cli, CLI), (sweep, SWEEP)])
def test_cli_and_sweep_parser_refusals(mod, base, extra):
    with pytest.raises(SystemExit) as e:
        mod.main(base + extra)
    assert e.value.code == 2


TRAIN = ['--xvec-ark-file', 'a', '--out-dir', 'o']


@pytest.mark.parametrize('extra', [
    ['--adapt-plda', 'p', '--utt2spk', 'u'],                                  # no transform
    ['--adapt-plda', 'p', '--xvec-transform', 't', '--utt2spk', 'u'],         # labels with adaptation
    ['--adapt-plda', 'p', '--xvec-transform', 't', '--segments-file', 's', '--ref-rttm', 'r'],
    ['--adapt-plda', 'p', '--xvec-transform', 't', '--interpolate-with', 'q', '--alpha', '0.5'],
    ['--xvec-transform', 't', '--utt2spk', 'u', '--recentre'],
    ['--xvec-transform', 't', '--utt2spk', 'u', '--within-scale', '0.5'],
    ['--xvec-transform', 't', '--utt2spk', 'u', '--chain', 'float64'],
    ['--adapt-plda', 'p', '--xvec-transform', 't', '--within-scale=-1'],
    ['--adapt-plda', 'p', '--xvec-transform', 't', '--mean-scale', 'nan'],
    ['--utt2spk', 'u', '--interpolate-with', 'q', '--alpha', '0.5'],          # no transform
    ['--xvec-transform', 't', '--utt2spk', 'u', '--interpolate-with', 'q'],    # no alpha
    ['--xvec-transform', 't', '--utt2spk', 'u', '--alpha', '0.5'],             # no PLDA
    ['--xvec-transform', 't', '--utt2spk', 'u', '--interpolate-with', 'q', '--alpha', '1.5'],
    ['--xvec-transform', 't', '--utt2spk', 'u', '--interpolate-with', 'q', '--alpha=-0.5'],
    ['--xvec-transform', 't', '--utt2spk', 'u', '--interpolate-with', 'q', '--alpha', 'nan'],
])
def test_train_parser_refusals(extra):
    with pytest.raises(SystemExit) as e:
        train.main(TRAIN + extra)
    assert e.value.code == 2


def write_model(root, transform, plda):
    from vbx_b200 import formats
    np.savez(os.path.join(root, 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    formats.write_kaldi_plda_binary(os.path.join(root, 'plda'), *plda)
    return os.path.join(root, 'transform.npz'), os.path.join(root, 'plda')


def test_train_refuses_models_that_do_not_fit(tmp_path):
    """Refusals that need the files' contents: a PLDA of another d than the transform, psi < 0, a singular transform,
    and PLDAs of different d to interpolate; all before any device work."""
    from vbx_b200 import formats
    recs, transform, plda = backend_case()
    ark = str(tmp_path / 'x.ark')
    formats.write_vec_flt_ark(ark, [f'{n}_{t}' for n, (x, _) in recs.items() for t in range(len(x))],
                              [v for x, _ in recs.values() for v in x])
    with open(tmp_path / 'utt2spk', 'w') as f:
        f.write(''.join(f'{n}_{t} {n}\n' for n, (x, _) in recs.items() for t in range(len(x))))
    t_path, _ = write_model(str(tmp_path), transform, plda)
    bad = {'d5': model(5, 3)[0], 'psi': (plda[0], plda[1], np.r_[plda[2][:-1], -1.0]),
           'singular': (plda[0], np.diag([1.0, 1.0, 1.0, 0.0]), plda[2])}
    for tag, p in bad.items():
        formats.write_kaldi_plda_binary(str(tmp_path / tag), *p)
    for tag, match in (('d5', 'maps to d = 4, the PLDA has d = 5'), ('psi', 'psi < 0'), ('singular', 'singular')):
        with pytest.raises(ValueError, match=re.escape(match)):
            train.main(TRAIN[:1] + [ark, '--out-dir', str(tmp_path / 'o'), '--xvec-transform', t_path,
                                    '--adapt-plda', str(tmp_path / tag), '--device', 'cpu'])
    for tag, match in (('d5', 'maps to d = 4, the PLDA has d = 5'), ('psi', 'psi < 0')):
        with pytest.raises(ValueError, match=re.escape(match)):
            train.main(TRAIN[:1] + [ark, '--out-dir', str(tmp_path / 'o'), '--xvec-transform', t_path,
                                    '--utt2spk', str(tmp_path / 'utt2spk'), '--interpolate-with', str(tmp_path / tag),
                                    '--alpha', '0.5', '--device', 'cpu'])
