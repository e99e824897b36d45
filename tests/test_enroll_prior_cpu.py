"""Enrolled speakers as state priors of the VB-HMM (DESIGN.md section 5.23), CPU side: the float64 oracle against the
plain oracle run on the recording with the enrolment x-vectors appended as frames held on their state, the zero prior,
and the host logic of diarize_batch(enroll_prior=True) and the command line."""
import numpy as np
import pytest

from oracle import prior_oracle as po
from oracle.vbx_oracle import vbx_oracle
from vbx_b200 import enroll
from vbx_b200.link import speaker_table


def _case(seed, T=240, R=8, S=4, n_e=(6, 0, 300, 0)):
    """A recording of S speakers with sticky turns and enrolment x-vectors of some of them (n_e per state)."""
    rng = np.random.default_rng(seed)
    Phi = np.sort(rng.uniform(0.5, 30.0, R))[::-1].copy()
    centres = rng.normal(0, 1.5, (S, R))
    spk = np.zeros(T, dtype=np.int64)
    for t in range(1, T):
        spk[t] = spk[t - 1] if rng.random() < 0.95 else rng.integers(S)
    X = centres[spk] + rng.normal(0, 1.0, (T, R))
    state_e = np.repeat(np.arange(S), n_e)
    X_e = centres[state_e] + rng.normal(0, 1.0, (len(state_e), R))
    q = np.exp(5.0 * np.eye(S)[rng.integers(S, size=T)])
    gamma0 = q / q.sum(1, keepdims=True)
    n = np.bincount(state_e, minlength=S).astype(np.float64)
    F = np.zeros((S, R))
    np.add.at(F, state_e, X_e)
    return X, Phi, X_e, state_e, gamma0, n, F


@pytest.mark.parametrize('seed', [0, 1, 2])
@pytest.mark.parametrize('Fa,Fb,loopP', [(0.3, 17.0, 0.99), (0.4, 64.0, 0.65), (1.0, 1.0, 0.9)])
def test_prior_equals_frames_held_on_their_state(seed, Fa, Fb, loopP):
    X, Phi, X_e, state_e, gamma0, n, F = _case(seed)
    S = gamma0.shape[1]
    trace = []
    po.vbx_prior_oracle(X, Phi, n, F, loopProb=loopP, Fa=Fa, Fb=Fb, pi=S, gamma=gamma0, maxIters=15, epsilon=-np.inf,
                        trace=trace)
    assert len(trace) == 15
    consts = []
    for it in trace:
        invL, alpha = po.augmented_model(it['gamma0'], X, Phi, Fa / Fb, X_e, state_e)
        np.testing.assert_allclose(it['invL'], invL, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(it['alpha'], alpha, rtol=1e-12, atol=1e-12)
        consts.append(po.augmented_elbo(it['tll'], it['alpha'], it['invL'], Phi, Fa, Fb, X_e, state_e) - it['elbo'])
    elbo = np.array([it['elbo'] for it in trace])
    aug = elbo + np.array(consts)
    np.testing.assert_allclose(np.diff(aug), np.diff(elbo), rtol=1e-9, atol=1e-9 * np.abs(elbo).max())
    # one constant, Fb log Z_e, that depends on the enrolment alone
    want = Fb * po.log_evidence(Phi, Fa, Fb, X_e, state_e, S)
    np.testing.assert_allclose(consts, want, rtol=1e-10, atol=1e-9 * np.abs(elbo).max())


@pytest.mark.parametrize('seed', [3, 4])
def test_zero_prior_is_the_plain_oracle(seed):
    X, Phi, _, _, gamma0, _, _ = _case(seed)
    S, R = gamma0.shape[1], X.shape[1]
    kw = dict(loopProb=0.99, Fa=0.3, Fb=17.0, pi=S, gamma=gamma0, maxIters=30, epsilon=1e-6, return_model=True)
    a = vbx_oracle(X, Phi, **kw)
    b = po.vbx_prior_oracle(X, Phi, np.zeros(S), np.zeros((S, R)), **kw)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_prior_pulls_a_state_to_its_enrolled_speaker():
    """Two states started on one merged speaker: the enrolled state keeps the frames of its enrolled speaker."""
    X, Phi, X_e, state_e, gamma0, n, F = _case(5, n_e=(40, 0, 0, 0))
    S = gamma0.shape[1]
    _, _, _, al0, _ = po.vbx_prior_oracle(X, Phi, np.zeros(S), np.zeros_like(F), Fa=0.3, Fb=17.0, pi=S, gamma=gamma0,
                                          maxIters=1, return_model=True)
    _, _, _, al1, _ = po.vbx_prior_oracle(X, Phi, n, F, Fa=0.3, Fb=17.0, pi=S, gamma=gamma0, maxIters=1,
                                          return_model=True)
    target = (X_e.mean(0) * np.sqrt(Phi))
    assert np.linalg.norm(al1[0] - target) < np.linalg.norm(al0[0] - target)
    assert np.array_equal(al1[1:], al0[1:])


# ---- host logic ----------------------------------------------------------------------------------------------------

def _result(labels, assign, best, E=3, R=4):
    table = speaker_table(labels)
    n_e = np.arange(1, E + 1, dtype=np.float64) * 10
    F_e = np.arange(E * R, dtype=np.float64).reshape(E, R)
    return enroll.EnrollResult(table, np.asarray(assign), np.asarray(best, dtype=np.float64), None, None, n_e, F_e,
                               None)


def test_prior_states_follow_the_ahc_states():
    labels = [np.array([0, 2, 2, 1, 0]), np.array([1, 0]), np.array([0, 0, 0])]
    # table rows: (0,0) (0,1) (0,2) | (1,0) (1,1) | (2,0)
    res = _result(labels, [2, -1, 0, -1, -1, 1], [9.0, -3.0, 4.0, -1.0, -2.0, 7.0])
    prior, named = enroll.prior_states(res, ['ann', 'bob', 'cy'], [3, 2, 1])
    n0, F0 = prior[0]
    assert n0.tolist() == [30.0, 0.0, 10.0] and F0.shape == (3, 4)
    assert np.array_equal(F0[0], res.F_enroll[2]) and not F0[1].any() and np.array_equal(F0[2], res.F_enroll[0])
    assert prior[1] is None
    assert prior[2][0].tolist() == [20.0] and np.array_equal(prior[2][1][0], res.F_enroll[1])
    assert named == [{0: 'cy', 2: 'ann'}, {}, {0: 'bob'}]
    # one enrolled speaker per recording at most: the assignment is one-to-one, and the states carry it as it is
    for b, x in enumerate(prior):
        if x is not None:
            nz = x[0][x[0] > 0]
            assert len(set(nz.tolist())) == len(nz)


def test_names_of_prior_states_and_free_states():
    ahc = [np.array([0, 1, 2, 1]), np.array([0, 1])]
    res = _result(ahc, [1, -1, 0, -1, -1], [8.0, -1.0, 5.0, -2.0, -4.0])
    # the VB-HMM dropped state 1 of recording 0; state 1 of recording 1 also appears as a second label only there
    final = [np.array([0, 2, 2, 0]), np.array([0, 0])]
    labels2 = [np.array([2, 0, 0, 2]), np.array([1, 1])]
    table, assign, best = enroll.carry_assignment(res, final)
    assert table.rec.tolist() == [0, 0, 1] and table.label.tolist() == [0, 2, 0]
    assert assign.tolist() == [1, 0, -1] and best.tolist() == [8.0, 5.0, -2.0]
    names, llrs = enroll.enroll_names(table, assign, best, ['ann', 'bob'], ['r0', 'r1'], labels2)
    assert names == [{0: 'bob', 2: 'ann'}, {0: 'unknown-r1-1', 1: 'unknown-r1-2'}]
    assert llrs == [{0: 8.0, 2: 5.0}, {0: -2.0}]


def test_prior_state_left_as_a_second_label_keeps_its_name():
    ahc = [np.array([0, 1, 2, 1])]
    res = _result(ahc, [1, 0, -1], [8.0, 6.0, -3.0])
    prior, named = enroll.prior_states(res, ['ann', 'bob'], [3])
    assert named == [{0: 'bob', 1: 'ann'}]
    final = [np.array([0, 2, 2, 0])]                 # state 1 survives as a second label only
    labels2 = [np.array([1, 0, 1, 2])]
    table, assign, best = enroll.carry_assignment(res, final)
    names, llrs = enroll.enroll_names(table, assign, best, ['ann', 'bob'], ['r0'], labels2)
    assert names == [{0: 'bob', 2: 'unknown-r0-3', 1: 'unknown-r0-2'}]
    assert enroll.name_prior_states(names, named) == [{0: 'bob', 2: 'unknown-r0-3', 1: 'ann'}]
    assert llrs == [{0: 8.0, 2: -3.0}]


def _fake_archive():
    recs = {'a': (np.zeros((3, 4)), np.zeros((3, 2)))}
    return recs, (None, None, None), (None, None, None)


@pytest.mark.parametrize('kw,msg', [
    (dict(enroll_prior=True), 'needs enroll'),
    (dict(enroll_prior=True, init='AHC', enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0), 'AHC'),
    (dict(enroll_prior=True, init='RANDOM+VB', init_states=3, enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0),
     'RANDOM'),
    (dict(enroll_prior=True, enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0, num_speakers=2), 'num_speakers'),
    (dict(enroll_prior=True, enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0, min_speakers=2), 'num_speakers'),
    (dict(enroll_prior=True, enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0, max_speakers=2), 'num_speakers'),
])
def test_diarize_batch_refusals(kw, msg):
    from vbx_b200 import pipeline
    recs, transform, plda = _fake_archive()
    with pytest.raises(ValueError, match=msg):
        pipeline.diarize_batch(recs, transform, plda, 0.3, 17.0, 0.99, **kw)


def test_rttm_init_refused(tmp_path):
    from vbx_b200 import pipeline
    recs, transform, plda = _fake_archive()
    (tmp_path / 'a.rttm').write_text('SPEAKER a 1 0.0 1.0 <NA> <NA> s1 <NA> <NA>\n')
    with pytest.raises(ValueError, match='RTTM'):
        pipeline.diarize_batch(recs, transform, plda, 0.3, 17.0, 0.99, init='RTTM+VB', init_rttm=str(tmp_path / 'a.rttm'),
                               enroll={'x': np.zeros((1, 4))}, enroll_threshold=0.0, enroll_prior=True)


BASE = ['--out-rttm-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 'x.seg', '--xvec-transform', 't.h5',
        '--plda-file', 'plda', '--threshold', '-0.015', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']
ENR = ['--enroll-ark', 'e.ark', '--enroll-utt2spk', 'utt2spk', '--enroll-threshold', '0']


@pytest.mark.parametrize('extra', [
    ['--init', 'AHC+VB', '--enroll-prior'],
    ['--init', 'AHC', '--enroll-prior'] + ENR,
    ['--init', 'RANDOM+VB', '--init-states', '3', '--enroll-prior'] + ENR,
    ['--init', 'RTTM+VB', '--init-rttm', 'i.rttm', '--enroll-prior'] + ENR,
    ['--init', 'AHC+VB', '--num-speakers', '2', '--enroll-prior'] + ENR,
    ['--init', 'AHC+VB', '--max-speakers', '2', '--enroll-prior'] + ENR,
])
def test_command_line_refusals(extra, capsys):
    from vbx_b200 import cli
    with pytest.raises(SystemExit) as e:
        cli.main(BASE + extra)
    assert e.value.code == 2
    assert '--enroll-prior' in capsys.readouterr().err


def test_command_line_accepts_the_option():
    from vbx_b200 import cli
    args = cli.build_parser().parse_args(BASE + ['--init', 'AHC+VB', '--enroll-prior'] + ENR)
    assert args.enroll_prior is True
    assert cli.build_parser().parse_args(BASE + ['--init', 'AHC+VB']).enroll_prior is False
