"""Enrolled speakers in live streams (DESIGN.md section 5.29) without a GPU: the float64 oracle on a worked case of two
streams and three pushes, stable names that are never shared within a stream, the prior's history, and every refusal of
StreamDiarizer and of the stream command line."""
import json

import numpy as np
import pytest

from oracle import stream_enroll_oracle as seo
from oracle.stream_oracle import StreamOracle
from vbx_b200 import stream, verify

R = 8
C_CTX = 6
FA, FB = 0.3, 17.0
THR = 2.0


def phi():
    return np.linspace(0.5, 4.0, R)


def enrolled_set(seed=3, E=3, n=20):
    """E enrolled speakers far apart, n x-vectors each: means, n_e, F_e."""
    rng = np.random.default_rng(seed)
    mu = rng.standard_normal((E, R)) * 4.0
    x = [mu[e] + 0.3 * rng.standard_normal((n, R)) for e in range(E)]
    return mu, np.full(E, float(n)), np.array([xe.sum(0) for xe in x])


def rows(rng, mean, h):
    return mean + 0.3 * rng.standard_normal((h, R))


def new_stream():
    return StreamOracle(phi(), FA, FB, 0.99, context=C_CTX, max_speakers=8)


def push(so, names, fea, labels, n_e, F_e, threshold, prior=False):
    so.commit(labels, fea)                    # labels are final: fresh speakers appear in order of their first row
    return seo.name_push(so, names, labels, n_e, F_e, phi(), FA / FB, threshold, prior)


def worked_case(prior=False):
    """Stream a: speaker 0 (enrolled 0) named at its first push; speaker 1 (enrolled 1) first seen with one x-vector
    far from every enrolled speaker, named only at the third push once its later x-vectors outweigh it.  Stream b:
    speaker 0 is enrolled 0 as well (a claim in one stream does not bind the other), speaker 1 is nobody."""
    mu, n_e, F_e = enrolled_set()
    rng = np.random.default_rng(11)
    far = np.full(R, 30.0)
    a, b = new_stream(), new_stream()
    na, nb = {}, {}
    out = []
    out.append((push(a, na, np.vstack([rows(rng, mu[0], 4), far[None]]), np.array([0, 0, 0, 0, 1]), n_e, F_e, THR,
                     prior),
                push(b, nb, np.vstack([rows(rng, mu[0], 3), rows(rng, -mu[2] * 3, 3)]), np.array([0, 0, 0, 1, 1, 1]),
                     n_e, F_e, THR, prior)))
    out.append((push(a, na, rows(rng, mu[1], 1), np.array([1]), n_e, F_e, THR, prior),
                push(b, nb, rows(rng, mu[0], 2), np.array([0, 0]), n_e, F_e, THR, prior)))
    out.append((push(a, na, np.vstack([rows(rng, mu[1], 6), rows(rng, mu[0], 2)]), np.array([1] * 6 + [0, 0]), n_e,
                     F_e, THR, prior),
                push(b, nb, rows(rng, -mu[2] * 3, 2), np.array([1, 1]), n_e, F_e, THR, prior)))
    return out, (a, na), (b, nb), (n_e, F_e)


def test_worked_case():
    out, (a, na), (b, nb), _ = worked_case()
    (a1, b1), (a2, b2), (a3, b3) = out
    assert a1['candidates'] == [0, 1] and a1['assign'].tolist() == [0, -1]
    assert b1['candidates'] == [0, 1] and b1['assign'].tolist() == [0, -1]       # enrolled 0 claimed in both streams
    assert a2['candidates'] == [1] and a2['assign'].tolist() == [-1]              # not yet: the far x-vector weighs in
    assert b2['candidates'] == []                                                 # speaker 0 is named: never rescored
    assert a3['candidates'] == [1] and a3['assign'].tolist() == [1]               # named at a later push
    assert b3['candidates'] == [1] and b3['assign'].tolist() == [-1]
    assert na == {0: 0, 1: 1} and nb == {0: 0}
    # an unnamed candidate's best LLR is over the enrolled speakers its stream has not claimed
    assert b3['best'][0] == pytest.approx(max(b3['llr'][0][1:]), abs=0)
    assert a2['best'][0] == pytest.approx(max(a2['llr'][0][1:]), abs=0) and a2['best'][0] < THR


def test_statistics_are_every_row_of_the_speaker():
    """History plus ring is every x-vector the stream gave the speaker, whatever the context cut off."""
    out, (a, _), _, _ = worked_case()
    fea, lab = np.vstack(a.final_fea), np.concatenate(a.final_lab)
    assert len(lab) > C_CTX
    n, F = seo.candidate_stats(a.n_hist, a.F_hist, a.ctx_fea, a.ctx_lab, [0, 1])
    for j, k in enumerate([0, 1]):
        assert n[j] == (lab == k).sum()
        np.testing.assert_allclose(F[j], fea[lab == k].sum(0), rtol=1e-13, atol=1e-12)


def test_names_are_stable_and_never_shared_within_a_stream():
    """Five speakers near the same enrolled speaker, pushed one at a time: the first takes the name, the others never."""
    mu, n_e, F_e = enrolled_set(E=2)
    rng = np.random.default_rng(5)
    so, names = new_stream(), {}
    for k in range(5):
        r = push(so, names, rows(rng, mu[0], 3), np.array([k] * 3), n_e, F_e, -1e3)
        assert r['candidates'] == [k]
        assert r['assign'].tolist() == ([0] if k == 0 else [1] if k == 1 else [-1])
        if k >= 2:
            assert r['best'][0] == -np.inf                        # every enrolled speaker is claimed
    assert names == {0: 0, 1: 1}


def test_prior_adds_the_enrolment_to_the_history():
    out, (a, na), (b, nb), (n_e, F_e) = worked_case(prior=True)
    plain = worked_case(prior=False)
    (pa, _), (pb, _) = plain[1], plain[2]
    for so, ref, names in ((a, pa, na), (b, pb, nb)):
        add_n, add_F = np.zeros_like(ref.n_hist), np.zeros_like(ref.F_hist)
        for k, e in names.items():
            add_n[k], add_F[k] = n_e[e], F_e[e]
        np.testing.assert_array_equal(so.n_hist, ref.n_hist + add_n)
        np.testing.assert_allclose(so.F_hist, ref.F_hist + add_F, rtol=1e-14, atol=1e-12)


def model(Dx=64):
    rng = np.random.default_rng(0)
    return (rng.standard_normal(Dx), rng.standard_normal(R), rng.standard_normal((Dx, R))), \
        (rng.standard_normal(R), np.eye(R), np.ones(R))


GOOD = {'alice': np.zeros((2, 64)), 'bob': np.ones((1, 64))}


@pytest.mark.parametrize('kw', [
    dict(enroll={'spk1': np.zeros((1, 64))}, enroll_threshold=0.0),          # the name of an unnamed stream speaker
    dict(enroll={'spk12': np.zeros((1, 64))}, enroll_threshold=0.0),
    dict(enroll={'a b': np.zeros((1, 64))}, enroll_threshold=0.0),
    dict(enroll={'unknown-x': np.zeros((1, 64))}, enroll_threshold=0.0),
    dict(enroll={'': np.zeros((1, 64))}, enroll_threshold=0.0),
    dict(enroll={}, enroll_threshold=0.0),
    dict(enroll={'alice': np.zeros((0, 64))}, enroll_threshold=0.0),
    dict(enroll={'alice': np.zeros((2, 32))}, enroll_threshold=0.0),       # dimension
    dict(enroll=GOOD),                                                       # no threshold: there is no default
    dict(enroll=GOOD, enroll_threshold=float('inf')),
    dict(enroll=GOOD, enroll_threshold=2e15),
    dict(enroll_threshold=0.0),                                              # flags without enroll
    dict(enroll_prior=True),
])
def test_refusals(kw):
    transform, plda = model()
    with pytest.raises(ValueError):
        stream.StreamDiarizer(transform, plda, FA, FB, 0.99, lda_dim=R, **kw)


def test_accepts_a_good_enrolment_without_a_device():
    transform, plda = model()
    sd = stream.StreamDiarizer(transform, plda, FA, FB, 0.99, lda_dim=R, enroll=GOOD, enroll_threshold=1.5,
                               enroll_prior=True)
    assert [n for n, _ in sd.enrolled] == ['alice', 'bob'] and sd.enroll_threshold == 1.5 and sd.state is None
    assert sd.enrolment is None                        # the enrolled x-vectors reach the device with the first stream
    enrolled, _ = stream.check_stream_enrolment({'spk1x': np.zeros((1, 64))}, 0.0, False, 64)
    assert enrolled[0][0] == 'spk1x'                   # spk followed by anything but digits is an ordinary name


BASE = ['--out-rttm-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform', 't', '--plda-file',
        'p', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99', '--threshold', '-0.015', '--lda-dim', '128']


def calibration(tmp_path, kind):
    t, p = tmp_path / 't', tmp_path / 'p'
    t.write_bytes(b'transform')
    p.write_bytes(b'plda')
    path = tmp_path / f'{kind}.json'
    verify.write_calibration(str(path), dict(a=2.0, b=-1.0, prior=0.5, n_target=10, n_nontarget=20), kind, 0.3, 17.0,
                             128, 200 if kind == 'as-norm' else None, str(t), str(p))
    return str(path), str(t), str(p)


@pytest.mark.parametrize('extra, message', [
    (['--enroll-ark', 'e'], 'go together'),
    (['--enroll-ark', 'e', '--enroll-utt2spk', 'u'], 'go together'),
    (['--enroll-threshold', '0'], 'go together'),
    (['--enroll-prior'], '--enroll-prior needs'),
])
def test_command_line_usage_errors(extra, message, capsys):
    with pytest.raises(SystemExit) as e:
        stream.main(BASE + extra)
    assert e.value.code == 2 and message in capsys.readouterr().err


def test_command_line_calibration(tmp_path, capsys):
    llr, t, p = calibration(tmp_path, 'llr')
    base = [a if a not in ('t', 'p') else {'t': t, 'p': p}[a] for a in BASE]
    cases = [(['--calibration', llr], '--calibration needs the enrolment options'),
             (['--calibration', calibration(tmp_path, 'as-norm')[0], '--enroll-ark', 'e', '--enroll-utt2spk', 'u'],
              "score_kind 'as-norm'"),
             (['--calibration', llr, '--enroll-ark', 'e', '--enroll-utt2spk', 'u', '--Fb', '16'], 'Fb'),
             (['--calibration', str(tmp_path / 'missing.json'), '--enroll-ark', 'e', '--enroll-utt2spk', 'u'],
              '--calibration')]
    for extra, message in cases:
        with pytest.raises(SystemExit) as e:
            stream.main(base + extra)
        assert e.value.code == 2 and message in capsys.readouterr().err
    ap = stream.build_parser()
    for thr, want in ((None, 0.5), ('3', 2.0)):           # (t - b) / a with a = 2, b = -1
        args = ap.parse_args(base + ['--calibration', llr, '--enroll-ark', 'e', '--enroll-utt2spk', 'u']
                             + ([] if thr is None else ['--enroll-threshold', thr]))
        assert stream.enrolment_options(ap, args) == want
    with open(llr) as f:
        assert json.load(f)['score_kind'] == 'llr'
