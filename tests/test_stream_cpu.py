"""Streaming diarization on the host (DESIGN.md section 5.25): the float64 oracle's properties, the host rules of
vbx_b200.stream and its refusals.  The device kernels are tested in test_stream_gpu.py."""
import numpy as np
import pytest
from scipy.cluster.hierarchy import fcluster

from oracle.ahc_oracle import ahc_labels
from oracle.stream_oracle import StreamOracle, block_ahc, nonnegative, soft_init
from oracle.vbx_oracle import vbx_oracle
from vbx_b200 import ahc as _ahc
from vbx_b200 import stream

R = 16
KW = dict(Fa=0.3, Fb=17.0, loopP=0.99, threshold=-0.015, smoothing=5.0, max_iters=20, epsilon=1e-6)


def speakers(seed, T, n_spk=3, stay=0.95, spread=3.0):
    """x-vectors of n_spk speakers with sticky turns: (x [T,R], truth [T]); x serves as the AHC input and as fea."""
    rng = np.random.default_rng(seed)
    centres = spread * rng.standard_normal((n_spk, R))
    spk = np.zeros(T, dtype=np.int64)
    for t in range(1, T):
        spk[t] = spk[t - 1] if rng.random() < stay else rng.integers(n_spk)
    return centres[spk] + rng.standard_normal((T, R)), spk


def phi():
    return np.linspace(2.0, 0.2, R)


def oracle(**kw):
    return StreamOracle(phi(), **dict(KW, **kw))


def by_first_row(labels):
    m = {}
    return np.array([m.setdefault(l, len(m)) for l in labels.tolist()])


def test_one_push_of_a_recording_is_the_offline_oracle():
    x, _ = speakers(1, 150)
    got = oracle(context=40).push(x, x)
    labels, _, _ = ahc_labels(x, KW['threshold'])
    S = int(labels.max()) + 1
    gamma, pi, Li = vbx_oracle(x, phi(), loopProb=KW['loopP'], Fa=KW['Fa'], Fb=KW['Fb'], pi=np.full(S, 1.0 / S),
                               gamma=soft_init(labels, S, KW['smoothing']), maxIters=KW['max_iters'],
                               epsilon=KW['epsilon'])
    assert got['iterations'] == len(Li)
    np.testing.assert_allclose(got['gamma'], gamma, rtol=0, atol=1e-12)
    np.testing.assert_array_equal(got['labels'], by_first_row(np.argsort(-gamma, axis=1, kind='stable')[:, 0]))
    assert got['window']['n_states'] == S and not got['window']['prior_n'].any()


@pytest.mark.parametrize('context', [0, 7, 40, 1000])
def test_history_plus_context_is_every_final_row(context):
    x, _ = speakers(2, 200)
    o = oracle(context=context)
    for lo, hi in [(0, 30), (30, 31), (31, 75), (75, 140), (140, 200)]:
        o.push(x[lo:hi], x[lo:hi])
        fea, lab = np.vstack(o.final_fea), np.concatenate(o.final_lab)
        assert len(o.ctx_lab) == min(context, hi)
        n = o.n_hist.copy()
        F = o.F_hist.copy()
        np.add.at(n, o.ctx_lab, 1.0)
        np.add.at(F, o.ctx_lab, o.ctx_fea)
        want_n, want_F = np.zeros_like(n), np.zeros_like(F)
        np.add.at(want_n, lab, 1.0)
        np.add.at(want_F, lab, fea)
        np.testing.assert_array_equal(n, want_n)
        np.testing.assert_allclose(F, want_F, rtol=1e-12, atol=1e-12)
        assert o.K == int(lab.max()) + 1


def test_context_rows_are_never_relabelled_and_streams_are_independent():
    x, _ = speakers(3, 180)
    y, _ = speakers(4, 120, n_spk=2)
    a, b, alone = oracle(context=50), oracle(context=50), oracle(context=50)
    emitted = []
    for lo in range(0, 180, 30):
        got = a.push(x[lo:lo + 30], x[lo:lo + 30])
        emitted.append(got['labels'])
        np.testing.assert_array_equal(a.ctx_lab, np.concatenate(emitted)[-len(a.ctx_lab):])
        # the window starts the context rows on exactly the labels emitted for them
        w = got['window']
        np.testing.assert_array_equal(np.argmax(w['gamma0'][:w['L']], 1), np.concatenate(emitted[:-1])[-w['L']:]
                                      if w['L'] else np.zeros(0))
        if lo < 120:
            b.push(y[lo:lo + 30], y[lo:lo + 30])
        np.testing.assert_array_equal(alone.push(x[lo:lo + 30], x[lo:lo + 30])['labels'], got['labels'])


def test_speaker_cap():
    x, _ = speakers(5, 60, n_spk=6, stay=0.5, spread=6.0)
    o = oracle(max_speakers=3, context=20)
    got = o.push(x[:30], x[:30])
    assert got['window']['n_states'] <= 3
    o.K = 3                                                      # a stream at S_max: no fresh state
    got = o.push(x[30:], x[30:])
    assert got['window']['n_states'] == 3 and got['labels'].max() < 3
    np.testing.assert_allclose(got['window']['gamma0'][got['window']['L']:], 1.0 / 3)


def test_block_clusters_recut_and_independence():
    xs = [speakers(s, T, n_spk=5, stay=0.6, spread=5.0)[0] for s, T in ((6, 40), (7, 25), (8, 3), (9, 1))]
    Zs, labels = [], []
    for x in xs:
        l, Z = block_ahc(x, KW['threshold'])
        labels.append(l)
        Zs.append(np.zeros((0, 4)) if Z is None else Z)
    lens = [len(x) for x in xs]
    K = [0, 62, 64, 10]
    out = stream.block_clusters(labels, Zs, lens, K, 64)
    for b in range(len(xs)):
        alone = stream.block_clusters([labels[b]], [Zs[b]], [lens[b]], [K[b]], 64)[0]
        np.testing.assert_array_equal(out[b][0], alone[0])
        assert out[b][1] == alone[1] and K[b] + out[b][1] <= 64
    assert out[2][1] == 0 and (out[2][0] == -1).all()
    c_free = int(labels[1].max()) + 1
    if c_free > 2:                                              # the maxclust cut at S_max - K, as scipy numbers it
        np.testing.assert_array_equal(out[1][0], fcluster(nonnegative(Zs[1]), 2, criterion='maxclust') - 1)
        np.testing.assert_array_equal(out[1][0], _ahc.cut_count([Zs[1]], [lens[1]], [2])[0])


def test_block_schedule_with_skipped_pushes():
    seg = lambda ends: np.stack([np.asarray(ends) - 1.5, np.asarray(ends)], 1)
    recs = {'a': (np.zeros((5, 4)), seg([0.0, 1.5, 9.9, 10.0, 25.0])),
            'b': (np.zeros((3, 4)), seg([12.0, 19.0, 20.5])),
            'c': (np.zeros((1, 4)), seg([31.0]))}
    pushes = stream.block_schedule(recs, 10.0)
    assert len(pushes) == 4
    want = [{'a': [0, 1, 2, 3]}, {'b': [0, 1]}, {'a': [4], 'b': [2]}, {'c': [0]}]
    assert [{k: v.tolist() for k, v in p.items()} for p in pushes] == want
    every = {n: np.sort(np.concatenate([p[n] for p in pushes if n in p])) for n in recs}
    assert all(np.array_equal(every[n], np.arange(len(recs[n][0]))) for n in recs)
    with pytest.raises(ValueError):
        stream.block_schedule(recs, 0.0)


def model(Dx=64):
    rng = np.random.default_rng(0)
    return (rng.standard_normal(Dx), rng.standard_normal(R), rng.standard_normal((Dx, R))), \
        (rng.standard_normal(R), np.eye(R), np.ones(R))


@pytest.mark.parametrize('kw', [dict(max_speakers=0), dict(max_speakers=129), dict(max_speakers=True),
                                dict(context=-1), dict(context=2.5), dict(Fb=0.0), dict(loopP=1.5),
                                dict(smoothing=float('nan')), dict(chain='cpu')])
def test_bad_settings(kw):
    transform, plda = model()
    args = dict(Fa=0.3, Fb=17.0, loopP=0.99)
    args.update(kw)
    with pytest.raises(ValueError):
        stream.StreamDiarizer(transform, plda, args.pop('Fa'), args.pop('Fb'), args.pop('loopP'), lda_dim=R, **args)


def test_bad_pushes_fail_before_any_device_work():
    transform, plda = model()
    sd = stream.StreamDiarizer(transform, plda, 0.3, 17.0, 0.99, lda_dim=R)
    seg = np.zeros((3, 2))
    for blocks in ({}, {'a': (np.zeros((0, 64)), np.zeros((0, 2)))}, {'a': (np.zeros((3, 32)), seg)},
                   {'a': (np.zeros((3, 64)), np.zeros((2, 2)))}, [('a', (np.zeros((3, 64)), seg))],
                   {'a': (np.full((3, 64), np.nan), seg)}):
        with pytest.raises(ValueError):
            sd.push(blocks)
    assert sd.state is None and not sd.streams


def test_stream_parser_takes_the_cli_options():
    ap = stream.build_parser()
    args = ap.parse_args(['--out-rttm-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform', 't',
                          '--plda-file', 'p', '--threshold', '-0.015', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17',
                          '--loopP', '0.99', '--block-seconds', '5', '--context', '120'])
    assert args.block_seconds == 5.0 and args.context == 120 and args.max_speakers == 64 and args.timing_json is None
    assert args.init_smoothing == 5.0 and args.chain == 'auto'
