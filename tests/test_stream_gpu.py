"""Streaming diarization on the H100 (DESIGN.md section 5.25): vbx_stream_window / vbx_stream_commit against numpy on
the same inputs, the VB-HMM of a window against the float64 oracle, the first push against diarize_batch, batch
independence, the synthetic archive against the streaming oracle, and a speaker returning after leaving the context."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle.prior_oracle import vbx_prior_oracle
from oracle.stream_oracle import StreamOracle, soft_init
from vbx_b200 import pipeline, synth
from vbx_b200.batch import StreamState, VbxBatch
from vbx_b200.stream import StreamDiarizer

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return dict(z=z, transform=(m['mean1'], m['mean2'], m['lda']), plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']),
                kw=dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb'])),
                opts=dict(smoothing=float(z['smoothing']), threshold=-0.015, max_iters=40, epsilon=1e-6))


def poisoned(dev, *specs):
    """Output buffers of the given (shape, dtype) filled with NaN bytes (all bits set: NaN as float, -1 as int), so
    that every element the entry does not write is caught."""
    return [torch.full(shape, float('nan') if dt.is_floating_point else -1, dtype=dt, device=dev) for shape, dt in specs]


# (K, c, count, h) per stream: every tier, a full ring, a ring that overflows, a block longer than the context, a
# stream at S_max (c = 0)
CASES = {'tier0': [(0, 3, 0, 17), (5, 2, 100, 40), (10, 1, 63, 9), (30, 4, 3, 80), (60, 4, 500, 40)],
         'tier1': [(70, 3, 200, 40), (2, 70, 10, 90), (128, 0, 300, 12)]}


def fill_state(st, cases, seed):
    rng = np.random.default_rng(seed)
    for slot, (K, _, count, _) in enumerate(cases):
        st.count[slot] = count
        st.K[slot] = K
        if K:
            st.ctx_lab[slot] = torch.from_numpy(rng.integers(0, K, st.C).astype(np.int32))
            st.n_hist[slot, :K] = torch.from_numpy(rng.integers(0, 50, K).astype(np.float64))
        st.ctx_fea[slot] = torch.from_numpy(rng.standard_normal((st.C, st.R)).astype(np.float32))
        st.F_hist[slot] = torch.from_numpy(rng.standard_normal((st.S_max, st.R)) * 30)


def host_state(st, slot):
    """The oracle's view of one slot: the context in time order, the history, K."""
    C, cnt = st.C, int(st.count[slot])
    L = min(C, cnt)
    pos = [(cnt - L + q) % C for q in range(L)] if C else []
    return (st.ctx_fea[slot].cpu().numpy()[pos].astype(np.float64), st.ctx_lab[slot].cpu().numpy()[pos].astype(np.int64),
            st.n_hist[slot].cpu().numpy().copy(), st.F_hist[slot].cpu().numpy().copy(), int(st.K[slot]))


@pytest.mark.parametrize('case', sorted(CASES))
def test_window_and_commit_against_numpy(dev, es, case):
    cases = CASES[case]
    C, R, S_max = 64, 32, 128
    rng = np.random.default_rng(5)
    st = StreamState(len(cases) + 3, C, R, S_max, dev)
    slots = [len(cases) + 2 - i for i in range(len(cases))]             # not in slot order
    tmp = StreamState(len(cases), C, R, S_max, dev)
    fill_state(tmp, cases, 7)
    for name in StreamState._FIELDS:
        getattr(st, name)[slots] = getattr(tmp, name)
    hs = [np.asarray(rng.integers(0, c, h) if c else np.zeros(h), dtype=np.int32) for K, c, _, h in cases]
    h = np.array([x[3] for x in cases])
    boff = np.concatenate([[0], np.cumsum(h)])
    blk = rng.standard_normal((int(boff[-1]), R)).astype(np.float32)
    blk_d = torch.from_numpy(blk).to(dev)
    lab_d = torch.from_numpy(np.concatenate(hs)).to(dev)
    ns = np.array([K + c for K, c, _, _ in cases])
    lens = np.minimum([x[2] for x in cases], C) + h
    before = [host_state(st, s) for s in slots]
    vb = VbxBatch(lens, R, ns, device=dev)
    f32, f64 = torch.float32, torch.float64
    out = poisoned(dev, ((vb.N, R), f32), ((vb.N, vb.S), f32), ((vb.B, vb.S), f32), ((vb.B,), torch.int32),
                   ((vb.B, vb.S), f64), ((vb.B, vb.S, R), f64))
    fea, g, p, n_states, (pn, pF) = vb.stream_window(st, slots, blk_d, boff, lab_d, [x[1] for x in cases], 5.0, out=out)
    assert fea.data_ptr() == out[0].data_ptr() and pF.data_ptr() == out[5].data_ptr()
    off = vb.offsets
    for b, (K, c, count, hb) in enumerate(cases):
        cf, cl, nh, Fh, _ = before[b]
        w = slice(off[b], off[b + 1])
        np.testing.assert_array_equal(fea[w].cpu().numpy(), np.vstack([cf.astype(np.float32), blk[boff[b]:boff[b + 1]]]))
        labels = np.concatenate([cl, K + hs[b] if c else np.full(hb, -1)])
        want = torch.zeros((len(labels), vb.S), dtype=torch.float32, device=dev)
        want[:, :K + c] = pipeline.soft_init(torch.from_numpy(np.maximum(labels, 0)).to(dev), K + c, 5.0)
        if not c:
            want[len(cl):, :K] = 1.0 / K
        got = g[w]
        assert torch.equal(got[:, K + c:], torch.zeros_like(got[:, K + c:]))
        ulp = torch.abs(got.view(torch.int32).long() - want.view(torch.int32).long()).max().item()
        assert ulp <= 1, (case, b, ulp)
        assert int(n_states[b]) == K + c
        np.testing.assert_array_equal(p[b].cpu().numpy(), np.r_[np.full(K + c, np.float32(1.0 / (K + c))),
                                                                np.zeros(vb.S - K - c, np.float32)])
        np.testing.assert_array_equal(pn[b].cpu().numpy(), np.r_[nh[:K], np.zeros(vb.S - K)])
        np.testing.assert_array_equal(pF[b].cpu().numpy(), np.vstack([Fh[:K], np.zeros((vb.S - K, R))]))
    # commit from arbitrary window labels: the renumbering, the ring and the sequential float64 history
    first = np.concatenate([rng.integers(0, n, l) for n, l in zip(ns, lens)]).astype(np.int32)
    lab_out, = poisoned(dev, ((len(blk),), torch.int32))
    final = vb.stream_commit(st, slots, blk_d, boff, torch.from_numpy(first).to(dev), out=lab_out).cpu().numpy()
    for b, (K, c, count, hb) in enumerate(cases):
        cf, cl, nh, Fh, _ = before[b]
        o = StreamOracle(np.ones(R), 1.0, 1.0, 0.9, context=C, max_speakers=S_max)
        o.ctx_fea, o.ctx_lab, o.n_hist, o.F_hist, o.K = cf, cl, nh, Fh, K
        want = o.commit(first[off[b] + len(cl):off[b + 1]], blk[boff[b]:boff[b + 1]].astype(np.float64))
        np.testing.assert_array_equal(final[boff[b]:boff[b + 1]], want)
        cf2, cl2, nh2, Fh2, K2 = host_state(st, slots[b])
        assert int(st.count[slots[b]]) == count + hb and K2 == o.K
        np.testing.assert_array_equal(cl2, o.ctx_lab)
        np.testing.assert_array_equal(cf2, o.ctx_fea)
        assert np.array_equal(nh2, o.n_hist) and np.array_equal(Fh2.view(np.int64), o.F_hist.view(np.int64))
    # every state tier: the VB-HMM with the prior over the window against the float64 oracle
    vb.prepare_scale(fea, torch.from_numpy(np.linspace(3.0, 0.5, R).astype(np.float32)).to(dev))
    iters, eps = 25, 1e-5
    res = vb.run(g, p, Fa=es['kw']['Fa'], Fb=es['kw']['Fb'], loopProb=es['kw']['loopP'], maxIters=iters,
                 epsilon=eps, prior=(pn, pF))
    Phi = np.linspace(3.0, 0.5, R).astype(np.float32).astype(np.float64)
    fea_h, g_h, p_h = fea.cpu().numpy().astype(np.float64), g.cpu().numpy(), p.cpu().numpy()
    for b, (K, c, _, _) in enumerate(cases):
        n = K + c
        w = slice(off[b], off[b + 1])
        ref = vbx_prior_oracle(fea_h[w], Phi, pn[b, :n].cpu().numpy(), pF[b, :n].cpu().numpy(), loopProb=es['kw']['loopP'],
                               Fa=es['kw']['Fa'], Fb=es['kw']['Fb'], pi=np.full(n, 1.0 / n),
                               gamma=soft_init(window_labels(before[b], hs[b], K, c), n, 5.0), maxIters=iters,
                               epsilon=eps)
        assert int(res['n_iters'][b]) == len(ref[2]), (case, b, int(res['n_iters'][b]), len(ref[2]))
        assert np.abs(g_h[w, :n] - ref[0]).max() < 1e-4, (case, b)
        assert np.abs(p_h[b, :n] - ref[1]).max() < 1e-4, (case, b)
    assert (res['n_iters'].cpu().numpy() < iters).any()         # the stop rule decided somewhere, not maxIters alone
    vb.close()


def window_labels(before, blk_lab, K, c):
    return np.concatenate([before[1], K + blk_lab if c else np.full(len(blk_lab), -1)])


def test_argument_errors(dev):
    vb = VbxBatch([3], 8, 2, device=dev)
    st = StreamState(2, 4, 8, 4, dev)
    L = vb.lib
    z = torch.zeros(64, dtype=torch.float64, device=dev)
    p = ctypes.c_void_p(z.data_ptr())
    args = lambda n=1, C=4, R=8, S_max=4, S=4, slot=p: (vb._h, n, C, R, S_max, S, slot, p, p, p, p, p, 5.0, p, p, p, p, p, p,
                                                        p, p, p, p, p, p, None)
    assert L.vbx_stream_window(*args(slot=None)) == -1
    assert L.vbx_stream_window(*args(n=-1)) == -1
    assert L.vbx_stream_window(*args(C=-1)) == -1
    assert L.vbx_stream_window(*args(R=0)) == -1 and L.vbx_stream_window(*args(R=129)) == -1
    assert L.vbx_stream_window(*args(S_max=129)) == -1 and L.vbx_stream_window(*args(S=0)) == -1
    assert L.vbx_stream_window(*args(n=0, slot=None)) == 0
    a = list(args())
    a[12] = float('nan')
    assert L.vbx_stream_window(*a) == -1
    cargs = lambda n=1, first=p: (vb._h, n, 4, 8, 4, p, p, p, p, first, p, p, p, p, p, p, p, None)
    assert L.vbx_stream_commit(*cargs(first=None)) == -1 and L.vbx_stream_commit(*cargs(n=-1)) == -1
    assert L.vbx_stream_window(None, *args()[1:]) == -1 and L.vbx_stream_commit(None, *cargs()[1:]) == -1
    blk = torch.zeros((3, 8), dtype=torch.float32, device=dev)
    lab = torch.zeros(3, dtype=torch.int32, device=dev)
    for bad in (dict(slots=[2]), dict(blk_off=[0, 2]), dict(n_clusters=[5]), dict(n_clusters=[0]),
                dict(blk=blk.double()), dict(blk=torch.full_like(blk, float('nan'))), dict(lab=lab + 7)):
        with pytest.raises(ValueError):
            vb.stream_window(st, bad.get('slots', [0]), bad.get('blk', blk), bad.get('blk_off', [0, 3]),
                             bad.get('lab', lab), bad.get('n_clusters', [2]), 5.0)
    with pytest.raises(ValueError):
        vb.stream_commit(st, [0], blk, [0, 3], torch.full((3,), 9, dtype=torch.int32, device=dev))
    vb.close()


def archive(es, n_rec=8, seed=13, lengths=(300, 600)):
    return synth.multi_session_archive(es['z']['x_raw'], n_rec=n_rec, seed=seed, lengths=lengths)


def test_first_push_is_diarize_batch(dev, es):
    recs, _, _ = archive(es, n_rec=6, lengths=(60, 400))
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=100)
    got = sd.push(recs)
    off = pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'], **es['opts'], init='AHC+VB')
    for n in recs:
        m = {}
        want = np.array([m.setdefault(l, len(m)) for l in off[n]['labels'].tolist()])
        np.testing.assert_array_equal(got[n]['labels'], want)
        assert got[n]['iterations'] == off[n]['iterations']
        assert [l.split()[:7] for l in sd.rttm(n)] == [l.split()[:7] for l in off[n]['rttm']]


def test_first_push_posteriors_are_diarize_batch_s(dev, es):
    """gamma, pi, iterations and labels of a first push against the VB stage of diarize_batch(init='AHC+VB') on the same
    blocks: the same front end and AHC, soft_init's gamma0 and a uniform pi0, vbx_run without a prior."""
    recs, _, _ = archive(es, n_rec=6, lengths=(60, 400))
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    fea, Phi, labels, _, _ = pipeline._front_end(recs, names, lens, es['transform'], es['plda'], 128, 'auto', dev,
                                                 es['opts']['threshold'])
    fea, Phi = pipeline._pad_features(fea, Phi)
    ns = np.array([int(l.max()) + 1 for l in labels])
    assert ns.max() <= 64
    offs = np.concatenate([[0], np.cumsum(lens)])
    run = dict(Fa=es['kw']['Fa'], Fb=es['kw']['Fb'], loopProb=es['kw']['loopP'], maxIters=40, epsilon=1e-6)
    off = VbxBatch(lens, fea.shape[1], ns, device=dev)
    g0 = torch.zeros((off.N, off.S), dtype=torch.float32, device=dev)
    p0 = torch.zeros((off.B, off.S), dtype=torch.float32, device=dev)
    for b in range(len(names)):
        g0[offs[b]:offs[b + 1], :ns[b]] = pipeline.soft_init(torch.from_numpy(labels[b]).to(dev), int(ns[b]),
                                                             es['opts']['smoothing'])
        p0[b, :ns[b]] = 1.0 / ns[b]
    off.prepare_scale(fea, Phi)
    r_off = off.run(g0, p0, **run)
    st = StreamState(len(names), 100, fea.shape[1], 64, dev)
    sv = VbxBatch(lens, fea.shape[1], ns, device=dev)
    lab_d = torch.from_numpy(np.concatenate(labels).astype(np.int32)).to(dev)
    w_fea, g, p, _, prior = sv.stream_window(st, list(range(len(names))), fea, offs, lab_d, ns, es['opts']['smoothing'])
    assert torch.equal(w_fea, fea) and not bool(prior[0].any()) and not bool(prior[1].any())
    sv.prepare_scale(w_fea, Phi)
    r_st = sv.run(g, p, prior=prior, **run)
    assert torch.equal(r_st['n_iters'], r_off['n_iters'])
    assert float((g - g0).abs().max()) <= 1e-6 and float((p - p0).abs().max()) <= 1e-6
    assert torch.equal(sv.hard_labels(g), off.hard_labels(g0))
    off.close()
    sv.close()


def test_a_failing_push_leaves_streams_consistent(dev, es):
    recs, _, _ = archive(es, n_rec=2, lengths=(100, 120), seed=4)
    a, b = list(recs)
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=50)
    sd.push({a: (recs[a][0][:40], recs[a][1][:40])})
    bad = recs[b][0][:40].copy()
    bad[3] = np.nan
    with pytest.raises(ValueError):
        sd.push({a: (recs[a][0][40:80], recs[a][1][40:80]), b: (bad, recs[b][1][:40])})
    assert sd.streams[a].count == 40 and int(sd.state.count[sd.streams[a].slot]) == 40
    got = sd.push({a: (recs[a][0][40:80], recs[a][1][40:80])})
    assert len(got[a]['labels']) == 40 and sd.streams[a].count == 80


def blocks_of(recs, names, k, h):
    return {n: (recs[n][0][k * h:(k + 1) * h], recs[n][1][k * h:(k + 1) * h]) for n in names if len(recs[n][0]) > k * h}


def test_a_stream_alone_equals_it_in_a_batch_of_64(dev, es):
    recs, _, _ = archive(es, n_rec=64, lengths=(60, 200), seed=3)
    names = list(recs)
    many = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=50)
    one = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=50)
    me = names[7]
    for k in range(5):
        h = 40 + 7 * (k % 2)
        push = {n: (recs[n][0][k * 40:k * 40 + h - (i % 5)], recs[n][1][k * 40:k * 40 + h - (i % 5)])
                for i, n in enumerate(names) if len(recs[n][0]) > k * 40 + 5}
        push = {n: v for n, v in push.items() if len(v[0])}
        if me not in push:
            break
        a, b = many.push(push), one.push({me: push[me]})
        np.testing.assert_array_equal(a[me]['labels'], b[me]['labels'])
        assert a[me]['iterations'] == b[me]['iterations']
        sa, sb = many.streams[me].slot, one.streams[me].slot
        for name in StreamState._FIELDS:
            x, y = getattr(many.state, name)[sa], getattr(one.state, name)[sb]
            assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                               y.view(torch.uint8) if y.is_floating_point() else y), name


def test_synthetic_archive_against_the_streaming_oracle(dev, es):
    recs, _, _ = archive(es, n_rec=4, lengths=(200, 330), seed=21)
    C, h = 120, 40
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=C)
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    x_all = np.concatenate([recs[n][0] for n in names])
    front, x, fea, Phi = pipeline._project(x_all, lens, es['transform'], es['plda'], 128, 'tcgen05', dev)
    front.close()
    offs = np.concatenate([[0], np.cumsum(lens)])
    xs = {n: x[offs[b]:offs[b + 1]].double().cpu().numpy() for b, n in enumerate(names)}
    fs = {n: fea[offs[b]:offs[b + 1]].double().cpu().numpy() for b, n in enumerate(names)}
    orc = {n: StreamOracle(Phi.double().cpu().numpy(), **es['kw'], **es['opts'], context=C) for n in names}
    for k in range(int(np.ceil(lens.max() / h))):
        got = sd.push(blocks_of(recs, names, k, h))
        for n in got:
            want = orc[n].push(xs[n][k * h:(k + 1) * h], fs[n][k * h:(k + 1) * h])
            np.testing.assert_array_equal(got[n]['labels'], want['labels'], err_msg=f'{n} push {k}')


def test_a_speaker_back_after_leaving_the_context(dev, es):
    recs, _, truth = archive(es, n_rec=8, lengths=(400, 600), seed=13)
    # two speakers of one recording: A's x-vectors, then B's, then A's again, one block each
    n = next(n for n in recs if len(np.unique(truth[n])) >= 2)
    spk = np.unique(truth[n])[:2]
    a = np.nonzero(truth[n] == spk[0])[0]
    b = np.nonzero(truth[n] == spk[1])[0]
    h = min(40, len(a) // 2, len(b))
    x, seg = recs[n]
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=h)
    first = sd.push({'s': (x[a[:h]], seg[:h])})
    second = sd.push({'s': (x[b[:h]], seg[h:2 * h])})
    third = sd.push({'s': (x[a[h:2 * h]], seg[2 * h:3 * h])})
    assert set(first['s']['speakers']) == {'spk1'}
    assert set(second['s']['speakers']) == {'spk2'}
    assert set(third['s']['speakers']) == {'spk1'}            # from the prior alone: A's block has left the context


def test_command_line_replays_an_archive(dev, es, tmp_path):
    import json

    from vbx_b200 import formats, score, stream
    z = es['z']
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    x, seg = z['x_raw'], z['seg_times']
    keys = [f'ES2005a_{i:04d}' for i in range(len(x))]
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, x)
    (tmp_path / 'x.seg').write_text(''.join(f'{k} ES2005a {float(s)!r} {float(e)!r}\n' for k, (s, e) in zip(keys, seg)))
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), m['plda_mu'], m['plda_tr'], m['plda_psi'])
    np.savez(str(tmp_path / 'transform.npz'), mean1=m['mean1'], mean2=m['mean2'], lda=m['lda'])
    out = tmp_path / 'out'
    argv = ['--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']), '--loopP',
            str(z['loopProb']), '--init-smoothing', str(z['smoothing']), '--out-rttm-dir', str(out),
            '--block-seconds', '30', '--context', '120', '--timing-json', str(tmp_path / 't.json')]
    assert stream.main(argv) == 0
    recs = {'ES2005a': (x, seg)}
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=120)
    pushes = stream.block_schedule(recs, 30.0)
    for push in pushes:
        if push:
            sd.push({n: (recs[n][0][r], recs[n][1][r]) for n, r in push.items()})
    assert (out / 'ES2005a.rttm').read_text().splitlines() == sd.rttm('ES2005a')
    t = json.load(open(tmp_path / 't.json'))
    assert len(t['pushes']) == len(pushes) and sum(p['xvectors'] for p in t['pushes']) == len(x)
    rows = score.read_rttm_path(str(out))
    assert len(rows) == len(sd.rttm('ES2005a'))
