"""Enrolled speakers in live streams on the H100 (DESIGN.md section 5.29): vbx_stream_enroll's statistics, LLRs and
assignments against the float64 oracle, the enrolled statistics against vbx_enroll_batch's, a first push against
diarize_batch(enroll=), a stream alone against it in a batch of 64, the prior, and the stream command line end to end."""
import io
import json
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from oracle import enroll_oracle
from oracle import stream_enroll_oracle as seo
from vbx_b200 import enroll, formats, pipeline, score
from vbx_b200.batch import StreamEnrolment, StreamState
from vbx_b200.stream import StreamDiarizer
from vbx_b200 import stream as stream_cli

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SPEAKER_WIDTHS = [1, 3, 7, 9, 24, 31, 33, 40, 63, 65, 96, 100, 127]
FA, FB = 0.3, 17.0


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


def sessions(es, seed=13, n_rec=8, pool=10, lengths=(300, 601)):
    """A multi-session archive of well-separated speakers around ES2005a's mean x-vector, with 20 held-out x-vectors of
    every pool speaker (p<index>) to enrol them by."""
    x_es = es['z']['x_raw']
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + 2.0 * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, rows = {}, []
    for r in range(n_rec):
        T = int(rng.integers(*lengths))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        recs[f'ses{r:02d}'] = (x, seg)
        rows += [(f'ses{r:02d}', round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    return recs, rows, held


def poisoned(dev, *specs):
    return [torch.full(shape, float('nan') if dt.is_floating_point else -1, dtype=dt, device=dev) for shape, dt in specs]


def host_ring(st, slot):
    C, cnt = st.C, int(st.count[slot])
    L = min(C, cnt)
    pos = [(cnt - L + q) % C for q in range(L)] if C else []
    return st.ctx_fea[slot].cpu().numpy()[pos].astype(np.float64), st.ctx_lab[slot].cpu().numpy()[pos].astype(np.int64)


# (count, K, named speakers) per stream: an empty ring (a history only), a ring of one row, a partial ring, a full ring,
# a ring that has wrapped (a block longer than C leaves its oldest rows in the history), and a stream whose every
# enrolled speaker is claimed
def fill(dev, C, R, S_max, E, seed):
    rng = np.random.default_rng(seed)
    streams = [(0, 4, []), (1, 3, []), (max(C // 2, 1), 9, [0]), (C, 20, [2, 5]), (5 * C + 7, S_max, [1, S_max - 1]),
               (3 * C + 1, min(S_max, E + 6), list(range(E)))]
    st = StreamState(len(streams) + 2, C, R, S_max, dev)
    en = StreamEnrolment(st, rng.integers(1, 40, E).astype(np.float64), rng.standard_normal((E, R)) * 20)
    slots = [len(streams) + 1 - i for i in range(len(streams))]
    cand = []
    for slot, (count, K, named) in zip(slots, streams):
        st.count[slot], st.K[slot] = count, K
        if C:
            st.ctx_lab[slot] = torch.from_numpy(rng.integers(0, K, C).astype(np.int32))
            st.ctx_fea[slot] = torch.from_numpy(rng.standard_normal((C, R)).astype(np.float32) * 3)
        st.n_hist[slot, :K] = torch.from_numpy(rng.integers(0, 60, K).astype(np.float64))
        st.F_hist[slot, :K] = torch.from_numpy(rng.standard_normal((K, R)) * 40)
        for j, k in enumerate(named):
            en.named[slot, k] = j % E
        free = [k for k in range(K) if k not in named]
        cand.append(sorted(rng.choice(free, max(1, len(free) // 2), replace=False).tolist()))
    return st, en, slots, cand, rng


@pytest.mark.parametrize('R, C, S_max', [(8, 16, 64), (16, 16, 128), (128, 240, 64), (128, 0, 64), (128, 33, 128)]
                         + [(R, 24, 64) for R in SPEAKER_WIDTHS])
def test_candidates_against_the_oracle(dev, R, C, S_max):
    E = 33
    st, en, slots, cand, rng = fill(dev, C, R, S_max, E, seed=R + C)
    Phi = torch.from_numpy(np.geomspace(0.05, 40.0, R).astype(np.float32)).to(dev)
    M = sum(len(c) for c in cand)
    before = {s: (st.n_hist[s].cpu().numpy().copy(), st.F_hist[s].cpu().numpy().copy(), en.named[s].cpu().numpy().copy())
              for s in slots}
    out = poisoned(dev, ((M,), torch.int32), ((M,), torch.float64), ((M, E), torch.float64), ((M,), torch.float64),
                   ((M, R), torch.float64))
    n_e, F_e, ph = en.n_enroll.cpu().numpy(), en.F_enroll.cpu().numpy(), Phi.double().cpu().numpy()
    tops = []                    # the threshold: the median best LLR, so that some candidates are named and some not
    for s, ks in zip(slots, cand):
        claimed = [int(x) for x in before[s][2] if x >= 0]
        if len(set(claimed)) < E:
            l = enroll_oracle.llr(*seo.candidate_stats(before[s][0], before[s][1], *host_ring(st, s), ks), n_e, F_e, ph,
                                  FA / FB)
            tops += np.delete(l, claimed, axis=1).max(1).tolist()
    thr = float(np.median(tops))
    a, best, llr, n, F = (t.cpu().numpy() for t in en.assign(st, slots, cand, Phi, FA, FB, thr, out=out))
    o = 0
    for s, ks in zip(slots, cand):
        m = slice(o, o + len(ks))
        ring_fea, ring_lab = host_ring(st, s)
        n_o, F_o = seo.candidate_stats(before[s][0], before[s][1], ring_fea, ring_lab, ks)
        np.testing.assert_array_equal(n[m], n_o)
        np.testing.assert_allclose(F[m], F_o, rtol=0, atol=1e-12 * max(1.0, np.abs(F_o).max()))
        want = enroll_oracle.llr(n[m], F[m], n_e, F_e, ph, FA / FB)
        np.testing.assert_allclose(llr[m], want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()))
        claimed = [int(x) for x in before[s][2] if x >= 0]
        a_o, best_o = seo.assign(llr[m], claimed, thr)
        np.testing.assert_array_equal(a[m], a_o)
        np.testing.assert_array_equal(best[m], best_o)
        if len(set(claimed)) == E:
            assert (a[m] == -1).all() and (best[m] == -np.inf).all()
        named = before[s][2].copy()
        named[np.array(ks)[a_o >= 0]] = a_o[a_o >= 0]
        np.testing.assert_array_equal(en.named[s].cpu().numpy(), named)
        np.testing.assert_array_equal(st.n_hist[s].cpu().numpy(), before[s][0])      # no prior: history untouched
        o += len(ks)
    assert (a >= 0).any() and (a == -1).any()


def test_prior_adds_the_enrolled_statistics_exactly(dev):
    E, R, C = 7, 128, 40
    st, en, slots, cand, _ = fill(dev, C, R, 64, E, seed=2)
    Phi = torch.from_numpy(np.geomspace(0.05, 40.0, R).astype(np.float32)).to(dev)
    n0, F0 = st.n_hist.clone(), st.F_hist.clone()
    a = en.assign(st, slots, cand, Phi, FA, FB, -1e6, prior=True)[0].cpu().numpy()
    n_want, F_want = n0.clone(), F0.clone()
    o = 0
    for s, ks in zip(slots, cand):
        for k in ks:
            if a[o] >= 0:
                n_want[s, k] += en.n_enroll[a[o]]
                F_want[s, k] += en.F_enroll[a[o]]
            o += 1
    assert (a >= 0).sum() > 3
    assert torch.equal(st.n_hist, n_want) and torch.equal(st.F_hist.view(torch.uint8), F_want.view(torch.uint8))


def test_refusals(dev):
    E, R, C = 3, 16, 8
    st, en, slots, cand, _ = fill(dev, C, R, 64, E, seed=1)
    Phi = torch.ones(R, dtype=torch.float32, device=dev)
    named_k = int(np.nonzero(en.named[slots[2]].cpu().numpy() >= 0)[0][0])
    for bad in (dict(candidates=[[0]] * (len(slots) - 1)), dict(candidates=[[]] + cand[1:]),
                dict(candidates=[[0, 0]] + cand[1:]), dict(candidates=[[4]] + cand[1:]),       # K = 4 in slot 0's stream
                dict(candidates=cand[:2] + [[named_k]] + cand[3:]), dict(slots=[slots[0]] * len(slots)),
                dict(slots=[st.slots] + slots[1:]), dict(threshold=float('nan')), dict(Fb=0.0),
                dict(Phi=torch.ones(R + 1, dtype=torch.float32, device=dev))):
        kw = dict(state=st, slots=slots, candidates=cand, Phi=Phi, Fa=FA, Fb=FB, threshold=0.0)
        kw.update(bad)
        with pytest.raises(ValueError):
            en.assign(**kw)
    with pytest.raises(ValueError):
        StreamEnrolment(st, np.ones(2), np.zeros((2, R + 1)))


def test_enrolled_statistics_are_vbx_enroll_batch_s(dev, es):
    recs, _, held = sessions(es, n_rec=1, lengths=(80, 81))
    name = next(iter(recs))
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], enroll=held, enroll_threshold=0.0)
    got = sd.push({name: (recs[name][0][:40], recs[name][1][:40])})
    x_e = np.concatenate(list(held.values()))
    front, _, fea_e, Phi = pipeline._project(x_e, [len(x_e)], es['transform'], es['plda'], 128, 'tcgen05', dev)
    front.close()
    fea_e, Phi = pipeline._pad_features(fea_e, Phi)
    front, _, fea, _ = pipeline._project(recs[name][0][:40], [40], es['transform'], es['plda'], 128, 'tcgen05', dev)
    front.close()
    res = enroll.enroll_speakers(fea, Phi, [0, 40], [got[name]['labels']], fea_e,
                                 np.repeat(np.arange(len(held)), 20), sd.Fa, sd.Fb, 0.0, dev)
    assert np.array_equal(sd.enrolment.n_enroll.cpu().numpy(), res.n_enroll)
    assert sd.enrolment.F_enroll.cpu().numpy().tobytes() == np.ascontiguousarray(res.F_enroll).tobytes()


def test_first_push_is_diarize_batch_with_enrolment(dev, es):
    recs, _, held = sessions(es, n_rec=6, seed=4)
    thr = 0.0
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=700, enroll=held,
                        enroll_threshold=thr)
    got = sd.push(recs)
    off = pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'], **es['opts'], init='AHC+VB',
                                 enroll=held, enroll_threshold=thr)
    n_named = 0
    for n in recs:
        m = {}
        want = np.array([m.setdefault(l, len(m)) for l in off[n]['labels'].tolist()])
        np.testing.assert_array_equal(got[n]['labels'], want)
        for l_off, k in m.items():
            name = off[n]['speaker_names'][l_off]
            if name.startswith(enroll.UNKNOWN):
                assert k not in got[n]['named']
            else:
                assert got[n]['named'][k] == name
                n_named += 1
            v, w = got[n]['enroll_llr'][k], off[n]['speaker_llr'][l_off]
            assert abs(v - w) <= 1e-12 * max(1.0, abs(w)), (n, k, v, w)
        assert got[n]['speakers'] == [got[n]['named'].get(k, f'spk{k + 1}') for k in got[n]['labels'].tolist()]
        assert [l.split()[:7] for l in sd.rttm(n)] == [l.split()[:7] for l in off[n]['rttm_named']]
    assert n_named >= len(recs)


def test_a_stream_alone_equals_it_in_a_batch_of_64(dev, es):
    recs, _, held = sessions(es, n_rec=64, seed=3, lengths=(60, 200))
    names = list(recs)
    kw = dict(context=50, enroll=held, enroll_threshold=0.0, enroll_prior=True)
    many = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], **kw)
    one = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], **kw)
    me = names[7]
    for k in range(5):
        push = {n: (recs[n][0][k * 40:k * 40 + 40 - (i % 5)], recs[n][1][k * 40:k * 40 + 40 - (i % 5)])
                for i, n in enumerate(names) if len(recs[n][0]) > k * 40 + 5}
        if me not in push:
            break
        a, b = many.push(push), one.push({me: push[me]})
        for key in ('labels', 'speakers', 'named', 'enroll_llr'):
            assert str(a[me][key]) == str(b[me][key]), key
        assert a[me]['enroll_llr'] == b[me]['enroll_llr']
        sa, sb = many.streams[me].slot, one.streams[me].slot
        for name in StreamState._FIELDS:
            x, y = getattr(many.state, name)[sa], getattr(one.state, name)[sb]
            assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x,
                               y.view(torch.uint8) if y.is_floating_point() else y), name
        assert torch.equal(many.enrolment.named[sa], one.enrolment.named[sb])
    assert many.streams[me].names


def test_enroll_prior_changes_the_next_window_prior_by_the_enrolment(dev, es):
    recs, _, held = sessions(es, n_rec=1, seed=8, lengths=(200, 201))
    name = next(iter(recs))
    block = {name: (recs[name][0][:60], recs[name][1][:60])}
    kw = dict(context=30, enroll=held, enroll_threshold=0.0)
    plain = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], **kw)
    prior = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], enroll_prior=True, **kw)
    a, b = plain.push(block), prior.push(block)
    assert a[name]['named'] == b[name]['named'] and b[name]['named']
    s = plain.streams[name].slot
    n_want, F_want = plain.state.n_hist[s].clone(), plain.state.F_hist[s].clone()
    enrolled = [k for k, _ in prior.enrolled]
    for k, nm in b[name]['named'].items():
        n_want[k] += prior.enrolment.n_enroll[enrolled.index(nm)]
        F_want[k] += prior.enrolment.F_enroll[enrolled.index(nm)]
    t = prior.streams[name].slot
    assert torch.equal(prior.state.n_hist[t], n_want)
    assert torch.equal(prior.state.F_hist[t].view(torch.uint8), F_want.view(torch.uint8))


def test_command_line_end_to_end(dev, es, tmp_path):
    recs, rows, held = sessions(es, seed=6, n_rec=3)
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    keys, seg_lines, xs = [], [], []
    for name, (x, seg) in recs.items():
        for i, (s, e) in enumerate(seg):
            keys.append(f'{name}_{i:04d}')
            seg_lines.append(f'{name}_{i:04d} {name} {float(s)!r} {float(e)!r}')
        xs.append(x)
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, np.concatenate(xs))
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    ekeys = [f'{k}-{i:02d}' for k, v in held.items() for i in range(len(v))]
    formats.write_vec_flt_ark(str(tmp_path / 'e.ark'), ekeys, np.concatenate(list(held.values())))
    (tmp_path / 'e.utt2spk').write_text(''.join(f'{k} {k.rsplit("-", 1)[0]}\n' for k in ekeys))
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), m['plda_mu'], m['plda_tr'], m['plda_psi'])
    np.savez(str(tmp_path / 'transform.npz'), mean1=m['mean1'], mean2=m['mean2'], lda=m['lda'])
    (tmp_path / 'ref').mkdir()
    for name in recs:
        (tmp_path / 'ref' / f'{name}.rttm').write_text(''.join(
            f'SPEAKER {r[0]} 1 {r[1]:.2f} {r[2]:.2f} <NA> <NA> {r[3]} <NA> <NA>\n' for r in rows if r[0] == name))
    z = es['z']
    out = tmp_path / 'out'
    argv = ['--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']), '--loopP',
            str(z['loopProb']), '--init-smoothing', str(z['smoothing']), '--out-rttm-dir', str(out),
            '--block-seconds', '10', '--enroll-ark', str(tmp_path / 'e.ark'), '--enroll-utt2spk',
            str(tmp_path / 'e.utt2spk'), '--enroll-threshold', '0', '--enroll-prior']
    assert stream_cli.main(argv) == 0
    enr = formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'e.utt2spk'))
    sd = StreamDiarizer(es['transform'], es['plda'], float(z['Fa']), float(z['Fb']), float(z['loopProb']),
                        smoothing=float(z['smoothing']), enroll=enr, enroll_threshold=0.0, enroll_prior=True)
    for push in stream_cli.block_schedule(recs, 10.0):
        if push:
            sd.push({n: (recs[n][0][r], recs[n][1][r]) for n, r in push.items()})
    names = set()
    for name in recs:
        lines = (out / f'{name}.rttm').read_text().splitlines()
        assert lines == sd.rttm(name)
        names |= {line.split()[7] for line in lines}
    assert names & set(held)
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert score.main(['--ref-rttm', str(tmp_path / 'ref'), '--sys-rttm', str(out), '--by-name', '--json']) == 0
    assert 'by_name' in json.loads(buf.getvalue())['overall']


def test_without_enrolment_a_stream_is_what_it_was(dev, es):
    """enroll=None: a multi-push run gives the labels of the streaming oracle, the spk<k+1> speakers, rttm_lines RTTMs,
    no new result or timing fields, no enrolment state, and a history equal to the oracle's."""
    from oracle.stream_oracle import StreamOracle
    recs, _, _ = sessions(es, n_rec=3, seed=21, lengths=(200, 330))
    C, h = 120, 40
    sd = StreamDiarizer(es['transform'], es['plda'], **es['kw'], **es['opts'], context=C)
    sd.timing = []
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    front, x, fea, Phi = pipeline._project(np.concatenate([recs[n][0] for n in names]), lens, es['transform'],
                                           es['plda'], 128, 'tcgen05', dev)
    front.close()
    offs = np.concatenate([[0], np.cumsum(lens)])
    xs = {n: x[offs[b]:offs[b + 1]].double().cpu().numpy() for b, n in enumerate(names)}
    fs = {n: fea[offs[b]:offs[b + 1]].double().cpu().numpy() for b, n in enumerate(names)}
    orc = {n: StreamOracle(Phi.double().cpu().numpy(), **es['kw'], **es['opts'], context=C) for n in names}
    for k in range(int(np.ceil(lens.max() / h))):
        blocks = {n: (recs[n][0][k * h:(k + 1) * h], recs[n][1][k * h:(k + 1) * h]) for n in names
                  if len(recs[n][0]) > k * h}
        got = sd.push(blocks)
        for n in got:
            want = orc[n].push(xs[n][k * h:(k + 1) * h], fs[n][k * h:(k + 1) * h])
            np.testing.assert_array_equal(got[n]['labels'], want['labels'])
            assert set(got[n]) == {'labels', 'speakers', 'iterations'}
            assert got[n]['speakers'] == [f'spk{l + 1}' for l in got[n]['labels'].tolist()]
    assert sd.enrolment is None and all('enroll' not in t for t in sd.timing)
    for n in names:
        st = sd.streams[n]
        seg = np.concatenate(st.seg)
        assert sd.rttm(n) == pipeline.rttm_lines(n, *pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1],
                                                                                     np.concatenate(st.labels)))
        assert int(sd.state.K[st.slot]) == orc[n].K
        np.testing.assert_array_equal(sd.state.n_hist[st.slot].cpu().numpy(), orc[n].n_hist)
