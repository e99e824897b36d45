"""Enrolment against known speakers on the device (DESIGN.md section 5.16): vbx_enroll's statistics, LLRs and
assignments against numpy float64 and scipy (oracle/enroll_oracle.py), bit-identity with vbx_link, determinism across
runs, recording orders and chunks, the tie rules, a synthetic multi-session archive through diarize_batch and the
name-level DER, composition with the other options, ES2005a, and both command lines."""
import io
import json
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from oracle import enroll_oracle, link_oracle, norm_oracle
from test_link_gpu import SPEAKER_WIDTHS, width_phi
from vbx_b200 import cohort, enroll, link, pipeline, score

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
C = 0.3 / 17
THRESHOLDS = (-1e6, -50.0, 0.0, 20.0, 1e6)


def _ragged(seed, R, R_live, E, counts=(3, 0, 128, 1, 17, 0, 2, 40, 150)):
    """A seeded archive (recordings without x-vectors, 1 .. 150 speakers per recording with gaps in the label values, a
    speaker with one x-vector, features >= R_live padded with zeros, Phi from width_phi at the SPEAKER_WIDTHS) and E
    enrolled speakers, packed by speaker, drawn around the same pool of centres."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((40, R_live)) * 2.0
    lens, labels, feas = [], [], []
    for k in counts:
        if k == 0:
            lens.append(0)
            labels.append(np.zeros(0, dtype=np.int64))
            continue
        vals = np.sort(rng.choice(k + 6, k, replace=False))
        per = rng.integers(1, 9, k)
        per[0] = 1
        lab = np.repeat(vals, per)
        rng.shuffle(lab)
        lens.append(len(lab))
        labels.append(lab)
        who = centres[rng.integers(0, 40, k)]
        f = np.zeros((len(lab), R), dtype=np.float32)
        f[:, :R_live] = who[np.searchsorted(vals, lab)] + rng.standard_normal((len(lab), R_live))
        feas.append(f)
    Phi = np.zeros(R, dtype=np.float32)
    Phi[:R_live] = width_phi(rng, R) if R in SPEAKER_WIDTHS else np.sort(rng.uniform(0.2, 6.0, R_live))[::-1]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    espk = np.repeat(np.arange(E), rng.integers(1, 7, E))
    efea = np.zeros((len(espk), R), dtype=np.float32)
    efea[:, :R_live] = centres[rng.integers(0, 40, E)][espk] + rng.standard_normal((len(espk), R_live))
    return np.concatenate(feas), Phi, offs, labels, efea, espk


def _oracle(fea, Phi, offs, labels, efea, espk):
    table = link.speaker_table(labels)
    spk = np.full(len(fea), -1)
    for i, (b, l) in enumerate(zip(table.rec, table.label)):
        seg = slice(offs[b], offs[b + 1])
        spk[seg] = np.where(labels[b] == l, i, spk[seg])
    n, F = link_oracle.statistics(fea, spk, len(table.rec))
    n_e, F_e = link_oracle.statistics(efea, espk, int(espk.max()) + 1)
    rec_off = np.searchsorted(table.rec, np.arange(len(labels) + 1))
    return table, n, F, n_e, F_e, enroll_oracle.llr(n, F, n_e, F_e, Phi, C), rec_off


@pytest.mark.gpu
@pytest.mark.parametrize('R,R_live,E', [(R, R_live, E) for E in (1, 7, 300)
                                        for R, R_live in ((128, 128), (16, 13), (8, 1))]
                         + [(R, R, 33) for R in SPEAKER_WIDTHS])            # E = 33: a tail tile of one column
def test_device_equals_the_oracle(R, R_live, E):
    fea, Phi, offs, labels, efea, espk = _ragged(R + E, R, R_live, E)
    table, n0, F0, ne0, Fe0, L0, rec_off = _oracle(fea, Phi, offs, labels, efea, espk)
    K = np.diff(rec_off)
    assert K.max() > 128 and (K == 0).any()
    scale = np.abs(L0).max()
    for t in THRESHOLDS:
        res = enroll.enroll_speakers(torch.from_numpy(fea).cuda(), torch.from_numpy(Phi).cuda(), offs, labels, efea,
                                     espk, 0.3, 17.0, t, llr=True)
        assert np.array_equal(res.table.rec, table.rec) and np.array_equal(res.table.label, table.label)
        assert np.array_equal(res.n, n0) and np.array_equal(res.n_enroll, ne0)
        np.testing.assert_allclose(res.F, F0, rtol=1e-12, atol=1e-12 * np.abs(F0).max())
        np.testing.assert_allclose(res.F_enroll, Fe0, rtol=1e-12, atol=1e-12 * np.abs(Fe0).max())
        np.testing.assert_allclose(res.llr, L0, rtol=1e-12, atol=1e-12 * scale)
        want, obj = enroll_oracle.assign(L0, rec_off, t)
        assert np.array_equal(res.assign, want), t
        got_obj = enroll_oracle.objective(L0, rec_off, t, res.assign)
        np.testing.assert_allclose(got_obj, obj, rtol=1e-9, atol=1e-9 * max(abs(t), 1.0))
        named = res.assign >= 0
        assert np.array_equal(res.best_llr[named], res.llr[named, res.assign[named]])
        assert np.array_equal(res.best_llr[~named], res.llr[~named].max(axis=1))
        for a, z in zip(rec_off[:-1], rec_off[1:]):           # one name per speaker within a recording
            got = res.assign[a:z][res.assign[a:z] >= 0]
            assert len(set(got.tolist())) == len(got)
        assert (res.llr[named, res.assign[named]] >= t).all()
        if t == -1e6:
            assert all((res.assign[a:z] >= 0).all() for a, z in zip(rec_off[:-1], rec_off[1:]) if z - a <= E)
        if t == 1e6:
            assert not named.any()


def _llr_is_minus_link(fea, Phi, offs, labels, efea, espk):
    """The enrolled speakers appended to the archive as one-speaker recordings: vbx_link's distances between archive and
    enrolled speakers are exactly -llr.  Returns the enrolment result."""
    res = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 0.0, llr=True)
    cnt = np.bincount(espk)
    ext_labels = labels + [np.zeros(k, dtype=np.int64) for k in cnt]
    ext_offs = np.concatenate([offs, offs[-1] + np.cumsum(cnt)])
    table, _, _, _, D = link.link_speakers(np.concatenate([fea, efea]), Phi, ext_offs, ext_labels, 0.3, 17.0, dist=True)
    M = len(res.table.rec)
    assert len(table.rec) == M + len(cnt)
    assert np.array_equal(res.llr, -D[:M, M:])
    return res


@pytest.mark.gpu
def test_llr_is_bit_identical_to_vbx_link():
    _llr_is_minus_link(*_ragged(5, 16, 13, 9))


@pytest.mark.gpu
@pytest.mark.parametrize('R', SPEAKER_WIDTHS)
def test_llr_is_bit_identical_to_vbx_link_and_the_cohort_scores(R):
    """At every width: enrolment llr = -link distance, and the enrolled speakers taken as a cohort score exactly llr."""
    fea, Phi, offs, labels, efea, espk = _ragged(R, R, R, 9)
    res = _llr_is_minus_link(fea, Phi, offs, labels, efea, espk)
    st = cohort.cohort_stats(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, top_k=2, scores=True)
    assert np.array_equal(st.scores, res.llr)


@pytest.mark.gpu
@pytest.mark.parametrize('E', [31, 32, 33])
@pytest.mark.parametrize('M', [32, 33, 64, 65])
def test_tile_edges_at_width_100(M, E):
    """R = 100 (a partial last chunk that ends in a partial log group) at the 32-speaker tile edges: an archive of
    exactly M speakers (M - 24 of them in one recording) linked, enrolled against E speakers and scored against them as
    a cohort of C = E, each against the oracle."""
    R = 100
    fea, Phi, offs, labels, efea, espk = _ragged(100 * M + E, R, R, E, counts=(3, 0, M - 24, 1, 17, 0, 2, 1))
    table, n0, F0, ne0, Fe0, L0, rec_off = _oracle(fea, Phi, offs, labels, efea, espk)
    assert len(table.rec) == M and len(ne0) == E
    t, n, F, Z, D = link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, dist=True)
    assert np.array_equal(n, n0)
    np.testing.assert_allclose(F, F0, rtol=1e-12, atol=1e-12 * np.abs(F0).max())
    D0 = link_oracle.distances(n0, F0, Phi, C, table.rec)
    big = D0 == link.BIG
    assert np.array_equal(D == link.BIG, big) and np.array_equal(D, D.T)
    scale = np.abs(D0[~big]).max()
    np.testing.assert_allclose(D[~big], D0[~big], rtol=1e-12, atol=1e-12 * scale)
    Zs = link_oracle.link(D0)
    low = Zs[:, 2] < 1e15
    assert np.array_equal(Z[:, 2] < 1e15, low)
    np.testing.assert_allclose(Z[low], Zs[low], rtol=1e-12, atol=1e-12 * scale)
    scale = np.abs(L0).max()
    for th in THRESHOLDS:
        res = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, th, llr=True)
        np.testing.assert_allclose(res.llr, L0, rtol=1e-12, atol=1e-12 * scale)
        want, obj = enroll_oracle.assign(L0, rec_off, th)
        assert np.array_equal(res.assign, want), th
    st = cohort.cohort_stats(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, top_k=17, scores=True)
    np.testing.assert_allclose(st.scores, L0, rtol=1e-12, atol=1e-12 * scale)
    mu0, sd0 = norm_oracle.top_stats(L0, 17)
    np.testing.assert_allclose(st.mean, mu0, rtol=1e-12, atol=1e-12 * scale)
    np.testing.assert_allclose(st.std, sd0, rtol=1e-12, atol=1e-12 * scale)


@pytest.mark.gpu
def test_deterministic_permutation_invariant_and_chunked():
    fea, Phi, offs, labels, efea, espk = _ragged(11, 128, 100, 23)
    a = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 10.0, llr=True)
    b = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 10.0, llr=True)
    c = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 10.0, llr=True, max_bytes=8 * 23 * 5)
    for x, y, z in zip(a[1:], b[1:], c[1:]):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    perm = [5, 2, 7, 0, 8, 6, 1, 4, 3]
    pf = np.concatenate([fea[offs[p]:offs[p + 1]] for p in perm])
    pl = [labels[p] for p in perm]
    po = np.concatenate([[0], np.cumsum([offs[p + 1] - offs[p] for p in perm])])
    d = enroll.enroll_speakers(pf, Phi, po, pl, efea, espk, 0.3, 17.0, 10.0)
    key = lambda r, rec_of: {(rec_of[q], l): (e, v) for q, l, e, v in
                             zip(r.table.rec.tolist(), r.table.label.tolist(), r.assign.tolist(), r.best_llr.tolist())}
    assert key(a, list(range(9))) == key(d, perm)


@pytest.mark.gpu
def test_ties():
    """Enrolled speakers 0 and 1 have identical x-vectors: the speaker takes the lower index.  With the threshold equal
    to its LLR the real column (cost exactly 0) wins over the unknown columns; one ulp above, the speaker is unknown."""
    rng = np.random.default_rng(2)
    R = 8
    fea = rng.standard_normal((6, R)).astype(np.float32)
    Phi = np.full(R, 2.0, dtype=np.float32)
    x = fea[:3] + 0.1
    efea = np.concatenate([x, x, rng.standard_normal((2, R)).astype(np.float32) * 3])
    espk = np.array([0, 0, 0, 1, 1, 1, 2, 2])
    labels = [np.zeros(6, dtype=np.int64)]
    r0 = enroll.enroll_speakers(fea, Phi, [0, 6], labels, efea, espk, 0.3, 17.0, -1e6, llr=True)
    assert r0.llr[0, 0] == r0.llr[0, 1] and r0.llr[0, 0] > r0.llr[0, 2]
    assert r0.assign.tolist() == [0]
    top = float(r0.llr[0, 0])
    r1 = enroll.enroll_speakers(fea, Phi, [0, 6], labels, efea, espk, 0.3, 17.0, top)
    assert r1.assign.tolist() == [0] and r1.best_llr.tolist() == [top]
    r2 = enroll.enroll_speakers(fea, Phi, [0, 6], labels, efea, espk, 0.3, 17.0, float(np.nextafter(top, np.inf)))
    assert r2.assign.tolist() == [-1] and r2.best_llr.tolist() == [top]
    print(f'tie case: LLR {top!r}')


# ---- diarize_batch ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return dict(z=z, recs={'ES2005a': (z['x_raw'], z['seg_times'])}, transform=(m['mean1'], m['mean2'], m['lda']),
                plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']),
                kw=dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']),
                        threshold=-0.015, max_iters=40, epsilon=1e-6))


def _sessions(es, seed=13, n_rec=8, pool=10):
    """A multi-session archive: a pool of well-separated speakers (random directions around ES2005a's mean x-vector),
    each recording drawing 2 .. 5 of them with sticky turns; reference rows name speakers p<pool index>.  Also returns
    20 held-out x-vectors of every pool speaker, drawn from the same centres."""
    x_es = es['z']['x_raw']
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + 2.0 * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, rows, truth = {}, [], {}
    for r in range(n_rec):
        T = int(rng.integers(300, 601))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        name = f'ses{r:02d}'
        recs[name] = (x, seg)
        truth[name] = who[spk]
        rows += [(name, round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    return recs, rows, truth, held


def _rows(items, key):
    return [tuple(line.split()[1:2]) + (float(line.split()[3]), float(line.split()[4]), line.split()[7])
            for it in items.values() for line in it[key]]


def _scores(es, recs, out, truth, held):
    """The device LLRs of every VB-HMM speaker against the enrolled pool speakers, from the features diarize_batch ran
    with, each speaker's own pool speaker (the one of most of its x-vectors), and Phi."""
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    dev = torch.device('cuda:0')
    fea, Phi, *_ = pipeline._front_end(recs, names, lens, es['transform'], es['plda'], 128, 'auto', dev,
                                       es['kw']['threshold'])
    fea, Phi = pipeline._pad_features(fea, Phi)
    chain = pipeline._resolve_chain('auto', es['transform'], es['plda'], 128, recs[names[0]][0].shape[1])
    x_e = np.concatenate(list(held.values()))
    front, _, fea_e, _ = pipeline._project(x_e, [len(x_e)], es['transform'], es['plda'], 128, chain, dev)
    front.close()
    fea_e, _ = pipeline._pad_features(fea_e, Phi[:fea_e.shape[1]])
    espk = np.repeat(np.arange(len(held)), [len(v) for v in held.values()])
    offs = np.concatenate([[0], np.cumsum(lens)])
    labels = [out[n]['labels'] for n in names]
    res = enroll.enroll_speakers(fea, Phi, offs, labels, fea_e, espk, es['kw']['Fa'], es['kw']['Fb'], 0.0, llr=True)
    who = np.array([np.bincount(truth[names[b]][labels[b] == l]).argmax()
                    for b, l in zip(res.table.rec, res.table.label)])
    return res, who, Phi.double().cpu().numpy()


@pytest.mark.gpu
def test_multi_session_archive(es):
    recs, rows, truth, held = _sessions(es)
    args = (recs, es['transform'], es['plda'])
    names = list(recs)
    plain = pipeline.diarize_batch(*args, **es['kw'])
    res, who, Phi = _scores(es, recs, plain, truth, held)
    table, M = res.table, len(who)
    own = res.llr[np.arange(M), who]
    other = res.llr.copy()
    other[np.arange(M), who] = -np.inf
    other = other.max(axis=1)
    # the LLR is not calibrated: a speaker with few x-vectors scores less against its own pool speaker than a large one
    # against a different speaker, so no one threshold separates all pairs; but every speaker scores its own pool
    # speaker above every other one, and below the smallest own LLR every speaker is named by its own
    msg = (f'own-speaker LLR {own.min():.1f} .. {own.max():.1f}, other-speaker LLR up to {other.max():.1f}, '
           f'smallest per-speaker margin {np.min(own - other):.1f}')
    print(msg)
    assert (own > other).all(), msg
    theta = float(own.min()) - 1.0
    out = pipeline.diarize_batch(*args, **es['kw'], enroll=held, enroll_threshold=theta)
    for i, (b, l) in enumerate(zip(table.rec.tolist(), table.label.tolist())):
        assert out[names[b]]['speaker_names'][l] == f'p{who[i]}', (names[b], l, msg)
    for n in recs:
        extra = {k: v for k, v in out[n].items() if k not in ('speaker_names', 'speaker_llr', 'rttm_named')}
        assert extra.keys() == plain[n].keys() and extra['rttm'] == plain[n]['rttm']
        assert np.array_equal(extra['labels'], plain[n]['labels'])
    for proto in score.PROTOCOLS:
        per, tot = score.score_rttm(rows, _rows(out, 'rttm_named'), proto[1], proto[2], by_name=True, across_files=True)
        per0, _ = score.score_rttm(rows, _rows(plain, 'rttm'), proto[1], proto[2])
        assert tot['by_name']['ticks']['conf'] == tot['ticks']['conf'], (proto, msg)
        assert tot['by_name']['ticks']['conf'] >= tot['across_files']['ticks']['conf']
        assert per == per0, proto
    # one pool speaker left out of the enrolment: its speakers are unknown, and linked among themselves they share one
    # name.  It is the pool speaker of two or more VB-HMM speakers whose best other-speaker LLR lies furthest below the
    # other speakers' own LLRs; the enrolment threshold lies in between, the link threshold below their pairwise LLRs.
    gap = {}
    for g in set(who.tolist()):
        if (who == g).sum() >= 2:
            gap[g] = (float(other[who == g].max()), float(own[who != g].min()))
    gone = max(gap, key=lambda g: (gap[g][1] - gap[g][0], -g))
    lo, hi = gap[gone]
    mine = np.nonzero(who == gone)[0]
    pair = link_oracle.llr(res.n[mine], res.F[mine], Phi, es['kw']['Fa'] / es['kw']['Fb'])
    link_t = float(pair[~np.eye(len(mine), dtype=bool)].min()) - 1.0
    print(f'left out p{gone} ({len(mine)} speakers): enrolment threshold between {lo:.1f} and {hi:.1f}, '
          f'pairwise LLRs from {link_t + 1.0:.1f}')
    assert lo < hi and len(set(table.rec[mine].tolist())) == len(mine)
    part = {k: v for k, v in held.items() if k != f'p{gone}'}
    for lt in (None, link_t):
        got = pipeline.diarize_batch(*args, **es['kw'], enroll=part, enroll_threshold=(lo + hi) / 2, link_threshold=lt)
        unk = set()
        for i, (b, l) in enumerate(zip(table.rec.tolist(), table.label.tolist())):
            nm = got[names[b]]['speaker_names'][l]
            if who[i] == gone:
                assert nm.startswith('unknown-'), nm
                unk.add(nm)
                if lt is None:
                    assert nm == f'unknown-{names[b]}-{l + 1}'
            else:
                assert nm == f'p{who[i]}'
        assert len(unk) == (1 if lt is not None else len(mine)), unk


@pytest.mark.gpu
def test_composes_and_changes_nothing_else(es):
    recs, _, _, held = _sessions(es, seed=4, n_rec=4)
    args = (recs, es['transform'], es['plda'])
    ovl = {n: [(10.0, 30.0), (50.0, 55.0)] for n in list(recs)[:3]}
    for kw in (dict(overlaps=ovl), dict(num_speakers=3), dict(init='AHC'), dict(overlaps=ovl, max_speakers=2),
               dict(output_2nd=True), dict(link_threshold=0.0)):
        base = pipeline.diarize_batch(*args, **es['kw'], **kw)
        got = pipeline.diarize_batch(*args, **es['kw'], **kw, enroll=held, enroll_threshold=0.0)
        for n in recs:
            extra = {k: v for k, v in got[n].items() if k not in ('speaker_names', 'speaker_llr', 'rttm_named')}
            assert extra.keys() == base[n].keys() and 'rttm_named' not in base[n], kw
            assert all(np.array_equal(extra[k], base[n][k]) if isinstance(base[n][k], np.ndarray) else extra[k] == base[n][k]
                       for k in base[n]), kw
            src = base[n]['rttm_overlap' if 'overlaps' in kw else 'rttm']
            mp = got[n]['speaker_names']
            want = [l.split()[:7] + [mp[int(l.split()[7]) - 1]] + l.split()[8:] for l in src]
            assert [l.split() for l in got[n]['rttm_named']] == want, kw
            assert len(set(mp.values())) == len(mp), kw
            assert set(got[n]['speaker_llr']) == set(np.unique(got[n]['labels']).tolist()), kw


@pytest.mark.gpu
def test_es2005a_enrolled_with_its_own_speakers(es):
    plain = pipeline.diarize_batch(es['recs'], es['transform'], es['plda'], **es['kw'])['ES2005a']
    x = es['z']['x_raw']
    own = {f'spk{l + 1}': x[plain['labels'] == l] for l in np.unique(plain['labels']).tolist()}
    it = pipeline.diarize_batch(es['recs'], es['transform'], es['plda'], **es['kw'], enroll=own,
                                enroll_threshold=0.0)['ES2005a']
    a = [l.split() for l in it['rttm']]
    b = [l.split() for l in it['rttm_named']]
    assert len(a) == len(b) and all(p[:7] == q[:7] and p[8:] == q[8:] for p, q in zip(a, b))
    assert all(q[7] == f'spk{p[7]}' for p, q in zip(a, b))
    print('ES2005a own-speaker LLRs', {k: round(v, 1) for k, v in it['speaker_llr'].items()})


@pytest.mark.gpu
def test_command_lines(es, tmp_path):
    from vbx_b200 import cli, formats
    recs, rows, _, held = _sessions(es, seed=6, n_rec=5)
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    keys, seg_lines, xs = [], [], []
    for name, (x, seg) in recs.items():
        for i, (s, e) in enumerate(seg):
            k = f'{name}_{i:04d}'
            keys.append(k)
            seg_lines.append(f'{k} {name} {float(s)!r} {float(e)!r}')
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
    argv = ['--init', 'AHC+VB', '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']), '--loopP',
            str(z['loopProb']), '--init-smoothing', str(z['smoothing']), '--out-rttm-dir', str(out),
            '--enroll-ark', str(tmp_path / 'e.ark'), '--enroll-utt2spk', str(tmp_path / 'e.utt2spk'),
            '--enroll-threshold', '0', '--output-2nd', 'True']
    with redirect_stdout(io.StringIO()):
        assert cli.main(argv) == 0
    enr = formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'e.utt2spk'))
    got = pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'], enroll=enr, enroll_threshold=0.0,
                                 output_2nd=True)
    for name, it in got.items():
        assert (out / f'{name}.rttm').read_text().splitlines() == it['rttm_named']
        if it['labels2nd'] is not None:
            want = pipeline.named_lines(name, recs[name][1], it['labels2nd'], None, it['speaker_names'])
            assert (tmp_path / 'out2nd' / f'{name}.rttm').read_text().splitlines() == want
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert score.main(['--ref-rttm', str(tmp_path / 'ref'), '--sys-rttm', str(out), '--by-name', '--json']) == 0
    res = json.loads(buf.getvalue())
    _, tot = score.score_rttm(score.read_rttm_path(str(tmp_path / 'ref')), score.read_rttm_path(str(out)), 0.25, False,
                              by_name=True)
    assert res['overall']['by_name'] == json.loads(json.dumps(tot['by_name']))
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert score.main(['--ref-rttm', str(tmp_path / 'ref'), '--sys-rttm', str(out), '--by-name']) == 0
    assert buf.getvalue().splitlines()[-1].startswith('BY NAME')
