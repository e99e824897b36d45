"""Score normalisation against a cohort on the device (DESIGN.md section 5.17): vbx_cohort_stats' mean and spread
against numpy float64 (oracle/norm_oracle.py) over top_k, cohort sizes and feature widths, ties at the K-th value,
bit-identity of the cohort LLRs with vbx_enroll, determinism across runs, chunks and cohort order, the normalised link
distances and enrolment assignment against scipy, the spread check, diarize_batch with a cohort, and the calibration
finding on synthetic multi-session archives of two recording lengths."""
import os

import numpy as np
import pytest
import torch

from oracle import enroll_oracle, link_oracle, norm_oracle
from test_link_gpu import SPEAKER_WIDTHS, width_phi
from vbx_b200 import cohort, enroll, link, pipeline

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
C0 = 0.3 / 17
THRESHOLDS = (-1e6, -20.0, -2.0, 0.0, 1.0, 5.0, 1e6)


def _ragged(seed, R, R_live, C, counts=(3, 0, 128, 1, 17, 0, 2, 40, 150)):
    """A seeded archive (recordings without x-vectors, 1 .. 150 speakers per recording with gaps in the label values, a
    speaker with one x-vector, features >= R_live padded with zeros, Phi from width_phi at the SPEAKER_WIDTHS) and C
    cohort speakers packed by speaker, drawn around the same pool of centres."""
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
    cspk = np.repeat(np.arange(C), rng.integers(1, 7, C))
    cfea = np.zeros((len(cspk), R), dtype=np.float32)
    cfea[:, :R_live] = centres[rng.integers(0, 40, C)][cspk] + rng.standard_normal((len(cspk), R_live))
    return np.concatenate(feas), Phi, offs, labels, cfea, cspk


def _oracle(fea, Phi, offs, labels, cfea, cspk):
    """table, n, F of the archive's speakers, and their cohort LLRs [M,C]."""
    table = link.speaker_table(labels)
    spk, M = link.speaker_index(offs, labels)
    n, F = link_oracle.statistics(fea, spk, M)
    n_c, F_c = link_oracle.statistics(cfea, cspk, int(cspk.max()) + 1)
    return table, n, F, norm_oracle.cohort_llr(n, F, n_c, F_c, Phi, C0)


@pytest.mark.gpu
@pytest.mark.parametrize('R,R_live,C', [(R, R_live, C) for C in (2, 33, 1000)
                                        for R, R_live in ((128, 128), (16, 13), (8, 1))]
                         + [(R, R, 33) for R in SPEAKER_WIDTHS])
def test_stats_equal_the_oracle(R, R_live, C):
    fea, Phi, offs, labels, cfea, cspk = _ragged(R + C, R, R_live, C)
    table, n, F, L0 = _oracle(fea, Phi, offs, labels, cfea, cspk)
    scale = np.abs(L0).max()
    for top_k in sorted({k for k in (2, 17, C - 1, C, C + 5) if k >= 2}):
        st = cohort.cohort_stats(torch.from_numpy(fea).cuda(), torch.from_numpy(Phi).cuda(), offs, labels, cfea, cspk,
                                 0.3, 17.0, top_k=top_k, scores=True)
        assert st.K == min(top_k, C)
        np.testing.assert_allclose(st.scores, L0, rtol=1e-12, atol=1e-12 * scale)
        mu0, sd0 = norm_oracle.top_stats(L0, top_k)
        np.testing.assert_allclose(st.mean, mu0, rtol=1e-12, atol=1e-12 * scale)
        np.testing.assert_allclose(st.std, sd0, rtol=1e-12, atol=1e-12 * scale)
        mu1, sd1 = norm_oracle.top_stats(st.scores, top_k)          # the definition on the device's own scores
        np.testing.assert_allclose(st.mean, mu1, rtol=1e-13, atol=1e-14 * scale)
        np.testing.assert_allclose(st.std, sd1, rtol=1e-12, atol=1e-13 * scale)


@pytest.mark.gpu
@pytest.mark.parametrize('top_k', [3, 5, 7, 40])
def test_duplicated_cohort_speakers_tie_at_the_kth_value(top_k):
    """Cohort speakers 20 .. 39 are copies of 0 .. 19: every score occurs twice, so an odd K ends inside a tie."""
    fea, Phi, offs, labels, cfea, cspk = _ragged(3, 16, 13, 20)
    cfea2, cspk2 = np.concatenate([cfea, cfea]), np.concatenate([cspk, cspk + 20])
    st = cohort.cohort_stats(fea, Phi, offs, labels, cfea2, cspk2, 0.3, 17.0, top_k=top_k, scores=True)
    assert np.array_equal(st.scores[:, :20], st.scores[:, 20:])
    mu1, sd1 = norm_oracle.top_stats(st.scores, top_k)
    scale = np.abs(st.scores).max()
    np.testing.assert_allclose(st.mean, mu1, rtol=1e-13, atol=1e-14 * scale)
    np.testing.assert_allclose(st.std, sd1, rtol=1e-12, atol=1e-13 * scale)
    _, _, _, L0 = _oracle(fea, Phi, offs, labels, cfea2, cspk2)
    mu0, sd0 = norm_oracle.top_stats(L0, top_k)
    np.testing.assert_allclose(st.mean, mu0, rtol=1e-12, atol=1e-12 * scale)
    np.testing.assert_allclose(st.std, sd0, rtol=1e-12, atol=1e-12 * scale)


@pytest.mark.gpu
def test_cohort_llr_is_bit_identical_to_vbx_enroll():
    fea, Phi, offs, labels, cfea, cspk = _ragged(5, 128, 100, 45)
    st = cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=10, scores=True)
    res = enroll.enroll_speakers(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, 0.0, llr=True)
    assert np.array_equal(st.scores, res.llr)


@pytest.mark.gpu
def test_deterministic_chunked_and_cohort_order():
    fea, Phi, offs, labels, cfea, cspk = _ragged(11, 128, 100, 300)
    run = lambda **kw: cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=17, scores=True, **kw)
    a, b, c = run(), run(), run(max_bytes=8 * 300 * 7)
    for x, y, z in zip(a[:2] + a[3:], b[:2] + b[3:], c[:2] + c[3:]):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    perm = np.random.default_rng(0).permutation(300)
    inv = np.argsort(perm)
    pf = np.concatenate([cfea[cspk == p] for p in perm])
    ps = np.repeat(np.arange(300), [int((cspk == p).sum()) for p in perm])
    d = cohort.cohort_stats(fea, Phi, offs, labels, pf, ps, 0.3, 17.0, top_k=17, scores=True)
    assert np.array_equal(d.scores[:, inv], a.scores)                 # the same scores, columns permuted
    np.testing.assert_allclose(d.mean, a.mean, rtol=1e-12)
    np.testing.assert_allclose(d.std, a.std, rtol=1e-12)
    # scored speakers given by a speaker index (the enrolled-speaker form) get the same bits as by labels
    spk, M = link.speaker_index(offs, labels)
    e = cohort.cohort_stats(fea, Phi, None, spk, cfea, cspk, 0.3, 17.0, top_k=17)
    assert np.array_equal(e.mean, a.mean) and np.array_equal(e.std, a.std)


def _partition(table, maps):
    g = {}
    for b, l in zip(table.rec.tolist(), table.label.tolist()):
        g.setdefault(maps[b][l], set()).add((b, l))
    return sorted(map(sorted, g.values()))


@pytest.mark.gpu
@pytest.mark.parametrize('R,R_live', [(128, 128), (16, 13)] + [(R, R) for R in SPEAKER_WIDTHS])
def test_normalised_link_distances(R, R_live):
    fea, Phi, offs, labels, cfea, cspk = _ragged(7 + R, R, R_live, 60, counts=(3, 0, 128, 1, 17, 0, 2, 40))
    table, n, F, L0 = _oracle(fea, Phi, offs, labels, cfea, cspk)
    st = cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=20)
    cohort.check_spread(st.std, [str(i) for i in range(len(st.std))])
    t, _, _, Z, D = link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, dist=True, norm=(st.mean, st.std))
    assert np.array_equal(D, D.T)                                        # symmetric bit for bit
    mu0, sd0 = norm_oracle.top_stats(L0, 20)
    np.testing.assert_allclose(st.mean, mu0, rtol=1e-12, atol=1e-12 * np.abs(L0).max())
    np.testing.assert_allclose(st.std, sd0, rtol=1e-12, atol=1e-12 * np.abs(L0).max())
    # the oracle's distances from the device's mu and sigma (checked above): what remains is the LLR's 1e-12, carried
    # through the division by sigma
    D0 = norm_oracle.link_distances(n, F, Phi, C0, table.rec, st.mean, st.std)
    big = D0 == link.BIG
    assert np.array_equal(D == link.BIG, big) and (np.diag(D) == 0).all()
    scale = max(np.abs(D0[~big]).max(), np.abs(link_oracle.llr(n, F, Phi, C0)).max() / st.std.min())
    np.testing.assert_allclose(D[~big], D0[~big], rtol=1e-12, atol=1e-12 * scale)
    Zs = norm_oracle.link(D0)
    low = Zs[:, 2] < 1e15
    assert np.array_equal(Z[:, 2] < 1e15, low)
    np.testing.assert_allclose(Z[low], Zs[low], rtol=1e-12, atol=1e-12 * scale)
    for thr in THRESHOLDS:
        maps = link.link_cut(Z, t, thr)
        ref = norm_oracle.partition(Zs, thr)
        want = {}
        for i, (b, l) in enumerate(zip(table.rec.tolist(), table.label.tolist())):
            want.setdefault(int(ref[i]), set()).add((b, l))
        assert _partition(t, maps) == sorted(map(sorted, want.values())), thr
        for grp in _partition(t, maps):
            assert len({b for b, _ in grp}) == len(grp), thr
    # without norm the call is vbx_link's as before
    plain = link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, dist=True)
    assert not np.array_equal(plain[4], D)


@pytest.mark.gpu
def test_normalised_enrolment():
    fea, Phi, offs, labels, cfea, cspk = _ragged(23, 16, 13, 80)
    rng = np.random.default_rng(1)
    E = 9
    espk = np.repeat(np.arange(E), rng.integers(1, 7, E))
    efea = np.zeros((len(espk), 16), dtype=np.float32)
    efea[:, :13] = rng.standard_normal((E, 13))[espk] * 2.0 + rng.standard_normal((len(espk), 13))
    a = cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, 0.3, 17.0, top_k=30)
    e = cohort.cohort_stats(efea, Phi, None, espk, cfea, cspk, 0.3, 17.0, top_k=30)
    norm = (a.mean, a.std, e.mean, e.std)
    raw = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 0.0, llr=True)
    S0 = norm_oracle.normalise(raw.llr, a.mean, a.std, e.mean, e.std)
    rec_off = np.searchsorted(raw.table.rec, np.arange(len(labels) + 1))
    for thr in THRESHOLDS:
        res = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, thr, llr=True, norm=norm)
        np.testing.assert_allclose(res.llr, S0, rtol=1e-14, atol=1e-14 * np.abs(S0).max())
        want, obj = norm_oracle.assign(res.llr, rec_off, thr)
        assert np.array_equal(res.assign, want), thr
        named = res.assign >= 0
        assert np.array_equal(res.best_llr[named], res.llr[named, res.assign[named]])
        assert np.array_equal(res.best_llr[~named], res.llr[~named].max(axis=1))
        np.testing.assert_allclose(enroll_oracle.objective(res.llr, rec_off, thr, res.assign), obj, rtol=1e-9,
                                   atol=1e-9 * max(abs(thr), 1.0))
    chunked = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 1.0, llr=True, norm=norm,
                                     max_bytes=8 * E * 20)
    whole = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, 0.3, 17.0, 1.0, llr=True, norm=norm)
    assert all(np.array_equal(x, y) for x, y in zip(chunked[1:], whole[1:]))


# ---- diarize_batch ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return dict(z=z, recs={'ES2005a': (z['x_raw'], z['seg_times'])}, transform=(m['mean1'], m['mean2'], m['lda']),
                plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']),
                kw=dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']),
                        threshold=-0.015, max_iters=40, epsilon=1e-6))


def _sessions(es, seed=13, n_rec=8, pool=10, T_range=(300, 601), n_cohort=0):
    """As tests/test_enroll_gpu.py's generator: a pool of well-separated speakers (random directions around ES2005a's
    mean x-vector), each recording drawing 2 .. 5 of them with sticky turns; 20 held-out x-vectors of every pool
    speaker.  T_range sets the recording lengths; n_cohort more speakers drawn the same way (after the rest, so the
    archive does not depend on it) form a disjoint cohort of 20 x-vectors each."""
    x_es = es['z']['x_raw']
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + 2.0 * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, truth = {}, {}
    for r in range(n_rec):
        T = int(rng.integers(*T_range))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        recs[f'ses{r:02d}'] = (x, seg)
        truth[f'ses{r:02d}'] = who[spk]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    cc = x_es.mean(0) + 2.0 * sd * rng.standard_normal((n_cohort, x_es.shape[1]))
    coh = {f'c{k}': cc[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(n_cohort)}
    return recs, truth, held, coh


def _scores(es, recs, out, truth, held, coh, top_k=200):
    """Raw LLRs and normalised scores of every VB-HMM speaker against the enrolled pool speakers, from the features
    diarize_batch ran with, and each speaker's own pool speaker (the one of most of its x-vectors)."""
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    dev = torch.device('cuda:0')
    fea, Phi, *_ = pipeline._front_end(recs, names, lens, es['transform'], es['plda'], 128, 'auto', dev,
                                       es['kw']['threshold'])
    fea, Phi = pipeline._pad_features(fea, Phi)
    side = lambda sets: pipeline._side_features(list(sets.items()), recs, names, es['transform'], es['plda'], 128,
                                                'auto', dev, fea, Phi)
    fea_e, espk = side(held)
    fea_c, cspk = side(coh)
    offs = np.concatenate([[0], np.cumsum(lens)])
    labels = [out[n]['labels'] for n in names]
    Fa, Fb = es['kw']['Fa'], es['kw']['Fb']
    raw = enroll.enroll_speakers(fea, Phi, offs, labels, fea_e, espk, Fa, Fb, 0.0, llr=True)
    a = cohort.cohort_stats(fea, Phi, offs, labels, fea_c, cspk, Fa, Fb, top_k)
    e = cohort.cohort_stats(fea_e, Phi, None, espk, fea_c, cspk, Fa, Fb, top_k)
    nrm = enroll.enroll_speakers(fea, Phi, offs, labels, fea_e, espk, Fa, Fb, 0.0, llr=True,
                                 norm=(a.mean, a.std, e.mean, e.std))
    who = np.array([np.bincount(truth[names[b]][labels[b] == l]).argmax()
                    for b, l in zip(raw.table.rec, raw.table.label)])
    return raw, nrm, who


def _ranges(L, who):
    M = len(who)
    own = L[np.arange(M), who]
    other = L.copy()
    other[np.arange(M), who] = -np.inf
    return own, other.max(axis=1)


@pytest.mark.gpu
def test_calibration_across_recording_lengths(es):
    """The finding of DESIGN.md section 5.17: per archive and for raw and normalised scores, the own-speaker range, the
    largest other-speaker score and whether one threshold separates them, within each archive and across both."""
    found = {}
    for tag, T_range in (('short', (300, 601)), ('long', (1200, 2401))):
        recs, truth, held, coh = _sessions(es, T_range=T_range, n_cohort=200)
        out = pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'])
        raw, nrm, who = _scores(es, recs, out, truth, held, coh)
        for kind, L in (('raw', raw.llr), ('norm', nrm.llr)):
            own, other = _ranges(L, who)
            found[(tag, kind)] = (float(own.min()), float(own.max()), float(other.max()))
            print(f'{tag} archive ({len(who)} speakers), {kind}: own {own.min():.2f} .. {own.max():.2f}, other up to '
                  f'{other.max():.2f}, one threshold separates: {bool(own.min() > other.max())}')
    shift = {}
    for kind in ('raw', 'norm'):
        lo = min(found[(t, kind)][0] for t in ('short', 'long'))
        hi = max(found[(t, kind)][2] for t in ('short', 'long'))
        print(f'both archives, {kind}: own from {lo:.2f}, other up to {hi:.2f}, one threshold separates: {lo > hi}')
        # how far the ranges move between the two lengths, in units of the short archive's own-speaker spread
        s_lo, s_hi, s_other = found[('short', kind)]
        l_lo, _, l_other = found[('long', kind)]
        shift[kind] = max(abs(l_lo - s_lo), abs(l_other - s_other)) / (s_hi - s_lo)
        print(f'{kind}: ranges move by {shift[kind]:.3f} own-speaker spreads between the two lengths')
    # as measured (DESIGN.md section 5.17): neither score separates own from other speakers inside an archive, and the
    # normalised ranges move less between the two lengths than the raw ones
    assert all(found[(t, k)][0] < found[(t, k)][2] for t in ('short', 'long') for k in ('raw', 'norm'))
    assert shift['norm'] < shift['raw']


@pytest.mark.gpu
def test_diarize_batch_with_a_cohort_changes_only_the_linking_and_naming_fields(es):
    recs, truth, held, coh = _sessions(es, seed=4, n_rec=4, n_cohort=40)
    args = (recs, es['transform'], es['plda'])
    ovl = {n: [(10.0, 30.0), (50.0, 55.0)] for n in list(recs)[:3]}
    changed = {'global_speakers', 'rttm_linked', 'speaker_names', 'speaker_llr', 'speaker_score', 'rttm_named',
               'score_norm'}
    for kw in (dict(link_threshold=0.0), dict(enroll=held, enroll_threshold=0.0, overlaps=ovl),
               dict(enroll=held, enroll_threshold=0.0, link_threshold=0.0, num_speakers=3, output_2nd=True)):
        base = pipeline.diarize_batch(*args, **es['kw'], **kw)
        got = pipeline.diarize_batch(*args, **es['kw'], **kw, cohort=coh, cohort_top=25)
        for n in recs:
            assert got[n]['score_norm'] == {'top_k': 25, 'cohort_speakers': 40}
            assert ('speaker_score' in got[n]) == ('enroll' in kw) and 'speaker_llr' not in got[n]
            assert set(got[n]) - changed == set(base[n]) - changed, kw
            for k in set(base[n]) - changed:
                v = base[n][k]
                assert np.array_equal(got[n][k], v) if isinstance(v, np.ndarray) else got[n][k] == v, (kw, k)
            if 'enroll' in kw:
                assert set(got[n]['speaker_score']) == set(np.unique(got[n]['labels']).tolist())
                assert len(set(got[n]['speaker_names'].values())) == len(got[n]['speaker_names'])


@pytest.mark.gpu
def test_a_cohort_without_spread_raises_before_linking_or_enrolment(es, monkeypatch):
    recs, _, held, _ = _sessions(es, seed=4, n_rec=2)
    x = held['p0']
    same = {'a': x, 'b': x.copy(), 'c': x.copy()}              # identical speakers: every cohort score is one number

    def refuse(*a, **k):
        raise AssertionError('a link or enrol kernel ran')
    monkeypatch.setattr(link, 'link_speakers', refuse)
    monkeypatch.setattr(enroll, 'enroll_speakers', refuse)
    for kw in (dict(link_threshold=0.0), dict(enroll=held, enroll_threshold=0.0)):
        with pytest.raises(ValueError, match='without spread'):
            pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'], **kw, cohort=same)
