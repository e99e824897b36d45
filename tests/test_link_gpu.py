"""Speaker linking across recordings on the device (DESIGN.md section 5.15): vbx_link's statistics, distances and
linkage against numpy float64 and scipy (oracle/link_oracle.py), its tie rule and determinism, a synthetic
multi-session archive through diarize_batch and the DER across files, ES2005a, and both command lines."""
import io
import json
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from oracle import link_oracle
from vbx_b200 import link, pipeline, score

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
C = 0.3 / 17
# Feature widths of the speaker-pair scores (the link and enrolment tiles and verify_score_kernel stage 32-feature
# chunks, and llr_step takes one log per group of 8 denominators): a single partial group (1, 3, 7), one group and one
# feature (9), whole groups inside a chunk (24), both sides of the 32-, 64- and 96-feature chunk edges, and a partial
# last chunk that ends in a partial group (100, 127).  Every feature is live (width_phi).
SPEAKER_WIDTHS = [1, 3, 7, 9, 24, 31, 33, 40, 63, 65, 96, 100, 127]


def width_phi(rng, R):
    """Phi [R] of a SPEAKER_WIDTHS case: every feature live, log-uniform over four decades (1e-2 .. 1e2), descending, so
    that every feature's term shows in the LLR at 1e-12."""
    return np.sort(10.0 ** rng.uniform(-2.0, 2.0, R))[::-1].astype(np.float32)


def _ragged(seed, R, R_live):
    """A seeded archive: recordings without x-vectors, 1 .. 128 speakers per recording with gaps in the label values, a
    speaker with one x-vector, features drawn around a pool of centres; features >= R_live padded with zeros, Phi from
    width_phi at the SPEAKER_WIDTHS."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((40, R_live)) * 2.0
    counts = [3, 0, 128, 1, 17, 0, 2, 40]
    lens, labels, feas = [], [], []
    for k in counts:
        if k == 0:
            lens.append(0)
            labels.append(np.zeros(0, dtype=np.int64))
            continue
        vals = np.sort(rng.choice(k + 6, k, replace=False))          # label values with gaps
        per = rng.integers(1, 9, k)
        per[0] = 1                                                    # a speaker with one x-vector
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
    return np.concatenate(feas), Phi, offs, labels


def _oracle(fea, Phi, offs, labels):
    table = link.speaker_table(labels)
    spk = np.full(len(fea), -1)
    for i, (b, l) in enumerate(zip(table.rec, table.label)):
        seg = slice(offs[b], offs[b + 1])
        spk[seg] = np.where(labels[b] == l, i, spk[seg])
    n, F = link_oracle.statistics(fea, spk, len(table.rec))
    return table, n, F, link_oracle.distances(n, F, Phi, C, table.rec)


def _partition(table, maps):
    g = {}
    for b, l in zip(table.rec.tolist(), table.label.tolist()):
        g.setdefault(maps[b][l], set()).add((b, l))
    return sorted(map(sorted, g.values()))


@pytest.mark.gpu
@pytest.mark.parametrize('seed,R,R_live', [(seed, R, R_live) for seed in (0, 1)
                                            for R, R_live in ((128, 128), (16, 13), (8, 1))]
                         + [(R, R, R) for R in SPEAKER_WIDTHS])
def test_device_equals_the_oracle(R, R_live, seed):
    fea, Phi, offs, labels = _ragged(seed, R, R_live)
    table, n, F, Z, D = link.link_speakers(torch.from_numpy(fea).cuda(), torch.from_numpy(Phi).cuda(), offs, labels,
                                           0.3, 17.0, dist=True)
    t2, n0, F0, D0 = _oracle(fea, Phi, offs, labels)
    M = len(t2.rec)
    assert np.array_equal(table.rec, t2.rec) and np.array_equal(table.label, t2.label) and M > 128
    assert np.array_equal(n, n0)
    np.testing.assert_allclose(F, F0, rtol=1e-12, atol=1e-12 * np.abs(F0).max())
    big = D0 == link.BIG
    assert np.array_equal(D == link.BIG, big) and np.array_equal(D, D.T)
    scale = np.abs(D0[~big]).max()
    np.testing.assert_allclose(D[~big], D0[~big], rtol=1e-12, atol=1e-12 * scale)
    Zs = link_oracle.link(D0)
    low = Zs[:, 2] < 1e15
    assert np.array_equal(Z[:, 2] < 1e15, low)
    np.testing.assert_allclose(Z[low], Zs[low], rtol=1e-12, atol=1e-12 * scale)
    for t in (-1e6, -200.0, -20.0, 0.0, 5.0, 50.0, 1e6):
        maps = link.link_cut(Z, table, t)
        ref = link_oracle.partition(Zs, t)
        want = {}
        for i, (b, l) in enumerate(zip(table.rec.tolist(), table.label.tolist())):
            want.setdefault(int(ref[i]), set()).add((b, l))
        assert _partition(table, maps) == sorted(map(sorted, want.values())), t
        for grp in _partition(table, maps):               # never two speakers of one recording
            assert len({b for b, _ in grp}) == len(grp), t


@pytest.mark.gpu
def test_ties_follow_the_lowest_slot_rule():
    """Four recordings with one speaker each and identical statistics: every distance ties.  The kernel merges the
    lowest slot with its lowest-slot nearest neighbour, and the merged cluster keeps the lower slot."""
    fea = np.tile(np.arange(1, 9, dtype=np.float32)[None, :] / 8, (8, 1))
    offs = np.array([0, 2, 4, 6, 8])
    labels = [np.zeros(2, dtype=np.int64)] * 4
    _, _, _, Z, D = link.link_speakers(fea, np.full(8, 2.0, dtype=np.float32), offs, labels, 0.3, 17.0, dist=True)
    d = D[0, 1]
    assert (D[~np.eye(4, dtype=bool)] == d).all()
    # the second merge is tied exactly (d/2 + d/2 = d); the last merge's height, 2d/3 + d/3, may round off d, and with
    # two clusters left it decides nothing
    assert Z[:, [0, 1, 3]].tolist() == [[0, 1, 2], [2, 4, 3], [3, 5, 4]]
    np.testing.assert_allclose(Z[:, 2], d, rtol=1e-15)


@pytest.mark.gpu
def test_bit_identical_and_permutation_invariant():
    fea, Phi, offs, labels = _ragged(3, 128, 100)
    a = link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, dist=True)
    b = link.link_speakers(fea, Phi, offs, labels, 0.3, 17.0, dist=True)
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)
    perm = [5, 2, 7, 0, 6, 1, 4, 3]
    pf = np.concatenate([fea[offs[p]:offs[p + 1]] for p in perm])
    pl = [labels[p] for p in perm]
    po = np.concatenate([[0], np.cumsum([offs[p + 1] - offs[p] for p in perm])])
    c = link.link_speakers(pf, Phi, po, pl, 0.3, 17.0)
    key = lambda tab, rec_of: [(rec_of[b], l) for b, l in zip(tab.rec.tolist(), tab.label.tolist())]
    ka, kc = key(a[0], list(range(8))), key(c[0], perm)
    order = [kc.index(k) for k in ka]
    assert np.array_equal(c[1][order], a[1]) and np.array_equal(c[2][order], a[2])      # the same sums, bit for bit
    for t in (-50.0, 0.0, 30.0):
        pa = _partition(a[0], link.link_cut(a[3], a[0], t))
        pc = _partition(c[0], link.link_cut(c[3], c[0], t))
        assert sorted(sorted((b, l) for b, l in g) for g in pa) == \
            sorted(sorted((perm[b], l) for b, l in g) for g in pc), t


@pytest.mark.gpu
@pytest.mark.parametrize('R', [100, 128])
@pytest.mark.parametrize('c', [1e30, 1e36, 1e40])
def test_large_c_does_not_overflow_the_log_groups(R, c):
    """Fa = 1, Fb = 1 / c: any finite positive Fa and Fb are accepted, and from c of about 1e36 on a product of 8
    denominators 1 + c (n_i + n_j) Phi_r exceeds DBL_MAX although each is below 1e44.  Zero features make every b 0, so
    an LLR is its log part alone (no cancellation in the oracle either).  The link distances, enrolment, cohort and
    verification LLRs equal the oracle to 1e-12 of the sum of their |log| terms, and are one another bit for bit."""
    from oracle import verify_oracle
    from vbx_b200 import cohort, enroll, verify
    Fa, Fb = 1.0, 1.0 / c
    cc = Fa / Fb                                              # the c of the kernels
    rng = np.random.default_rng(R + int(np.log10(c)))
    Phi = np.sort(10.0 ** rng.uniform(np.log10(0.5), np.log10(40.0), R))[::-1].astype(np.float32)
    n_a = [1, 50, 3, 17, 50, 8, 2, 40, 5, 50, 11, 29]         # two speakers per recording
    labels = [np.repeat([0, 1], n_a[k:k + 2]) for k in range(0, len(n_a), 2)]
    offs = np.concatenate([[0], np.cumsum([len(l) for l in labels])]).astype(np.int64)
    fea = np.zeros((int(offs[-1]), R), dtype=np.float32)
    n_e = [1, 50, 4, 30, 2, 50, 9, 15, 50]
    espk = np.repeat(np.arange(len(n_e)), n_e)
    efea = np.zeros((len(espk), R), dtype=np.float32)
    M, E = len(n_a), len(n_e)
    # the oracle over the archive's speakers and then the enrolled ones
    n = np.array(n_a + n_e, dtype=np.float64)
    L0 = link_oracle.llr(n, np.zeros((M + E, R)), Phi, cc)
    ph = Phi.astype(np.float64)
    logs = np.log(1.0 + cc * n[:, None] * ph[None, :]).sum(1)
    pair = np.array([[np.log(1.0 + cc * (a + b) * ph).sum() for b in n] for a in n])
    scale = pair + logs[:, None] + logs[None, :]              # sum over r of |log L_su| + |log L_s| + |log L_u|
    groups = np.log(1.0 + cc * (n[:, None, None] + n[None, :, None]) * ph[None, None, :])
    groups = np.add.reduceat(groups, np.arange(0, R, 8), axis=2)
    assert ((groups > np.log(np.finfo(np.float64).max)).any()) == (c > 1e33)   # the edge is reached from 1e36 on
    assert np.isfinite(L0).all() and (1.0 + cc * 100 * ph.max()) < 1e300

    def check(got, want, sc):
        assert np.isfinite(got).all()
        assert (np.abs(got - want) <= 1e-12 * np.abs(want) + 1e-12 * sc).all(), np.abs(got - want).max()

    table, nd, _, _, D = link.link_speakers(fea, Phi, offs, labels, Fa, Fb, dist=True)
    assert np.array_equal(nd, n[:M])
    cross = table.rec[:, None] != table.rec[None, :]
    assert np.array_equal(D == link.BIG, ~cross & ~np.eye(M, dtype=bool))
    check(D[cross], -L0[:M, :M][cross], scale[:M, :M][cross])
    res = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, Fa, Fb, 0.0, llr=True)
    check(res.llr, L0[:M, M:], scale[:M, M:])
    st = cohort.cohort_stats(fea, Phi, offs, labels, efea, espk, Fa, Fb, top_k=2, scores=True)
    spk, _ = link.speaker_index(offs, labels)
    ii, jj = np.meshgrid(np.arange(M), np.arange(E), indexing='ij')
    tr = np.stack([ii.ravel(), jj.ravel()], 1)
    v = verify.score_trials(fea, spk, efea, espk, Phi, tr, Fa=Fa, Fb=Fb)
    ne_v, Fe_v = verify_oracle.statistics(fea, spk, M)
    nt_v, Ft_v = verify_oracle.statistics(efea, espk, E)
    check(v, verify_oracle.llr_trials(ne_v, Fe_v, nt_v, Ft_v, ph, cc, tr[:, 0], tr[:, 1]), scale[:M, M:].ravel())
    # the chain: verify = cohort = enrol = -link (the enrolled speakers appended as one-speaker recordings)
    ext = labels + [np.zeros(k, dtype=np.int64) for k in n_e]
    ext_offs = np.concatenate([offs, offs[-1] + np.cumsum(n_e)])
    D2 = link.link_speakers(np.concatenate([fea, efea]), Phi, ext_offs, ext, Fa, Fb, dist=True)[4]
    assert v.tobytes() == st.scores.tobytes() == res.llr.tobytes() == (-D2[:M, M:]).tobytes()


def test_too_many_speakers_is_a_value_error(monkeypatch):
    from vbx_b200 import _lib
    monkeypatch.setattr(_lib, 'LINK_MAX_SPEAKERS', 3)
    with pytest.raises(ValueError, match=r'4 speakers to link.*128 bytes'):
        link.link_speakers(np.zeros((4, 4), np.float32), np.ones(4, np.float32), [0, 4], [np.arange(4)], 0.3, 17.0)


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
    each recording drawing 2 .. 5 of them with sticky turns; reference rows name speakers by pool index."""
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
    return recs, rows, truth


def _rows(items, key):
    return [tuple(line.split()[1:2]) + (float(line.split()[3]), float(line.split()[4]), line.split()[7])
            for it in items.values() for line in it[key]]


def _speaker_llrs(es, recs, out, truth):
    """The smallest same-speaker and the largest different-speaker LLR of the archive's VB-HMM speakers (each taken as
    the pool speaker of most of its x-vectors), recomputed from the features diarize_batch ran with."""
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    fea, Phi, *_ = pipeline._front_end(recs, names, lens, es['transform'], es['plda'], 128, 'auto',
                                       torch.device('cuda:0'), es['kw']['threshold'])
    fea, Phi = pipeline._pad_features(fea, Phi)
    offs = np.concatenate([[0], np.cumsum(lens)])
    labels = [out[n]['labels'] for n in names]
    table, _, _, _, D = link.link_speakers(fea, Phi, offs, labels, es['kw']['Fa'], es['kw']['Fb'], dist=True)
    who = np.array([np.bincount(truth[names[b]][labels[b] == l]).argmax() for b, l in zip(table.rec, table.label)])
    cross = table.rec[:, None] != table.rec[None, :]
    same = cross & (who[:, None] == who[None, :])
    return float((-D[same]).min()), float((-D[cross & ~same]).max())


@pytest.mark.gpu
def test_multi_session_archive(es):
    recs, rows, truth = _sessions(es)
    args = (recs, es['transform'], es['plda'])
    plain = pipeline.diarize_batch(*args, **es['kw'])
    # the synthetic speakers share the offset of ES2005a's mean x-vector, so even different speakers score a positive LLR
    # (with the true labels up to 34.5 here, same speakers from 62.6): the threshold lies in between
    out = pipeline.diarize_batch(*args, **es['kw'], link_threshold=48.0)
    lo_same, hi_diff = _speaker_llrs(es, recs, out, truth)
    msg = f'smallest same-speaker LLR {lo_same:.1f}, largest different-speaker LLR {hi_diff:.1f}'
    for n in recs:
        assert {k: v for k, v in out[n].items() if k not in ('global_speakers', 'rttm_linked')}.keys() == plain[n].keys()
        assert out[n]['rttm'] == plain[n]['rttm'] and np.array_equal(out[n]['labels'], plain[n]['labels'])
    for proto in score.PROTOCOLS:
        _, linked = score.score_rttm(rows, _rows(out, 'rttm_linked'), proto[1], proto[2], across_files=True)
        _, unlinked = score.score_rttm(rows, _rows(plain, 'rttm'), proto[1], proto[2], across_files=True)
        assert linked['across_files']['ticks']['conf'] == linked['ticks']['conf'], (proto, msg)
        assert unlinked['across_files']['der'] > linked['across_files']['der'], (proto, msg)
        assert linked['der'] == unlinked['der'], proto
    print(msg)


@pytest.mark.gpu
def test_es2005a_linked_is_rttm_renamed(es):
    it = pipeline.diarize_batch(es['recs'], es['transform'], es['plda'], **es['kw'], link_threshold=0.0)['ES2005a']
    a = [l.split() for l in it['rttm']]
    b = [l.split() for l in it['rttm_linked']]
    assert len(a) == len(b) and all(x[:7] == y[:7] and x[8:] == y[8:] for x, y in zip(a, b))
    ren = {}
    for x, y in zip(a, b):
        assert ren.setdefault(x[7], y[7]) == y[7]
    assert len(set(ren.values())) == len(ren) == it['n_speakers']
    assert sorted(it['global_speakers'].values()) == list(range(len(it['global_speakers'])))


@pytest.mark.gpu
def test_composes_with_overlaps_counts_and_ahc(es):
    recs, rows, truth = _sessions(es, seed=4, n_rec=4)
    args = (recs, es['transform'], es['plda'])
    ovl = {n: [(10.0, 30.0), (50.0, 55.0)] for n in list(recs)[:3]}
    for kw in (dict(overlaps=ovl), dict(num_speakers=3), dict(init='AHC'), dict(overlaps=ovl, max_speakers=2)):
        base = pipeline.diarize_batch(*args, **es['kw'], **kw)
        got = pipeline.diarize_batch(*args, **es['kw'], **kw, link_threshold=0.0)
        for n in recs:
            extra = {k: v for k, v in got[n].items() if k not in ('global_speakers', 'rttm_linked')}
            assert extra.keys() == base[n].keys() and 'rttm_linked' not in base[n], kw
            assert all(np.array_equal(extra[k], base[n][k]) if isinstance(base[n][k], np.ndarray) else extra[k] == base[n][k]
                       for k in base[n]), kw
            src = base[n]['rttm_overlap' if 'overlaps' in kw else 'rttm']
            assert [l.split()[:7] for l in got[n]['rttm_linked']] == [l.split()[:7] for l in src], kw
            mp = got[n]['global_speakers']
            want = [l.split()[:7] + [str(mp[int(l.split()[7]) - 1] + 1)] + l.split()[8:] for l in src]
            assert [l.split() for l in got[n]['rttm_linked']] == want, kw


@pytest.mark.gpu
def test_command_lines(es, tmp_path):
    from vbx_b200 import cli, formats
    recs, rows, _ = _sessions(es, seed=6, n_rec=5)
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
            '--link-threshold', '0', '--output-2nd', 'True']
    with redirect_stdout(io.StringIO()):
        assert cli.main(argv) == 0
    got = pipeline.diarize_batch(recs, es['transform'], es['plda'], **es['kw'], link_threshold=0.0, output_2nd=True)
    for name, it in got.items():
        assert (out / f'{name}.rttm').read_text().splitlines() == it['rttm_linked']
        if it['labels2nd'] is not None:
            want = pipeline.linked_lines(name, recs[name][1], it['labels2nd'], None, it['global_speakers'])
            assert (tmp_path / 'out2nd' / f'{name}.rttm').read_text().splitlines() == want
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert score.main(['--ref-rttm', str(tmp_path / 'ref'), '--sys-rttm', str(out), '--across-files', '--json']) == 0
    res = json.loads(buf.getvalue())
    _, tot = score.score_rttm(score.read_rttm_path(str(tmp_path / 'ref')), score.read_rttm_path(str(out)), 0.25, False,
                              across_files=True)
    assert res['overall']['across_files'] == json.loads(json.dumps(tot['across_files']))
    buf = io.StringIO()
    with redirect_stdout(buf):
        assert score.main(['--ref-rttm', str(tmp_path / 'ref'), '--sys-rttm', str(out), '--across-files']) == 0
    assert buf.getvalue().splitlines()[-1].startswith('ACROSS FILES')
