"""Speaker-count constraints on the device (DESIGN.md section 5.14): vbx_hard_labels_keep against the numpy rules of
oracle/count_oracle.py, ES2005a through diarize_batch under every rule, a synthetic archive with known speaker counts
through diarize_batch and sweep_batch(num_speakers='oracle'), and the command line."""
import os

import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import fcluster

from oracle import ahc_oracle, count_oracle, vbx_oracle
from vbx_b200 import VbxError, pipeline, sweep, synth
from vbx_b200.batch import VbxBatch

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return dict(z=z, recs={'ES2005a': (z['x_raw'], z['seg_times'])}, transform=(m['mean1'], m['mean2'], m['lda']),
                plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']),
                kw=dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']),
                        threshold=-0.015, max_iters=40, epsilon=1e-6))


def _diarize(es, **kw):
    return pipeline.diarize_batch(es['recs'], es['transform'], es['plda'], **es['kw'], **kw)['ES2005a']


# ---- the kernel ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('S', [4, 7, 16, 33, 64, 100, 128])
def test_hard_labels_keep_equals_the_oracle(S):
    """Ragged batch with recordings without frames, random live-state counts and a random keep (also 1 and >= n_states),
    tied columns (tied masses) and tied entries: labels equal the numpy rule exactly, masses to rounding."""
    rng = np.random.default_rng(S)
    dev = torch.device('cuda:0')
    lens = [0, 50, 1, 129, 0, 300, 64, 65, 700]
    ns = rng.integers(1, S + 1, len(lens)).astype(np.int32)
    ns[5] = S
    vb = VbxBatch(lens, 128, ns, device=dev, allocate=False)
    offs = np.concatenate([[0], np.cumsum(lens)])
    g = np.zeros((vb.N, vb.S), dtype=np.float32)
    for b in range(len(lens)):
        if lens[b] == 0:
            continue
        q = rng.dirichlet(np.full(ns[b], 0.3), size=lens[b])
        if ns[b] > 2:
            q[:, ns[b] - 1] = q[:, 0]                 # a tied pair of columns: equal masses
            q[::4, 1] = q[::4, 0]                     # ties inside rows
        g[offs[b]:offs[b + 1], :ns[b]] = q
    keep = np.array([int(rng.integers(1, n + 2)) for n in ns], dtype=np.int32)
    keep[1], keep[3] = 1, ns[3] + 3
    first, second, mass = vb.hard_labels_keep(torch.from_numpy(g).to(dev), keep)
    first, second, mass = first.cpu().numpy(), second.cpu().numpy(), mass.cpu().numpy()
    for b in range(len(lens)):
        n = int(ns[b])
        gb = g[offs[b]:offs[b + 1]].astype(np.float64)
        f, s, m = count_oracle.keep_labels(gb, n, int(keep[b]))
        assert np.array_equal(first[offs[b]:offs[b + 1]], f), b
        assert np.array_equal(second[offs[b]:offs[b + 1]], s), b
        np.testing.assert_allclose(mass[b, :n], m, rtol=1e-13, atol=0)
        assert not mass[b, n:].any()
        if lens[b] == 0:
            assert not mass[b].any()
    vb.close()


@pytest.mark.gpu
@pytest.mark.parametrize('gemm', [0, 1])
@pytest.mark.parametrize('S', [8, 128])
def test_keep_all_states_is_hard_labels(gemm, S):
    """keep >= n_states: bit for bit vbx_hard_labels, on posteriors of a real VB-HMM run in either contraction mode."""
    dev = torch.device('cuda:0')
    lens = [300, 0, 45, 1, 129]
    ns = np.array([S, 1, max(S // 2, 1), 3, S - 1], dtype=np.int32)
    d = synth.make_batch([t for t in lens if t], R=128, S=S, seed=5, dtype=np.float32)
    vb = VbxBatch(lens, 128, ns, device=dev)
    vb.set_option('gemm', gemm)
    offs = np.concatenate([[0], np.cumsum(lens)])
    g0 = d['gamma0'].copy()
    for b in range(len(lens)):
        g0[offs[b]:offs[b + 1], ns[b]:] = 0
        g0[offs[b]:offs[b + 1]] /= g0[offs[b]:offs[b + 1]].sum(1, keepdims=True)
    g = torch.zeros((vb.N, vb.S), device=dev)
    g[:, :S] = torch.from_numpy(g0).to(dev)
    p = torch.zeros((len(lens), vb.S), device=dev)
    for b in range(len(lens)):
        p[b, :ns[b]] = 1.0 / ns[b]
    vb.prepare_scale(torch.from_numpy(d['fea']).to(dev), torch.from_numpy(d['Phi']).to(dev))
    vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=5, epsilon=-float('inf'))
    f0, s0 = vb.hard_labels(g, second=True)
    for keep in (ns, ns + 4):
        f1, s1, mass = vb.hard_labels_keep(g, keep)
        assert torch.equal(f0, f1) and torch.equal(s0, s1)
    assert mass[1].abs().sum().item() == 0.0
    with pytest.raises(VbxError):
        vb.hard_labels_keep(g, np.where(np.arange(len(lens)) == 2, 0, ns))
    vb.close()


# ---- ES2005a --------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_es2005a_counts_inside_the_bounds_change_nothing(es):
    base = _diarize(es)
    assert base['n_speakers'] == 5 and 'count_rule' not in base
    for c in (dict(num_speakers=5), dict(max_speakers=5), dict(min_speakers=1), dict(min_speakers=2, max_speakers=9)):
        it = _diarize(es, **c)
        assert it['count_rule'] == 'vb' and it['n_speakers_vb'] == 5, c
        assert it['rttm'] == base['rttm'] and it['iterations'] == base['iterations'], c
        assert np.array_equal(it['labels'], base['labels']) and np.array_equal(it['labels2nd'], base['labels2nd']), c
    assert _diarize(es, min_speakers=1)['count'] == (1, None) and _diarize(es, max_speakers=5)['count'] == (1, 5)


def _es_posteriors(es):
    """The final posteriors of diarize_batch's unconstrained run, recomputed the way its single tier computes them."""
    dev = torch.device('cuda:0')
    recs = es['recs']
    lens = np.array([len(es['z']['x_raw'])])
    fea, Phi, ahc_labels, _, _ = pipeline._front_end(recs, list(recs), lens, es['transform'], es['plda'], 128, 'auto', dev,
                                                     -0.015)
    fea, Phi = pipeline._pad_features(fea, Phi)
    S = int(ahc_labels[0].max()) + 1
    vb = VbxBatch(lens, int(fea.shape[1]), [S], device=dev)
    g = torch.zeros((vb.N, vb.S), device=dev)
    g[:, :S] = pipeline.soft_init(torch.from_numpy(ahc_labels[0]).to(dev), S, es['kw']['smoothing'])
    p = torch.zeros((1, vb.S), device=dev)
    p[0, :S] = 1.0 / S
    vb.prepare_scale(fea, Phi)
    kw = es['kw']
    vb.run(g, p, Fa=kw['Fa'], Fb=kw['Fb'], loopProb=kw['loopP'], maxIters=40, epsilon=1e-6)
    out = g[:, :S].double().cpu().numpy()
    vb.close()
    return out


@pytest.mark.gpu
def test_es2005a_four_speakers_by_posterior_mass(es):
    base = _diarize(es)
    it = _diarize(es, num_speakers=4)
    g = _es_posteriors(es)
    assert np.array_equal(np.argsort(-g, axis=1, kind='stable')[:, 0], base['labels'])
    f, s, _ = count_oracle.keep_labels(g, g.shape[1], 4)
    assert it['count_rule'] == 'mass' and it['n_speakers_vb'] == 5 and it['n_speakers'] == 4
    assert np.array_equal(it['labels'], f) and np.array_equal(it['labels2nd'], s)
    assert it['iterations'] == base['iterations']
    one = _diarize(es, max_speakers=1)
    assert one['count_rule'] == 'mass' and one['n_speakers'] == 1 and one['labels2nd'] is None


@pytest.mark.gpu
def test_es2005a_seven_speakers_recut(es):
    """min_speakers=7: rule 3 against the oracle pipeline (the float64 linkage cut with maxclust at 7, then the float64
    VBx oracle from that initialisation)."""
    z = es['z']
    it = _diarize(es, min_speakers=7)
    _, _, Z = ahc_oracle.ahc_labels(z['x_lda'])
    Z = Z.copy()
    Z[:, 2] += abs(Z[:, 2].min())          # scipy's fcluster wants distances >= 0; the shift does not change the cut
    mc = fcluster(Z, 7, criterion='maxclust') - 1
    ns = int(mc.max()) + 1
    q0 = np.exp(np.eye(ns)[mc] * float(z['smoothing']))
    q0 /= q0.sum(1, keepdims=True)
    gamma, _, _ = vbx_oracle.vbx_oracle(z['fea'], z['Phi'], loopProb=float(z['loopProb']), Fa=float(z['Fa']),
                                        Fb=float(z['Fb']), pi=ns, gamma=q0, maxIters=40, epsilon=1e-6)
    order = np.argsort(-gamma, axis=1, kind='stable')

    def rerun(init):
        assert np.array_equal(init, mc)
        return order[:, 0], order[:, 1]

    lab, lab2, rule, k1 = count_oracle.vb_rules(np.zeros(len(mc), dtype=np.int64), None, None, 7, pipeline.UNBOUNDED,
                                                Z, rerun)
    print('ES2005a min_speakers=7:', rule, len(np.unique(lab)), 'speakers')
    assert it['count_rule'] == rule and it['n_speakers_vb'] == 5
    assert np.array_equal(it['labels'], lab)
    if rule == 'recut':
        assert np.array_equal(it['labels2nd'], lab2) and it['n_speakers'] >= 7
    else:
        assert it['labels2nd'] is None and it['iterations'] == 0


# ---- a synthetic archive with known speaker counts ---------------------------------------------------------------------

def _synthetic(es, seed=1):
    """6 recordings of 300 .. 700 x-vectors with 2 .. 6 speakers (sticky turns around ES2005a x-vectors), and the
    reference RTTM rows of their true speakers."""
    x_es = es['z']['x_raw']
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    recs, rows, counts = {}, [], {}
    for r in range(6):
        T = int(rng.integers(300, 701))
        K = 2 + r % 5
        centers = x_es[rng.choice(len(x_es), K, replace=False)]
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(K)
        x = centers[spk] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        name = f'syn{r:02d}'
        recs[name] = (x, seg)
        rows += [(name, round(t * 0.24, 2), 0.24, f'spk{k}') for t, k in enumerate(spk)]
        counts[name] = len(np.unique(spk))
    return recs, rows, counts


def _count_calls(monkeypatch):
    """Record every _vb_tier call: (number of entries, largest state count, float64, first pass)."""
    calls = []
    real = pipeline._vb_tier

    def spy(lens, ns, *a, hi=None, **kw):
        calls.append((len(lens), int(np.max(ns)), bool(a[3]), hi is not None))
        return real(lens, ns, *a, hi=hi, **kw)
    monkeypatch.setattr(pipeline, '_vb_tier', spy)
    return calls


def _check_rules(item, lo, hi):
    assert item['count'] == (lo, None if hi >= pipeline.UNBOUNDED else hi)
    n = item['n_speakers']
    if item['count_rule'] in ('vb', 'recut'):
        assert lo <= n <= hi, item['count_rule']
    if item['count_rule'] == 'vb':
        assert lo <= item['n_speakers_vb'] <= hi
    if item['count_rule'] == 'mass':
        assert item['n_speakers_vb'] > hi and n <= hi
    if item['count_rule'] == 'ahc':
        assert item['labels2nd'] is None and n <= lo


@pytest.mark.gpu
def test_synthetic_archive_known_counts(es, monkeypatch):
    recs, _, counts = _synthetic(es)
    args = (recs, es['transform'], es['plda'])
    base = pipeline.diarize_batch(*args, **es['kw'])
    assert all('count_rule' not in it for it in base.values())
    calls = _count_calls(monkeypatch)
    got = pipeline.diarize_batch(*args, **es['kw'], num_speakers=counts)
    for n, it in got.items():
        _check_rules(it, counts[n], counts[n])
        if it['count_rule'] == 'vb':
            assert it['rttm'] == base[n]['rttm']
        print(n, counts[n], it['n_speakers_vb'], it['count_rule'], it['n_speakers'])
    # every recording too few: one re-run batch per state tier, and every recording takes rule 3
    calls.clear()
    got = pipeline.diarize_batch(*args, **es['kw'], min_speakers=20)
    reruns = [c for c in calls if not c[3]]
    assert len(reruns) == 1 and reruns[0][0] == len(recs) and reruns[0][1] <= 20
    assert all(it['count_rule'] in ('recut', 'ahc') for it in got.values())
    # every recording too many
    got = pipeline.diarize_batch(*args, **es['kw'], max_speakers=1)
    assert all(it['count_rule'] == 'mass' and it['n_speakers'] == 1 for it in got.values())


@pytest.mark.gpu
def test_sweep_with_the_oracle_count(es, monkeypatch):
    recs, rows, counts = _synthetic(es)
    grid = dict(Fa=[0.3], Fb=[17.0], loopP=[0.5, 0.99], threshold=[-0.015, 0.3], smoothing=[5.0])
    args = (recs, es['transform'], es['plda'], grid)
    plain = sweep.sweep_batch(*args, ref_rttm=rows)
    calls = _count_calls(monkeypatch)
    out = sweep.sweep_batch(*args, ref_rttm=rows, num_speakers='oracle')
    for s, per in out.items():
        for n, it in per.items():
            _check_rules(it, counts[n], counts[n])
            if it['count_rule'] == 'vb':
                assert it['rttm'] == plain[s][n]['rttm'] and it['der'] == plain[s][n]['der']
            assert 'count_rule' not in plain[s][n]
    reruns = [c for c in calls if not c[3]]
    assert len(reruns) <= 1
    calls.clear()
    out = sweep.sweep_batch(*args, min_speakers=20)
    reruns = [c for c in calls if not c[3]]
    assert len(reruns) == 1 and reruns[0][0] == len(recs) * len(sweep.grid_settings(grid))
    assert all(it['count_rule'] in ('recut', 'ahc') for per in out.values() for it in per.values())


# ---- the command line ------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_command_line_with_a_count(es, tmp_path):
    from vbx_b200 import cli, formats
    z = es['z']
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    keys, seg_lines = [], []
    for i, (s, e) in enumerate(z['seg_times']):
        k = f'ES2005a_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
        keys.append(k)
        seg_lines.append(f'{k} ES2005a {float(s)!r} {float(e)!r}')
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, z['x_raw'])
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), m['plda_mu'], m['plda_tr'], m['plda_psi'])
    np.savez(str(tmp_path / 'transform.npz'), mean1=m['mean1'], mean2=m['mean2'], lda=m['lda'])
    span = float(z['seg_times'][-1, 1])
    ovl = [(0.1 * span, 0.2 * span), (0.5 * span, 0.7 * span)]
    (tmp_path / 'ovl.rttm').write_text(''.join(f'SPEAKER ES2005a 1 {a:.2f} {b - a:.2f} <NA> <NA> ovl <NA> <NA>\n'
                                               for a, b in ovl))
    (tmp_path / 'counts').write_text('ES2005a 7\n')
    base = ['--init', 'AHC+VB', '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']), '--loopP',
            str(z['loopProb']), '--init-smoothing', str(z['smoothing'])]
    from vbx_b200.score import overlap_ticks, read_overlaps
    overlaps = read_overlaps(str(tmp_path / 'ovl.rttm'))
    for i, (opts, c) in enumerate(((['--num-speakers', '4'], dict(num_speakers=4)),
                                   (['--min-speakers', str(tmp_path / 'counts')], dict(min_speakers={'ES2005a': 7})))):
        for with_ovl in (False, True):
            out = tmp_path / f'out{i}{int(with_ovl)}'
            extra = ['--overlap-rttm', str(tmp_path / 'ovl.rttm')] if with_ovl else []
            assert cli.main(base + ['--out-rttm-dir', str(out)] + opts + extra) == 0
            it = _diarize(es, **c, overlaps=overlaps if with_ovl else None)
            lines = (out / 'ES2005a.rttm').read_text().splitlines()
            assert lines == it['rttm_overlap' if with_ovl else 'rttm'], (opts, with_ovl)
            if with_ovl:
                want = pipeline.rttm_lines('ES2005a', *pipeline.overlap_segments(
                    z['seg_times'], it['labels'], it['labels2nd'], overlap_ticks(overlaps['ES2005a'])))
                assert lines == want
                if it['labels2nd'] is not None:
                    assert len(lines) > len(it['rttm'])
