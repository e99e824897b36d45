"""PLDA adaptation on the GPU (DESIGN.md section 5.26): the archive statistics against numpy float64 on the same float32
rows, adapt_backend against the float64 oracle, the command line's --adapt against the files train --adapt-plda writes,
the sweep against the command line, train --xvec-transform against train, and enrolment through the adapted model."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import adapt_oracle as O
from vbx_b200 import adapt, cli, formats, pipeline, sweep, synth, train

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')
ES = np.load(os.path.join(GOLD, 'es2005a.npz'))
MODEL = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
TRANSFORM = (MODEL['mean1'], MODEL['mean2'], MODEL['lda'])
PLDA = (MODEL['plda_mu'], MODEL['plda_tr'], MODEL['plda_psi'])
HYPER = ['--Fa', str(float(ES['Fa'])), '--Fb', str(float(ES['Fb'])), '--loopP', str(float(ES['loopProb']))]


def shifted_archive(n_rec=6, seed=31):
    """A multi-session archive around ES2005a's x-vectors moved by a seeded offset, so that the archive differs from the
    shipped model's domain."""
    recs, rows, truth = synth.multi_session_archive(ES['x_raw'], n_rec=n_rec, pool=12, seed=seed)
    rng = np.random.default_rng(seed)
    off = 0.5 * ES['x_raw'].std(0) * rng.standard_normal(ES['x_raw'].shape[1])
    return {n: (x + off[None, :], seg) for n, (x, seg) in recs.items()}, rows, truth


def write_archive(root, recs):
    ark, seg = os.path.join(root, 'x.ark'), os.path.join(root, 'x.seg')
    keys, vecs = [], []
    with open(seg, 'w') as f:
        for name, (x, times) in recs.items():
            for t, (s, e) in enumerate(times):
                keys.append(f'{name}_{t:05d}')
                vecs.append(x[t])
                f.write(f'{name}_{t:05d} {name} {s:.2f} {e:.2f}\n')
    formats.write_vec_flt_ark(ark, keys, vecs)
    return ark, seg


def write_model(root, transform, plda):
    os.makedirs(root, exist_ok=True)
    np.savez(os.path.join(root, 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    formats.write_kaldi_plda_binary(os.path.join(root, 'plda'), *plda)
    return os.path.join(root, 'transform.npz'), os.path.join(root, 'plda')


def read_dir(d):
    return {f: open(os.path.join(d, f), 'rb').read() for f in sorted(os.listdir(d)) if f.endswith('.rttm')}


def ark_recordings(ark):
    """The archive as the command line reads it (float32 x-vectors from the ark)."""
    return {n: (x, None) for n, (_, x) in formats.read_xvectors_by_recording(ark).items()}


@pytest.mark.gpu
@pytest.mark.parametrize('chain', ['tcgen05', 'float64'])
def test_archive_stats_match_numpy(chain):
    rng = np.random.default_rng(5)
    lens = [1, 700, 33, 1500, 2, 257]                   # ragged, with recordings of one and two x-vectors
    x = 2.0 + rng.standard_normal((sum(lens), 256)) * ES['x_raw'].std(0)[None, :]
    z = adapt.project_archive(x, lens, TRANSFORM, PLDA, 128, chain, DEV)
    assert z.dtype == torch.float32 and tuple(z.shape) == (sum(lens), 128)
    m, C = adapt.archive_stats(z, DEV)
    m_ref, C_ref = O.stats(z.cpu().numpy())
    scale = np.abs(np.diag(C_ref)).max()
    assert np.abs(m.cpu().numpy() - m_ref).max() <= 1e-12 * np.abs(m_ref).max()
    assert np.abs(C.cpu().numpy() - C_ref).max() <= 1e-12 * scale


@pytest.mark.gpu
@pytest.mark.parametrize('recentre', [False, True])
def test_adapt_backend_matches_the_oracle(recentre):
    recs, _, _ = shifted_archive()
    transform, plda, rep = adapt.adapt_backend(recs, TRANSFORM, PLDA, device=DEV, recentre=recentre)
    x = np.concatenate([r[0] for r in recs.values()])
    lens = [len(r[0]) for r in recs.values()]
    if recentre:
        m1 = x.mean(0)
        y = (x - m1) / np.linalg.norm(x - m1, axis=1, keepdims=True)
        assert np.abs(transform[0] - m1).max() <= 1e-12 * np.abs(m1).max()
        assert np.abs(transform[1] - y.mean(0) @ TRANSFORM[2]).max() <= 1e-12
        assert np.array_equal(transform[2], TRANSFORM[2])
    else:
        assert all(np.array_equal(a, b) for a, b in zip(transform, TRANSFORM))
    z = adapt.project_archive(x, lens, transform, PLDA, 128, 'auto', DEV).cpu().numpy()
    m, C = O.stats(z)
    mu2, W2, B2, lam = O.adapt(PLDA[0], *O.covariances(PLDA[1], PLDA[2]), m, C)
    got = adapt.plda_covariances(plda)
    assert np.abs(got[0] - mu2).max() <= 1e-12
    for g, w in zip(got[1:], (W2, B2)):
        assert np.abs(g - w).max() <= 1e-9 * np.abs(w).max()
    assert rep['N'] == len(x) and rep['inflated'] == int((lam > 1).sum()) > 0 and rep['chain'] == 'tcgen05'
    assert np.allclose(rep['eigenvalues'], lam[::-1], rtol=1e-9, atol=1e-12)


def es2005a_archive():
    return {'ES2005a': (ES['x_raw'], ES['seg_times'])}


@pytest.mark.gpu
@pytest.mark.parametrize('recentre', [False, True])
@pytest.mark.parametrize('which', ['es2005a', 'synthetic'])
def test_cli_adapt_equals_the_written_model(tmp_path, which, recentre):
    recs = es2005a_archive() if which == 'es2005a' else shifted_archive()[0]
    ark, seg = write_archive(str(tmp_path), recs)
    t_path, p_path = write_model(str(tmp_path / 'shipped'), TRANSFORM, PLDA)
    extra = ['--recentre'] if recentre else []
    base = ['--init', 'AHC+VB', '--xvec-ark-file', ark, '--segments-file', seg, '--threshold', '-0.015',
            '--lda-dim', '128'] + HYPER
    assert cli.main(base + ['--out-rttm-dir', str(tmp_path / 'a'), '--xvec-transform', t_path, '--plda-file', p_path,
                            '--adapt'] + extra) == 0
    mdir = str(tmp_path / 'adapted')
    assert train.main(['--xvec-ark-file', ark, '--adapt-plda', p_path, '--xvec-transform', t_path, '--out-dir', mdir]
                      + extra) == 0
    rep = json.load(open(os.path.join(mdir, 'train.json')))
    assert rep['N'] == sum(len(r[0]) for r in recs.values()) and rep['recentre'] == recentre
    assert cli.main(base + ['--out-rttm-dir', str(tmp_path / 'b'), '--xvec-transform', os.path.join(mdir, 'transform.npz'),
                            '--plda-file', os.path.join(mdir, 'plda')]) == 0
    assert cli.main(base + ['--out-rttm-dir', str(tmp_path / 'c'), '--xvec-transform', t_path,
                            '--plda-file', p_path]) == 0
    a, b, c = (read_dir(str(tmp_path / d)) for d in 'abc')
    assert len(a) == len(recs) and a == b
    if which == 'synthetic':
        assert a != c                              # the adapted model does diarize this archive differently


@pytest.mark.gpu
def test_sweep_adapt_equals_cli_adapt(tmp_path):
    recs = shifted_archive(n_rec=4, seed=41)[0]
    ark, seg = write_archive(str(tmp_path), recs)
    t_path, p_path = write_model(str(tmp_path / 'shipped'), TRANSFORM, PLDA)
    model = ['--xvec-ark-file', ark, '--segments-file', seg, '--xvec-transform', t_path, '--plda-file', p_path,
             '--lda-dim', '128', '--adapt', '--recentre', '--adapt-within-scale', '0.5', '--adapt-between-scale', '0.4']
    assert sweep.main(['--out-dir', str(tmp_path / 'sw'), '--Fa', '0.3,0.5', '--Fb', '17', '--loopP', '0.99',
                       '--threshold=-0.015,0.2'] + model) == 0
    summary = json.load(open(tmp_path / 'sw' / 'summary.json'))
    assert len(summary) == 4
    for name, block in summary.items():
        s = block['setting']
        out = str(tmp_path / f'cli_{name}')
        assert cli.main(['--init', 'AHC+VB', '--out-rttm-dir', out, '--threshold', repr(s['threshold']),
                         '--Fa', repr(s['Fa']), '--Fb', repr(s['Fb']), '--loopP', repr(s['loopP'])] + model) == 0
        assert read_dir(out) == read_dir(str(tmp_path / 'sw' / name)), name


@pytest.mark.gpu
def test_train_with_the_fitted_transform_reproduces_the_plda(tmp_path):
    rng = np.random.default_rng(9)
    K, Dx = 300, 64
    centres = 2.0 + rng.standard_normal((K, Dx))
    keys, vecs, utt = [], [], []
    for k in range(K):
        for i in range(int(rng.integers(3, 12))):
            keys.append(f's{k}_{i}')
            vecs.append(centres[k] + 0.5 * rng.standard_normal(Dx))
            utt.append(f's{k}_{i} s{k}\n')
    ark = str(tmp_path / 'x.ark')
    formats.write_vec_flt_ark(ark, keys, vecs)
    with open(tmp_path / 'utt2spk', 'w') as f:
        f.write(''.join(utt))
    base = ['--xvec-ark-file', ark, '--utt2spk', str(tmp_path / 'utt2spk'), '--lda-dim', '24']
    assert train.main(base + ['--out-dir', str(tmp_path / 'a')]) == 0
    assert train.main(base + ['--out-dir', str(tmp_path / 'b'), '--xvec-transform',
                              str(tmp_path / 'a' / 'transform.npz')]) == 0
    pa, pb = (formats.read_kaldi_plda(str(tmp_path / d / 'plda')) for d in 'ab')
    for a, b in zip(pa, pb):
        assert np.abs(a - b).max() <= 1e-12 * np.abs(a).max()
    ta, tb = (formats.read_xvec_transform(str(tmp_path / d / 'transform.npz')) for d in 'ab')
    assert all(np.array_equal(a, b) for a, b in zip(ta, tb))
    rb = json.load(open(tmp_path / 'b' / 'train.json'))
    assert rb['transform'] == 'given' and 'lda_eigenvalues' not in rb
    # interpolation at alpha = 1 keeps the trained PLDA, at alpha = 0 the other
    write_model(str(tmp_path / 'o'), ta, PLDA_d(24))
    for alpha, want in (('1', pa), ('0', PLDA_d(24))):
        out = str(tmp_path / f'i{alpha}')
        assert train.main(base + ['--out-dir', out, '--xvec-transform', str(tmp_path / 'a' / 'transform.npz'),
                                  '--interpolate-with', str(tmp_path / 'o' / 'plda'), '--alpha', alpha]) == 0
        got = formats.read_kaldi_plda(os.path.join(out, 'plda'))
        for g, w in zip(got, want):
            assert np.abs(g - w).max() <= 1e-10 * np.abs(w).max()


def PLDA_d(d, seed=3):
    """A PLDA of dimension d in the form train_backend writes."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    W = (q * np.linspace(0.5, 1.5, d)[None, :]) @ q.T
    return adapt.plda_from_covariances(0.1 * rng.standard_normal(d), W, np.diag(np.linspace(3.0, 0.2, d)))


@pytest.mark.gpu
def test_enrolment_through_the_adapted_model(tmp_path):
    recs, _, truth = shifted_archive(n_rec=4, seed=51)
    ark, seg = write_archive(str(tmp_path), recs)
    t_path, p_path = write_model(str(tmp_path / 'shipped'), TRANSFORM, PLDA)
    # enrolment: 20 x-vectors of three pool speakers taken from the archive itself
    keys, vecs, utt = [], [], []
    for name, (x, _) in recs.items():
        for k in np.unique(truth[name])[:1]:
            for t in np.nonzero(truth[name] == k)[0][:20]:
                keys.append(f'e_{name}_{t}')
                vecs.append(x[t])
                utt.append(f'e_{name}_{t} p{k}\n')
    e_ark, e_utt = str(tmp_path / 'e.ark'), str(tmp_path / 'e.utt2spk')
    formats.write_vec_flt_ark(e_ark, keys, vecs)
    with open(e_utt, 'w') as f:
        f.write(''.join(utt))
    base = ['--init', 'AHC+VB', '--xvec-ark-file', ark, '--segments-file', seg, '--threshold', '-0.015',
            '--lda-dim', '128', '--enroll-ark', e_ark, '--enroll-utt2spk', e_utt, '--enroll-threshold', '0'] + HYPER
    assert cli.main(base + ['--out-rttm-dir', str(tmp_path / 'a'), '--xvec-transform', t_path, '--plda-file', p_path,
                            '--adapt']) == 0
    mdir = str(tmp_path / 'adapted')
    assert train.main(['--xvec-ark-file', ark, '--adapt-plda', p_path, '--xvec-transform', t_path,
                       '--out-dir', mdir]) == 0
    assert cli.main(base + ['--out-rttm-dir', str(tmp_path / 'b'), '--xvec-transform', os.path.join(mdir, 'transform.npz'),
                            '--plda-file', os.path.join(mdir, 'plda')]) == 0
    a, b = read_dir(str(tmp_path / 'a')), read_dir(str(tmp_path / 'b'))
    assert len(a) == len(recs) and a == b
    assert any(b'SPEAKER' in v and b' p' in v for v in a.values())     # some speakers took enrolled names
