"""Back-end training on the GPU (DESIGN.md section 5.24): vbx_class_scatter against float64 numpy on the same float32
rows at every tile and split edge, its determinism and refusals; train_backend against the float64 oracle; and a model
trained from a synthetic archive diarizing unseen speakers through the command line."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import train_oracle as O
from vbx_b200 import _lib, cli, formats, score, synth, train

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')


def reference(X, off):
    """float64 means and scatter of the float32 rows, and the scale of each class mean (mean |x|)."""
    m, S = O.class_stats(X, off)
    a, _ = O.class_stats(np.abs(X), off)
    return m, S, a


def check(X, off, means, S):
    m_ref, S_ref, scale = reference(X, off)
    means, S = means.cpu().numpy(), S.cpu().numpy()
    assert np.all(np.abs(means - m_ref) <= 1e-13 * scale + 1e-300)
    dg = np.sqrt(np.maximum(np.diag(S_ref), 0))
    assert np.all(np.abs(S - S_ref) <= 1e-11 * np.outer(dg, dg) + 1e-300)
    assert np.array_equal(S, S.T)


def rows(sizes, D, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    K = len(sizes)
    centre = rng.standard_normal((K, D)) * 2.0
    X = np.repeat(centre, sizes, axis=0) + rng.standard_normal((int(off[-1]), D)) + offset
    return X.astype(np.float32), off


@pytest.mark.gpu
@pytest.mark.parametrize('D', [1, 3, 4, 100, 128, 192, 256, 512, 1024])
def test_scatter_every_width(D):
    rng = np.random.default_rng(D)
    # the first N sits on a 32-row chunk edge, the others one row past and short of a split edge
    per = train_split_rows(5000, D)
    for N in (32, per + 1, 3 * per - 1, 5000):
        sizes = rng.multinomial(N, np.ones(40) / 40)
        sizes[3] = 0
        sizes[7] = 1
        X, off = rows(sizes, D, D * 7 + N)
        check(X, off, *train.class_stats(X, off, DEV))


def train_split_rows(N, D):
    """Rows per split of vbx_train.cu for (N, D): ceil(N / want) rounded up to 32, want = ceil(1024 / tile pairs)."""
    T = (D + 63) // 64
    want = max(1, -(-1024 // (T * (T + 1) // 2)))
    return max(32, -(-(-(-N // want)) // 32) * 32)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['one_class', 'singletons', 'tiny_classes', 'offset', 'empty'])
def test_scatter_class_layouts(case):
    D = 96
    if case == 'one_class':
        X, off = rows([20000], D, 1)
    elif case == 'singletons':
        X, off = rows([1] * 300 + [50], D, 2)
    elif case == 'tiny_classes':
        rng = np.random.default_rng(3)
        X, off = rows(rng.integers(0, 4, 100000), 16, 3)
    elif case == 'offset':                           # S = G - n m m^T would lose every digit here
        X, off = rows(np.full(64, 150), D, 4, offset=1e3)
    else:
        X, off = np.zeros((0, D), dtype=np.float32), np.zeros(4, dtype=np.int64)
    means, S = train.class_stats(X, off, DEV)
    if case == 'empty':
        assert not means.any() and not S.any()
    else:
        check(X, off, means, S)


def raw_call(lib, h, X, off, ws, means, S, nbytes=None):
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    N, D = X.shape
    return lib.vbx_class_scatter(h, p(X), N, D, len(off) - 1, off.ctypes.data_as(ctypes.c_void_p) if off is not None
                                 else None, p(ws), ws.numel() if nbytes is None else nbytes, p(means), p(S),
                                 ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))


@pytest.fixture
def handle():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    yield lib, h
    lib.vbx_destroy(h)


@pytest.mark.gpu
def test_scatter_is_deterministic_and_ignores_the_workspace(handle):
    lib, h = handle
    Xn, off = rows(np.random.default_rng(5).integers(1, 300, 400), 256, 5)
    X = torch.from_numpy(Xn).to(DEV)
    need = ctypes.c_size_t()
    assert lib.vbx_class_scatter_workspace_bytes(h, X.shape[0], 256, len(off) - 1, ctypes.byref(need)) == 0
    outs = []
    for poison in (0.0, float('nan'), 0.0):
        ws = torch.full((need.value // 8 + 1,), poison, dtype=torch.float64, device=DEV)
        means = torch.full((len(off) - 1, 256), float('nan'), dtype=torch.float64, device=DEV)
        S = torch.full((256, 256), float('nan'), dtype=torch.float64, device=DEV)
        assert raw_call(lib, h, X, off, ws, means, S, need.value) == 0, lib.vbx_last_error(h)
        torch.cuda.synchronize()
        outs.append((means.cpu().numpy(), S.cpu().numpy()))
    for m, S in outs[1:]:
        assert np.array_equal(m.view(np.int64), outs[0][0].view(np.int64))
        assert np.array_equal(S.view(np.int64), outs[0][1].view(np.int64))
    check(Xn, off, torch.from_numpy(outs[0][0]), torch.from_numpy(outs[0][1]))


@pytest.mark.gpu
def test_scatter_refusals(handle):
    lib, h = handle
    X = torch.zeros((100, 8), dtype=torch.float32, device=DEV)
    off = np.array([0, 40, 100], dtype=np.int64)
    need = ctypes.c_size_t()
    assert lib.vbx_class_scatter_workspace_bytes(h, 100, 8, 2, ctypes.byref(need)) == 0
    ws = torch.zeros(need.value + 256, dtype=torch.uint8, device=DEV)
    means = torch.zeros((2, 8), dtype=torch.float64, device=DEV)
    S = torch.zeros((8, 8), dtype=torch.float64, device=DEV)
    assert raw_call(lib, h, X, off, ws, means, S) == 0
    err = -1                                                            # VBX_ERR_ARG
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    o = off.ctypes.data_as(ctypes.c_void_p)
    call = lambda X_, N, D, K, o_, ws_, nb, m_, S_: lib.vbx_class_scatter(h, X_, N, D, K, o_, ws_, nb, m_, S_, st)
    base = (vp(X), 100, 8, 2, o, vp(ws), ws.numel(), vp(means), vp(S))
    for i in (0, 4, 5, 7, 8):                                           # null pointers (X only matters with N > 0)
        a = list(base)
        a[i] = None
        assert call(*a) == err
    for i, v in ((2, 0), (2, 1025), (3, 0), (1, -1)):                   # D, K, N out of range
        a = list(base)
        a[i] = v
        assert call(*a) == err
    for bad in ([0, 40, 99], [1, 40, 100], [0, 60, 50]):                # offsets not 0 .. N or decreasing
        b = np.array(bad, dtype=np.int64)
        a = list(base)
        a[4] = b.ctypes.data_as(ctypes.c_void_p)
        assert call(*a) == err
    a = list(base)
    a[0] = ctypes.c_void_p(X.data_ptr() + 4)                            # X off the 16-byte grid
    assert call(*a) == err
    a = list(base)
    a[5] = ctypes.c_void_p(ws.data_ptr() + 8)                           # misaligned workspace
    assert call(*a) == err
    a = list(base)
    a[6] = need.value - 1                                               # short workspace
    assert call(*a) == err
    assert lib.vbx_class_scatter_workspace_bytes(h, 100, 0, 2, ctypes.byref(need)) == err


def speaker_set(K, Dx, seed, nmin=4, nmax=30):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((Dx, Dx)))
    within = q * np.exp(np.linspace(0, -2, Dx))[None, :]
    centres = 3.0 + rng.standard_normal((K, Dx)) * np.exp(np.linspace(0.5, -1.5, Dx))[None, :]
    return {f'spk{k}': centres[k] + rng.standard_normal((int(rng.integers(nmin, nmax + 1)), Dx)) @ within.T
            for k in range(K)}


def rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b))


@pytest.mark.gpu
@pytest.mark.parametrize('Dx, K, d', [(64, 150, 24), (256, 400, 128)])
def test_train_backend_matches_the_oracle(Dx, K, d):
    sets = speaker_set(K, Dx, Dx + K)
    sets['solo'] = np.ones((1, Dx))                                     # dropped: below min_per_speaker
    (mean1, mean2, lda), (mu, tr, psi), rep = train.train_backend(sets, lda_dim=d, em_iters=10, device=DEV)
    ref = O.train(sets, lda_dim=d, em_iters=10)
    assert rep['K'] == ref['K'] == K and rep['N'] == ref['N'] and rep['speakers_dropped'] == 1
    assert rep['xvectors_dropped'] == 1 and rep['Dx'] == Dx and rep['lda_dim'] == d
    W = np.linalg.inv(tr.T @ tr)
    B = np.linalg.inv((tr.T / psi) @ tr)
    for got, want in ((W, ref['W']), (B, ref['B']), (lda, ref['lda']), (mean1, ref['mean1']), (mean2, ref['mean2']),
                      (psi, ref['psi']), (mu, ref['mu']), (rep['lda_eigenvalues'], ref['lam'])):
        assert rel(got, want) <= 1e-8, rel(got, want)
    assert np.allclose(rep['objective'], ref['trace'], rtol=1e-9, atol=0)
    assert np.all(np.diff(rep['objective']) >= -1e-12 * np.abs(rep['objective'][1:]))


def write_archive(root, recs, rows):
    """ark + segments + one reference RTTM for a synth.multi_session_archive archive; returns the three paths."""
    ark, seg, ref = (os.path.join(root, f) for f in ('x.ark', 'x.seg', 'ref.rttm'))
    keys, vecs = [], []
    with open(seg, 'w') as f:
        for name, (x, times) in recs.items():
            for t, (s, e) in enumerate(times):
                keys.append(f'{name}_{t:05d}')
                vecs.append(x[t])
                f.write(f'{name}_{t:05d} {name} {s:.2f} {e:.2f}\n')
    formats.write_vec_flt_ark(ark, keys, vecs)
    with open(ref, 'w') as f:
        for name, on, dur, spk in rows:
            f.write(f'SPEAKER {name} 1 {on:.2f} {dur:.2f} <NA> <NA> {spk} <NA> <NA>\n')
    return ark, seg, ref


@pytest.mark.gpu
def test_trained_model_diarizes_unseen_speakers(tmp_path):
    x_es = np.load(os.path.join(GOLD, 'es2005a.npz'))['x_raw']
    model = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    recs, rows, truth = synth.multi_session_archive(x_es, n_rec=150, pool=300, seed=21)
    ark, seg, ref = write_archive(str(tmp_path), recs, rows)
    utt2spk = os.path.join(str(tmp_path), 'utt2spk')
    with open(utt2spk, 'w') as f:
        for name, who in truth.items():
            f.write(''.join(f'{name}_{t:05d} p{k}\n' for t, k in enumerate(who)))
    out_rttm, out_utt = (os.path.join(str(tmp_path), d) for d in ('m_rttm', 'm_utt'))
    assert train.main(['--xvec-ark-file', ark, '--segments-file', seg, '--ref-rttm', ref, '--out-dir', out_rttm,
                       '--speakers-across-recordings']) == 0
    assert train.main(['--xvec-ark-file', ark, '--utt2spk', utt2spk, '--out-dir', out_utt, '--text-plda']) == 0
    held, held_rows, _ = synth.multi_session_archive(x_es, n_rec=12, pool=40, seed=977)
    hdir = tmp_path / 'held'
    hdir.mkdir()
    h_ark, h_seg, h_ref = write_archive(str(hdir), held, held_rows)
    shipped = tmp_path / 'shipped'
    shipped.mkdir()
    np.savez(shipped / 'transform.npz', mean1=model['mean1'], mean2=model['mean2'], lda=model['lda'])
    formats.write_kaldi_plda_binary(str(shipped / 'plda'), model['plda_mu'], model['plda_tr'], model['plda_psi'])
    ders = {}
    for tag, mdir in (('rttm', out_rttm), ('utt2spk', out_utt), ('shipped', str(shipped))):
        sys_dir = os.path.join(str(tmp_path), f'sys_{tag}')
        assert cli.main(['--init', 'AHC+VB', '--out-rttm-dir', sys_dir, '--xvec-ark-file', h_ark, '--segments-file', h_seg,
                         '--xvec-transform', os.path.join(mdir, 'transform.npz'), '--plda-file',
                         os.path.join(mdir, 'plda'), '--threshold', '-0.015', '--lda-dim', '128',
                         '--Fa', str(float(z['Fa'])), '--Fb', str(float(z['Fb'])),
                         '--loopP', str(float(z['loopProb']))]) == 0
        _, tot = score.score_rttm(score.read_rttm_path(h_ref), score.read_rttm_path(sys_dir), 0.25, False, device=DEV)
        ders[tag] = tot['der']
    print('held-out DER', ders)
    assert ders['rttm'] <= ders['shipped'] and ders['utt2spk'] <= ders['shipped'], ders
