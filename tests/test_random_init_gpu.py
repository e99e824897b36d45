"""Random starts of the VB-HMM on the device (init='RANDOM+VB', DESIGN.md section 5.22): vbx_init_random against the
float64 oracle of oracle/random_init_oracle.py, rows independent of the batch, every restart's VB-HMM against the float64
oracle VB-HMM from the oracle's gamma0, no AHC without count bounds, sweep_batch against diarize_batch, rule 2 on the
chosen restart, and the command line on ES2005a."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import random_init_oracle as ro
from oracle.vbx_oracle import vbx_oracle
from vbx_b200 import VbxError, ahc, pipeline, random_init, sweep, synth
from vbx_b200.batch import VbxBatch

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
M64 = (1 << 64) - 1


@pytest.fixture(scope='module')
def model():
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    return dict(z=z, transform=(m['mean1'], m['mean2'], m['lda']), plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']))


# ---- the kernel -----------------------------------------------------------------------------------------------------------

def draw(lens, ns, keys, seeds, f64, S=None):
    """gamma0, pi0 of vbx_init_random on a plan of lens / ns, written into NaN-filled tensors (host arrays)."""
    dev = torch.device('cuda:0')
    vb = VbxBatch(lens, 128, ns, device=dev, allocate=False, f64_only=f64, S_pad=S)
    dt = torch.float64 if f64 else torch.float32
    g = torch.full((vb.N, vb.S), float('nan'), dtype=dt, device=dev)
    p = torch.full((vb.B, vb.S), float('nan'), dtype=dt, device=dev)
    vb.init_random(keys, seeds, g, p)
    out = g.cpu().numpy(), p.cpu().numpy(), vb.S
    vb.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('f64', [False, True])
def test_init_random_equals_the_oracle(f64):
    """Ragged batch with an empty recording and N = 1, 4, 64, 65, 128 (and 129 on the float64 plan): float32 within 1 ulp
    of the float64 oracle, float64 within 1e-14 relative, pi0 = 1/N exactly, no NaN left."""
    lens = [400, 0, 300, 250, 200, 150, 1, 37] + ([180] if f64 else [])
    ns = [4, 3, 1, 64, 65, 128, 7, 10] + ([129] if f64 else [])
    keys = [ro.name_key(f'rec{b}') for b in range(len(lens))]
    seeds = [0, 1, M64, 2 ** 63, 12345, 7, M64 - 1, 99, 3][:len(lens)]
    g, p, S = draw(lens, ns, keys, seeds, f64)
    assert not np.isnan(g).any() and not np.isnan(p).any()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        want, pi = ro.init_gamma(lens[b], ns[b], keys[b], seeds[b], S=S)
        got = g[offs[b]:offs[b + 1]]
        if f64:
            np.testing.assert_allclose(got, want, rtol=1e-14, atol=0, err_msg=str(b))
        else:
            assert np.all(np.abs(got.astype(np.float64) - want) <= np.spacing(want.astype(np.float32))), b
        assert np.all(got[:, ns[b]:] == 0), b
        assert np.array_equal(p[b], pi.astype(p.dtype)), b


@pytest.mark.gpu
def test_rows_do_not_depend_on_the_batch():
    """A recording's gamma0 is bit-identical alone, inside a larger batch of another S, and at another position."""
    key, seed, T, N = ro.name_key('meeting'), 41, 333, 10
    alone, _, _ = draw([T], [N], [key], [seed], False)
    others = dict(lens=[120, 80, 50], ns=[64, 3, 17], keys=[5, 6, 7], seeds=[1, 2, 3])
    for pos in (0, 2, 3):
        lens = others['lens'][:pos] + [T] + others['lens'][pos:]
        ns = others['ns'][:pos] + [N] + others['ns'][pos:]
        keys = others['keys'][:pos] + [key] + others['keys'][pos:]
        seeds = others['seeds'][:pos] + [seed] + others['seeds'][pos:]
        for S in (None, 128):
            g, _, _ = draw(lens, ns, keys, seeds, False, S=S)
            o = int(np.sum(lens[:pos]))
            assert np.array_equal(g[o:o + T, :N], alone[:, :N]), (pos, S)
    a64, _, _ = draw([T], [N], [key], [seed], True)
    b64, _, _ = draw([50, T], [140, N], [1, key], [1, seed], True)
    assert np.array_equal(a64, b64[50:, :N])


@pytest.mark.gpu
def test_init_random_argument_errors():
    dev = torch.device('cuda:0')
    vb = VbxBatch([20, 5], 128, [3, 4], device=dev, allocate=False)
    g = torch.zeros((vb.N, vb.S), device=dev)
    p = torch.zeros((2, vb.S), device=dev)
    with pytest.raises(ValueError, match='rec_keys'):
        vb.init_random([1], [0, 0], g, p)
    with pytest.raises(ValueError, match='seeds'):
        vb.init_random([1, 2], [0, 1 << 64], g, p)
    with pytest.raises(ValueError):
        vb.init_random([1, 2], [0, 0], g.double(), p)
    vb.close()
    from vbx_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    assert lib.vbx_init_random(h, None, None, None, None, None, 0, None) == -3     # VBX_ERR_STATE: no plan
    offs = np.array([0, 4], dtype=np.int64)
    assert lib.vbx_plan_f64(h, offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 1, 8, 4) == 0
    assert lib.vbx_init_random(h, None, None, None, None, None, 0, None) == -1     # VBX_ERR_ARG: null arrays
    lib.vbx_destroy(h)
    assert lib.vbx_init_random(None, None, None, None, None, None, 0, None) == -1


# ---- the VB-HMM from random starts ------------------------------------------------------------------------------------

KW = dict(Fa=0.3, Fb=17.0, loopP=0.99, smoothing=5.0, threshold=-0.015, max_iters=40, epsilon=1e-6)


@pytest.mark.gpu
def test_every_restart_follows_the_float64_oracle(model):
    """diarize_batch(init='RANDOM+VB', restarts=4): every restart's final ELBO is the float64 oracle VB-HMM's from the
    oracle's gamma0 within the parity bar (1e-4 relative), and the chosen restart's oracle ELBO is the oracle's best
    within that bar."""
    recs, _, _ = synth.multi_session_archive(model['z']['x_raw'], n_rec=3, lengths=(150, 250), seed=5)
    N, R, seed = 6, 4, 2024
    out = pipeline.diarize_batch(recs, model['transform'], model['plda'], init='RANDOM+VB', init_states=N, restarts=R,
                                 seed=seed, **KW)
    names = list(recs)
    lens = np.array([len(recs[n][0]) for n in names])
    dev = torch.device('cuda:0')
    fea, Phi, *_ = pipeline._front_end(recs, names, lens, model['transform'], model['plda'], 128, 'auto', dev, 0.0,
                                       ahc=False)
    fea, Phi = fea.double().cpu().numpy(), Phi.double().cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for b, n in enumerate(names):
        item = out[n]
        assert len(item['restart_elbos']) == R and item['elbo'] == item['restart_elbos'][item['restart']]
        assert item['init_seed'] == seed + item['restart']
        oracle_final = []
        for r in range(R):
            g0, _ = ro.init_gamma(int(lens[b]), N, ro.name_key(n), ro.restart_seed(seed, r))
            _, _, Li = vbx_oracle(fea[offs[b]:offs[b + 1]], Phi, loopProb=KW['loopP'], Fa=KW['Fa'], Fb=KW['Fb'], pi=N,
                                  gamma=g0, maxIters=KW['max_iters'], epsilon=KW['epsilon'])
            oracle_final.append(Li[-1][0])
            assert abs(item['restart_elbos'][r] - Li[-1][0]) <= 1e-4 * abs(Li[-1][0]), (n, r)
        best = max(oracle_final)
        assert oracle_final[item['restart']] >= best - 1e-4 * abs(best), n


@pytest.mark.gpu
def test_no_ahc_without_lower_count_bounds(model, monkeypatch):
    recs, _, _ = synth.multi_session_archive(model['z']['x_raw'], n_rec=2, seed=7)

    def refuse(*a, **k):
        raise AssertionError('ahc_batch ran')
    monkeypatch.setattr(ahc, 'ahc_batch', refuse)
    out = pipeline.diarize_batch(recs, model['transform'], model['plda'], init='RANDOM+VB', init_states=8, restarts=2,
                                 **KW)
    assert all(item['n_speakers'] >= 1 for item in out.values())
    grid = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99, 0.5], threshold=[-0.015], smoothing=[5.0])
    sweep.sweep_batch(recs, model['transform'], model['plda'], grid, init='RANDOM+VB', init_states=8)
    with pytest.raises(AssertionError, match='ahc_batch ran'):
        pipeline.diarize_batch(recs, model['transform'], model['plda'], init='RANDOM+VB', init_states=8,
                               min_speakers=2, **KW)


@pytest.mark.gpu
def test_sweep_entries_equal_diarize_batch(model):
    """Every setting's entries equal diarize_batch(init='RANDOM+VB') with that setting's scalars: labels, iterations, the
    chosen restart and its ELBOs."""
    recs, _, _ = synth.multi_session_archive(model['z']['x_raw'], n_rec=4, seed=9)
    grid = dict(Fa=[0.3, 0.5], Fb=[17.0], loopP=[0.99, 0.6], threshold=[-0.015], smoothing=[5.0])
    opts = dict(init='RANDOM+VB', init_states=9, restarts=3, seed=77)
    out = sweep.sweep_batch(recs, model['transform'], model['plda'], grid, **opts)
    for s, per_rec in out.items():
        want = pipeline.diarize_batch(recs, model['transform'], model['plda'], Fa=s.Fa, Fb=s.Fb, loopP=s.loopP,
                                      smoothing=s.smoothing, threshold=s.threshold, **opts)
        for n in recs:
            a, b = per_rec[n], want[n]
            assert np.array_equal(a['labels'], b['labels']) and a['iterations'] == b['iterations'], (s, n)
            assert a['rttm'] == b['rttm'] and a['restart'] == b['restart'] and a['init_seed'] == b['init_seed'], (s, n)
            np.testing.assert_allclose(a['restart_elbos'], b['restart_elbos'], rtol=1e-9)


@pytest.mark.gpu
def test_max_speakers_applies_rule_2_to_the_chosen_restart(model):
    recs, _, _ = synth.multi_session_archive(model['z']['x_raw'], n_rec=4, seed=11)
    opts = dict(init='RANDOM+VB', init_states=10, restarts=3, seed=5)
    free = pipeline.diarize_batch(recs, model['transform'], model['plda'], **opts, **KW)
    bound = pipeline.diarize_batch(recs, model['transform'], model['plda'], max_speakers=2, **opts, **KW)
    for n in recs:
        a, b = free[n], bound[n]
        assert b['restart'] == a['restart'] and b['restart_elbos'] == a['restart_elbos'], n
        assert b['n_speakers_vb'] == a['n_speakers'] and b['n_speakers'] <= 2, n
        assert b['count_rule'] == ('mass' if a['n_speakers'] > 2 else 'vb'), n
        if b['count_rule'] == 'vb':
            assert np.array_equal(a['labels'], b['labels']), n
        else:
            assert set(np.unique(b['labels'])) <= set(np.unique(a['labels'])), n


# ---- the command line on ES2005a ----------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_command_line_on_es2005a(model, tmp_path):
    from vbx_b200 import cli, formats
    z = model['z']
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
    out = tmp_path / 'out'
    argv = ['--init', 'RANDOM+VB', '--init-states', '10', '--restarts', '8', '--out-rttm-dir', str(out),
            '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']),
            '--loopP', str(z['loopProb']), '--init-smoothing', str(z['smoothing'])]
    assert cli.main(argv) == 0
    lines = (out / 'ES2005a.rttm').read_text().splitlines()
    it = pipeline.diarize_batch({'ES2005a': (z['x_raw'], z['seg_times'])}, model['transform'], model['plda'],
                                Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']),
                                smoothing=float(z['smoothing']), init='RANDOM+VB', init_states=10, restarts=8)
    assert lines and lines == it['ES2005a']['rttm']
    assert len(it['ES2005a']['restart_elbos']) == 8 and np.isfinite(it['ES2005a']['elbo'])
