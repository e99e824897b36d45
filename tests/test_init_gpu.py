"""VB resegmentation on the device (DESIGN.md section 5.20): vbx_init_turns against the float64 numpy oracle of
oracle/init_oracle.py, the tie to the AHC-initialised path (an RTTM of the archive's own AHC labels on back-to-back
segments gives soft_init's gamma0 and init='AHC+VB''s labels and iterations), sweep_batch against diarize_batch per
setting, and the command line on ES2005a from the reference's own RTTM."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import init_oracle
from vbx_b200 import VbxError, pipeline, resegment, score, sweep, synth
from vbx_b200.batch import VbxBatch

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture(scope='module')
def model():
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    return dict(z=z, transform=(m['mean1'], m['mean2'], m['lda']), plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']))


# ---- the kernel ---------------------------------------------------------------------------------------------------------

def speakers(rng, K, span, many=False):
    """K speakers' sorted disjoint turns in ticks on [0, span); many: the first one has thousands of short turns."""
    out = []
    for k in range(K):
        n = 3000 if many and k == 0 else int(rng.integers(1, 12))
        b = np.unique(rng.integers(0, span, 2 * n))
        b = b[:len(b) // 2 * 2]
        out.append((f's{k:04d}', score.merge_turns(b[0::2], b[1::2])))
    if K >= 2:
        out[1] = (out[1][0], (np.array([0], dtype=np.int64), np.array([span // 2], dtype=np.int64)))   # spans many
    return out


def segments(rng, T, span):
    """T segments in seconds on a 10 ms grid inside [0, span + 1 s): overlapping, some of zero length, some after every
    turn, some touching a turn end."""
    lo = rng.integers(0, span // 10000, T) / 100.0
    seg = np.stack([lo, lo + rng.integers(0, 300, T) / 100.0], 1)
    seg[::7, 1] = seg[::7, 0]                                  # zero length
    seg[3::11] = (span / 1e6 + 0.2, span / 1e6 + 0.9)          # uncovered
    return seg


def batch_case(Ks, lens, seed):
    rng = np.random.default_rng(seed)
    span = 60_000_000
    items = []
    for b, (K, T) in enumerate(zip(Ks, lens)):
        spk = speakers(rng, K, span, many=b == 0)
        seg = segments(rng, T, span)
        if K >= 2 and T > 5:                                  # a segment ending exactly where speaker 1's turn ends
            seg[5] = (span / 2e6 - 1.0, span / 2e6)
        items.append((seg, spk))
    return items


@pytest.mark.gpu
@pytest.mark.parametrize('f64', [False, True])
def test_init_turns_equals_the_oracle(f64):
    """Ragged batch with an empty recording and K = 1, 64, 65, 128 (and 129 on the float64 plan) speakers, one with
    3000 turns: float32 within 1 ulp of the float64 oracle, float64 within 1e-14 relative; pi0 = 1/K exactly."""
    dev = torch.device('cuda:0')
    Ks = [2, 1, 64, 65, 128, 7, 3] + ([129] if f64 else [])
    lens = [400, 300, 250, 200, 150, 0, 1] + ([180] if f64 else [])
    items = batch_case(Ks, lens, seed=3 + int(f64))
    pack = resegment.pack_turns(items)
    vb = VbxBatch(lens, 128, Ks, device=dev, allocate=False, f64_only=f64)
    dt = torch.float64 if f64 else torch.float32
    g = torch.full((vb.N, vb.S), float('nan'), dtype=dt, device=dev)
    p = torch.full((vb.B, vb.S), float('nan'), dtype=dt, device=dev)
    sm = np.array([5.0, 1.0, 11.0, 0.5, 5.0, 3.0, 7.0, 5.0])[:len(Ks)]
    vb.init_turns(pack, sm, g, p)
    g, p = g.cpu().numpy(), p.cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for b, (seg, spk) in enumerate(items):
        want, pi = init_oracle.init_gamma(score.to_ticks(seg), [t for _, t in spk], sm[b], S=vb.S)
        got = g[offs[b]:offs[b + 1]]
        if f64:
            np.testing.assert_allclose(got, want, rtol=1e-14, atol=0, err_msg=str(b))
        else:
            ulp = np.spacing(want.astype(np.float32))
            assert np.all(np.abs(got.astype(np.float64) - want) <= ulp), b
        assert np.array_equal(p[b], pi.astype(p.dtype)), b
    vb.close()


@pytest.mark.gpu
def test_init_turns_argument_errors():
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(0)
    items = [(segments(rng, 20, 10_000_000), speakers(rng, 5, 10_000_000))]
    vb = VbxBatch([20], 128, [3], device=dev, allocate=False)              # S = 4 < 5 speakers
    g = torch.zeros((vb.N, vb.S), device=dev)
    p = torch.zeros((1, vb.S), device=dev)
    with pytest.raises(VbxError, match='more than the plan'):
        vb.init_turns(resegment.pack_turns(items), 5.0, g, p)
    vb.close()
    two = resegment.pack_turns([items[0], (items[0][0][:0], items[0][1][:2])])
    vb = VbxBatch([20, 0], 128, [4, 4], device=dev, allocate=False)
    g = torch.zeros((vb.N, vb.S), device=dev)
    p = torch.zeros((2, vb.S), device=dev)
    bad = two._replace(spk_off=np.array([0, 2, 1]))                      # recording 1 with a negative speaker count
    with pytest.raises(VbxError, match='negative speaker count'):
        vb.init_turns(bad, 5.0, g, p)
    with pytest.raises(ValueError):
        vb.init_turns(two, 5.0, g.double(), p)                           # gamma and pi of different types
    vb.close()
    from vbx_b200 import _lib
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    assert lib.vbx_init_turns(h, *([None] * 9), 0, None) == -3              # VBX_ERR_STATE: no plan
    assert lib.vbx_init_turns(None, *([None] * 9), 0, None) == -1
    lib.vbx_destroy(h)


# ---- the tie to the AHC-initialised path ----------------------------------------------------------------------------------

def back_to_back(model, n_rec=6, seed=21):
    """multi_session_archive recordings with non-overlapping segments [0.24 t, 0.24 (t + 1))."""
    recs, rows, truth = synth.multi_session_archive(model['z']['x_raw'], n_rec=n_rec, seed=seed)
    out = {}
    for n, (x, _) in recs.items():
        T = len(x)
        out[n] = (x, np.stack([np.arange(T) * 0.24, np.arange(T + 1)[1:] * 0.24], 1))
    return out, rows, truth


KW = dict(Fa=0.3, Fb=17.0, loopP=0.99, smoothing=5.0, threshold=-0.015, max_iters=40, epsilon=1e-6)


@pytest.mark.gpu
def test_rttm_of_the_own_ahc_labels_is_the_ahc_path(model):
    """An RTTM written from the archive's own AHC labels (names that sort in label order) on back-to-back segments:
    every segment lies inside one speaker's turns, so gamma0 is soft_init's within 1 ulp, and diarize_batch gives
    init='AHC+VB''s labels, second labels and iteration counts."""
    recs, _, _ = back_to_back(model)
    ahc = pipeline.diarize_batch(recs, model['transform'], model['plda'], init='AHC', **KW)
    rows = [(n, float(s), float(e - s), f'L{int(l):04d}') for n, it in ahc.items()
            for (s, e), l in zip(recs[n][1], it['labels'])]
    dev = torch.device('cuda:0')
    init = resegment.load_init(rows, list(recs))
    for n in recs:
        labels = ahc[n]['labels']
        K = int(labels.max()) + 1
        assert resegment.speaker_names(init[n]) == [f'L{k:04d}' for k in range(K)]
        vb = VbxBatch([len(labels)], 128, [K], device=dev, allocate=False)
        g = torch.zeros((vb.N, vb.S), device=dev)
        p = torch.zeros((1, vb.S), device=dev)
        vb.init_turns(resegment.pack_turns([(recs[n][1], init[n])]), 5.0, g, p)
        want = pipeline.soft_init(torch.from_numpy(labels).to(dev), K, 5.0).cpu().numpy()
        got = g[:, :K].cpu().numpy()
        assert np.all(np.abs(got - want) <= np.spacing(want)), n
        assert np.all(p[0, :K].cpu().numpy() == np.float32(1.0 / K)) and not g[:, K:].any()
        vb.close()
    base = pipeline.diarize_batch(recs, model['transform'], model['plda'], init='AHC+VB', **KW)
    got = pipeline.diarize_batch(recs, model['transform'], model['plda'], init='RTTM+VB', init_rttm=rows, **KW)
    for n in recs:
        assert np.array_equal(got[n]['labels'], base[n]['labels']), n
        assert (got[n]['labels2nd'] is None) == (base[n]['labels2nd'] is None), n
        if base[n]['labels2nd'] is not None:
            assert np.array_equal(got[n]['labels2nd'], base[n]['labels2nd']), n
        assert got[n]['iterations'] == base[n]['iterations'], n
        assert got[n]['rttm'] == base[n]['rttm']
        assert got[n]['init_speakers'] == [f'L{k:04d}' for k in range(int(ahc[n]['labels'].max()) + 1)]
        assert [l.split()[7] for l in got[n]['rttm_init']] == [f'L{int(l.split()[7]) - 1:04d}' for l in got[n]['rttm']]


# ---- sweep_batch against diarize_batch ------------------------------------------------------------------------------------

def partial_rows(rows, keep=0.6):
    """The first `keep` share of each recording's reference rows: a partial annotation."""
    out = []
    for rec in dict.fromkeys(r[0] for r in rows):
        mine = [r for r in rows if r[0] == rec]
        out += mine[:int(len(mine) * keep)]
    return out


@pytest.mark.gpu
def test_sweep_entries_equal_diarize_batch(model):
    """Every setting's entries equal diarize_batch(init='RTTM+VB') with that setting's scalars (labels, iterations,
    init names, rttm_init), plain and with count bounds, overlaps, linking and enrolment each switched on once."""
    recs, rows, truth = synth.multi_session_archive(model['z']['x_raw'], n_rec=5, seed=4)
    init_rows = partial_rows(rows)
    grid = dict(Fa=[0.3, 0.5], Fb=[17.0], loopP=[0.99, 0.6], threshold=[-0.015], smoothing=[5.0, 2.0])
    names = list(recs)
    pool = sorted({int(k) for n in names for k in truth[n]})[:3]
    enroll = {f'p{k}': np.concatenate([recs[n][0][truth[n] == k] for n in names])[:15] for k in pool}
    span = {n: float(recs[n][1][-1, 1]) for n in names}
    overlaps = {n: [(0.2 * span[n], 0.3 * span[n])] for n in names}
    options = [(dict(ref_rttm=rows), dict()),                  # scored too: the sweep's reference turns are its own
               (dict(max_speakers=2, min_speakers=2), dict(max_speakers=2, min_speakers=2)),
               (dict(overlaps=overlaps), dict(overlaps=overlaps)),
               (dict(link_thresholds=[0.0]), dict(link_threshold=0.0)),
               (dict(enroll=enroll, enroll_thresholds=[0.0]), dict(enroll=enroll, enroll_threshold=0.0))]
    for sw_kw, d_kw in options:
        out = sweep.sweep_batch(recs, model['transform'], model['plda'], grid, init='RTTM+VB', init_rttm=init_rows,
                                **sw_kw)
        for s, per_rec in out.items():
            want = pipeline.diarize_batch(recs, model['transform'], model['plda'], Fa=s.Fa, Fb=s.Fb, loopP=s.loopP,
                                          smoothing=s.smoothing, threshold=s.threshold, init='RTTM+VB',
                                          init_rttm=init_rows, **d_kw)
            for n in names:
                a, b = per_rec[n], want[n]
                assert np.array_equal(a['labels'], b['labels']), (sw_kw.keys(), s, n)
                assert a['iterations'] == b['iterations'] and a['rttm'] == b['rttm'], (sw_kw.keys(), s, n)
                assert a['init_speakers'] == b['init_speakers'] and a['rttm_init'] == b['rttm_init'], (sw_kw.keys(), s, n)
                for key in ('count_rule', 'rttm_overlap'):
                    assert a.get(key) == b.get(key), (key, s, n)
                if 'link_threshold' in d_kw:
                    assert a['global_speakers'][0.0] == b['global_speakers'], (s, n)
                if 'enroll' in d_kw:
                    assert a['speaker_names'][0.0] == b['speaker_names'], (s, n)
                if 'overlaps' not in d_kw and b['init_speakers'] is not None:
                    assert all(l.split()[7] in b['init_speakers'] for l in b['rttm_init'])


# ---- the command line on ES2005a --------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_command_line_resegments_es2005a_from_the_reference(model, tmp_path):
    """cli --init RTTM+VB from ES2005a's reference RTTM: the written speakers are the input's names, and the file is
    diarize_batch's rttm_init."""
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
    ref_names = [f'FEE{int(l):03d}' for l in z['rttm_ref_labels']]
    (tmp_path / 'init').mkdir()
    (tmp_path / 'init' / 'ES2005a.rttm').write_text(''.join(
        f'SPEAKER ES2005a 1 {s:.2f} {e - s:.2f} <NA> <NA> {k} <NA> <NA>\n'
        for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], ref_names)))
    out = tmp_path / 'out'
    argv = ['--init', 'RTTM+VB', '--init-rttm', str(tmp_path / 'init'), '--out-rttm-dir', str(out),
            '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']),
            '--loopP', str(z['loopProb']), '--init-smoothing', str(z['smoothing'])]
    assert cli.main(argv) == 0
    lines = (out / 'ES2005a.rttm').read_text().splitlines()
    written = {l.split()[7] for l in lines}
    assert written and written <= set(ref_names)
    it = pipeline.diarize_batch({'ES2005a': (z['x_raw'], z['seg_times'])}, model['transform'], model['plda'],
                                Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']),
                                smoothing=float(z['smoothing']), init='RTTM+VB', init_rttm=str(tmp_path / 'init'))
    assert lines == it['ES2005a']['rttm_init']
    assert it['ES2005a']['init_speakers'] == sorted(set(ref_names))
