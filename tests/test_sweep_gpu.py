"""The hyperparameter sweep (vbx_b200/sweep.py) on the shipped ES2005a inputs: every setting equals diarize_batch with
that setting's scalars, across all three state tiers; the example setting reproduces the reference; the batch budget
does not change results; the command line writes what sweep_batch returns."""
import json
import os

import numpy as np
import pytest
import torch

from vbx_b200 import pipeline, sweep

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
# thresholds -0.015 / 0.1 / 0.2 give 31 / 80 / 144 AHC clusters on ES2005a: the <= 64, S = 128 and float64 tiers
GRID = dict(Fa=[0.3, 0.4], Fb=[17.0], loopP=[0.99, 0.5], threshold=[-0.015, 0.1, 0.2], smoothing=[5.0])
EXAMPLE = sweep.Setting(0.3, 17.0, 0.99, -0.015, 5.0)


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    return z, recs, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])


@pytest.fixture(scope='module')
def swept(es):
    z, recs, transform, plda = es
    return sweep.sweep_batch(recs, transform, plda, GRID, device=torch.device('cuda:0'))


def same(a, b):
    assert np.array_equal(a['labels'], b['labels'])
    assert a['n_speakers'] == b['n_speakers'] and a['iterations'] == b['iterations']
    assert a['rttm'] == b['rttm']


def test_every_setting_equals_diarize_batch(es, swept):
    z, recs, transform, plda = es
    assert [s for s in swept] == sweep.grid_settings(GRID)
    for s, per_rec in swept.items():
        ref = pipeline.diarize_batch(recs, transform, plda, s.Fa, s.Fb, s.loopP, threshold=s.threshold,
                                     smoothing=s.smoothing, max_iters=40, epsilon=1e-6, device=torch.device('cuda:0'))
        same(per_rec['ES2005a'], ref['ES2005a'])
        assert per_rec['ES2005a']['flags'] & 1 == 0


def test_example_setting_reproduces_the_reference(es, swept):
    z = es[0]
    item = swept[EXAMPLE]['ES2005a']
    assert np.array_equal(item['labels'], z['labels'])
    assert len(item['rttm']) == len(z['rttm_starts'])
    for line, s, e in zip(item['rttm'], z['rttm_starts'], z['rttm_ends']):
        f = line.split()
        assert abs(float(f[3]) - s) < 1e-5 and abs(float(f[4]) - (e - s)) < 1e-5


def test_small_batch_budget_gives_the_same_results(es, swept, monkeypatch):
    z, recs, transform, plda = es
    dev = torch.device('cuda:0')
    T = z['x_raw'].shape[0]
    budget = 2 * max(sweep.entry_bytes(T, 32, 128, dev), sweep.entry_bytes(T, 128, 128, dev))
    calls = []
    pack = sweep.pack
    monkeypatch.setattr(sweep, 'pack', lambda sizes, b: calls.append(pack(sizes, b)) or calls[-1])
    small = sweep.sweep_batch(recs, transform, plda, GRID, device=dev, max_batch_bytes=budget)
    assert sum(len(c) for c in calls) >= 3
    for s in swept:
        same(small[s]['ES2005a'], swept[s]['ES2005a'])


def test_command_line_writes_one_directory_per_setting(es, swept, tmp_path):
    from vbx_b200 import formats
    z, recs, transform, plda = es
    keys, seg_lines = [], []
    for i, (s, e) in enumerate(z['seg_times']):
        k = f'ES2005a_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
        keys.append(k)
        seg_lines.append(f'{k} ES2005a {float(s)!r} {float(e)!r}')
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, z['x_raw'])
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    out = tmp_path / 'out'
    rc = sweep.main(['--out-dir', str(out), '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file',
                     str(tmp_path / 'x.seg'), '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file',
                     str(tmp_path / 'plda.txt'), '--lda-dim', '128', '--Fa', '0.3,0.4', '--Fb', '17', '--loopP', '0.99,0.5',
                     '--threshold=-0.015,0.1,0.2', '--init-smoothing', '5'])     # a list starting with '-': the = form
    assert rc == 0
    summary = json.loads((out / 'summary.json').read_text())
    assert sorted(summary) == sorted(s.name for s in swept)
    for s, per_rec in swept.items():
        item = per_rec['ES2005a']
        got = summary[s.name]['recordings']['ES2005a']
        assert got == dict(speakers=item['n_speakers'], iterations=item['iterations'], flags=item['flags'])
        lines = (out / s.name / 'ES2005a.rttm').read_text().splitlines()
        assert len(lines) == len(item['rttm'])
