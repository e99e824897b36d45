"""The VB-HMM stage after AHC (pipeline._vb_stage) that diarize_batch and sweep_batch share: state tiers, batch packing,
the hyperparameter form and the speaker-count rules 2 and 3 (DESIGN.md section 5.14), driven on CPU tensors with
_vb_tier replaced by a fake that records its calls.  Runs without a GPU."""
import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import linkage

from vbx_b200 import ahc, pipeline, sweep

DEV = torch.device('cpu')
MAKE = object()          # stands for the batch planner: the stage only hands it on
HYPER = [(0.3, 17.0, 0.99, 5.0), (0.4, 6.0, 0.5, 3.0), (0.2, 64.0, 0.9, 7.0)]


def archive(lens, seed=0):
    """fea [N,4] whose column 0 is the global row, Phi, and a seeded average-linkage matrix per recording."""
    rng = np.random.default_rng(seed)
    N = int(np.sum(lens))
    fea = torch.zeros((N, 4))
    fea[:, 0] = torch.arange(N, dtype=torch.float32)
    Zs = [linkage(rng.standard_normal((T, 3)), 'average') if T > 1 else np.zeros((0, 4)) for T in lens]
    return np.asarray(lens, dtype=np.int64), fea, torch.ones(4), Zs


def labels_for(lens, ns):
    """AHC labels of ns[b] clusters on recording b."""
    return [np.arange(T, dtype=np.int64) % n for T, n in zip(lens, ns)]


def fake_tier(monkeypatch, offs, rerun_one=()):
    """Replace _vb_tier: record each call; return every recording's input labels as its VB-HMM labels, except on
    re-runs (no hi) of the recordings in rerun_one, which end with one speaker."""
    calls = []

    def tier(lens, ns, fea, Phi, labels, f64, smoothing, dev, make=None, hi=None, **kw):
        o = np.concatenate([[0], np.cumsum(lens)])
        recs = [int(np.searchsorted(offs, float(fea[o[j], 0]), 'right')) - 1 for j in range(len(lens))]
        calls.append(dict(lens=[int(t) for t in lens], ns=[int(n) for n in ns], recs=recs, fea=fea,
                          labels=labels.numpy().copy(), f64=f64, smoothing=smoothing, make=make, hi=hi, kw=kw))
        out = []
        for j in range(len(lens)):
            l = labels.numpy()[o[j]:o[j + 1]].astype(np.int64)
            if hi is None and recs[j] in rerun_one:
                l = np.zeros_like(l)
            r = (l, (l + 1) % max(int(ns[j]), 1), 10 + j, 0)
            out.append(r if hi is None else r + (len(np.unique(l)), 'vb'))
        return out
    monkeypatch.setattr(pipeline, '_vb_tier', tier)
    return calls


def stage(hyper, labels, lens, fea, Phi, Zs, bounds=None, init='AHC+VB', split=None):
    labels_d = [torch.from_numpy(np.concatenate(l)) for l in labels]
    return pipeline._vb_stage(hyper, labels, labels_d, Zs, lens, fea, Phi, bounds, init, DEV, MAKE, split,
                              maxIters=40, epsilon=1e-6)


def test_tiers_split_at_64_and_128_states(monkeypatch):
    ns = [129, 64, 1, 65, 200, 128]
    lens, fea, Phi, Zs = archive([n + 7 for n in ns])
    calls = fake_tier(monkeypatch, np.concatenate([[0], np.cumsum(lens)]))
    out = stage(HYPER[:1], [labels_for(lens, ns)], lens, fea, Phi, Zs)
    assert [(c['ns'], c['f64']) for c in calls] == [([64, 1], False), ([65, 128], False), ([129, 200], True)]
    assert [c['recs'] for c in calls] == [[1, 2], [3, 5], [0, 4]]
    for c in calls:
        assert c['make'] is MAKE and c['hi'] is None and c['kw']['maxIters'] == 40
        # one setting: numbers, not per-recording tensors
        assert (c['kw']['Fa'], c['kw']['Fb'], c['kw']['loopProb'], c['smoothing']) == HYPER[0]
        assert np.array_equal(c['labels'], np.concatenate([labels_for(lens, ns)[b] for b in c['recs']]))
    assert sorted(out) == [(0, b) for b in range(len(ns))]
    assert all(np.array_equal(out[(0, b)][0], labels_for(lens, ns)[b]) for b in range(len(ns)))


def test_a_tier_of_every_recording_takes_the_features_as_they_are(monkeypatch):
    lens, fea, Phi, Zs = archive([30, 50, 20])
    calls = fake_tier(monkeypatch, np.concatenate([[0], np.cumsum(lens)]))
    stage(HYPER[:1], [labels_for(lens, [3, 5, 2])], lens, fea, Phi, Zs)
    assert len(calls) == 1 and calls[0]['fea'] is fea


def test_several_settings_take_tensors_and_float64_runs_once_per_setting(monkeypatch):
    lens, fea, Phi, Zs = archive([150, 40, 90])
    calls = fake_tier(monkeypatch, np.concatenate([[0], np.cumsum(lens)]))
    labels = [labels_for(lens, [140, 10, 70]), labels_for(lens, [140, 10, 3]), labels_for(lens, [5, 10, 70])]
    out = stage(HYPER, labels, lens, fea, Phi, Zs)
    f32 = [c for c in calls if not c['f64']]
    f64 = [c for c in calls if c['f64']]
    assert [c['ns'] for c in f32] == [[10, 10, 3, 5, 10], [70, 70]]
    assert [c['recs'] for c in f32] == [[1, 1, 2, 0, 1], [2, 2]]
    settings = [[0, 1, 1, 2, 2], [0, 2]]            # entries in setting-major order
    for c, ks in zip(f32, settings):
        for i, name in enumerate(('Fa', 'Fb', 'loopProb')):
            assert c['kw'][name].dtype == torch.float64
            assert c['kw'][name].tolist() == [HYPER[k][i] for k in ks]
        assert list(c['smoothing']) == [HYPER[k][3] for k in ks]
    # the float64 tier: one run per setting that has entries there, with that setting's numbers
    assert [(c['ns'], c['kw']['Fa'], c['smoothing']) for c in f64] == [([140], 0.3, 5.0), ([140], 0.4, 3.0)]
    assert len(out) == 9


def test_sweep_packing_follows_entry_order_under_the_budget(monkeypatch):
    lens, fea, Phi, Zs = archive([100, 300, 200, 50])
    calls = fake_tier(monkeypatch, np.concatenate([[0], np.cumsum(lens)]))
    monkeypatch.setattr(sweep, 'entry_bytes', lambda T, S, R, dev: int(T))
    labels = [labels_for(lens, [4, 8, 80, 6])] * 2
    stage(HYPER[:2], labels, lens, fea, Phi, Zs, split=sweep.packer(lens, 4, DEV, 400))
    # tier 0 entries (0,0) (0,1) (0,3) (1,0) (1,1) (1,3): 100 300 50 100 300 50 bytes; tier 1 (0,2) (1,2): 200 200
    assert [c['recs'] for c in calls] == [[0, 1], [3, 0], [1, 3], [2, 2]]
    assert [c['kw']['Fa'].tolist() for c in calls] == [[0.3, 0.3], [0.3, 0.4], [0.4, 0.4], [0.3, 0.4]]
    assert not any(c['f64'] for c in calls)
    calls.clear()
    stage(HYPER[:2], labels, lens, fea, Phi, Zs)         # no split: one batch per tier
    assert [len(c['lens']) for c in calls] == [6, 2]
    with pytest.raises(ValueError, match='max_batch_bytes'):
        stage(HYPER[:2], labels, lens, fea, Phi, Zs, split=sweep.packer(lens, 4, DEV, 250))


def test_count_rules_share_one_rerun_per_tier(monkeypatch):
    # 0: too few, re-run in tier 0, ends in bounds (recut); 1: too few, re-run in tier 1, ends short (ahc);
    # 2: fewer x-vectors than lo (unmet); 3: in bounds (vb)
    lens, fea, Phi, Zs = archive([150, 120, 5, 40])
    offs = np.concatenate([[0], np.cumsum(lens)])
    calls = fake_tier(monkeypatch, offs, rerun_one={1})
    lo = np.array([10, 100, 8, 3])
    hi = np.array([20, 110, 9, 6])
    labels = [labels_for(lens, [3, 3, 2, 4])] * 2
    out = stage(HYPER[:2], labels, lens, fea, Phi, Zs, bounds=(lo, hi))
    first = [c for c in calls if c['hi'] is not None]
    again = [c for c in calls if c['hi'] is None]
    assert len(first) == 1 and first[0]['hi'].tolist() == hi.tolist() * 2
    mc = ahc.cut_count(Zs, lens, lo)
    assert [(c['recs'], c['ns'], c['f64']) for c in again] == [([0, 0], [10, 10], False), ([1, 1], [100, 100], False)]
    for c in again:
        b = c['recs'][0]
        assert np.array_equal(c['labels'], np.concatenate([mc[b], mc[b]]))
        assert c['kw']['Fa'].tolist() == [0.3, 0.4]
    for k in range(2):
        assert out[(k, 0)][4:] == (3, 'recut') and np.array_equal(out[(k, 0)][0], mc[0]) and out[(k, 0)][2] == 10 + k
        assert out[(k, 1)][4:] == (3, 'ahc') and out[(k, 1)][1:4] == (None, 0, 0)
        assert np.array_equal(out[(k, 1)][0], mc[1])
        assert out[(k, 2)][4:] == (2, 'unmet') and np.array_equal(out[(k, 2)][0], np.arange(5))
        assert out[(k, 3)][4:] == (4, 'vb') and np.array_equal(out[(k, 3)][0], labels[k][3])


def test_init_ahc_takes_rule_4_without_the_vb_hmm(monkeypatch):
    lens, fea, Phi, Zs = archive([60, 40])
    calls = fake_tier(monkeypatch, np.concatenate([[0], np.cumsum(lens)]))
    labels = [labels_for(lens, [3, 9]), labels_for(lens, [5, 4])]
    plain = stage(HYPER[:2], labels, lens, fea, Phi, Zs, init='AHC')
    assert all(np.array_equal(plain[(k, b)][0], labels[k][b]) and plain[(k, b)][1:] == (None, 0, 0)
               for k in range(2) for b in range(2))
    bounds = (np.array([4, 2]), np.array([4, 6]))
    out = stage(HYPER[:2], labels, lens, fea, Phi, Zs, bounds=bounds, init='AHC')
    for k in range(2):
        want, k1, rules = pipeline._count_ahc(Zs, lens, labels[k], bounds)
        for b in range(2):
            assert np.array_equal(out[(k, b)][0], want[b]) and out[(k, b)][1:] == (None, 0, 0, k1[b], rules[b])
    assert [out[(k, b)][5] for k in range(2) for b in range(2)] == ['ahc', 'ahc', 'ahc', 'vb']
    assert calls == []
