"""Speaker-count constraints (DESIGN.md section 5.14) on the host: the maxclust cut against scipy, the rules' numpy
restatement (oracle/count_oracle.py) and the float64 tier's torch restatement of rule 2 against it, the argument
checks, the command-line parsing and the oracle speaker count.  CPU-only."""
import argparse

import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.spatial.distance import pdist

from oracle import count_oracle
from vbx_b200 import ahc, cli, formats, pipeline, score, sweep


def _linkages():
    for seed in range(24):
        rng = np.random.default_rng(seed)
        T = int(rng.integers(3, 60))
        x = rng.standard_normal((T, 4))
        yield f'seed{seed}', linkage(pdist(x), method='average'), T
    for seed in range(12):                 # few distinct points: many merges at tied heights
        rng = np.random.default_rng(100 + seed)
        T = int(rng.integers(3, 40))
        x = rng.integers(0, 3, (T, 2)).astype(np.float64)
        yield f'ties{seed}', linkage(pdist(x), method='average'), T


@pytest.mark.parametrize('name,Z,T', list(_linkages()), ids=lambda v: v if isinstance(v, str) else '')
def test_cut_count_is_scipy_maxclust(name, Z, T):
    for k in range(1, T + 1):
        got = ahc.cut_count([Z], [T], [k])[0]
        want = fcluster(Z, k, criterion='maxclust') - 1
        assert np.array_equal(got, want), (name, k)
        # the numbering is flat_clusters' at the chosen height
        if k < T:
            assert len(np.unique(got)) <= k


def test_cut_count_ties_leave_fewer_clusters():
    x = np.array([[0.0], [0.0], [1.0], [1.0], [2.0], [2.0]])
    Z = linkage(pdist(x), method='average')
    got = ahc.cut_count([Z], [6], [5])[0]                   # the three zero-height merges happen together
    assert len(np.unique(got)) == 3
    assert np.array_equal(got, fcluster(Z, 5, 'maxclust') - 1)


def test_cut_count_one_and_two_xvectors():
    assert ahc.cut_count([np.zeros((0, 4))], [1], [1])[0].tolist() == [0]
    assert ahc.cut_count([np.zeros((0, 4))], [1], [3])[0].tolist() == [0]
    assert ahc.cut_count([np.zeros((0, 4))], [0], [2])[0].tolist() == []
    Z = linkage(pdist(np.array([[0.0], [1.0]])), method='average')
    for k in (1, 2, 5):
        assert np.array_equal(ahc.cut_count([Z], [2], [k])[0], fcluster(Z, k, 'maxclust') - 1)
    with pytest.raises(ValueError):
        ahc.cut_count([Z], [2], [0])


def _posteriors(rng, T, S, ties=False):
    g = rng.dirichlet(np.full(S, 0.3), size=T)
    if ties:                                   # tied columns (tied masses) and tied entries inside rows
        g[:, S // 2] = g[:, 0]
        g[::3, 1] = g[::3, 0]
        g /= g.sum(1, keepdims=True)
    return g


@pytest.mark.parametrize('seed', range(8))
def test_float64_tier_rule2_equals_the_oracle(seed):
    """pipeline.keep_labels (the float64 tier's torch ops) == count_oracle.keep_labels: ties in mass and in gamma go to
    the lower state, dead states (no mass) are dropped first, keep >= n_states is the plain argsort."""
    rng = np.random.default_rng(seed)
    S = int(rng.integers(2, 12))
    g = _posteriors(rng, int(rng.integers(1, 200)), S, ties=seed % 2 == 0)
    if seed % 3 == 0:
        g[:, S - 1] = 0.0                                       # a dead state
    for keep in range(1, S + 2):
        f, s, mass = count_oracle.keep_labels(g, S, keep)
        tf, ts = pipeline.keep_labels(torch.from_numpy(g), keep)
        assert np.array_equal(tf.numpy(), f), keep
        assert np.array_equal(ts.numpy(), s), keep
        np.testing.assert_allclose(mass, g.sum(0), rtol=1e-15)
        if keep >= S:
            order = np.argsort(-g, axis=1, kind='stable')
            assert np.array_equal(f, order[:, 0]) and (S == 1 or np.array_equal(s, order[:, 1]))
        assert len(np.unique(f)) <= keep


def test_oracle_mass_ties_go_to_the_lower_state():
    g = np.array([[0.5, 0.2, 0.3], [0.1, 0.5, 0.4], [0.4, 0.3, 0.3]])      # masses 1.0, 1.0, 1.0
    f, s, _ = count_oracle.keep_labels(g, 3, 2)
    assert set(np.unique(f)) <= {0, 1} and f.tolist() == [0, 1, 0] and s.tolist() == [1, 0, 1]
    f, s, _ = count_oracle.keep_labels(g[:, :1], 1, 1)                      # one-state recording
    assert f.tolist() == [0, 0, 0] and s.tolist() == [-1, -1, -1]


def test_oracle_rules():
    rng = np.random.default_rng(3)
    T, S = 40, 6
    g = _posteriors(rng, T, S)
    lab = np.argmax(g, 1)
    k1 = len(np.unique(lab))
    lab2 = np.argsort(-g, 1, kind='stable')[:, 1]
    Z = linkage(rng.standard_normal((T, 3)), method='average')
    calls = []

    def rerun(init):
        calls.append(init)
        return init, None

    assert count_oracle.vb_rules(lab, lab2, g, 1, k1, Z, rerun)[2] == 'vb'
    f, s, rule, kk = count_oracle.vb_rules(lab, lab2, g, 2, 2, Z, rerun)
    assert rule == 'mass' and kk == k1 and len(np.unique(f)) <= 2
    f, s, rule, _ = count_oracle.vb_rules(lab, lab2, g, 1, 1, Z, rerun)
    assert rule == 'mass' and s is None and len(np.unique(f)) == 1
    f, s, rule, _ = count_oracle.vb_rules(lab, lab2, g, k1 + 2, k1 + 3, Z, rerun)
    assert rule == 'recut' and np.array_equal(f, fcluster(Z, k1 + 2, 'maxclust') - 1)
    f, s, rule, _ = count_oracle.vb_rules(lab, lab2, g, k1 + 2, k1 + 3, Z, lambda init: (np.zeros(T, int), None))
    assert rule == 'ahc' and s is None and np.array_equal(f, fcluster(Z, k1 + 2, 'maxclust') - 1)
    f, s, rule, _ = count_oracle.vb_rules(lab[:3], lab2[:3], g[:3], 5, 5, linkage(rng.standard_normal((3, 2))), rerun)
    assert rule == 'unmet' and len(np.unique(f)) == 3
    assert len(calls) == 1
    thr = fcluster(Z, 0.5 * Z[-1, 2], 'distance') - 1
    K = len(np.unique(thr))
    assert count_oracle.ahc_rules(thr, 1, K, Z)[1] == 'vb'
    lab4, rule, _ = count_oracle.ahc_rules(thr, 1, max(K - 1, 1), Z)
    assert rule == 'ahc' and len(np.unique(lab4)) <= max(K - 1, 1)
    assert count_oracle.ahc_rules(thr[:3], 4, 6, linkage(rng.standard_normal((3, 2))))[1] == 'unmet'


def test_host_rule4_equals_the_oracle():
    """pipeline._count_ahc (rule 4, init='AHC') == count_oracle.ahc_rules on seeded linkages."""
    rng = np.random.default_rng(9)
    lens, Zs, labels = [], [], []
    for T in (30, 50, 2, 1, 20):
        Z = linkage(rng.standard_normal((T, 3)), method='average') if T > 1 else np.zeros((0, 4))
        lens.append(T)
        Zs.append(Z)
        labels.append(fcluster(Z, 0.6 * Z[-1, 2], 'distance') - 1 if T > 1 else np.zeros(T, dtype=np.int64))
    for lo, hi in ((1, 1), (2, 3), (4, 4), (1, 100), (3, 8)):
        bounds = (np.full(5, lo), np.full(5, hi))
        got, k1, rules = pipeline._count_ahc(Zs, np.array(lens), labels, bounds)
        for b in range(5):
            want, rule, kk = count_oracle.ahc_rules(labels[b], lo, hi, Zs[b])
            assert np.array_equal(got[b], want) and rules[b] == rule and k1[b] == kk, (lo, hi, b)


def test_count_bounds_argument_checks():
    names = ['a', 'b']
    assert pipeline.count_bounds(names) is None
    lo, hi = pipeline.count_bounds(names, num_speakers=3)
    assert lo.tolist() == [3, 3] and hi.tolist() == [3, 3]
    lo, hi = pipeline.count_bounds(names, min_speakers={'a': 2, 'b': 1, 'c': 9}, max_speakers=4)
    assert lo.tolist() == [2, 1] and hi.tolist() == [4, 4]
    lo, hi = pipeline.count_bounds(names, min_speakers=2)
    assert hi.tolist() == [pipeline.UNBOUNDED] * 2
    with pytest.raises(ValueError, match='not both'):
        pipeline.count_bounds(names, num_speakers=2, max_speakers=3)
    with pytest.raises(ValueError, match='not both'):
        pipeline.count_bounds(names, num_speakers=2, min_speakers=1)
    with pytest.raises(ValueError, match='min_speakers > max_speakers'):
        pipeline.count_bounds(names, min_speakers=4, max_speakers=3)
    for bad in (0, -1):
        with pytest.raises(ValueError, match='>= 1'):
            pipeline.count_bounds(names, num_speakers=bad)
        with pytest.raises(ValueError, match='>= 1'):
            pipeline.count_bounds(names, max_speakers={'a': 2, 'b': bad})
    with pytest.raises(ValueError, match=r"\['b'\]"):
        pipeline.count_bounds(names, num_speakers={'a': 2})
    with pytest.raises(ValueError, match='integer'):
        pipeline.count_bounds(names, num_speakers=2.5)


def test_entry_points_check_before_running():
    recs = {'a': (np.zeros((4, 256)), np.zeros((4, 2)))}
    grid = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
    with pytest.raises(ValueError, match='ref_rttm'):
        sweep.sweep_batch(recs, None, None, grid, num_speakers='oracle')
    with pytest.raises(ValueError, match='oracle'):
        sweep.sweep_batch(recs, None, None, grid, num_speakers='estimate')
    with pytest.raises(ValueError, match='not both'):
        sweep.sweep_batch(recs, None, None, grid, num_speakers=2, min_speakers=1)
    with pytest.raises(ValueError, match=r"\['a'\]"):
        sweep.sweep_batch(recs, None, None, grid, max_speakers={'b': 2})
    with pytest.raises(ValueError, match='>= 1'):
        pipeline.diarize_batch(recs, None, None, 0.3, 17.0, 0.99, num_speakers=0)
    with pytest.raises(ValueError, match='min_speakers > max_speakers'):
        pipeline.diarize_batch(recs, None, None, 0.3, 17.0, 0.99, min_speakers=3, max_speakers=2)


def test_command_line_count_options(tmp_path):
    f = tmp_path / 'counts'
    f.write_text('# recording count\nrecA 2\n\nrecB 5\n')
    assert cli.speaker_count_arg('4') == 4
    assert cli.speaker_count_arg(str(f)) == {'recA': 2, 'recB': 5}
    with pytest.raises(argparse.ArgumentTypeError):
        cli.speaker_count_arg('oracle')
    assert cli.speaker_count_arg('oracle', allow_oracle=True) == 'oracle'
    (tmp_path / 'bad').write_text('recA two\n')
    with pytest.raises(argparse.ArgumentTypeError):
        cli.speaker_count_arg(str(tmp_path / 'bad'))
    base = ['--init', 'AHC+VB', '--out-rttm-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform',
            't', '--plda-file', 'p', '--threshold', '-0.015', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP',
            '0.99']
    a = cli.build_parser().parse_args(base)
    assert a.num_speakers is None and a.min_speakers is None and a.max_speakers is None
    a = cli.build_parser().parse_args(base + ['--num-speakers', '2'])
    assert a.num_speakers == 2
    a = cli.build_parser().parse_args(base + ['--min-speakers', str(f), '--max-speakers', '6'])
    assert a.min_speakers == {'recA': 2, 'recB': 5} and a.max_speakers == 6
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(base + ['--num-speakers', 'oracle'])
    sb = ['--out-dir', 'o', '--xvec-ark-file', 'x', '--segments-file', 's', '--xvec-transform', 't', '--plda-file', 'p',
          '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99', '--threshold=-0.015']
    assert sweep.build_parser().parse_args(sb + ['--num-speakers', 'oracle']).num_speakers == 'oracle'
    assert sweep.build_parser().parse_args(sb + ['--num-speakers', str(f)]).num_speakers == {'recA': 2, 'recB': 5}
    assert sweep.build_parser().parse_args(sb + ['--max-speakers', '3']).max_speakers == 3
    assert sweep.build_parser().parse_args(sb).num_speakers is None
    assert formats.read_speaker_counts(str(f)) == {'recA': 2, 'recB': 5}


def test_reference_speaker_counts():
    rows = [('r1', 0.0, 1.0, 'A'), ('r1', 2.0, 1.0, 'B'), ('r1', 5.0, 0.0, 'C'), ('r1', 4.0, 1.0, 'A'),
            ('r2', 0.0, 3.0, 'X')]
    turns = score.reference_turns(rows)
    assert score.reference_speaker_counts(turns) == {'r1': 2, 'r2': 1}
    uem = {'r1': [(0.0, 1.5), (4.5, 9.0)], 'r2': [(3.0, 4.0)]}              # B talks only outside the UEM; X as well
    assert score.reference_speaker_counts(turns, uem) == {'r1': 1, 'r2': 0}
    assert score.reference_speaker_counts(turns, {'r1': [(2.9, 3.1)], 'r2': [(0.0, 9.0)]}) == {'r1': 1, 'r2': 1}
