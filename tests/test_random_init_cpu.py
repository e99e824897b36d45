"""Random initialisation of the VB-HMM (init='RANDOM+VB', DESIGN.md section 5.22) without a GPU: the oracle's Philox
against numpy's, the rows it draws, the stream keys, the restart choice, the VB stage's restart entries (with _vb_tier
replaced by a fake) and the argument checks of diarize_batch, sweep_batch and both command lines."""
import hashlib
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import random_init_oracle as oracle
from vbx_b200 import cli, pipeline, random_init, sweep

M64 = (1 << 64) - 1


# ---- the generator ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('seed, counter', [
    (0, 1), (1, 2), (12345, 1 << 64), (7, (1 << 64) + 5), (M64, (1 << 128)), (2 ** 63, (1 << 192) + 3),
    (0xDEADBEEF, (1 << 256) - 1), (99, 3 + (17 << 64) + (5 << 128)),
])
def test_oracle_philox_equals_numpy(seed, counter):
    """np.random.Philox(key=seed, counter=c - 1).random_raw(4) is Philox4x64-10 of counter c (four little-endian words)
    under key (seed, 0): numpy advances its counter before each block, also across the carries between the words."""
    want = np.random.Philox(key=seed, counter=counter - 1).random_raw(4)
    words = [(counter >> (64 * i)) & M64 for i in range(4)]
    got = oracle.philox4x64([words], (seed, 0))[0]
    assert [int(v) for v in got] == [int(v) for v in want]


def test_oracle_exponentials_follow_the_definition():
    """e[t, 4j + i] = -log(((w_i >> 11) + 0.5) 2^-53) of the block (t, j, key, 0), drawn through numpy's Philox."""
    key, seed = oracle.name_key('rec-α'), M64 - 2
    e = oracle.exponentials(5, 7, key, seed)
    assert e.shape == (5, 8)
    for t in range(5):
        for j in range(2):
            c = t + (j << 64) + (key << 128)
            w = np.random.Philox(key=seed, counter=c - 1).random_raw(4)
            u = np.array([((int(x) >> 11) + 0.5) * 2.0 ** -53 for x in w])
            assert np.array_equal(e[t, 4 * j:4 * j + 4], -np.log(u))


def test_rows_sum_to_one_with_zero_padding():
    for N, S in ((1, 4), (3, 4), (8, 8), (65, 128), (129, 129), (10, 16)):
        g, pi = oracle.init_gamma(40, N, oracle.name_key(f'r{N}'), N, S=S)
        assert g.shape == (40, S) and np.all(g[:, N:] == 0) and np.all(g[:, :N] > 0)
        np.testing.assert_allclose(g.sum(axis=1), 1.0, rtol=1e-14)
        assert np.all(pi[:N] == 1.0 / N) and np.all(pi[N:] == 0)
    g, pi = oracle.init_gamma(0, 5, 1, 2, S=8)
    assert g.shape == (0, 8) and np.all(pi[:5] == 0.2)


def test_a_column_is_the_flat_dirichlet_marginal():
    """Column s of N = 8 flat-Dirichlet rows is Beta(1, N - 1): a KS test on 50 000 rows."""
    g, _ = oracle.init_gamma(50_000, 8, oracle.name_key('rec2'), 2)
    for s in (0, 5):
        assert stats.kstest(g[:, s], stats.beta(1, 7).cdf).pvalue > 1e-3


def test_restart_r_of_seed_s_is_restart_0_of_seed_s_plus_r():
    key = oracle.name_key('meeting')
    for s, r in ((0, 3), (41, 7), (M64 - 1, 3), (M64, 1)):
        assert random_init.restart_seed(s, r) == oracle.restart_seed(s, r) == (s + r) % (1 << 64)
        a, _ = oracle.init_gamma(20, 6, key, random_init.restart_seed(s, r))
        b, _ = oracle.init_gamma(20, 6, key, oracle.restart_seed(s + r, 0) if s + r < 1 << 64 else s + r - (1 << 64))
        assert np.array_equal(a, b)
    c, _ = oracle.init_gamma(20, 6, key, 1)
    d, _ = oracle.init_gamma(20, 6, key, 2)
    assert not np.array_equal(c, d)


def test_name_key_is_stable_and_the_archive_does_not_matter():
    assert random_init.name_key('ES2005a') == 9716333371497247983
    for n in ('ES2005a', 'rec-α', '', 'a b/c'):
        assert random_init.name_key(n) == oracle.name_key(n) == \
            int.from_bytes(hashlib.sha256(n.encode('utf-8')).digest()[:8], 'little')
    # one key per name: the same list whatever the order or the other recordings
    assert [random_init.name_key(n) for n in ('b', 'a')][::-1] == [random_init.name_key(n) for n in ('a', 'b')]


# ---- the restart choice -----------------------------------------------------------------------------------------------

def test_restart_choice_on_hand_built_traces():
    nan = math.nan
    cases = [
        # Li rows (NaN padded), n_iters, chosen restart
        ([[-5.0, -3.0, nan], [-6.0, -2.0, -1.5], [-4.0, nan, nan]], [2, 3, 1], 1),
        ([[-5.0, -3.0], [-6.0, nan]], [2, 0], 0),                                 # a restart that ran no iteration
        ([[-5.0, nan], [-1.0, nan], [-1.0, nan]], [2, 1, 1], 1),                  # a NaN final ELBO never wins; ties: lowest
        ([[-2.0, -1.0], [-3.0, -1.0], [0.0, -1.0]], [2, 2, 2], 0),                # a tie of all three
        ([[nan, nan], [nan, nan]], [1, 2], 0),                                    # nothing finite: restart 0
        ([[-1.0, math.inf], [-3.0, -2.0]], [2, 2], 1),                            # an infinite ELBO never wins
    ]
    for Li, n, want in cases:
        final = random_init.final_elbo(np.array(Li), n)
        r, o_final = oracle.choose(Li, n)
        assert random_init.best_restart(final) == r == want, (Li, n)
        np.testing.assert_array_equal(final, np.array(o_final))


# ---- the VB stage: restarts as entries --------------------------------------------------------------------------------

DEV = torch.device('cpu')
MAKE = object()
HYPER = [(0.3, 17.0, 0.99, 5.0), (0.4, 6.0, 0.5, 5.0)]


def fake_tier(monkeypatch, offs, elbo_of):
    """Replace _vb_tier: record each call; labels t % ns of every entry; the final ELBO elbo_of(recording, seed)."""
    calls = []

    def tier(lens, ns, fea, Phi, labels, f64, smoothing, dev, make=None, hi=None, random=None, elbo=False, **kw):
        o = np.concatenate([[0], np.cumsum(lens)])
        recs = [int(np.searchsorted(offs, float(fea[o[j], 0]), 'right')) - 1 for j in range(len(lens))]
        calls.append(dict(recs=recs, ns=[int(n) for n in ns], f64=f64, random=random, elbo=elbo, hi=hi, kw=kw,
                          labels=labels))
        out = []
        for j in range(len(lens)):
            l = np.arange(lens[j], dtype=np.int64) % int(ns[j])
            r = (l, None, 5, 0)
            if hi is not None:
                r += (len(np.unique(l)), 'vb')
            out.append(r + (elbo_of(recs[j], random[1][j]),) if elbo else r)
        return out
    monkeypatch.setattr(pipeline, '_vb_tier', tier)
    return calls


def test_vb_stage_runs_every_restart_and_keeps_the_best(monkeypatch):
    lens = np.array([30, 20, 10], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)])
    fea = torch.zeros((int(offs[-1]), 4))
    fea[:, 0] = torch.arange(int(offs[-1]), dtype=torch.float32)
    seed = M64 - 1                                        # the third restart's seed wraps to 0
    table = {(0, seed): -5.0, (0, M64): -3.0, (0, 0): -3.0,      # recording 0: a tie of restarts 1 and 2
             (1, seed): math.nan, (1, M64): -9.0, (1, 0): -8.0,
             (2, seed): math.nan, (2, M64): math.nan, (2, 0): math.nan}
    calls = fake_tier(monkeypatch, offs, lambda b, s: table[(b, s)])
    keys = [11, 22, 33]
    rs = random_init.RandomStart(n_states=7, restarts=3, seed=seed, keys=keys)
    out = pipeline._vb_stage(HYPER, None, None, None, lens, fea, torch.ones(4), None, 'RANDOM+VB', DEV, MAKE, None,
                             random=rs, maxIters=40, epsilon=1e-6)
    assert len(calls) == 1 and not calls[0]['f64'] and calls[0]['elbo'] and calls[0]['labels'] is None
    # (setting, recording, restart) in that order, the restarts of a recording side by side
    assert calls[0]['recs'] == [0, 0, 0, 1, 1, 1, 2, 2, 2] * 2 and calls[0]['ns'] == [7] * 18
    assert calls[0]['random'] == (([11] * 3 + [22] * 3 + [33] * 3) * 2, [seed, M64, 0] * 6)
    assert calls[0]['kw']['Fa'].tolist() == [0.3] * 9 + [0.4] * 9
    for k in range(2):
        assert out[(k, 0)][-1] == (1, [-5.0, -3.0, -3.0])
        assert out[(k, 1)][-1][0] == 2
        assert out[(k, 2)][-1][0] == 0
        assert out[(k, 0)][:4][2:] == (5, 0) and len(out[(k, 0)]) == 5


def test_vb_stage_float64_tier_holds_every_restart_of_a_setting(monkeypatch):
    lens = np.array([200, 150], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)])
    fea = torch.zeros((int(offs[-1]), 4))
    fea[:, 0] = torch.arange(int(offs[-1]), dtype=torch.float32)
    calls = fake_tier(monkeypatch, offs, lambda b, s: -float(s))
    rs = random_init.RandomStart(n_states=130, restarts=4, seed=10, keys=[1, 2])
    out = pipeline._vb_stage(HYPER, None, None, None, lens, fea, torch.ones(4), None, 'RANDOM+VB', DEV, MAKE, None,
                             random=rs, maxIters=40, epsilon=1e-6)
    assert [(c['f64'], c['recs']) for c in calls] == [(True, [0] * 4 + [1] * 4)] * 2
    assert [c['kw']['Fa'] for c in calls] == [0.3, 0.4]
    assert all(out[(k, b)][-1][0] == 0 for k in range(2) for b in range(2))     # -seed: seed 10 is largest


def test_vb_stage_count_rules_follow_the_chosen_restart(monkeypatch):
    from scipy.cluster.hierarchy import linkage
    lens = np.array([40, 30], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)])
    fea = torch.zeros((int(offs[-1]), 4))
    fea[:, 0] = torch.arange(int(offs[-1]), dtype=torch.float32)
    rng = np.random.default_rng(0)
    Zs = [linkage(rng.standard_normal((T, 3)), 'average') for T in lens]
    calls = fake_tier(monkeypatch, offs, lambda b, s: float(s))               # the last restart wins
    rs = random_init.RandomStart(n_states=3, restarts=2, seed=0, keys=[5, 6])
    lo, hi = np.array([6, 1]), np.array([8, 2])
    out = pipeline._vb_stage(HYPER[:1], None, None, Zs, lens, fea, torch.ones(4), (lo, hi), 'RANDOM+VB', DEV, MAKE,
                             None, random=rs, maxIters=40, epsilon=1e-6)
    assert calls[0]['hi'].tolist() == [8, 8, 2, 2]
    again = [c for c in calls[1:]]                 # rule 3 for recording 0 (3 < lo = 6) from the AHC cut, as for AHC+VB
    assert len(again) == 1 and again[0]['recs'] == [0] and again[0]['random'] is None
    assert out[(0, 0)][4:6] == (3, 'recut') and out[(0, 0)][-1] == (1, [0.0, 1.0])
    assert out[(0, 1)][4:6] == (3, 'vb') and out[(0, 1)][-1][0] == 1


# ---- argument checks --------------------------------------------------------------------------------------------------

def rec(T=6, D=4):
    return {'r': (np.zeros((T, D)), np.stack([np.arange(T), np.arange(T) + 1.0], 1))}


def test_check_init_options():
    assert pipeline._check_init('RANDOM+VB', False, None, 5) == (5, 1, 0, None)
    assert pipeline._check_init('RANDOM+VB', True, None, 5, 8, M64) == (5, 8, M64, None)
    assert pipeline._check_init('AHC+VB', False) is None
    with pytest.raises(ValueError, match='Wrong option'):
        pipeline._check_init('RTTM', False)
    with pytest.raises(ValueError, match='Wrong option'):
        pipeline._check_init('RANDOM', False, None, 5)
    bad = [dict(init_states=None), dict(init_states=0), dict(init_states=2.0), dict(init_states=True),
           dict(init_states=3, restarts=0), dict(init_states=3, restarts=1.5), dict(init_states=3, seed=-1),
           dict(init_states=3, seed=1 << 64), dict(init_states=3, seed=0.5)]
    for kw in bad:
        with pytest.raises(ValueError):
            pipeline._check_init('RANDOM+VB', False, None, **kw)
    for init in ('AHC', 'AHC+VB'):
        for kw in (dict(init_states=3), dict(restarts=2), dict(seed=0)):
            with pytest.raises(ValueError, match='RANDOM'):
                pipeline._check_init(init, False, None, **kw)
    with pytest.raises(ValueError, match='init_rttm'):
        pipeline._check_init('RANDOM+VB', False, 'x.rttm', 3)


def test_diarize_batch_refuses_bad_options_before_device_work():
    kw = dict(transform=None, plda=None, Fa=0.3, Fb=17.0, loopP=0.99)
    with pytest.raises(ValueError, match='init_states'):
        pipeline.diarize_batch(rec(), init='RANDOM+VB', **kw)
    with pytest.raises(ValueError, match='RANDOM'):
        pipeline.diarize_batch(rec(), init='AHC+VB', restarts=4, **kw)
    with pytest.raises(ValueError, match='RANDOM'):
        pipeline.diarize_batch(rec(), init='RTTM+VB', init_rttm=[], seed=4, **kw)
    with pytest.raises(ValueError, match='seed'):
        pipeline.diarize_batch(rec(), init='RANDOM+VB', init_states=4, seed=-3, **kw)
    with pytest.raises(ValueError, match='Wrong option'):
        pipeline.diarize_batch(rec(), init='RTTM', **kw)


def test_sweep_batch_refuses_bad_options_before_device_work():
    grid = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
    with pytest.raises(ValueError, match='init_states'):
        sweep.sweep_batch(rec(), None, None, grid, init='RANDOM+VB')
    with pytest.raises(ValueError, match='RANDOM'):
        sweep.sweep_batch(rec(), None, None, grid, init='AHC+VB', init_states=3)
    for axis in ('threshold', 'smoothing'):
        g = dict(grid, **{axis: [0.1, 0.2]})
        with pytest.raises(ValueError, match=f'{axis} axis'):
            sweep.sweep_batch(rec(), None, None, g, init='RANDOM+VB', init_states=3)


BASE = ['--out-rttm-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 'x.seg', '--xvec-transform', 't.h5',
        '--plda-file', 'plda', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']


@pytest.mark.parametrize('argv, message', [
    (['--init', 'RANDOM+VB', '--threshold', '0'], 'go together'),
    (['--init', 'AHC+VB', '--init-states', '5', '--threshold', '0'], 'go together'),
    (['--init', 'AHC+VB', '--restarts', '5', '--threshold', '0'], 'options of --init RANDOM'),
    (['--init', 'RTTM+VB', '--init-rttm', 'r', '--seed', '5', '--threshold', '0'], 'options of --init RANDOM'),
    (['--init', 'RANDOM+VB', '--init-states', '0', '--threshold', '0'], 'init-states must'),
    (['--init', 'RANDOM+VB', '--init-states', '4', '--restarts', '0', '--threshold', '0'], 'restarts must'),
    (['--init', 'RANDOM+VB', '--init-states', '4', '--seed', str(1 << 64), '--threshold', '0'], 'seed must'),
    (['--init', 'RANDOM+VB', '--init-states', '4'], 'threshold'),           # still required, as by the reference
    (['--init', 'RANDOM', '--init-states', '4', '--threshold', '0'], 'invalid choice'),
])
def test_cli_usage_errors(argv, message, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(argv + BASE)
    assert e.value.code == 2 and message in capsys.readouterr().err


SWEEP = ['--out-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 'x.seg', '--xvec-transform', 't.h5',
         '--plda-file', 'plda', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']


@pytest.mark.parametrize('argv, message', [
    (['--init', 'RANDOM+VB', '--threshold', '0'], 'go together'),
    (['--init-states', '5', '--threshold', '0'], 'go together'),
    (['--restarts', '2', '--threshold', '0'], 'options of --init RANDOM'),
    (['--seed', '2', '--threshold', '0'], 'options of --init RANDOM'),
    (['--init', 'RANDOM+VB', '--init-states', '4'], 'threshold'),
])
def test_sweep_usage_errors(argv, message, capsys):
    with pytest.raises(SystemExit) as e:
        sweep.main(argv + SWEEP)
    assert e.value.code == 2 and message in capsys.readouterr().err


def test_parsers_take_the_options():
    a = cli.build_parser().parse_args(['--init', 'RANDOM+VB', '--init-states', '10', '--restarts', '8', '--seed',
                                       str(M64), '--threshold', '-0.015'] + BASE)
    assert (a.init, a.init_states, a.restarts, a.seed) == ('RANDOM+VB', 10, 8, M64)
    a = sweep.build_parser().parse_args(['--init', 'RANDOM+VB', '--init-states', '3', '--threshold', '0'] + SWEEP)
    assert (a.init, a.init_states, a.restarts, a.seed) == ('RANDOM+VB', 3, None, None)
