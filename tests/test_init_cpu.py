"""VB resegmentation, init='RTTM+VB' (DESIGN.md section 5.20), without a GPU: the oracle's coverage against a per-tick
count, its rows against soft_init, the host packing of the init turns against score.named_reference_turns, and the
argument checks of diarize_batch, sweep_batch and both command lines, which raise before any device work."""
import numpy as np
import pytest
import torch

from oracle import init_oracle
from vbx_b200 import cli, pipeline, resegment, score, sweep


def random_case(rng, T=40, K=4, span=400):
    """Segments and per-speaker sorted disjoint turns on a small tick range, with the edge cases of the definition:
    turns touching segment ends exactly, turns spanning many segments, overlapping speakers, zero-length and uncovered
    segments."""
    lo = rng.integers(0, span - 60, T)
    seg = np.stack([lo, lo + rng.integers(0, 60, T)], 1).astype(np.int64)
    seg[0] = (seg[1, 0], seg[1, 0])                               # zero length
    seg[2] = (span + 50, span + 90)                               # after every turn: uncovered
    seg[3] = (100, 140)
    turns = []
    for k in range(K):
        b = np.unique(rng.integers(0, span, 2 * int(rng.integers(1, 6))))
        if len(b) % 2:
            b = b[:-1]
        s, e = score.merge_turns(b[0::2], b[1::2])
        turns.append((s, e))
    turns[0] = (np.array([100, 300]), np.array([140, 320]))                                # touches segment 3's ends
    turns[1] = (np.array([0], dtype=np.int64), np.array([span], dtype=np.int64))          # spans every segment
    return seg, turns


def per_tick(seg, turns):
    """The coverage by counting covered ticks one by one."""
    c = np.zeros((len(seg), len(turns)))
    for t, (a, b) in enumerate(seg):
        if b <= a:
            continue
        for k, (lo, hi) in enumerate(turns):
            ticks = np.arange(a, b)
            inside = ((ticks[:, None] >= lo[None, :]) & (ticks[:, None] < hi[None, :])).any(1)
            c[t, k] = inside.sum() / (b - a)
    return c


@pytest.mark.parametrize('seed', range(6))
def test_oracle_coverage_is_the_per_tick_count(seed):
    rng = np.random.default_rng(seed)
    seg, turns = random_case(rng, K=int(rng.integers(1, 6)))
    c = init_oracle.coverage(seg, turns)
    np.testing.assert_array_equal(c, per_tick(seg, turns))
    assert not c[0].any() and not c[2].any()
    assert c[3, 0] == 1.0 and np.all(c[3:, 1][seg[3:, 1] > seg[3:, 0]] == 1.0)
    g, pi = init_oracle.init_gamma(seg, turns, 5.0, S=8)
    K = len(turns)
    np.testing.assert_allclose(g[:, :K].sum(1), 1.0, rtol=1e-15)
    assert not g[:, K:].any() and np.array_equal(pi, np.where(np.arange(8) < K, 1.0 / K, 0.0))
    np.testing.assert_array_equal(g[2, :K], np.full(K, 1.0 / K))          # uncovered: uniform


def test_one_speaker_segment_is_the_references_qinit():
    """A segment inside one speaker's turns alone gives softmax(onehot * smoothing), soft_init's row."""
    turns = [(np.array([0, 500]), np.array([100, 600])), (np.array([100]), np.array([500])),
             (np.array([700]), np.array([800]))]
    seg = np.array([[0, 100], [120, 480], [500, 600], [10, 90], [700, 800]], dtype=np.int64)
    labels = np.array([0, 1, 0, 0, 2])
    for sm in (5.0, 0.5, 11.0):
        g, _ = init_oracle.init_gamma(seg, turns, sm)
        want = pipeline.soft_init(torch.from_numpy(labels), 3, sm, dtype=torch.float64).numpy()
        np.testing.assert_allclose(g, want, rtol=1e-15, atol=0)
    g, _ = init_oracle.init_gamma(np.array([[50, 150]]), turns, 5.0)      # half speaker 0, half speaker 1: a split
    assert g[0, 0] == g[0, 1] > g[0, 2]


def kernel_coverage(pack, b, seg_rows):
    """The kernel's algorithm in numpy over a TurnPack: P(hi) - P(lo), P(x) by binary search plus turn_cum."""
    out = []
    for k in range(pack.spk_off[b], pack.spk_off[b + 1]):
        f, l = pack.turn_off[k], pack.turn_off[k + 1]
        lo, hi, cum = pack.turn_lo[f:l], pack.turn_hi[f:l], pack.turn_cum[f:l]

        def P(x):
            j = np.searchsorted(lo, x, 'left')            # turns that start before x
            return np.where(j > 0, cum[np.maximum(j - 1, 0)] + np.minimum(hi[np.maximum(j - 1, 0)], x)
                            - lo[np.maximum(j - 1, 0)], 0) if len(lo) else np.zeros_like(x)
        length = seg_rows[:, 1] - seg_rows[:, 0]
        out.append(np.where(length > 0, (P(seg_rows[:, 1]) - P(seg_rows[:, 0])) / np.maximum(length, 1), 0.0))
    return np.stack(out, 1)


@pytest.mark.parametrize('n_spk', [1, 2, 17, 64])
def test_packing_matches_named_reference_turns(n_spk):
    """load_init orders and merges as named_reference_turns; pack_turns' offsets, turns and prefix sums restate them,
    and the kernel's prefix-sum coverage over the pack equals the oracle's."""
    rng = np.random.default_rng(n_spk)
    rows = []
    for rec, T in (('b', 30), ('a', 50), ('c', 0)):
        for i in range(3 * n_spk):
            start = round(float(rng.uniform(0, 20)), 2)
            rows.append((rec, start, round(float(rng.uniform(0, 2)), 2), f'spk{int(rng.integers(n_spk)):03d}'))
        rows.append((rec, 1.0, 0.0, 'zz-empty'))           # only empty turns: not a speaker
    rows.append(('other', 0.0, 1.0, 'x'))                  # not in the archive: ignored
    names = ['a', 'b']
    init = resegment.load_init(rows, names)
    ref = score.named_reference_turns([r for r in rows if r[0] in names])
    assert list(init) == names
    for n in names:
        assert [k for k, _ in init[n]] == [k for k, _ in ref[n]] and 'zz-empty' not in resegment.speaker_names(init[n])
        for (_, (s, e)), (_, (s2, e2)) in zip(init[n], ref[n]):
            assert np.array_equal(s, s2) and np.array_equal(e, e2)
    segs = {n: np.sort(rng.uniform(0, 22, (T, 1)), 0) + np.array([[0.0, 1.5]]) for n, T in (('a', 50), ('b', 30))}
    items = [(segs['b'], init['b']), (segs['a'], init['a']), (segs['b'], init['b'])]     # a recording twice, as a sweep packs
    pack = resegment.pack_turns(items)
    K = [len(init['b']), len(init['a']), len(init['b'])]
    assert np.array_equal(pack.spk_off, np.concatenate([[0], np.cumsum(K)]))
    spk = [t for _, turns in items for _, t in turns]
    assert np.array_equal(np.diff(pack.turn_off), [len(s) for s, _ in spk])
    for k, (s, e) in enumerate(spk):
        f, l = pack.turn_off[k], pack.turn_off[k + 1]
        assert np.array_equal(pack.turn_lo[f:l], s) and np.array_equal(pack.turn_hi[f:l], e)
        assert np.array_equal(pack.turn_cum[f:l], np.concatenate([[0], np.cumsum(e - s)[:-1]]))
    assert pack.seg.shape == (110, 2) and pack.seg.dtype == np.int64
    offs = np.concatenate([[0], np.cumsum([50 if i == 1 else 30 for i in range(3)])])
    for b, (seg, turns) in enumerate(items):
        rows_b = pack.seg[offs[b]:offs[b + 1]]
        assert np.array_equal(rows_b, score.to_ticks(seg))
        np.testing.assert_array_equal(kernel_coverage(pack, b, rows_b), init_oracle.coverage(rows_b, [t for _, t in turns]))


def test_129_speakers_pack_without_the_score_cap():
    rows = [('r', 0.5 * k, 0.5, f's{k:03d}') for k in range(129)]
    with pytest.raises(ValueError, match='at most 64'):
        score.named_reference_turns(rows)
    init = resegment.load_init(rows, ['r'])
    assert len(init['r']) == 129
    pack = resegment.pack_turns([(np.array([[0.0, 1.5], [10.0, 11.5]]), init['r'])])
    assert list(pack.spk_off) == [0, 129] and len(pack.turn_lo) == 129 and not pack.turn_cum.any()
    assert pipeline._tier(129) == 2                   # more than 128 states: the float64 tier


# ---- argument checks before any device work -------------------------------------------------------------------------------

def archive():
    rng = np.random.default_rng(0)
    seg = np.stack([np.arange(10) * 0.24, np.arange(10) * 0.24 + 1.5], 1)
    return {'r1': (rng.standard_normal((10, 32)), seg), 'r2': (rng.standard_normal((10, 32)), seg)}


ROWS = [('r1', 0.0, 2.0, 'A'), ('r1', 2.0, 1.0, 'B'), ('r2', 0.0, 3.0, 'B'), ('r9', 0.0, 1.0, 'C')]
MODEL = dict(transform=None, plda=None, Fa=0.3, Fb=17.0, loopP=0.99)
GRID = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])


def test_diarize_batch_argument_errors():
    recs = archive()
    with pytest.raises(ValueError, match=r"recordings missing from the init RTTM: \['r2'\]"):
        pipeline.diarize_batch(recs, init='RTTM+VB', init_rttm=ROWS[:2], **MODEL)
    with pytest.raises(ValueError, match=r"without a speaker in the init RTTM: \['r2'\]"):
        pipeline.diarize_batch(recs, init='RTTM+VB', init_rttm=ROWS[:2] + [('r2', 1.0, 0.0, 'B')], **MODEL)
    with pytest.raises(ValueError, match='needs init_rttm'):
        pipeline.diarize_batch(recs, init='RTTM+VB', **MODEL)
    for init in ('AHC', 'AHC+VB'):
        with pytest.raises(ValueError, match='init_rttm'):
            pipeline.diarize_batch(recs, init=init, init_rttm=ROWS, **MODEL)
    with pytest.raises(ValueError, match='Wrong option'):
        pipeline.diarize_batch(recs, init='RTTM', **MODEL)


def test_diarize_batch_reads_an_init_rttm_path(tmp_path):
    """A file goes through score.read_rttm_path: its missing recording is named before any device work."""
    p = tmp_path / 'init.rttm'
    p.write_text(''.join(f'SPEAKER {r} 1 {s:.2f} {d:.2f} <NA> <NA> {k} <NA> <NA>\n' for r, s, d, k in ROWS[:2]))
    with pytest.raises(ValueError, match=r"\['r2'\]"):
        pipeline.diarize_batch(archive(), init='RTTM+VB', init_rttm=str(p), **MODEL)
    with pytest.raises(ValueError, match=r"\['r2'\]"):
        pipeline.diarize_batch(archive(), init='RTTM+VB', init_rttm=str(tmp_path), **MODEL)


def test_sweep_batch_argument_errors():
    recs = archive()
    grid = dict(GRID, threshold=[-0.015, 0.1])
    with pytest.raises(ValueError, match='threshold axis must hold one value'):
        sweep.sweep_batch(recs, None, None, grid, init='RTTM+VB', init_rttm=ROWS)
    with pytest.raises(ValueError, match=r"recordings missing from the init RTTM: \['r2'\]"):
        sweep.sweep_batch(recs, None, None, GRID, init='RTTM+VB', init_rttm=ROWS[:2])
    with pytest.raises(ValueError, match='needs init_rttm'):
        sweep.sweep_batch(recs, None, None, GRID, init='RTTM+VB')
    with pytest.raises(ValueError, match='init_rttm'):
        sweep.sweep_batch(recs, None, None, GRID, init='AHC+VB', init_rttm=ROWS)


CLI_ARGS = ['--out-rttm-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 's', '--xvec-transform', 't.h5',
            '--plda-file', 'p', '--threshold', '-0.015', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99']
SWEEP_ARGS = ['--out-dir', 'o', '--xvec-ark-file', 'x.ark', '--segments-file', 's', '--xvec-transform', 't.h5',
              '--plda-file', 'p', '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99',
              '--threshold=-0.015']


@pytest.mark.parametrize('module, base', [(cli, CLI_ARGS), (sweep, SWEEP_ARGS)])
def test_command_line_init_rttm_options(module, base, capsys):
    args = module.build_parser().parse_args(base + ['--init', 'RTTM+VB', '--init-rttm', 'init_dir'])
    assert args.init == 'RTTM+VB' and args.init_rttm == 'init_dir'
    for extra in (['--init', 'RTTM+VB'], ['--init', 'AHC+VB', '--init-rttm', 'init_dir']):
        with pytest.raises(SystemExit) as e:
            module.main(base + extra)
        assert e.value.code == 2
        assert '--init RTTM+VB and --init-rttm go together' in capsys.readouterr().err
    with pytest.raises(SystemExit):                  # --threshold stays required, as in the reference's parser
        module.build_parser().parse_args([a for a in base if not a.startswith('--threshold') and a != '-0.015']
                                         + ['--init', 'RTTM+VB', '--init-rttm', 'x'])
