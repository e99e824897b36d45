"""DER scoring on the device (vbx_score through vbx_b200/score.py): exact tick equality with the line-sweep oracle
(oracle/der_oracle.py) on seeded ragged archives, batch independence, label checks, and the sweep scored against the
reference system's own ES2005a RTTM."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import der_oracle
from vbx_b200 import VbxError, pipeline, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')


def ref_layers(rng, span_cs, K, layers):
    """Reference turns (start cs, end cs, speaker) over [0, span_cs): `layers` independent sequences of turns, so at most
    that many speakers overlap; every one of the K speakers gets at least one turn."""
    turns, spk = [], 0
    for _ in range(layers):
        t = int(rng.integers(0, 200))
        while t < span_cs:
            d = int(rng.integers(10, 200))
            turns.append((t, t + d, f'spk{spk % K}'))
            spk += 1 if spk < K else int(rng.integers(1, K + 1))
            t += d + int(rng.integers(0, 150))
    return turns


def sticky(rng, T, L, stay=0.9):
    lab = np.zeros(T, dtype=np.int64)
    if T:
        lab[0] = rng.integers(L)
    for t in range(1, T):
        lab[t] = lab[t - 1] if rng.random() < stay else rng.integers(L)
    if T > 1:
        lab[-1] = L - 1                       # the entry's label count is L
    return lab


def ragged_case(seed, with_uem):
    """Recordings: length 1, gaps, no reference speech, 1 .. 64 reference speakers with up to 4 overlapping; entries with
    label counts up to 128 and 200."""
    rng = np.random.default_rng(seed)
    lens = [1, 37, 260, 180, 90, 0, 300]
    segs = synth.make_scoring_archive(lens, seed=seed, gap_prob=0.08)
    spec = [(1, 1), (3, 2), (64, 4), (9, 3), (0, 0), (2, 1), (40, 4)]     # (reference speakers, overlap layers)
    names, ref_rows, recs, uem = [], [], [], {}
    for (n, (seg, _)), (K, layers) in zip(segs.items(), spec):
        span = int(round(seg[:, 1].max() * 100)) + 200 if len(seg) else 500
        turns = ref_layers(rng, span, K, layers) if K else []
        ref_rows += [(n, s / 100.0, (e - s) / 100.0, k) for s, e, k in turns]
        names.append(n)
        uem[n] = [(0.5, span / 200.0), (span / 200.0 + 1.0, span / 100.0 - 0.3)]
    turns = score.reference_turns(ref_rows)
    for n in names:
        recs.append(score.prepare_recording(n, turns.get(n, []), score.owned_intervals(segs[n][0]),
                                            uem[n] if with_uem else None))
    entries = []
    for b, n in enumerate(names):
        T = len(segs[n][0])
        for L in (1, 2, 7, 128, 200):
            entries.append((b, sticky(rng, T, L)))
    return names, segs, ref_rows, recs, entries, (uem if with_uem else None)


def oracle_entry(n, seg, labels, ref_rows, uem, collar, ignore):
    t = score.to_ticks
    s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], labels)
    ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows if r[0] == n]
    return der_oracle.der_ticks(ref, list(zip(t(s).tolist(), t(e).tolist(), l.tolist())), int(t(collar)), ignore,
                                None if uem is None else [(int(t(a)), int(t(b))) for a, b in uem[n]])


@pytest.mark.parametrize('with_uem', [False, True])
def test_device_equals_oracle_on_ragged_archives(with_uem):
    names, segs, ref_rows, recs, entries, uem = ragged_case(3 + with_uem, with_uem)
    got = score.score_entries(recs, entries, device=DEV)
    assert any(r.n_ref == 64 for r in recs) and any(len(r.sys_lo) == 1 for r in recs)
    for (b, lab), res in zip(entries, got):
        n = names[b]
        for p, c, io in score.PROTOCOLS:
            want = oracle_entry(n, segs[n][0], lab, ref_rows, uem, c, io)
            assert res[p]['ticks'] == want, (n, int(lab.max()) + 1 if len(lab) else 0, p)
            if want['scored'] == 0:
                assert res[p]['der'] is None


def test_entry_alone_equals_entry_in_batch_and_second_run():
    names, segs, ref_rows, recs, entries, _ = ragged_case(5, True)
    batch = score.score_entries(recs, entries, device=DEV)
    again = score.score_entries(recs, entries, device=DEV)
    assert batch == again
    for i in (0, 12, len(entries) - 1):
        assert score.score_entries(recs, [entries[i]], device=DEV)[0] == batch[i]


def test_out_of_range_label_raises():
    names, segs, ref_rows, recs, entries, _ = ragged_case(6, False)
    b, lab = entries[8]
    bad = lab.copy()
    bad[len(bad) // 2] = -1
    with pytest.raises(VbxError, match='labels must lie'):
        score.score_entries(recs, [entries[0], (b, bad)], device=DEV)


def test_ground_truth_of_a_synthetic_archive_scores_zero():
    arch = synth.make_scoring_archive([40, 700, 1, 2500], seed=9, gap_prob=0.03)
    rows, recs, entries = [], [], []
    for b, (n, (seg, lab)) in enumerate(arch.items()):
        s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
        rows += [(n, float(a), float(z - a), f'gt{k}') for a, z, k in zip(s, e, l)]
    turns = score.reference_turns(rows)
    for b, (n, (seg, lab)) in enumerate(arch.items()):
        recs.append(score.prepare_recording(n, turns[n], score.owned_intervals(seg)))
        entries.append((b, (lab + 3) % 11))                     # any relabelling
    for res in score.score_entries(recs, entries, device=DEV):
        for p in res:
            assert res[p]['der'] == 0.0 and res[p]['ticks']['scored'] > 0


# ---- the sweep, scored against the reference system's own RTTM -----------------------------------------------------
GRID = dict(Fa=[0.3, 0.4], Fb=[17.0], loopP=[0.99, 0.5], threshold=[-0.015, 0.2], smoothing=[5.0])   # 31 / 144 clusters
EXAMPLE = sweep.Setting(0.3, 17.0, 0.99, -0.015, 5.0)


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    rows = [('ES2005a', float(s), float(e - s), str(int(k)))
            for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], z['rttm_ref_labels'])]
    return z, recs, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi']), rows


def test_sweep_scores_the_example_setting_zero_and_ranks_it_first(es):
    z, recs, transform, plda, rows = es
    out = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=rows)
    item = out[EXAMPLE]['ES2005a']
    assert not np.array_equal(z['rttm_labels'], z['rttm_ref_labels'])      # the same segments under other labels
    for p, _, _ in score.PROTOCOLS:
        assert item['der'][p]['der'] == 0.0
    tot, ranking = sweep.summarize_der(out)
    for p, _, _ in score.PROTOCOLS:
        assert tot[ranking[p][0]][p]['der'] == 0.0
        ders = [tot[n][p]['der'] for n in ranking[p]]
        assert ders == sorted(ders)
    # every entry, float64 tier included, against the oracle
    for s, per_rec in out.items():
        for p, c, io in score.PROTOCOLS:
            want = oracle_entry('ES2005a', z['seg_times'], per_rec['ES2005a']['labels'], rows, None, c, io)
            assert per_rec['ES2005a']['der'][p]['ticks'] == want, (s.name, p)


def test_sweep_with_ahc_init_is_scored(es):
    z, recs, transform, plda, rows = es
    grid = dict(GRID, Fa=[0.3], loopP=[0.99])
    out = sweep.sweep_batch(recs, transform, plda, grid, device=DEV, init='AHC', ref_rttm=rows)
    for s, per_rec in out.items():
        for p, c, io in score.PROTOCOLS:
            want = oracle_entry('ES2005a', z['seg_times'], per_rec['ES2005a']['labels'], rows, None, c, io)
            assert per_rec['ES2005a']['der'][p]['ticks'] == want


def shifted(es, shift):
    """ES2005a with every segment and reference time moved by `shift` seconds."""
    z, recs, transform, plda, rows = es
    recs = {'ES2005a': (z['x_raw'], z['seg_times'] + shift)}
    return recs, [(r[0], r[1] + shift, r[2], r[3]) for r in rows]


def test_sweep_past_1000_s_equals_the_oracle(es):
    """At 3000 s merge_adjacent_labels joins equal labels across the 10 and 20 ms pauses of ES2005a: every entry still scores
    exactly the segments it would write."""
    z, _, transform, plda, _ = es
    recs, rows = shifted(es, 3000.0)
    seg = recs['ES2005a'][1]
    lo, hi, join_hi = score.owned_intervals(seg)
    assert np.sum(join_hi > hi) == 2
    out = sweep.sweep_batch(recs, transform, plda, dict(GRID, Fa=[0.3], loopP=[0.99]), device=DEV, ref_rttm=rows)
    for s, per_rec in out.items():
        for p, c, io in score.PROTOCOLS:
            want = oracle_entry('ES2005a', seg, per_rec['ES2005a']['labels'], rows, None, c, io)
            assert per_rec['ES2005a']['der'][p]['ticks'] == want, (s.name, p)


def test_sweep_without_speaker_in_reference_is_an_error(es):
    z, recs, transform, plda, rows = es
    with pytest.raises(ValueError, match='missing from the reference'):
        sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=[('IS1009a', 0.0, 1.0, 'a')])


@pytest.mark.parametrize('shift', [0.0, 3000.0])
def test_sweep_command_line_der_equals_the_score_command(es, tmp_path, capsys, shift):
    """shift = 3000 s: there the written RTTM joins equal labels across 10 and 20 ms pauses."""
    from vbx_b200 import formats
    z, _, transform, plda, _ = es
    recs, rows = shifted(es, shift)
    keys, seg_lines = [], []
    for i, (s, e) in enumerate(recs['ES2005a'][1]):
        k = f'ES2005a_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
        keys.append(k)
        seg_lines.append(f'{k} ES2005a {float(s)!r} {float(e)!r}')
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, z['x_raw'])
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    ref = tmp_path / 'ref.rttm'
    ref.write_text(''.join(f'SPEAKER {r[0]} 1 {r[1]:.6f} {r[2]:.6f} <NA> <NA> {r[3]} <NA> <NA>\n' for r in rows)
                   + 'SPEAKER IS1009a 1 0.0 1.0 <NA> <NA> x <NA> <NA>\n')          # not in the archive: ignored
    out = tmp_path / 'out'
    assert sweep.main(['--out-dir', str(out), '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file',
                       str(tmp_path / 'x.seg'), '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file',
                       str(tmp_path / 'plda.txt'), '--lda-dim', '128', '--Fa', '0.3,0.4', '--Fb', '17', '--loopP',
                       '0.99,0.5', '--threshold=-0.015,0.2', '--init-smoothing', '5', '--ref-rttm', str(ref)]) == 0
    summary = json.loads((out / 'summary.json').read_text())
    names = [s.name for s in sweep.grid_settings(GRID)]
    assert sorted(summary) == sorted(names + ['ranking'])
    for p, _, _ in score.PROTOCOLS:
        ders = [summary[n]['der'][p]['der'] for n in summary['ranking'][p]]
        assert ders == sorted(ders)
        if shift == 0.0:
            assert ders[0] == 0.0
    (tmp_path / 'only_es.rttm').write_text(''.join(l for l in ref.read_text().splitlines(True) if ' ES2005a ' in l))
    capsys.readouterr()
    for name in names:
        n_seg = len((out / name / 'ES2005a.rttm').read_text().splitlines())
        tol = 2 * n_seg + 2                  # each written boundary is rounded to 1 us
        for p, c, io in score.PROTOCOLS:
            argv = ['--ref-rttm', str(tmp_path / 'only_es.rttm'), '--sys-rttm', str(out / name), '--collar', str(c), '--json']
            assert score.main(argv + (['--ignore-overlaps'] if io else [])) == 0
            cli = json.loads(capsys.readouterr().out)['files']['ES2005a']
            mine = summary[name]['recordings']['ES2005a']['der'][p]
            assert cli['ticks']['scored'] == mine['ticks']['scored']
            for k in ('miss', 'fa', 'conf'):
                assert abs(cli['ticks'][k] - mine['ticks'][k]) <= tol, (name, p, k)
            assert summary[name]['der'][p]['ticks'] == mine['ticks']          # one recording: overall = it
