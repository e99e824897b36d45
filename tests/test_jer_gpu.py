"""Jaccard error rate on the device (vbx_score_jer through vbx_b200/score.py, DESIGN.md section 5.13): label time and
intersections equal to the line-sweep oracle (oracle/jer_oracle.py) on the segments the project writes, the DER outputs
bit-identical to vbx_score / vbx_score_overlap, batch independence, score_rttm on parsed files, and the sweep against
the score command on ES2005a."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.jer_oracle import jer_ticks
from vbx_b200 import pipeline, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')
LABEL_COUNTS = (1, 2, 7, 128, 129, 200)          # 129 and 200: the label block takes the global path


def ref_layers(rng, span_cs, K, layers):
    """Reference turns (start cs, end cs, speaker): `layers` independent sequences, so at most that many overlap."""
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
        lab[-1] = L - 1
    return lab


def ragged_case(seed, with_uem, two_stream):
    """Recordings of length 1, with pauses, empty, without reference speech, with 64 reference speakers; entries with
    1 .. 200 labels (two-stream: second labels with -1 rows, overlap regions the reference's own or seeded)."""
    rng = np.random.default_rng(seed)
    lens = [1, 37, 260, 180, 90, 0, 300]
    segs = synth.make_scoring_archive(lens, seed=seed, gap_prob=0.08)
    spec = [(1, 1), (3, 2), (64, 4), (9, 3), (0, 0), (2, 1), (40, 4)]
    names, ref_rows, uem = [], [], {}
    for (n, (seg, _)), (K, layers) in zip(segs.items(), spec):
        span = int(round(seg[:, 1].max() * 100)) + 200 if len(seg) else 500
        turns = ref_layers(rng, span, K, layers) if K else []
        ref_rows += [(n, s / 100.0, (e - s) / 100.0, k) for s, e, k in turns]
        names.append(n)
        uem[n] = [(0.5, span / 200.0), (span / 200.0 + 1.0, span / 100.0 - 0.3)]
    turns = score.reference_turns(ref_rows)
    recs, ovl = [], []
    for b, n in enumerate(names):
        o = None
        if two_stream:
            if b % 2 == 0:
                o = score.oracle_overlaps(turns.get(n, []))
            else:
                span = float(segs[n][0][:, 1].max()) + 2 if len(segs[n][0]) else 5.0
                o = score.overlap_ticks(np.sort(rng.uniform(0, span, 2 * int(rng.integers(1, 9)))).reshape(-1, 2).tolist())
        ovl.append(o)
        recs.append(score.prepare_recording(n, turns.get(n, []), score.owned_intervals(segs[n][0]),
                                            uem[n] if with_uem else None, overlap=o))
    entries = []
    for b, n in enumerate(names):
        T = len(segs[n][0])
        for L in LABEL_COUNTS:
            lab = sticky(rng, T, L)
            if not two_stream:
                entries.append((b, lab))
                continue
            lab2 = None if L == 1 else (lab + sticky(rng, T, L - 1, 0.8) + 1) % L
            if lab2 is not None and L == 7:
                lab2[rng.random(T) < 0.3] = -1
            entries.append((b, lab, lab2))
    return names, segs, ref_rows, recs, ovl, entries, (uem if with_uem else None)


def system_segments(seg, labels, labels2, overlap):
    """The segments the project writes, in ticks: stream 1 merged, stream 2 with its own join clipped to the overlap
    regions; -1 second labels say nothing."""
    t = score.to_ticks
    s, e, l = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], labels) if len(seg) else ([], [], [])
    out = list(zip(t(np.asarray(s)).tolist(), t(np.asarray(e)).tolist(), np.asarray(l).tolist()))
    if labels2 is not None:
        timeline = score.owned_intervals(seg)
        end2 = score.effective_hi(timeline, labels2)
        for a, b, k in zip(timeline[0].tolist(), end2.tolist(), labels2.tolist()):
            if k >= 0:
                out += [(max(a, c), min(b, d), k) for c, d in zip(*(v.tolist() for v in overlap)) if min(b, d) > max(a, c)]
    return out


def capture(monkeypatch):
    """Records the exact inputs score_entries hands to finish() and jer_finish()."""
    seen = dict(finish=[], jer=[])
    real_finish, real_jer = score.finish, score.jer_finish

    def finish(cov, fa, O, ref_total):
        seen['finish'].append((int(cov), int(fa), np.array(O, dtype=np.int64)))
        return real_finish(cov, fa, O, ref_total)

    def jer_finish(R, S, O):
        seen['jer'].append((list(R), np.array(S, dtype=np.int64), np.array(O, dtype=np.int64)))
        return real_jer(R, S, O)

    monkeypatch.setattr(score, 'finish', finish)
    monkeypatch.setattr(score, 'jer_finish', jer_finish)
    return seen


def check_against_oracle(R, S, O, want, spk_names):
    """Device R [K], S [L], O [K x L] against jer_ticks (speakers by name, labels by number), exactly."""
    assert R == [want['R'].get(k, 0) for k in spk_names]
    assert S.tolist() == [want['S'].get(s, 0) for s in range(len(S))]
    assert set(want['S']) <= set(range(len(S)))
    assert O.tolist() == [[want['I'].get((k, s), 0) for s in range(len(S))] for k in spk_names]


@pytest.mark.parametrize('two_stream', [False, True])
@pytest.mark.parametrize('with_uem', [False, True])
def test_label_time_and_intersections_equal_the_oracle(monkeypatch, with_uem, two_stream):
    names, segs, ref_rows, recs, ovl, entries, uem = ragged_case(31 + 2 * with_uem + two_stream, with_uem, two_stream)
    assert any(r.n_ref == 64 for r in recs) and any(len(r.sys_lo) == 1 for r in recs)
    assert any(r.n_ref == 0 for r in recs) and any(len(r.sys_lo) == 0 for r in recs)
    seen = capture(monkeypatch)
    got = score.score_entries(recs, entries, device=DEV, jer='full')
    assert len(seen['jer']) == len(entries)
    t = score.to_ticks
    for e, res, (R, S, O) in zip(entries, got, seen['jer']):
        b, lab = e[0], e[1]
        n = names[b]
        ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows if r[0] == n]
        sysseg = system_segments(segs[n][0], lab, e[2] if two_stream else None, ovl[b])
        want = jer_ticks(ref, sysseg, None if uem is None else [(int(t(a)), int(t(c))) for a, c in uem[n]])
        spk = sorted({r[3] for r in ref_rows if r[0] == n})
        check_against_oracle(R, S, O, want, spk)
        assert res['jer'] == score.jer_finish(R, S, O)
        assert res['jer']['speakers'] == len(want['R'])


@pytest.mark.parametrize('two_stream', [False, True])
def test_der_outputs_are_bit_identical_to_the_plain_launches(monkeypatch, two_stream):
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(41 + two_stream, True, two_stream)
    seen = capture(monkeypatch)
    plain = score.score_entries(recs, entries, device=DEV)
    raw_plain = list(seen['finish'])
    seen['finish'].clear()
    withjer = score.score_entries(recs, entries, device=DEV, jer='full')
    assert len(raw_plain) == len(seen['finish']) == len(entries) * len(score.PROTOCOLS)
    for (c0, f0, o0), (c1, f1, o1) in zip(raw_plain, seen['finish']):
        assert (c0, f0) == (c1, f1) and np.array_equal(o0, o1)
    assert [{p: r[p] for p, _, _ in score.PROTOCOLS} for r in withjer] == plain
    assert all(set(r) == {p for p, _, _ in score.PROTOCOLS} for r in plain)


@pytest.mark.parametrize('two_stream', [False, True])
def test_entry_alone_equals_entry_in_batch_and_second_run(two_stream):
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(51 + two_stream, True, two_stream)
    batch = score.score_entries(recs, entries, device=DEV, jer='full')
    assert score.score_entries(recs, entries, device=DEV, jer='full') == batch
    for i in (0, 3, 5, 15, 17, len(entries) - 1):
        assert score.score_entries(recs, [entries[i]], device=DEV, jer='full')[0] == batch[i]


def rows_of(n, segments, names_of=str):
    return [(n, a / 1e6, (z - a) / 1e6, names_of(k)) for a, z, k in segments]


@pytest.mark.parametrize('collar', [0.0, 0.25])
@pytest.mark.parametrize('overlapping', [False, True])
def test_score_rttm_equals_the_oracle_on_parsed_files(monkeypatch, collar, overlapping):
    names, segs, ref_rows, recs, ovl, entries, uem = ragged_case(61 + overlapping, True, overlapping)
    sys_rows = []
    with_ref = {r[0] for r in ref_rows}
    # one system per recording that has a reference: its 7-label entry (second labels with -1 rows)
    by_rec = {e[0]: e for i, e in enumerate(entries) if LABEL_COUNTS[i % len(LABEL_COUNTS)] == 7 and names[e[0]] in with_ref}
    for b, e in by_rec.items():
        sys_rows += rows_of(names[b], system_segments(segs[names[b]][0], e[1], e[2] if overlapping else None, ovl[b]),
                            lambda k: f'L{k}')
    seen = capture(monkeypatch)
    per, tot = score.score_rttm(ref_rows, sys_rows, collar, False, uem, device=DEV, overlapping=overlapping, jer=True)
    t = score.to_ticks
    jers = []
    for (R, S, O), n in zip(seen['jer'], sorted(per)):
        ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows if r[0] == n]
        sysseg = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in sys_rows if r[0] == n]
        want = jer_ticks(ref, sysseg, [(int(t(a)), int(t(c))) for a, c in uem[n]])
        labels = sorted({r[3] for r in sys_rows if r[0] == n})
        want = dict(want, S={labels.index(k): v for k, v in want['S'].items()},
                    I={(r, labels.index(k)): v for (r, k), v in want['I'].items()})
        check_against_oracle(R, S, O, want, sorted({r[3] for r in ref_rows if r[0] == n}))
        fin = score.jer_finish(R, S, O)
        assert per[n]['jer'] == fin['jer'] and per[n]['jer_ticks'] == fin['ticks']
        jers.append(fin)
    assert tot['jer'] == score.overall_jer(jers)['jer']
    plain, plain_tot = score.score_rttm(ref_rows, sys_rows, collar, False, uem, device=DEV, overlapping=overlapping)
    assert {n: {k: v for k, v in r.items() if k not in ('jer', 'jer_ticks')} for n, r in per.items()} == plain
    assert {k: v for k, v in tot.items() if k != 'jer'} == plain_tot


# ---- ES2005a: the sweep against the score command on the files it wrote ---------------------------------------------
GRID = dict(Fa=[0.3, 0.4], Fb=[17.0], loopP=[0.99, 0.5], threshold=[-0.015, 0.2], smoothing=[5.0])   # 31 / 144 clusters


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    rows = [('ES2005a', float(s), float(e - s), str(int(k)))
            for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], z['rttm_ref_labels'])]
    rng = np.random.default_rng(5)                       # seeded second-speaker turns: the reference overlaps
    spk = sorted({r[3] for r in rows})
    span = float(z['seg_times'][:, 1].max())
    rows += [('ES2005a', round(float(a), 2), round(float(d), 2), str(rng.choice(spk)))
             for a, d in zip(rng.uniform(0, span - 3, 40), rng.uniform(0.3, 3.0, 40))]
    return z, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi']), rows


def write_inputs(tmp_path, seg_times, x_raw, transform, plda, rows):
    from vbx_b200 import formats
    keys, seg_lines = [], []
    for i, (s, e) in enumerate(seg_times):
        k = f'ES2005a_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
        keys.append(k)
        seg_lines.append(f'{k} ES2005a {float(s)!r} {float(e)!r}')
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, x_raw)
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    ref = tmp_path / 'ref.rttm'
    ref.write_text(''.join(f'SPEAKER {r[0]} 1 {r[1]:.6f} {r[2]:.6f} <NA> <NA> {r[3]} <NA> <NA>\n' for r in rows))
    return ['--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'), '--xvec-transform',
            str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'), '--lda-dim', '128'], ref


@pytest.mark.parametrize('shift', [0.0, 3000.0])
def test_sweep_jer_equals_the_score_command(es, tmp_path, capsys, shift):
    """shift = 3000 s: there the written RTTM joins equal labels across 10 and 20 ms pauses."""
    z, transform, plda, rows = es
    rows = [(r[0], r[1] + shift, r[2], r[3]) for r in rows]
    seg_times = z['seg_times'] + shift
    if shift:
        lo, hi, join_hi = score.owned_intervals(seg_times)
        assert np.sum(join_hi > hi) == 2
    common, ref = write_inputs(tmp_path, seg_times, z['x_raw'], transform, plda, rows)
    grid = ['--Fa', '0.3,0.4', '--Fb', '17', '--loopP', '0.99,0.5', '--threshold=-0.015,0.2', '--init-smoothing', '5',
            '--ref-rttm', str(ref), '--oracle-overlaps']
    base, out = tmp_path / 'base', tmp_path / 'jer'
    assert sweep.main(['--out-dir', str(base)] + common + grid) == 0
    assert sweep.main(['--out-dir', str(out)] + common + grid + ['--jer']) == 0
    s0 = json.loads((base / 'summary.json').read_text())
    s1 = json.loads((out / 'summary.json').read_text())
    names = [s.name for s in sweep.grid_settings(GRID)]
    assert sorted(s0) == sorted(names + ['ranking', 'ranking_overlap'])        # without --jer: the keys of before
    assert sorted(s1) == sorted(names + ['ranking', 'ranking_overlap', 'ranking_jer', 'ranking_jer_overlap'])
    assert s1['ranking'] == s0['ranking'] and s1['ranking_overlap'] == s0['ranking_overlap']
    for key in ('jer', 'jer_overlap'):
        jers = [s1[n][key]['jer'] for n in s1['ranking_' + key]]
        assert sorted(s1['ranking_' + key]) == sorted(names) and jers == sorted(jers)
    capsys.readouterr()
    for name in names:
        r0, r1 = s0[name]['recordings']['ES2005a'], s1[name]['recordings']['ES2005a']
        assert {k: v for k, v in r1.items() if k not in ('jer', 'jer_overlap')} == r0
        assert {k: v for k, v in s1[name].items() if k not in ('jer', 'jer_overlap', 'recordings')} == \
            {k: v for k, v in s0[name].items() if k != 'recordings'}
        assert (out / name / 'ES2005a.rttm').read_bytes() == (base / name / 'ES2005a.rttm').read_bytes()
        for key, sub, extra in (('jer', out / name, []), ('jer_overlap', out / name / 'overlap', ['--overlapping-system'])):
            n_seg = len((sub / 'ES2005a.rttm').read_text().splitlines())
            argv = ['--ref-rttm', str(ref), '--sys-rttm', str(sub), '--collar', '0.25', '--json', '--jer'] + extra
            assert score.main(argv) == 0
            cli = json.loads(capsys.readouterr().out)['files']['ES2005a']
            mine = r1[key]
            assert [t['R'] for t in cli['jer_ticks']] == [t['R'] for t in mine['ticks']]
            # each written boundary is rounded to 1 us, moving S and I by at most tol ticks: every cost, and so the
            # best mapping's mean, moves by at most 3 tol / R per speaker
            tol = 2 * n_seg + 2
            bound = sum(3.0 * tol / t['R'] for t in mine['ticks']) / len(mine['ticks'])
            assert abs(cli['jer'] - mine['jer']) <= bound, (name, key)


def test_sweep_jer_with_ahc_init_and_item_keys(es):
    z, transform, plda, rows = es
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    grid = dict(GRID, Fa=[0.3], loopP=[0.99])
    out = sweep.sweep_batch(recs, transform, plda, grid, device=DEV, init='AHC', ref_rttm=rows, jer=True)
    t = score.to_ticks
    ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in rows]
    for s, per_rec in out.items():
        item = per_rec['ES2005a']
        assert set(item['der']) == {p for p, _, _ in score.PROTOCOLS} and 'jer_overlap' not in item
        want = jer_ticks(ref, system_segments(z['seg_times'], item['labels'], None, None))
        assert [x['R'] for x in item['jer']['ticks']] == [want['R'][k] for k in sorted(want['R'])]
        for x in item['jer']['ticks']:
            if x['label'] is not None:
                assert x['S'] == want['S'][x['label']]
