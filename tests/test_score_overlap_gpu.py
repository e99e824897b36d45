"""Overlap-aware scoring on the device (vbx_score_overlap through vbx_b200/score.py, DESIGN.md section 5.12): exact tick
equality with the line-sweep oracle (oracle/der_oracle.py) on the segments the project writes, agreement with vbx_score
when there is nothing to add, batch independence, label checks, and the sweep and the command line with overlap
regions on ES2005a."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import der_oracle
from vbx_b200 import VbxError, cli, formats, pipeline, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')


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


def ragged_case(seed, with_uem):
    """The recordings of test_score_gpu's ragged archives (length 1, gaps, none, no reference speech, 1 .. 64 reference
    speakers, up to 4 overlapping) with overlap regions: the reference's own on even recordings, seeded ones on odd;
    entries with 1 .. 200 labels and second labels (None, or with -1 rows)."""
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
        for L in (1, 2, 7, 128, 200):
            lab = sticky(rng, T, L)
            lab2 = None if L == 1 else (lab + sticky(rng, T, L - 1, 0.8) + 1) % L
            if lab2 is not None and L == 7:
                lab2[rng.random(T) < 0.3] = -1
            entries.append((b, lab, lab2))
    return names, segs, ref_rows, recs, ovl, entries, (uem if with_uem else None)


def oracle_entry(n, seg, labels, labels2, overlap, ref_rows, uem, collar, ignore):
    """The oracle on the written segments; -1 second labels say nothing."""
    t = score.to_ticks
    s, e, l = pipeline.overlap_segments(seg, labels, None, overlap)
    sysseg = list(zip(t(s).tolist(), t(e).tolist(), l.tolist()))
    if labels2 is not None:
        timeline = score.owned_intervals(seg)
        end2 = score.effective_hi(timeline, labels2)
        for a, b, k in zip(timeline[0].tolist(), end2.tolist(), labels2.tolist()):
            if k >= 0:
                sysseg += [(max(a, c), min(b, d), k) for c, d in zip(*(v.tolist() for v in overlap)) if min(b, d) > max(a, c)]
    ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows if r[0] == n]
    return der_oracle.der_ticks(ref, sysseg, int(t(collar)), ignore,
                                None if uem is None else [(int(t(a)), int(t(b))) for a, b in uem[n]])


@pytest.mark.parametrize('with_uem', [False, True])
def test_device_equals_oracle_on_ragged_archives(with_uem):
    names, segs, ref_rows, recs, ovl, entries, uem = ragged_case(13 + with_uem, with_uem)
    got = score.score_entries(recs, entries, device=DEV)
    assert any(r.n_ref == 64 for r in recs) and any(len(r.sys_lo) == 1 for r in recs)
    assert any(len(o[0]) for o in ovl[::2]) and any(len(o[0]) for o in ovl[1::2])
    for (b, lab, lab2), res in zip(entries, got):
        n = names[b]
        for p, c, io in score.PROTOCOLS:
            want = oracle_entry(n, segs[n][0], lab, lab2, ovl[b], ref_rows, uem, c, io)
            assert res[p]['ticks'] == want, (n, int(lab.max()) + 1 if len(lab) else 0, p)


def test_written_segments_score_like_the_device():
    """Where no second label is -1, the oracle on pipeline.overlap_segments (what the RTTM holds) is the device's count."""
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(21, False)
    entries = [(b, l, l2) for b, l, l2 in entries if l2 is None or not np.any(l2 < 0)]
    got = score.score_entries(recs, entries, device=DEV)
    t = score.to_ticks
    for (b, lab, lab2), res in zip(entries, got):
        n = names[b]
        s, e, l = pipeline.overlap_segments(segs[n][0], lab, lab2, ovl[b])
        ref = [(int(t(r[1])), int(t(r[1] + r[2])), r[3]) for r in ref_rows if r[0] == n]
        for p, c, io in score.PROTOCOLS:
            want = der_oracle.der_ticks(ref, list(zip(t(s).tolist(), t(e).tolist(), l.tolist())), int(t(c)), io)
            assert res[p]['ticks'] == want, (n, p)


def test_nothing_to_add_equals_vbx_score():
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(15, True)
    single = score.score_entries(recs, [(b, l) for b, l, _ in entries], device=DEV)
    none = [score.prepare_recording(r.name, score.reference_turns(ref_rows).get(r.name, []),
                                    (r.sys_lo, r.sys_hi, r.sys_join_hi), None, overlap=score.overlap_ticks([]))
            for r in recs]
    plain = [score.prepare_recording(r.name, score.reference_turns(ref_rows).get(r.name, []),
                                     (r.sys_lo, r.sys_hi, r.sys_join_hi)) for r in recs]
    single_plain = score.score_entries(plain, [(b, l) for b, l, _ in entries], device=DEV)
    assert score.score_entries(none, [(b, l, l2) for b, l, l2 in entries], device=DEV) == single_plain
    minus = [(b, l, None if l2 is None else np.full(len(l), -1)) for b, l, l2 in entries]
    assert score.score_entries(recs, minus, device=DEV) == single
    assert score.score_entries(recs, [(b, l, None) for b, l, _ in entries], device=DEV) == single


def test_entry_alone_equals_entry_in_batch_and_second_run():
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(16, True)
    batch = score.score_entries(recs, entries, device=DEV)
    assert score.score_entries(recs, entries, device=DEV) == batch
    for i in (0, 13, 14, len(entries) - 1):
        assert score.score_entries(recs, [entries[i]], device=DEV)[0] == batch[i]


def test_bad_second_label_raises():
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(17, False)
    b, lab, lab2 = entries[9]
    i = len(lab2) // 2
    for value in (int(lab[i]), -2):                   # equal to the first label; below -1
        bad = lab2.copy()
        bad[i] = value
        with pytest.raises(VbxError, match=r'entry 1 .*second labels'):
            score.score_entries(recs, [entries[0], (b, lab, bad)], device=DEV)
    with pytest.raises(ValueError, match='all'):
        score.score_entries(recs, [entries[0], (b, lab)], device=DEV)


# ---- ES2005a: the sweep and the command line with overlap regions -----------------------------------------------------
GRID = dict(Fa=[0.3, 0.4], Fb=[17.0], loopP=[0.99, 0.5], threshold=[-0.015, 0.2], smoothing=[5.0])   # 31 / 144 clusters


@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    rows = [('ES2005a', float(s), float(e - s), str(int(k)))
            for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], z['rttm_ref_labels'])]
    rng = np.random.default_rng(5)                       # seeded second-speaker turns: the reference overlaps
    spk = sorted({r[3] for r in rows})
    span = float(z['seg_times'][:, 1].max())
    rows += [('ES2005a', round(float(a), 2), round(float(d), 2), str(rng.choice(spk)))
             for a, d in zip(rng.uniform(0, span - 3, 40), rng.uniform(0.3, 3.0, 40))]
    return z, recs, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi']), rows


def write_inputs(tmp_path, z, transform, plda, rows):
    keys, seg_lines = [], []
    for i, (s, e) in enumerate(z['seg_times']):
        k = f'ES2005a_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
        keys.append(k)
        seg_lines.append(f'{k} ES2005a {float(s)!r} {float(e)!r}')
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, z['x_raw'])
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    ref = tmp_path / 'ref.rttm'
    ref.write_text(''.join(f'SPEAKER {r[0]} 1 {r[1]:.6f} {r[2]:.6f} <NA> <NA> {r[3]} <NA> <NA>\n' for r in rows))
    return ['--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'), '--xvec-transform',
            str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'), '--lda-dim', '128'], ref


def test_sweep_with_oracle_overlaps(es, tmp_path, capsys):
    z, recs, transform, plda, rows = es
    turns = score.reference_turns(rows)['ES2005a']
    assert len(score.oracle_overlaps(turns)[0]) > 10
    common, ref = write_inputs(tmp_path, z, transform, plda, rows)
    grid = ['--Fa', '0.3,0.4', '--Fb', '17', '--loopP', '0.99,0.5', '--threshold=-0.015,0.2', '--init-smoothing', '5',
            '--ref-rttm', str(ref)]
    plain, ovl = tmp_path / 'plain', tmp_path / 'ovl'
    assert sweep.main(['--out-dir', str(plain)] + common + grid) == 0
    assert sweep.main(['--out-dir', str(ovl)] + common + grid + ['--oracle-overlaps']) == 0
    s0 = json.loads((plain / 'summary.json').read_text())
    s1 = json.loads((ovl / 'summary.json').read_text())
    names = [s.name for s in sweep.grid_settings(GRID)]
    assert sorted(s0) == sorted(names + ['ranking'])
    assert sorted(s1) == sorted(names + ['ranking', 'ranking_overlap'])
    assert s1['ranking'] == s0['ranking']
    capsys.readouterr()
    for name in names:
        assert sorted(os.listdir(plain / name)) == ['ES2005a.rttm']
        assert (ovl / name / 'ES2005a.rttm').read_bytes() == (plain / name / 'ES2005a.rttm').read_bytes()
        r0, r1 = s0[name]['recordings']['ES2005a'], s1[name]['recordings']['ES2005a']
        assert r1['der'] == r0['der'] and s1[name]['der'] == s0[name]['der']
        assert {k: v for k, v in r1.items() if k not in ('der_overlap', 'overlap_seconds')} == r0
        assert r1['overlap_seconds'] > 0
        for p, _, _ in score.PROTOCOLS:
            one, two = r0['der'][p]['ticks'], r1['der_overlap'][p]['ticks']
            if p == 'forgiving':
                assert two == one
            else:
                assert two['fa'] == one['fa'] and two['miss'] + two['conf'] <= one['miss'] + one['conf'], (name, p)
        written = (ovl / name / 'overlap' / 'ES2005a.rttm').read_text().splitlines()
        assert written[:len((plain / name / 'ES2005a.rttm').read_text().splitlines())] == \
            (plain / name / 'ES2005a.rttm').read_text().splitlines()
        tol = 2 * len(written) + 2                       # each written boundary is rounded to 1 us
        for p, c, io in score.PROTOCOLS:
            argv = ['--ref-rttm', str(ref), '--sys-rttm', str(ovl / name / 'overlap'), '--collar', str(c), '--json',
                    '--overlapping-system'] + (['--ignore-overlaps'] if io else [])
            assert score.main(argv) == 0
            got = json.loads(capsys.readouterr().out)['files']['ES2005a']['ticks']
            mine = r1['der_overlap'][p]['ticks']
            assert got['scored'] == mine['scored']
            for k in ('miss', 'fa', 'conf'):
                assert abs(got[k] - mine[k]) <= tol, (name, p, k)
    for p, _, _ in score.PROTOCOLS:
        ders = [s1[n]['der_overlap'][p]['der'] for n in s1['ranking_overlap'][p]]
        assert ders == sorted(ders)
    assert any(s1[n]['der_overlap']['full']['der'] < s1[n]['der']['full']['der'] for n in names)


def test_command_line_writes_overlap_aware_rttm(es, tmp_path):
    z, recs, transform, plda, rows = es
    common, _ = write_inputs(tmp_path, z, transform, plda, rows)
    osd = tmp_path / 'osd.rttm'
    osd.write_text('SPEAKER ES2005a 1 20.000 15.500 <NA> <NA> ovl <NA> <NA>\n'
                   'SPEAKER ES2005a 1 30.000 12.000 <NA> <NA> other <NA> <NA>\n'
                   'SPEAKER ES2005a 1 120.250 40.000 <NA> <NA> ovl <NA> <NA>\n'
                   'SPEAKER IS1009a 1 0.0 1.0 <NA> <NA> ovl <NA> <NA>\n')
    argv = ['--init', 'AHC+VB', '--threshold', '-0.015', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99'] + common
    assert cli.main(argv + ['--out-rttm-dir', str(tmp_path / 'a')]) == 0
    assert cli.main(argv + ['--out-rttm-dir', str(tmp_path / 'b'), '--overlap-rttm', str(osd)]) == 0
    out = pipeline.diarize_batch(recs, transform, plda, 0.3, 17.0, 0.99, threshold=-0.015)
    plain = (tmp_path / 'a' / 'ES2005a.rttm').read_bytes()
    assert plain == ''.join(line + os.linesep for line in out['ES2005a']['rttm']).encode()
    assert set(out['ES2005a']) == {'rttm', 'labels', 'labels2nd', 'iterations', 'n_speakers', 'rttm2nd'}
    ovl = pipeline.diarize_batch(recs, transform, plda, 0.3, 17.0, 0.99, threshold=-0.015,
                                 overlaps=score.read_overlaps(str(osd)))['ES2005a']
    assert ovl['overlap_seconds'] == pytest.approx(22.0 + 40.0)
    written = (tmp_path / 'b' / 'ES2005a.rttm').read_text()
    assert written == ''.join(line + os.linesep for line in ovl['rttm_overlap'])
    lines = written.splitlines()
    n1 = len(out['ES2005a']['rttm'])
    assert lines[:n1] == out['ES2005a']['rttm'] and len(lines) > n1
    for line in lines[n1:]:
        a, d = float(line.split()[3]), float(line.split()[4])
        assert (20.0 <= a and a + d <= 42.0 + 1e-6) or (120.25 <= a and a + d <= 160.25 + 1e-6)
