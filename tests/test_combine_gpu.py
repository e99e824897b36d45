"""Combination of diarizations on the device (DESIGN.md section 5.21): vbx_combine through combine.combine_labels against
oracle/dover_oracle.py bit for bit on seeded ragged batches, batch independence, the global-label limit, the C ABI's
argument errors, combine_rttm against combine_labels on the common timeline, and sweep --combine."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import dover_oracle
from vbx_b200 import _lib, combine, formats, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')


def _batch(seed, K, n_lab, lens, bad=False):
    """Ragged recordings whose hypotheses are noisy relabelled copies of a sticky truth, with second labels, silent
    intervals and (bad=True) bad labels."""
    rng = np.random.default_rng(seed)
    intervals, hyps = [], [[] for _ in range(K)]
    for T in lens:
        d = rng.integers(0, 400_000, T)                       # some empty intervals
        gap = rng.integers(0, 50_000, T) * (rng.random(T) < 0.2)
        lo = np.cumsum(np.concatenate([[0], (d + gap)[:-1]])).astype(np.int64) if T else np.zeros(0, dtype=np.int64)
        intervals.append((lo, lo + d))
        n_true = int(rng.integers(1, n_lab + 1))
        truth = np.repeat(rng.integers(0, n_true, T // 7 + 1), 7)[:T]
        for k in range(K):
            n = int(rng.integers(n_true, n_lab + 1))
            l1 = rng.permutation(n)[truth]
            flip = rng.random(T) < rng.uniform(0.02, 0.3)
            l1[flip] = rng.integers(0, n, int(flip.sum()))
            l1[rng.random(T) < 0.1] = -1
            l2 = np.where((rng.random(T) < 0.15) & (l1 >= 0), (l1 + rng.integers(1, max(n, 2), T)) % max(n, 2), -1)
            l2[l2 >= n] = -1
            l2[l2 == l1] = -1
            if bad and T:
                i = rng.integers(0, T, 3)
                l2[i[0]] = l1[i[0]] if l1[i[0]] >= 0 else 0   # equal to the first, or a second without a first
                l1[i[1]], l2[i[1]] = -1, 0
            hyps[k].append((l1, l2))
    return intervals, hyps


def _compare(intervals, hyps, weights=None, bad=False):
    got = combine.combine_labels(intervals, hyps, weights, DEV, strict=False, blocks=True)
    K = len(hyps)
    for b, (g, (lo, hi)) in enumerate(zip(got, intervals)):
        l1 = np.stack([hyps[k][b][0] for k in range(K)]) if len(lo) else np.zeros((K, 0), dtype=np.int64)
        l2 = np.stack([hyps[k][b][1] for k in range(K)]) if len(lo) else np.zeros((K, 0), dtype=np.int64)
        n_labels = [max(int(max(hyps[k][b][0].max(initial=-1), hyps[k][b][1].max(initial=-1))) + 1, 0) for k in range(K)]
        want = dover_oracle.combine(lo, hi, l1, l2, n_labels, weights)
        assert g['flags'] == want['flags'], b
        for pr, blk in want['O'].items():
            assert np.array_equal(g['O'][pr], blk), (b, pr)
        for k in range(K):
            assert np.array_equal(g['L'][k], want['L'][k]), (b, k)
        assert np.array_equal(g['D'], want['D']) and np.array_equal(g['D'], g['D'].T), b
        assert g['order'] == want['order'], b
        assert np.array_equal(g['weights'], want['weights']), b          # bit for bit
        # every assignment reaches scipy's total on the costs the earlier maps give, and is scipy's where that is unique
        mapped, ng = {g['order'][0]: g['map'][g['order'][0]]}, int((want['L'][g['order'][0]] > 0).sum())
        assert np.array_equal(mapped[g['order'][0]], want['map'][g['order'][0]])
        for r in range(1, K):
            h = g['order'][r]
            C = np.zeros((n_labels[h], ng), dtype=np.int64)
            for q, m in mapped.items():
                blk = want['O'][(h, q)] if h < q else want['O'][(q, h)].T
                for u, gid in enumerate(m):
                    if gid >= 0:
                        C[:, gid] += blk[:, u]
            col, total, unique = dover_oracle.assign(C)
            m = g['map'][h]
            old = np.nonzero((m >= 0) & (m < ng))[0]
            assert len(set(m[old].tolist())) == len(old) and np.all(C[old, m[old]] > 0), (b, r)
            assert int(C[old, m[old]].sum()) == total, (b, r)
            if unique:
                assert np.array_equal(np.where((m >= 0) & (m < ng), m, -1), col), (b, r)
            fresh = np.nonzero(m >= ng)[0]
            assert np.array_equal(m[fresh], ng + np.arange(len(fresh))), (b, r)
            assert np.array_equal(m < 0, (want['L'][h] <= 0)), (b, r)
            mapped[h] = m
            ng += len(fresh)
        assert g['n_global'] == ng
        if all(want['unique']):
            assert np.array_equal(g['labels'], want['labels']) and np.array_equal(g['labels2'], want['labels2']), b
    return got


@pytest.mark.parametrize('K,n_lab', [(2, 3), (3, 6), (8, 12), (32, 5), (3, 128)])
def test_against_the_oracle(K, n_lab):
    lens = [60, 0, 131, 7, 300, 1, 0, 45] if n_lab < 128 else [900, 0, 400]
    intervals, hyps = _batch(K * 1000 + n_lab, K, n_lab, lens)
    _compare(intervals, hyps)
    _compare(intervals, hyps, weights=np.linspace(1.0, 0.3, K))
    intervals, hyps = _batch(K * 1000 + n_lab + 1, K, n_lab, lens, bad=True)
    got = _compare(intervals, hyps, bad=True)
    assert any(g['flags'] & _lib.COMBINE_BAD_LABEL for g in got)
    with pytest.raises(_lib.VbxError, match='second label'):
        combine.combine_labels(intervals, hyps, device=DEV)


def test_a_recording_alone_and_inside_a_batch():
    intervals, hyps = _batch(5, 8, 9, [200, 33, 0, 512, 90])
    whole = combine.combine_labels(intervals, hyps, device=DEV, blocks=True)
    for b in range(len(intervals)):
        alone = combine.combine_labels([intervals[b]], [[h[b]] for h in hyps], device=DEV, blocks=True)[0]
        for key in ('labels', 'labels2', 'weights', 'D'):
            assert np.array_equal(alone[key], whole[b][key]), (b, key)
        assert alone['order'] == whole[b]['order'] and alone['n_global'] == whole[b]['n_global']
        assert all(np.array_equal(x, y) for x, y in zip(alone['map'], whole[b]['map']))


def test_too_many_global_labels_are_flagged():
    T = 128 * 3
    lo = np.arange(T, dtype=np.int64) * 1000
    i = np.arange(T)
    a = np.where(i % 3 == 0, i // 3, -1)                                  # 128 labels
    b = np.where((i % 3 == 1) & (i // 3 < 127), i // 3, -1)               # 127 that share no time with them: 255 in all
    c = np.where(i % 3 == 2, 0, -1)                                       # and one more
    hyps = [[(a, None)], [(b, None)], [(c, None)]]
    got = combine.combine_labels([(lo, lo + 1000)], hyps, device=DEV, strict=False)[0]
    assert got['flags'] == _lib.COMBINE_TOO_MANY_LABELS and got['n_global'] == 0
    assert np.all(got['labels'] == -1) and np.all(got['labels2'] == -1)
    with pytest.raises(_lib.VbxError, match='255 global labels'):
        combine.combine_labels([(lo, lo + 1000)], hyps, device=DEV)
    ok = combine.combine_labels([(lo, lo + 1000)], hyps[:2], device=DEV)[0]
    assert ok['n_global'] == 255 and ok['flags'] == 0


def test_argument_errors():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    try:
        need = ctypes.c_size_t()
        for n_rec, K, ML in ((-1, 2, 4), (1, 1, 4), (1, 33, 4), (1, 2, 0), (1, 2, 129), (1 << 30, 32, 4)):
            assert lib.vbx_combine_workspace_bytes(h, n_rec, K, ML, ctypes.byref(need)) == -1, (n_rec, K, ML)
        assert lib.vbx_combine_workspace_bytes(h, 2, 3, 4, ctypes.byref(need)) == 0 and need.value > 0
        ws = torch.empty(need.value, dtype=torch.uint8, device=DEV)
        z64 = torch.zeros(64, dtype=torch.int64, device=DEV)
        z32 = torch.zeros(4096, dtype=torch.int32, device=DEV)
        d64 = torch.zeros(64, dtype=torch.int64, device=DEV)
        o32 = [torch.zeros(4096, dtype=torch.int32, device=DEV) for _ in range(6)]
        zd = torch.zeros(64, dtype=torch.float64, device=DEV)
        off = torch.tensor([0, 2, 4], dtype=torch.int64, device=DEV)
        nl = np.full((2, 3), 2, dtype=np.int32)
        p = lambda t: ctypes.c_void_p(t.data_ptr())

        def call(n_rec=2, K=3, N=4, ML=4, n_labels=nl, weights=None, wsp=p(ws), size=need.value, offsets=p(off),
                 order=p(o32[2])):
            w = None if weights is None else np.asarray(weights, dtype=np.float64).ctypes.data_as(ctypes.c_void_p)
            return lib.vbx_combine(h, n_rec, offsets, N, p(z64), p(z64), K, p(z32), p(z32),
                                   n_labels.ctypes.data_as(ctypes.c_void_p), ML, w, wsp, size, p(o32[0]), p(o32[1]), order,
                                   p(zd), p(d64), p(o32[3]), p(o32[4]), p(o32[5]), None, None, None)

        assert call() == 0
        torch.cuda.synchronize()
        for bad in (dict(K=1), dict(K=33), dict(n_rec=-1), dict(N=-1), dict(ML=0), dict(ML=1), dict(weights=[1, 0, 1]),
                    dict(weights=[1, float('nan'), 1]), dict(weights=[1, float('inf'), 1]), dict(weights=[1, -2, 1]),
                    dict(size=need.value - 1), dict(wsp=ctypes.c_void_p(ws.data_ptr() + 8)), dict(offsets=None),
                    dict(order=None), dict(n_labels=np.full((2, 3), -1, dtype=np.int32))):
            assert call(**bad) == -1, bad
            assert lib.vbx_last_error(h)
    finally:
        lib.vbx_destroy(h)


def _rttm(rows):
    return ''.join(f'SPEAKER {r[0]} 1 {r[1]:.6f} {r[2]:.6f} <NA> <NA> {r[3]} <NA> <NA>\n' for r in rows)


def test_combine_rttm_is_combine_labels_on_the_common_timeline(tmp_path, capsys):
    rng = np.random.default_rng(3)
    arch = synth.make_scoring_archive([300, 180, 240], seed=4, gap_prob=0.05)
    from vbx_b200.pipeline import merge_adjacent_labels
    hyp_rows = []
    for k in range(3):
        rows = []
        for n, (seg, lab) in arch.items():
            if k == 2 and n == list(arch)[1]:
                continue                                       # this hypothesis lacks the recording
            sysl = rng.permutation(int(lab.max()) + 1)[lab]
            flip = rng.random(len(lab)) < 0.1
            sysl[flip] = rng.integers(0, int(lab.max()) + 1, int(flip.sum()))
            s, e, l = merge_adjacent_labels(seg[:, 0] + 0.01 * k, seg[:, 1] + 0.01 * k, sysl)
            rows += [(n, float(a), float(z - a), f'h{k}s{x}') for a, z, x in zip(s, e, l)]
            rows.append((n, float(s[3]), float(e[3] - s[3]) / 2, f'h{k}extra'))         # a second speaker
        hyp_rows.append(rows)
        (tmp_path / f'h{k}.rttm').write_text(_rttm(rows))
    names, intervals, hyps = combine.common_timeline(hyp_rows)
    want = combine.combine_labels(intervals, hyps, device=DEV)
    got = combine.combine_rttm([str(tmp_path / f'h{k}.rttm') for k in range(3)], device=DEV)
    assert list(got) == names == sorted(arch)
    for n, w in zip(names, want):
        assert np.array_equal(got[n]['labels'], w['labels']) and np.array_equal(got[n]['labels2'], w['labels2'])
        assert got[n]['order'] == w['order'] and np.array_equal(got[n]['D'], w['D'])
    argv = ['--sys-rttm'] + [str(tmp_path / f'h{k}.rttm') for k in range(3)] + ['--out-rttm-dir', str(tmp_path / 'out'),
                                                                                 '--json', '--weights', '1,0.9,0.8']
    assert combine.main(argv) == 0
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    weighted = combine.combine_rttm(hyp_rows, [1, 0.9, 0.8], device=DEV)
    for n in names:
        assert printed[n]['weights'] == [1.0, 0.9, 0.8] and printed[n]['order'] == weighted[n]['order']
        assert (tmp_path / 'out' / f'{n}.rttm').read_text().splitlines() == weighted[n]['rttm']
    # the combination of a hypothesis with itself and a renamed copy is that hypothesis
    same = combine.combine_rttm([hyp_rows[0], hyp_rows[0], [(r[0], r[1], r[2], 'x' + r[3]) for r in hyp_rows[0]]],
                                device=DEV)
    for n in same:
        assert not same[n]['D'].any()
        ref = [r for r in hyp_rows[0] if r[0] == n]
        per, tot = score.score_rttm(ref, [(n,) + tuple(float(x) for x in l.split()[3:5]) + (l.split()[7],)
                                          for l in same[n]['rttm']], 0.0, False, overlapping=True, device=DEV)
        assert tot['der'] == 0.0


GRID = dict(Fa=[0.3, 0.5], Fb=[17.0], loopP=[0.99, 0.9], threshold=[-0.015], smoothing=[5.0])


def test_sweep_combine_command_line(tmp_path):
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    transform, plda = (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])
    recs, rows, _ = synth.multi_session_archive(z['x_raw'], n_rec=3, seed=6)
    keys, seg_lines, xs = [], [], []
    for name, (x, seg) in recs.items():
        for i, (s, e) in enumerate(seg):
            keys.append(f'{name}_{i:04d}')
            seg_lines.append(f'{keys[-1]} {name} {float(s)!r} {float(e)!r}')
        xs.append(x)
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, np.concatenate(xs))
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    (tmp_path / 'ref.rttm').write_text(_rttm(rows))
    base = ['--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'), '--xvec-transform',
            str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'), '--lda-dim', '128', '--Fa',
            '0.3,0.5', '--Fb', '17', '--loopP', '0.99,0.9', '--threshold=-0.015', '--ref-rttm', str(tmp_path / 'ref.rttm'),
            '--jer']
    assert sweep.main(['--out-dir', str(tmp_path / 'plain')] + base) == 0
    plain = json.loads((tmp_path / 'plain' / 'summary.json').read_text())
    for how, n_hyp in (('all', 4), ('3', 3)):
        out = tmp_path / f'c{how}'
        assert sweep.main(['--out-dir', str(out), '--combine', how] + base) == 0
        summary = json.loads((out / 'summary.json').read_text())
        comb = summary.pop('combined')
        assert summary == plain
        assert len(comb['hypotheses']) == n_hyp and set(comb['hypotheses']) <= set(plain) - {'ranking', 'ranking_jer'}
        if how == '3':
            assert comb['hypotheses'] == plain['ranking']['full'][:3]
        assert sorted(comb['recordings']) == sorted(recs)
        sys_rows = score.read_rttm_path(str(out / 'combined'))
        for p, c, io in score.PROTOCOLS:
            _, tot = score.score_rttm(rows, sys_rows, c, io, device=DEV, jer=True)
            assert comb['der'][p] == json.loads(json.dumps({k: v for k, v in tot.items() if k != 'jer'})), p
        assert comb['jer']['jer'] == tot['jer']
    with pytest.raises(SystemExit):
        sweep.main(['--out-dir', str(tmp_path / 'bad'), '--combine', '2'] + [a for a in base if a not in
                                                                              ('--ref-rttm', str(tmp_path / 'ref.rttm'), '--jer')])
