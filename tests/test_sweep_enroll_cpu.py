"""Enrolment and cohort normalisation inside the sweep (DESIGN.md section 5.19) without a GPU: the argument checks of
sweep_batch before any device work, threshold lists, summarize_by_name on hand-built blocks against a direct
restatement of the name-level DER, stable rankings, greedy packing by batch workspace, threshold names, and the argument
checks of enroll_many and of the command line.  The batched assignment against oracle/enroll_oracle.py, looped over
problems and thresholds, is in tests/test_sweep_enroll_gpu.py (it needs the device's LLRs)."""
import numpy as np
import pytest

from vbx_b200 import enroll, score, sweep
from vbx_b200.sweep import Setting

GRID = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
REC = {'r': (np.zeros((3, 256)), np.zeros((3, 2)))}
ENR = {'alice': np.zeros((2, 256)), 'bob': np.zeros((1, 256))}
COH = {'c1': np.zeros((1, 256)), 'c2': np.zeros((1, 256))}


@pytest.mark.parametrize('kw, msg', [
    (dict(enroll=ENR, enroll_thresholds=[]), 'at least one'),
    (dict(enroll=ENR, enroll_thresholds=[0.0, float('nan')]), 'enrolment threshold'),
    (dict(enroll=ENR, enroll_thresholds=[2e15]), 'enrolment threshold'),
    (dict(enroll=ENR), 'no default'),
    (dict(enroll_thresholds=[0.0]), 'without enroll'),
    (dict(cohort=COH), 'needs link_thresholds or enroll'),
    (dict(enroll={'unknown-1': np.zeros((1, 256))}, enroll_thresholds=[0.0]), 'reserved'),
    (dict(enroll={'a': np.zeros((1, 8))}, enroll_thresholds=[0.0]), 'dimension'),
    (dict(enroll=ENR, enroll_thresholds=[0.0], cohort={'c1': np.zeros((1, 256))}), 'at least 2'),
    (dict(enroll=ENR, enroll_thresholds=[0.0], cohort=COH, cohort_top=1), 'top_k'),
    (dict(link_thresholds=[0.0], cohort={'c1': np.zeros((1, 256)), 'c2': np.zeros((1, 7))}), 'dimension'),
])
def test_argument_errors_before_device_work(kw, msg):
    with pytest.raises(ValueError, match=msg):
        sweep.sweep_batch(REC, None, None, GRID, **kw)


def test_thresholds_are_deduplicated_in_order():
    assert enroll.check_thresholds([20, -10, 20.0, 0, -10]) == [20.0, -10.0, 0.0]
    assert sweep.check_enroll_options(None, None, 256) == (None, None)
    enrolled, thr = sweep.check_enroll_options(ENR, [40, 40, -1e15], 256)
    assert [k for k, _ in enrolled] == ['alice', 'bob'] and thr == [40.0, -1e15]


def _by_name(tot, ref_names, sys_names, blocks):
    """The name-level DER restated: every cell whose reference and system names agree counts as matched."""
    matched = 0
    for rk, sk, blk in zip(ref_names, sys_names, blocks):
        for i, r in enumerate(rk):
            for j in range(min(blk.shape[1], len(sk))):
                if sk[j] == r:
                    matched += int(blk[i, j])
    t = tot['ticks']
    return score.result(t['miss'], t['fa'], t['scored'] - t['miss'] - matched, t['scored'])


def _fake_out(rng, with_overlap):
    """Two settings over three files with random blocks, per-setting names at two thresholds (names that repeat across
    files, unknown speakers, a label without turns)."""
    s1, s2 = Setting(0.3, 17.0, 0.99, -0.015, 5.0), Setting(0.5, 17.0, 0.99, -0.015, 5.0)
    pool = ['p0', 'p1', 'p2', 'p3']
    out = {}
    for s in (s1, s2):
        out[s] = {}
        for f in range(3):
            rk = list(rng.choice(pool, int(rng.integers(1, 4)), replace=False))
            n = int(rng.integers(1, 4))
            item = dict(ref_speakers=rk)
            for key in ('der', 'der_overlap') if with_overlap else ('der',):
                item[key + '_blocks'] = {p: rng.integers(0, 50, (len(rk), n)).astype(np.int64)
                                         for p, _, _ in score.PROTOCOLS}
                item[key] = {p: score.result(*rng.integers(0, 30, 3), 400) for p, _, _ in score.PROTOCOLS}
            names = {}
            for t in (0.0, 20.0):
                names[t] = {l: (str(rng.choice(pool)) if rng.random() < 0.6 else f'unknown-f{f}-{l + 1}')
                            for l in range(n - 1)}        # the last label has no name: its column counts nothing
                names[t] = {l: v if list(names[t].values()).count(v) == 1 else f'unknown-f{f}-{l + 1}'
                            for l, v in names[t].items()}
            item['speaker_names'] = names
            out[s][f'f{f}'] = item
    return s1, s2, out


@pytest.mark.parametrize('seed', range(6))
@pytest.mark.parametrize('with_overlap', [False, True])
def test_summarize_by_name_equals_the_name_level_der(seed, with_overlap):
    rng = np.random.default_rng(seed)
    _, _, out = _fake_out(rng, with_overlap)
    for key in ('der', 'der_overlap') if with_overlap else ('der',):
        tot, ranking = sweep.summarize_by_name(out, key)
        assert len(tot) == 4
        for s, per_rec in out.items():
            items = list(per_rec.values())
            for t in (0.0, 20.0):
                for p, _, _ in score.PROTOCOLS:
                    sys_names = [[it['speaker_names'][t].get(l, f'unknown-{rec}-{l + 1}')
                                  for l in range(it[key + '_blocks'][p].shape[1])] for rec, it in per_rec.items()]
                    want = _by_name(score.overall([it[key][p] for it in items]), [it['ref_speakers'] for it in items],
                                    sys_names, [it[key + '_blocks'][p] for it in items])
                    assert tot[sweep.enroll_key(s, t)][p] == want
                    # by_name DER is at least the DER across files of the same names (no assignment to help)
                    assert want['ticks']['conf'] >= score.across_files_result(
                        score.overall([it[key][p] for it in items]), [it['ref_speakers'] for it in items],
                        sys_names, [it[key + '_blocks'][p] for it in items])['ticks']['conf']
        for p, _, _ in score.PROTOCOLS:
            assert sorted(ranking[p]) == sorted(tot)


def test_ranking_ties_keep_grid_then_threshold_order():
    s1, s2, out = _fake_out(np.random.default_rng(1), False)
    for per_rec in out.values():                      # every name unknown: every entry scores the same
        for it in per_rec.values():
            it['speaker_names'] = {t: {l: f'unknown-x{id(it)}-{l}' for l in m} for t, m in it['speaker_names'].items()}
        for i, it in enumerate(per_rec.values()):
            it['der'] = {p: score.result(1, 1, 0, 100) for p, _, _ in score.PROTOCOLS}
            it['ref_speakers'] = list(out[s1][f'f{i}']['ref_speakers'])
            it['der_blocks'] = {p: np.zeros_like(b) for p, b in out[s1][f'f{i}']['der_blocks'].items()}
    tot, ranking = sweep.summarize_by_name(out)
    order = [sweep.enroll_key(s, t) for s in (s1, s2) for t in (0.0, 20.0)]
    assert list(tot) == order
    assert all(ranking[p] == order for p, _, _ in score.PROTOCOLS)
    assert sweep.enroll_key(s1, -10.0) == 'Fa0.3_Fb17_loopP0.99_thr-0.015_sm5_enroll-10'


def test_pack_by_keeps_order_and_budget():
    sizes = [5, 1, 7, 3, 3, 9]
    size_of = lambda idx: sum(sizes[i] for i in idx) + 4 * max(sizes[i] for i in idx)   # not a plain sum
    for budget in (45, 60, 100):                     # the largest entry alone needs 9 + 4 * 9
        batches = sweep.pack_by(len(sizes), size_of, budget)
        assert sum(batches, []) == list(range(len(sizes)))
        assert all(size_of(b) <= budget for b in batches)
    assert sweep.pack_by(3, size_of, None) == [[0, 1, 2]] and sweep.pack_by(0, size_of, 10) == []
    with pytest.raises(ValueError, match='max_batch_bytes'):
        sweep.pack_by(len(sizes), size_of, 44)


@pytest.mark.parametrize('flags', [['--enroll-ark', 'e.ark'], ['--enroll-utt2spk', 'e.utt2spk'],
                                   ['--cohort-ark', 'c.ark'], ['--cohort-utt2spk', 'c.utt2spk']])
def test_command_line_pairs_go_together(flags, capsys):
    req = ['--out-dir', 'o', '--xvec-ark-file', 'a', '--segments-file', 's', '--xvec-transform', 't', '--plda-file', 'p',
           '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99', '--threshold=-0.015',
           '--enroll-threshold=-10,0']
    with pytest.raises(SystemExit):
        sweep.main(req + flags)
    assert 'go together' in capsys.readouterr().err


def test_sweep_thresholds_with_the_same_name_are_refused():
    with pytest.raises(ValueError, match='same name'):
        sweep.check_enroll_options(ENR, [1.0, 1.0000001], 256)   # both _enroll1 in enroll_key and summary.json
    with pytest.raises(ValueError, match='same name'):
        sweep.sweep_batch(REC, None, None, GRID, enroll=ENR, enroll_thresholds=[0.5, 0.50000001])
    assert sweep.check_enroll_options(ENR, [1.0, 1.00001], 256)[1] == [1.0, 1.00001]
    assert enroll.check_thresholds([1.0, 1.0000001]) == [1.0, 1.0000001]   # enroll_many keys by position


@pytest.mark.parametrize('kw, msg', [
    (dict(thresholds=[]), 'at least one'),
    (dict(norm=[(np.zeros(1), np.ones(1), np.zeros(2), np.ones(2))]), 'norm must hold'),
    (dict(enroll_speaker=[0, 2]), 'every enrolled speaker'),
])
def test_enroll_many_argument_errors_before_device_work(kw, msg):
    args = dict(fea=np.zeros((3, 4)), Phi=np.ones(4), offsets=[0, 3], labels_per_problem=[[np.array([0, 0, 1])]],
                enroll_fea=np.zeros((2, 4)), enroll_speaker=[0, 1], Fa=0.3, Fb=17.0, thresholds=[0.0])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        enroll.enroll_many(**args)
