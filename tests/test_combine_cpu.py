"""Combination of diarizations without a device (DESIGN.md section 5.21): the hand-worked cases of the section on
oracle/dover_oracle.py, combine.common_timeline, every ValueError of combine.py and sweep.combine_settings, the command
lines' parsing, and the C ABI's refusal of a null handle."""
import ctypes

import numpy as np
import pytest

from oracle import dover_oracle
from vbx_b200 import combine, sweep

SEC = 1_000_000


def _run(labels, labels2=None, weights=None, dur=None):
    l1 = np.asarray(labels, dtype=np.int64)
    l2 = np.full_like(l1, -1) if labels2 is None else np.asarray(labels2, dtype=np.int64)
    T = l1.shape[1]
    d = np.full(T, SEC, dtype=np.int64) if dur is None else np.asarray(dur, dtype=np.int64) * SEC
    lo = np.concatenate([[0], np.cumsum(d)[:-1]])
    n = [int(max(a.max(), b.max())) + 1 for a, b in zip(l1, l2)]
    return dover_oracle.combine(lo, lo + d, l1, l2, n, weights)


def test_swapped_names_give_the_anchor_back():
    r = _run([[0, 0, 1, 1, -1, 2], [1, 1, 0, 0, -1, 2]])
    assert r['order'] == [0, 1] and not r['D'].any()
    assert r['labels'].tolist() == [0, 0, 1, 1, -1, 2] and np.all(r['labels2'] == -1)
    assert r['map'][1].tolist() == [1, 0, 2] and r['n_global'] == 3
    assert r['weights'].tolist() == [1.0, 2.0 ** -0.1]


def test_one_dissenter_of_three_loses():
    r = _run([[0, 0, 1, 1], [0, 0, 1, 1], [0, 1, 1, 1]])
    # D: the dissenter is 2 s of confusion-twice away from each of the others
    assert r['D'].tolist() == [[0, 0, 2 * SEC], [0, 0, 2 * SEC], [2 * SEC, 2 * SEC, 0]]
    assert r['order'] == [0, 1, 2] and r['labels'].tolist() == [0, 0, 1, 1]
    assert r['weights'].tolist() == [1.0, 2.0 ** -0.1, 3.0 ** -0.1]


def test_an_extra_speaker_gets_a_new_id_and_wins_only_unopposed():
    #            both others silent | others say 0 | others split
    r = _run([[-1, 0, 0, 0], [-1, 0, 0, 1], [2, 2, 0, 1]], weights=[1.0, 1.0, 1.5])
    assert r['map'][2].tolist() == [0, 1, 2] and r['n_global'] == 3
    # interval 0: count vote floor(0.5 + 1.5 / 3.5) = 0 -> silence although only label 2 is said
    # interval 1: 0 has 2.0 against 2's 1.5; interval 3: labels 0 (1.0) and 1 (2.5)
    assert r['labels'].tolist() == [-1, 0, 0, 1]
    r = _run([[-1, 0, 0, 0], [-1, 0, 0, 1], [2, 2, 0, 1]], weights=[1.0, 1.0, 2.5])
    assert r['labels'].tolist() == [2, 2, 0, 1]                   # outvoted by weight: 2.5 against 2.0


def test_count_vote():
    one = _run([[0, 0], [0, 0], [0, 0]], [[-1, -1], [-1, -1], [1, -1]], weights=[1, 1, 1])
    assert one['labels'].tolist() == [0, 0] and one['labels2'].tolist() == [-1, -1]       # counts 1, 1, 2 -> 1
    two = _run([[0, 0], [0, 0], [0, 0]], [[1, -1], [1, -1], [-1, -1]], weights=[1, 1, 1])
    assert two['labels'].tolist() == [0, 0] and two['labels2'].tolist() == [1, -1]        # counts 2, 2, 1 -> 2


def test_ties_go_to_the_lower_id():
    r = _run([[0, 1, 0], [0, 1, 1]], weights=[1, 1], dur=[5, 5, 1])
    assert r['D'][0, 1] == 2 * SEC and r['order'] == [0, 1]       # equal row sums: the lower index is the anchor
    assert r['labels'].tolist() == [0, 1, 0]                       # interval 2: 0 and 1 tie at weight 1


def test_D_is_symmetric_and_zero_up_to_renaming():
    rng = np.random.default_rng(0)
    l = rng.integers(-1, 5, (4, 200))
    l[1] = np.where(l[0] >= 0, (l[0] + 2) % 5, -1)
    l2 = np.where((rng.random((4, 200)) < 0.2) & (l >= 0), (l + 1) % 5, -1)
    l2[1] = np.where(l2[0] >= 0, (l2[0] + 2) % 5, -1)
    r = _run(l, l2, dur=rng.integers(0, 4, 200))
    assert np.array_equal(r['D'], r['D'].T) and r['D'][0, 1] == 0 and not np.diag(r['D']).any()
    assert r['D'][0, 2] > 0 and np.array_equal(r['D'][0], r['D'][1])
    assert r['order'][0] in (0, 1)
    # miss + false alarm + twice the confusion: here 3 s of one-sided speech and 2 s of confusion
    assert _run([[0, 0, -1, 1, 1], [0, -1, 0, 0, 1]], dur=[1, 1, 2, 2, 1])['D'][0, 1] == (3 + 2 * 2) * SEC


def test_bad_labels_are_ignored_and_flagged():
    r = _run([[0, 0, 1], [0, 1, 1]], [[-1, 0, -1], [-1, -1, -1]])
    assert r['flags'] == dover_oracle.BAD_LABEL and r['L'][0].tolist() == [SEC, SEC]
    assert _run([[0, -1], [0, 0]], [[-1, 0], [-1, -1]])['flags'] == dover_oracle.BAD_LABEL


def test_common_timeline():
    a = [('r1', 0.0, 2.0, 'x'), ('r1', 2.0, 2.0, 'y'), ('r2', 1.0, 1.0, 'x')]
    b = [('r1', 0.5, 2.0, 'p'), ('r1', 1.5, 1.0, 'q'), ('r1', 6.0, 1.0, 'p')]
    names, intervals, hyps = combine.common_timeline([a, b])
    assert names == ['r1', 'r2']
    lo, hi = intervals[0]
    assert (lo / 1e6).tolist() == [0.0, 0.5, 1.5, 2.0, 2.5, 6.0] and (hi / 1e6).tolist() == [0.5, 1.5, 2.0, 2.5, 4.0, 7.0]
    assert hyps[0][0][0].tolist() == [0, 0, 0, 1, 1, -1] and hyps[0][0][1].tolist() == [-1] * 6
    assert hyps[1][0][0].tolist() == [-1, 0, 0, 0, -1, 0] and hyps[1][0][1].tolist() == [-1, -1, 1, 1, -1, -1]
    assert hyps[1][1][0].tolist() == [-1] and hyps[0][1][0].tolist() == [0]           # r2 is silent in b
    with pytest.raises(ValueError, match=r"'r1'.*3 system speakers at 1\.5"):
        combine.common_timeline([a, b + [('r1', 1.5, 0.2, 'z')]])
    lines = combine.combined_lines('r1', lo, hi, [0, 0, 0, 1, -1, 1], [-1, -1, 2, 2, -1, -1])
    assert [l.split()[3:5] + [l.split()[7]] for l in lines] == [['0.000000', '2.000000', '1'], ['2.000000', '0.500000', '2'],
                                                                ['6.000000', '1.000000', '2'], ['1.500000', '1.000000', '3']]


def test_value_errors():
    iv = [(np.array([0, 10]), np.array([10, 20]))]
    h = [(np.array([0, 1]), None)]
    for bad, match in ((dict(hypotheses=[h]), '2 .. 32'), (dict(hypotheses=[h] * 33), '2 .. 32'),
                       (dict(weights=[1.0]), '1 weights for 2'), (dict(weights=[1.0, 0.0]), 'finite and > 0'),
                       (dict(weights=[1.0, float('nan')]), 'finite and > 0'),
                       (dict(hypotheses=[h, [(np.array([0]), None)]]), '1 labels for 2 intervals'),
                       (dict(hypotheses=[h, [(np.array([0, 128]), None)]]), r'\[-1, 128\)'),
                       (dict(hypotheses=[h, [(np.array([0, -2]), None)]]), r'\[-1, 128\)'),
                       (dict(hypotheses=[h, h + h]), 'all 1 recordings')):
        kw = dict(intervals=iv, hypotheses=[h, h], weights=None)
        kw.update(bad)
        with pytest.raises(ValueError, match=match):
            combine.combine_labels(**kw)
    assert combine.combine_labels([], [[], []]) == []
    with pytest.raises(ValueError, match='2 .. 32'):
        combine.combine_rttm([[('r', 0.0, 1.0, 'a')]])
    out = {s: {} for s in sweep.grid_settings(dict(Fa=[0.1, 0.2], Fb=[1], loopP=[0.5], threshold=[0], smoothing=[5]))}
    with pytest.raises(ValueError, match='2 .. 32'):
        sweep.combine_settings(out, {}, settings=list(out)[:1])
    with pytest.raises(ValueError, match='did not run'):
        sweep.combine_settings(out, {}, settings=list(out) + [sweep.Setting(9, 9, 0.5, 0, 5)])


def test_command_lines():
    args = combine.build_parser().parse_args(['--sys-rttm', 'a', 'b', 'c', '--weights', '1,0.9,0.8', '--out-rttm-dir', 'o'])
    assert args.sys_rttm == ['a', 'b', 'c'] and args.weights == [1.0, 0.9, 0.8] and not args.json
    for argv in (['--sys-rttm', 'a', '--out-rttm-dir', 'o'], ['--sys-rttm', 'a', 'b', '--weights', '1', '--out-rttm-dir', 'o'],
                 ['--sys-rttm', 'a', 'b', '--weights', 'x,1', '--out-rttm-dir', 'o'], ['--sys-rttm', 'a', 'b']):
        with pytest.raises(SystemExit):
            combine.main(argv)
    base = ['--out-dir', 'o', '--xvec-ark-file', 'a', '--segments-file', 's', '--xvec-transform', 't', '--plda-file', 'p',
            '--lda-dim', '128', '--Fa', '1', '--Fb', '1', '--loopP', '0.5', '--threshold', '0']
    ap = sweep.build_parser()
    assert ap.parse_args(base).combine is None and ap.parse_args(base + ['--combine', 'all']).combine == 'all'
    assert ap.parse_args(base + ['--combine', '3']).combine == 3
    for bad in ('1', 'best', '-2'):
        with pytest.raises(SystemExit):
            ap.parse_args(base + ['--combine', bad])
    with pytest.raises(SystemExit):
        sweep.main(base + ['--combine', '2'])                      # the N best need a reference


def test_c_abi_refuses_a_null_handle():
    from vbx_b200 import _lib, build
    build.build_library()
    lib = _lib.load()
    need = ctypes.c_size_t()
    assert lib.vbx_combine_workspace_bytes(None, 1, 2, 4, ctypes.byref(need)) == -1            # VBX_ERR_ARG
    assert lib.vbx_combine(None, 0, None, 0, None, None, 2, None, None, None, 1, None, None, 0, None, None, None, None,
                           None, None, None, None, None, None, None) == -1
