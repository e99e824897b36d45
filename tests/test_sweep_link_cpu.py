"""Speaker linking inside the sweep (DESIGN.md section 5.18) without a GPU: a numpy restatement of vbx_link_batch's flat
score-tile decoding and workspace layout, packing of problems under a budget, the DER across files summed by global
id against score.across_files_result, the argument checks, and the summary and ranking of a faked sweep output."""
import math

import numpy as np
import pytest

from vbx_b200 import link, score, sweep
from vbx_b200.sweep import Setting


# ---- restatements of vbx_link.cu ----------------------------------------------------------------------------------------

def al(v):
    return (v + 255) & ~255


def linkage_bytes(T):              # linkage_workspace_bytes (vbx_ahc.cu)
    return T * T * 8 + T * (8 + 4 + 4 + 4 + 4) + T


def batch_layout(Ms):
    """(linkage region offsets [G+1], total bytes) of vbx_link_batch_workspace_bytes: the problems' linkage regions,
    then n, e, b, first, last over all speakers, then the problem arrays (off, lk_off, tile_off, dist_off, c)."""
    lk = [0]
    for M in Ms:
        lk.append(lk[-1] + al(linkage_bytes(M)))
    M = sum(Ms)
    G = len(Ms)
    return lk, lk[-1] + 4 * al(8 * M) + al(8 * 128 * M) + al((5 * G + 4) * 8)


def tiles(M):
    t = (M + 31) // 32
    return t * (t + 1) // 2


def find_problem(pref, G, x):
    lo, hi = 0, G
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if pref[mid] <= x:
            lo = mid
        else:
            hi = mid
    return lo


def decode(Ms, t):
    """link_score_kernel's decoding of flat tile t -> (problem, bi, bj)."""
    off = np.concatenate([[0], np.cumsum([tiles(M) for M in Ms])])
    g = find_problem(off, len(Ms), t)
    lt = t - int(off[g])
    n = (Ms[g] + 31) // 32
    tt = 2.0 * n + 1.0
    row0 = lambda b: b * n - b * (b - 1) // 2
    bi = int((tt - math.sqrt(tt * tt - 8.0 * lt)) / 2.0)
    while bi > 0 and row0(bi) > lt:
        bi -= 1
    while bi + 1 < n and row0(bi + 1) <= lt:
        bi += 1
    return g, bi, bi + (lt - row0(bi))


@pytest.mark.parametrize('order', [0, 1, 2])
def test_every_tile_of_every_problem_once(order):
    Ms = [0, 1, 2, 31, 32, 33, 1000]
    Ms = [Ms[(i * (order + 1)) % len(Ms)] for i in range(len(Ms))] if order else Ms
    Ms = Ms + [0, 33]
    total = sum(tiles(M) for M in Ms)
    grid = total // 3 + 1                     # below the tile count: CTAs stride
    assert grid < total
    seen = []
    for cta in range(grid):
        for t in range(cta, total, grid):
            seen.append(decode(Ms, t))
    want = [(g, bi, bj) for g, M in enumerate(Ms) for bi in range((M + 31) // 32) for bj in range(bi, (M + 31) // 32)]
    assert len(seen) == len(set(seen)) == total
    assert sorted(seen) == sorted(want)


def test_workspace_layout_and_packing():
    rng = np.random.default_rng(3)
    for _ in range(20):
        Ms = rng.integers(0, 300, int(rng.integers(1, 12))).tolist()
        lk, total = batch_layout(Ms)
        assert all(o % 256 == 0 for o in lk)                 # every problem's linkage region 256-byte aligned
        assert [lk[g + 1] - lk[g] for g in range(len(Ms))] == [al(linkage_bytes(M)) for M in Ms]
        single = [batch_layout([M])[1] for M in Ms]          # each problem sized alone, as link_many packs them
        assert total <= sum(single)                          # so packing by the single sizes bounds every launch
        budget = max(single) + int(rng.integers(0, 2 * max(single)))
        batches = sweep.pack(single, budget)
        assert sum(batches, []) == list(range(len(Ms)))
        assert all(batch_layout([Ms[g] for g in b])[1] <= budget for b in batches)
    assert batch_layout([0])[1] == 256                       # M = 0: the problem arrays only
    with pytest.raises(ValueError, match='more than max_batch_bytes'):
        sweep.pack([batch_layout([40])[1]], batch_layout([40])[1] - 1)


# ---- DER across files by global id --------------------------------------------------------------------------------------

def _random_files(rng, n_files):
    ref_names, blocks, maps = [], [], []
    pool = [f'spk{k}' for k in range(7)]
    for f in range(n_files):
        rk = sorted(rng.choice(pool, int(rng.integers(0, 4)), replace=False).tolist())
        n_lab = int(rng.integers(0, 5))
        blk = rng.integers(0, 1000, (len(rk), n_lab)).astype(np.int64)
        m = {}
        for l in range(n_lab):
            if rng.random() < 0.2:                          # a label without turns: no map entry, empty column
                blk[:, l] = 0
            else:
                m[l] = int(rng.integers(0, 6))
        if f % 4 == 3:                                      # a file without system speakers
            blk, m = np.zeros((len(rk), 0), dtype=np.int64), {}
        ids = list(m.values())
        if len(set(ids)) != len(ids):                       # one global id per label of a file (link_cut is one-to-one)
            m = {l: 10 + 7 * f + i for i, l in enumerate(m)}
        ref_names.append(rk)
        blocks.append(blk)
        maps.append(m)
    return ref_names, blocks, maps


@pytest.mark.parametrize('seed', range(8))
def test_across_files_by_id_equals_named_matching(seed):
    rng = np.random.default_rng(seed)
    ref_names, blocks, maps = _random_files(rng, 6)
    scored = int(sum(b.sum() for b in blocks)) + 5000
    tot = score.result(int(rng.integers(0, 500)), int(rng.integers(0, 500)), 0, scored)
    got = sweep.across_files_by_id(tot, ref_names, blocks, maps)
    sys_names, kept = [], []
    for blk, m in zip(blocks, maps):
        cols = [l for l in range(blk.shape[1]) if l in m]
        sys_names.append([f'g{m[l]}' for l in cols])
        kept.append(blk[:, cols])
    order = [np.argsort(n, kind='stable') for n in sys_names]      # across_files_result wants sorted names per file
    want = score.across_files_result(tot, ref_names, [sorted(n) for n in sys_names],
                                     [k[:, o] for k, o in zip(kept, order)])
    assert got == want


def test_across_files_by_id_without_speakers():
    tot = score.result(10, 5, 0, 100)
    got = sweep.across_files_by_id(tot, [[], ['a']], [np.zeros((0, 2), np.int64), np.zeros((1, 0), np.int64)], [{}, {}])
    assert got['ticks'] == dict(miss=10, fa=5, conf=90, scored=100)


# ---- argument checks ----------------------------------------------------------------------------------------------------

GRID = dict(Fa=[0.3], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])


@pytest.mark.parametrize('bad', [[float('nan')], [float('inf')], [-float('inf')], [1.5e15], [0.0, -2e15], []])
def test_bad_link_thresholds_before_device_work(bad):
    with pytest.raises(ValueError, match='link threshold|at least one'):
        sweep.sweep_batch({'r': (np.zeros((3, 256)), np.zeros((3, 2)))}, None, None, GRID, link_thresholds=bad)


def test_link_thresholds_are_deduplicated_in_order():
    assert sweep.check_link_thresholds(None) is None
    assert sweep.check_link_thresholds([48, -10, 48.0, 0, -10]) == [48.0, -10.0, 0.0]
    assert sweep.check_link_thresholds(np.array([1e15, -1e15])) == [1e15, -1e15]


def test_command_line_list():
    ap = sweep.build_parser()
    req = ['--out-dir', 'o', '--xvec-ark-file', 'a', '--segments-file', 's', '--xvec-transform', 't', '--plda-file', 'p',
           '--lda-dim', '128', '--Fa', '0.3', '--Fb', '17', '--loopP', '0.99', '--threshold=-0.015']
    assert ap.parse_args(req).link_threshold is None
    assert ap.parse_args(req + ['--link-threshold=-10,0,48']).link_threshold == [-10.0, 0.0, 48.0]
    with pytest.raises(SystemExit):
        ap.parse_args(req + ['--link-threshold', 'x'])


# ---- summary and ranking from a faked sweep output ----------------------------------------------------------------------

def _fake_out():
    """Two settings x two recordings, one reference speaker per recording ('a' in both), linked at two thresholds."""
    s1, s2 = Setting(0.3, 17.0, 0.99, -0.015, 5.0), Setting(0.4, 17.0, 0.99, -0.015, 5.0)
    per_p = lambda v: {p: v for p, _, _ in score.PROTOCOLS}
    item = lambda m: dict(der=per_p(score.result(0, 0, 0, 100)), ref_speakers=['a'],
                          der_blocks=per_p(np.array([[60, 40]], dtype=np.int64)), global_speakers=m)
    out = {}
    for s in (s1, s2):
        # threshold 5: both files' labels 0 -> id 0 and labels 1 -> id 1; threshold -5: everything id 0 in file 1
        out[s] = {'r1': item({5.0: {0: 0, 1: 1}, -5.0: {0: 0, 1: 1}}),
                  'r2': item({5.0: {0: 0, 1: 1}, -5.0: {0: 1, 1: 0}})}
    return s1, s2, out


def test_summary_and_ranking_ties_are_stable():
    s1, s2, out = _fake_out()
    tot, ranking = sweep.summarize_across_files(out)
    keys = [sweep.link_key(s, t) for s in (s1, s2) for t in (5.0, -5.0)]
    assert list(tot) == keys and keys[0] == s1.name + '_link5' and keys[1] == s1.name + '_link-5'
    for p, _, _ in score.PROTOCOLS:
        # link5: id 0 gets 120 of 200 ticks; link-5: ids 0 and 1 each get 100 -> matched 100
        assert tot[keys[0]][p]['ticks'] == dict(miss=0, fa=0, conf=80, scored=200)
        assert tot[keys[1]][p]['ticks'] == dict(miss=0, fa=0, conf=100, scored=200)
        assert ranking[p] == [keys[0], keys[2], keys[1], keys[3]]      # equal DERs keep grid, then threshold order
