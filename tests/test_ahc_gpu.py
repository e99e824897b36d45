"""Device AHC (csrc/vbx_ahc.cu) against the float64 oracle (oracle/ahc_oracle.py) at meeting length, every feature
width, ties and degenerate calibrations.

`check_dendrogram` judges a linkage without depending on merge order: every height must be the mean of the oracle's
distances over the leaf pairs it joins, and the partitions at every cut must be the oracle's.  So it holds for any
correct average linkage, whichever way ties are broken.  The CPU tests here show that it rejects wrong linkages; the
`gpu` tests hold the device to it and, where there are no ties, to the oracle's linkage merge for merge.
"""
import os
import sys
import warnings
from fractions import Fraction

import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import cophenet, fcluster, linkage
from scipy.spatial.distance import squareform

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ahc_oracle                      # noqa: E402
from vbx_b200 import ahc as host_ahc               # noqa: E402

TOL = 1e-12
SWEEP = np.round(np.linspace(-0.3, 0.3, 13), 3).tolist() + [-0.015]      # AHC thresholds a sweep typically tries
LINK_ROWS_PER_PASS = 32          # warps of ahc_linkage_kernel: rows it recomputes per pass of its step-3 loop


# ---- data and oracle --------------------------------------------------------------------------------------------
def synth(T, dim, seed, spk=6):
    """Speaker centres plus noise, in runs of 5 x-vectors (as tools/bench_ahc.py), rows scaled to varied norms."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((spk, dim))
    who = np.repeat(rng.integers(0, spk, T // 5 + 1), 5)[:T]
    x = centres[who] + 0.8 * rng.standard_normal((T, dim))
    return x * rng.uniform(0.5, 4.0, (T, 1))


def gmm_threshold_torch(s, device):
    """ahc_oracle.two_gaussian_threshold line for line in torch float64, for score matrices too large for numpy to
    calibrate quickly (tens of millions of scores); test_torch_threshold_restates_the_oracle pins it to the oracle."""
    s = torch.as_tensor(np.ascontiguousarray(s), dtype=torch.float64, device=device).reshape(-1)
    sign = torch.tensor([-1.0, 1.0], dtype=torch.float64, device=device)
    w = torch.tensor([0.5, 0.5], dtype=torch.float64, device=device)
    m = s.mean() + s.std(unbiased=False) * sign
    var = s.var(unbiased=False)
    thr = torch.tensor(float('inf'), dtype=torch.float64)
    for _ in range(20):
        ll = torch.log(w) - 0.5 * torch.log(var) - 0.5 * (s[:, None] - m) ** 2 / var
        ll -= ll.max(dim=1, keepdim=True).values
        g = torch.exp(ll)
        g /= g.sum(dim=1, keepdim=True)
        cnt = g.sum(dim=0)
        w = cnt / cnt.sum()
        m = s @ g / cnt
        var = ((s * s) @ g / cnt - m * m) @ w
        thr = -0.5 * ((torch.log(w * w / var) - m * m / var) @ -sign) / ((m / var) @ -sign)
    return float(thr)


def oracle(x, device=None):
    """float64 distances D = -cos, threshold and scipy average linkage of the x-vectors x (cast to float64)."""
    x = np.asarray(x, dtype=np.float64)
    s = ahc_oracle.cosine_similarity(x)
    T = len(x)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)          # degenerate calibrations divide by zero
        thr = ahc_oracle.two_gaussian_threshold(s) if T <= 256 else gmm_threshold_torch(s, device or 'cpu')
    Z = linkage(squareform(-s, checks=False), method='average') if T >= 2 else np.zeros((0, 4))
    return -s, thr, Z


def oracle_labels(Zref, cut):
    """fcluster(..., 'distance') of the oracle linkage at height `cut` (0-based), shifted as in ahc_oracle.ahc_labels."""
    T = len(Zref) + 1
    if T < 2 or np.isnan(cut):
        return np.arange(T)
    adjust = abs(Zref[:, 2].min())
    shifted = Zref.copy()
    shifted[:, 2] += adjust
    return fcluster(shifted, cut + adjust, criterion='distance') - 1


def partition(labels):
    """Labels renumbered by first appearance: equal iff the two labelings group the x-vectors the same way."""
    _, first, inv = np.unique(np.asarray(labels), return_index=True, return_inverse=True)
    rank = np.empty(len(first), dtype=np.int64)
    rank[np.argsort(first)] = np.arange(len(first))
    return rank[inv.reshape(-1)]


# ---- the dendrogram checker ---------------------------------------------------------------------------------------
def check_dendrogram(Z, D, Zref, thr=np.nan, tol=TOL):
    """Raise AssertionError unless the linkage Z [T-1, 4] (scipy layout) is an average linkage of the distances D
    [T, T] that cuts like the oracle's linkage Zref at every height, to within `tol`.  O(T^2): every leaf pair is
    visited once, inside the block of the merge that joins it.  Independent of merge order and of tie breaking."""
    T = D.shape[0]
    Z = np.asarray(Z, dtype=np.float64)
    assert Z.shape == (max(T - 1, 0), 4), f'linkage shape {Z.shape} for {T} x-vectors'
    if T < 2:
        return
    assert np.isfinite(Z).all(), 'linkage has non-finite entries'
    ids = Z[:, :2]
    assert np.array_equal(ids, np.round(ids)), 'cluster ids are not integers'
    ids = ids.astype(np.int64)
    size = np.ones(2 * T - 1, dtype=np.int64)
    used = np.zeros(2 * T - 1, dtype=bool)
    for r in range(T - 1):
        for c in ids[r]:
            assert 0 <= c < T + r, f'merge {r} uses cluster {c}, which does not exist yet'
            assert not used[c], f'cluster {c} merged twice'
            used[c] = True
        size[T + r] = size[ids[r, 0]] + size[ids[r, 1]]
        assert Z[r, 3] == size[T + r], f'merge {r}: size {Z[r, 3]}, children hold {size[T + r]}'
    # leaf order in which every cluster is a contiguous range: merge r joins [lo[a], hi[a]) and [lo[b], hi[b])
    order = []
    stack = [2 * T - 2]
    while stack:
        c = stack.pop()
        if c < T:
            order.append(c)
        else:
            stack += [ids[c - T, 1], ids[c - T, 0]]
    order = np.asarray(order)
    pos = np.empty(T, dtype=np.int64)
    pos[order] = np.arange(T)
    lo = np.concatenate([pos, np.zeros(T - 1, dtype=np.int64)])
    for r in range(T - 1):
        lo[T + r] = min(lo[ids[r, 0]], lo[ids[r, 1]])
    Dp = D[np.ix_(order, order)]
    shift = abs(Zref[:, 2].min())                                 # cophenet wants nonnegative heights
    shifted = Zref.copy()
    shifted[:, 2] += shift
    Cp = squareform(cophenet(shifted))[np.ix_(order, order)] - shift    # oracle's merge height of every leaf pair
    h = Z[:, 2]
    for r in range(T - 1):
        a, b = ids[r]
        a0, b0 = lo[a], lo[b]
        if b0 < a0:
            a, b, a0, b0 = b, a, b0, a0
        a1, b1 = a0 + size[a], b0 + size[b]
        assert a1 == b0, f'merge {r}: children are not adjacent in the leaf order'
        mean = Dp[a0:a1, b0:b1].sum() / (size[a] * size[b])
        assert abs(h[r] - mean) <= tol, f'merge {r}: height {h[r]!r}, mean distance of its leaf pairs {mean!r}'
        dev = np.abs(Cp[a0:a1, b0:b1] - h[r]).max()
        assert dev <= tol, f'merge {r} at {h[r]!r} joins leaves the oracle joins {dev:.3g} away: partitions differ'
    assert np.all(np.diff(h) >= -tol), f'heights decrease by up to {-np.diff(h).min():.3g}'
    # the host cut (ahc.cut, what diarization and the sweep run) against fcluster of the oracle linkage
    href = Zref[:, 2]
    cuts = [(0.0, -c) for c in np.linspace(href.min() - 0.01, href.max() + 0.01, 23)]
    if np.isfinite(thr):
        cuts += [(thr, t) for t in SWEEP]
    for th, t in cuts:
        height = -(th + t)
        if np.abs(href - height).min() <= 100 * tol:             # a cut on a merge height: either side is right
            continue
        got = host_ahc.cut([Z], np.array([th]), [T], t)[0]
        np.testing.assert_array_equal(partition(got), partition(oracle_labels(Zref, height)),
                                      err_msg=f'partition at cut {height}')


def check_against_oracle(Z, thr, labels, ref, exact=True, thr_tol=1e-9, msg=''):
    """Device results of one recording against ref = oracle(x): threshold (NaN exactly when the oracle's is),
    the checker, and with exact=True (no ties) the oracle's linkage merge for merge and its labels."""
    D, thr_ref, Zref = ref
    assert np.isnan(thr) == np.isnan(thr_ref), f'{msg}: threshold {thr} against the oracle {thr_ref}'
    if not np.isnan(thr_ref):
        assert abs(thr - thr_ref) <= thr_tol, f'{msg}: threshold {thr!r} against the oracle {thr_ref!r}'
    try:
        check_dendrogram(Z, D, Zref, thr_ref)
    except AssertionError as e:
        raise AssertionError(f'{msg}: {e}') from None
    cut = -(thr_ref - 0.015)
    if exact:
        np.testing.assert_array_equal(Z[:, [0, 1, 3]], Zref[:, [0, 1, 3]], err_msg=msg)
        np.testing.assert_allclose(Z[:, 2], Zref[:, 2], rtol=0, atol=TOL, err_msg=msg)
        np.testing.assert_array_equal(labels, oracle_labels(Zref, cut), err_msg=msg)
    else:
        np.testing.assert_array_equal(partition(labels), partition(oracle_labels(Zref, cut)), err_msg=msg)


# ---- CPU: the checker has teeth -------------------------------------------------------------------------------------
def naive_average_linkage(D, detour=None):
    """O(T^3) average linkage in scipy's layout; at step `detour` it merges the second-closest pair instead."""
    T = len(D)
    members = {i: [i] for i in range(T)}
    Z = []
    for step in range(T - 1):
        keys = sorted(members)
        pairs = sorted((D[np.ix_(members[a], members[b])].mean(), a, b)
                       for i, a in enumerate(keys) for b in keys[i + 1:])
        d, a, b = pairs[1] if step == detour else pairs[0]
        members[T + step] = members.pop(a) + members.pop(b)
        Z.append([a, b, d, len(members[T + step])])
    return np.array(Z, dtype=np.float64)


@pytest.fixture(scope='module')
def small_case():
    D, thr, Zref = oracle(synth(40, 16, seed=1))
    return D, thr, Zref


def test_checker_accepts_the_oracle_linkage(small_case):
    D, thr, Zref = small_case
    check_dendrogram(Zref, D, Zref, thr)
    check_dendrogram(naive_average_linkage(D), D, Zref, thr)


def test_checker_rejects_children_swapped_across_rows(small_case):
    D, thr, Zref = small_case
    rejected = 0
    for r1, r2 in ((3, 20), (10, 11), (0, 38), (25, 37)):
        Z = Zref.copy()
        Z[r1, 1], Z[r2, 0] = Zref[r2, 0], Zref[r1, 1]
        with pytest.raises(AssertionError):
            check_dendrogram(Z, D, Zref, thr)
        rejected += 1
    assert rejected == 4


@pytest.mark.parametrize('row', [0, 17, 38])
def test_checker_rejects_a_height_moved_by_1e9(small_case, row):
    D, thr, Zref = small_case
    Z = Zref.copy()
    Z[row, 2] += 1e-9
    with pytest.raises(AssertionError, match='mean distance'):
        check_dendrogram(Z, D, Zref, thr)


def test_checker_rejects_a_merge_of_a_non_closest_pair(small_case):
    """Heights all correct means and nondecreasing: only the partition check can tell the linkage is wrong."""
    D, thr, Zref = small_case
    tested = 0
    for detour in range(len(D) - 2):
        Z = naive_average_linkage(D, detour)
        if np.all(np.diff(Z[:, 2]) >= 0):
            with pytest.raises(AssertionError, match='partitions differ'):
                check_dendrogram(Z, D, Zref, thr)
            tested += 1
    assert tested >= 3


def test_checker_is_independent_of_tie_breaking():
    """Duplicated x-vectors tie; a linkage that breaks every tie the other way passes as well."""
    x = synth(30, 8, seed=2)
    x = np.concatenate([x, x[:10], x[5:8]])
    D, thr, Zref = oracle(x)
    D = (D + D.T) / 2                   # the same distance both ways, so that ties are exact
    Zrev = linkage(squareform(D[::-1, ::-1], checks=False), method='average')
    perm = np.arange(len(x))[::-1]
    T = len(x)
    ids = Zrev[:, :2].astype(np.int64)
    ids = np.where(ids < T, perm[np.minimum(ids, T - 1)], ids)
    Zrev[:, :2] = np.sort(ids, axis=1)
    assert not np.array_equal(Zrev[:, :2], Zref[:, :2])
    check_dendrogram(Zrev, D, Zref, thr)


def test_torch_threshold_restates_the_oracle():
    for T, dim, seed in ((150, 32, 4), (129, 3, 5), (200, 128, 6)):
        s = ahc_oracle.cosine_similarity(synth(T, dim, seed))
        assert abs(gmm_threshold_torch(s, 'cpu') - ahc_oracle.two_gaussian_threshold(s)) <= 1e-12


def replay_nn_arrays(D):
    """The nearest-neighbour schedule of ahc_linkage_kernel on the host (slot a = min(p, q) keeps the merge, ties go
    to the lowest slot): returns its linkage and, per merge, how many rows its step 3 recomputes."""
    D = D.copy()
    T = len(D)
    np.fill_diagonal(D, np.inf)
    alive = np.ones(T, dtype=bool)
    nn = D.argmin(axis=1)
    nnd = D[np.arange(T), nn]
    cid = np.arange(T)
    csize = np.ones(T, dtype=np.int64)
    Z = np.zeros((T - 1, 4))
    rows = []
    for step in range(T - 1):
        p = int(np.where(alive, nnd, np.inf).argmin())
        q = int(nn[p])
        a, b = min(p, q), max(p, q)
        na, nb = csize[a], csize[b]
        Z[step] = [min(cid[a], cid[b]), max(cid[a], cid[b]), nnd[p], na + nb]
        alive[b] = False
        live = alive.copy()
        live[a] = False
        dn = (na / (na + nb)) * D[a] + (nb / (na + nb)) * D[b]
        D[a, live] = dn[live]
        D[live, a] = dn[live]
        D[b, :] = np.inf
        D[:, b] = np.inf
        todo = live & ((nn == a) | (nn == b))
        closer = live & ~todo & (D[a] < nnd)
        nn[closer] = a
        nnd[closer] = D[a, closer]
        cid[a], csize[a] = T + step, na + nb
        redo = np.concatenate([np.flatnonzero(todo), [a]])
        rows.append(len(redo))
        if step < T - 2:
            nn[redo] = D[redo].argmin(axis=1)
            nnd[redo] = D[redo, nn[redo]]
    return Z, np.array(rows)


LONG_T = 8000


@pytest.fixture(scope='module')
def long_x():
    """The long case of tools/bench_ahc.py, as the float32 x-vectors the front end hands over."""
    return synth(LONG_T, 128, seed=8000).astype(np.float32)


def test_long_recording_needs_more_than_one_recompute_pass(long_x):
    """On the long recording some merge leaves more rows without their nearest neighbour than one pass of the
    linkage kernel's step 3 recomputes, so the device tests below exercise the loop's later passes."""
    s = ahc_oracle.cosine_similarity(long_x.astype(np.float64))
    Zref = linkage(squareform(-s, checks=False), method='average')
    Z, rows = replay_nn_arrays(-s)
    np.testing.assert_array_equal(Z[:, [0, 1, 3]], Zref[:, [0, 1, 3]])
    assert rows.max() > LINK_ROWS_PER_PASS, rows.max()


# ---- GPU --------------------------------------------------------------------------------------------------------------
DEV = 'cuda:0'


def device_ahc(xs, dtype, dim=None):
    """vbx_ahc on one ragged batch: (labels, thresholds, linkages), linkages copied out of the batch buffer."""
    from vbx_b200.batch import VbxBatch
    dim = dim or xs[0].shape[1]
    lens = [len(x) for x in xs]
    vb = VbxBatch(lens, 128, 2, device=torch.device(DEV), allocate=False)
    try:
        x = torch.from_numpy(np.concatenate([np.asarray(x, dtype=np.float64).reshape(-1, dim) for x in xs]))
        x = x.to(DEV).to(dtype).contiguous()
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', RuntimeWarning)
            labels, thr, Zs = host_ahc.ahc_batch(vb, x)
        torch.cuda.synchronize()
    finally:
        vb.close()
    return labels, thr, [z.copy() for z in Zs]


def as_input(x, dtype):
    """The x-vectors as the device sees them, in float64 for the oracle."""
    return np.asarray(x, dtype=np.float32 if dtype == torch.float32 else np.float64).astype(np.float64)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


SMALL_T = [2, 3, 4, 5, 7, 8, 31, 32, 33, 63, 64, 65]
LARGE_T = {1: [1023], 3: [1024], 31: [1025], 32: [1056], 33: [2049, 4097], 100: [1023], 128: [4097], 200: [1025],
           256: [2049], 512: [1024, 1056]}


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float64, torch.float32], ids=['f64', 'f32'])
@pytest.mark.parametrize('dim', sorted(LARGE_T))
def test_device_ahc_shapes(dim, dtype):
    """Every T of SMALL_T and some of LARGE_T at this feature width, as one ragged batch: 32 x 32 cosine tiles and their
    feature tail, fewer than 64 scores per recording (GMM chunks), and more x-vectors than the linkage kernel's 1024
    threads.  float32 input is converted to float64 before any arithmetic, so it is held to the same bars.
    At dim = 1 every cosine is +-1: all ties, so only the checker and the partitions apply.  At T = 2 the calibration
    has zero variance in exact arithmetic, so whether its threshold is NaN hangs on the last bit of the diagonal
    cosines; test_device_ahc_two_and_three_xvectors pins that case with cosines both sides compute exactly."""
    Ts = SMALL_T + LARGE_T[dim]
    xs = [as_input(synth(T, dim, seed=1000 * dim + T), dtype) for T in Ts]
    labels, thr, Zs = device_ahc(xs, dtype)
    for b, T in enumerate(Ts):
        ref = oracle(xs[b], DEV)
        if T == 2:
            ref = (ref[0], thr[b], ref[2])
        check_against_oracle(Zs[b], thr[b], labels[b], ref, exact=dim > 1, msg=f'T={T} dim={dim}')


@pytest.fixture(scope='module')
def long_batch(long_x):
    """The long recording alone, then in one batch with recordings of 0, 1, 2, 3, 40 and 1025 x-vectors."""
    others = {T: synth(T, 128, seed=T).astype(np.float32) for T in (0, 1, 2, 3, 40, 1025)}
    order = [0, 1025, 1, 2, LONG_T, 3, 40]
    xs = [long_x if T == LONG_T else others[T] for T in order]
    return order, xs, device_ahc(xs, torch.float32, 128)


@pytest.mark.gpu
def test_device_ahc_long_recording_against_the_oracle(long_x, long_batch):
    labels, thr, Zs = device_ahc([long_x], torch.float32)
    check_against_oracle(Zs[0], thr[0], labels[0], oracle(as_input(long_x, torch.float32), DEV), msg='T=8000')
    order, xs, (blabels, bthr, bZs) = long_batch
    k = order.index(LONG_T)
    assert bits(bthr[k]) == bits(thr[0])
    np.testing.assert_array_equal(bits(bZs[k]), bits(Zs[0]))
    np.testing.assert_array_equal(blabels[k], labels[0])


@pytest.mark.gpu
def test_device_ahc_ragged_batch_equals_solo_runs(long_batch):
    """Each recording of the batch is bit-identical to its run alone (workspace carve, blockIdx.z, early exit of
    recordings shorter than the longest), and the oracle's."""
    order, xs, (blabels, bthr, bZs) = long_batch
    for k, T in enumerate(order):
        if T == LONG_T:
            continue
        labels, thr, Zs = device_ahc([xs[k]], torch.float32, 128)
        assert bits(bthr[k]) == bits(thr[0]), T
        np.testing.assert_array_equal(bits(bZs[k]), bits(Zs[0]), err_msg=f'T={T}')
        np.testing.assert_array_equal(blabels[k], labels[0], err_msg=f'T={T}')
        if T >= 3:
            check_against_oracle(bZs[k], bthr[k], blabels[k], oracle(as_input(xs[k], torch.float32), DEV), msg=f'T={T}')
        else:
            assert blabels[k].tolist() == list(range(T)), T


@pytest.mark.gpu
def test_device_ahc_is_deterministic(long_batch):
    order, xs, (blabels, bthr, bZs) = long_batch
    labels, thr, Zs = device_ahc(xs, torch.float32, 128)
    np.testing.assert_array_equal(bits(thr), bits(bthr))
    for k, T in enumerate(order):
        np.testing.assert_array_equal(bits(Zs[k]), bits(bZs[k]), err_msg=f'T={T}')
        np.testing.assert_array_equal(labels[k], blabels[k], err_msg=f'T={T}')


def exact_pairs(n, seed):
    """Unit vectors (a, b) whose cosines with e1 and with themselves every evaluation order gets exactly: a^2 + b^2
    rounds to 1 whether summed plainly or with either product fused, so numpy and the device see the same scores.
    a^2 itself is inexact; a in [0.97, 1) puts the two x-vectors within merging distance of a finite threshold."""
    def fma(p, q, r):
        return float(Fraction(p) * Fraction(q) + Fraction(r))
    rng = np.random.default_rng(seed)
    up, down = [], []
    while len(up) < n or len(down) < n:
        a = float(rng.uniform(0.97, 1.0))
        b = float(np.sqrt(1.0 - a * a))
        if not (a * a + b * b == 1.0 and fma(a, a, b * b) == 1.0 and fma(b, b, a * a) == 1.0):
            continue
        err = Fraction(a * a) - Fraction(a) ** 2
        if err > 0 and len(up) < n:
            up.append((a, b))
        elif err < 0 and len(down) < n:
            down.append((a, b))
    return up + down


@pytest.mark.gpu
@pytest.mark.parametrize('dim', [2, 33])
def test_device_ahc_two_and_three_xvectors(dim):
    """T = 2: the calibration's variance is exactly 0 in the reference, so its threshold is NaN and each x-vector
    stays its own cluster.  The x-vectors are cut so that the device's and numpy's scores agree to the bit, and half of
    them make a^2 round up, so a fused multiply-add in the variance would leave a positive residual: a finite
    threshold, and the two x-vectors would merge.  T = 3: seeded x-vectors, threshold and labels against the oracle."""
    xs = []
    for a, b in exact_pairs(4, seed=dim):
        x = np.zeros((2, dim))
        x[0, 0] = 1.0
        x[1, :2] = a, b
        xs.append(x)
    rng = np.random.default_rng(3)
    xs += [rng.standard_normal((3, dim)) for _ in range(4)]
    labels, thr, Zs = device_ahc(xs, torch.float64)
    for k, x in enumerate(xs):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', RuntimeWarning)
            ref_labels, ref_thr, ref_Z = ahc_oracle.ahc_labels(x)
        if len(x) == 2:
            assert np.isnan(ref_thr)
            assert np.isnan(thr[k]), f'x-vectors {k}: threshold {thr[k]!r}, the reference has NaN'
        else:
            assert abs(thr[k] - ref_thr) <= 1e-9, (k, thr[k], ref_thr)
        np.testing.assert_array_equal(labels[k], ref_labels, err_msg=f'recording {k}')
        np.testing.assert_array_equal(Zs[k][:, [0, 1, 3]], ref_Z[:, [0, 1, 3]])
        np.testing.assert_allclose(Zs[k][:, 2], ref_Z[:, 2], rtol=0, atol=TOL)


@pytest.mark.gpu
def test_device_ahc_identical_xvectors():
    """All x-vectors equal: every score is the same, the calibration has no variance and its threshold is NaN, so the
    reference leaves every x-vector on its own.  Rows e1 give scores of exactly 1; random rows the scores numpy and the
    device round to.  Random rows stop at T = 65: numpy's mean of a million equal scores is off by its own rounding,
    and from that noise the reference calibrates a finite threshold that depends on the machine's BLAS."""
    rng = np.random.default_rng(11)
    xs = []
    for T, dim in ((4, 8), (32, 33), (40, 128), (65, 3), (1025, 128)):
        e1 = np.zeros((T, dim))
        e1[:, 0] = 1.0
        xs += [e1] if T > 65 else [e1, np.tile(rng.standard_normal(dim), (T, 1))]
    for dim in (8, 33, 128, 3):
        group = [x for x in xs if x.shape[1] == dim]
        labels, thr, Zs = device_ahc(group, torch.float64)
        for k, x in enumerate(group):
            T = len(x)
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', RuntimeWarning)
                ref_labels, ref_thr, ref_Z = ahc_oracle.ahc_labels(x)
            assert np.isnan(ref_thr)
            assert np.isnan(thr[k]), f'T={T} dim={dim} recording {k}: threshold {thr[k]!r}'
            np.testing.assert_array_equal(np.sort(labels[k]), np.arange(T))
            check_dendrogram(Zs[k], -ahc_oracle.cosine_similarity(x), ref_Z)
            if x[0, 0] == 1.0:
                # every distance exactly -1 on both sides: each tie goes to the lowest slot, as scipy breaks it, so
                # the linkage and the numbering of the singletons are scipy's (for random rows numpy's last bits
                # break the ties, and with them the numbering)
                np.testing.assert_array_equal(Zs[k], ref_Z, err_msg=f'T={T} dim={dim}')
                np.testing.assert_array_equal(labels[k], ref_labels)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float64, torch.float32], ids=['f64', 'f32'])
def test_device_ahc_duplicate_rows(dtype):
    """Exact duplicates tie at distance -1 and with every third x-vector: merge ids may differ from scipy's, but every
    height and the partition at every cut are the oracle's."""
    xs = []
    for T, dim, seed in ((33, 31, 1), (1056, 33, 2), (600, 128, 3), (200, 1, 4)):
        x = synth(T, dim, seed)
        rng = np.random.default_rng(seed)
        src = rng.integers(0, T, T // 3)
        dst = rng.choice(T, T // 3, replace=False)
        x[dst] = x[src]
        xs.append(as_input(x, dtype))
    for x in xs:
        labels, thr, Zs = device_ahc([x], dtype)
        check_against_oracle(Zs[0], thr[0], labels[0], oracle(x, DEV), exact=False, msg=f'T={len(x)} dim={x.shape[1]}')


@pytest.mark.gpu
def test_device_ahc_zero_row():
    """An all-zero x-vector has cosine 0 with everything, itself included (the reference's norm + 1e-32).  The other
    x-vectors are positive, so all their distances are negative and the zero row, at distance 0 from every cluster,
    merges last and alone (with mixed signs it would tie with several clusters at 0, and a tie there changes the tree)."""
    xs = []
    for T, dim, row in ((33, 33, 0), (100, 128, 57), (1025, 31, 1024)):
        x = np.abs(synth(T, dim, seed=T))
        x[row] = 0.0
        xs.append(x)
    for x in xs:
        labels, thr, Zs = device_ahc([x], torch.float64)
        ref = oracle(x, DEV)
        assert not np.any(ref[0][np.all(x == 0, axis=1)])
        check_against_oracle(Zs[0], thr[0], labels[0], ref, msg=f'T={len(x)}')


@pytest.mark.gpu
def test_device_ahc_nan_row():
    """A NaN x-vector (scipy refuses those, so there is no reference): no fault; it never merges, so the last linkage
    row is NaN and the rest is the oracle's linkage of the other x-vectors; the threshold is NaN and every x-vector
    its own cluster; the other recordings of the batch are bit-identical to a batch without it."""
    others = [synth(T, 33, seed=T) for T in (40, 1056, 3)]
    T, j = 300, 123
    bad = synth(T, 33, seed=7)
    bad[j, 5] = np.nan
    labels, thr, Zs = device_ahc(others[:2] + [bad] + others[2:], torch.float64)
    clean_labels, clean_thr, clean_Zs = device_ahc(others, torch.float64)
    for k, kc in ((0, 0), (1, 1), (3, 2)):
        assert bits(thr[k]) == bits(clean_thr[kc])
        np.testing.assert_array_equal(bits(Zs[k]), bits(clean_Zs[kc]))
        np.testing.assert_array_equal(labels[k], clean_labels[kc])
    Z = Zs[2]
    assert np.isnan(thr[2])
    assert np.isfinite(Z[:T - 2]).all() and np.isnan(Z[T - 2:]).all()
    assert sorted(labels[2].tolist()) == list(range(T))
    # the finite rows: the oracle's linkage of the other 299 x-vectors, leaves past j and merges renumbered
    _, _, Zref = oracle(np.delete(bad, j, axis=0))
    ids = Zref[:, :2].copy()
    ids = np.where(ids >= j, ids + 1, ids)
    ids = np.where(Zref[:, :2] >= T - 1, Zref[:, :2] + 1, ids)
    np.testing.assert_array_equal(Z[:T - 2, :2], ids)
    np.testing.assert_array_equal(Z[:T - 2, 3], Zref[:, 3])
    np.testing.assert_allclose(Z[:T - 2, 2], Zref[:, 2], rtol=0, atol=TOL)
