"""Combination of K diarizations of one recording by label mapping and weighted voting: the rule of DESIGN.md section
5.21 in plain numpy with scipy's linear_sum_assignment.  Test infrastructure: nothing under vbx_b200/ imports it.

    combine(lo, hi, labels, labels2, n_labels, weights=None) -> dict(labels, labels2, order, weights, D, map, n_global,
                                                                   flags, O, L, totals)
labels, labels2: int [K, T]; n_labels: int [K]; weights: None or K positive floats.  O is {(a, b): int64 [n_a, n_b]} for
a < b, L a list of int64 [n_a], map a list of int arrays [n_a] (-1 = no time), totals the K - 1 assignment totals in
rank order (what any optimal assignment must reach) and unique a list of K - 1 booleans: whether that assignment's
optimum is the only one (found by brute force over single-cell perturbations of the cost).
"""
import numpy as np
from scipy.optimize import linear_sum_assignment

BAD_LABEL, TOO_MANY_LABELS = 1, 2
MAX_GLOBAL = 255


def clean(labels, labels2, n_labels):
    """-> (labels, labels2, bad) with the bad intervals of each hypothesis set to (-1, -1)."""
    l1, l2 = np.array(labels, dtype=np.int64), np.array(labels2, dtype=np.int64)
    n = np.asarray(n_labels, dtype=np.int64).reshape(-1, 1)
    bad = (l1 < -1) | (l1 >= n) | (l2 < -1) | (l2 >= n) | ((l1 < 0) & (l2 >= 0)) | ((l1 >= 0) & (l2 == l1))
    l1[bad] = -1
    l2[bad] = -1
    return l1, l2, bool(bad.any())


def says(l1, l2, n):
    """[T, n] bool: the interval has label s in either stream."""
    out = np.zeros((l1.shape[0], n), dtype=bool)
    for l in (l1, l2):
        i = np.nonzero(l >= 0)[0]
        out[i, l[i]] = True
    return out


def matching_total(O):
    if O.size == 0:
        return 0
    r, c = linear_sum_assignment(O, maximize=True)
    return int(O[r, c].sum())


def default_weight(rank):
    """DOVER's default: rank ** -0.1 with rank 1 for the anchor, the C library's pow on float64."""
    return float(rank) ** -0.1


def assign(C):
    """Maximum-total one-to-one assignment of the rows of C (int64) that never pairs a row with a column it shares
    nothing with: -> (column or -1 per row, total, whether the optimum is unique)."""
    n, m = C.shape
    col = np.full(n, -1, dtype=np.int64)
    if n == 0 or m == 0:
        return col, 0, True
    r, c = linear_sum_assignment(C, maximize=True)
    keep = C[r, c] > 0
    col[r[keep]] = c[keep]
    total = int(C[r, c].sum())
    # unique iff forbidding any one matched pair lowers the optimum
    unique = True
    for i, j in zip(r[keep], c[keep]):
        Cx = C.copy()
        Cx[i, j] = 0
        ri, ci = linear_sum_assignment(Cx, maximize=True)
        if int(Cx[ri, ci].sum()) == total:
            unique = False
            break
    return col, total, unique


def combine(lo, hi, labels, labels2, n_labels, weights=None):
    lo, hi = np.asarray(lo, dtype=np.int64), np.asarray(hi, dtype=np.int64)
    K = len(n_labels)
    l1, l2, bad = clean(labels, labels2, n_labels)
    d = np.maximum(hi - lo, 0)
    S = [says(l1[k], l2[k], int(n_labels[k])) for k in range(K)]
    L = [(S[k] * d[:, None]).sum(0).astype(np.int64) for k in range(K)]
    O = {(a, b): (S[a].astype(np.int64).T * d[None, :]) @ S[b].astype(np.int64) for a in range(K) for b in range(a + 1, K)}
    block = lambda a, b: O[(a, b)] if a < b else O[(b, a)].T
    D = np.zeros((K, K), dtype=np.int64)
    for (a, b), blk in O.items():
        D[a, b] = D[b, a] = int(L[a].sum()) + int(L[b].sum()) - 2 * matching_total(blk)
    order = sorted(range(K), key=lambda k: (int(D[k].sum()), k))
    if weights is None:
        w = np.zeros(K, dtype=np.float64)
        for r, k in enumerate(order):
            w[k] = default_weight(r + 1)
    else:
        w = np.asarray(weights, dtype=np.float64)
    maps = [np.full(int(n), -1, dtype=np.int64) for n in n_labels]
    anchor = order[0]
    have = np.nonzero(L[anchor] > 0)[0]
    maps[anchor][have] = np.arange(len(have))
    ng, flags = len(have), BAD_LABEL if bad else 0
    totals, unique = [], []
    for r in range(1, K):
        h = order[r]
        C = np.zeros((int(n_labels[h]), ng), dtype=np.int64)
        for b in order[:r]:
            blk = block(h, b)
            for u, g in enumerate(maps[b]):
                if g >= 0:
                    C[:, g] += blk[:, u]
        col, total, uniq = assign(C)
        totals.append(total)
        unique.append(uniq)
        for s in range(int(n_labels[h])):
            if L[h][s] <= 0:
                continue
            if col[s] >= 0:
                maps[h][s] = col[s]
            else:
                maps[h][s] = ng
                ng += 1
        if ng > MAX_GLOBAL:
            T = len(lo)
            return dict(labels=np.full(T, -1), labels2=np.full(T, -1), order=order, weights=w, D=D, map=maps, n_global=0,
                        flags=flags | TOO_MANY_LABELS, O=O, L=L, totals=totals, unique=unique)
    out1, out2 = np.full(len(lo), -1, dtype=np.int64), np.full(len(lo), -1, dtype=np.int64)
    for i in range(len(lo)):
        num = den = 0.0
        tally = {}
        for k in range(K):
            mine = [int(x) for x in (l1[k, i], l2[k, i]) if x >= 0]
            num += w[k] * float(len(mine))
            den += w[k]
            for s in mine:
                g = int(maps[k][s])
                if g >= 0:
                    tally[g] = tally.get(g, 0.0) + w[k]
        n = int(np.floor(0.5 + num / den))
        best = sorted(tally, key=lambda g: (-tally[g], g))[:n]
        if len(best) > 0:
            out1[i] = best[0]
        if len(best) > 1:
            out2[i] = best[1]
    return dict(labels=out1, labels2=out2, order=order, weights=w, D=D, map=maps, n_global=ng, flags=flags, O=O, L=L,
                totals=totals, unique=unique)
