"""TEST INFRASTRUCTURE ONLY - numpy restatement of the speaker-count rules of DESIGN.md section 5.14.

Only tests/ may import this.  The maxclust cut is scipy's own fcluster; masses are float64 sums.
"""
import numpy as np
from scipy.cluster.hierarchy import fcluster


def top2(gamma, states):
    """argsort(-gamma)[:, :2] restricted to the columns `states` (ascending): ties go to the lower state, second -1
    when there is one state (VBx/vbhmm.py:160-162)."""
    states = np.asarray(states, dtype=np.int64)
    order = np.argsort(-gamma[:, states], axis=1, kind='stable')
    first = states[order[:, 0]]
    second = states[order[:, 1]] if len(states) > 1 else np.full(len(gamma), -1, dtype=np.int64)
    return first, second


def keep_labels(gamma, n_states, keep):
    """Rule 2 for one recording: gamma [T, >= n_states] posteriors, the first n_states live.  Returns (first, second,
    mass): mass [n_states] float64 sums over frames; the `keep` states of largest mass survive (ties: lower index)."""
    g = np.asarray(gamma, dtype=np.float64)[:, :n_states]
    mass = g.sum(axis=0)
    kept = np.sort(np.argsort(-mass, kind='stable')[:keep])
    first, second = top2(g, kept)
    return first, second, mass


def maxclust(Z, T, k):
    """fcluster(Z, k, 'maxclust') - 1 (0-based), every x-vector on its own when T <= 1."""
    if T <= 1:
        return np.zeros(T, dtype=np.int64)
    return fcluster(Z, k, criterion='maxclust').astype(np.int64) - 1


def vb_rules(labels, labels2, gamma, lo, hi, Z, rerun):
    """Rules 1-3 for one recording of AHC+VB.  labels / labels2: the unconstrained output; gamma [T, S] its final
    posteriors over the live states; Z: the recording's linkage; rerun(init_labels) -> (labels, labels2) of the VB-HMM
    started from init_labels.  Returns (labels, labels2 or None, rule, K1)."""
    T = len(labels)
    k1 = len(np.unique(labels))
    if lo <= k1 <= hi:
        return labels, labels2, 'vb', k1
    if k1 > hi:
        f, s, _ = keep_labels(gamma, gamma.shape[1], hi)
        return f, (s if hi > 1 else None), 'mass', k1
    mc = maxclust(Z, T, lo)
    if T < lo:
        return mc, None, 'unmet', k1
    r1, r2 = rerun(mc)
    if len(np.unique(r1)) >= lo:
        return r1, r2, 'recut', k1
    return mc, None, 'ahc', k1


def ahc_rules(labels, lo, hi, Z):
    """Rule 4 (init='AHC'): labels of the threshold cut -> (labels, rule, K1)."""
    T = len(labels)
    k1 = len(np.unique(labels))
    if lo <= k1 <= hi:
        return labels, 'vb', k1
    return maxclust(Z, T, hi if k1 > hi else lo), 'unmet' if T < lo else 'ahc', k1
