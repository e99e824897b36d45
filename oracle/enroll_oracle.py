"""Enrolment against known speakers (DESIGN.md section 5.16) restated in numpy float64 and scipy (test infrastructure;
product code never imports it): statistics of archive and enrolled speakers, the rectangular LLR, the cost matrix of
each recording, scipy's linear_sum_assignment and the naming rule."""
import numpy as np
from scipy.optimize import linear_sum_assignment

from oracle import link_oracle


def llr(n, F, n_e, F_e, Phi, c):
    """LLR [M,E] of every archive speaker (n [M], F [M,R]) against every enrolled speaker (n_e [E], F_e [E,R]):
    section 5.15's score on the stacked speakers."""
    M = len(n)
    full = link_oracle.llr(np.concatenate([n, n_e]), np.vstack([F, F_e]), Phi, c)
    return full[:M, M:]


def cost(llr_rec, threshold):
    """C [K, E + K] of one recording: threshold - LLR for the enrolled columns, 0 for the K unknown columns."""
    K = llr_rec.shape[0]
    return np.hstack([threshold - llr_rec, np.zeros((K, K))])


def assign(llr_all, rec_offsets, threshold):
    """(assign [M] enrolled index or -1, objective per recording) from scipy's linear_sum_assignment of each recording's
    cost matrix; rec_offsets [n_rec+1] gives each recording's speakers."""
    M, E = llr_all.shape
    out = np.full(M, -1, dtype=np.int64)
    obj = []
    for a, b in zip(rec_offsets[:-1], rec_offsets[1:]):
        if b == a:
            obj.append(0.0)
            continue
        C = cost(llr_all[a:b], threshold)
        r, col = linear_sum_assignment(C)
        out[a + r] = np.where(col < E, col, -1)
        obj.append(float(C[r, col].sum()))
    return out, np.array(obj)


def objective(llr_all, rec_offsets, threshold, assignment):
    """The cost of an assignment per recording: sum of threshold - LLR over its named speakers."""
    return np.array([sum(threshold - llr_all[s, assignment[s]] for s in range(a, b) if assignment[s] >= 0)
                     for a, b in zip(rec_offsets[:-1], rec_offsets[1:])], dtype=np.float64)


def names(rec, label, assignment, enrolled, recordings, labels2=None):
    """Per recording {label: name}: the enrolled name, or unknown-<recording>-<label+1>; a label used only as a second
    label (labels2: per recording None or an int array) is unknown."""
    out = [{} for _ in recordings]
    for b, l, a in zip(rec, label, assignment):
        out[b][int(l)] = enrolled[a] if a >= 0 else f'unknown-{recordings[b]}-{int(l) + 1}'
    for b, l2 in enumerate(labels2 or []):
        for l in ([] if l2 is None else np.unique(np.asarray(l2)).tolist()):
            if l >= 0 and l not in out[b]:
                out[b][l] = f'unknown-{recordings[b]}-{l + 1}'
    return out
