"""CPU oracle of enrolled speakers in live streams (TEST INFRASTRUCTURE - never on the product path; DESIGN.md section
5.29), on the state of oracle/stream_oracle.StreamOracle.

After a push's commit, for one stream with its names {label: enrolled index}:
  candidates  the speakers of the push's block (its final labels) that are not yet named, in increasing label order;
  statistics  n = n_hist[k] + the ring rows labelled k, F = F_hist[k] + those rows added oldest first in float64: every
              x-vector the stream has given speaker k (the history holds the rows that left the ring);
  scores      section 5.15's LLR of every candidate against every enrolled speaker (enroll_oracle.llr, c = Fa / Fb);
  assignment  scipy's linear_sum_assignment of enroll_oracle.cost over the enrolled speakers the stream has not
              claimed (the claimed columns removed): a name only where LLR >= threshold; best LLR = the assigned pair's,
              or for an unnamed candidate its largest LLR over the unclaimed enrolled speakers (-inf when none is left);
  prior       with prior, a speaker named now gets n_hist[k] += n_e, F_hist[k] += F_e.
Named speakers keep their names and are never scored again.
"""
import numpy as np
from scipy.optimize import linear_sum_assignment

from oracle import enroll_oracle


def candidate_stats(n_hist, F_hist, ring_fea, ring_lab, ks):
    """n [len(ks)], F [len(ks), R] float64: the history of each speaker plus its ring rows, oldest first."""
    n = np.array([float(n_hist[k]) for k in ks])
    F = np.array([np.asarray(F_hist[k], dtype=np.float64) for k in ks]).reshape(len(ks), np.shape(F_hist)[1])
    for x, l in zip(np.asarray(ring_fea, dtype=np.float64), np.asarray(ring_lab).tolist()):
        if l in ks:
            j = ks.index(l)
            n[j] += 1.0
            F[j] = F[j] + x
    return n, F


def assign(llr, claimed, threshold):
    """(assign [M] enrolled index or -1, best [M]) of one stream's candidates with LLRs llr [M, E], the enrolled
    speakers in `claimed` removed."""
    M, E = llr.shape
    free = np.array([e for e in range(E) if e not in set(claimed)], dtype=np.int64)
    out, best = np.full(M, -1, dtype=np.int64), np.full(M, -np.inf)
    if M == 0 or len(free) == 0:
        return out, best
    sub = llr[:, free]
    r, col = linear_sum_assignment(enroll_oracle.cost(sub, threshold))
    for i, j in zip(r.tolist(), col.tolist()):
        if j < len(free):
            out[i] = free[j]
    best = np.where(out >= 0, llr[np.arange(M), np.maximum(out, 0)], sub.max(axis=1))
    return out, best


def name_push(stream, names, block_labels, n_e, F_e, Phi, c, threshold, prior=False):
    """Steps of the module docstring for one StreamOracle `stream` after its commit of a block with final labels
    block_labels; names {label: enrolled index} is updated in place, and with prior stream.n_hist / F_hist.  Returns
    dict(candidates, n, F, llr, assign, best)."""
    ks = [k for k in np.unique(np.asarray(block_labels, dtype=np.int64)).tolist() if k not in names]
    n, F = candidate_stats(stream.n_hist, stream.F_hist, stream.ctx_fea, stream.ctx_lab, ks)
    if not ks:
        return dict(candidates=ks, n=n, F=F, llr=np.zeros((0, len(n_e))), assign=np.zeros(0, dtype=np.int64),
                    best=np.zeros(0))
    llr = enroll_oracle.llr(n, F, np.asarray(n_e, dtype=np.float64), np.asarray(F_e, dtype=np.float64),
                            np.asarray(Phi, dtype=np.float64), c)
    a, best = assign(llr, list(names.values()), threshold)
    for k, e in zip(ks, a.tolist()):
        if e >= 0:
            names[k] = e
            if prior:
                stream.n_hist[k] += n_e[e]
                stream.F_hist[k] = stream.F_hist[k] + np.asarray(F_e[e], dtype=np.float64)
    return dict(candidates=ks, n=n, F=F, llr=llr, assign=a, best=best)
