"""numpy float64 restatement of the turn initialisation of VB resegmentation (DESIGN.md section 5.20, vbx_init_turns).
Coverage by brute-force interval intersection (every segment against every turn), not by the kernel's prefix sums."""
import numpy as np


def coverage(seg, turns):
    """seg [T,2] int64 ticks; turns: per speaker (lo, hi) int64 ticks, sorted and disjoint -> c [T,K] float64, c[t,k] =
    (ticks of [seg lo, seg hi) inside speaker k's turns) / (seg hi - seg lo), 0 for a segment of no positive length."""
    seg = np.asarray(seg, dtype=np.int64).reshape(-1, 2)
    c = np.zeros((len(seg), len(turns)), dtype=np.float64)
    length = seg[:, 1] - seg[:, 0]
    for k, (lo, hi) in enumerate(turns):
        lo, hi = np.asarray(lo, dtype=np.int64), np.asarray(hi, dtype=np.int64)
        inter = np.minimum(seg[:, 1:2], hi[None, :]) - np.maximum(seg[:, 0:1], lo[None, :])
        covered = np.maximum(inter, 0).sum(1)
        c[:, k] = np.where(length > 0, covered / np.where(length > 0, length, 1), 0.0)
    return c


def init_gamma(seg, turns, smoothing, S=None):
    """gamma0 [T,S] = softmax(smoothing * coverage) over the K = len(turns) speakers, 0 in columns K .. S-1, and
    pi0 [S] = 1/K on the first K columns."""
    c = coverage(seg, turns)
    K = c.shape[1]
    S = K if S is None else S
    g = np.zeros((c.shape[0], S), dtype=np.float64)
    pi = np.zeros(S, dtype=np.float64)
    if K:
        z = smoothing * c
        e = np.exp(z - z.max(1, keepdims=True))
        g[:, :K] = e / e.sum(1, keepdims=True)
        pi[:K] = 1.0 / K
    return g, pi
