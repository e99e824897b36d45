"""Speaker linking across recordings (DESIGN.md section 5.15) restated in numpy float64 and scipy (test infrastructure;
product code never imports it): per-speaker statistics, the closed-form same-speaker LLR, the cannot-link distances,
scipy's average linkage and its fcluster cut."""
import numpy as np
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.spatial.distance import squareform

BIG = 1e30


def statistics(fea, speaker, M):
    """n [M] and F [M,R] float64: the x-vectors whose speaker index (in [0, M), -1 = none) is s, and their feature sum."""
    fea = np.asarray(fea, dtype=np.float64)
    speaker = np.asarray(speaker, dtype=np.int64)
    n = np.zeros(M)
    F = np.zeros((M, fea.shape[1]))
    ok = (speaker >= 0) & (speaker < M)
    np.add.at(n, speaker[ok], 1.0)
    np.add.at(F, speaker[ok], fea[ok])
    return n, F


def llr(n, F, Phi, c):
    """LLR [M,M] of every pair of speakers with statistics n [M], F [M,R] under c = Fa / Fb (0 where either n is 0)."""
    n = np.asarray(n, dtype=np.float64)
    Phi = np.asarray(Phi, dtype=np.float64)
    L = 1.0 + c * n[:, None] * Phi[None, :]
    b = c * np.sqrt(Phi)[None, :] * np.asarray(F, dtype=np.float64)
    e = np.sum(b * b / L - np.log(L), axis=1)
    out = np.zeros((len(n), len(n)))
    for s in range(len(n)):
        Lsu = L[s][None, :] + L - 1.0
        x = b[s][None, :] + b
        out[s] = 0.5 * (np.sum(x * x / Lsu - np.log(Lsu), axis=1) - e[s] - e)
    out[(n[:, None] == 0) | (n[None, :] == 0)] = 0.0
    return out


def distances(n, F, Phi, c, speaker_rec):
    """-LLR, BIG between two speakers of one recording, 0 on the diagonal."""
    d = -llr(n, F, Phi, c)
    rec = np.asarray(speaker_rec)
    d[rec[:, None] == rec[None, :]] = BIG
    np.fill_diagonal(d, 0.0)
    return d


def link(d):
    """scipy's average linkage of the distance matrix d [M,M]."""
    return linkage(squareform(d, checks=False), method='average')


def partition(Z, threshold):
    """fcluster(Z, -threshold, 'distance'): the speakers whose average LLR is at least `threshold` share a cluster.
    fcluster refuses negative heights, so heights and cut are shifted by the same amount (the same merges lie below)."""
    Z = np.array(Z, dtype=np.float64)
    k = max(0.0, -float(Z[:, 2].min())) if len(Z) else 0.0
    Z[:, 2] += k
    return fcluster(Z, -threshold + k, criterion='distance')
