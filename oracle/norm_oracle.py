"""Score normalisation against a cohort (DESIGN.md section 5.17) restated in numpy float64 and scipy (test
infrastructure; product code never imports it): cohort LLRs, the mean and population standard deviation of each
speaker's top-K cohort scores, the normalised score S, the normalised link distances with scipy's average linkage and
fcluster cut, and the normalised enrolment assignment by linear_sum_assignment."""
import numpy as np

from oracle import enroll_oracle, link_oracle


def cohort_llr(n, F, n_c, F_c, Phi, c):
    """LLR [M,C] of every scored speaker against every cohort speaker: section 5.15's score (enroll_oracle.llr)."""
    return enroll_oracle.llr(n, F, n_c, F_c, Phi, c)


def top_stats(scores, top_k):
    """(mean [M], std [M]) of each row's K = min(top_k, C) largest values, std with ddof 0."""
    scores = np.asarray(scores, dtype=np.float64)
    K = min(int(top_k), scores.shape[1])
    top = -np.sort(-scores, axis=1)[:, :K]
    return top.mean(axis=1), top.std(axis=1)


def normalise(llr, mean_r, std_r, mean_c, std_c):
    """S [rows, cols] = 1/2 [ (LLR - mu_row) / sigma_row + (LLR - mu_col) / sigma_col ]."""
    llr = np.asarray(llr, dtype=np.float64)
    return 0.5 * ((llr - mean_r[:, None]) / std_r[:, None] + (llr - mean_c[None, :]) / std_c[None, :])


def link_distances(n, F, Phi, c, speaker_rec, mean, std):
    """-S, BIG between two speakers of one recording, 0 on the diagonal."""
    d = -normalise(link_oracle.llr(n, F, Phi, c), mean, std, mean, std)
    rec = np.asarray(speaker_rec)
    d[rec[:, None] == rec[None, :]] = link_oracle.BIG
    np.fill_diagonal(d, 0.0)
    return d


def link(d):
    return link_oracle.link(d)


def partition(Z, threshold):
    return link_oracle.partition(Z, threshold)


def assign(S, rec_offsets, threshold):
    """enroll_oracle.assign on the normalised scores S [M,E]."""
    return enroll_oracle.assign(S, rec_offsets, threshold)
