"""Float64 numpy/scipy restatement of the back-end training of DESIGN.md section 5.24 (vbx_b200/train.py), with a loop
per class and the EM in its textbook form (a d x d inverse per class) rather than in the jointly diagonal basis.  Test
infrastructure only: the package never imports it.

The rows enter the class statistics as float32, as the device's do: y and z are computed in float64 and rounded once."""
import math

import numpy as np
from scipy.linalg import cholesky, eigh, solve_triangular


def l2_norm(x):
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def class_stats(X, offsets):
    """(means [K, D], scatter [D, D]) of the rows X (promoted to float64) packed by class."""
    X = np.asarray(X, dtype=np.float64)
    K, D = len(offsets) - 1, X.shape[1]
    means, S = np.zeros((K, D)), np.zeros((D, D))
    for i in range(K):
        xi = X[offsets[i]:offsets[i + 1]]
        if len(xi):
            means[i] = xi.mean(0)
            c = xi - means[i]
            S += c.T @ c
    return means, S


def lda(Sw, Sb, d):
    """(eigenvalues [d] descending, lda [D, d]) of S_B v = lambda S_W v, v^T S_W v = 1, columns' largest entry > 0."""
    lam, V = eigh(Sb, Sw)
    lam, V = lam[::-1][:d], V[:, ::-1][:, :d]
    s = np.sign(V[np.argmax(np.abs(V), 0), np.arange(d)])
    return lam.copy(), V * s[None, :]


def objective(W, B, Mc, n, S):
    """The marginal log-likelihood of the training vectors given mu (not yet divided by N)."""
    d = W.shape[0]
    Wi = np.linalg.inv(W)
    ldw = np.linalg.slogdet(W)[1]
    L = -0.5 * np.trace(Wi @ S)
    for m, ni in zip(Mc, n):
        C = B + W / ni
        L += -0.5 * d * math.log(2 * math.pi) - 0.5 * np.linalg.slogdet(C)[1] - 0.5 * m @ np.linalg.solve(C, m)
        L += -(ni - 1) * d / 2 * math.log(2 * math.pi) - (ni - 1) / 2 * ldw - d / 2 * math.log(ni)
    return L


def plda_em(Mc, n, S, em_iters):
    """(W, B, objective trace / N): the two-covariance EM from W = S / N, B = mean m_i m_i^T."""
    N, K = float(np.sum(n)), len(n)
    W, B = S / N, Mc.T @ Mc / K
    trace = [objective(W, B, Mc, n, S) / N]
    for _ in range(em_iters):
        Wi, Bi = np.linalg.inv(W), np.linalg.inv(B)
        Bn, Wn = np.zeros_like(B), S.copy()
        for m, ni in zip(Mc, n):
            C = np.linalg.inv(Bi + ni * Wi)
            z = C @ (ni * Wi @ m)
            Bn += C + np.outer(z, z)
            Wn += ni * (C + np.outer(m - z, m - z))
        B, W = Bn / K, Wn / N
        B, W = 0.5 * (B + B.T), 0.5 * (W + W.T)
        trace.append(objective(W, B, Mc, n, S) / N)
    return W, B, trace


def kaldi_form(W, B):
    """(transform, psi): W = L L^T, L^-1 B L^-T = U diag(psi) U^T with psi descending, transform = U^T L^-1 with every
    row's largest-magnitude entry positive."""
    L = cholesky(W, lower=True)
    A = solve_triangular(L, solve_triangular(L, B, lower=True).T, lower=True)
    psi, U = np.linalg.eigh(0.5 * (A + A.T))
    psi, U = psi[::-1], U[:, ::-1]
    T = U.T @ np.linalg.inv(L)
    s = np.sign(T[np.arange(len(T)), np.argmax(np.abs(T), 1)])
    return T * s[:, None], psi.copy()


def train(xvectors, lda_dim=128, em_iters=10, min_per_speaker=2):
    """The whole training: {speaker: x [n, Dx]} -> dict of mean1, mean2, lda, lam, mu, W, B, transform, psi, trace."""
    kept = [np.asarray(x, dtype=np.float64) for x in xvectors.values() if len(x) >= min_per_speaker]
    n = np.array([len(x) for x in kept], dtype=np.float64)
    off = np.concatenate([[0], np.cumsum([len(x) for x in kept])]).astype(np.int64)
    x = np.concatenate(kept)
    N = float(len(x))
    mean1 = x.mean(0)
    y = l2_norm(x - mean1).astype(np.float32).astype(np.float64)
    my, Sw = class_stats(y, off)
    mu_y = n @ my / N
    Sb = sum(ni * np.outer(m - mu_y, m - mu_y) for m, ni in zip(my, n)) / N
    lam, A = lda(Sw / N, Sb, lda_dim)
    mean2 = (y @ A).mean(0)
    z = l2_norm(y @ A - mean2).astype(np.float32).astype(np.float64)
    mz, S = class_stats(z, off)
    mu = n @ mz / N
    W, B, trace = plda_em(mz - mu, n, S, em_iters)
    tr, psi = kaldi_form(W, B)
    return dict(mean1=mean1, mean2=mean2, lda=A, lam=lam, mu=mu, W=W, B=B, transform=tr, psi=psi, trace=trace,
                N=int(N), K=len(kept))
