"""CPU oracle of streaming diarization (TEST INFRASTRUCTURE - never on the product path; DESIGN.md section 5.25).

One `StreamOracle` is one stream.  Its state: K speakers so far (speaker k is spk<k+1> for the stream's life), the
projected features `fea` of its last min(C, pushed) x-vectors and their final labels (the context), and the history
n_hist[k], F_hist[k] = sum of fea over the x-vectors that have LEFT the context, by final label, float64, summed
sequentially in time order.

A push delivers a block of h >= 1 x-vectors, as the transformed x-vectors `x` (the AHC input) and the projected
features `fea`:
  1. AHC of the block alone (ahc_oracle), cut at `threshold`: c clusters; if K + c > S_max the maxclust cut at S_max - K
     (scipy fcluster 'maxclust'), and c = 0 when K = S_max (the block rows then start uniform over the K states);
  2. the window [context rows; block rows] with K + c states: context rows start on their final label, block rows on
     K + cluster; gamma0 = softmax(smoothing * onehot), pi0 = 1 / (K + c); states k < K carry the prior
     (n_hist[k], F_hist[k]), fresh states none;
  3. the VB-HMM with that prior (prior_oracle.vbx_prior_oracle) over the window, and hard labels (first best, ties to
     the lower state);
  4. commit: a block row on a state k < K is speaker k; fresh states that hold block rows become speakers K, K+1, ... in
     order of their first row; the block enters the context, and the rows pushed out of it add (1, fea) to n_hist /
     F_hist in time order.  Context rows are never relabelled.
Context x-vectors enter the window once, as frames, and older x-vectors once, through the prior.  A fresh stream's
first push is therefore the offline AHC + VB-HMM of its block.
"""
import numpy as np
from scipy.cluster.hierarchy import fcluster

from oracle.ahc_oracle import ahc_labels
from oracle.prior_oracle import vbx_prior_oracle


def block_ahc(x, threshold):
    """The threshold cut of the block's AHC as the device path makes it: one x-vector is one cluster, and a NaN
    calibration leaves every x-vector on its own.  Returns (labels, Z) (Z None for one x-vector)."""
    x = np.asarray(x, dtype=np.float64)
    if len(x) == 1:
        return np.zeros(1, dtype=np.int64), None
    labels, thr, Z = ahc_labels(x, threshold)
    if not np.isfinite(thr):
        return np.arange(len(x), dtype=np.int64), Z
    return np.asarray(labels, dtype=np.int64), Z


def nonnegative(Z):
    """Z with its heights shifted to start at 0 (VBx/vbhmm.py:142-143; scipy refuses negative heights, and a shift does not
    change a maxclust cut)."""
    Z = np.array(Z, dtype=np.float64)
    Z[:, 2] += abs(Z[:, 2].min())
    return Z


def soft_init(labels, n, smoothing):
    """softmax(smoothing * onehot(labels)) over n states in float64; label -1 gives a uniform row."""
    q = np.zeros((len(labels), n))
    hot = labels >= 0
    q[np.nonzero(hot)[0], labels[hot]] = smoothing
    q = np.exp(q - q.max(1, keepdims=True))
    return q / q.sum(1, keepdims=True)


class StreamOracle:
    def __init__(self, Phi, Fa, Fb, loopP, threshold=-0.015, smoothing=5.0, context=240, max_speakers=64,
                 max_iters=40, epsilon=1e-6):
        self.Phi = np.asarray(Phi, dtype=np.float64)
        self.Fa, self.Fb, self.loopP = Fa, Fb, loopP
        self.threshold, self.smoothing, self.C, self.S_max = threshold, smoothing, context, max_speakers
        self.max_iters, self.epsilon = max_iters, epsilon
        R = len(self.Phi)
        self.K = 0
        self.ctx_fea = np.zeros((0, R))
        self.ctx_lab = np.zeros(0, dtype=np.int64)
        self.n_hist = np.zeros(max_speakers)
        self.F_hist = np.zeros((max_speakers, R))
        self.final_fea, self.final_lab = [], []       # every committed row, for the statistics identity

    def clusters(self, x):
        """Step 1: (block labels, c)."""
        labels, Z = block_ahc(x, self.threshold)
        c = int(labels.max()) + 1
        if self.K + c > self.S_max:
            if self.K >= self.S_max:
                return np.full(len(labels), -1, dtype=np.int64), 0
            labels = fcluster(nonnegative(Z), self.S_max - self.K, criterion='maxclust').astype(np.int64) - 1
            c = int(labels.max()) + 1
        return labels, c

    def window(self, fea, labels, c):
        """Step 2: dict(fea, gamma0, pi0, n_states, prior_n, prior_F, L) of the window (float64)."""
        ns = self.K + c
        fea_w = np.vstack([self.ctx_fea, np.asarray(fea, dtype=np.float64)])
        lab = np.concatenate([self.ctx_lab, np.where(labels >= 0, self.K + labels, -1)])
        pn, pF = np.zeros(ns), np.zeros((ns, len(self.Phi)))
        pn[:self.K], pF[:self.K] = self.n_hist[:self.K], self.F_hist[:self.K]
        return dict(fea=fea_w, gamma0=soft_init(lab, ns, self.smoothing), pi0=np.full(ns, 1.0 / ns), n_states=ns,
                    prior_n=pn, prior_F=pF, L=len(self.ctx_lab))

    def commit(self, first_block, fea):
        """Step 4 from the block rows' window labels; returns the block's final labels."""
        first_block = np.asarray(first_block, dtype=np.int64)
        new = {}
        for w in first_block.tolist():
            if w >= self.K and w not in new:
                new[w] = self.K + len(new)
        final = np.array([w if w < self.K else new[w] for w in first_block.tolist()], dtype=np.int64)
        self.K += len(new)
        fea = np.asarray(fea, dtype=np.float64)
        all_fea = np.vstack([self.ctx_fea, fea])
        all_lab = np.concatenate([self.ctx_lab, final])
        out = len(all_lab) - min(self.C, len(all_lab))
        for t in range(out):                          # sequential float64 sums in time order
            self.n_hist[all_lab[t]] += 1.0
            self.F_hist[all_lab[t]] += all_fea[t]
        self.ctx_fea, self.ctx_lab = all_fea[out:], all_lab[out:]
        self.final_fea.append(fea)
        self.final_lab.append(final)
        return final

    def push(self, x, fea, clusters=None):
        """One push of the block (x transformed [h, dx], fea projected [h, R]).  clusters: None, or the (labels, c) of
        step 1 to use instead of the oracle's own AHC.  Returns dict(labels, iterations, window, gamma, pi)."""
        labels, c = self.clusters(x) if clusters is None else clusters
        w = self.window(fea, np.asarray(labels, dtype=np.int64), c)
        gamma, pi, Li = vbx_prior_oracle(w['fea'], self.Phi, w['prior_n'], w['prior_F'], loopProb=self.loopP, Fa=self.Fa,
                                         Fb=self.Fb, pi=w['pi0'], gamma=w['gamma0'], maxIters=self.max_iters,
                                         epsilon=self.epsilon)
        first = np.argsort(-gamma, axis=1, kind='stable')[:, 0]
        final = self.commit(first[w['L']:], fea)
        return dict(labels=final, iterations=len(Li), window=w, gamma=gamma, pi=pi, first=first)
