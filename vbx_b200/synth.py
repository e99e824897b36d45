"""Seeded synthetic x-vector batches shaped like the reference's inputs (SURVEY.md section 8d).

A recording is a sticky Markov chain over a few speakers; each frame is the speaker's mean (drawn
from the PLDA across-class prior N(0, diag Phi)) plus unit within-class noise - exactly the
generative model VBx assumes (VBx/VBx.py:33-36).  Raw D-dim x-vectors are built so that one
projection V (D x R) maps them to `rho`:  X @ V0 = fea,  V = V0 * sqrt(Phi),  rho = X @ V.
"""
import math

import numpy as np


def plda_phi(R=128):
    """Across-class variances spanning the range of the shipped 16 kHz PLDA (5.60 ... 0.534)."""
    return np.exp(np.linspace(math.log(5.6), math.log(0.53), R))


def projection_basis(D=256, R=128, seed=1234):
    """Fixed D x R matrix with orthonormal columns."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((D, R)))
    return q


def make_recording(T, R, Phi, rng, stay=0.99, n_spk=None):
    """-> fea (T x R float64), path (T,) of true speaker ids."""
    n_spk = int(rng.integers(2, 9)) if n_spk is None else n_spk
    means = rng.standard_normal((n_spk, R)) * np.sqrt(Phi)[None, :]
    switch = rng.random(T) >= stay
    jump = rng.integers(0, n_spk, size=T)
    z = np.empty(T, dtype=np.int64)
    cur = int(jump[0])
    for t in range(T):
        if switch[t]:
            cur = int(jump[t])
        z[t] = cur
    fea = means[z] + rng.standard_normal((T, R))
    return fea, z


def dirichlet_rows(T, S, rng, conc=1.0):
    """Flat-Dirichlet responsibilities like the reference's default init (VBx/VBx.py:82-83)."""
    g = rng.gamma(conc, size=(T, S))
    return g / g.sum(axis=1, keepdims=True)


def make_batch(lengths, R=128, S=16, seed=0, D=None, dtype=np.float32):
    """Packed ragged batch.  Returns dict with
       fea   [N, R]   (the reference's `X` argument, per recording slices)
       X     [N, D]   raw x-vectors (only if D is given) and V [D, R] with rho = X @ V
       Phi   [R], gamma0 [N, S], offsets [B+1] (int64), paths [N]"""
    Phi = plda_phi(R)
    lengths = [int(t) for t in lengths]
    offsets = np.zeros(len(lengths) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum(lengths)
    N = int(offsets[-1])
    fea = np.empty((N, R), dtype=np.float64)
    gamma0 = np.empty((N, S), dtype=np.float64)
    paths = np.empty(N, dtype=np.int64)
    for b, T in enumerate(lengths):
        rng = np.random.default_rng(seed * 1000003 + b)
        f, z = make_recording(T, R, Phi, rng)
        lo, hi = offsets[b], offsets[b + 1]
        fea[lo:hi] = f
        paths[lo:hi] = z
        gamma0[lo:hi] = dirichlet_rows(T, S, rng)
    out = {'fea': fea.astype(dtype), 'Phi': Phi.astype(dtype), 'gamma0': gamma0.astype(dtype),
           'offsets': offsets, 'paths': paths}
    if D is not None:
        V0 = projection_basis(D, R)
        rng = np.random.default_rng(seed * 7919 + 17)
        noise = rng.standard_normal((N, D))
        noise -= (noise @ V0) @ V0.T                      # keep only the null-space of V0^T
        out['X'] = (out['fea'].astype(np.float64) @ V0.T + 0.5 * noise).astype(dtype)
        out['V'] = (V0 * np.sqrt(Phi)[None, :]).astype(dtype)
    return out


def make_scoring_archive(lengths, seed=0, n_spk=(2, 9), stay=0.97, gap_prob=0.0):
    """Seeded recordings with ground-truth speaker labels for DER scoring, shaped like an x-vector archive: 1.5 s segments
    every 0.24 s, after a segment a pause of 1.5 .. 4.5 s with probability gap_prob (times on a 10 ms grid), and a sticky
    speaker chain over n_spk[0] .. n_spk[1]-1 speakers.  Returns {name: (seg_times [T,2] seconds, labels int64 [T])};
    the reference turns are the merged label segments (pipeline.merge_adjacent_labels), so the labels score DER 0."""
    rng = np.random.default_rng(seed)
    out = {}
    for r, T in enumerate(lengths):
        T = int(T)
        K = int(rng.integers(n_spk[0], n_spk[1]))
        step = np.where(rng.random(T) < gap_prob, rng.integers(150, 451, T) + 150, 24)     # centiseconds
        start = np.concatenate([[0], np.cumsum(step[:-1])]) if T else np.zeros(0, dtype=np.int64)
        lab = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            lab[t] = lab[t - 1] if rng.random() < stay else rng.integers(K)
        out[f'syn{r:02d}'] = (np.stack([start / 100.0, (start + 150) / 100.0], 1).reshape(-1, 2), lab)
    return out


def multi_session_archive(x_ref, n_rec=8, pool=10, lengths=(300, 600), speakers=(2, 5), seed=13, stay=0.97):
    """Seeded recordings whose speakers are drawn from one shared pool, as in an archive of meetings with recurring
    participants (speaker linking, DESIGN.md sections 5.15 and 5.18).  x_ref [n, D]: real x-vectors whose mean and
    per-dimension spread place the pool: speaker k's centre is mean + 2 sd * N(0, 1), its x-vectors the centre plus
    0.5 sd * N(0, 1) noise.  Each recording has lengths[0] .. lengths[1] x-vectors (1.5 s segments every 0.24 s) and
    speakers[0] .. speakers[1] distinct pool speakers with sticky turns.  Returns (recordings {name: (x [T,D] float64,
    seg_times [T,2])}, reference rows [(recording, onset, duration, 'p<k>')], one 0.24 s row per x-vector, and the pool
    index of every x-vector {name: int64 [T]})."""
    rng = np.random.default_rng(seed)
    x_ref = np.asarray(x_ref, dtype=np.float64)
    sd = x_ref.std(0)
    centres = x_ref.mean(0) + 2.0 * sd * rng.standard_normal((pool, x_ref.shape[1]))
    recs, rows, truth = {}, [], {}
    for r in range(n_rec):
        T = int(rng.integers(lengths[0], lengths[1] + 1))
        who = rng.choice(pool, int(rng.integers(speakers[0], speakers[1] + 1)), replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < stay else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_ref.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        name = f'ses{r:02d}'
        recs[name] = (x, seg)
        truth[name] = who[spk]
        rows += [(name, round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    return recs, rows, truth
