"""Float64 oracle of the random VB-HMM initialisation (DESIGN.md section 5.22; TEST INFRASTRUCTURE).

Philox4x64-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) in Python integers, vectorised
over numpy object arrays; the uniform, exponential and normalisation in float64; the restart choice.  Shares no code
with vbx_init_random or vbx_b200.random_init, and is itself checked against numpy's np.random.Philox."""
import hashlib
import math

import numpy as np

M64 = (1 << 64) - 1
PHILOX_M = (0xD2E7470EE14C6C93, 0xCA5A826395121157)
PHILOX_W = (0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B)


def philox4x64(counter, key, rounds=10):
    """Philox4x64-`rounds` of counters [..., 4] (Python ints or an object array) under key (k0, k1).  Returns an
    object array [..., 4] of the output words."""
    c = np.array(counter, dtype=object).reshape(-1, 4)
    c0, c1, c2, c3 = (c[:, i].copy() for i in range(4))
    k0, k1 = int(key[0]) & M64, int(key[1]) & M64
    for r in range(rounds):
        if r:
            k0, k1 = (k0 + PHILOX_W[0]) & M64, (k1 + PHILOX_W[1]) & M64
        p0 = c0 * PHILOX_M[0]
        p1 = c2 * PHILOX_M[1]
        c0, c1, c2, c3 = (p1 >> 64) ^ c1 ^ k0, p1 & M64, (p0 >> 64) ^ c3 ^ k1, p0 & M64
    return np.stack([c0, c1, c2, c3], axis=1).reshape(np.shape(counter))


def name_key(name):
    """First 8 bytes of SHA-256(name, UTF-8), little-endian."""
    return int.from_bytes(hashlib.sha256(name.encode('utf-8')).digest()[:8], 'little')


def exponentials(T, N, rec_key, seed):
    """e [T, 4 * ceil(N / 4)] float64: e[t, 4j + i] = -log(((w_i >> 11) + 0.5) 2^-53) with w = Philox4x64-10 of
    counter (t, j, rec_key, 0) and key (seed, 0)."""
    nb = (N + 3) // 4
    t, j = np.meshgrid(np.arange(T), np.arange(nb), indexing='ij')
    ctr = np.empty((T, nb, 4), dtype=object)
    ctr[..., 0] = t.astype(object)
    ctr[..., 1] = j.astype(object)
    ctr[..., 2] = int(rec_key)
    ctr[..., 3] = 0
    w = philox4x64(ctr, (seed, 0)) if T * nb else np.zeros((T, nb, 4), dtype=object)
    top = np.vectorize(lambda x: float(x >> 11), otypes=[np.float64])(w) if T * nb else np.zeros((T, nb, 4))
    u = (top + 0.5) * 2.0 ** -53
    return (-np.log(u)).reshape(T, 4 * nb)


def init_gamma(T, N, rec_key, seed, S=None):
    """(gamma0 [T, S], pi0 [S]) float64 of one recording: the exponentials of the N live states normalised per row, 0 in
    the padded columns; pi0 = 1 / N on the live states."""
    S = N if S is None else S
    e = exponentials(T, N, rec_key, seed)[:, :N]
    g = np.zeros((T, S))
    if N:
        g[:, :N] = e / e.sum(axis=1, keepdims=True)
    pi = np.zeros(S)
    pi[:N] = 1.0 / N if N else 0.0
    return g, pi


def restart_seed(seed, r):
    return (seed + r) & M64


def choose(Li, n_iters):
    """(restart index, final ELBOs) of one recording's restarts: final ELBO Li[r, n_iters[r] - 1] (NaN when a restart
    ran no iteration); the largest finite one wins, ties to the lowest r, restart 0 when none is finite."""
    final = [float(Li[r][n - 1]) if n > 0 else math.nan for r, n in enumerate(n_iters)]
    finite = [(v, -r) for r, v in enumerate(final) if math.isfinite(v)]
    return (-max(finite)[1] if finite else 0), final
