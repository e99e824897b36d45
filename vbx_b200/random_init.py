"""Random initialisation of the VB-HMM with restarts (init='RANDOM+VB', DESIGN.md section 5.22): the host side.

Recording b, restart r starts from gamma0 rows drawn by vbx_init_random with the recording's key (name_key: the first
8 bytes, little-endian, of SHA-256 of its name) and the seed (seed + r) mod 2^64, so a recording draws the same numbers
in any archive and restart r of seed s is restart 0 of seed s + r.  After the VB-HMM every recording keeps the restart
with the largest final ELBO (best_restart)."""
import hashlib
import math
from collections import namedtuple

import numpy as np

SEED_LIMIT = 1 << 64

# What _vb_stage needs: init_states N, restarts R, seed, and one name_key per recording of the archive.
RandomStart = namedtuple('RandomStart', 'n_states restarts seed keys')


def name_key(name):
    """The recording's stream key: the first 8 bytes, little-endian, of SHA-256 of its name (UTF-8)."""
    return int.from_bytes(hashlib.sha256(str(name).encode('utf-8')).digest()[:8], 'little')


def restart_seed(seed, r):
    """The Philox key of restart r: (seed + r) mod 2^64."""
    return (int(seed) + int(r)) % SEED_LIMIT


def _is_int(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))


def check_options(init, init_states, restarts, seed):
    """ValueError unless init_states / restarts / seed fit init: with 'RANDOM+VB' init_states is an int >= 1 (required),
    restarts an int >= 1 and seed an int in [0, 2^64) (None: 1 and 0); with any other init all three are None.
    Returns RandomStart(N, R, seed, None) for 'RANDOM+VB', else None."""
    if init != 'RANDOM+VB':
        given = [k for k, v in (('init_states', init_states), ('restarts', restarts), ('seed', seed)) if v is not None]
        if given:
            raise ValueError(f"{', '.join(given)}: options of init='RANDOM+VB', not of init={init!r}")
        return None
    if init_states is None:
        raise ValueError("init='RANDOM+VB' needs init_states, the number of HMM states to start from (no default)")
    if not _is_int(init_states) or init_states < 1:
        raise ValueError(f'init_states must be an integer >= 1, got {init_states!r}')
    restarts = 1 if restarts is None else restarts
    if not _is_int(restarts) or restarts < 1:
        raise ValueError(f'restarts must be an integer >= 1, got {restarts!r}')
    seed = 0 if seed is None else seed
    if not _is_int(seed) or not 0 <= seed < SEED_LIMIT:
        raise ValueError(f'seed must be an integer in [0, 2**64), got {seed!r}')
    return RandomStart(int(init_states), int(restarts), int(seed), None)


def final_elbo(Li, n_iters):
    """Each entry's final ELBO Li[e, n_iters[e] - 1] (NaN for an entry that ran no iteration).  Li [E, maxIters],
    n_iters [E]: host arrays."""
    Li = np.asarray(Li, dtype=np.float64)
    n = np.asarray(n_iters, dtype=np.int64)
    out = np.full(len(n), np.nan)
    ran = n > 0
    out[ran] = Li[np.nonzero(ran)[0], n[ran] - 1]
    return out


def best_restart(elbos):
    """The restart to keep: the largest finite final ELBO, ties to the lowest index; 0 when none is finite."""
    best, r_best = -math.inf, 0
    for r, v in enumerate(elbos):
        if math.isfinite(v) and v > best:
            best, r_best = v, r
    return r_best
