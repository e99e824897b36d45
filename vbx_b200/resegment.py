"""VB resegmentation (DESIGN.md section 5.20): the VB-HMM started from a diarization the user already has (another
system's output, an earlier run, a partial manual annotation) instead of this project's AHC, init='RTTM+VB'.

Every speaker of a recording in the init RTTM is one HMM state, in name order (score.named_turns, the grouping of
score.named_reference_turns without its 64-speaker cap).  X-vector t with segment [lo, hi) ticks starts from
gamma0[t] = softmax(smoothing * c), c_k the share of [lo, hi) inside speaker k's turns (vbx_init_turns): a segment one
speaker covers gets the reference's qinit row (VBx/vbhmm.py:150-152), one two speakers cover splits its mass between
them, and one nobody covers gets a uniform row, so a partial annotation needs no special case.

This module holds the host side: reading and checking the init RTTM, and packing the turns of a batch's entries into
the arrays vbx_init_turns takes.
"""
import os
from collections import namedtuple

import numpy as np

# The turns of a batch of entries, packed for vbx_init_turns (HOST int64 arrays): seg [N,2] ticks; spk_off [B+1] (entry b
# has speakers spk_off[b] .. spk_off[b+1]-1); turn_off [n_spk+1]; turn_lo, turn_hi [n_turns] each speaker's sorted,
# disjoint turns; turn_cum [n_turns] the exclusive prefix sum of the turn lengths within each speaker.
TurnPack = namedtuple('TurnPack', 'seg spk_off turn_off turn_lo turn_hi turn_cum')


def load_init(init_rttm, names):
    """The init turns of the recordings `names`: {name: [(speaker name, (lo, hi) merged ticks)]}, speakers in name
    order.  init_rttm: an RTTM file or directory of *.rttm (score.read_rttm_path) or formats.read_rttm rows.  Recordings
    the RTTM lacks, or in which it has no speaker with a non-empty turn, raise ValueError naming them; RTTM recordings
    outside `names` are ignored."""
    from . import score
    rows = score.read_rttm_path(init_rttm) if isinstance(init_rttm, (str, os.PathLike)) else list(init_rttm)
    wanted = set(names)
    turns = score.named_turns([r for r in rows if r[0] in wanted])
    missing = [n for n in names if n not in turns]
    if missing:
        raise ValueError(f'recordings missing from the init RTTM: {missing}')
    empty = [n for n in names if not turns[n]]
    if empty:
        raise ValueError(f'recordings without a speaker in the init RTTM: {empty}')
    return {n: turns[n] for n in names}


def pack_turns(items):
    """items: one (seg_times [T,2] seconds, load_init speaker list) per entry of a batch, in batch order -> TurnPack."""
    from .score import to_ticks
    z = np.zeros(0, dtype=np.int64)
    seg = [to_ticks(np.asarray(s, dtype=np.float64).reshape(-1, 2)) for s, _ in items]
    spk = [t for _, turns in items for _, t in turns]
    n_turns = np.array([len(lo) for lo, _ in spk], dtype=np.int64)
    cum = [np.concatenate([[0], np.cumsum(hi - lo)[:-1]]).astype(np.int64) for lo, hi in spk]
    return TurnPack(seg=np.concatenate(seg) if seg else np.zeros((0, 2), dtype=np.int64),
                    spk_off=np.concatenate([[0], np.cumsum([len(t) for _, t in items])]).astype(np.int64),
                    turn_off=np.concatenate([[0], np.cumsum(n_turns)]).astype(np.int64),
                    turn_lo=np.concatenate([lo for lo, _ in spk] + [z]).astype(np.int64),
                    turn_hi=np.concatenate([hi for _, hi in spk] + [z]).astype(np.int64),
                    turn_cum=np.concatenate(cum + [z]))


def speaker_names(turns):
    """The state names of one recording's load_init speaker list: the init RTTM's name of each state."""
    return [k for k, _ in turns]
