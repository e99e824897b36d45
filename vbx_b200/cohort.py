"""Score normalisation against a cohort (DESIGN.md section 5.17).

The same-speaker LLR of section 5.15 is not calibrated: it grows with the number of x-vectors and with a speaker's
offset from the PLDA mean, so one threshold means different things for different speakers and archives.  Adaptive
symmetric normalisation (AS-norm) standardises every score by the scores of both speakers against a cohort of speakers
known to be someone else: speaker x scores LLR(x, c) against each cohort speaker c, mu_x and sigma_x are the mean and
population standard deviation of its K = min(top_k, C) largest cohort scores (on the device, vbx_cohort_stats_batch),
and

    S(x, y) = 1/2 [ (LLR(x, y) - mu_x) / sigma_x + (LLR(x, y) - mu_y) / sigma_y ].

link.link_speakers and enroll.enroll_speakers take the statistics (norm=) and then decide on S.
"""
import ctypes
from collections import namedtuple

import numpy as np

DEFAULT_TOP_K = 200        # a conventional AS-norm value, not tuned here; top_k >= C is plain S-norm
SIGMA_MIN = 1e-6           # smallest accepted sigma_x (DESIGN.md section 5.17: keeps |S| far below the cannot-link regime)

# mean [M], std [M] float64 numpy; K = min(top_k, C); scores [M,C] or None
CohortStats = namedtuple('CohortStats', 'mean std K scores')


def check_top_k(top_k):
    """top_k as an int; ValueError below 2 (one score has no spread)."""
    if isinstance(top_k, (bool, np.bool_)) or not isinstance(top_k, (int, np.integer)) or top_k < 2:
        raise ValueError(f'cohort top_k must be an integer >= 2, got {top_k!r}')
    return int(top_k)


def check_cohort(cohort, dim):
    """cohort = {name: x [n, dim]} checked: at least two speakers, each with at least one x-vector of dimension dim.
    Returns [(name, float64 array)] in dict order."""
    if not isinstance(cohort, dict) or not cohort:
        raise ValueError('cohort must be a non-empty {name: x-vectors} dict')
    if len(cohort) < 2:
        raise ValueError(f'a cohort needs at least 2 speakers, got {len(cohort)}')
    out = []
    for name, x in cohort.items():
        x = np.asarray(x, dtype=np.float64)
        if x.ndim != 2 or x.shape[0] == 0:
            raise ValueError(f'cohort speaker {name!r}: needs at least one x-vector as an [n, {dim}] array')
        if x.shape[1] != dim:
            raise ValueError(f'cohort speaker {name!r}: x-vectors of dimension {x.shape[1]}, the archive has {dim}')
        out.append((name, x))
    return out


def check_spread(std, names):
    """ValueError naming the speakers whose sigma is not finite or below SIGMA_MIN (e.g. a cohort of identical
    speakers: every top-K score is the same number)."""
    std = np.asarray(std, dtype=np.float64)
    bad = np.nonzero(~(std >= SIGMA_MIN) | ~np.isfinite(std))[0]
    if len(bad):
        shown = ', '.join(f'{names[i]} ({std[i]!r})' for i in bad[:10])
        raise ValueError(f'cohort scores without spread (sigma not finite or below {SIGMA_MIN:g}) for {len(bad)} '
                         f'speaker(s): {shown}')


def _cohort_speakers(cohort_speaker):
    """(cspk [N_c] int64, C) checked: at least two cohort speakers, each with an x-vector."""
    cspk = np.asarray(cohort_speaker, dtype=np.int64).reshape(-1)
    if len(cspk) == 0 or cspk.min() < 0:
        raise ValueError('cohort_speaker must hold at least one speaker index, all >= 0')
    C = int(cspk.max()) + 1
    if C < 2:
        raise ValueError(f'a cohort needs at least 2 speakers, got {C}')
    if np.bincount(cspk, minlength=C).min() == 0:
        raise ValueError('every cohort speaker 0 .. C-1 needs at least one x-vector')
    return cspk, C


def _scored_speakers(offsets, labels):
    """(speaker [N] int64, M) of the scored speakers as cohort_stats takes them (see there)."""
    from .link import speaker_index
    if offsets is not None:
        return speaker_index(offsets, labels)
    spk = np.asarray(labels, dtype=np.int64).reshape(-1)
    M = int(spk.max()) + 1 if len(spk) else 0
    if M and np.bincount(spk[spk >= 0], minlength=M).min() == 0:
        raise ValueError('every scored speaker 0 .. M-1 needs at least one x-vector')
    return spk, M


def cohort_stats(fea, Phi, offsets, labels, cohort_fea, cohort_speaker, Fa, Fb, top_k=DEFAULT_TOP_K, device=None,
                 max_bytes=2 ** 31, scores=False):
    """mu and sigma of every scored speaker's top_k cohort scores on the device (vbx_cohort_stats_batch on a batch of
    one).  fea [N,R], Phi [R]: the features the VB-HMM ran with.  Scored speakers: with offsets [B+1], labels holds each
    recording's first labels and the speakers are link.speaker_table's; with offsets None, labels is a speaker index [N]
    in [0, M) (-1: none), every speaker with at least one x-vector.  cohort_fea [N_c,R]: the cohort x-vectors through
    the same front end; cohort_speaker [N_c]: their speaker in [0, C), C >= 2, every one with an x-vector.  Speakers
    whose M x C score block exceeds max_bytes are split into chunks of consecutive speakers, one cohort_stats_many call
    each (the same bits).  Returns CohortStats (numpy), with the scores [M,C] when scores=True."""
    K_req = check_top_k(top_k)
    C = _cohort_speakers(cohort_speaker)[1]
    spk, M = _scored_speakers(offsets, labels)
    N = int(fea.shape[0])
    if len(spk) != N:
        raise ValueError(f'{len(spk)} speaker indices for {N} x-vectors')
    # chunks of consecutive speakers with at most max_bytes of scores (one speaker alone may exceed it)
    per = max(1, int(max_bytes) // (8 * C))
    parts = []
    for s0 in range(0, M, per) if M else [0]:
        s1 = min(s0 + per, M)
        x0, x1 = 0, N
        if M:
            mine = np.nonzero((spk >= s0) & (spk < s1))[0]
            x0, x1 = int(mine[0]), int(mine[-1]) + 1    # every speaker has an x-vector
        sp = spk[x0:x1]
        parts += cohort_stats_many(fea[x0:x1], Phi, None, [np.where((sp >= s0) & (sp < s1), sp - s0, -1)],
                                   cohort_fea, cohort_speaker, Fa, Fb, top_k=K_req, device=device, scores=scores)
    return CohortStats(np.concatenate([c.mean for c in parts]), np.concatenate([c.std for c in parts]), min(K_req, C),
                       np.concatenate([c.scores for c in parts]) if scores else None)


def cohort_stats_many(fea, Phi, offsets, labels_per_problem, cohort_fea, cohort_speaker, Fa, Fb, top_k=DEFAULT_TOP_K,
                      device=None, max_bytes=None, scores=False):
    """cohort_stats for G independent problems over the same features and cohort in few launches
    (vbx_cohort_stats_batch, DESIGN.md section 5.19), e.g. the final labels of every setting of a sweep.  fea, Phi,
    offsets, cohort_fea, cohort_speaker, top_k: as for cohort_stats; labels_per_problem: G label sets as cohort_stats
    takes them (per recording first labels with offsets, or a speaker index [N] with offsets None); Fa, Fb: numbers or
    G values.  The enrolled speakers of every setting: fea = the enrolled features, offsets None and their speaker index
    once per setting.  Launches as enroll_many packs them (max_bytes None: one).  Returns one CohortStats per problem,
    with its scores [M_g,C] when scores=True, bit-identical to cohort_stats on that problem alone."""
    import torch
    from . import _lib
    from ._lib import VbxError
    from .sweep import pack_by
    K_req = check_top_k(top_k)
    G = len(labels_per_problem)
    Fa, Fb = (np.broadcast_to(np.asarray(v, dtype=np.float64), (G,)).copy() for v in (Fa, Fb))
    cspk, C = _cohort_speakers(cohort_speaker)
    spks, Ms = zip(*[_scored_speakers(offsets, labels) for labels in labels_per_problem]) if G else ((), ())
    Ms = np.array(Ms, dtype=np.int64)
    if not torch.cuda.is_available():
        raise VbxError('cohort_stats_many(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    fea = torch.as_tensor(fea).to(dev, torch.float32).contiguous()
    Phi = torch.as_tensor(Phi).to(dev, torch.float32).contiguous()
    cfea = torch.as_tensor(cohort_fea).to(dev, torch.float32).contiguous()
    N, R = int(fea.shape[0]), int(fea.shape[1])
    if any(len(s) != N for s in spks):
        raise ValueError(f'every problem needs one speaker index per x-vector ({N})')
    if tuple(cfea.shape) != (len(cspk), R):
        raise ValueError(f'cohort_fea must be [{len(cspk)}, {R}], got {tuple(cfea.shape)}')
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    v = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    out = [None] * G

    def ws_bytes(idx):
        need = ctypes.c_size_t()
        M_h = np.ascontiguousarray(Ms[idx])
        if lib.vbx_cohort_stats_batch_workspace_bytes(h, len(idx), v(M_h), C, len(cspk), ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_cohort_stats_batch_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        return int(need.value)
    try:
        batches = pack_by(G, ws_bytes, max_bytes)
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            cspk_d = torch.from_numpy(cspk.astype(np.int32)).to(dev)
            for idx in batches:
                M_h = np.ascontiguousarray(Ms[idx])
                tot = int(M_h.sum())
                ws = torch.empty(max(ws_bytes(idx), 1), dtype=torch.uint8, device=dev)
                spk_d = torch.from_numpy(np.stack([spks[g] for g in idx]).astype(np.int32)).to(dev)
                fa, fb = np.ascontiguousarray(Fa[idx]), np.ascontiguousarray(Fb[idx])
                mean = torch.empty(tot, dtype=torch.float64, device=dev)
                std = torch.empty(tot, dtype=torch.float64, device=dev)
                L = torch.empty((tot, C), dtype=torch.float64, device=dev) if scores else None
                rc = lib.vbx_cohort_stats_batch(h, p(fea), p(Phi), N, R, len(idx), p(spk_d), v(M_h), p(cfea),
                                                len(cspk), p(cspk_d), C, v(fa), v(fb), K_req, p(ws), ws.numel(),
                                                p(mean), p(std), p(L), stream)
                if rc != 0:
                    raise VbxError(f'vbx_cohort_stats_batch failed ({rc}): {lib.vbx_last_error(h).decode()}')
                mean, std = mean.cpu().numpy(), std.cpu().numpy()
                L = L.cpu().numpy() if scores else None
                o = 0
                for g, M in zip(idx, M_h.tolist()):
                    out[g] = CohortStats(mean[o:o + M], std[o:o + M], min(K_req, C), L[o:o + M] if scores else None)
                    o += M
    finally:
        lib.vbx_destroy(h)
    return out
