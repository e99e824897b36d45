"""Enrolment against known speakers (DESIGN.md section 5.16).

Each recording's VB-HMM numbers its speakers 1..K.  Enrolment names them: every archive speaker (section 5.15's table)
is scored against every enrolled speaker with section 5.15's same-speaker LLR, and each recording's speakers are
assigned one-to-one to enrolled speakers, or to "unknown", by a minimum-cost assignment on the device
(vbx_enroll_batch).  A speaker takes an enrolled name only where its LLR reaches the threshold, two speakers of one
recording never share a name, and the sum of LLR - threshold over the named speakers is the largest possible.
"""
import ctypes
from collections import namedtuple

import numpy as np

from .link import speaker_table, table_index

UNKNOWN = 'unknown-'       # prefix of the names of speakers that match no enrolled speaker (reserved)
MAX_THRESHOLD = 1e15

# table: link.SpeakerTable; assign [M] enrolled index or -1; best_llr [M] the LLR of the assigned pair, or for an unknown
# speaker its largest LLR; n [M], F [M,R], n_enroll [E], F_enroll [E,R] float64 statistics; llr [M,E] or None
EnrollResult = namedtuple('EnrollResult', 'table assign best_llr n F n_enroll F_enroll llr')


def check_threshold(threshold):
    """The enrolment threshold as a float; ValueError when it is missing, not finite or beyond +-1e15."""
    if threshold is None:
        raise ValueError('enrolment needs a threshold: the LLR is not calibrated, so there is no default')
    t = float(threshold)
    if not abs(t) <= MAX_THRESHOLD:
        raise ValueError(f'enrolment threshold must lie in [-{MAX_THRESHOLD:g}, {MAX_THRESHOLD:g}], got {threshold!r}')
    return t


def check_enrolment(enroll, dim):
    """enroll = {name: x [n, dim]} checked: a name is non-empty, has no whitespace and does not start with 'unknown-';
    every speaker has at least one x-vector of dimension dim.  Returns [(name, float64 array)] in dict order."""
    if not isinstance(enroll, dict) or not enroll:
        raise ValueError('enroll must be a non-empty {name: x-vectors} dict')
    out = []
    for name, x in enroll.items():
        if not isinstance(name, str) or not name or any(ch.isspace() for ch in name):
            raise ValueError(f'enrolled speaker name {name!r}: must be a non-empty string without whitespace')
        if name.startswith(UNKNOWN):
            raise ValueError(f'enrolled speaker name {name!r}: the prefix {UNKNOWN!r} is reserved')
        x = np.asarray(x, dtype=np.float64)
        if x.ndim != 2 or x.shape[0] == 0:
            raise ValueError(f'enrolled speaker {name!r}: needs at least one x-vector as an [n, {dim}] array')
        if x.shape[1] != dim:
            raise ValueError(f'enrolled speaker {name!r}: x-vectors of dimension {x.shape[1]}, the archive has {dim}')
        out.append((name, x))
    return out


def enroll_speakers(fea, Phi, offsets, labels, enroll_fea, enroll_speaker, Fa, Fb, threshold, device=None, llr=False,
                    max_bytes=2 ** 31, norm=None):
    """Statistics, LLRs and the per-recording assignment of every archive speaker against the enrolled speakers on the
    device (vbx_enroll_batch on a batch of one).  fea [N,R], Phi [R]: the features the VB-HMM ran with, packed by
    recording at offsets [B+1]; labels: each recording's final first labels.  enroll_fea [N_e,R]: the enrolled
    x-vectors through the same front end; enroll_speaker [N_e]: their speaker in [0, E), every speaker with at least one
    x-vector.  Archives whose M x E LLR block exceeds max_bytes are split into chunks of whole recordings, one
    enroll_many call each (the results are the same bits).  norm: None, or (mean [M], std [M], enroll_mean [E],
    enroll_std [E]) of the archive and enrolled speakers' cohort scores (cohort.cohort_stats): the assignment then runs
    on the normalised scores S of DESIGN.md section 5.17 with the threshold on S, and best_llr and llr hold S.
    Returns EnrollResult (numpy, speaker_table order), with llr [M,E] when llr=True."""
    t = check_threshold(threshold)
    offsets = np.asarray(offsets, dtype=np.int64)
    espk = np.asarray(enroll_speaker, dtype=np.int64).reshape(-1)
    if len(espk) == 0 or espk.min() < 0:
        raise ValueError('enroll_speaker must hold at least one speaker index, all >= 0')
    E = int(espk.max()) + 1
    if np.bincount(espk, minlength=E).min() == 0:
        raise ValueError('every enrolled speaker 0 .. E-1 needs at least one x-vector')
    table = speaker_table(labels)
    M, B = len(table.rec), len(labels)
    if int(offsets[-1]) != int(fea.shape[0]) or len(offsets) != B + 1:
        raise ValueError('offsets must hold one more entry than labels and end at the number of x-vectors')
    if norm is not None:
        norm = [np.asarray(a, dtype=np.float64) for a in norm]
        if [a.shape for a in norm] != [(M,), (M,), (E,), (E,)]:
            raise ValueError(f'norm must hold mean and std of the {M} archive and the {E} enrolled speakers')
    first = np.searchsorted(table.rec, np.arange(B + 1)).astype(np.int64)     # each recording's first speaker
    # chunks of whole recordings with at most max_bytes of LLRs (a recording alone may exceed it)
    chunks, b0 = [], 0
    for b in range(B):
        if b > b0 and (first[b + 1] - first[b0]) * E * 8 > max_bytes:
            chunks.append((b0, b))
            b0 = b
    chunks.append((b0, B))
    parts = []
    for a, z in chunks:
        s0, s1, x0 = int(first[a]), int(first[z]), int(offsets[a])
        nm = None if norm is None else [(norm[0][s0:s1], norm[1][s0:s1], norm[2], norm[3])]
        parts += enroll_many(fea[x0:int(offsets[z])], Phi, offsets[a:z + 1] - x0, [labels[a:z]], enroll_fea, espk,
                             Fa, Fb, [t], device=device, llr=llr, norm=nm)
    cat = lambda f: np.concatenate([f(r) for r in parts])
    return EnrollResult(table, cat(lambda r: r.assign[0]), cat(lambda r: r.best_llr[0]), cat(lambda r: r.n),
                        cat(lambda r: r.F), parts[0].n_enroll, parts[0].F_enroll, cat(lambda r: r.llr) if llr else None)


def check_thresholds(thresholds):
    """The enrolment thresholds of a sweep as floats without duplicates (first occurrence kept); each as check_threshold
    takes it.  An empty list raises ValueError."""
    out = list(dict.fromkeys(check_threshold(t) for t in thresholds))
    if not out:
        raise ValueError('enroll_thresholds needs at least one value')
    return out


def enroll_many(fea, Phi, offsets, labels_per_problem, enroll_fea, enroll_speaker, Fa, Fb, thresholds, device=None,
                llr=False, max_bytes=None, norm=None):
    """enroll_speakers for G independent problems over the same features and enrolled set, at every threshold, in few
    launches (vbx_enroll_batch, DESIGN.md section 5.19), e.g. the final labels of every setting of a sweep.  fea, Phi,
    offsets, enroll_fea, enroll_speaker: as for enroll_speakers; labels_per_problem: G lists of first labels per
    recording; Fa, Fb: numbers or G values; thresholds: a list (check_thresholds).  Each problem's LLR block is computed
    once and assigned at every threshold.  norm: None, or per problem (mean [M_g], std [M_g], enroll_mean [E],
    enroll_std [E]) (cohort.cohort_stats_many): the normalised path of enroll_speakers(norm=).  The problems are packed
    in order into launches whose workspace stays within max_bytes (None: one launch; sweep.pack_by with the batch's own
    vbx_enroll_batch_workspace_bytes; a problem larger than max_bytes alone raises ValueError).
    Returns one EnrollResult per problem with assign and best_llr [n_thr, M_g] (row h: thresholds[h]); row h is
    bit-identical to enroll_speakers(threshold=thresholds[h]) on that problem alone, and so are n, F, n_enroll, F_enroll
    and llr [M_g, E] (llr=True)."""
    import torch
    from . import _lib
    from ._lib import VbxError
    from .sweep import pack_by
    thr = np.ascontiguousarray(check_thresholds(thresholds), dtype=np.float64)
    G, T = len(labels_per_problem), len(thr)
    Fa, Fb = (np.broadcast_to(np.asarray(v, dtype=np.float64), (G,)).copy() for v in (Fa, Fb))
    offsets = np.asarray(offsets, dtype=np.int64)
    espk = np.asarray(enroll_speaker, dtype=np.int64).reshape(-1)
    if len(espk) == 0 or espk.min() < 0:
        raise ValueError('enroll_speaker must hold at least one speaker index, all >= 0')
    E = int(espk.max()) + 1
    if np.bincount(espk, minlength=E).min() == 0:
        raise ValueError('every enrolled speaker 0 .. E-1 needs at least one x-vector')
    tables = [speaker_table(l) for l in labels_per_problem]
    Ms = np.array([len(t.rec) for t in tables], dtype=np.int64)
    B = len(offsets) - 1
    firsts = [np.searchsorted(t.rec, np.arange(B + 1)).astype(np.int64) for t in tables]
    if norm is not None:
        norm = [tuple(np.asarray(a, dtype=np.float64) for a in nm) for nm in norm]
        if len(norm) != G or any([a.shape for a in nm] != [(M,), (M,), (E,), (E,)] for nm, M in zip(norm, Ms.tolist())):
            raise ValueError('norm must hold per problem mean and std of its archive speakers and of the E enrolled ones')
    if not torch.cuda.is_available():
        raise VbxError('enroll_many(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    fea = torch.as_tensor(fea).to(dev, torch.float32).contiguous()
    Phi = torch.as_tensor(Phi).to(dev, torch.float32).contiguous()
    efea = torch.as_tensor(enroll_fea).to(dev, torch.float32).contiguous()
    N, R = int(fea.shape[0]), int(fea.shape[1])
    for labels in labels_per_problem:
        if int(offsets[-1]) != N or len(labels) != B:
            raise ValueError('offsets must hold one more entry than labels and end at the number of x-vectors')
    if tuple(efea.shape) != (len(espk), R):
        raise ValueError(f'enroll_fea must be [{len(espk)}, {R}], got {tuple(efea.shape)}')
    max_k = [int(np.diff(f).max()) if B else 0 for f in firsts]
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
        if lib.vbx_enroll_batch_workspace_bytes(h, len(idx), v(M_h), E, len(espk), max(max_k[g] for g in idx), T,
                                                ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_enroll_batch_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        return int(need.value)
    try:
        batches = pack_by(G, ws_bytes, max_bytes)
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            espk_d = torch.from_numpy(espk.astype(np.int32)).to(dev)
            thr_h = np.ascontiguousarray(thr)
            for idx in batches:
                M_h = np.ascontiguousarray(Ms[idx])
                tot, Gb = int(M_h.sum()), len(idx)
                ws = torch.empty(max(ws_bytes(idx), 1), dtype=torch.uint8, device=dev)
                spk = np.stack([table_index(offsets, labels_per_problem[g], tables[g]) for g in idx]).astype(np.int32)
                spk_d = torch.from_numpy(spk).to(dev)
                rec_off = np.ascontiguousarray(np.stack([firsts[g] for g in idx]))
                fa, fb = np.ascontiguousarray(Fa[idx]), np.ascontiguousarray(Fb[idx])
                assign = torch.empty((T, tot), dtype=torch.int32, device=dev)
                best = torch.empty((T, tot), dtype=torch.float64, device=dev)
                n = torch.empty(tot, dtype=torch.float64, device=dev)
                F = torch.empty((tot, R), dtype=torch.float64, device=dev)
                n_e = torch.empty((Gb, E), dtype=torch.float64, device=dev)
                F_e = torch.empty((Gb, E, R), dtype=torch.float64, device=dev)
                L = torch.empty((tot, E), dtype=torch.float64, device=dev) if llr else None
                stats = [None] * 4
                if norm is not None:
                    stats = [torch.from_numpy(np.concatenate([norm[g][k] for g in idx])).to(dev) for k in range(4)]
                rc = lib.vbx_enroll_batch(h, p(fea), p(Phi), N, R, Gb, p(spk_d), v(M_h), v(rec_off), B, p(efea),
                                          len(espk), p(espk_d), E, v(fa), v(fb), v(thr_h), T, p(ws), ws.numel(),
                                          p(assign), p(best), p(L), p(n), p(F), p(n_e), p(F_e), *map(p, stats), stream)
                if rc != 0:
                    raise VbxError(f'vbx_enroll_batch failed ({rc}): {lib.vbx_last_error(h).decode()}')
                assign = assign.cpu().numpy().astype(np.int64)
                best, n, F = best.cpu().numpy(), n.cpu().numpy(), F.cpu().numpy()
                n_e, F_e = n_e.cpu().numpy(), F_e.cpu().numpy()
                L = L.cpu().numpy() if llr else None
                o = 0
                for j, (g, M) in enumerate(zip(idx, M_h.tolist())):
                    out[g] = EnrollResult(tables[g], assign[:, o:o + M], best[:, o:o + M], n[o:o + M], F[o:o + M],
                                          n_e[j], F_e[j], L[o:o + M] if llr else None)
                    o += M
    finally:
        lib.vbx_destroy(h)
    return out


def enroll_names(table, assign, best_llr, enrolled_names, recording_names, labels2=None, link=None):
    """The names of every recording's speakers (DESIGN.md section 5.16): per recording ({label: name}, {label: llr}).
    A speaker assigned to enrolled speaker e is enrolled_names[e]; any other is unknown-<recording>-<label + 1>, or with
    `link` (per recording {label: id}, link.link_cut over the unknown speakers) unknown-<id + 1>.  labels2: None, or per
    recording None or its second labels; a label used only there has no model and is unknown (it has no llr entry)."""
    names = [{} for _ in range(table.n_recordings)]
    llrs = [{} for _ in range(table.n_recordings)]
    unknown = (lambda b, l: f'{UNKNOWN}{recording_names[b]}-{l + 1}') if link is None else \
        (lambda b, l: f'{UNKNOWN}{link[b][l] + 1}')
    for b, l, a, v in zip(table.rec.tolist(), table.label.tolist(), np.asarray(assign).tolist(),
                          np.asarray(best_llr).tolist()):
        names[b][l] = enrolled_names[a] if a >= 0 else unknown(b, l)
        llrs[b][l] = float(v)
    for b, l2 in enumerate(labels2 or []):
        if l2 is None:
            continue
        for l in np.unique(np.asarray(l2, dtype=np.int64)).tolist():
            if l >= 0 and l not in names[b]:
                names[b][l] = unknown(b, l)
    return names, llrs


def prior_states(result, enrolled_names, n_states):
    """The enrolment prior of the VB-HMM's states (DESIGN.md section 5.23) from an assignment of each recording's AHC
    clusters (enroll_speakers over the AHC labels: cluster l of recording b is state l).  n_states: the state count of
    every recording.  Returns (prior, prior_speakers): prior[b] is None when no cluster of recording b was assigned,
    else (n [n_states[b]], F [n_states[b], R]) float64 with the assigned enrolled speaker's n_enroll, F_enroll in the
    row of its state and zeros elsewhere; prior_speakers[b] = {state: enrolled name}."""
    R = np.asarray(result.F_enroll).shape[1]
    prior = [None] * len(n_states)
    named = [{} for _ in n_states]
    for b, l, a in zip(result.table.rec.tolist(), result.table.label.tolist(), np.asarray(result.assign).tolist()):
        if a < 0:
            continue
        if prior[b] is None:
            prior[b] = (np.zeros(int(n_states[b])), np.zeros((int(n_states[b]), R)))
        prior[b][0][l] = result.n_enroll[a]
        prior[b][1][l] = result.F_enroll[a]
        named[b][l] = enrolled_names[a]
    return prior, named


def carry_assignment(result, labels):
    """The assignment of an enroll_speakers result over the AHC labels carried to the final labels of the VB-HMM that
    started from them (every final label is one of the AHC clusters, its state).  Returns (table, assign, best) over
    link.speaker_table(labels), for enroll_names."""
    row = {(b, l): i for i, (b, l) in enumerate(zip(result.table.rec.tolist(), result.table.label.tolist()))}
    table = speaker_table(labels)
    idx = np.array([row[(b, l)] for b, l in zip(table.rec.tolist(), table.label.tolist())], dtype=np.int64)
    return table, np.asarray(result.assign)[idx], np.asarray(result.best_llr)[idx]


def name_prior_states(names, prior_speakers):
    """The names of enroll_names with every state that carried an enrolment prior (prior_states' prior_speakers) named
    by its enrolled speaker, also where it survived the VB-HMM as a second label only.  Changes names in place and
    returns it."""
    for nm, pr in zip(names, prior_speakers):
        for l, name in pr.items():
            if l in nm:
                nm[l] = name
    return names


def mask_named(labels, names):
    """An int label array with the labels of enrolled (not unknown-) speakers set to -1 (None stays None)."""
    if labels is None:
        return None
    l = np.asarray(labels, dtype=np.int64)
    named = [k for k, v in names.items() if not v.startswith(UNKNOWN)]
    return np.where(np.isin(l, named), -1, l)
