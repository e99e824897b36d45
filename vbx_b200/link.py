"""Speaker linking across the recordings of an archive (DESIGN.md section 5.15).

Each recording's VB-HMM numbers its speakers 1..K on its own.  Linking gives them archive-wide ids: every speaker's
VB-HMM posterior (from its x-vectors' features) is scored against every other speaker's with the closed-form
same-speaker log-likelihood ratio, the scores are clustered by average linkage on the device (vbx_link), and the
linkage is cut on the host at an LLR threshold, so another threshold is another cut of the same linkage.
"""
import ctypes
from collections import namedtuple

import numpy as np

BIG = 1e30                 # distance between two speakers of one recording (vbx_link)
MAX_THRESHOLD = 1e15       # |threshold| above this would reach the cannot-link merges

# The speakers of an archive: speaker i is label `label[i]` of recording `rec[i]`, ordered by recording, then label;
# n_recordings counts the archive's recordings, those without speakers included.
SpeakerTable = namedtuple('SpeakerTable', 'rec label n_recordings')


def speaker_table(labels_by_recording):
    """The speakers of an archive: every (recording, label) that is the first label of at least one x-vector.
    labels_by_recording: one int array of first labels per recording, in archive order (negative entries: none)."""
    rec, lab = [], []
    for b, l in enumerate(labels_by_recording):
        u = np.unique(np.asarray(l, dtype=np.int64).reshape(-1))
        u = u[u >= 0]
        rec.append(np.full(len(u), b, dtype=np.int64))
        lab.append(u)
    cat = lambda a: np.concatenate(a) if a else np.zeros(0, dtype=np.int64)
    return SpeakerTable(cat(rec), cat(lab), len(labels_by_recording))


def check_threshold(threshold):
    t = float(threshold)
    if not abs(t) <= MAX_THRESHOLD:
        raise ValueError(f'link threshold must lie in [-{MAX_THRESHOLD:g}, {MAX_THRESHOLD:g}], got {threshold!r}')
    return t


def speaker_index(offsets, labels):
    """(speaker [N] int64, M): the speaker_table index of every x-vector (-1 where its label is negative) of the
    recordings packed at offsets [B+1] with first labels `labels`."""
    table = speaker_table(labels)
    return table_index(offsets, labels, table), len(table.rec)


def table_index(offsets, labels, table):
    """speaker_index's speaker [N] with table = speaker_table(labels) already at hand."""
    offsets = np.asarray(offsets, dtype=np.int64)
    if len(offsets) != len(labels) + 1:
        raise ValueError('offsets must hold one more entry than labels')
    spk = np.full(int(offsets[-1]), -1, dtype=np.int64)
    first = np.searchsorted(table.rec, np.arange(len(labels) + 1))
    for b, l in enumerate(labels):
        l = np.asarray(l, dtype=np.int64).reshape(-1)
        if len(l) != offsets[b + 1] - offsets[b]:
            raise ValueError(f'recording {b}: {len(l)} labels for {offsets[b + 1] - offsets[b]} x-vectors')
        own = table.label[first[b]:first[b + 1]]
        spk[offsets[b]:offsets[b + 1]] = np.where(l >= 0, first[b] + np.searchsorted(own, l), -1)
    return spk


def link_speakers(fea, Phi, offsets, labels, Fa, Fb, device=None, dist=False, norm=None):
    """Statistics, pairwise scores and average linkage of every speaker of an archive on the device (vbx_link_batch on a
    batch of one).  fea [N,R] and Phi [R]: the features the VB-HMM ran with (CUDA tensors or arrays, float32), packed
    by recording at offsets [B+1]; labels: the final first labels of each recording; Fa, Fb: the VB-HMM's scalars.
    norm: None, or (mean [M], std [M]) of the speakers' cohort scores (cohort.cohort_stats over the same speakers):
    the distances are then -S, the normalised scores of DESIGN.md section 5.17.
    Returns (table, n [M], F [M,R], Z [M-1,4]) as numpy float64 (speaker_table order), and dist [M,M] with dist=True.
    ValueError when the archive has more speakers than the linkage kernel indexes."""
    return link_many(fea, Phi, offsets, [labels], Fa, Fb, device=device, dist=dist,
                     norm=None if norm is None else [norm])[0]


def link_many(fea, Phi, offsets, labels_per_problem, Fa, Fb, device=None, max_bytes=None, dist=False, norm=None):
    """link_speakers for G independent problems over the same features in few launches (vbx_link_batch, DESIGN.md
    section 5.18), e.g. the final labels of every setting of a sweep.  fea, Phi, offsets: as for link_speakers;
    labels_per_problem: G lists of first labels per recording; Fa, Fb: numbers or G values, problem g's scalars.
    The problems are packed in order into launches whose workspaces stay within max_bytes (None: one launch), each
    problem sized by vbx_link_batch_workspace_bytes on it alone (sweep.pack: a problem larger than max_bytes on its own
    raises ValueError).  norm: None, or per problem (mean [M_g], std [M_g]) of its speakers' cohort scores
    (cohort.cohort_stats_many): the distances are then -S (DESIGN.md sections 5.17, 5.19).
    Returns one (table, n, F, Z) per problem (with dist=True also dist [M,M]), bit-identical to link_speakers on that
    problem alone (with the same norm)."""
    import torch
    from . import _lib
    from ._lib import VbxError
    from .sweep import pack
    G = len(labels_per_problem)
    Fa, Fb = (np.broadcast_to(np.asarray(v, dtype=np.float64), (G,)).copy() for v in (Fa, Fb))
    offsets = np.asarray(offsets, dtype=np.int64)
    tables = [speaker_table(l) for l in labels_per_problem]
    Ms = [len(t.rec) for t in tables]
    for g, M in enumerate(Ms):
        if M > _lib.LINK_MAX_SPEAKERS:
            raise ValueError(f'problem {g}: {M} speakers to link: at most {_lib.LINK_MAX_SPEAKERS} are supported (the '
                             f'workspace would need more than {8 * M * M} bytes)')
    if not torch.cuda.is_available():
        raise VbxError('link_many(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    fea = torch.as_tensor(fea).to(dev, torch.float32).contiguous()
    Phi = torch.as_tensor(Phi).to(dev, torch.float32).contiguous()
    N, R = int(fea.shape[0]), int(fea.shape[1])
    for labels in labels_per_problem:
        if int(offsets[-1]) != N or len(offsets) != len(labels) + 1:
            raise ValueError('offsets must hold one more entry than labels and end at the number of x-vectors')
    if norm is not None:
        norm = [tuple(np.asarray(a, dtype=np.float64) for a in nm) for nm in norm]
        if len(norm) != G or any([a.shape for a in nm] != [(M,), (M,)] for nm, M in zip(norm, Ms)):
            raise ValueError('norm must hold per problem mean and std of its speakers')
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    out = [None] * G
    try:
        def ws_bytes(M_h):
            need = ctypes.c_size_t()
            if lib.vbx_link_batch_workspace_bytes(h, len(M_h), M_h.ctypes.data_as(ctypes.c_void_p),
                                                  ctypes.byref(need)) != 0:
                raise VbxError(f'vbx_link_batch_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
            return int(need.value)
        batches = [list(range(G))] if max_bytes is None else \
            pack([ws_bytes(np.array([M], dtype=np.int64)) for M in Ms], max_bytes)
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            for idx in batches:
                if not idx:
                    continue
                M_h = np.array([Ms[g] for g in idx], dtype=np.int64)
                tot = int(M_h.sum())
                spk = np.stack([table_index(offsets, labels_per_problem[g], tables[g]) for g in idx]).astype(np.int32)
                rec = np.concatenate([tables[g].rec for g in idx]).astype(np.int32)
                fa, fb = np.ascontiguousarray(Fa[idx]), np.ascontiguousarray(Fb[idx])
                ws = torch.empty(max(ws_bytes(M_h), 1), dtype=torch.uint8, device=dev)
                spk_d = torch.from_numpy(spk).to(dev)
                rec_d = torch.from_numpy(rec).to(dev)
                n = torch.empty(tot, dtype=torch.float64, device=dev)
                F = torch.empty((tot, R), dtype=torch.float64, device=dev)
                D = torch.empty(int((M_h * M_h).sum()), dtype=torch.float64, device=dev) if dist else None
                Z = torch.empty((tot, 4), dtype=torch.float64, device=dev)
                mean = std = None
                if norm is not None:
                    mean, std = (torch.from_numpy(np.concatenate([norm[g][k] for g in idx])).to(dev) for k in (0, 1))
                rc = lib.vbx_link_batch(h, p(fea), p(Phi), N, R, len(idx), p(spk_d), M_h.ctypes.data_as(ctypes.c_void_p),
                                        p(rec_d), fa.ctypes.data_as(ctypes.c_void_p), fb.ctypes.data_as(ctypes.c_void_p),
                                        p(ws), ws.numel(), p(n), p(F), p(D), p(Z), p(mean), p(std), stream)
                if rc != 0:
                    raise VbxError(f'vbx_link_batch failed ({rc}): {lib.vbx_last_error(h).decode()}')
                n, F, Z = n.cpu().numpy(), F.cpu().numpy(), Z.cpu().numpy()
                D = D.cpu().numpy() if dist else None
                o = d = 0
                for g, M in zip(idx, M_h.tolist()):
                    out[g] = (tables[g], n[o:o + M], F[o:o + M], Z[o:o + max(M - 1, 0)])
                    if dist:
                        out[g] += (D[d:d + M * M].reshape(M, M),)
                    o += M
                    d += M * M
    finally:
        lib.vbx_destroy(h)
    return out


def link_cut(Z, table, threshold, labels2=None):
    """Archive-wide speaker ids from the linkage Z of table's speakers: speakers whose average LLR is at least
    `threshold` share an id (ahc.flat_clusters(Z, -threshold)); ids are numbered by first appearance over the table.
    labels2: None, or per recording its second labels (None or an int array, -1 = none); a label that occurs only there
    gets an id of its own after all linked ones, by recording, then label.  Returns per recording {label: id}."""
    from .ahc import flat_clusters
    t = check_threshold(threshold)
    M = len(table.rec)
    flat = flat_clusters(Z, -t) if M > 1 else np.ones(M, dtype=np.int32)
    ids = {}
    gid = [ids.setdefault(int(f), len(ids)) for f in flat]
    maps = [{} for _ in range(table.n_recordings)]
    for b, l, g in zip(table.rec.tolist(), table.label.tolist(), gid):
        maps[b][l] = g
    nxt = len(ids)
    for b, l2 in enumerate(labels2 or []):
        if l2 is None:
            continue
        for l in np.unique(np.asarray(l2, dtype=np.int64)).tolist():
            if l >= 0 and l not in maps[b]:
                maps[b][l] = nxt
                nxt += 1
    return maps


def relabel(labels, mapping):
    """An int label array through a {label: id} map (None stays None, -1 stays -1)."""
    if labels is None:
        return None
    l = np.asarray(labels, dtype=np.int64)
    lut = np.full(max(mapping, default=-1) + 2, -1, dtype=np.int64)    # lut[label + 1]; lut[0] = -1 for label -1
    lut[np.fromiter(mapping, dtype=np.int64, count=len(mapping)) + 1] = list(mapping.values())
    return lut[l + 1]
