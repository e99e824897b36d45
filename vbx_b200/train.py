"""Train the x-vector transform and the PLDA from labelled x-vectors (DESIGN.md section 5.24), so that embeddings of any
extractor, or a back end fitted to one's own domain, can be diarized without Kaldi:

    python -m vbx_b200.train --xvec-ark-file train.ark --utt2spk train.utt2spk --out-dir model
    python -m vbx_b200.train --xvec-ark-file train.ark --segments-file train.seg --ref-rttm ref/ --out-dir model

and then `python -m vbx_b200.cli --xvec-transform model/transform.npz --plda-file model/plda --lda-dim d ...`.

The model, all float64 (classes with fewer than min_per_speaker x-vectors dropped first; K classes, N x-vectors):
  transform  mean1 = mean of x; y = l2_norm(x - mean1); S_W, S_B the within- and between-class scatters of y over N;
             lda [Dx, d] the generalised eigenvectors of S_B v = lambda S_W v of the d largest lambda, descending,
             v^T S_W v = 1, each column's largest-magnitude entry positive; mean2 = mean of y lda;
             z = l2_norm(y lda - mean2)
  PLDA       two-covariance model z = mu + s + e, s ~ N(0, B), e ~ N(0, W), fitted by EM from W = S / N, B = the mean of
             m_i m_i^T (m_i the class means of z - mu, S the within-class scatter), in the basis that makes W = I and B
             diagonal; written in Kaldi form: W = L L^T, L^-1 B L^-T = U diag(psi) U^T with psi descending,
             transform = U^T L^-1 (each row's largest-magnitude entry positive), mean = mu.
The class means and within-class scatters run on the FP64 tensor cores (vbx_class_scatter); the K-row algebra is float64
torch on the device and the d x d eigenproblems float64 scipy on the host.
"""
import argparse
import ctypes
import json
import math
import os
import sys
import time

import numpy as np
import torch

from . import _lib, formats, pipeline, score
from ._lib import VbxError

MAX_DIM = 1024      # widest x-vector vbx_class_scatter takes


def _device(device):
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if dev.type != 'cuda':
        raise ValueError(f'back-end training runs on a CUDA device, got {dev}')
    return torch.device('cuda', torch.cuda.current_device()) if dev.index is None else dev


def class_stats(X, offsets, device=None):
    """Class means and within-class scatter of rows packed by class, on the FP64 tensor cores.  X [N, D] float32 (a
    tensor or array; moved to the device), offsets [K+1] int64 host (class i is rows offsets[i] .. offsets[i+1]-1,
    empty classes allowed).  Returns (means [K, D], scatter [D, D]) float64 tensors on the device: scatter =
    sum_rows (x - m_class)(x - m_class)^T, symmetric bit for bit."""
    dev = _device(device)
    X = torch.as_tensor(X).to(dev, torch.float32).contiguous()
    off = np.ascontiguousarray(np.asarray(offsets, dtype=np.int64).reshape(-1))
    if X.dim() != 2:
        raise ValueError(f'X must be [N, D], got shape {tuple(X.shape)}')
    N, D = int(X.shape[0]), int(X.shape[1])
    if not 1 <= D <= MAX_DIM:
        raise ValueError(f'x-vector dimension {D} outside 1 .. {MAX_DIM}')
    if len(off) < 2 or off[0] != 0 or off[-1] != N or np.any(np.diff(off) < 0):
        raise ValueError(f'offsets must run from 0 to N = {N} without decreasing')
    K = len(off) - 1
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    try:
        need = ctypes.c_size_t()
        if lib.vbx_class_scatter_workspace_bytes(h, N, D, K, ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_class_scatter_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        with torch.cuda.device(dev):
            ws = torch.empty(max(int(need.value), 1), dtype=torch.uint8, device=dev)
            means = torch.empty((K, D), dtype=torch.float64, device=dev)
            scatter = torch.empty((D, D), dtype=torch.float64, device=dev)
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            rc = lib.vbx_class_scatter(h, p(X), N, D, K, off.ctypes.data_as(ctypes.c_void_p), p(ws), ws.numel(),
                                       p(means), p(scatter), stream)
            if rc != 0:
                raise VbxError(f'vbx_class_scatter failed ({rc}): {lib.vbx_last_error(h).decode()}')
    finally:
        lib.vbx_destroy(h)
    return means, scatter


def _positive_largest(v, axis):
    """Flip the sign of every column (axis 0) or row (axis 1) whose entry of largest magnitude is negative."""
    idx = np.argmax(np.abs(v), axis=axis)
    big = v[idx, np.arange(v.shape[1])] if axis == 0 else v[np.arange(v.shape[0]), idx]
    s = np.where(big < 0, -1.0, 1.0)
    return v * (s[None, :] if axis == 0 else s[:, None])


def joint_diagonalise(W, B):
    """(L, U, psi, T): W = L L^T (lower), L^-1 B L^-T = U diag(psi) U^T with psi descending, T = U^T L^-1, so that
    T W T^T = I and T B T^T = diag(psi); T^-1 = L U."""
    from scipy.linalg import cholesky, eigh, solve_triangular
    L = cholesky(W, lower=True)
    A = solve_triangular(L, solve_triangular(L, B, lower=True).T, lower=True)
    psi, U = eigh(0.5 * (A + A.T))
    U, psi = U[:, ::-1].copy(), psi[::-1].copy()
    return L, U, psi, solve_triangular(L, U, lower=True, trans='T').T


def plda_em(Mc, n, S, N, em_iters):
    """Two-covariance EM.  Mc [K, d] class means of z - mu and n [K] float64 (tensors, any device), S [d, d] the
    within-class scatter (numpy).  Returns (W, B, objective trace [em_iters + 1]): the objective of the start and after
    every iteration, per x-vector."""
    K, d = int(Mc.shape[0]), int(Mc.shape[1])
    dev = Mc.device
    host = lambda t: t.cpu().numpy()
    W = S / N
    B = host(Mc.T @ Mc) / K
    nc = n[:, None]
    const = -0.5 * N * d * math.log(2 * math.pi) - 0.5 * d * float(torch.log(n).sum())
    trace = []
    for it in range(em_iters + 1):
        L, U, psi, T = joint_diagonalise(W, B)
        Td, psid = torch.from_numpy(T).to(dev), torch.from_numpy(psi).to(dev)
        Mt = Mc @ Td.T
        var = psid[None, :] + 1.0 / nc                       # diagonal of T (B + W / n_i) T^T
        logdet_w = 2.0 * float(np.log(np.diag(L)).sum())
        obj = const - 0.5 * N * logdet_w - 0.5 * float(torch.log(var).sum() + (Mt * Mt / var).sum()) \
            - 0.5 * float(np.trace(T @ S @ T.T))
        trace.append(obj / N)
        if it == em_iters:
            break
        c = psid[None, :] / (1.0 + nc * psid[None, :])      # C_i in the basis T
        zh = nc * c * Mt                                     # z-hat_i
        R = Mt - zh
        Bt = host(torch.diag(c.sum(0)) + zh.T @ zh) / K
        Wt = host(torch.diag((nc * c).sum(0)) + (nc * R).T @ R)
        Ti = L @ U
        B = Ti @ Bt @ Ti.T
        W = (S + Ti @ Wt @ Ti.T) / N
        B, W = 0.5 * (B + B.T), 0.5 * (W + W.T)
    return W, B, trace


def _sync(dev):
    torch.cuda.synchronize(dev)
    return time.perf_counter()


def check_training_set(xvectors, lda_dim, em_iters, min_per_speaker):
    """The refusals of DESIGN.md section 5.24 on the host.  Returns (names kept, arrays kept, speakers dropped,
    x-vectors dropped, Dx)."""
    for what, v, lo in (('min_per_speaker', min_per_speaker, 1), ('lda_dim', lda_dim, 1), ('em_iters', em_iters, 0)):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < lo:
            raise ValueError(f'{what} must be an integer >= {lo}, got {v!r}')
    if not isinstance(xvectors, dict):
        raise ValueError('xvectors must be a {speaker: x [n, Dx]} dict')
    names, arrays, drop_spk, drop_x, Dx = [], [], 0, 0, None
    for name, x in xvectors.items():
        x = np.asarray(x, dtype=np.float64)
        if x.ndim != 2:
            raise ValueError(f'speaker {name!r}: x-vectors must be an [n, Dx] array, got shape {x.shape}')
        if Dx is None:
            Dx = x.shape[1]
        if x.shape[1] != Dx:
            raise ValueError(f'speaker {name!r}: x-vectors of dimension {x.shape[1]}, the others have {Dx}')
        if not np.all(np.isfinite(x)):
            raise ValueError(f'speaker {name!r}: {int((~np.isfinite(x)).any(1).sum())} non-finite x-vector(s)')
        if x.shape[0] < min_per_speaker:
            drop_spk, drop_x = drop_spk + 1, drop_x + x.shape[0]
            continue
        names.append(name)
        arrays.append(x)
    K, N = len(arrays), sum(a.shape[0] for a in arrays)
    if K < 2:
        raise ValueError(f'{K} speaker(s) with at least {min_per_speaker} x-vectors; training needs at least 2')
    if not 1 <= Dx <= MAX_DIM:
        raise ValueError(f'x-vector dimension {Dx} outside 1 .. {MAX_DIM}')
    if lda_dim > Dx or lda_dim > K - 1:
        raise ValueError(f'lda_dim = {lda_dim} exceeds Dx = {Dx} or K - 1 = {K - 1} (the rank of the between-class '
                         f'scatter with K = {K} speakers)')
    if N - K < Dx:
        raise ValueError(f'N - K = {N} - {K} = {N - K} is below Dx = {Dx}: the within-class scatter would be singular')
    return names, arrays, drop_spk, drop_x, Dx


def train_backend(xvectors, lda_dim=128, em_iters=10, min_per_speaker=2, device=None):
    """Fit the x-vector transform and the PLDA (the definition in this module's docstring) to {speaker: x [n, Dx]}
    (e.g. formats.read_enrolment).  Returns (transform, plda, report): transform = (mean1, mean2, lda) and plda =
    (mean, transform, psi), float64 numpy, the tuples diarize_batch, sweep_batch and the command line take; report a
    dict of N, K, dropped speakers and x-vectors, Dx, d, the LDA eigenvalues, psi, the objective trace and the seconds
    of each stage."""
    from scipy.linalg import eigh
    _, arrays, drop_spk, drop_x, Dx = check_training_set(xvectors, lda_dim, em_iters, min_per_speaker)
    dev = _device(device)
    t = {}
    t0 = _sync(dev)
    counts = np.array([a.shape[0] for a in arrays], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    K, N, d = len(arrays), int(off[-1]), lda_dim
    x = torch.from_numpy(np.concatenate(arrays)).to(dev)
    n = torch.from_numpy(counts.astype(np.float64)).to(dev)
    t1 = _sync(dev)
    t['upload'] = t1 - t0

    mean1 = x.mean(0)
    y = pipeline.l2_norm_rows(x - mean1[None, :]).float()
    del x
    my, Sw = class_stats(y, off, dev)
    mu_y = (n @ my) / N
    dm = my - mu_y[None, :]
    Sb = (dm.T * n[None, :]) @ dm / N
    t2 = _sync(dev)
    t['lda_stats'] = t2 - t1
    lam, V = eigh(Sb.cpu().numpy(), Sw.cpu().numpy() / N)
    lam, lda = lam[::-1][:d].copy(), _positive_largest(V[:, ::-1][:, :d].copy(), 0)
    t3 = time.perf_counter()
    t['lda_eig'] = t3 - t2

    lda_d = torch.from_numpy(lda).to(dev)
    mean2 = mu_y @ lda_d
    z = pipeline.l2_norm_rows(y.double() @ lda_d - mean2[None, :]).float()
    del y
    mz, S = class_stats(z, off, dev)
    del z
    mu = (n @ mz) / N
    Mc = mz - mu[None, :]
    t4 = _sync(dev)
    t['plda_stats'] = t4 - t3
    W, B, trace = plda_em(Mc, n, S.cpu().numpy(), N, em_iters)
    _, _, psi, T = joint_diagonalise(W, B)
    tr = _positive_largest(T, 1)
    t['plda_em'] = time.perf_counter() - t4
    transform = (mean1.cpu().numpy(), mean2.cpu().numpy(), lda)
    plda = (mu.cpu().numpy(), tr, psi)
    report = dict(N=N, K=K, speakers_dropped=drop_spk, xvectors_dropped=drop_x, min_per_speaker=min_per_speaker,
                  Dx=Dx, lda_dim=d, em_iters=em_iters, lda_eigenvalues=lam.tolist(), psi=psi.tolist(),
                  objective=trace, seconds=t)
    return transform, plda, report


def speaker_shares(seg_ticks, turns):
    """c [T, n_spk]: the share of x-vector t's segment [lo, hi) ticks inside each speaker's sorted, disjoint turns
    (score.named_turns), as vbx_init_turns defines it; 0 for an empty segment."""
    lo, hi = seg_ticks[:, 0], seg_ticks[:, 1]
    length = (hi - lo).astype(np.float64)
    c = np.zeros((len(lo), len(turns)), dtype=np.float64)
    for k, (_, (s, e)) in enumerate(turns):
        cum = np.concatenate([[0], np.cumsum(e - s)])

        def covered(x):                                   # speaker time in [-inf, x)
            i = np.searchsorted(s, x, side='right') - 1
            inside = np.clip(x - s[np.maximum(i, 0)], 0, (e - s)[np.maximum(i, 0)])
            return np.where(i >= 0, cum[np.maximum(i, 0)] + inside, 0)
        c[:, k] = np.where(length > 0, (covered(hi) - covered(lo)) / np.maximum(length, 1), 0.0)
    return c


def speakers_from_rttm(recordings, ref_rttm, min_share=0.75, across_recordings=False):
    """Training classes from a diarization archive with reference RTTMs.  recordings {name: (x [T, Dx], seg_times [T, 2]
    seconds)} (formats.read_xvectors_by_recording with formats.read_segments); ref_rttm an RTTM file or directory, or
    formats.read_rttm rows.  X-vector t is kept for speaker k when k's share of its segment is >= min_share and no other
    speaker has any; overlapped x-vectors (two speakers with a share), uncovered ones (no speaker reaches min_share) and
    those of recordings the RTTM lacks are dropped.  A class is (recording, RTTM name), or the RTTM name alone with
    across_recordings (names are archive-wide ids).  Returns ({class: x [n, Dx]} in order of first appearance,
    counts {'kept', 'overlapped', 'uncovered'})."""
    if not 0.0 < min_share <= 1.0:
        raise ValueError(f'min_share must lie in (0, 1], got {min_share!r}')
    rows = score.read_rttm_path(ref_rttm) if isinstance(ref_rttm, (str, os.PathLike)) else list(ref_rttm)
    turns = score.named_turns([r for r in rows if r[0] in recordings])
    out, counts = {}, dict(kept=0, overlapped=0, uncovered=0)
    for rec, (x, seg) in recordings.items():
        x = np.asarray(x, dtype=np.float64)
        spk = turns.get(rec, [])
        if not spk:
            counts['uncovered'] += len(x)
            continue
        c = speaker_shares(score.to_ticks(np.asarray(seg, dtype=np.float64).reshape(-1, 2)), spk)
        over = (c > 0).sum(1) > 1
        best = np.argmax(c, 1)
        keep = ~over & (c[np.arange(len(c)), best] >= min_share)
        counts['overlapped'] += int(over.sum())
        counts['uncovered'] += int((~over & ~keep).sum())
        counts['kept'] += int(keep.sum())
        for t in np.nonzero(keep)[0]:
            name = spk[best[t]][0]
            out.setdefault(name if across_recordings else (rec, name), []).append(x[t])
    return {k: np.stack(v) for k, v in out.items()}, counts


def write_backend(out_dir, transform, plda, report, binary=True):
    """out_dir/transform.npz (formats.read_xvec_transform), out_dir/plda (Kaldi binary, or text with binary=False) and
    out_dir/train.json (the report).  Returns the three paths."""
    os.makedirs(out_dir, exist_ok=True)
    mean1, mean2, lda = transform
    paths = [os.path.join(out_dir, f) for f in ('transform.npz', 'plda', 'train.json')]
    np.savez(paths[0], mean1=np.asarray(mean1, dtype=np.float64), mean2=np.asarray(mean2, dtype=np.float64),
             lda=np.asarray(lda, dtype=np.float64))
    (formats.write_kaldi_plda_binary if binary else formats.write_kaldi_plda_text)(paths[1], *plda)
    with open(paths[2], 'w') as f:
        json.dump(report, f, indent=1, sort_keys=True, default=str)
    return paths


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--xvec-ark-file', required=True, help='Kaldi ark of the training x-vectors')
    ap.add_argument('--utt2spk', default=None, help='speaker of every x-vector of the ark')
    ap.add_argument('--ref-rttm', default=None, help='reference RTTM file or directory (with --segments-file)')
    ap.add_argument('--segments-file', default=None, help='Kaldi segments of the ark (with --ref-rttm)')
    ap.add_argument('--out-dir', required=True, help='directory for transform.npz, plda and train.json')
    ap.add_argument('--lda-dim', type=int, default=128, help='dimension d after the LDA (default 128)')
    ap.add_argument('--em-iters', type=int, default=10, help='PLDA EM iterations (default 10)')
    ap.add_argument('--min-per-speaker', type=int, default=2, help='speakers with fewer x-vectors are dropped')
    ap.add_argument('--min-share', type=float, default=None,
                    help='with --ref-rttm: least share of a segment its one speaker must cover (default 0.75)')
    ap.add_argument('--speakers-across-recordings', action='store_true',
                    help='with --ref-rttm: an RTTM name is the same speaker in every recording')
    ap.add_argument('--text-plda', action='store_true', help='write the PLDA as Kaldi text instead of binary')
    ap.add_argument('--device', default=None, help='CUDA device (default: the current one)')
    return ap


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if (args.utt2spk is None) == (args.ref_rttm is None):
        ap.error('give exactly one of --utt2spk and --ref-rttm')
    if (args.ref_rttm is None) != (args.segments_file is None):
        ap.error('--ref-rttm and --segments-file go together')
    if args.utt2spk is not None and (args.speakers_across_recordings or args.min_share is not None):
        ap.error('--min-share and --speakers-across-recordings need --ref-rttm')
    min_share = 0.75 if args.min_share is None else args.min_share
    extra = {}
    if args.utt2spk is not None:
        xvectors = formats.read_enrolment(args.xvec_ark_file, args.utt2spk)
    else:
        segs = formats.read_segments(args.segments_file)
        recs = {}
        for name, (keys, x) in formats.read_xvectors_by_recording(args.xvec_ark_file).items():
            if name not in segs or list(segs[name][0]) != list(keys):
                raise ValueError(f'recording {name!r}: the segments file does not list the ark keys in ark order')
            recs[name] = (x, segs[name][1])
        xvectors, extra = speakers_from_rttm(recs, args.ref_rttm, min_share, args.speakers_across_recordings)
    transform, plda, report = train_backend(xvectors, args.lda_dim, args.em_iters, args.min_per_speaker, args.device)
    if extra:
        report['rttm'] = dict(extra, min_share=min_share, across_recordings=args.speakers_across_recordings)
    paths = write_backend(args.out_dir, transform, plda, report, binary=not args.text_plda)
    print(f'trained on N = {report["N"]} x-vectors of K = {report["K"]} speakers ({report["speakers_dropped"]} speakers, '
          f'{report["xvectors_dropped"]} x-vectors dropped), Dx = {report["Dx"]}, d = {report["lda_dim"]}, objective '
          f'{report["objective"][0]:.4f} -> {report["objective"][-1]:.4f}; wrote {", ".join(paths)}')
    return 0


if __name__ == '__main__':
    sys.exit(main())
