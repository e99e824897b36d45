"""Speaker-verification trials scored with the back end (DESIGN.md section 5.27).

    python -m vbx_b200.verify --trials trials --enroll-ark enrol.ark [--enroll-utt2spk enrol.utt2spk] \\
        --test-ark test.ark [--test-utt2spk test.utt2spk] --xvec-transform model/transform.npz --plda-file model/plda \\
        [--cohort-ark c.ark --cohort-utt2spk c.utt2spk] [--p-target 0.01,0.001] --scores-out scores --json metrics.json

Sides.  A trial compares an enrolment item with a test item.  An item is a speaker of a utt2spk file (all of its
x-vectors) or, without one, one ark key with its one x-vector.  Both sides go through the front end of the command line
(pipeline._project, --chain auto|tcgen05|float64), and each item gets the statistics n, F, b, e of section 5.15 with
c = Fa / Fb.  The default Fa = Fb = 1 gives the plain two-covariance PLDA LLR in the diagonalised space; --Fa/--Fb give
exactly the LLR that enrolment (section 5.16) thresholds at those diarization settings.

Score.  Without a cohort a trial scores section 5.15's LLR(s, u).  With --cohort-ark/--cohort-utt2spk [--cohort-top K]
it scores section 5.17's S = 1/2 [(LLR - mu_s) / sigma_s + (LLR - mu_u) / sigma_u], mu and sigma each item's top-K
cohort statistics (cohort.cohort_stats with offsets None and the item index as labels, checked by cohort.check_spread).

Trials file.  Kaldi's 'enrol-id test-id target|nontarget' lines (formats.read_trials); a file of two-column lines is
scored only.  Mixed column counts, another label word, an id that is not an item of its side and an empty list are
ValueErrors before any device work; duplicate trials are scored twice.

Metrics.  A trial is accepted at threshold t when score >= t; the candidate thresholds are every distinct score value
(-0.0 and +0.0 one value) and +inf.  P_miss(t) = #targets with score < t / N_tar and P_fa(t) = #nontargets with
score >= t / N_non, exact integer counts and one float64 division each.
  EER: k is the first candidate, ascending, with P_miss >= P_fa (k >= 1 when both classes are present);
       a = P_miss(k-1) - P_fa(k-1), b = P_miss(k) - P_fa(k), lambda = a / (a - b), and
       EER = P_fa(k-1) + lambda (P_fa(k) - P_fa(k-1)), where the segment between the two points crosses P_miss = P_fa.
  minDCF at (p, C_miss, C_fa): min_t (C_miss p P_miss + C_fa (1-p) P_fa) / min(C_miss p, C_fa (1-p)); the threshold
       reported is the lowest that attains it.
  actDCF: the same normalised cost at the Bayes threshold log(C_fa (1-p) / (C_miss p)), score >= it accepted.
  Cllr = 1 / (2 ln 2) [mean over targets of softplus(-s) + mean over nontargets of softplus(s)],
       softplus(x) = max(x, 0) + log1p(exp(-|x|)); meaningful for LLRs only, so the score kind (llr or as-norm) is
       reported next to it.
Defaults p = 0.01, C_miss = C_fa = 1.  The metrics need at least one target and one nontarget trial.

Calibration (DESIGN.md section 5.28).  --calibrate-out FILE fits llr = a s + b to the labelled list by prior-weighted
logistic regression (--calibration-prior, default 0.5) on the device (vbx_verify_calibrate), writes it with the score
kind, Fa, Fb, --lda-dim, --cohort-top and the SHA-256 of the model files, and reports minCllr and the metrics of the
calibrated scores on the same list (self-calibrated: an optimistic figure).  --calibration FILE scores a s + b instead
of s; the file must match this run's kind, Fa, Fb, --lda-dim, --cohort-top and model files.  python -m vbx_b200.cli
--calibration FILE states --link-threshold and --enroll-threshold as calibrated LLRs.

Statistics and scores run in vbx_verify_score, the metrics in vbx_verify_metrics (sort, scans and fixed-order
reductions on the device: bit-identical from run to run and for any order of the trials).
"""
import argparse
import ctypes
import json
import math
import sys
import time

import numpy as np

DEFAULT_P_TARGET = 0.01


def _device(device):
    import torch
    from ._lib import VbxError
    if not torch.cuda.is_available():
        raise VbxError('vbx_b200.verify: no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    return torch.device('cuda', torch.cuda.current_device()) if dev.index is None else dev


def _positive(name, v):
    v = float(v)
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError(f'{name} must be finite and > 0, got {v!r}')
    return v


def check_p_targets(p_targets):
    """The operating points as a list of floats, each in (0, 1); ValueError otherwise or when there is none."""
    out = [float(p) for p in np.atleast_1d(np.asarray(p_targets, dtype=np.float64))]
    if not out:
        raise ValueError('give at least one p_target')
    if len(out) > 64:
        raise ValueError(f'at most 64 operating points, got {len(out)}')
    for p in out:
        if not 0.0 < p < 1.0:
            raise ValueError(f'p_target must lie in (0, 1), got {p!r}')
    return out


def _side(name, fea, item, R=None):
    """(fea [N,R] float32 numpy packed by item, item [N] int32 packed, M) of one side, checked."""
    x = np.asarray(fea.detach().cpu().numpy() if hasattr(fea, 'detach') else fea)
    if x.ndim != 2 or x.shape[0] == 0:
        raise ValueError(f'{name}_fea must be a non-empty [N, R] array')
    if R is not None and x.shape[1] != R:
        raise ValueError(f'{name}_fea has dimension {x.shape[1]}, Phi has {R}')
    if not np.all(np.isfinite(x)):
        raise ValueError(f'{name}_fea holds non-finite values')
    it = np.asarray(item, dtype=np.int64).reshape(-1)
    if len(it) != x.shape[0]:
        raise ValueError(f'{name}_item needs one item per x-vector ({x.shape[0]}), got {len(it)}')
    if it.min() < 0:
        raise ValueError(f'{name}_item must be >= 0')
    M = int(it.max()) + 1
    if np.bincount(it, minlength=M).min() == 0:
        raise ValueError(f'every {name} item 0 .. {M - 1} needs at least one x-vector')
    if M > np.iinfo(np.int32).max:
        raise ValueError(f'more than 2^31 - 1 {name} items')
    order = np.argsort(it, kind='stable')             # each item's x-vectors together: its statistics read one span
    return np.ascontiguousarray(x[order], dtype=np.float32), it[order].astype(np.int32), M


def score_trials(enroll_fea, enroll_item, test_fea, test_item, Phi, trials, Fa=1.0, Fb=1.0, norm=None, device=None):
    """Scores [T] float64 of the trials on the device (vbx_verify_score).  enroll_fea [N_e,R] / test_fea [N_t,R]: the two
    sides' x-vectors through the front end, enroll_item [N_e] / test_item [N_t] their item in [0, M), every item with at
    least one x-vector; Phi [R]; trials [T, 2]: (enrolment item, test item) per trial.  Fa, Fb: c = Fa / Fb of the
    statistics.  norm: None (section 5.15's LLR) or (enroll_mean [M_e], enroll_std [M_e], test_mean [M_t], test_std
    [M_t]) cohort statistics (section 5.17's AS-norm S).  ValueError before any device work: non-finite x-vectors, a
    dimension mismatch, Fa or Fb not finite and positive, a trial index outside its side, bad statistics."""
    import torch
    from . import _lib
    from ._lib import VbxError
    Fa, Fb = _positive('Fa', Fa), _positive('Fb', Fb)
    Phi = np.asarray(Phi.detach().cpu().numpy() if hasattr(Phi, 'detach') else Phi, dtype=np.float32).reshape(-1)
    R = len(Phi)
    if not 1 <= R <= 128 or not np.all(np.isfinite(Phi)):
        raise ValueError(f'Phi must hold 1 .. 128 finite values, got {R}')
    xe, ie, M_e = _side('enroll', enroll_fea, enroll_item, R)
    xt, it, M_t = _side('test', test_fea, test_item, R)
    tr = np.asarray(trials, dtype=np.int64).reshape(-1, 2)
    T = len(tr)
    for k, (side, M) in enumerate((('enrolment', M_e), ('test', M_t))):
        bad = np.nonzero((tr[:, k] < 0) | (tr[:, k] >= M))[0]
        if len(bad):
            raise ValueError(f'trial {int(bad[0])}: {side} item {int(tr[bad[0], k])} outside [0, {M})')
    if norm is not None:
        from .cohort import check_spread
        norm = [np.ascontiguousarray(a, dtype=np.float64) for a in norm]
        if [a.shape for a in norm] != [(M_e,), (M_e,), (M_t,), (M_t,)]:
            raise ValueError(f'norm must hold mean and std of the {M_e} enrolment and the {M_t} test items')
        if not (np.all(np.isfinite(norm[0])) and np.all(np.isfinite(norm[2]))):
            raise ValueError('norm: non-finite cohort means')
        check_spread(norm[1], [f'enrolment item {i}' for i in range(M_e)])
        check_spread(norm[3], [f'test item {j}' for j in range(M_t)])
    dev = _device(device)
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    try:
        need = ctypes.c_size_t()
        if lib.vbx_verify_score_workspace_bytes(h, M_e, M_t, ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_verify_score_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
            fe, fie, ft, fit, ph = d(xe), d(ie), d(xt), d(it), d(Phi)
            ti, tj = d(tr[:, 0].astype(np.int32)), d(tr[:, 1].astype(np.int32))
            st = [d(a) for a in norm] if norm is not None else [None] * 4
            ws = torch.empty(max(int(need.value), 1), dtype=torch.uint8, device=dev)
            out = torch.empty(T, dtype=torch.float64, device=dev)
            rc = lib.vbx_verify_score(h, p(fe), len(xe), p(fie), M_e, p(ft), len(xt), p(fit), M_t, R, p(ph), Fa, Fb,
                                      p(ti), p(tj), T, *map(p, st), p(ws), ws.numel(), p(out), stream)
            if rc != 0:
                raise VbxError(f'vbx_verify_score failed ({rc}): {lib.vbx_last_error(h).decode()}')
            return out.cpu().numpy()
    finally:
        lib.vbx_destroy(h)


def error_rates(scores, labels, p_targets=(DEFAULT_P_TARGET,), c_miss=1.0, c_fa=1.0, device=None):
    """EER, minDCF with its threshold, actDCF and Cllr of scored trials on the device (vbx_verify_metrics).  scores [T]
    (numpy or a torch tensor), labels [T] (true / 1: target trial).  Returns dict(n_target, n_nontarget, eer, cllr,
    p_target, min_dcf, threshold, act_dcf), the last four lists in the order of p_targets.  ValueError before any
    device work: an empty list, labels of another length, no target or no nontarget trial, a p outside (0, 1), costs
    not finite and positive; after the device pass: non-finite scores."""
    import torch
    from . import _lib
    from ._lib import VbxError
    ps = check_p_targets(p_targets)
    c_miss, c_fa = _positive('c_miss', c_miss), _positive('c_fa', c_fa)
    lab = np.asarray(labels).reshape(-1)
    T = int(scores.shape[0]) if hasattr(scores, 'shape') else len(scores)
    if T == 0:
        raise ValueError('no trials')
    if len(lab) != T:
        raise ValueError(f'{len(lab)} labels for {T} scores')
    lab = lab.astype(bool)
    n_tar = int(lab.sum())
    if n_tar == 0 or n_tar == T:
        raise ValueError(f'the metrics need target and nontarget trials, got {n_tar} targets of {T}')
    dev = _device(device)
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    n_op = len(ps)
    try:
        need = ctypes.c_size_t()
        if lib.vbx_verify_metrics_workspace_bytes(h, T, n_op, ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_verify_metrics_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            s = torch.as_tensor(scores).to(dev, torch.float64).contiguous().reshape(-1)
            y = torch.from_numpy(lab.astype(np.uint8)).to(dev)
            ws = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
            counts = torch.empty(3, dtype=torch.int64, device=dev)
            res = torch.empty(2 + 3 * n_op, dtype=torch.float64, device=dev)
            pt = np.ascontiguousarray(ps, dtype=np.float64)
            at = lambda k: ctypes.c_void_p(res.data_ptr() + 8 * k)      # eer, cllr, min_dcf, threshold, act_dcf
            rc = lib.vbx_verify_metrics(h, p(s), p(y), T, n_op, pt.ctypes.data_as(ctypes.c_void_p), c_miss, c_fa,
                                        p(ws), ws.numel(), p(counts), at(0), at(1), at(2), at(2 + n_op),
                                        at(2 + 2 * n_op), stream)
            if rc != 0:
                raise VbxError(f'vbx_verify_metrics failed ({rc}): {lib.vbx_last_error(h).decode()}')
            counts, res = counts.cpu().numpy(), res.cpu().numpy()
    finally:
        lib.vbx_destroy(h)
    if counts[2]:
        raise ValueError(f'{int(counts[2])} non-finite score(s): the metrics need finite scores')
    return dict(n_target=int(counts[0]), n_nontarget=int(counts[1]), eer=float(res[0]), cllr=float(res[1]),
                p_target=ps, min_dcf=res[2:2 + n_op].tolist(), threshold=res[2 + n_op:2 + 2 * n_op].tolist(),
                act_dcf=res[2 + 2 * n_op:].tolist())


CALIBRATION_VERSION = 1
CALIBRATION_KEYS = ('version', 'a', 'b', 'prior', 'score_kind', 'Fa', 'Fb', 'lda_dim', 'cohort_top',
                    'xvec_transform_sha256', 'plda_file_sha256', 'n_target', 'n_nontarget')
SEPARABLE, NONFINITE, NOT_CONVERGED = 1, 2, 3       # vbx_verify_calibrate statuses


def calibrate(scores, labels, prior=0.5, device=None):
    """The linear calibration llr = a s + b of scored trials on the device (vbx_verify_calibrate, DESIGN.md section
    5.28): (a, b) minimise the prior-weighted logistic cost, cllr_prior = C(a, b) / ln 2 (at prior 0.5 the Cllr of
    a s + b), min_cllr the Cllr of the optimal monotone transform of the scores (PAV; at prior 0.5).  Returns dict(a, b,
    prior, cllr_prior, min_cllr, passes, n_target, n_nontarget, hull_vertices).  ValueError before any device work: an
    empty list, labels of another length, no target or no nontarget trial, a prior outside (0, 1); after the device
    pass: separable classes or non-finite scores.  VbxError: the fit did not converge."""
    import torch
    from . import _lib
    from ._lib import VbxError
    prior = float(prior)
    if not 0.0 < prior < 1.0:
        raise ValueError(f'prior must lie in (0, 1), got {prior!r}')
    lab = np.asarray(labels).reshape(-1)
    T = int(scores.shape[0]) if hasattr(scores, 'shape') else len(scores)
    if T == 0:
        raise ValueError('no trials')
    if len(lab) != T:
        raise ValueError(f'{len(lab)} labels for {T} scores')
    lab = lab.astype(bool)
    n_tar = int(lab.sum())
    if n_tar == 0 or n_tar == T:
        raise ValueError(f'a calibration needs target and nontarget trials, got {n_tar} targets of {T}')
    dev = _device(device)
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise VbxError('vbx_create failed: no usable sm_90 device')
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    try:
        need = ctypes.c_size_t()
        if lib.vbx_verify_calibrate_workspace_bytes(h, T, ctypes.byref(need)) != 0:
            raise VbxError(f'vbx_verify_calibrate_workspace_bytes failed: {lib.vbx_last_error(h).decode()}')
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            s = torch.as_tensor(scores).to(dev, torch.float64).contiguous().reshape(-1)
            y = torch.from_numpy(lab.astype(np.uint8)).to(dev)
            ws = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
            info = torch.empty(5, dtype=torch.int64, device=dev)
            res = torch.empty(4, dtype=torch.float64, device=dev)
            rc = lib.vbx_verify_calibrate(h, p(s), p(y), T, prior, p(ws), ws.numel(), p(info), p(res), stream)
            if rc != 0:
                raise VbxError(f'vbx_verify_calibrate failed ({rc}): {lib.vbx_last_error(h).decode()}')
            info, res = info.cpu().numpy(), res.cpu().numpy()
    finally:
        lib.vbx_destroy(h)
    status = int(info[0])
    if status == NONFINITE:
        raise ValueError('non-finite score(s): a calibration needs finite scores')
    if status == SEPARABLE:
        s = np.asarray(scores.detach().cpu().numpy() if hasattr(scores, 'detach') else scores, dtype=np.float64)
        s = s.reshape(-1)
        how = 'at or above' if s[lab].min() >= s[~lab].max() else 'at or below'
        raise ValueError(f'the classes are separable: every target trial scores {how} every nontarget trial, so the '
                         f'logistic regression has no finite minimiser (minCllr {float(res[3]):.6g})')
    if status == NOT_CONVERGED:
        raise VbxError(f'vbx_verify_calibrate: the fit did not converge in {int(info[1])} passes')
    return dict(a=float(res[0]), b=float(res[1]), prior=prior, cllr_prior=float(res[2]), min_cllr=float(res[3]),
                passes=int(info[1]), n_target=int(info[2]), n_nontarget=int(info[3]), hull_vertices=int(info[4]))


def file_sha256(path):
    """The SHA-256 of a file's bytes, hex."""
    import hashlib
    d = hashlib.sha256()
    with open(path, 'rb') as f:
        for chunk in iter(lambda: f.read(1 << 20), b''):
            d.update(chunk)
    return d.hexdigest()


def write_calibration(path, fit, score_kind, Fa, Fb, lda_dim, cohort_top, xvec_transform, plda_file):
    """Write a calibration file (JSON): calibrate's a, b, prior and trial counts, and what the scores it was fitted on
    depend on: the score kind ('llr' / 'as-norm'), Fa, Fb, lda_dim, cohort_top (as-norm only, else None) and the
    SHA-256 of the x-vector transform and PLDA files."""
    if score_kind not in ('llr', 'as-norm'):
        raise ValueError(f'score_kind must be llr or as-norm, got {score_kind!r}')
    doc = dict(version=CALIBRATION_VERSION, a=float(fit['a']), b=float(fit['b']), prior=float(fit['prior']),
               score_kind=score_kind, Fa=float(Fa), Fb=float(Fb), lda_dim=int(lda_dim),
               cohort_top=None if score_kind == 'llr' else int(cohort_top),
               xvec_transform_sha256=file_sha256(xvec_transform), plda_file_sha256=file_sha256(plda_file),
               n_target=int(fit['n_target']), n_nontarget=int(fit['n_nontarget']))
    with open(path, 'w') as f:
        json.dump(doc, f, indent=1)
        f.write('\n')
    return doc


def read_calibration(path):
    """A calibration file as a dict, checked: ValueError for an unknown version, a missing key, a non-finite number, a
    prior outside (0, 1), an unknown score kind, a cohort_top that does not fit the kind, bad counts or hashes."""
    with open(path) as f:
        try:
            doc = json.load(f)
        except json.JSONDecodeError as e:
            raise ValueError(f'{path}: not a calibration file ({e})')
    if not isinstance(doc, dict):
        raise ValueError(f'{path}: not a calibration file')
    if doc.get('version') != CALIBRATION_VERSION:
        raise ValueError(f'{path}: calibration format version {doc.get("version")!r}, this reader knows '
                         f'{CALIBRATION_VERSION}')
    missing = [k for k in CALIBRATION_KEYS if k not in doc]
    if missing:
        raise ValueError(f'{path}: missing {", ".join(missing)}')
    for k in ('a', 'b', 'prior', 'Fa', 'Fb'):
        v = doc[k]
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
            raise ValueError(f'{path}: {k} must be a finite number, got {v!r}')
        doc[k] = float(v)
    if not 0.0 < doc['prior'] < 1.0:
        raise ValueError(f'{path}: prior must lie in (0, 1), got {doc["prior"]!r}')
    if not (doc['Fa'] > 0 and doc['Fb'] > 0):
        raise ValueError(f'{path}: Fa and Fb must be > 0')
    if doc['score_kind'] not in ('llr', 'as-norm'):
        raise ValueError(f'{path}: score_kind must be llr or as-norm, got {doc["score_kind"]!r}')
    for k in ('lda_dim', 'n_target', 'n_nontarget'):
        if isinstance(doc[k], bool) or not isinstance(doc[k], int) or doc[k] < 1:
            raise ValueError(f'{path}: {k} must be an integer >= 1, got {doc[k]!r}')
    top = doc['cohort_top']
    if doc['score_kind'] == 'llr' and top is not None:
        raise ValueError(f'{path}: cohort_top is for as-norm scores only')
    if doc['score_kind'] == 'as-norm' and (isinstance(top, bool) or not isinstance(top, int) or top < 2):
        raise ValueError(f'{path}: as-norm scores need an integer cohort_top >= 2, got {top!r}')
    for k in ('xvec_transform_sha256', 'plda_file_sha256'):
        v = doc[k]
        if not (isinstance(v, str) and len(v) == 64 and all(c in '0123456789abcdef' for c in v)):
            raise ValueError(f'{path}: {k} must be a SHA-256 in hex')
    return doc


def raw_threshold(cal, t):
    """The raw score threshold (t - b) / a in float64 of a calibrated LLR threshold t: a calibrated score a s + b is
    >= t exactly where s >= (t - b) / a, up to the rounding of this division.  ValueError when a <= 0 (the
    calibration does not keep the scores' order)."""
    a, b = float(cal['a']), float(cal['b'])
    if not a > 0.0:
        raise ValueError(f'the calibration\'s slope a = {a!r} is not positive: a threshold cannot be carried over')
    return (float(t) - b) / a


def calibration_mismatch(cal, score_kind, Fa, Fb, lda_dim, cohort_top, xvec_transform, plda_file):
    """The first way in which a calibration does not fit a run's scores, as a message, or None."""
    want = dict(score_kind=score_kind, Fa=float(Fa), Fb=float(Fb), lda_dim=int(lda_dim),
                cohort_top=None if score_kind == 'llr' else int(cohort_top))
    for k, v in want.items():
        if cal[k] != v:
            return f'the calibration was fitted with {k} {cal[k]!r}, this run has {v!r}'
    for k, path in (('xvec_transform_sha256', xvec_transform), ('plda_file_sha256', plda_file)):
        if cal[k] != file_sha256(path):
            return f'the calibration was fitted with another {k[:-7].replace("_", "-")} ({path} differs)'
    return None


def trial_norm(enroll_fea, enroll_item, test_fea, test_item, Phi, cohort_fea, cohort_speaker, Fa=1.0, Fb=1.0,
               top_k=None, device=None):
    """The norm= of score_trials: each side's items' top-K cohort statistics (cohort.cohort_stats with offsets None and
    the item index as labels), checked by cohort.check_spread.  Returns (enroll_mean, enroll_std, test_mean,
    test_std)."""
    from . import cohort
    top_k = cohort.DEFAULT_TOP_K if top_k is None else top_k
    out = []
    for name, fea, item in (('enrolment', enroll_fea, enroll_item), ('test', test_fea, test_item)):
        x, it, M = _side(name, fea, item, len(np.asarray(Phi).reshape(-1)))
        st = cohort.cohort_stats(x, Phi, None, it, cohort_fea, cohort_speaker, Fa, Fb, top_k, device)
        cohort.check_spread(st.std, [f'{name} item {k}' for k in range(M)])
        out += [st.mean, st.std]
    return tuple(out)


# ---- command line ------------------------------------------------------------------------------------------------------

def read_items(ark, utt2spk=None):
    """(names, x [N, Dx] float64, item [N]) of one side: the speakers of utt2spk (formats.read_enrolment), or every ark
    key as an item of one x-vector.  ValueError: a key listed twice without utt2spk."""
    from . import formats
    if utt2spk is not None:
        sets = formats.read_enrolment(ark, utt2spk)
        names = list(sets)
        return names, np.concatenate([sets[n] for n in names]), np.repeat(np.arange(len(names)),
                                                                          [len(sets[n]) for n in names])
    names, rows = [], []
    for key, vec in formats.read_vec_flt_ark(ark):
        names.append(key)
        rows.append(np.asarray(vec, dtype=np.float64))
    if len(set(names)) != len(names):
        raise ValueError(f'{ark}: a key is listed twice (give a utt2spk file to group x-vectors into items)')
    if not names:
        raise ValueError(f'{ark}: no x-vectors')
    return names, np.stack(rows), np.arange(len(names))


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--trials', required=True, help='Kaldi trial list: "enrol-id test-id [target|nontarget]" lines')
    ap.add_argument('--enroll-ark', required=True, help='x-vectors of the enrolment side (Kaldi ark)')
    ap.add_argument('--enroll-utt2spk', default=None,
                    help='speaker of each enrolment x-vector: items are speakers (default: every ark key is an item)')
    ap.add_argument('--test-ark', required=True, help='x-vectors of the test side (Kaldi ark)')
    ap.add_argument('--test-utt2spk', default=None,
                    help='speaker of each test x-vector: items are speakers (default: every ark key is an item)')
    ap.add_argument('--xvec-transform', required=True, help='x-vector transform (transform.h5 or train\'s .npz)')
    ap.add_argument('--plda-file', required=True, help='Kaldi PLDA, binary or text')
    ap.add_argument('--lda-dim', type=int, default=128, help='dimension after the LDA (default 128)')
    ap.add_argument('--chain', default='auto', choices=['auto', 'tcgen05', 'float64'],
                    help='front end arithmetic, as for the command line')
    ap.add_argument('--device', default=None, help='CUDA device, e.g. cuda:0 (default: the current device)')
    ap.add_argument('--Fa', type=float, default=1.0, help='Fa of the statistics (default 1: the plain PLDA LLR)')
    ap.add_argument('--Fb', type=float, default=1.0, help='Fb of the statistics (default 1)')
    ap.add_argument('--cohort-ark', default=None, help='x-vectors of cohort speakers (Kaldi ark): AS-norm scores')
    ap.add_argument('--cohort-utt2spk', default=None, help='the speaker of each x-vector of --cohort-ark')
    ap.add_argument('--cohort-top', type=int, default=None,
                    help='how many of each item\'s largest cohort scores set its mean and spread (default 200)')
    ap.add_argument('--p-target', default=str(DEFAULT_P_TARGET),
                    help='comma list of target priors in (0, 1) for minDCF and actDCF (default 0.01)')
    ap.add_argument('--c-miss', type=float, default=1.0, help='cost of a miss (default 1)')
    ap.add_argument('--c-fa', type=float, default=1.0, help='cost of a false alarm (default 1)')
    ap.add_argument('--scores-out', default=None, help='write "enrol test score" lines in trial order')
    ap.add_argument('--json', default=None, help='write the metrics, score kind, counts and timings as JSON')
    ap.add_argument('--calibrate-out', default=None,
                    help='fit the calibration llr = a s + b to the labelled trials (DESIGN.md section 5.28) and write '
                         'it to this file; the metrics of the calibrated scores on the same list are reported too')
    ap.add_argument('--calibration-prior', type=float, default=None,
                    help='with --calibrate-out: the prior of the logistic regression (default 0.5)')
    ap.add_argument('--calibration', default=None,
                    help='a calibration file of --calibrate-out: score a s + b for the metrics and --scores-out')
    return ap


def check_args(ap, args):
    """Usage errors (exit 2); returns the operating points."""
    if (args.cohort_ark is None) != (args.cohort_utt2spk is None):
        ap.error('--cohort-ark and --cohort-utt2spk go together')
    if args.cohort_top is not None and args.cohort_ark is None:
        ap.error('--cohort-top needs --cohort-ark and --cohort-utt2spk')
    if args.cohort_top is not None and args.cohort_top < 2:
        ap.error('--cohort-top must be >= 2')
    if args.lda_dim < 1:
        ap.error('--lda-dim must be >= 1')
    if args.calibrate_out is not None and args.calibration is not None:
        ap.error('--calibrate-out and --calibration do not combine: fit on one list, apply to another')
    if args.calibration_prior is not None:
        if args.calibrate_out is None:
            ap.error('--calibration-prior needs --calibrate-out')
        if not 0.0 < args.calibration_prior < 1.0:
            ap.error('--calibration-prior must lie in (0, 1)')
    for name in ('Fa', 'Fb', 'c_miss', 'c_fa'):
        v = getattr(args, name)
        if not (math.isfinite(v) and v > 0):
            ap.error(f'--{name.replace("_", "-")} must be finite and > 0')
    try:
        return check_p_targets([float(t) for t in args.p_target.split(',')])
    except ValueError as e:
        ap.error(f'--p-target: {e}')


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    ps = check_args(ap, args)
    cal = None
    if args.calibration is not None:
        try:
            cal = read_calibration(args.calibration)
            why = calibration_mismatch(cal, 'llr' if args.cohort_ark is None else 'as-norm', args.Fa, args.Fb,
                                       args.lda_dim, 200 if args.cohort_top is None else args.cohort_top,
                                       args.xvec_transform, args.plda_file)
        except (OSError, ValueError) as e:
            ap.error(f'--calibration: {e}')
        if why is not None:
            ap.error(f'--calibration: {why}')
    from . import formats, pipeline
    t0 = time.perf_counter()
    en, xe, ie = read_items(args.enroll_ark, args.enroll_utt2spk)
    tn, xt, it = read_items(args.test_ark, args.test_utt2spk)
    e_ids, t_ids, labels = formats.read_trials(args.trials, en, tn)
    if args.calibrate_out is not None and labels is None:
        ap.error('--calibrate-out needs a labelled trial list')
    ei, ti = {n: k for k, n in enumerate(en)}, {n: k for k, n in enumerate(tn)}
    trials = np.stack([np.array([ei[n] for n in e_ids], dtype=np.int64), np.array([ti[n] for n in t_ids], dtype=np.int64)], 1)
    cohort = formats.read_enrolment(args.cohort_ark, args.cohort_utt2spk) if args.cohort_ark is not None else None
    plda = formats.read_kaldi_plda(args.plda_file)
    transform = formats.read_xvec_transform(args.xvec_transform)
    Dx = np.asarray(transform[0]).shape[0]
    for name, D in [('enrolment', xe.shape[1]), ('test', xt.shape[1])] + [('cohort', v.shape[1]) for v in
                                                                           (cohort or {}).values()]:
        if D != Dx:
            raise ValueError(f'{name} x-vectors have dimension {D}, the transform takes {Dx}')
    t1 = time.perf_counter()
    dev = _device(args.device)
    parts = [xe, xt] + ([np.concatenate(list(cohort.values()))] if cohort else [])
    x_all = np.concatenate(parts)
    chain = pipeline._resolve_chain(args.chain, transform, plda, args.lda_dim, x_all.shape[1])
    front, _, fea, Phi = pipeline._project(x_all, [len(x_all)], transform, plda, args.lda_dim, chain, dev)
    front.close()
    fea = fea.cpu().numpy()
    Phi = Phi.cpu().numpy()
    fe, ft = fea[:len(xe)], fea[len(xe):len(xe) + len(xt)]
    t2 = time.perf_counter()
    norm = None
    if cohort is not None:
        fc = fea[len(xe) + len(xt):]
        cspk = np.repeat(np.arange(len(cohort)), [len(v) for v in cohort.values()])
        norm = trial_norm(fe, ie, ft, it, Phi, fc, cspk, args.Fa, args.Fb, args.cohort_top, dev)
    t3 = time.perf_counter()
    scores = score_trials(fe, ie, ft, it, Phi, trials, Fa=args.Fa, Fb=args.Fb, norm=norm, device=dev)
    t4 = time.perf_counter()
    kind = 'llr' if norm is None else 'as-norm'
    if cal is not None:
        scores = cal['a'] * scores + cal['b']
    metrics = None
    if labels is not None:
        metrics = error_rates(scores, labels, ps, args.c_miss, args.c_fa, device=dev)
    t5 = time.perf_counter()
    fit = fit_metrics = None
    if args.calibrate_out is not None:
        fit = calibrate(scores, labels, 0.5 if args.calibration_prior is None else args.calibration_prior, device=dev)
        write_calibration(args.calibrate_out, fit, kind, args.Fa, args.Fb, args.lda_dim,
                          200 if args.cohort_top is None else args.cohort_top, args.xvec_transform, args.plda_file)
        fit_metrics = error_rates(fit['a'] * scores + fit['b'], labels, ps, args.c_miss, args.c_fa, device=dev)
    t6 = time.perf_counter()
    if args.scores_out is not None:
        with open(args.scores_out, 'w') as f:
            f.write(''.join(f'{a} {b} {float(s)!r}\n' for a, b, s in zip(e_ids, t_ids, scores.tolist())))
    n_tar = None if labels is None else int(labels.sum())
    if args.json is not None:
        doc = dict(score_kind=kind, n_trials=len(scores), n_target=n_tar,
                   n_nontarget=None if labels is None else len(scores) - n_tar,
                   n_enroll_items=len(en), n_test_items=len(tn), Fa=args.Fa, Fb=args.Fb,
                   cohort_speakers=None if cohort is None else len(cohort),
                   cohort_top=None if cohort is None else (200 if args.cohort_top is None else args.cohort_top),
                   c_miss=args.c_miss, c_fa=args.c_fa, chain=chain,
                   timings_s=dict(read=t1 - t0, front_end=t2 - t1, cohort=t3 - t2, score=t4 - t3, metrics=t5 - t4))
        if metrics is not None:
            doc.update(eer=metrics['eer'], cllr=metrics['cllr'],
                       operating_points=[dict(p_target=p, min_dcf=m, threshold=th, act_dcf=a) for p, m, th, a in
                                         zip(ps, metrics['min_dcf'], metrics['threshold'], metrics['act_dcf'])])
        if cal is not None:
            doc.update(calibration_applied=dict(file=args.calibration, a=cal['a'], b=cal['b'], prior=cal['prior']))
        if fit is not None:
            doc['timings_s']['calibrate'] = t6 - t5
            doc.update(min_cllr=fit['min_cllr'], calibration=dict(
                a=fit['a'], b=fit['b'], prior=fit['prior'], cllr_prior=fit['cllr_prior'], passes=fit['passes'],
                hull_vertices=fit['hull_vertices'], self_calibrated=True, eer=fit_metrics['eer'],
                cllr=fit_metrics['cllr'],
                operating_points=[dict(p_target=p, min_dcf=m, threshold=th, act_dcf=a) for p, m, th, a in
                                  zip(ps, fit_metrics['min_dcf'], fit_metrics['threshold'], fit_metrics['act_dcf'])]))
        with open(args.json, 'w') as f:
            json.dump(doc, f, indent=1)
    if metrics is None:
        print(f'verify: {len(scores)} trials scored ({kind}), no labels: no metrics')
    else:
        ops = ', '.join(f'minDCF(p={p:g}) {m:.4f} at {th:.4g}, actDCF {a:.4f}' for p, m, th, a in
                        zip(ps, metrics['min_dcf'], metrics['threshold'], metrics['act_dcf']))
        print(f'verify: {len(scores)} trials ({n_tar} target), {kind}: EER {100 * metrics["eer"]:.3f} %, {ops}, '
              f'Cllr ({kind}) {metrics["cllr"]:.4f}')
    if fit is not None:
        print(f'verify: calibration a {fit["a"]:.6g}, b {fit["b"]:.6g} at prior {fit["prior"]:g} written to '
              f'{args.calibrate_out}: minCllr {fit["min_cllr"]:.4f}, Cllr of the calibrated scores (self-calibrated) '
              f'{fit_metrics["cllr"]:.4f}')
    return 0


if __name__ == '__main__':
    sys.exit(main())
