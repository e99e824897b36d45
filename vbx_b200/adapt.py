"""Adapt the back end to the archive being diarized (DESIGN.md section 5.26): unsupervised adaptation of an existing
PLDA to the archive's own x-vectors, interpolation of two PLDAs, and a transform whose centring means are re-estimated
on the archive.  The model is Kaldi's ivector-adapt-plda with its three knobs and their defaults; Kaldi is not run here
and nothing is claimed to match it.

    python -m vbx_b200.cli ... --adapt [--recentre] [--adapt-within-scale 0.3 --adapt-between-scale 0.7 ...]
    python -m vbx_b200.train --xvec-ark-file archive.ark --adapt-plda plda --xvec-transform transform.h5 --out-dir model

The definition, all float64:
  covariance form  a PLDA (mu, T, psi) of dimension d has W = T^-1 T^-T and B = T^-1 diag(psi) T^-T
                   (plda_covariances); plda_from_covariances turns (mu, W, B) back into Kaldi form, as train_backend
                   writes it.
  re-centring      (recentre_transform) from the raw x-vectors x of the adaptation set: mean1' = mean(x),
                   mean2' = mean(l2_norm(x - mean1')) lda, lda unchanged.
  statistics       z = the adaptation set through the (possibly re-centred) transform, as the archive's own front end
                   computes it (pipeline._project's first pass, float32, on the chain the diarization uses); m = mean(z)
                   and C = scatter / N, the scatter from vbx_class_scatter on those rows as one class.
  adaptation       scales w (within, 0.3), b (between, 0.7), s (mean, 1.0): Delta = m - mu, C' = C + s Delta Delta^T,
                   Sigma = W + B; C' v = lambda Sigma v with V^T Sigma V = I; e_i = max(0, lambda_i - 1),
                   E = Sigma V diag(e) V^T Sigma (the variance the archive shows beyond the model's total along each
                   generalised direction); W' = W + w E, B' = B + b E, mu' = m.  If C' <= Sigma, W' and B' are W and B
                   bit for bit; if w + b = 1, V^T (W' + B') V = diag(max(lambda, 1)).
  interpolation    for alpha in [0, 1]: (mu, W, B) = alpha (in-domain) + (1 - alpha) (other), both PLDAs of the same d
                   in the same transform's space.
The d x d eigenproblems run in float64 scipy on the host, the re-centring means in float64 torch on the device.
"""
import math
import time

import numpy as np
import torch

from . import pipeline, train
from .train import plda_from_covariances  # noqa: F401  (part of this module's interface)

SCALES = dict(within_scale=0.3, between_scale=0.7, mean_scale=1.0)


def check_scales(**scales):
    """The adaptation scales with their defaults filled in: ValueError for an unknown name or a negative or
    non-finite value."""
    unknown = sorted(set(scales) - set(SCALES))
    if unknown:
        raise ValueError(f'unknown adaptation scale(s) {unknown}; expected {sorted(SCALES)}')
    out = dict(SCALES, **scales)
    for k, v in out.items():
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) \
                or not math.isfinite(v) or v < 0:
            raise ValueError(f'{k} must be a finite number >= 0, got {v!r}')
        out[k] = float(v)
    return out


def check_alpha(alpha):
    if isinstance(alpha, (bool, np.bool_)) or not isinstance(alpha, (int, float, np.integer, np.floating)) \
            or not 0.0 <= alpha <= 1.0:
        raise ValueError(f'alpha must lie in [0, 1], got {alpha!r}')
    return float(alpha)


def check_plda(plda):
    """(mu, T, psi) as float64 arrays, checked: shapes, finite values, psi >= 0 and T not singular."""
    mu, T, psi = (np.asarray(a, dtype=np.float64) for a in plda)
    d = mu.shape[0] if mu.ndim == 1 else -1
    if mu.ndim != 1 or T.shape != (d, d) or psi.shape != (d,):
        raise ValueError(f'inconsistent PLDA dimensions: mean {mu.shape}, transform {T.shape}, psi {psi.shape}')
    if not all(np.all(np.isfinite(a)) for a in (mu, T, psi)):
        raise ValueError('the PLDA holds non-finite values')
    if np.any(psi < 0):
        raise ValueError(f'the PLDA has psi < 0: {int((psi < 0).sum())} value(s), the smallest {psi.min():.6g}')
    cond = np.linalg.cond(T)
    if not cond < 1.0 / np.finfo(np.float64).eps:
        raise ValueError(f'the PLDA transform is singular (condition number {cond:.3g})')
    return mu, T, psi


def plda_covariances(plda):
    """(mu, W, B) of a Kaldi-form PLDA (mu, T, psi): W = T^-1 T^-T, B = T^-1 diag(psi) T^-T (checked as check_plda)."""
    mu, T, psi = check_plda(plda)
    Ti = np.linalg.inv(T)
    W, B = Ti @ Ti.T, (Ti * psi[None, :]) @ Ti.T
    return mu, 0.5 * (W + W.T), 0.5 * (B + B.T)


def check_compatible(transform, plda):
    """ValueError unless the transform's lda width is the PLDA's d."""
    d_t, d_p = int(np.asarray(transform[2]).shape[1]), int(np.asarray(plda[0]).shape[0])
    if d_t != d_p:
        raise ValueError(f'the x-vector transform maps to d = {d_t}, the PLDA has d = {d_p}')


def adapt_covariances(mu, W, B, mean, cov, within_scale, between_scale, mean_scale):
    """The adaptation of the module docstring on the covariance form.  Returns (mu', W', B', lambda ascending, V)."""
    from scipy.linalg import eigh
    delta = np.asarray(mean, dtype=np.float64) - mu
    Cp = np.asarray(cov, dtype=np.float64) + mean_scale * np.outer(delta, delta)
    Sigma = W + B
    lam, V = eigh(0.5 * (Cp + Cp.T), Sigma)
    e = np.maximum(lam - 1.0, 0.0)
    SV = Sigma @ V
    E = (SV * e[None, :]) @ SV.T
    E = 0.5 * (E + E.T)
    return np.asarray(mean, dtype=np.float64).copy(), W + within_scale * E, B + between_scale * E, lam, V


def adapt_plda(plda, mean, cov, within_scale=0.3, between_scale=0.7, mean_scale=1.0):
    """Adapt the Kaldi-form PLDA (mu, T, psi) to an adaptation set of mean [d] and covariance cov [d, d] (the module
    docstring's definition).  Returns (adapted PLDA in Kaldi form, report: |Delta|, lambda descending, the number of
    inflated directions, the scales)."""
    scales = check_scales(within_scale=within_scale, between_scale=between_scale, mean_scale=mean_scale)
    mu, W, B = plda_covariances(plda)
    mean, cov = np.asarray(mean, dtype=np.float64), np.asarray(cov, dtype=np.float64)
    if mean.shape != mu.shape or cov.shape != W.shape:
        raise ValueError(f'adaptation statistics of shape {mean.shape}, {cov.shape} for a PLDA of d = {mu.shape[0]}')
    if not (np.all(np.isfinite(mean)) and np.all(np.isfinite(cov))):
        raise ValueError('non-finite adaptation statistics')
    mu2, W2, B2, lam, _ = adapt_covariances(mu, W, B, mean, cov, **scales)
    report = dict(delta_norm=float(np.linalg.norm(mean - mu)), eigenvalues=lam[::-1].tolist(),
                  inflated=int((lam > 1.0).sum()), scales=scales)
    return plda_from_covariances(mu2, W2, B2), report


def interpolate_plda(plda_in, plda_out, alpha):
    """alpha (plda_in) + (1 - alpha) (plda_out) on the covariance form (mu, W, B), in Kaldi form; both PLDAs must have
    the same d and live in the same transform's space."""
    alpha = check_alpha(alpha)
    a, b = plda_covariances(plda_in), plda_covariances(plda_out)
    if a[0].shape != b[0].shape:
        raise ValueError(f'PLDAs of different dimension: d = {a[0].shape[0]} and d = {b[0].shape[0]}')
    return plda_from_covariances(*(alpha * p + (1.0 - alpha) * q for p, q in zip(a, b)))


def _archive_x(recordings):
    """(lens, x [N, Dx] float64) of {name: (x, seg_times)}, checked: at least 2 x-vectors, all finite."""
    names = list(recordings)
    lens = np.array([np.asarray(recordings[n][0]).shape[0] for n in names], dtype=np.int64)
    x = np.concatenate([np.asarray(recordings[n][0], dtype=np.float64).reshape(int(lens[i]), -1)
                        for i, n in enumerate(names)]) if names else np.zeros((0, 0))
    if x.shape[0] < 2:
        raise ValueError(f'adaptation needs at least 2 x-vectors, the archive has {x.shape[0]}')
    bad = int((~np.isfinite(x)).any(1).sum())
    if bad:
        raise ValueError(f'the archive holds {bad} non-finite x-vector(s)')
    return lens, x


def recentre_transform(transform, x_raw, device=None):
    """(mean1', mean2', lda) from raw x-vectors x_raw [N, Dx] (array or tensor): mean1' = mean(x), mean2' =
    mean(l2_norm(x - mean1')) lda, in float64 torch on `device` (default: the current CUDA device)."""
    dev = torch.device(device) if device is not None else train._device(None)
    x = torch.as_tensor(x_raw).to(dev, torch.float64)
    mean1, mean2, lda = train.check_transform(transform, int(x.shape[1]) if x.dim() == 2 else None)
    if x.dim() != 2 or x.shape[0] < 2:
        raise ValueError(f're-centring needs at least 2 x-vectors of shape [N, Dx], got {tuple(x.shape)}')
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f'{int((~torch.isfinite(x)).any(1).sum())} non-finite x-vector(s)')
    m1 = x.mean(0)
    y = pipeline.l2_norm_rows(x - m1[None, :]).mean(0)
    return m1.cpu().numpy(), (y @ torch.from_numpy(lda).to(dev)).cpu().numpy(), lda


def project_archive(x, lens, transform, plda, lda_dim=128, chain='auto', device=None):
    """The first-pass output z [N, d] float32 on the device of the archive's front end (pipeline._project's x) for raw
    x-vectors x [N, Dx] packed as recordings of lens, on the chain diarize_batch resolves for these arguments."""
    dev = train._device(device)
    x = np.asarray(x, dtype=np.float64)
    chain = pipeline._resolve_chain(chain, transform, plda, lda_dim, int(x.shape[1]))
    front, z, _, _ = pipeline._project(x, np.asarray(lens, dtype=np.int64), transform, plda, lda_dim, chain, dev)
    front.close()
    return z.float().contiguous()


def archive_stats(z, device=None):
    """(mean [d], covariance [d, d]) float64 on the device of the rows z [N, d] (rounded to float32), from one
    vbx_class_scatter call with the archive as one class: covariance = scatter / N."""
    z = torch.as_tensor(z).to(train._device(device), torch.float32).contiguous()
    N = int(z.shape[0])
    means, scatter = train.class_stats(z, [0, N], z.device)
    return means[0], scatter / N


def adapt_backend(recordings, transform, plda, lda_dim=128, chain='auto', device=None, recentre=False, adapt=True,
                  **scales):
    """The back end adapted to an archive {name: (x_raw [T, Dx], seg_times)} (diarize_batch's recordings): with recentre
    the transform's centring means re-estimated on the archive's raw x-vectors, with adapt the PLDA adapted to the
    archive's statistics through that transform (scales: within_scale, between_scale, mean_scale).  Everything is
    checked before any device work.  Returns (transform', plda', report: N, recentre, adapt, chain, and with adapt
    delta_norm, the eigenvalues lambda descending, the number of inflated directions and the scales; seconds per
    stage)."""
    if scales and not adapt:
        raise ValueError(f'adaptation scales {sorted(scales)} without adapt')
    scales = check_scales(**scales)
    transform = train.check_transform(transform)
    check_plda(plda)
    check_compatible(transform, plda)
    lens, x = _archive_x(recordings)
    train.check_transform(transform, int(x.shape[1]))
    dev = train._device(device)
    t = {}
    t0 = train._sync(dev)
    report = dict(N=int(x.shape[0]), recentre=bool(recentre), adapt=bool(adapt))
    if recentre:
        transform = recentre_transform(transform, x, dev)
        t1 = train._sync(dev)
        t['recentre'], t0 = t1 - t0, t1
    if adapt:
        report['chain'] = pipeline._resolve_chain(chain, transform, plda, lda_dim, int(x.shape[1]))
        z = project_archive(x, lens, transform, plda, lda_dim, chain, dev)
        t1 = train._sync(dev)
        t['project'] = t1 - t0
        m, C = archive_stats(z, dev)
        del z
        t2 = train._sync(dev)
        t['stats'] = t2 - t1
        plda, rep = adapt_plda(plda, m.cpu().numpy(), C.cpu().numpy(), **scales)
        t['adapt'] = time.perf_counter() - t2
        report.update(rep)
    report['seconds'] = t
    return transform, plda, report
