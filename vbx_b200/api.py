"""Drop-in replacement for the reference's `VBx()` (VBx/VBx.py:27-126) running on the H100.

Same positional/keyword arguments, same `(gamma, pi, Li[, alpha, invL])` return with float64 numpy
arrays, same exceptions for bad arguments; the work itself happens in the CUDA library.  The
reference's single call site is VBx/vbhmm.py:154-158.
"""
import os

import numpy as np
import torch

from . import _lib
from .batch import VbxBatch, run_f64

# Arithmetic of the drop-in call.  'float64' (default): every quantity in float64 on the GPU, reproduces the
# reference's iteration count and values to ~1e-9 (VBx/vbhmm.py:157 stops on an ELBO step of 1e-6).  'float32': the
# fast kernels of the batched path with their float64 finish near the stop rule (DESIGN.md section 3): same iteration
# counts, values within 1e-4 relative (measured 2e-7 on ES2005a), half the latency.
PRECISION = os.environ.get('VBX_B200_PRECISION', 'float64')


def set_precision(name):
    global PRECISION
    if name not in ('float32', 'float64'):
        raise ValueError("precision must be 'float32' or 'float64'")
    PRECISION = name


def DER(q, ref, expected=True, xentropy=False):
    """The optional diagnostic of the reference module (VBx/VBx.py:129-143; never called by vbhmm.py): diarization error
    rate or per-frame cross-entropy of the posteriors q [T,S] against integer reference labels ref [T], under the best
    one-to-one mapping of reference speakers to HMM states.  expected=False scores the hard decisions argmax(q).
    Host-side (numpy + scipy's Hungarian solver): it is a scoring aid, not part of the GPU path."""
    from scipy.optimize import linear_sum_assignment
    q = np.asarray(q, dtype=np.float64)
    ref = np.asarray(ref).astype(np.int64).reshape(-1)
    n_frames = ref.shape[0]
    if q.shape[0] != n_frames:
        raise ValueError('DER: q and ref disagree on the number of frames')
    if not expected:
        hard = np.zeros_like(q)
        hard[np.arange(n_frames), q.argmax(axis=1)] = 1.0
        q = hard
    frame_cost = -np.log(q + np.nextafter(0, 1)) if xentropy else -q
    # cost[r, s] = total cost of explaining the frames of reference speaker r with state s
    cost = np.zeros((int(ref.max()) + 1 if n_frames else 0, q.shape[1]))
    np.add.at(cost, ref, frame_cost)
    rows, cols = linear_sum_assignment(cost)
    best = cost[rows, cols].sum()
    return best / float(n_frames) if xentropy else (n_frames + best) / float(n_frames)


def forward_backward(lls, tr, ip):
    """The module-level forward_backward() of the reference (VBx/VBx.py:146-175) on the GPU, for any transition matrix:
    returns (state posteriors [T,S], total log-likelihood, log-forward [T,S], log-backward [T,S]) as float64 numpy."""
    import ctypes
    lls = np.ascontiguousarray(lls, dtype=np.float64)
    tr = np.ascontiguousarray(tr, dtype=np.float64)
    ip = np.ascontiguousarray(ip, dtype=np.float64)
    T, S = lls.shape
    assert tr.shape == (S, S) and ip.shape == (S,)
    if not torch.cuda.is_available():
        raise _lib.VbxError('forward_backward(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device())
    lib = _lib.load()
    h = ctypes.c_void_p()
    if lib.vbx_create(dev.index, ctypes.byref(h)) != 0:
        raise _lib.VbxError('vbx_create failed: no usable sm_90 device')
    try:
        d = lambda a: torch.from_numpy(a).to(dev)
        lls_d, tr_d, ip_d = d(lls), d(tr), d(ip)
        post, lfw, lbw = (torch.empty((T, S), dtype=torch.float64, device=dev) for _ in range(3))
        tll = torch.empty(1, dtype=torch.float64, device=dev)
        ptr = lambda t: ctypes.c_void_p(t.data_ptr())
        rc = lib.vbx_forward_backward(h, ptr(lls_d), ptr(tr_d), ptr(ip_d), T, S, ptr(post), ptr(tll), ptr(lfw), ptr(lbw),
                                      ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        if rc != 0:
            raise _lib.VbxError(f'vbx_forward_backward failed ({rc}): {lib.vbx_last_error(h).decode()}')
        return post.cpu().numpy(), float(tll.item()), lfw.cpu().numpy(), lbw.cpu().numpy()
    finally:
        lib.vbx_destroy(h)


# Plans (handle + device plan + workspace) of the most recent call shapes: vbhmm.py calls VBx() once per recording, a
# service calls it with recurring shapes; re-planning costs a cudaMalloc and a dozen synchronous copies per call.
_PLAN_CACHE = {}
_PLAN_CACHE_SIZE = 8


def _cached_batch(T, D, S, dev, allocate, f64_only=False):
    key = (int(T), int(D), int(S), dev.index, bool(allocate), bool(f64_only))
    vb = _PLAN_CACHE.pop(key, None)
    if vb is None:
        vb = VbxBatch([T], D, S, device=dev, allocate=allocate, f64_only=f64_only)
        vb.rho = None
    _PLAN_CACHE[key] = vb                       # most recently used last
    while len(_PLAN_CACHE) > _PLAN_CACHE_SIZE:
        _PLAN_CACHE.pop(next(iter(_PLAN_CACHE))).close()
    return vb


def clear_plan_cache():
    """Drop the cached plans (frees their device memory)."""
    while _PLAN_CACHE:
        _PLAN_CACHE.popitem()[1].close()


def VBx(X, Phi, loopProb=0.9, Fa=1.0, Fb=1.0, pi=10, gamma=None, maxIters=10,
        epsilon=1e-4, alphaQInit=1.0, ref=None, plot=False,
        return_model=False, alpha=None, invL=None):
    """See VBx/VBx.py:30-68 for the meaning of every argument (kept identical).

    Runs on the GPU in float64 by default (module variable PRECISION / env VBX_B200_PRECISION; 'float32' selects the
    fast kernels of the batched path); outputs are float64 numpy like the reference's."""
    X = np.asarray(X)
    Phi = np.asarray(Phi)
    T, D = X.shape                                    # VBx/VBx.py:74
    if PRECISION == 'float32' and D % 4 != 0 and D < 128:
        # The kernels want a feature dimension that is a multiple of 4.  Zero features with zero across-class
        # variance are inert: invL = 1, alpha = 0, no bias, no regulariser term; only the constant D*log(2*pi) of G
        # (VBx/VBx.py:87) depends on D, which is put back into the ELBO trace below.
        pad = 4 - D % 4
        res = VBx(np.concatenate([X, np.zeros((T, pad), dtype=X.dtype)], axis=1),
                  np.concatenate([Phi, np.zeros(pad, dtype=Phi.dtype)]), loopProb=loopProb, Fa=Fa, Fb=Fb, pi=pi, gamma=gamma,
                  maxIters=maxIters, epsilon=epsilon, alphaQInit=alphaQInit, ref=ref, plot=plot, return_model=return_model,
                  alpha=None if alpha is None else np.concatenate([alpha, np.zeros((alpha.shape[0], pad))], axis=1),
                  invL=None if invL is None else np.concatenate([invL, np.ones((invL.shape[0], pad))], axis=1))
        shift = 0.5 * Fa * T * pad * np.log(2 * np.pi)
        Li = [[l[0] + shift] + l[1:] for l in res[2]]
        out = (res[0], res[1], Li)
        if return_model:
            out = out + (res[3][:, :D], res[4][:, :D])
        return out
    if type(pi) is int:                               # VBx/VBx.py:76-77 (np.int64 is *not* accepted there either)
        pi = np.ones(pi) / pi
    S = len(pi)
    if gamma is None:                                 # VBx/VBx.py:79-83: global np.random, drawn on the host
        gamma = np.random.gamma(alphaQInit, size=(T, S))
        gamma = gamma / gamma.sum(1, keepdims=True)
    assert (gamma.shape[1] == len(pi) and gamma.shape[0] == X.shape[0])   # VBx/VBx.py:85
    if plot:
        raise NotImplementedError('plot=True (matplotlib diagnostics, VBx/VBx.py:111-120) is not part of the GPU path')

    dev = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else None
    if dev is None:
        raise _lib.VbxError('VBx(): no CUDA device - vbx_b200 has no CPU fallback')
    if PRECISION == 'float64' or S > 64 or D > 128:
        # float64 kernels: any number of states / features, like the reference (the float32 kernels hold S <= 64, D <= 128)
        return _vbx_f64(X, Phi, loopProb, Fa, Fb, pi, gamma, maxIters, epsilon, ref, return_model, alpha, invL, dev)
    vb = _cached_batch(T, D, S, dev, True)
    vb.set_option('gemm', 1)      # single recording: float32 FFMA contractions (closest to the float64 reference);
    Sp = vb.S                     # the batched API defaults to tensor cores in split-precision 3xTF32
    fea_d = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
    phi_d = torch.from_numpy(np.ascontiguousarray(Phi, dtype=np.float32)).to(dev)
    g = torch.zeros((T, Sp), dtype=torch.float32, device=dev)
    g[:, :S] = torch.from_numpy(np.ascontiguousarray(gamma, dtype=np.float32)).to(dev)
    p = torch.zeros((1, Sp), dtype=torch.float32, device=dev)
    p[0, :S] = torch.from_numpy(np.ascontiguousarray(pi, dtype=np.float32)).to(dev)
    vb.prepare_scale(fea_d, phi_d)
    warm = alpha is not None and invL is not None    # VBx/VBx.py:94
    kw = {}
    if warm:
        a = torch.zeros((1, Sp, D), dtype=torch.float32, device=dev)
        il = torch.zeros((1, Sp, D), dtype=torch.float32, device=dev)
        a[0, :S] = torch.from_numpy(np.ascontiguousarray(alpha, dtype=np.float32)).to(dev)
        il[0, :S] = torch.from_numpy(np.ascontiguousarray(invL, dtype=np.float32)).to(dev)
        kw = dict(alpha=a, invL=il, warm_start=True)

    if ref is None:
        out = vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, maxIters=maxIters, epsilon=epsilon,
                     return_model=return_model, **kw)
        n = int(out['n_iters'][0].item())
        flags = int(out['flags'][0].item())
        Li = [[float(v)] for v in out['Li'][0, :n].cpu().numpy()]
    else:
        # the per-iteration DER / cross-entropy diagnostics (VBx/VBx.py:108-109) need gamma on the host
        # after every iteration: run one iteration per call, warm-starting nothing (the M-step reruns).
        Li, flags, out = [], 0, None
        for ii in range(maxIters):
            out = vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, maxIters=1, epsilon=epsilon,
                         return_model=return_model, **(kw if ii == 0 else {}))
            elbo = float(out['Li'][0, 0].item())
            gh = g[:, :S].double().cpu().numpy()
            Li.append([elbo, DER(gh, ref), DER(gh, ref, xentropy=True)])
            if ii > 0 and elbo - Li[-2][0] < epsilon:
                if elbo - Li[-2][0] < 0:
                    flags |= _lib.FLAG_ELBO_DECREASED
                break
    if flags & _lib.FLAG_ELBO_DECREASED:
        print('WARNING: Value of auxiliary function has decreased!')   # VBx/VBx.py:123-124
    gamma_out = g[:, :S].double().cpu().numpy()
    pi_out = p[0, :S].double().cpu().numpy()
    res = (gamma_out, pi_out, Li)
    if return_model:
        res = res + (out['alpha'][0, :S].double().cpu().numpy(), out['invL'][0, :S].double().cpu().numpy())
    return res


def _vbx_f64(X, Phi, loopProb, Fa, Fb, pi, gamma, maxIters, epsilon, ref, return_model, alpha, invL, dev):
    """Float64 evaluation through vbx_run_f64 (include/vbx_b200.h)."""
    T, D = X.shape
    S = len(pi)
    vb = _cached_batch(T, D, S, dev, False, f64_only=True)      # any S, any D: no padding (the reference has no limits)
    Sp = vb.S
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    fea_d, phi_d = f64(X), f64(Phi)
    g = torch.zeros((T, Sp), dtype=torch.float64, device=dev)
    g[:, :S] = f64(gamma)
    p = torch.zeros((1, Sp), dtype=torch.float64, device=dev)
    p[0, :S] = f64(pi)
    warm = alpha is not None and invL is not None
    kw = {}
    if warm:
        a = torch.zeros((1, Sp, D), dtype=torch.float64, device=dev)
        il = torch.zeros((1, Sp, D), dtype=torch.float64, device=dev)
        a[0, :S] = f64(alpha)
        il[0, :S] = f64(invL)
        kw = dict(alpha=a, invL=il, warm_start=True)
    flags, out = 0, None
    if ref is None:
        out = run_f64(vb, fea_d, phi_d, g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, maxIters=maxIters, epsilon=epsilon,
                      return_model=return_model, **kw)
        n = int(out['n_iters'][0].item())
        flags = int(out['flags'][0].item())
        Li = [[float(v)] for v in out['Li'][0, :n].cpu().numpy()]
    else:
        Li = []
        for ii in range(maxIters):     # one iteration per call so that DER() can look at gamma (VBx/VBx.py:108-109)
            out = run_f64(vb, fea_d, phi_d, g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, maxIters=1, epsilon=epsilon,
                          return_model=return_model, **(kw if ii == 0 else {}))
            elbo = float(out['Li'][0, 0].item())
            gh = g[:, :S].cpu().numpy()
            Li.append([elbo, DER(gh, ref), DER(gh, ref, xentropy=True)])
            if ii > 0 and elbo - Li[-2][0] < epsilon:
                if elbo - Li[-2][0] < 0:
                    flags |= _lib.FLAG_ELBO_DECREASED
                break
    if flags & _lib.FLAG_ELBO_DECREASED:
        print('WARNING: Value of auxiliary function has decreased!')   # VBx/VBx.py:123-124
    res = (g[:, :S].cpu().numpy(), p[0, :S].cpu().numpy(), Li)
    if return_model:
        res = res + (out['alpha'][0, :S].cpu().numpy(), out['invL'][0, :S].cpu().numpy())
    return res
