"""Batched VB-HMM on the GPU: host-side driver over the C ABI (torch is only the owner of device
memory and streams).

A `VbxBatch` describes B independent recordings packed along the frame axis - the batched
equivalent of the reference's per-recording loop VBx/vbhmm.py:120-158, where every iteration calls
VBx() (VBx/VBx.py:27).  `run()` executes VBx/VBx.py:91-125 for all of them at once.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import VbxError


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class VbxBatch:
    """Plan + workspace for one packed ragged batch on one device."""

    def __init__(self, lengths, R, n_states, device=None, allocate=True, exact_stop=True, fb_split=0, S_pad=None, f64_only=False):
        """lengths: per-recording frame counts T_b; R: feature dim seen by VBx() (VBx/VBx.py:74);
        n_states: int or per-recording ints (the `pi`-as-int / len(pi) of VBx/VBx.py:76-77).
        exact_stop: reserve the buffers of the float64 finishing phase, so that run() with a finite epsilon applies the
        reference's stop rule (VBx/VBx.py:122-125) at float64 resolution; False = float32 only (smaller workspace).
        fb_split: 0 = auto, 1 = always, 2 = never run the forward / backward sweeps concurrently (include/vbx_b200.h).
        f64_only: plan for run_f64() only (vbx_plan_f64): any R and any number of states, no padding."""
        if not torch.cuda.is_available():
            raise VbxError('vbx_b200 needs a CUDA device (H100, sm_90); there is no CPU path')
        self.lib = _lib.load()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.index is None:       # a bare 'cuda' means the CURRENT device, not device 0
            self.device = torch.device('cuda', torch.cuda.current_device())
        lengths = np.asarray(lengths, dtype=np.int64).reshape(-1)
        self.B = int(lengths.shape[0])
        self.lengths = lengths
        self.offsets = np.zeros(self.B + 1, dtype=np.int64)
        np.cumsum(lengths, out=self.offsets[1:])
        self.N = int(self.offsets[-1])
        self.R = int(R)
        ns = np.asarray(n_states, dtype=np.int32).reshape(-1)
        if ns.size == 1:
            ns = np.full(self.B, int(ns[0]), dtype=np.int32)
        if ns.shape[0] != self.B:
            raise ValueError('n_states must be an int or one int per recording')
        self.n_states_host = ns
        self.f64_only = bool(f64_only)
        if self.f64_only:
            self.S = int(ns.max()) if self.B else 1
        else:
            self.S = _lib.padded_states(int(ns.max()) if self.B else 1) if S_pad is None else int(S_pad)
        self.uniform_states = bool(np.all(ns == self.S))
        self._h = ctypes.c_void_p()
        rc = self.lib.vbx_create(self.device.index, ctypes.byref(self._h))
        if rc != 0:
            raise VbxError(f'vbx_create failed ({rc}): no usable sm_90 device')
        self.exact_stop = bool(exact_stop)
        self._check(self.lib.vbx_set_option(self._h, b'exact_stop', int(self.exact_stop)))
        self._check(self.lib.vbx_set_option(self._h, b'fb_split', int(fb_split)))
        need = ctypes.c_size_t()
        if self.f64_only:
            self._check(self.lib.vbx_plan_f64(self._h, self.offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                              self.B, self.R, self.S))
            allocate = False
        else:
            self._check(self.lib.vbx_plan(self._h, self.offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                          self.B, self.R, self.S, ctypes.byref(need)))
        self.workspace_bytes = int(need.value)
        with torch.cuda.device(self.device):
            self.n_states = None if self.uniform_states else torch.from_numpy(ns).to(self.device)
        self.workspace = None
        self.rho = None
        if allocate:
            self.bind(torch.empty(self.workspace_bytes, dtype=torch.uint8, device=self.device))

    def bind(self, workspace):
        """Attach a caller-owned uint8 CUDA tensor of at least `workspace_bytes` as the scratch space."""
        self._check(self.lib.vbx_bind_workspace(self._h, _ptr(workspace), workspace.numel()))
        self.workspace = workspace

    # ---- plumbing -------------------------------------------------------------------------
    def _check(self, rc):
        if rc != 0:
            msg = self.lib.vbx_last_error(self._h)
            raise VbxError(f'vbx_b200 error {rc}: {msg.decode() if msg else "?"}')

    def close(self):
        if getattr(self, '_h', None) is not None and self._h.value:
            self.lib.vbx_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def attach_comm(self, group=None):
        """Hand torch.distributed's NCCL communicator of `group` (default: the world) to the library, which then
        all-reduces the ELBO trace itself (vbx_elbo_trace; SURVEY.md 8e).  No-op outside a multi-rank NCCL job."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) < 2:
            return False
        pg = (group or dist.distributed_c10d._get_default_group())._get_backend(self.device)
        if not hasattr(pg, '_comm_ptr'):
            raise VbxError('this torch build does not expose the NCCL communicator (ProcessGroupNCCL._comm_ptr)')
        try:
            ptr = pg._comm_ptr()
        except Exception:
            ptr = 0
        if not ptr:           # communicators are created lazily: force it with one collective, then ask again
            t = torch.zeros(1, device=self.device)
            dist.all_reduce(t, group=group)
            torch.cuda.current_stream(self.device).synchronize()
            ptr = pg._comm_ptr()
        nccl_lib = None
        try:
            import nvidia.nccl
            cand = os.path.join(list(nvidia.nccl.__path__)[0], 'lib', 'libnccl.so.2')
            nccl_lib = cand.encode() if os.path.exists(cand) else None
        except Exception:
            pass
        self._check(self.lib.vbx_attach_comm(self._h, ctypes.c_void_p(ptr), dist.get_world_size(group), nccl_lib))
        return True

    def elbo_trace(self, Li):
        """Li [B,maxIters] (float64 CUDA, NaN padded, as returned by run()) -> float64 CUDA tensor [2*maxIters]:
        per-iteration ELBO sums followed by the number of recordings that ran the iteration, summed over all ranks
        when a communicator is attached."""
        Li = Li.contiguous()
        n = int(Li.shape[1])
        out = torch.empty(2 * n, dtype=torch.float64, device=self.device)
        self._check(self.lib.vbx_elbo_trace(self._h, _ptr(Li), n, _ptr(out), self._stream()))
        return out

    def set_option(self, name, value):
        self._check(self.lib.vbx_set_option(self._h, name.encode(), int(value)))

    def hard_labels(self, gamma, second=False):
        """VBx/vbhmm.py:160-162 on the device: the most likely speaker per frame (int32 [N]); with second=True also
        the runner-up.  Only these labels need to leave the GPU, not gamma."""
        self._f32(gamma, (self.N, self.S), 'gamma', need_workspace=False)
        first = torch.empty(self.N, dtype=torch.int32, device=self.device)
        sec = torch.empty(self.N, dtype=torch.int32, device=self.device) if second else None
        self._check(self.lib.vbx_hard_labels(self._h, _ptr(gamma), _ptr(self.n_states), _ptr(first), _ptr(sec), self._stream()))
        return (first, sec) if second else first

    @property
    def launches(self):
        return int(self.lib.vbx_launch_count(self._h))

    def timings(self, reset=True):
        """{kernel class: (total device ms, launches)} accumulated while option 'timing' was on."""
        n = len(_lib.KERNEL_CLASSES)
        ms = (ctypes.c_double * n)()
        cnt = (ctypes.c_int64 * n)()
        self._check(self.lib.vbx_get_timings(self._h, ms, cnt, int(reset)))
        return {k: (ms[i], cnt[i]) for i, k in enumerate(_lib.KERNEL_CLASSES)}

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _f32(self, t, shape, name, need_workspace=True):
        if need_workspace and self.workspace is None:
            raise VbxError('no workspace bound (VbxBatch(..., allocate=False) needs bind())')
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise ValueError(f'{name}: expected a contiguous float32 CUDA tensor')
        if tuple(t.shape) != tuple(shape):
            raise ValueError(f'{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}')
        return t

    # ---- VBx/VBx.py:87-89 -----------------------------------------------------------------
    def prepare_scale(self, fea, Phi, out=None):
        """rho = fea * sqrt(Phi) (+ the ELBO constant G).  fea [N,R], Phi [R]."""
        self._f32(fea, (self.N, self.R), 'fea')
        self._f32(Phi, (self.R,), 'Phi')
        rho = torch.empty_like(fea) if out is None else self._f32(out, (self.N, self.R), 'out')
        self._check(self.lib.vbx_prepare_scale(self._h, _ptr(fea), _ptr(Phi), _ptr(rho), self._stream()))
        self.rho, self.Phi = rho, Phi
        return rho

    def prepare_project(self, X, V, Phi, out=None):
        """rho = X @ V for raw D-dim x-vectors (SURVEY.md 8d; VBx/vbhmm.py:129,153 folded with VBx/VBx.py:88-89)."""
        D = int(X.shape[1])
        self._f32(X, (self.N, D), 'X')
        self._f32(V, (D, self.R), 'V')
        self._f32(Phi, (self.R,), 'Phi')
        rho = torch.empty((self.N, self.R), dtype=torch.float32, device=self.device) if out is None \
            else self._f32(out, (self.N, self.R), 'out')
        self._check(self.lib.vbx_prepare_project(self._h, _ptr(X), D, _ptr(V), _ptr(Phi), _ptr(rho), self._stream()))
        self.rho, self.Phi = rho, Phi
        return rho

    def prepare_xvectors(self, x_raw, mean1, lda, mean2, plda_mu, plda_tr, plda_psi, out=None):
        """The real-data chain in front of VBx() on the tensor cores (VBx/vbhmm.py:125-129 and :153, with the scale
        of VBx/VBx.py:88-89): raw x-vectors [N,Dx] -> rho [N,128].  plda_tr / plda_psi are the diagonalised model
        (pipeline.diagonalise_plda).  Returns (rho, x_norm); x_norm is the l2-normalised LDA output [N,128]."""
        Dx = int(x_raw.shape[1])
        self._f32(x_raw, (self.N, Dx), 'x_raw')
        self._f32(mean1, (Dx,), 'mean1')
        self._f32(lda, (Dx, 128), 'lda')
        self._f32(mean2, (128,), 'mean2')
        self._f32(plda_mu, (128,), 'plda_mu')
        self._f32(plda_tr, (128, 128), 'plda_tr')
        self._f32(plda_psi, (128,), 'plda_psi')
        rho = torch.empty((self.N, self.R), dtype=torch.float32, device=self.device) if out is None \
            else self._f32(out, (self.N, self.R), 'out')
        x_norm = torch.empty((self.N, 128), dtype=torch.float32, device=self.device)
        self._check(self.lib.vbx_prepare_xvectors(self._h, _ptr(x_raw), Dx, _ptr(mean1), _ptr(lda), _ptr(mean2),
                                                  _ptr(plda_mu), _ptr(plda_tr), _ptr(plda_psi), _ptr(x_norm), _ptr(rho),
                                                  self._stream()))
        self.rho, self.Phi = rho, plda_psi
        return rho, x_norm

    def output_buffers(self, maxIters):
        """Preallocated outputs for run(buffers=...): with the same tensors every call the library sees identical
        arguments and replays the whole run as one CUDA graph (option 'graph')."""
        dev = self.device
        return dict(Li=torch.empty((self.B, max(int(maxIters), 1)), dtype=torch.float64, device=dev),
                    n_iters=torch.empty(self.B, dtype=torch.int32, device=dev),
                    flags=torch.empty(self.B, dtype=torch.int32, device=dev))

    # ---- VBx/VBx.py:91-125 ----------------------------------------------------------------
    def run(self, gamma, pi, Fa=1.0, Fb=1.0, loopProb=0.9, maxIters=10, epsilon=1e-4,
            alpha=None, invL=None, warm_start=False, return_model=False, buffers=None):
        """gamma [N,S] and pi [B,S] float32 CUDA tensors, updated IN PLACE (padded columns must be 0).
        Returns dict(gamma, pi, Li [B,maxIters] float64 (NaN padded), n_iters [B], flags [B][, alpha, invL]).
        buffers: optional dict(Li, n_iters, flags) of preallocated output tensors (see `output_buffers`)."""
        if self.rho is None:
            raise VbxError('call prepare_scale() or prepare_project() first')
        self._f32(gamma, (self.N, self.S), 'gamma')
        self._f32(pi, (self.B, self.S), 'pi')
        dev = self.device
        if return_model or warm_start:
            if alpha is None:
                alpha = torch.zeros((self.B, self.S, self.R), dtype=torch.float32, device=dev)
            if invL is None:
                invL = torch.zeros((self.B, self.S, self.R), dtype=torch.float32, device=dev)
            self._f32(alpha, (self.B, self.S, self.R), 'alpha')
            self._f32(invL, (self.B, self.S, self.R), 'invL')
        if buffers is not None:      # caller-owned outputs: identical pointers from call to call let the library replay the
            Li, n_iters, flags = buffers['Li'], buffers['n_iters'], buffers['flags']       # run as one CUDA graph
            assert Li.shape == (self.B, max(int(maxIters), 1)) and Li.dtype == torch.float64 and Li.is_contiguous()
        else:
            Li = torch.empty((self.B, max(int(maxIters), 1)), dtype=torch.float64, device=dev)
            n_iters = torch.empty(self.B, dtype=torch.int32, device=dev)
            flags = torch.empty(self.B, dtype=torch.int32, device=dev)
        self._check(self.lib.vbx_run(
            self._h, _ptr(self.rho), _ptr(self.Phi), _ptr(gamma), _ptr(pi), _ptr(self.n_states),
            float(Fa), float(Fb), float(loopProb), int(maxIters), float(epsilon),
            _ptr(alpha), _ptr(invL), int(bool(warm_start)), _ptr(Li), _ptr(n_iters), _ptr(flags),
            self._stream()))
        out = dict(gamma=gamma, pi=pi, Li=Li[:, :int(maxIters)], n_iters=n_iters, flags=flags)
        if return_model or warm_start:
            out.update(alpha=alpha, invL=invL)
        return out


def run_f64(vb, fea, Phi, gamma, pi, Fa=1.0, Fb=1.0, loopProb=0.9, maxIters=10, epsilon=1e-4, alpha=None, invL=None,
            warm_start=False, return_model=False):
    """Float64 evaluation of the EM loop on the planned batch `vb` (VbxBatch(..., allocate=False) is enough).
    fea [N,R], Phi [R], gamma [N,S], pi [B,S] float64 CUDA tensors (gamma, pi updated in place)."""
    dev = vb.device
    for t, shape, name in ((fea, (vb.N, vb.R), 'fea'), (Phi, (vb.R,), 'Phi'), (gamma, (vb.N, vb.S), 'gamma'), (pi, (vb.B, vb.S), 'pi')):
        if not (t.is_cuda and t.dtype == torch.float64 and t.is_contiguous() and tuple(t.shape) == shape):
            raise ValueError(f'{name}: expected a contiguous float64 CUDA tensor of shape {shape}')
    need = ctypes.c_size_t()
    vb._check(vb.lib.vbx_f64_workspace_bytes(vb._h, ctypes.byref(need)))
    ws = torch.empty(int(need.value), dtype=torch.uint8, device=dev)
    if return_model or warm_start:
        if alpha is None:
            alpha = torch.zeros((vb.B, vb.S, vb.R), dtype=torch.float64, device=dev)
        if invL is None:
            invL = torch.zeros((vb.B, vb.S, vb.R), dtype=torch.float64, device=dev)
    Li = torch.empty((vb.B, max(int(maxIters), 1)), dtype=torch.float64, device=dev)
    n_iters = torch.empty(vb.B, dtype=torch.int32, device=dev)
    flags = torch.empty(vb.B, dtype=torch.int32, device=dev)
    vb._check(vb.lib.vbx_run_f64(vb._h, _ptr(ws), ws.numel(), _ptr(fea), _ptr(Phi), _ptr(gamma), _ptr(pi), _ptr(vb.n_states),
                                 float(Fa), float(Fb), float(loopProb), int(maxIters), float(epsilon), _ptr(alpha), _ptr(invL),
                                 int(bool(warm_start)), _ptr(Li), _ptr(n_iters), _ptr(flags), vb._stream()))
    torch.cuda.current_stream(dev).synchronize()     # ws is released when this function returns
    out = dict(gamma=gamma, pi=pi, Li=Li[:, :int(maxIters)], n_iters=n_iters, flags=flags)
    if return_model or warm_start:
        out.update(alpha=alpha, invL=invL)
    return out


def vbx_batch(fea, Phi, lengths, gamma, pi=None, n_states=None, loopProb=0.9, Fa=1.0, Fb=1.0, maxIters=10,
              epsilon=1e-4, return_model=False, alpha=None, invL=None):
    """One-call batched VBx on CUDA tensors.

    fea [N,R] float32 (the reference's X per recording, packed), Phi [R], lengths [B] (host ints),
    gamma [N,S_user] initial responsibilities, pi [B,S_user] or None (uniform over the live states).
    Returns dict with gamma [N,S_user], pi [B,S_user], Li, n_iters, flags (CUDA tensors)."""
    N, S_user = gamma.shape
    ns = np.full(len(lengths), S_user, dtype=np.int32) if n_states is None else np.asarray(n_states, dtype=np.int32)
    vb = VbxBatch(lengths, fea.shape[1], ns, device=fea.device)
    S = vb.S
    g = torch.zeros((N, S), dtype=torch.float32, device=fea.device)
    g[:, :S_user] = gamma
    p = torch.zeros((vb.B, S), dtype=torch.float32, device=fea.device)
    if pi is None:
        nsd = torch.from_numpy(ns).to(fea.device)
        cols = torch.arange(S, device=fea.device)[None, :]
        p[:] = (cols < nsd[:, None]).float() / nsd[:, None].float()
    else:
        p[:, :S_user] = pi
    kw = {}
    warm = alpha is not None and invL is not None
    if warm:
        a = torch.zeros((vb.B, S, vb.R), dtype=torch.float32, device=fea.device)
        il = torch.zeros_like(a)
        a[:, :S_user] = alpha
        il[:, :S_user] = invL
        kw = dict(alpha=a, invL=il, warm_start=True)
    vb.prepare_scale(fea.contiguous(), Phi.contiguous())
    out = vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, maxIters=maxIters, epsilon=epsilon,
                 return_model=return_model, **kw)
    res = dict(gamma=out['gamma'][:, :S_user], pi=out['pi'][:, :S_user], Li=out['Li'], n_iters=out['n_iters'],
               flags=out['flags'], launches=vb.launches)
    if return_model or warm:
        res.update(alpha=out['alpha'][:, :S_user], invL=out['invL'][:, :S_user])
    torch.cuda.current_stream(fea.device).synchronize()
    vb.close()
    return res
