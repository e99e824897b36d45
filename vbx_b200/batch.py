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

    def g_sum(self):
        """The ELBO constant of every recording from the last prepare_*() call (a diagnostic, vbx_get_gsum):
        float64 CUDA tensor [B], G_b = sum_t -0.5 * (sum_r rho_tr^2 / Phi_r + R log 2pi)."""
        out = torch.empty(self.B, dtype=torch.float64, device=self.device)
        self._check(self.lib.vbx_get_gsum(self._h, _ptr(out), self._stream()))
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

    def hard_labels_keep(self, gamma, keep):
        """Labels under an upper bound on the speaker count (vbx_hard_labels_keep, DESIGN.md section 5.14): of recording b
        only the keep[b] live states of largest posterior mass compete.  keep: ints [B] (host sequence or int32 CUDA
        tensor), each >= 1; keep >= n_states gives hard_labels(second=True).  Returns (first, second) int32 [N] (second
        -1 where one state is kept) and the masses N_s, float64 [B, S]."""
        self._f32(gamma, (self.N, self.S), 'gamma', need_workspace=False)
        if isinstance(keep, torch.Tensor):
            if not (keep.is_cuda and keep.dtype == torch.int32 and tuple(keep.shape) == (self.B,)):
                raise ValueError(f'keep: expected an int32 CUDA tensor of shape ({self.B},)')
            keep = keep.contiguous()
        else:
            keep = torch.from_numpy(np.asarray(keep, dtype=np.int32).reshape(-1)).to(self.device)
            if tuple(keep.shape) != (self.B,):
                raise ValueError(f'keep: expected {self.B} counts, got {tuple(keep.shape)}')
        first = torch.empty(self.N, dtype=torch.int32, device=self.device)
        sec = torch.empty(self.N, dtype=torch.int32, device=self.device)
        mass = torch.empty((self.B, self.S), dtype=torch.float64, device=self.device)
        self._check(self.lib.vbx_hard_labels_keep(self._h, _ptr(gamma), _ptr(self.n_states), _ptr(keep), _ptr(first),
                                                  _ptr(sec), _ptr(mass), self._stream()))
        return first, sec, mass

    def init_turns(self, pack, smoothing, gamma, pi):
        """Initial responsibilities and priors of VB resegmentation (vbx_init_turns, DESIGN.md section 5.20) on this
        batch's plan: pack, a resegment.TurnPack of the batch's recordings (host arrays); smoothing, a number or one per
        recording.  gamma [N,S] and pi [B,S]: contiguous CUDA tensors, both float32 or both float64, overwritten."""
        dt = gamma.dtype
        for t, shape, name in ((gamma, (self.N, self.S), 'gamma'), (pi, (self.B, self.S), 'pi')):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dt and t.is_contiguous()
                    and dt in (torch.float32, torch.float64) and tuple(t.shape) == shape):
                raise ValueError(f'{name}: expected a contiguous float32 or float64 CUDA tensor of shape {shape}, '
                                 'gamma and pi of one type')
        if tuple(pack.seg.shape) != (self.N, 2) or len(pack.spk_off) != self.B + 1:
            raise ValueError(f'pack: expected the segments of {self.N} x-vectors and the speakers of {self.B} recordings')
        sm = np.broadcast_to(np.asarray(smoothing, dtype=np.float64), (self.B,)).copy()
        if not np.all(np.isfinite(sm)):
            raise ValueError('smoothing must be finite')
        dev = lambda a, t=np.int64: torch.from_numpy(np.ascontiguousarray(a, dtype=t)).to(self.device)
        arrays = [dev(a) for a in pack] + [dev(sm, np.float64)]
        self._check(self.lib.vbx_init_turns(self._h, *(_ptr(a) for a in arrays), _ptr(gamma), _ptr(pi),
                                            int(dt == torch.float64), self._stream()))

    def init_random(self, rec_keys, seeds, gamma, pi):
        """Random initial responsibilities and uniform priors (vbx_init_random, DESIGN.md section 5.22) on this batch's
        plan and live state counts: rec_keys and seeds, one integer in [0, 2^64) per recording (random_init.name_key and
        the restart's seed).  gamma [N,S] and pi [B,S]: contiguous CUDA tensors, both float32 or both float64,
        overwritten."""
        dt = gamma.dtype
        for t, shape, name in ((gamma, (self.N, self.S), 'gamma'), (pi, (self.B, self.S), 'pi')):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dt and t.is_contiguous()
                    and dt in (torch.float32, torch.float64) and tuple(t.shape) == shape):
                raise ValueError(f'{name}: expected a contiguous float32 or float64 CUDA tensor of shape {shape}, '
                                 'gamma and pi of one type')
        words = []
        for vals, name in ((rec_keys, 'rec_keys'), (seeds, 'seeds')):
            vals = list(vals)
            if len(vals) != self.B or not all(isinstance(v, (int, np.integer)) and 0 <= int(v) < 1 << 64 for v in vals):
                raise ValueError(f'{name}: expected {self.B} integers in [0, 2**64)')
            a = np.array([int(v) for v in vals], dtype=np.uint64).view(np.int64)     # the bits, as torch has no uint64
            words.append(torch.from_numpy(a).to(self.device))
        self._check(self.lib.vbx_init_random(self._h, _ptr(words[0]), _ptr(words[1]), _ptr(self.n_states), _ptr(gamma),
                                             _ptr(pi), int(dt == torch.float64), self._stream()))

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
    def _hyper(self, Fa, Fb, loopProb, arrays=False):
        """None when Fa, Fb and loopProb are all numbers (and not `arrays`), else the three as float64 CUDA tensors [B]
        (numbers broadcast), checked on the host: the library reads per-recording values on the device and cannot
        validate them, so the check copies them to the host and a per-recording run() waits for the device's current
        stream.  A broadcast number keeps its tensor between calls (stable pointers: option 'graph' can replay the run)."""
        vals = dict(Fa=Fa, Fb=Fb, loopProb=loopProb)
        if not arrays and not any(isinstance(v, torch.Tensor) for v in vals.values()):
            return None
        out = []
        for name, v in vals.items():
            if isinstance(v, torch.Tensor):
                if not (v.dtype == torch.float64 and v.device == self.device and tuple(v.shape) == (self.B,)):
                    raise ValueError(f'{name}: expected a float64 tensor of shape ({self.B},) on {self.device}, got '
                                     f'{v.dtype} {tuple(v.shape)} on {v.device}')
                t = v.contiguous()
            else:
                cache = self.__dict__.setdefault('_broadcast', {})
                if (name, float(v)) not in cache:
                    cache[(name, float(v))] = torch.full((self.B,), float(v), dtype=torch.float64, device=self.device)
                t = cache[(name, float(v))]
            out.append(t)
        Fa_t, Fb_t, lp_t = out
        host = torch.stack(out).cpu()
        if not bool(torch.isfinite(host).all()):
            raise ValueError('Fa, Fb and loopProb must be finite')
        if bool((host[1] == 0).any()):
            raise ValueError('Fb must be non-zero')
        if bool(((host[2] < 0) | (host[2] > 1)).any()):
            raise ValueError('loopProb must lie in [0, 1]')
        return Fa_t, Fb_t, lp_t

    def run(self, gamma, pi, Fa=1.0, Fb=1.0, loopProb=0.9, maxIters=10, epsilon=1e-4,
            alpha=None, invL=None, warm_start=False, return_model=False, buffers=None, prior=None):
        """gamma [N,S] and pi [B,S] float32 CUDA tensors, updated IN PLACE (padded columns must be 0).
        Fa, Fb, loopProb: numbers for the whole batch, or any of them a float64 CUDA tensor [B] of per-recording values
        (vbx_run_per_recording; numbers are then broadcast).  A recording gets bit-identical results either way.  The
        per-recording values are validated on the host, so such a call synchronises with the current stream.
        prior: None, or (n [B,S], F [B,S,R]) float64 CUDA tensors, the enrolment prior of each state (vbx_run_prior,
        DESIGN.md section 5.23): n_e x-vectors with feature sum F_e in fea units.  Checked on the host (synchronises).
        Returns dict(gamma, pi, Li [B,maxIters] float64 (NaN padded), n_iters [B], flags [B][, alpha, invL]).
        buffers: optional dict(Li, n_iters, flags) of preallocated output tensors (see `output_buffers`)."""
        if self.rho is None:
            raise VbxError('call prepare_scale() or prepare_project() first')
        self._f32(gamma, (self.N, self.S), 'gamma')
        self._f32(pi, (self.B, self.S), 'pi')
        if prior is not None:
            prior = check_prior(prior, self.B, self.S, self.R, self.device)
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
        hyper = self._hyper(Fa, Fb, loopProb, arrays=prior is not None)
        if prior is not None:
            self._check(self.lib.vbx_run_prior(
                self._h, _ptr(self.rho), _ptr(self.Phi), _ptr(gamma), _ptr(pi), _ptr(self.n_states),
                *(_ptr(t) for t in hyper), int(maxIters), float(epsilon),
                _ptr(alpha), _ptr(invL), int(bool(warm_start)), _ptr(Li), _ptr(n_iters), _ptr(flags),
                _ptr(prior[0]), _ptr(prior[1]), self._stream()))
        elif hyper is None:
            self._check(self.lib.vbx_run(
                self._h, _ptr(self.rho), _ptr(self.Phi), _ptr(gamma), _ptr(pi), _ptr(self.n_states),
                float(Fa), float(Fb), float(loopProb), int(maxIters), float(epsilon),
                _ptr(alpha), _ptr(invL), int(bool(warm_start)), _ptr(Li), _ptr(n_iters), _ptr(flags),
                self._stream()))
        else:
            self._check(self.lib.vbx_run_per_recording(
                self._h, _ptr(self.rho), _ptr(self.Phi), _ptr(gamma), _ptr(pi), _ptr(self.n_states),
                *(_ptr(t) for t in hyper), int(maxIters), float(epsilon),
                _ptr(alpha), _ptr(invL), int(bool(warm_start)), _ptr(Li), _ptr(n_iters), _ptr(flags),
                self._stream()))
        out = dict(gamma=gamma, pi=pi, Li=Li[:, :int(maxIters)], n_iters=n_iters, flags=flags)
        if return_model or warm_start:
            out.update(alpha=alpha, invL=invL)
        return out

    # ---- streaming diarization, DESIGN.md section 5.25 ----------------------------------------------------------------
    def _stream_args(self, state, slots, blk_fea, blk_off):
        """The per-stream arrays of a push on this batch's plan (the window plan: recording b is stream slots[b]'s
        window), checked on the host: slots distinct and in range, blk_fea [*, R] float32 finite, blk_off [B+1] with
        blocks of >= 1 rows, every window length min(C, count) + h.  Returns (slot, blk_off, win_off) CUDA tensors."""
        if not isinstance(state, StreamState) or state.device != self.device or state.R != self.R:
            raise ValueError(f'state: expected a StreamState with R = {self.R} on {self.device}')
        sl = np.asarray(slots, dtype=np.int64).reshape(-1)
        if len(sl) != self.B or len(np.unique(sl)) != self.B or (self.B and (sl.min() < 0 or sl.max() >= state.slots)):
            raise ValueError(f'slots: expected {self.B} distinct slots in [0, {state.slots})')
        bo = np.asarray(blk_off, dtype=np.int64).reshape(-1)
        if len(bo) != self.B + 1 or bo[0] != 0 or np.any(np.diff(bo) < 1):
            raise ValueError(f'blk_off: expected {self.B + 1} increasing offsets from 0, one block of >= 1 rows per stream')
        if not (isinstance(blk_fea, torch.Tensor) and blk_fea.is_cuda and blk_fea.device == self.device
                and blk_fea.dtype == torch.float32 and blk_fea.is_contiguous() and tuple(blk_fea.shape) == (int(bo[-1]), self.R)):
            raise ValueError(f'blk_fea: expected a contiguous float32 tensor of shape ({int(bo[-1])}, {self.R}) on {self.device}')
        if not bool(torch.isfinite(blk_fea).all()):
            raise ValueError('blk_fea must be finite')
        slot_d = torch.from_numpy(sl.astype(np.int32)).to(self.device)
        count = state.count[slot_d.long()].cpu().numpy()
        if not np.array_equal(self.lengths, np.minimum(count, state.C) + np.diff(bo)):
            raise ValueError('the plan\'s lengths must be min(C, count) + h for every stream (the window of the push)')
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(self.device)
        return slot_d, dev(bo), dev(self.offsets)

    def _stream_out(self, out, specs):
        """Caller-owned outputs of the stream entries, checked (contiguous tensors of the given (shape, dtype) on this
        batch's device); out None allocates them."""
        if out is None:
            return [torch.empty(shape, dtype=dt, device=self.device) for shape, dt in specs]
        if len(out) != len(specs):
            raise ValueError(f'out: expected {len(specs)} tensors')
        for t, (shape, dt) in zip(out, specs):
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == dt and t.is_contiguous()
                    and tuple(t.shape) == tuple(shape)):
                raise ValueError(f'out: expected a contiguous {dt} tensor of shape {tuple(shape)} on {self.device}')
        return list(out)

    def _timed(self, events, call):
        """call() with the CUDA events pair `events` (None: no timing) recorded right around it on the current stream,
        so that their interval holds the kernel and not the host checks before it."""
        if events is not None:
            events[0].record()
        self._check(call())
        if events is not None:
            events[1].record()

    def stream_window(self, state, slots, blk_fea, blk_off, blk_lab, n_clusters, smoothing, out=None, events=None):
        """The window of a push on this batch's plan (vbx_stream_window): stream slots[b] (a StreamState slot) takes the
        block rows blk_off[b] .. blk_off[b+1]-1 of blk_fea [*, R] float32 (projected x-vectors) with its block AHC
        labels blk_lab (int32 CUDA [*], 0 .. c-1) and c = n_clusters[b] (host ints; K + c <= min(S, S_max), c = 0 only
        when K = S_max).  Everything is checked on the host first (synchronises).  Returns (fea [N,R] float32,
        gamma0 [N,S], pi0 [B,S] float32, n_states int32 [B], (prior_n [B,S], prior_F [B,S,R]) float64): the inputs of
        prepare_scale and run(prior=).  out: None, or those six tensors to write into; events: None, or two CUDA events
        recorded right before and after the kernel (a measurement aid)."""
        slot_d, bo_d, wo_d = self._stream_args(state, slots, blk_fea, blk_off)
        c = np.asarray(n_clusters, dtype=np.int64).reshape(-1)
        sm = float(smoothing)
        if not np.isfinite(sm):
            raise ValueError('smoothing must be finite')
        if len(c) != self.B or np.any(c < 0):
            raise ValueError(f'n_clusters: expected {self.B} counts >= 0')
        K = state.K[slot_d.long()].cpu().numpy().astype(np.int64)
        if np.any(K + c > min(self.S, state.S_max)) or np.any((c == 0) & (K != state.S_max)):
            raise ValueError(f'n_clusters: K + c must lie in [1, {min(self.S, state.S_max)}], and c = 0 only at S_max speakers')
        if not (isinstance(blk_lab, torch.Tensor) and blk_lab.device == self.device and blk_lab.dtype == torch.int32
                and tuple(blk_lab.shape) == (int(blk_fea.shape[0]),)):
            raise ValueError(f'blk_lab: expected an int32 tensor of shape ({int(blk_fea.shape[0])},) on {self.device}')
        blk_lab = blk_lab.contiguous()
        c_d = torch.from_numpy(c.astype(np.int32)).to(self.device)
        per_row = torch.repeat_interleave(c_d, torch.diff(bo_d))
        if bool(((per_row > 0) & ((blk_lab < 0) | (blk_lab >= per_row))).any()):
            raise ValueError('blk_lab: every label must lie in [0, c) of its stream (not read where c = 0)')
        f32, f64 = torch.float32, torch.float64
        fea, gamma, pi, ns, pn, pF = self._stream_out(out, [((self.N, self.R), f32), ((self.N, self.S), f32),
                                                            ((self.B, self.S), f32), ((self.B,), torch.int32),
                                                            ((self.B, self.S), f64), ((self.B, self.S, self.R), f64)])
        self._timed(events, lambda: self.lib.vbx_stream_window(
            self._h, self.B, state.C, self.R, state.S_max, self.S, _ptr(slot_d), _ptr(bo_d), _ptr(wo_d), _ptr(blk_lab),
            _ptr(c_d), _ptr(blk_fea), sm, _ptr(state.ctx_fea), _ptr(state.ctx_lab), _ptr(state.count), _ptr(state.K),
            _ptr(state.n_hist), _ptr(state.F_hist), _ptr(fea), _ptr(gamma), _ptr(pi), _ptr(ns), _ptr(pn), _ptr(pF),
            self._stream()))
        return fea, gamma, pi, ns, (pn, pF)

    def stream_commit(self, state, slots, blk_fea, blk_off, first, out=None, events=None):
        """Fold a push's result into the streams' state (vbx_stream_commit): first (int32 CUDA [N]) holds the window's
        first labels, as hard_labels leaves them; slots, blk_fea and blk_off as for stream_window.  Checked on the host
        first (synchronises).  Returns the blocks' final labels, int32 CUDA [blk_off[-1]] (written into out, when given);
        state is updated in place.  events: as for stream_window."""
        slot_d, bo_d, wo_d = self._stream_args(state, slots, blk_fea, blk_off)
        if not (isinstance(first, torch.Tensor) and first.device == self.device and first.dtype == torch.int32
                and tuple(first.shape) == (self.N,)):
            raise ValueError(f'first: expected an int32 tensor of shape ({self.N},) on {self.device}')
        first = first.contiguous()
        if self.N and bool(((first < 0) | (first >= min(self.S, state.S_max))).any()):
            raise ValueError(f'first: every label must lie in [0, {min(self.S, state.S_max)})')
        labels, = self._stream_out(None if out is None else [out], [((int(blk_fea.shape[0]),), torch.int32)])
        self._timed(events, lambda: self.lib.vbx_stream_commit(
            self._h, self.B, state.C, self.R, state.S_max, _ptr(slot_d), _ptr(bo_d), _ptr(wo_d), _ptr(blk_fea),
            _ptr(first), _ptr(state.ctx_fea), _ptr(state.ctx_lab), _ptr(state.count), _ptr(state.K), _ptr(state.n_hist),
            _ptr(state.F_hist), _ptr(labels), self._stream()))
        return labels


class StreamState:
    """The device-resident state of `slots` live streams (include/vbx_b200.h vbx_stream_window, DESIGN.md section
    5.25): a ring of the last C projected x-vectors of each stream and their final labels, its x-vector count, its
    speaker count K and the float64 history statistics n_hist [slots, S_max], F_hist [slots, S_max, R] of the x-vectors
    that have left the ring.  Every slot starts empty."""

    def __init__(self, slots, C, R, S_max, device):
        self.C, self.R, self.S_max = int(C), int(R), int(S_max)
        self.device = torch.device(device)
        self.slots = 0
        self.ctx_fea = torch.zeros((0, max(self.C, 1), self.R), dtype=torch.float32, device=self.device)
        self.ctx_lab = torch.zeros((0, max(self.C, 1)), dtype=torch.int32, device=self.device)
        self.count = torch.zeros(0, dtype=torch.int64, device=self.device)
        self.K = torch.zeros(0, dtype=torch.int32, device=self.device)
        self.n_hist = torch.zeros((0, self.S_max), dtype=torch.float64, device=self.device)
        self.F_hist = torch.zeros((0, self.S_max, self.R), dtype=torch.float64, device=self.device)
        self.grow(slots)

    _FIELDS = ('ctx_fea', 'ctx_lab', 'count', 'K', 'n_hist', 'F_hist')

    def grow(self, slots):
        """At least `slots` slots, the existing ones kept (a larger allocation and one copy per array)."""
        if slots <= self.slots:
            return
        for name in self._FIELDS:
            old = getattr(self, name)
            new = torch.zeros((int(slots),) + tuple(old.shape[1:]), dtype=old.dtype, device=self.device)
            new[:self.slots] = old
            setattr(self, name, new)
        self.slots = int(slots)

    def reset(self, slot):
        """Empty slot `slot` for a new stream."""
        for name in self._FIELDS:
            getattr(self, name)[int(slot)].zero_()


def check_prior(prior, B, S, R, device):
    """The enrolment prior of run() / run_f64() checked on the host (ValueError): a pair (n [B,S], F [B,S,R]) of float64
    tensors on `device`, finite, n >= 0.  Returns the pair contiguous."""
    if not (isinstance(prior, (tuple, list)) and len(prior) == 2):
        raise ValueError('prior must be a pair (n [B,S], F [B,S,R]) of float64 CUDA tensors')
    out = []
    for t, shape, name in ((prior[0], (B, S), 'prior n'), (prior[1], (B, S, R), 'prior F')):
        if not (isinstance(t, torch.Tensor) and t.dtype == torch.float64 and t.device == torch.device(device)
                and tuple(t.shape) == shape):
            got = f'{t.dtype} {tuple(t.shape)} on {t.device}' if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f'{name}: expected a float64 tensor of shape {shape} on {device}, got {got}')
        out.append(t.contiguous())
    n, F = out
    if not (bool(torch.isfinite(n).all()) and bool(torch.isfinite(F).all())):
        raise ValueError('prior n and F must be finite')
    if bool((n < 0).any()):
        raise ValueError('prior n (enrolment x-vector counts) must be >= 0')
    return n, F


def run_f64(vb, fea, Phi, gamma, pi, Fa=1.0, Fb=1.0, loopProb=0.9, maxIters=10, epsilon=1e-4, alpha=None, invL=None,
            warm_start=False, return_model=False, prior=None):
    """Float64 evaluation of the EM loop on the planned batch `vb` (VbxBatch(..., allocate=False) is enough).
    fea [N,R], Phi [R], gamma [N,S], pi [B,S] float64 CUDA tensors (gamma, pi updated in place).  prior: None, or
    (n [B,S], F [B,S,R]) float64 CUDA tensors, the enrolment prior of VbxBatch.run (vbx_run_f64_prior)."""
    dev = vb.device
    for t, shape, name in ((fea, (vb.N, vb.R), 'fea'), (Phi, (vb.R,), 'Phi'), (gamma, (vb.N, vb.S), 'gamma'), (pi, (vb.B, vb.S), 'pi')):
        if not (t.is_cuda and t.dtype == torch.float64 and t.is_contiguous() and tuple(t.shape) == shape):
            raise ValueError(f'{name}: expected a contiguous float64 CUDA tensor of shape {shape}')
    if prior is not None:
        prior = check_prior(prior, vb.B, vb.S, vb.R, dev)
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
    args = (vb._h, _ptr(ws), ws.numel(), _ptr(fea), _ptr(Phi), _ptr(gamma), _ptr(pi), _ptr(vb.n_states), float(Fa), float(Fb),
            float(loopProb), int(maxIters), float(epsilon), _ptr(alpha), _ptr(invL), int(bool(warm_start)), _ptr(Li),
            _ptr(n_iters), _ptr(flags))
    if prior is None:
        vb._check(vb.lib.vbx_run_f64(*args, vb._stream()))
    else:
        vb._check(vb.lib.vbx_run_f64_prior(*args, _ptr(prior[0]), _ptr(prior[1]), vb._stream()))
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
