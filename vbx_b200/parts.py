"""A large batch as two (or more) independently scheduled parts.

Recordings are independent, so the EM loop of one half of a batch never waits for the other half.  Run as ONE sequence of
kernels, the latency-bound forward-backward sweep (a tenth of the warps the GPU can hold, half of the DRAM bandwidth)
alternates with the bandwidth-bound contractions and neither fills the machine.  Here every part is its own planned batch
on its own CUDA stream: while one part walks its recordings sequentially, the other streams rho through the tensor cores.
The parts are contiguous ranges of recordings of about equal frame counts; all tensors handed in stay whole (parts work on
row ranges of them), results are bit-identical to the unpartitioned batch (a recording's arithmetic never depends on its
neighbours).  Host-side orchestration only: streams and events, no new kernels.
"""
import numpy as np
import torch

from .batch import VbxBatch


def auto_parts(lengths, n_states_max):
    """2 for batches that are large enough for both halves to keep the GPU's bandwidth busy, else 1."""
    lengths = np.asarray(lengths)
    return 2 if (len(lengths) >= 2048 and int(lengths.sum()) >= 2_000_000 and int(lengths.max()) < 4096) else 1


def make_batch(lengths, R, n_states, device=None, parts=0, **kw):
    """VbxBatch, or a PartitionedBatch when `parts` (0 = auto) says so."""
    ns = np.asarray(n_states).reshape(-1)
    if parts == 0:
        parts = auto_parts(lengths, int(ns.max()))
    if parts <= 1 or len(lengths) < 2 * parts:
        return VbxBatch(lengths, R, n_states, device=device, **kw)
    return PartitionedBatch(lengths, R, n_states, device=device, parts=parts, **kw)


class PartitionedBatch:
    """Same calls as VbxBatch (prepare_*, run, hard_labels, elbo_trace, ...) over `parts` sub-batches on separate streams."""

    def __init__(self, lengths, R, n_states, device=None, parts=2, exact_stop=True, fb_split=0):
        lengths = np.asarray(lengths, dtype=np.int64).reshape(-1)
        # the whole batch, planned but without workspace: batch-wide calls (ELBO trace + collective, labels)
        self.whole = VbxBatch(lengths, R, n_states, device=device, allocate=False, exact_stop=False, fb_split=fb_split)
        w = self.whole
        self.device, self.B, self.N, self.R, self.S, self.lengths = w.device, w.B, w.N, w.R, w.S, lengths
        csum = np.cumsum(lengths)
        cuts = [0]
        for k in range(1, parts):
            cuts.append(int(np.searchsorted(csum, self.N * k / parts, side='left')) + 1)
        cuts.append(self.B)
        cuts = sorted(set(min(max(c, 0), self.B) for c in cuts))
        self.rec_bounds = cuts
        offs = np.concatenate([[0], csum])
        self.frame_bounds = [int(offs[c]) for c in cuts]
        ns = w.n_states_host
        self.children = [VbxBatch(lengths[a:b], R, ns[a:b], device=self.device, exact_stop=exact_stop, fb_split=fb_split, S_pad=self.S)
                         for a, b in zip(cuts[:-1], cuts[1:])]
        self.streams = [None] + [torch.cuda.Stream(device=self.device) for _ in self.children[1:]]   # part 0: the caller's stream
        self.workspace_bytes = sum(c.workspace_bytes for c in self.children)
        self.rho = None
        self._n_states = w.n_states

    # ---- attributes VbxBatch users touch --------------------------------------------------------
    @property
    def n_states(self):
        return self._n_states

    @n_states.setter
    def n_states(self, t):
        self._n_states = t
        self.whole.n_states = t
        for c, a, b in zip(self.children, self.rec_bounds[:-1], self.rec_bounds[1:]):
            c.n_states = None if t is None else t[a:b]

    @property
    def workspace(self):
        return self.children[0].workspace

    @property
    def launches(self):
        return self.whole.launches + sum(c.launches for c in self.children)

    def set_option(self, name, value):
        for c in self.children:
            c.set_option(name, value)

    def timings(self, reset=True):
        """Summed over the parts; with the parts overlapping on the device the classes add up to MORE than the step time."""
        out = {}
        for c in self.children:
            for k, (ms, n) in c.timings(reset=reset).items():
                a = out.get(k, (0.0, 0))
                out[k] = (a[0] + ms, a[1] + n)
        return out

    def close(self):
        for c in self.children:
            c.close()
        self.whole.close()

    # ---- fork / join ----------------------------------------------------------------------------
    def _each(self, fn):
        """fn(child, frame slice, recording slice) for every part on its stream; the caller's stream continues after all."""
        main = torch.cuda.current_stream(self.device)
        fork = torch.cuda.Event()
        fork.record(main)
        results, done = [], []
        for i, (c, st) in enumerate(zip(self.children, self.streams)):
            fs = slice(self.frame_bounds[i], self.frame_bounds[i + 1])
            rs = slice(self.rec_bounds[i], self.rec_bounds[i + 1])
            if st is None:
                results.append(fn(c, fs, rs))
            else:
                st.wait_event(fork)
                with torch.cuda.stream(st):
                    results.append(fn(c, fs, rs))
                    ev = torch.cuda.Event()
                    ev.record(st)
                done.append(ev)
        for ev in done:
            main.wait_event(ev)
        return results

    def _keep(self, t, main):
        if isinstance(t, torch.Tensor):
            t.record_stream(main)       # allocated on a part's stream, consumed on the caller's
        return t

    # ---- VBx/VBx.py:87-89 and the caller-side front ends -----------------------------------------
    def prepare_scale(self, fea, Phi, out=None):
        rho = torch.empty_like(fea) if out is None else out
        self._each(lambda c, fs, rs: c.prepare_scale(fea[fs], Phi, out=rho[fs]))
        self.rho, self.Phi = rho, Phi
        return rho

    def prepare_project(self, X, V, Phi, out=None):
        rho = torch.empty((self.N, self.R), dtype=torch.float32, device=self.device) if out is None else out
        self._each(lambda c, fs, rs: c.prepare_project(X[fs], V, Phi, out=rho[fs]))
        self.rho, self.Phi = rho, Phi
        return rho

    def prepare_xvectors(self, x_raw, mean1, lda, mean2, plda_mu, plda_tr, plda_psi, out=None):
        rho = torch.empty((self.N, self.R), dtype=torch.float32, device=self.device) if out is None else out
        main = torch.cuda.current_stream(self.device)
        xn = self._each(lambda c, fs, rs: c.prepare_xvectors(x_raw[fs], mean1, lda, mean2, plda_mu, plda_tr, plda_psi, out=rho[fs])[1])
        self.rho, self.Phi = rho, plda_psi
        return rho, torch.cat([self._keep(t, main) for t in xn])

    # ---- VBx/VBx.py:91-125 --------------------------------------------------------------------
    def output_buffers(self, maxIters):
        return None               # the parts allocate their own outputs

    def run(self, gamma, pi, alpha=None, invL=None, buffers=None, prior=None, **kw):
        main = torch.cuda.current_stream(self.device)
        if prior is not None:      # checked whole, so that a bad prior is refused before any part launches
            from .batch import check_prior
            prior = check_prior(prior, self.B, self.S, self.R, self.device)

        def one(c, fs, rs):
            extra = {}
            if prior is not None:
                extra['prior'] = (prior[0][rs], prior[1][rs])
            if alpha is not None:
                extra['alpha'] = alpha[rs]
            if invL is not None:
                extra['invL'] = invL[rs]
            for k in ('Fa', 'Fb', 'loopProb'):      # per-recording values: each part takes its recordings' rows
                if isinstance(kw.get(k), torch.Tensor):
                    extra[k] = kw[k][rs]
            return c.run(gamma[fs], pi[rs], **{**kw, **extra})

        outs = self._each(one)
        res = dict(gamma=gamma, pi=pi)
        for k in ('Li', 'n_iters', 'flags', 'alpha', 'invL'):
            if k in outs[0]:
                res[k] = torch.cat([self._keep(o[k], main) for o in outs])
        return res

    def hard_labels(self, gamma, second=False):
        self.whole.n_states = self._n_states
        return self.whole.hard_labels(gamma, second=second)

    def hard_labels_keep(self, gamma, keep):
        self.whole.n_states = self._n_states
        return self.whole.hard_labels_keep(gamma, keep)

    def init_turns(self, pack, smoothing, gamma, pi):
        return self.whole.init_turns(pack, smoothing, gamma, pi)

    def init_random(self, rec_keys, seeds, gamma, pi):
        self.whole.n_states = self._n_states
        return self.whole.init_random(rec_keys, seeds, gamma, pi)

    # ---- multi-GPU: the batch-wide ELBO trace and its collective live in the whole-batch handle ----
    def attach_comm(self, group=None):
        return self.whole.attach_comm(group)

    def elbo_trace(self, Li):
        return self.whole.elbo_trace(Li)
