"""Per-recording Fa, Fb and loopP in the batched float32 VB-HMM (vbx_run_per_recording, VbxBatch.run with tensors).

The core property: on the same plan and options, a recording run with per-recording arrays gets bit-identical results to
a run of the whole batch with that recording's values as scalars.  Oracle bars as in test_parity_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import c_oracle as co
from vbx_b200 import synth

pytestmark = pytest.mark.gpu
TOL = 1e-4
VBX_ERR_ARG, VBX_ERR_STATE = -1, -3
# the recipe settings (Fa, Fb, loopP): example, AMI, DIHARD II, CALLHOME
RECIPES = [(0.3, 17.0, 0.99), (0.4, 64.0, 0.65), (0.2, 6.0, 0.35), (0.4, 17.0, 0.40)]


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def inputs(lens, n, seed):
    d = synth.make_batch(lens, R=128, S=n, seed=seed, dtype=np.float32)
    return d, d['gamma0'].astype(np.float32), np.full((len(lens), n), 1.0 / n, dtype=np.float32)


def hyper_arrays(settings, assign):
    return [cuda(np.array([settings[k][i] for k in assign]), torch.float64) for i in range(3)]


class Runner:
    """One planned batch; run() starts every call from the same inputs."""

    def __init__(self, lens, n, seed, fb_split=0, opts=None, make=None):
        from vbx_b200.batch import VbxBatch
        self.d, self.g0, self.pi0 = inputs(lens, n, seed)
        self.n = n
        self.vb = (make or VbxBatch)(lens, 128, n, device=dev(), fb_split=fb_split)
        for k, v in (opts or {}).items():
            self.vb.set_option(k, v)
        self.S = self.vb.S
        self.vb.prepare_scale(cuda(self.d['fea']), cuda(self.d['Phi']))

    def fresh(self):
        g = torch.zeros((self.vb.N, self.S), device=dev())
        g[:, :self.n] = cuda(self.g0)
        p = torch.zeros((self.vb.B, self.S), device=dev())
        p[:, :self.n] = cuda(self.pi0)
        return g, p

    def run(self, Fa, Fb, loopProb, warm=None, **kw):
        g, p = self.fresh()
        extra = {}
        if warm is not None:
            extra = dict(alpha=warm[0].clone(), invL=warm[1].clone(), warm_start=True)
        out = self.vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, **extra, **kw)
        torch.cuda.synchronize()
        res = {k: out[k].cpu().numpy() for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags')}
        for k in ('alpha', 'invL'):
            if k in out:
                res[k] = out[k].cpu().numpy()
        return res


def assert_entry_equal(a, b, rec, offsets):
    lo, hi = offsets[rec], offsets[rec + 1]
    assert np.array_equal(a['gamma'][lo:hi], b['gamma'][lo:hi]), rec
    assert np.array_equal(a['pi'][rec], b['pi'][rec]), rec
    assert np.array_equal(a['Li'][rec], b['Li'][rec], equal_nan=True), rec
    assert a['n_iters'][rec] == b['n_iters'][rec], rec
    assert a['flags'][rec] == b['flags'][rec], rec
    for k in ('alpha', 'invL'):
        if k in a:
            assert np.array_equal(a[k][rec], b[k][rec]), (k, rec)


def ragged(seed, B, tmax):
    lens = np.random.default_rng(seed).integers(1, tmax, size=B)
    lens[:3] = [1, 2, 513]
    return lens


LONG = np.array([5000, 4200, 300, 900, 4096, 17, 700, 6000])   # >= 4096 frames: the chunked scan on non-split plans
# id: (lengths, live states, fb_split, options)
CASES = {
    'lookahead-S16': (ragged(1, 24, 900), 16, 2, {}),
    'lookahead-S32-ffma': (ragged(2, 24, 900), 30, 2, dict(gemm=1)),
    'lookahead-S64': (ragged(3, 16, 700), 64, 2, {}),
    'classic-S16': (ragged(4, 24, 900), 13, 2, dict(fb_classic=1)),
    'classic-S64-ffma': (ragged(5, 16, 700), 50, 2, dict(fb_classic=1, gemm=1)),
    'split-S16': (ragged(6, 12, 900), 16, 1, {}),
    'split-S32-ffma': (ragged(7, 12, 900), 32, 1, dict(gemm=1)),
    'split-S64': (ragged(8, 12, 700), 64, 1, {}),
    'split-S128': (ragged(9, 8, 700), 100, 1, {}),
    'split-S128-ffma': (ragged(10, 8, 700), 128, 1, dict(gemm=1)),
    'chunked-S16': (LONG, 16, 2, {}),
    'chunked-S64-ffma': (LONG, 64, 2, dict(gemm=1)),
    'chunked-S32-classic': (LONG, 20, 2, dict(fb_classic=1)),
}


@pytest.mark.parametrize('epsilon', [-np.inf, 1e-6], ids=['fixed', 'eps1e-6'])
@pytest.mark.parametrize('case', list(CASES))
def test_bitwise_equal_to_scalar_runs(case, epsilon):
    lens, n, fb_split, opts = CASES[case]
    r = Runner(lens, n, seed=len(case), fb_split=fb_split, opts=opts)
    settings = RECIPES + [(0.3, 17.0, 0.0), (0.3, 17.0, 1.0)]
    assign = [b % len(settings) for b in range(len(lens))]      # every setting appears in every case
    kw = dict(maxIters=12, epsilon=epsilon, return_model=True)
    per = r.run(*hyper_arrays(settings, assign), **kw)
    for k, s in enumerate(settings):
        ref = r.run(*s, **kw)
        for b in np.nonzero(np.array(assign) == k)[0]:
            assert_entry_equal(per, ref, int(b), r.d['offsets'])


@pytest.mark.parametrize('case', ['lookahead-S16', 'split-S64', 'split-S128', 'chunked-S16'])
def test_warm_start_bitwise(case):
    lens, n, fb_split, opts = CASES[case]
    r = Runner(lens, n, seed=7, fb_split=fb_split, opts=opts)
    B, S = len(lens), r.S
    rng = np.random.default_rng(3)
    alpha = cuda(rng.normal(0, 0.3, (B, S, 128)))
    invL = cuda(rng.uniform(0.2, 1.0, (B, S, 128)))
    alpha[:, n:] = 0
    invL[:, n:] = 0
    assign = [b % len(RECIPES) for b in range(B)]
    kw = dict(maxIters=8, epsilon=1e-6, return_model=True, warm=(alpha, invL))
    per = r.run(*hyper_arrays(RECIPES, assign), **kw)
    for k, s in enumerate(RECIPES):
        ref = r.run(*s, **kw)
        for b in np.nonzero(np.array(assign) == k)[0]:
            assert_entry_equal(per, ref, int(b), r.d['offsets'])


@pytest.mark.parametrize('fb_split', [1, 2], ids=['split', 'fused'])
def test_mixed_settings_vs_oracle(fb_split):
    lens = ragged(21, 18, 800)
    n = 12
    settings = RECIPES + [(0.3, 17.0, 0.0), (0.3, 17.0, 1.0)]
    assign = [b % len(settings) for b in range(len(lens))]
    r = Runner(lens, n, seed=5, fb_split=fb_split)
    out = r.run(*hyper_arrays(settings, assign), maxIters=20, epsilon=1e-6)
    offs = r.d['offsets']
    for k, (Fa, Fb, lp) in enumerate(settings):
        ref = co.vbx_oracle_batch(r.d['fea'], r.d['Phi'], offs, r.g0.astype(np.float64), r.pi0.astype(np.float64),
                                  Fa, Fb, lp, 20, 1e-6)
        for b in np.nonzero(np.array(assign) == k)[0]:
            lo, hi = offs[b], offs[b + 1]
            assert out['n_iters'][b] == ref['n_iters'][b], (k, b)
            assert np.abs(out['gamma'][lo:hi, :n] - ref['gamma'][lo:hi]).max() <= TOL
            assert np.abs(out['pi'][b, :n] - ref['pi'][b]).max() <= TOL
            m = int(out['n_iters'][b])
            np.testing.assert_allclose(out['Li'][b, :m], ref['Li'][b, :m], rtol=TOL)


def test_graph_replay_reads_current_values():
    lens = ragged(31, 10, 600)
    n = 8
    r = Runner(lens, n, seed=9, fb_split=1, opts=dict(graph=1))
    direct = Runner(lens, n, seed=9, fb_split=1, opts=dict(graph=2))
    B = len(lens)
    bufs = r.vb.output_buffers(10)
    g, p = r.fresh()
    hyper = hyper_arrays(RECIPES, [b % 4 for b in range(B)])
    rng = np.random.default_rng(0)
    for call in range(4):      # call 0 runs directly, call 1 is captured, calls 2 and 3 replay the graph
        vals = [rng.uniform(0.1, 0.5, B), rng.uniform(2.0, 60.0, B), rng.uniform(0.0, 1.0, B)]
        for t, v in zip(hyper, vals):
            t.copy_(cuda(v, torch.float64))
        g0, p0 = r.fresh()
        g.copy_(g0)
        p.copy_(p0)
        out = r.vb.run(g, p, Fa=hyper[0], Fb=hyper[1], loopProb=hyper[2], maxIters=10, epsilon=1e-6, buffers=bufs)
        torch.cuda.synchronize()
        got = {k: out[k].cpu().numpy() for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags')}
        ref = direct.run(*[cuda(v, torch.float64) for v in vals], maxIters=10, epsilon=1e-6)
        for b in range(B):
            assert_entry_equal(got, ref, b, r.d['offsets'])


def test_partitioned_batch_equals_whole():
    from vbx_b200.parts import make_batch, PartitionedBatch
    lens = ragged(41, 16, 900)
    n = 16
    assign = [b % 4 for b in range(len(lens))]
    whole = Runner(lens, n, seed=11, fb_split=1)
    parts = Runner(lens, n, seed=11, fb_split=1, make=lambda *a, **k: make_batch(*a, parts=2, **k))
    assert isinstance(parts.vb, PartitionedBatch)
    kw = dict(maxIters=15, epsilon=1e-6, return_model=True)
    a = whole.run(*hyper_arrays(RECIPES, assign), **kw)
    b = parts.run(*hyper_arrays(RECIPES, assign), **kw)
    for rec in range(len(lens)):
        assert_entry_equal(a, b, rec, whole.d['offsets'])
    # a number and a tensor mixed: the number is broadcast
    c = parts.run(0.3, hyper_arrays(RECIPES, assign)[1], 0.99, **kw)
    d = whole.run(0.3, hyper_arrays(RECIPES, assign)[1], 0.99, **kw)
    for rec in range(len(lens)):
        assert_entry_equal(c, d, rec, whole.d['offsets'])


def _raw_run(vb, g, p, hyper, Li, it, fl, maxIters=10, epsilon=1e-4):
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    return vb.lib.vbx_run_per_recording(vb._h, P(vb.rho), P(getattr(vb, 'Phi', None)), P(g), P(p), P(vb.n_states), *(P(t) for t in hyper),
                                        maxIters, epsilon, None, None, 0, P(Li), P(it), P(fl), vb._stream())


@pytest.mark.parametrize('fb_split', [1, 2], ids=['split', 'fused'])
def test_bad_entry_is_flagged_and_isolated(fb_split):
    lens = ragged(51, 12, 800)
    n, B, bad = 10, 12, 5
    r = Runner(lens, n, seed=13, fb_split=fb_split)
    assign = [b % 4 for b in range(B)]
    good = hyper_arrays(RECIPES, assign)
    broken = [t.clone() for t in good]
    broken[1][bad] = 0.0
    outs = []
    for hyper in (good, broken):
        g, p = r.fresh()
        bufs = r.vb.output_buffers(10)
        assert _raw_run(r.vb, g, p, hyper, bufs['Li'], bufs['n_iters'], bufs['flags']) == 0
        torch.cuda.synchronize()
        outs.append(dict(gamma=g.cpu().numpy(), pi=p.cpu().numpy(), Li=bufs['Li'].cpu().numpy(),
                         n_iters=bufs['n_iters'].cpu().numpy(), flags=bufs['flags'].cpu().numpy()))
    assert outs[1]['flags'][bad] & 1
    assert not np.any(outs[0]['flags'] & 1)
    for b in range(B):
        if b != bad:
            assert_entry_equal(outs[0], outs[1], b, r.d['offsets'])


def test_abi_and_host_errors():
    from vbx_b200.batch import VbxBatch
    lens = np.array([300, 200, 500])
    r = Runner(lens, 8, seed=17, fb_split=1)
    g, p = r.fresh()
    bufs = r.vb.output_buffers(10)
    hyper = hyper_arrays(RECIPES, [0, 1, 2])
    for i in range(3):
        h = list(hyper)
        h[i] = None
        assert _raw_run(r.vb, g, p, h, bufs['Li'], bufs['n_iters'], bufs['flags']) == VBX_ERR_ARG
    fresh = VbxBatch(lens, 128, 8, device=dev())
    assert _raw_run(fresh, g, p, hyper, bufs['Li'], bufs['n_iters'], bufs['flags']) == VBX_ERR_STATE
    fresh.close()
    Fa, Fb, lp = hyper
    bad = [
        dict(Fa=Fa[:2]),                                                       # wrong shape
        dict(Fa=Fa.float()),                                                   # wrong dtype
        dict(Fa=torch.tensor([0.3, float('nan'), 0.3], dtype=torch.float64, device=dev())),
        dict(Fb=torch.tensor([17.0, 0.0, 6.0], dtype=torch.float64, device=dev())),
        dict(loopProb=torch.tensor([0.5, 1.5, 0.5], dtype=torch.float64, device=dev())),
        dict(loopProb=torch.tensor([-0.1, 0.5, 0.5], dtype=torch.float64, device=dev())),
    ]
    for kw in bad:
        args = dict(Fa=Fa, Fb=Fb, loopProb=lp)
        args.update(kw)
        with pytest.raises(ValueError):
            r.vb.run(g, p, maxIters=5, **args)
