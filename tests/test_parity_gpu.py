"""GPU parity: the CUDA path (through the C ABI) against the reference goldens and the CPU oracle.

Tolerances (north_star: gamma/pi/Li within 1e-4 relative in float32; SURVEY.md 8c):
  gamma, pi : max|delta| <= 1e-4 * max|ref|      ELBO : |delta| <= 1e-4 * |ELBO| per iteration
The ELBO of a *transient* iteration amplifies rounding differences (EM far from its fixed point), so on top of the
official per-iteration bound the typical (median) relative ELBO error must be below 1e-6.
"""
import os

import numpy as np
import pytest
import torch

from oracle import c_oracle as co
from vbx_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
G_TOL, PI_TOL, L_RTOL = 1e-4, 1e-4, 1e-4


def check_elbo(got, want, median_tol=3e-6):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    np.testing.assert_allclose(got, want, rtol=L_RTOL)
    rel = np.abs(got - want) / np.abs(want)
    assert np.nanmedian(rel) < median_tol, np.nanmedian(rel)


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def load_cases():
    z = np.load(os.path.join(GOLD, 'synthetic_cases.npz'))
    cases = {}
    for k in z.files:
        tag, name = k.split('/')
        cases.setdefault(tag, {})[name] = z[k]
    return cases


CASES = load_cases()


def run_gpu(fea, Phi, lengths, gamma0, pi0=None, n_states=None, spl=0, gemm=0, fb_classic=0, exact_stop=True, fb_split=0, **kw):
    from vbx_b200.batch import VbxBatch
    import vbx_b200._lib as L
    lengths = np.asarray(lengths)
    S_user = gamma0.shape[1]
    ns = np.full(len(lengths), S_user, dtype=np.int32) if n_states is None else np.asarray(n_states, dtype=np.int32)
    if spl or fb_classic:
        fb_split = 2                  # these knobs belong to the fused sweep
    vb = VbxBatch(lengths, fea.shape[1], ns, device=dev(), exact_stop=exact_stop, fb_split=fb_split)
    vb.workspace.fill_(0xFF)       # poison (NaN in float32 and float64): nothing may be read before it is written
    if spl:
        vb.set_option('fb_states_per_lane', spl)
    vb.set_option('gemm', gemm)
    vb.set_option('fb_classic', fb_classic)
    S = vb.S
    g = torch.zeros((fea.shape[0], S), device=dev())
    g[:, :S_user] = cuda(gamma0)
    p = torch.zeros((len(lengths), S), device=dev())
    if pi0 is None:
        for b in range(len(lengths)):
            p[b, :ns[b]] = 1.0 / ns[b]
    else:
        p[:, :S_user] = cuda(np.broadcast_to(pi0, (len(lengths), S_user)))
    vb.prepare_scale(cuda(fea), cuda(Phi))
    extra = {}
    if 'alpha0' in kw:
        a = torch.zeros((len(lengths), S, fea.shape[1]), device=dev())
        il = torch.zeros_like(a)
        a[:, :S_user] = cuda(kw.pop('alpha0'))
        il[:, :S_user] = cuda(kw.pop('invL0'))
        extra = dict(alpha=a, invL=il, warm_start=True)
    out = vb.run(g, p, return_model=True, **extra, **kw)
    torch.cuda.synchronize()
    res = dict(gamma=g[:, :S_user].double().cpu().numpy(), pi=p[:, :S_user].double().cpu().numpy(),
               Li=out['Li'].cpu().numpy(), n_iters=out['n_iters'].cpu().numpy(), flags=out['flags'].cpu().numpy(),
               alpha=out['alpha'][:, :S_user].double().cpu().numpy(), invL=out['invL'][:, :S_user].double().cpu().numpy(),
               gamma_pad=g[:, S_user:].cpu().numpy())
    vb.close()
    return res


@pytest.mark.parametrize('fb', [2, 1], ids=['fused', 'split'])
@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('tag', sorted(CASES))
def test_reference_goldens(tag, gemm, fb):
    """Every reference-generated case through both contraction modes - tensor cores in split-precision 3xTF32 (the
    batch default) and float32 FFMA (the default of the drop-in VBx(), tighter) - and both forward-backward schedules:
    the fused sweep (large batches) and forward / backward on separate warps + combine pass (small batches)."""
    c = CASES[tag]
    T = c['fea'].shape[0]
    kw = dict(Fa=float(c['Fa']), Fb=float(c['Fb']), loopProb=float(c['loopProb']), maxIters=int(c['maxIters']),
              epsilon=float(c['epsilon']))
    if 'alpha0' in c:
        kw.update(alpha0=c['alpha0'][None], invL0=c['invL0'][None])
    out = run_gpu(c['fea'], c['Phi'], [T], c['gamma0'], pi0=c['pi0'], gemm=gemm, fb_split=fb, **kw)
    n = int(out['n_iters'][0])
    # identical iteration counts in both modes: the stop test of VBx/VBx.py:122 is decided on float64 ELBO values
    # (vbx_exact64.cu) whenever the float32 ELBO step is not safely away from epsilon ('early_stop': epsilon = 1e-3
    # on |ELBO| = 2e4, at float32 resolution)
    assert n == len(c['Li']), (n, len(c['Li']))
    m = n
    assert np.abs(out['gamma'] - c['gamma']).max() <= G_TOL * np.abs(c['gamma']).max()
    assert np.abs(out['pi'][0] - c['pi']).max() <= PI_TOL * np.abs(c['pi']).max()
    check_elbo(out['Li'][0, :m], c['Li'][:m], median_tol=1e-6 if gemm == 1 else 3e-6)
    assert np.all(np.isnan(out['Li'][0, n:]))
    assert np.abs(out['alpha'][0] - c['alpha']).max() <= 1e-4 * max(1.0, np.abs(c['alpha']).max())
    assert np.abs(out['invL'][0] - c['invL']).max() <= 1e-4
    assert np.all(out['gamma_pad'] == 0)
    assert not (out['flags'][0] & 1)


def es_inputs():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    lab = z['labels_ahc'].astype(int)
    q = np.zeros((len(lab), lab.max() + 1))
    q[np.arange(len(lab)), lab] = 1.0
    q = np.exp(q * float(z['smoothing']))
    q /= q.sum(1, keepdims=True)
    return z, q


@pytest.mark.parametrize('fb', [2, 1], ids=['fused', 'split'])
def test_es2005a_fixed_iterations(fb):
    """Config 1: the real recording, same 13 iterations as the reference (VBx/vbhmm.py:154-158)."""
    z, q = es_inputs()
    out = run_gpu(z['fea'], z['Phi'], [q.shape[0]], q, Fa=float(z['Fa']), Fb=float(z['Fb']),
                  loopProb=float(z['loopProb']), maxIters=13, epsilon=-np.inf, fb_split=fb)
    assert np.abs(out['gamma'] - z['gamma']).max() <= G_TOL
    assert np.abs(out['pi'][0] - z['pi']).max() <= PI_TOL
    check_elbo(out['Li'][0], z['Li'])
    assert np.array_equal(out['gamma'].argmax(1), z['labels'])


@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
def test_es2005a_reference_stop_rule(gemm):
    """The reference's own call (VBx/vbhmm.py:154-158: maxIters=40, epsilon=1e-6 on |ELBO| ~ 7e4, far below float32
    resolution) through the batched float32 path: the recording is handed to the float64 finishing kernels once its
    ELBO step nears epsilon, stops at the reference's iteration 13 and meets the 1e-4 bar."""
    z, q = es_inputs()
    out = run_gpu(z['fea'], z['Phi'], [q.shape[0]], q, Fa=float(z['Fa']), Fb=float(z['Fb']),
                  loopProb=float(z['loopProb']), maxIters=40, epsilon=1e-6, gemm=gemm)
    n = int(out['n_iters'][0])
    assert n == len(z['Li']) == 13, n
    assert np.abs(out['gamma'] - z['gamma']).max() <= G_TOL
    assert np.abs(out['pi'][0] - z['pi']).max() <= PI_TOL
    check_elbo(out['Li'][0, :n], z['Li'])
    # the float64 iterations reproduce the reference's ELBO steps far below epsilon
    d_ref, d_got = np.diff(z['Li'])[-4:], np.diff(out['Li'][0, :n])[-4:]
    assert np.abs(d_ref - d_got).max() < 1e-7, (d_ref, d_got)
    assert np.all(np.isnan(out['Li'][0, n:]))
    assert bool(out['flags'][0] & 4)
    assert np.array_equal(out['gamma'].argmax(1), z['labels'])


def test_es2005a_stop_rule_float32_only():
    """exact_stop=False keeps everything in float32: the stop iteration then depends on float32 ELBO noise (documented
    behaviour of that option), the result stays close to the reference's."""
    z, q = es_inputs()
    out = run_gpu(z['fea'], z['Phi'], [q.shape[0]], q, Fa=float(z['Fa']), Fb=float(z['Fb']),
                  loopProb=float(z['loopProb']), maxIters=40, epsilon=1e-6, exact_stop=False)
    n = int(out['n_iters'][0])
    assert 5 <= n <= 40
    assert abs(out['Li'][0, n - 1] - z['Li'][-1]) <= 1e-6 * abs(z['Li'][-1])
    assert np.abs(out['gamma'] - z['gamma']).max() <= 2e-2, n      # stops some iterations early on float32 ELBO noise
    assert np.array_equal(out['gamma'].argmax(1), z['labels'])


def ragged_batch(B, S, seed, tmax=700, R=128):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, tmax, size=B)
    lens[0] = 1
    lens[1] = 2
    d = synth.make_batch(lens, R=R, S=S, seed=seed, dtype=np.float32)
    return lens, d


@pytest.mark.parametrize('spl', [1, 2, 4])
def test_ragged_batch_vs_oracle(spl):
    S = 16
    lens, d = ragged_batch(37, S, seed=21)
    ns = np.random.default_rng(3).integers(1, S + 1, size=len(lens)).astype(np.int32)
    ns[:4] = S
    g0 = d['gamma0'].astype(np.float64)
    for b, (lo, hi) in enumerate(zip(d['offsets'][:-1], d['offsets'][1:])):
        g0[lo:hi, ns[b]:] = 0
        g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
    pi0 = np.zeros((len(lens), S))
    for b in range(len(lens)):
        pi0[b, :ns[b]] = 1.0 / ns[b]
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, 0.3, 17.0, 0.99, 8, -np.inf, n_states=ns)
    out = run_gpu(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0=None, n_states=ns, spl=spl,
                  Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=8, epsilon=-np.inf)
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= PI_TOL
    check_elbo(out['Li'], ref['Li'])
    assert np.all(out['n_iters'] == 8)


@pytest.mark.parametrize('tag', ['ami_hp', 'dead_speaker', 'loop0', 'loop1', 't1', 's64', 'dihard_hp'])
def test_classic_forward_backward_sweep(tag):
    """The normalise-every-frame sweep (option fb_classic = 1) stays selectable for A/B runs: it meets the same goldens
    and the two sweeps agree with each other far inside the parity bar."""
    c = CASES[tag]
    T = c['fea'].shape[0]
    kw = dict(Fa=float(c['Fa']), Fb=float(c['Fb']), loopProb=float(c['loopProb']), maxIters=len(c['Li']), epsilon=-np.inf)
    classic, ahead = (run_gpu(c['fea'], c['Phi'], [T], c['gamma0'], pi0=c['pi0'], fb_classic=v, **kw) for v in (1, 0))
    assert np.abs(classic['gamma'] - c['gamma']).max() <= G_TOL * np.abs(c['gamma']).max()
    assert np.abs(classic['pi'][0] - c['pi']).max() <= PI_TOL * np.abs(c['pi']).max()
    check_elbo(classic['Li'][0], c['Li'])
    assert np.abs(classic['gamma'] - ahead['gamma']).max() <= 2e-5
    check_elbo(classic['Li'][0], ahead['Li'][0])


@pytest.mark.parametrize('fb', [2, 1], ids=['fused', 'split'])
@pytest.mark.parametrize('S', [3, 4, 8, 10, 16, 31, 32, 64])
def test_state_counts_vs_oracle(S, fb):
    lens, d = ragged_batch(9, S, seed=30 + S, tmax=400)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S),
                              0.2, 6.0, 0.35, 6, -np.inf)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=0.2, Fb=6.0, loopProb=0.35, maxIters=6, epsilon=-np.inf, fb_split=fb)
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= PI_TOL
    check_elbo(out['Li'], ref['Li'])


@pytest.mark.parametrize('fb', [2, 1], ids=['chunked_scan', 'split'])
@pytest.mark.parametrize('S', [6, 16, 30, 64])
def test_long_recordings_chunked_scan(S, fb):
    """Recordings of >= 4096 frames: inside a large batch they take the chunked-scan forward-backward (three phases per
    sweep), in a small batch the concurrent forward / backward sweeps; mixed with short ones in the same batch.  Same
    parity bar against the oracle."""
    lens = np.array([4096, 300, 5000, 4097, 1, 9000 if S <= 16 else 4500])
    d = synth.make_batch(lens, R=128, S=S, seed=90 + S, dtype=np.float32)
    ns = np.full(len(lens), S, dtype=np.int32)
    ns[2] = max(2, S - 3)
    g0 = d['gamma0'].astype(np.float64)
    lo, hi = d['offsets'][2], d['offsets'][3]
    g0[lo:hi, ns[2]:] = 0
    g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
    pi0 = np.zeros((len(lens), S))
    for b in range(len(lens)):
        pi0[b, :ns[b]] = 1.0 / ns[b]
    kw = dict(Fa=0.2, Fb=6.0, loopProb=0.35) if S == 30 else dict(Fa=0.3, Fb=17.0, loopProb=0.99)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, kw['Fa'], kw['Fb'], kw['loopProb'], 6, -np.inf, n_states=ns)
    out = run_gpu(d['fea'], d['Phi'], lens, g0.astype(np.float32), n_states=ns, maxIters=6, epsilon=-np.inf, fb_split=fb, **kw)
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= PI_TOL
    check_elbo(out['Li'], ref['Li'])
    assert np.abs(out['gamma'].sum(1) - 1).max() < 1e-5
    # a long recording alone == inside the batch, bit for bit
    lo, hi = d['offsets'][0], d['offsets'][1]
    one = run_gpu(d['fea'][lo:hi], d['Phi'], [hi - lo], g0[lo:hi].astype(np.float32), maxIters=6, epsilon=-np.inf, fb_split=fb, **kw)
    assert np.array_equal(one['gamma'], out['gamma'][lo:hi]) and np.array_equal(one['Li'][0], out['Li'][0])


@pytest.mark.parametrize('name,B,T,S,iters,hp,fb', [
    ('config2_headline_shape', 48, 1000, 16, 10, (0.3, 17.0, 0.99), 2),
    ('config2_small_batch', 48, 1000, 16, 10, (0.3, 17.0, 0.99), 1),
    ('config3_ragged_20_iterations', 48, (200, 3000), 16, 20, (0.3, 17.0, 0.99), 2),
    ('config4_long_40_iterations_chunked', 3, 12000, 30, 40, (0.2, 6.0, 0.35), 2),
    ('config4_long_40_iterations_split', 3, 12000, 30, 40, (0.2, 6.0, 0.35), 1),
    ('config5_s64', 6, 2000, 64, 10, (0.3, 17.0, 0.99), 2),
])
def test_baseline_configs_at_their_sizes(name, B, T, S, iters, hp, fb):
    """BASELINE.json's configs at their own recording length, state count and ITERATION count (error growth over 20-40
    float32 iterations included), a sample of recordings each, against the float64 oracle; bench.py repeats this check on
    recordings of the full-size batch it times."""
    rng = np.random.default_rng(len(name))
    lens = rng.integers(T[0], T[1] + 1, size=B) if isinstance(T, tuple) else np.full(B, T)
    d = synth.make_batch(lens, R=128, S=S, seed=400 + B + S, dtype=np.float32)
    Fa, Fb, lp = hp
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), Fa, Fb, lp, iters, -np.inf)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=Fa, Fb=Fb, loopProb=lp, maxIters=iters, epsilon=-np.inf, fb_split=fb)
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= PI_TOL
    check_elbo(out['Li'], ref['Li'])
    assert np.array_equal(out['gamma'].argmax(1), ref['gamma'].argmax(1)) or \
        (out['gamma'].argmax(1) != ref['gamma'].argmax(1)).mean() < 1e-3


def test_partitioned_batch_equals_the_whole_batch():
    """vbx_b200.parts: two sub-batches on two streams give bit-identical results to one batch (recordings are independent),
    through the projection, both stop-rule phases, hard labels and the ELBO trace."""
    from vbx_b200.batch import VbxBatch
    from vbx_b200.parts import make_batch, PartitionedBatch
    S = 7
    lens, d = ragged_batch(41, S, seed=99, tmax=500)
    dd = synth.make_batch(lens, R=128, S=S, seed=99, D=256, dtype=np.float32)
    ns = np.full(len(lens), S, dtype=np.int32)
    ns[5] = 3
    g0 = dd['gamma0'].astype(np.float32).copy()
    lo, hi = dd['offsets'][5], dd['offsets'][6]
    g0[lo:hi, 3:] = 0
    g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
    results = []
    for parts in (1, 2, 3):
        vb = make_batch(lens, 128, ns, device=dev(), parts=parts)
        assert isinstance(vb, PartitionedBatch) == (parts > 1)
        g = torch.zeros((int(lens.sum()), vb.S), device=dev())
        g[:, :S] = cuda(g0)
        p = torch.zeros((len(lens), vb.S), device=dev())
        for b in range(len(lens)):
            p[b, :ns[b]] = 1.0 / ns[b]
        rho = vb.prepare_project(cuda(dd['X']), cuda(dd['V']), cuda(dd['Phi']))
        out = vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=25, epsilon=1e-5, return_model=True)
        lab = vb.hard_labels(g)
        tr = vb.elbo_trace(out['Li'])
        torch.cuda.synchronize()
        results.append([t.cpu().numpy() for t in (rho, g, p, out['Li'], out['n_iters'], out['flags'], out['alpha'], lab, tr)])
        vb.close()
    for other in results[1:]:
        for a, b in zip(results[0], other):
            assert np.array_equal(a, b, equal_nan=True)
    assert len(set(results[0][4].tolist())) > 1          # recordings stopped at different iterations


@pytest.mark.parametrize('eps', [-np.inf, 1e-5])
def test_cuda_graph_replay_is_identical(eps):
    """Option 'graph' (auto for small batches): the second call with identical arguments is captured, later ones replay the
    whole run as one CUDA graph launch.  Results equal the directly launched first run bit for bit, through both stop-rule
    phases; a call with different arguments falls back to direct launches."""
    from vbx_b200.batch import VbxBatch
    S = 6
    lens, d = ragged_batch(14, S, seed=71, tmax=400)
    vb = VbxBatch(lens, 128, S, device=dev())
    vb.set_option('graph', 1)
    g0 = torch.zeros((int(lens.sum()), vb.S), device=dev())
    g0[:, :S] = cuda(d['gamma0'])
    g, p = torch.empty_like(g0), torch.empty((len(lens), vb.S), device=dev())
    vb.prepare_scale(cuda(d['fea']), cuda(d['Phi']))
    # fixed output buffers: identical pointers from call to call (run() allocates Li / n_iters / flags itself, so bind them)
    outs, launches = [], []
    import ctypes
    Li = torch.empty((len(lens), 30), dtype=torch.float64, device=dev())
    ni = torch.empty(len(lens), dtype=torch.int32, device=dev())
    fl = torch.empty(len(lens), dtype=torch.int32, device=dev())
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    for rep in range(5):
        g.copy_(g0)
        p.zero_()
        p[:, :S] = 1.0 / S
        l0 = vb.launches
        vb._check(vb.lib.vbx_run(vb._h, ptr(vb.rho), ptr(vb.Phi), ptr(g), ptr(p), None, 0.3, 17.0, 0.99, 30, float(eps), None, None, 0,
                                 ptr(Li), ptr(ni), ptr(fl), vb._stream()))
        torch.cuda.synchronize()
        launches.append(vb.launches - l0)
        outs.append([t.clone().cpu().numpy() for t in (g, p, Li, ni, fl)])
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b, equal_nan=True)
    assert len(set(launches)) == 1 and launches[0] > 30           # the counter counts the kernels a replay runs
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), 0.3, 17.0, 0.99, 30, eps)
    assert np.array_equal(outs[0][3], ref['n_iters'])
    assert np.abs(outs[0][0][:, :S] - ref['gamma']).max() <= G_TOL
    # different arguments on the same handle: direct launches again, still right
    g.copy_(g0)
    p.zero_()
    p[:, :S] = 1.0 / S
    out = vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.9, maxIters=5, epsilon=-np.inf)
    ref2 = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), 0.3, 17.0, 0.9, 5, -np.inf)
    torch.cuda.synchronize()
    assert np.abs(g[:, :S].double().cpu().numpy() - ref2['gamma']).max() <= G_TOL
    vb.close()


def test_small_feature_dims():
    for R in (16, 32, 64):
        lens, d = ragged_batch(6, 5, seed=50 + R, tmax=200, R=R)
        ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(5, 0.2), 0.4, 17.0, 0.4, 5, -np.inf)
        out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=0.4, Fb=17.0, loopProb=0.4, maxIters=5, epsilon=-np.inf)
        assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
        check_elbo(out['Li'], ref['Li'])


def test_per_recording_early_stop_in_a_batch():
    """Recordings stop independently (VBx/VBx.py:122-125); stopped ones stay frozen; Li is NaN padded."""
    lens, d = ragged_batch(12, 8, seed=77, tmax=500)
    eps = 0.5
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(8, 0.125), 0.3, 17.0, 0.99, 30, eps)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=30, epsilon=eps)
    assert len(set(ref['n_iters'].tolist())) > 1, 'test needs recordings that stop at different iterations'
    assert np.array_equal(out['n_iters'], ref['n_iters']), (out['n_iters'], ref['n_iters'])
    for b in range(len(lens)):
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        n = int(ref['n_iters'][b])
        assert np.abs(out['gamma'][lo:hi] - ref['gamma'][lo:hi]).max() <= G_TOL
        check_elbo(out['Li'][b, :n], ref['Li'][b, :n])
        assert np.all(np.isnan(out['Li'][b, n:]))
        assert bool(out['flags'][b] & 4) == (n < 30)


@pytest.mark.parametrize('eps,S,hp', [(1e-4, 8, (0.3, 17.0, 0.99)), (1e-6, 16, (0.3, 17.0, 0.99)), (1e-5, 30, (0.2, 6.0, 0.35))])
def test_stop_rule_of_a_batch_matches_the_float64_oracle(eps, S, hp):
    """epsilon far below float32 resolution (the values the recipes use): every recording of a ragged batch finishes in
    the float64 kernels and stops at exactly the iteration the float64 oracle stops at."""
    lens, d = ragged_batch(20, S, seed=300 + S, tmax=900)
    Fa, Fb, lp = hp
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), Fa, Fb, lp, 40, eps)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=Fa, Fb=Fb, loopProb=lp, maxIters=40, epsilon=eps)
    assert np.array_equal(out['n_iters'], ref['n_iters']), (out['n_iters'], ref['n_iters'])
    assert len(set(ref['n_iters'].tolist())) > 2
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= PI_TOL
    for b in range(len(lens)):
        n = int(ref['n_iters'][b])
        check_elbo(out['Li'][b, :n], ref['Li'][b, :n])
        assert np.all(np.isnan(out['Li'][b, n:]))
        assert bool(out['flags'][b] & 4) == (n < 40)
    # alone == inside the batch, bit for bit, through both phases
    for b in (2, 7):
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        one = run_gpu(d['fea'][lo:hi], d['Phi'], [hi - lo], d['gamma0'][lo:hi], Fa=Fa, Fb=Fb, loopProb=lp, maxIters=40, epsilon=eps)
        assert np.array_equal(one['gamma'], out['gamma'][lo:hi]) and np.array_equal(one['Li'][0], out['Li'][b], equal_nan=True)


@pytest.mark.parametrize('eps', [1e-3, 1e-5])
def test_stop_rule_many_tiny_recordings(eps):
    """Very short recordings have a small |ELBO| and therefore the tightest float32 noise bound: 300 recordings of 1 .. 40
    frames must all stop at the float64 oracle's iteration."""
    rng = np.random.default_rng(8)
    lens = rng.integers(1, 41, size=300)
    S = 5
    d = synth.make_batch(lens, R=128, S=S, seed=808, dtype=np.float32)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), 0.3, 17.0, 0.9, 40, eps)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=0.3, Fb=17.0, loopProb=0.9, maxIters=40, epsilon=eps)
    bad = np.nonzero(out['n_iters'] != ref['n_iters'])[0]
    assert len(bad) == 0, [(int(b), int(lens[b]), int(out['n_iters'][b]), int(ref['n_iters'][b])) for b in bad[:10]]
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL


def test_stop_rule_long_recording_and_model_output():
    """A recording that takes the chunked-scan path in float32 finishes sequentially in float64; alpha / invL returned
    with return_model come from the last (float64) M-step."""
    lens = np.array([4200, 350])
    S = 6
    d = synth.make_batch(lens, R=128, S=S, seed=123, dtype=np.float32)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), 0.3, 17.0, 0.99, 40, 1e-5)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=40, epsilon=1e-5)
    assert np.array_equal(out['n_iters'], ref['n_iters']), (out['n_iters'], ref['n_iters'])
    assert np.abs(out['gamma'] - ref['gamma']).max() <= G_TOL
    assert np.abs(out['alpha'] - ref['alpha']).max() <= 1e-4 * max(1.0, np.abs(ref['alpha']).max())
    assert np.abs(out['invL'] - ref['invL']).max() <= 1e-4


def test_batch_is_independent_and_deterministic():
    """A recording gives bit-identical results alone, inside a batch, and on a second run."""
    lens, d = ragged_batch(10, 16, seed=5, tmax=600)
    kw = dict(Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=5, epsilon=-np.inf)
    full = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], **kw)
    again = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], **kw)
    assert np.array_equal(full['gamma'], again['gamma']) and np.array_equal(full['Li'], again['Li'])
    for b in (0, 3, 9):
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        one = run_gpu(d['fea'][lo:hi], d['Phi'], [hi - lo], d['gamma0'][lo:hi], **kw)
        assert np.array_equal(one['gamma'], full['gamma'][lo:hi])
        assert np.array_equal(one['pi'][0], full['pi'][b])
        assert np.array_equal(one['Li'][0], full['Li'][b])


def test_projection_matches_fp32_matmul():
    from vbx_b200.batch import VbxBatch
    lens = [300, 45, 129, 1]
    d = synth.make_batch(lens, R=128, S=4, seed=9, D=256, dtype=np.float32)
    vb = VbxBatch(lens, 128, 4, device=dev())
    rho = vb.prepare_project(cuda(d['X']), cuda(d['V']), cuda(d['Phi']))
    torch.cuda.synchronize()
    want = d['X'].astype(np.float64) @ d['V'].astype(np.float64)
    got = rho.double().cpu().numpy()
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max()
    # and it equals the scale path on the projected features (rho = fea * sqrt(Phi))
    want2 = d['fea'].astype(np.float64) * np.sqrt(d['Phi'].astype(np.float64))
    assert np.abs(got - want2).max() <= 1e-4 * np.abs(want2).max()
    vb.close()


@pytest.mark.parametrize('n_rec,T', [(4, 119), (300, 1000)])
def test_projection_tcgen05(n_rec, T):
    """The tensor-core (wgmma) 3xTF32 projection kernel against a float64 matmul (several tiles per persistent CTA)."""
    from vbx_b200.batch import VbxBatch
    lens = [T] * n_rec
    rng = np.random.default_rng(7)
    N = n_rec * T
    X = rng.standard_normal((N, 256)).astype(np.float32) * 3.0
    V = (synth.projection_basis(256, 128) * np.sqrt(synth.plda_phi(128))[None, :]).astype(np.float32)
    vb = VbxBatch(lens, 128, 4, device=dev())
    vb.set_option('projection', 2)
    rho = vb.prepare_project(cuda(X), cuda(V), cuda(synth.plda_phi(128)))
    torch.cuda.synchronize()
    got = rho.double().cpu().numpy()
    want = X.astype(np.float64) @ V.astype(np.float64)
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err <= 5e-6, err
    vb.set_option('projection', 1)
    rho2 = vb.prepare_project(cuda(X), cuda(V), cuda(synth.plda_phi(128)))
    torch.cuda.synchronize()
    err2 = np.abs(rho2.double().cpu().numpy() - want).max() / np.abs(want).max()
    print("projection error: wgmma 3xTF32 %.2e, FFMA %.2e" % (err, err2))
    assert err <= 32 * err2 + 1e-7, (err, err2)       # split-precision tensor cores stay near FFMA-level accuracy
    vb.close()


def _synthetic_xvector_model(rng, Dx=256):
    """A model with the shapes of the shipped one (VBx/models/ResNet101_16kHz: 256 -> LDA 128 -> PLDA 128)."""
    mean1 = rng.standard_normal(Dx) * 0.5
    lda = rng.standard_normal((Dx, 128)) / np.sqrt(Dx)
    mean2 = rng.standard_normal(128) * 0.05
    plda_mu = rng.standard_normal(128) * 0.02
    q, _ = np.linalg.qr(rng.standard_normal((128, 128)))
    plda_tr = q * rng.uniform(2.0, 20.0, 128)[:, None]        # already-diagonalised model: any full-rank transform
    plda_psi = synth.plda_phi(128).astype(np.float64)
    return mean1, lda, mean2, plda_mu, plda_tr, plda_psi


@pytest.mark.parametrize('n_rec,T', [(3, 77), (1, 256), (200, 1000)])
def test_xvector_chain_tcgen05(n_rec, T):
    """vbx_prepare_xvectors (VBx/vbhmm.py:125-129,153 + VBx/VBx.py:88-89 on the tensor cores) against the float64
    host chain of vbx_b200.pipeline, then the EM loop on top of it against the oracle."""
    from vbx_b200.batch import VbxBatch
    from vbx_b200 import pipeline
    rng = np.random.default_rng(101 + T)
    lens = [T] * n_rec
    N = n_rec * T
    mean1, lda, mean2, mu, tr, psi = _synthetic_xvector_model(rng)
    x_raw = (rng.standard_normal((N, 256)) * 2.0 + mean1[None, :]).astype(np.float32)
    f32 = lambda a: cuda(np.ascontiguousarray(a, dtype=np.float32))
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).double()   # the float32 model, in float64
    xn64 = pipeline.xvector_transform(t64(x_raw), t64(mean1), t64(mean2), t64(lda))
    fea64 = pipeline.plda_project(xn64, t64(mu), t64(tr), 128).numpy()
    xn64 = xn64.numpy()
    psi32 = t64(psi).numpy()
    rho64 = fea64 * np.sqrt(psi32)[None, :]
    S = 4
    vb = VbxBatch(lens, 128, S, device=dev())
    rho, x_norm = vb.prepare_xvectors(cuda(x_raw), f32(mean1), f32(lda), f32(mean2), f32(mu), f32(tr), f32(psi))
    torch.cuda.synchronize()
    e1 = np.abs(x_norm.double().cpu().numpy() - xn64).max() / np.abs(xn64).max()
    e2 = np.abs(rho.double().cpu().numpy() - rho64).max() / np.abs(rho64).max()
    print("x-vector chain error: x_norm %.2e, rho %.2e" % (e1, e2))
    assert e1 <= 5e-6, e1
    assert e2 <= 1e-5, e2
    assert np.abs(np.linalg.norm(x_norm.double().cpu().numpy(), axis=1) - 1.0).max() <= 1e-6
    if N <= 4096:      # EM on top (G comes from the fused epilogue): compare with the oracle on the float64 features
        offsets = np.concatenate([[0], np.cumsum(lens)])
        g0 = rng.random((N, S))
        g0 /= g0.sum(1, keepdims=True)
        ref = co.vbx_oracle_batch(fea64, psi32, offsets, g0, np.full(S, 1.0 / S), 0.3, 17.0, 0.99, 5, -np.inf)
        g = cuda(g0.astype(np.float32))
        p = torch.full((n_rec, S), 1.0 / S, device=dev())
        out = vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=5, epsilon=-np.inf)
        torch.cuda.synchronize()
        assert np.abs(g.double().cpu().numpy() - ref['gamma']).max() <= G_TOL
        check_elbo(out['Li'].cpu().numpy(), ref['Li'])
    vb.close()


def test_hard_labels_kernel():
    """vbx_hard_labels == argsort(-q)[:, 0] / [:, 1] (VBx/vbhmm.py:160-162) on a ragged batch with per-recording
    state counts; padded columns never win even when they hold garbage."""
    from vbx_b200.batch import VbxBatch
    rng = np.random.default_rng(5)
    lens = [1, 63, 64, 65, 300, 2]
    ns = [3, 5, 1, 7, 6, 2]
    vb = VbxBatch(lens, 128, ns, device=dev())
    N, S = sum(lens), vb.S
    g = rng.random((N, S)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(lens)])
    first, second = vb.hard_labels(cuda(g), second=True)
    torch.cuda.synchronize()
    first, second = first.cpu().numpy(), second.cpu().numpy()
    for b, n in enumerate(ns):
        q = g[off[b]:off[b + 1], :n]
        order = np.argsort(-q, axis=1, kind='stable')
        assert np.array_equal(first[off[b]:off[b + 1]], order[:, 0])
        if n > 1:
            assert np.array_equal(second[off[b]:off[b + 1]], order[:, 1])
        else:
            assert np.all(second[off[b]:off[b + 1]] == -1)
    vb.close()


def test_full_pipeline_from_raw_xvectors():
    """X (D=256) -> rho = X.V -> EM: equals the oracle run on fea = X.V0."""
    from vbx_b200.batch import VbxBatch
    lens = [257, 64, 400]
    S = 8
    d = synth.make_batch(lens, R=128, S=S, seed=19, D=256, dtype=np.float32)
    fea64 = d['X'].astype(np.float64) @ synth.projection_basis(256, 128)
    ref = co.vbx_oracle_batch(fea64, d['Phi'], d['offsets'], d['gamma0'], np.full(S, 1.0 / S), 0.3, 17.0, 0.99, 6, -np.inf)
    vb = VbxBatch(lens, 128, S, device=dev())
    vb.prepare_project(cuda(d['X']), cuda(d['V']), cuda(d['Phi']))
    g = cuda(d['gamma0'])
    p = torch.full((3, S), 1.0 / S, device=dev())
    out = vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=6, epsilon=-np.inf)
    torch.cuda.synchronize()
    assert np.abs(g.double().cpu().numpy() - ref['gamma']).max() <= G_TOL
    check_elbo(out['Li'].cpu().numpy(), ref['Li'])
    vb.close()


def test_properties_at_scale():
    """Size-independent properties on a batch too big for the numpy oracle: rows of gamma sum to 1, pi sums to 1,
    ELBO does not decrease (up to float32 noise), permuting speaker columns permutes the result; a sample of
    recordings is compared against the C oracle."""
    B, T, S = 512, 1000, 16
    lens = np.full(B, T)
    d = synth.make_batch(lens, R=128, S=S, seed=123, dtype=np.float32)
    kw = dict(Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=10, epsilon=-np.inf)
    out = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'], **kw)
    assert np.abs(out['gamma'].sum(1) - 1).max() < 1e-4
    assert np.abs(out['pi'].sum(1) - 1).max() < 1e-5
    dl = np.diff(out['Li'], axis=1)
    assert (dl >= -1e-6 * np.abs(out['Li'][:, 1:])).all()
    perm = np.random.default_rng(0).permutation(S)
    outp = run_gpu(d['fea'], d['Phi'], lens, d['gamma0'][:, perm], **kw)
    np.testing.assert_allclose(outp['Li'], out['Li'], rtol=1e-6)
    assert np.abs(outp['gamma'] - out['gamma'][:, perm]).max() < 1e-4
    sel = np.arange(0, B, 37)
    offs = np.arange(len(sel) + 1) * T
    fea = np.concatenate([d['fea'][b * T:(b + 1) * T] for b in sel])
    g0 = np.concatenate([d['gamma0'][b * T:(b + 1) * T] for b in sel])
    ref = co.vbx_oracle_batch(fea, d['Phi'], offs, g0, np.full(S, 1.0 / S), 0.3, 17.0, 0.99, 10, -np.inf)
    got = np.concatenate([out['gamma'][b * T:(b + 1) * T] for b in sel])
    assert np.abs(got - ref['gamma']).max() <= G_TOL
    check_elbo(out['Li'][sel], ref['Li'])


def run_gpu_f64(fea, Phi, T, gamma0, pi0, **kw):
    from vbx_b200.batch import VbxBatch, run_f64
    S_user = gamma0.shape[1]
    vb = VbxBatch([T], fea.shape[1], S_user, device=dev(), allocate=False)
    g = torch.zeros((T, vb.S), dtype=torch.float64, device=dev())
    g[:, :S_user] = cuda(gamma0, torch.float64)
    p = torch.zeros((1, vb.S), dtype=torch.float64, device=dev())
    p[0, :S_user] = cuda(pi0, torch.float64)
    extra = {}
    if 'alpha0' in kw:
        a = torch.zeros((1, vb.S, fea.shape[1]), dtype=torch.float64, device=dev())
        il = torch.zeros_like(a)
        a[0, :S_user] = cuda(kw.pop('alpha0'), torch.float64)
        il[0, :S_user] = cuda(kw.pop('invL0'), torch.float64)
        extra = dict(alpha=a, invL=il, warm_start=True)
    out = run_f64(vb, cuda(fea, torch.float64), cuda(Phi, torch.float64), g, p, return_model=True, **extra, **kw)
    res = dict(gamma=g[:, :S_user].cpu().numpy(), pi=p[0, :S_user].cpu().numpy(), Li=out['Li'][0].cpu().numpy(),
               n=int(out['n_iters'][0].item()), flags=int(out['flags'][0].item()),
               alpha=out['alpha'][0, :S_user].cpu().numpy(), invL=out['invL'][0, :S_user].cpu().numpy())
    vb.close()
    return res


@pytest.mark.parametrize('tag', sorted(CASES))
def test_float64_mode_matches_reference_tightly(tag):
    """The float64 evaluation path (the drop-in's default): iteration counts identical, values to ~1e-8."""
    c = CASES[tag]
    kw = dict(Fa=float(c['Fa']), Fb=float(c['Fb']), loopProb=float(c['loopProb']), maxIters=int(c['maxIters']),
              epsilon=float(c['epsilon']))
    if 'alpha0' in c:
        kw.update(alpha0=c['alpha0'], invL0=c['invL0'])
    out = run_gpu_f64(c['fea'], c['Phi'], c['fea'].shape[0], c['gamma0'], c['pi0'], **kw)
    assert out['n'] == len(c['Li'])
    np.testing.assert_allclose(out['gamma'], c['gamma'], rtol=0, atol=1e-7)
    np.testing.assert_allclose(out['pi'], c['pi'], rtol=0, atol=1e-8)
    np.testing.assert_allclose(out['Li'][:out['n']], c['Li'], rtol=1e-9)
    np.testing.assert_allclose(out['alpha'], c['alpha'], rtol=0, atol=1e-7)
    np.testing.assert_allclose(out['invL'], c['invL'], rtol=0, atol=1e-9)
    if tag == 'early_stop':       # the reference printed its 'auxiliary function has decreased' warning here
        assert out['flags'] & 2 and out['flags'] & 4


def test_float64_mode_es2005a_reference_call():
    """The reference's own call VBx/vbhmm.py:154-158 (maxIters=40, epsilon=1e-6): 13 iterations, same trace."""
    z, q = es_inputs()
    S = q.shape[1]
    out = run_gpu_f64(z['fea'], z['Phi'], q.shape[0], q, np.full(S, 1.0 / S), Fa=float(z['Fa']), Fb=float(z['Fb']),
                      loopProb=float(z['loopProb']), maxIters=40, epsilon=1e-6)
    assert out['n'] == 13
    np.testing.assert_allclose(out['Li'][:13], z['Li'], rtol=1e-11)
    np.testing.assert_allclose(out['gamma'], z['gamma'], rtol=0, atol=1e-7)
    np.testing.assert_allclose(out['pi'], z['pi'], rtol=0, atol=1e-8)
    assert np.array_equal(out['gamma'].argmax(1), z['labels'])
    assert np.all(np.isnan(out['Li'][13:]))


def test_dropin_vbx_function():
    """The reference-facing call: numpy in, (gamma, pi, Li) out (VBx/VBx.py:27-29,126)."""
    from vbx_b200 import VBx
    c = CASES['example_hp']
    g, p, L = VBx(c['fea'], c['Phi'], loopProb=float(c['loopProb']), Fa=float(c['Fa']), Fb=float(c['Fb']),
                  pi=int(len(c['pi0'])), gamma=c['gamma0'], maxIters=int(c['maxIters']), epsilon=float(c['epsilon']))
    assert g.dtype == np.float64 and p.dtype == np.float64 and isinstance(L, list) and isinstance(L[0], list)
    assert g.shape == c['gamma'].shape and p.shape == c['pi'].shape and len(L) == len(c['Li'])
    assert np.abs(g - c['gamma']).max() <= 1e-7          # float64 evaluation is the drop-in's default
    np.testing.assert_allclose([l[0] for l in L], c['Li'], rtol=1e-9)
    import vbx_b200.api as api
    api.set_precision('float32')
    try:
        g32, p32, L32 = VBx(c['fea'], c['Phi'], loopProb=float(c['loopProb']), Fa=float(c['Fa']), Fb=float(c['Fb']),
                            pi=int(len(c['pi0'])), gamma=c['gamma0'], maxIters=int(c['maxIters']), epsilon=float(c['epsilon']))
    finally:
        api.set_precision('float64')
    assert np.abs(g32 - c['gamma']).max() <= G_TOL and len(L32) == len(c['Li'])
    check_elbo([l[0] for l in L32], c['Li'])
    g2, p2, L2, a2, il2 = VBx(c['fea'], c['Phi'], loopProb=float(c['loopProb']), Fa=float(c['Fa']), Fb=float(c['Fb']),
                              pi=c['pi0'], gamma=c['gamma0'], maxIters=3, epsilon=-np.inf, return_model=True)
    assert a2.shape == c['alpha'].shape and il2.shape == c['invL'].shape
    with pytest.raises(AssertionError):
        VBx(c['fea'], c['Phi'], pi=5, gamma=c['gamma0'])
    with pytest.raises(TypeError):
        VBx(c['fea'], c['Phi'], pi=np.int64(16), gamma=c['gamma0'])
    np.random.seed(4)
    g3, p3, L3 = VBx(c['fea'], c['Phi'], pi=6, maxIters=2)          # gamma=None: global np.random draw
    assert g3.shape == (c['fea'].shape[0], 6) and np.abs(g3.sum(1) - 1).max() < 1e-5


def test_c_abi_argument_errors():
    import ctypes
    import vbx_b200._lib as L
    lib = L.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    need = ctypes.c_size_t()
    off = np.array([0, 10], dtype=np.int64)
    po = off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    assert lib.vbx_plan(h, po, 1, 130, 16, ctypes.byref(need)) == -1      # R not supported
    assert lib.vbx_plan(h, po, 1, 128, 17, ctypes.byref(need)) == -1      # S not padded
    assert b'S must' in lib.vbx_last_error(h)
    assert lib.vbx_run(h, None, None, None, None, None, 1.0, 1.0, 0.9, 1, 0.0, None, None, 0, None, None, None, None) == -3
    assert lib.vbx_plan(h, po, 1, 128, 16, ctypes.byref(need)) == 0 and need.value > 0
    assert lib.vbx_bind_workspace(h, None, 0) == -3
    # entry points added with the section-8f rows: state and argument checks before anything is launched
    assert lib.vbx_set_option(h, b'fb_classic', 1) == 0 and lib.vbx_set_option(h, b'no_such_knob', 1) == -1
    for removed in (b'fold_speaker', b'fb_priority', b'stop_noise_c', b'stop_guard_mult'):
        assert lib.vbx_set_option(h, removed, 2) == -1 and b'unknown option' in lib.vbx_last_error(h), removed
    assert lib.vbx_prepare_xvectors(h, None, 256, None, None, None, None, None, None, None, None, None) == -3   # no workspace
    assert lib.vbx_hard_labels(h, None, None, None, None, None) == -1                                          # null pointers
    ahc_need = ctypes.c_size_t()
    assert lib.vbx_ahc_workspace_bytes(h, ctypes.byref(ahc_need)) == 0 and ahc_need.value >= 10 * 10 * 8
    assert lib.vbx_ahc(h, None, 0, 128, None, 0, None, None, None) == -1
    assert lib.vbx_ahc(h, None, 0, 0, None, 0, None, None, None) == -1 and b'dim' in lib.vbx_last_error(h)
    assert lib.vbx_destroy(h) == 0
    h2 = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h2)) == 0
    assert lib.vbx_ahc_workspace_bytes(h2, ctypes.byref(ahc_need)) == -3      # not planned yet
    assert lib.vbx_hard_labels(h2, None, None, None, None, None) == -3
    assert lib.vbx_destroy(h2) == 0


def test_float64_mode_ragged_batch_vs_oracle():
    """vbx_run_f64 on a ragged multi-recording batch with per-recording state counts."""
    from vbx_b200.batch import VbxBatch, run_f64
    S = 10
    lens, d = ragged_batch(7, S, seed=61, tmax=300)
    ns = np.array([10, 3, 10, 7, 1, 10, 5], dtype=np.int32)
    g0 = d['gamma0'].astype(np.float64)
    for b, (lo, hi) in enumerate(zip(d['offsets'][:-1], d['offsets'][1:])):
        g0[lo:hi, ns[b]:] = 0
        g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
    pi0 = np.zeros((len(lens), S))
    for b in range(len(lens)):
        pi0[b, :ns[b]] = 1.0 / ns[b]
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, 0.4, 17.0, 0.4, 9, 1e-3, n_states=ns)
    vb = VbxBatch(lens, 128, ns, device=dev(), allocate=False)
    g = torch.zeros((int(lens.sum()), vb.S), dtype=torch.float64, device=dev())
    g[:, :S] = cuda(g0, torch.float64)
    p = torch.zeros((len(lens), vb.S), dtype=torch.float64, device=dev())
    p[:, :S] = cuda(pi0, torch.float64)
    out = run_f64(vb, cuda(d['fea'], torch.float64), cuda(d['Phi'], torch.float64), g, p, Fa=0.4, Fb=17.0, loopProb=0.4,
                  maxIters=9, epsilon=1e-3)
    assert np.array_equal(out['n_iters'].cpu().numpy(), ref['n_iters'])
    np.testing.assert_allclose(g[:, :S].cpu().numpy(), ref['gamma'], rtol=0, atol=1e-8)
    np.testing.assert_allclose(p[:, :S].cpu().numpy(), ref['pi'], rtol=0, atol=1e-9)
    Li = out['Li'].cpu().numpy()
    assert np.array_equal(np.isnan(Li), np.isnan(ref['Li']))
    np.testing.assert_allclose(np.nan_to_num(Li), np.nan_to_num(ref['Li']), rtol=1e-10)
    vb.close()


def test_host_pipeline_equals_resident_path():
    """The host-buffer API (pinned host X / gamma0 in, gamma / pi / Li out, chunked over streams) gives bit-identical
    results to the device-resident calls, including per-recording state padding."""
    from vbx_b200.batch import VbxBatch
    from vbx_b200.host_pipeline import HostPipeline
    lens = np.array([700, 20, 333, 1, 512, 90, 1500, 64])
    S = 6
    d = synth.make_batch(lens, R=128, S=S, seed=41, D=256, dtype=np.float32)
    kw = dict(Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=5, epsilon=-np.inf)
    vb = VbxBatch(lens, 128, S, device=dev())
    vb.prepare_project(cuda(d['X']), cuda(d['V']), cuda(d['Phi']))
    g = torch.zeros((int(lens.sum()), vb.S), device=dev())
    g[:, :S] = cuda(d['gamma0'])
    p = torch.zeros((len(lens), vb.S), device=dev())
    p[:, :S] = 1.0 / S
    res = vb.run(g, p, **kw)
    torch.cuda.synchronize()
    hp = HostPipeline(lens, 256, 128, S, device=dev(), n_chunks=3)
    Xh = torch.from_numpy(d['X']).pin_memory()
    Gh = torch.from_numpy(d['gamma0']).pin_memory()
    out = hp.run(Xh, cuda(d['V']), cuda(d['Phi']), Gh, **kw)
    assert hp.n_chunks == 3
    assert torch.equal(out['gamma'], g[:, :S].cpu())
    assert torch.equal(out['pi'], p[:, :S].cpu())
    assert torch.equal(out['Li'], res['Li'].cpu())
    assert hp.h2d_bytes == int(lens.sum()) * (256 + S) * 4
    vb.close()


@pytest.mark.parametrize('T,R,S,precision', [(60, 200, 100, 'float64'), (90, 131, 70, 'float32'), (40, 3, 2, 'float64'), (1, 7, 65, 'float64')])
def test_dropin_has_no_size_limits(T, R, S, precision):
    """The reference accepts any number of states and any feature dimension; so does the drop-in: its float64 kernels
    loop over states / features (vbx_plan_f64), and the float32 mode hands sizes beyond S = 64 / D = 128 to them."""
    import vbx_b200.api as api
    from oracle import vbx_oracle as po
    rng = np.random.default_rng(T + R + S)
    Phi = np.exp(np.linspace(np.log(5.6), np.log(0.53), R))
    fea, _ = synth.make_recording(T, R, Phi, rng, n_spk=3)
    g0 = synth.dirichlet_rows(T, S, rng)
    api.set_precision(precision)
    try:
        g, p, L, a, il = api.VBx(fea, Phi, loopProb=0.9, Fa=0.4, Fb=11.0, pi=S, gamma=g0, maxIters=6, epsilon=1e-6, return_model=True)
    finally:
        api.set_precision('float64')
    gr, pr, Lr, ar, ilr = po.vbx_oracle(fea, Phi, loopProb=0.9, Fa=0.4, Fb=11.0, pi=S, gamma=g0, maxIters=6, epsilon=1e-6, return_model=True)
    assert g.shape == (T, S) and p.shape == (S,) and a.shape == (S, R) and len(L) == len(Lr)
    np.testing.assert_allclose(g, gr, atol=1e-7)
    np.testing.assert_allclose(p, pr, atol=1e-8)
    np.testing.assert_allclose([l[0] for l in L], [l[0] for l in Lr], rtol=1e-9)
    np.testing.assert_allclose(a, ar, atol=1e-7)
    np.testing.assert_allclose(il, ilr, atol=1e-9)


def test_dropin_pads_odd_feature_dims():
    """lda_dim values that are not a multiple of 4 (VBx/vbhmm.py --lda-dim is free): float64 mode takes them as they are,
    float32 mode zero-pads on the host (R = 50 runs as 52, a width of 4 (mod 8) for the contraction kernels)."""
    import vbx_b200.api as api
    from oracle import vbx_oracle as po
    rng = np.random.default_rng(12)
    T, R, S = 150, 50, 5
    Phi = synth.plda_phi(R)
    fea, _ = synth.make_recording(T, R, Phi, rng, n_spk=3)
    g0 = synth.dirichlet_rows(T, S, rng)
    gr, pr, Lr, ar, ilr = po.vbx_oracle(fea, Phi, loopProb=0.8, Fa=0.4, Fb=17.0, pi=S, gamma=g0, maxIters=8, epsilon=1e-4,
                                        return_model=True)
    for precision in ('float64', 'float32'):
        api.set_precision(precision)
        try:
            g, p, L, a, il = api.VBx(fea, Phi, loopProb=0.8, Fa=0.4, Fb=17.0, pi=S, gamma=g0, maxIters=8, epsilon=1e-4,
                                     return_model=True)
        finally:
            api.set_precision('float64')
        assert len(L) == len(Lr) and a.shape == (S, R) and il.shape == (S, R), precision
        f32 = precision == 'float32'
        np.testing.assert_allclose(g, gr, atol=G_TOL if f32 else 1e-7)
        np.testing.assert_allclose([l[0] for l in L], [l[0] for l in Lr], rtol=L_RTOL if f32 else 1e-9)
        np.testing.assert_allclose(a, ar, atol=1e-4 * max(1.0, np.abs(ar).max()) if f32 else 1e-7)
        np.testing.assert_allclose(il, ilr, atol=1e-4 if f32 else 1e-9)
