"""The EM iteration against float64 one stage at a time (VBx/VBx.py:91-125), at every feature width, state tier, schedule
and tile edge.  The stages are isolated through the public API:

  1. M-step + speaker model: a cold start with maxIters = 1 and return_model: alpha and invL are the M-step and the
     speaker model applied to gamma0, compared with float64 computed here from gamma0 and the rho the device holds, under
     the per-element and normwise bounds of tests/test_em_stage_bounds_math.py; with one-hot gamma and integer rho every
     tile sum is exact and alpha is predicted bit for bit from the device's invL.
  2. Log-likelihood: a warm start from a given float32 model (no M-step), maxIters = 1, loopProb = 0: a gamma row is then
     the normalised p_t w, a per-frame view of the ll row, held to the stage-2 bounds; Li[0] to the sum of those bounds.
  3. Forward-backward: a warm start from the M-step on the true speaker turns, loopProb 0.35 / 0.99 and maxIters
     1 / 2, through every schedule (split,
     fused ring for every (S, states per lane), register burst, classic, chunked scan, S = 128): under the 1e-4 bar
     against the C oracle and within FB_FACTOR of the classic sweep's error on the same inputs.

Every batch carries the edges where kernels go wrong: T = 1, 2, 3, empty recordings mid-batch, frame offsets = 1, 2, 3
(mod 4), T - 1 at F - 1, F, F + 1, 2F, 2F + 1 for the sweeps' stages of F = 16 / 10 / 5 backward steps, M-tile edges
511 / 512 / 513 and 1023 / 1024 / 1025, L-tile edges 63 / 64 / 65, the ring limit 2047 / 2048 / 2049 and the chunked scan's
4095 / 4096 / 4097 and 4096 + 256 +- 1.  The workspace is poisoned with 0xFF, gamma is followed by NaN guard rows, dead
and padded columns must stay 0 and Li must be NaN past n_iters."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import c_oracle as co
from test_em_stage_bounds_math import U, ll_emulated, loglik_errors, loglik_parts, mstep_errors
from test_fb_ring_gpu import VARIANTS
from test_split_precision_math import mm
from vbx_b200 import synth

pytestmark = pytest.mark.gpu
G_TOL = 1e-4
FA, FB = 0.3, 17.0
GUARD = 3                  # NaN rows after gamma
# An optimised sweep may not be less accurate than the plain one: its max |gamma error| stays within FB_FACTOR times the
# classic sweep's on the same inputs (FB_FLOOR absorbs errors at the float32 rounding level).
FB_FACTOR, FB_FLOOR = 3.0, 1e-6
STAGE_F = (16, 10, 5)      # backward steps per stage of the fused sweeps at 1 / 2 / 4 states per lane (forward: 2F)


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def edge_lengths(extra=()):
    lens = [1, 2, 3, 0, 63, 64, 65]
    for F in STAGE_F:
        lens += [F, F + 1, F + 2, 2 * F + 1, 2 * F + 2]
    return np.array(lens + [511, 512, 513, 1023, 1024, 1025, 0, 2047, 2048, 7] + list(extra), dtype=np.int64)


def inputs(lens, R, S_user, seed, case='random'):
    """A packed batch with fewer live states than S_user in most recordings (dead columns of gamma0 are 0).
    case: 'random'; 'cancel' (rho with a large common offset); 'lowbits' (gamma values whose TF32 low part is not 0);
    'neardead' (the last live state of every recording holds N_s = 1e-6)."""
    lens = np.asarray(lens, dtype=np.int64)
    d = synth.make_batch(np.maximum(lens, 1), R=R, S=S_user, seed=seed, dtype=np.float32)   # synth needs T >= 1:
    rows = np.repeat(lens > 0, np.maximum(lens, 1))                                       # drop the empty ones' row
    d['gamma0'] = d['gamma0'][rows]
    fea, off = d['fea'][rows], np.concatenate([[0], np.cumsum(lens)])
    if case == 'cancel':
        fea = (fea + np.float32(40.0)).astype(np.float32)
    rng = np.random.default_rng(seed + 1)
    B = len(lens)
    ns = rng.integers(max(1, S_user // 2 + 1), S_user + 1, size=B).astype(np.int32)
    ns[0] = S_user
    g = d['gamma0'].astype(np.float64)
    for b in range(B):
        lo, hi = off[b], off[b + 1]
        g[lo:hi, ns[b]:] = 0.0
        g[lo:hi] /= np.maximum(g[lo:hi].sum(1, keepdims=True), 1e-300)
        if case == 'neardead' and ns[b] >= 2 and hi > lo:
            k = ns[b] - 1
            g[lo:hi, k] = 1e-6 / (hi - lo)
            g[lo:hi, :k] *= (1.0 - 1e-6 / (hi - lo)) / g[lo:hi, :k].sum(1, keepdims=True)
    g = g.astype(np.float32)
    if case == 'lowbits':
        bits = g.view(np.uint32)
        g = np.where(g > 0, (bits | np.uint32(0xFFF)).view(np.float32), g)
    pi0 = np.zeros((B, S_user), dtype=np.float32)
    for b in range(B):
        pi0[b, :ns[b]] = 1.0 / ns[b]
    return dict(fea=fea, Phi=d['Phi'], gamma0=g, pi0=pi0, ns=ns, offsets=off, lens=lens, R=R, S_user=S_user,
                paths=d['paths'][rows])


def warm_model(x, seed):
    """A float32 speaker model to start from (alpha, invL [B, S_user, R]); dead states are 0."""
    rng = np.random.default_rng(seed)
    B, S, R = len(x['lens']), x['S_user'], x['R']
    alpha = (0.6 * rng.standard_normal((B, S, R)) * np.sqrt(x['Phi'])[None, None, :]).astype(np.float32)
    invL = rng.uniform(0.02, 0.6, (B, S, R)).astype(np.float32)
    for b in range(B):
        alpha[b, x['ns'][b]:] = 0
        invL[b, x['ns'][b]:] = 0
    return alpha, invL


def mstep_model(x):
    """The float32 rounding of the float64 M-step and speaker model on the true speaker turns (one-hot, speaker k of a
    recording in state k mod n_states): the model of a run that has found its speakers.  The second iteration from an
    uninformative model (random, or the M-step of a flat gamma0) amplifies float32 rounding past the 1e-4 bar in every
    sweep alike, the classic one included; from this one the posteriors are as well conditioned as late in a real run."""
    B, S, R = len(x['lens']), x['S_user'], x['R']
    alpha = np.zeros((B, S, R), dtype=np.float32)
    invL = np.zeros_like(alpha)
    Phi = x['Phi'].astype(np.float64)
    rho = x['fea'].astype(np.float64) * np.sqrt(Phi)[None, :]
    off = x['offsets']
    for b in range(B):
        lo, hi, n = off[b], off[b + 1], x['ns'][b]
        g = np.zeros((hi - lo, n))
        g[np.arange(hi - lo), x['paths'][lo:hi] % n] = 1.0
        il = 1.0 / (1.0 + FA / FB * g.sum(0)[:, None] * Phi[None, :])
        invL[b, :n] = il
        alpha[b, :n] = FA / FB * il * (g.T @ rho[lo:hi])
    return alpha, invL


def run_device(x, gemm=0, fb_split=0, spl=0, ring=1, classic=0, maxIters=1, loopProb=0.99, epsilon=-np.inf, warm=None):
    """One vbx_run over the batch with the guards of the module docstring checked; numpy results."""
    from vbx_b200.batch import VbxBatch
    lens, ns, S_user, R = x['lens'], x['ns'], x['S_user'], x['R']
    vb = VbxBatch(lens, R, ns, device=dev(), fb_split=fb_split)
    vb.workspace.fill_(0xFF)           # NaN in float32 and float64: nothing may be read before it is written
    vb.set_option('gemm', gemm)
    vb.set_option('fb_ring', ring)
    vb.set_option('fb_classic', classic)
    if spl:
        vb.set_option('fb_states_per_lane', spl)
    S, N, B = vb.S, vb.N, vb.B
    buf = torch.full((N + GUARD, S), float('nan'), device=dev())
    g = buf[:N]
    g.zero_()
    g[:, :S_user] = cuda(x['gamma0'])
    p = torch.zeros((B, S), device=dev())
    p[:, :S_user] = cuda(x['pi0'])
    vb.prepare_scale(cuda(x['fea']), cuda(x['Phi']))
    kw = {}
    if warm is not None:
        a = torch.zeros((B, S, R), device=dev())
        il = torch.zeros_like(a)
        a[:, :S_user] = cuda(warm[0])
        il[:, :S_user] = cuda(warm[1])
        kw = dict(alpha=a, invL=il, warm_start=True)
    out = vb.run(g, p, Fa=FA, Fb=FB, loopProb=loopProb, maxIters=maxIters, epsilon=epsilon, return_model=True, **kw)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[N:]).all()), 'gamma written past its last row'
    gam = g.cpu().numpy()
    res = dict(gamma=gam[:, :S_user], pi=p[:, :S_user].cpu().numpy(), Li=out['Li'].cpu().numpy(),
               n_iters=out['n_iters'].cpu().numpy(), flags=out['flags'].cpu().numpy(), rho=vb.rho.cpu().numpy(),
               alpha=out['alpha'][:, :S_user].cpu().numpy(), invL=out['invL'][:, :S_user].cpu().numpy())
    vb.close()
    off = x['offsets']
    for b in range(B):
        assert np.all(gam[off[b]:off[b + 1], ns[b]:] == 0), f'recording {b}: a dead or padded column of gamma is not 0'
        n = int(res['n_iters'][b])
        assert np.all(np.isnan(res['Li'][b, n:])) and np.all(np.isfinite(res['Li'][b, :n])), (b, n, res['Li'][b])
        assert lens[b] > 0 or n == 0, f'empty recording {b} ran {n} iterations'
    assert not np.any(res['flags'] & 1), 'non-finite ELBO'
    return res


def oracle(x, maxIters, loopProb, epsilon=-np.inf, warm=None):
    """The C oracle over the non-empty recordings; returns (result, mask of the non-empty recordings)."""
    keep = x['lens'] > 0
    off = np.concatenate([[0], np.cumsum(x['lens'][keep])])
    kw = {} if warm is None else dict(alpha0=warm[0][keep], invL0=warm[1][keep])
    r = co.vbx_oracle_batch(x['fea'], x['Phi'], off, x['gamma0'], x['pi0'][keep], FA, FB, loopProb, maxIters, epsilon,
                            n_states=x['ns'][keep], **kw)
    return r, keep


def check_mstep(x, out, tag):
    off, ns = x['offsets'], x['ns']
    recs, alphas, invLs = [], [], []
    for b in range(len(x['lens'])):
        lo, hi, n = off[b], off[b + 1], ns[b]
        if hi == lo:
            continue
        assert np.all(out['alpha'][b, n:] == 0) and np.all(out['invL'][b, n:] == 0), f'recording {b}: dead state model'
        recs.append((x['gamma0'][lo:hi, :n], out['rho'][lo:hi]))
        alphas.append(out['alpha'][b, :n])
        invLs.append(out['invL'][b, :n])
    r_inv, r_a, nw, ceil = mstep_errors(recs, x['Phi'], FA, FB, alphas, invLs)
    print(f'{tag}: invL err / bound {r_inv:.3g}, alpha err / bound {r_a:.3g}, normwise {nw:.3g} = {nw / ceil:.3g} of the ceiling')
    assert r_inv <= 1 and r_a <= 1 and nw <= ceil, (tag, r_inv, r_a, nw, ceil)


def check_loglik(x, out, warm, ref, keep, tag):
    """Stage 2 through gamma (maxIters = 1, loopProb = 0) and Li[0] against the sum of the per-frame bounds."""
    off, ns, Phi, R = x['offsets'], x['ns'], x['Phi'], x['R']
    recs, gams, ws, grefs, ffma, li_ratio = [], [], [], [], [], 0.0
    ko = np.concatenate([[0], np.cumsum(x['lens'][keep])])
    for k, b in enumerate(np.flatnonzero(keep)):
        lo, hi, n = off[b], off[b + 1], ns[b]
        rho, a, il = out['rho'][lo:hi], warm[0][b, :n], warm[1][b, :n]
        gr = ref['gamma'][ko[k]:ko[k + 1], :n]
        assert np.abs(out['gamma'][lo:hi, :n] - gr).max() <= G_TOL
        recs.append((rho, a, il))
        gams.append(out['gamma'][lo:hi, :n])
        ws.append(x['pi0'][b, :n].astype(np.float64) + 1e-8)
        grefs.append(gr)
        ffma.append(ll_emulated(rho, a, il, Phi, FA, mm))
        # Li[0] = sum_t (rowmax_t + log sigma_t) + Fa G + Fb / 2 reg: per frame the log-sum-exp moves by at most max_s E,
        # sigma (a float32 sum of S terms) by (S + 8) u; G and reg are float32 sums of R terms per frame / state
        ll, E, _ = loglik_parts(rho, a, il, Phi, FA)
        x2 = (x['fea'][lo:hi].astype(np.float64)) ** 2
        reg = np.abs(np.log(il.astype(np.float64))) + il + a.astype(np.float64) ** 2 + 1.0
        bound = (E.max(1) + (n + 8) * U * (1.0 + np.abs(ll).max(1))).sum() + FA * 0.5 * (R + 8) * U * x2.sum() \
            + 0.5 * FB * 48 * U * reg.sum()
        li_ratio = max(li_ratio, abs(out['Li'][b, 0] - ref['Li'][k, 0]) / bound)
    worst, nw, ceil = loglik_errors(recs, Phi, FA, gams, ws, grefs, ffma)
    print(f'{tag}: ll err / bound {worst:.3g}, normwise {nw:.3g} = {nw / ceil:.3g} of the ceiling, Li[0] err / bound {li_ratio:.3g}')
    assert worst <= 1 and nw <= ceil and li_ratio <= 1, (tag, worst, nw, ceil, li_ratio)


def gamma_error(x, out, ref, keep, only=None):
    """max |gamma - gamma_ref| (and |pi - pi_ref|) over the non-empty recordings (or those where `only` holds)."""
    ko = np.concatenate([[0], np.cumsum(x['lens'][keep])])
    off, eg, ep = x['offsets'], 0.0, 0.0
    for k, b in enumerate(np.flatnonzero(keep)):
        if only is not None and not only[b]:
            continue
        eg = max(eg, float(np.abs(out['gamma'][off[b]:off[b + 1]] - ref['gamma'][ko[k]:ko[k + 1]]).max()))
        ep = max(ep, float(np.abs(out['pi'][b] - ref['pi'][k]).max()))
    return eg, ep


# ---- stage 1 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('case', ['random', 'cancel', 'lowbits', 'neardead'])
def test_mstep_and_speaker_model(case, gemm):
    x = inputs(edge_lengths(), 128, 13, seed=len(case) * 17 + gemm, case=case)
    for fb in (2, 1):
        out = run_device(x, gemm=gemm, fb_split=fb)
        check_mstep(x, out, f'{case} gemm={gemm} fb_split={fb}')


@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('R,S_user', [(12, 5), (52, 13), (128, 13), (128, 50), (36, 100)])
def test_mstep_exact_probe(R, S_user, gemm):
    """One-hot gamma and integer rho (Phi = 1): every tile sum is exact, so alpha = float32(float64(float32(FaFb invL))
    Sigma) bit for bit from the device's own invL; any layout, permutation or tile-tail error shows at any tolerance."""
    lens = np.array([513, 1, 0, 1025, 64, 511, 2, 65, 1024, 3], dtype=np.int64)
    x = inputs(lens, R, S_user, seed=R + S_user)
    rng = np.random.default_rng(R * S_user)
    N = int(lens.sum())
    x['fea'] = rng.integers(-8, 9, size=(N, R)).astype(np.float32)
    x['Phi'] = np.ones(R, dtype=np.float32)
    g = np.zeros((N, S_user), dtype=np.float32)
    off = x['offsets']
    for b in range(len(lens)):
        lo, hi = off[b], off[b + 1]
        g[np.arange(lo, hi), rng.integers(0, x['ns'][b], size=hi - lo)] = 1.0
    x['gamma0'] = g
    out = run_device(x, gemm=gemm, fb_split=1 if S_user > 64 else 0)
    assert np.array_equal(out['rho'], x['fea'])
    FaFb = np.float32(FA / FB)
    for b in range(len(lens)):
        lo, hi, n = off[b], off[b + 1], x['ns'][b]
        if hi == lo:
            continue
        Sig = g[lo:hi, :n].astype(np.float64).T @ x['fea'][lo:hi].astype(np.float64)
        want = ((FaFb * out['invL'][b, :n]).astype(np.float32).astype(np.float64) * Sig).astype(np.float32)
        bad = np.argwhere(out['alpha'][b, :n] != want)
        assert bad.size == 0, f'recording {b} (T = {hi - lo}): alpha differs at (state, r) {bad[:5].tolist()}'


# ---- stage 2 ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('S_user,fb', [(13, 2), (13, 1), (50, 2), (50, 1), (100, 1)],
                         ids=['S16-fused', 'S16-split', 'S64-fused', 'S64-split', 'S128-split'])
def test_loglik(S_user, fb, gemm):
    x = inputs(edge_lengths(), 128, S_user, seed=S_user + fb)
    warm = warm_model(x, seed=S_user)
    ref, keep = oracle(x, 1, 0.0, warm=warm)
    out = run_device(x, gemm=gemm, fb_split=fb, loopProb=0.0, warm=warm)
    check_loglik(x, out, warm, ref, keep, f'S={S_user} fb_split={fb} gemm={gemm}')


# ---- stage 3 ------------------------------------------------------------------------------------------------------
SCHEDULES = {'split': (16, dict(fb_split=1), ()),
             'burst': (16, dict(fb_split=2, ring=0), ()),
             'burst-T2049': (8, dict(fb_split=2), (2049,)),
             'chunked': (16, dict(fb_split=2), (4095, 4096, 4097, 4351, 4352, 4353)),
             'split-S128': (100, dict(fb_split=1), ())}
SCHEDULES.update({f'ring-S{s}-spl{l}': (s, dict(fb_split=2, spl=l), ()) for s, l in VARIANTS})


@pytest.mark.parametrize('name', list(SCHEDULES))
def test_forward_backward_schedule(name):
    S_user, opts, extra = SCHEDULES[name]
    x = inputs(edge_lengths(extra), 128, S_user, seed=len(name) * 31 + S_user)
    warm = mstep_model(x)
    long_rec = x['lens'] >= 4096
    for lp in (0.35, 0.99):
        for iters in (1, 2):
            ref, keep = oracle(x, iters, lp, warm=warm)
            kw = dict(maxIters=iters, loopProb=lp, warm=warm)
            out = run_device(x, **opts, **kw)
            eg, ep = gamma_error(x, out, ref, keep)
            msg = f'{name} loopProb={lp} maxIters={iters}: max |dgamma| {eg:.3g}, |dpi| {ep:.3g}'
            if S_user <= 64:        # the classic sweep is a fused-schedule sweep: there is none at S = 128
                base = run_device(x, fb_split=2, classic=1, spl=opts.get('spl', 0), **kw)
                eb, _ = gamma_error(x, base, ref, keep, only=~long_rec)
                if long_rec.any():  # the fused sweeps hand recordings of >= 4096 frames to the chunked scan: the split
                    sp = run_device(x, fb_split=1, **kw)          # sweep is the plain yardstick there
                    eb = max(eb, gamma_error(x, sp, ref, keep, only=long_rec)[0])
                msg += f', classic {eb:.3g} (ratio {eg / max(eb, 1e-30):.3g})'
                assert eg <= FB_FACTOR * eb + FB_FLOOR, msg
            print(msg)
            assert eg <= G_TOL and ep <= G_TOL, msg


# ---- feature widths -----------------------------------------------------------------------------------------------
WIDTHS = [4, 8, 12, 20, 24, 36, 52, 100, 124, 128]


@pytest.mark.parametrize('S_user', [4, 16, 64, 100], ids=['S4', 'S16', 'S64', 'S128'])
@pytest.mark.parametrize('R', WIDTHS)
def test_feature_widths(R, S_user):
    """Stages 1-3 at every width class of the contraction kernels (R = 4 (mod 8) meets the clamped columns and the zero
    fragments), both gemm modes and both schedules."""
    lens = np.array([1, 2, 3, 0, 17, 65, 513, 300, 1025, 64], dtype=np.int64)
    x = inputs(lens, R, S_user, seed=R * 7 + S_user)
    warm = warm_model(x, seed=R)
    ref2, keep = oracle(x, 1, 0.0, warm=warm)
    ref3, _ = oracle(x, 2, 0.99, warm=mstep_model(x))
    for gemm in (0, 1):
        for fb in ((1,) if S_user > 64 else (2, 1)):
            tag = f'R={R} S={S_user} gemm={gemm} fb_split={fb}'
            check_mstep(x, run_device(x, gemm=gemm, fb_split=fb), tag)
            check_loglik(x, run_device(x, gemm=gemm, fb_split=fb, loopProb=0.0, warm=warm), warm, ref2, keep, tag)
            eg, ep = gamma_error(x, run_device(x, gemm=gemm, fb_split=fb, maxIters=2, warm=mstep_model(x)), ref3, keep)
            assert eg <= G_TOL and ep <= G_TOL, (tag, eg, ep)


@pytest.mark.parametrize('R', [12, 52])
def test_float64_finishing_at_narrow_widths(R):
    """With a finite epsilon recordings hand over to the float64 kernels at different iterations; at R != 128 they stop
    where the float64 oracle stops."""
    lens = np.random.default_rng(R).integers(40, 700, size=14)
    lens[3] = 0
    x = inputs(lens, R, 8, seed=R + 5)
    ref, keep = oracle(x, 25, 0.99, epsilon=1e-5)
    assert len(set(ref['n_iters'].tolist())) > 1 and (ref['n_iters'] < 25).any()
    for fb in (2, 1):
        for gemm in (0, 1):
            out = run_device(x, gemm=gemm, fb_split=fb, maxIters=25, epsilon=1e-5)
            assert np.array_equal(out['n_iters'][keep], ref['n_iters']), (fb, gemm, out['n_iters'][keep], ref['n_iters'])
            eg, ep = gamma_error(x, out, ref, keep)
            assert eg <= G_TOL and ep <= G_TOL, (fb, gemm, eg, ep)


# ---- the benchmark's configuration at test size -------------------------------------------------------------------
@pytest.mark.parametrize('tmax', [2048, 3000], ids=['ring', 'register-burst'])
def test_benchmark_configuration(tmax):
    """Two sub-batches of 1100 recordings on the fused schedule: each half runs its sweep on the high-priority side stream
    (>= 1024 recordings), ordered by events against the snapshot, the float64 finishing round and the next M-step.
    epsilon = 1e-6 makes recordings switch to float64 at different iterations.  Results equal one whole batch and
    sampled recordings run alone bit for bit, and the samples stop where the oracle stops."""
    from vbx_b200.batch import VbxBatch
    from vbx_b200.parts import PartitionedBatch, make_batch
    rng = np.random.default_rng(tmax)
    B, S = 2200, 16
    lens = rng.integers(1, 300, size=B)
    lens[::97] = rng.integers(1500, tmax + 1, size=len(lens[::97]))
    lens[5], lens[1500] = tmax, tmax - 1
    ns = rng.integers(9, S + 1, size=B).astype(np.int32)
    d = synth.make_batch(lens, R=128, S=S, seed=tmax + 1, dtype=np.float32)
    g0 = d['gamma0'].astype(np.float32)
    pi0 = np.zeros((B, S), dtype=np.float32)
    for b in range(B):
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        g0[lo:hi, ns[b]:] = 0
        g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
        pi0[b, :ns[b]] = 1.0 / ns[b]
    kw = dict(Fa=FA, Fb=FB, loopProb=0.99, maxIters=20, epsilon=1e-6)

    def run(vb, sl=slice(None), rs=slice(None)):
        g, p = cuda(g0[sl]), cuda(pi0[rs])
        vb.prepare_scale(cuda(d['fea'][sl]), cuda(d['Phi']))
        o = vb.run(g, p, **kw)
        torch.cuda.synchronize()
        res = [t.cpu().numpy() for t in (g, p, o['Li'], o['n_iters'], o['flags'])]
        vb.close()
        return res

    whole = {}
    for parts in (1, 2):
        vb = make_batch(lens, 128, ns, device=dev(), parts=parts, fb_split=2)
        if parts == 2:
            assert isinstance(vb, PartitionedBatch) and min(c.B for c in vb.children) >= 1024
        whole[parts] = run(vb)
    for a, b in zip(whole[1], whole[2]):
        assert np.array_equal(a, b, equal_nan=True)
    n_iters = whole[1][3]
    assert len(set(n_iters.tolist())) > 2 and (n_iters < 20).any()
    off = d['offsets']
    sample = [5, 1500] + rng.choice(B, 5, replace=False).tolist()
    for b in sample:
        lo, hi = off[b], off[b + 1]
        alone = run(VbxBatch([lens[b]], 128, ns[b:b + 1], device=dev(), fb_split=2), slice(lo, hi), slice(b, b + 1))
        for a, w in zip(alone, (whole[1][0][lo:hi], whole[1][1][b:b + 1], whole[1][2][b:b + 1], n_iters[b:b + 1],
                                whole[1][4][b:b + 1])):
            assert np.array_equal(a, w, equal_nan=True), f'recording {b} alone differs from the batch'
        ref = co.vbx_oracle_batch(d['fea'][lo:hi], d['Phi'], np.array([0, hi - lo]), g0[lo:hi], pi0[b:b + 1], FA, FB, 0.99,
                                  20, 1e-6, n_states=ns[b:b + 1])
        assert int(ref['n_iters'][0]) == int(n_iters[b]), (b, ref['n_iters'], n_iters[b])
        assert np.abs(whole[1][0][lo:hi] - ref['gamma']).max() <= G_TOL


# ---- alignment ----------------------------------------------------------------------------------------------------
def test_misaligned_arrays_are_refused():
    """rho and gamma are read and written with 16-byte vectors: an address off that grid (a view with a storage offset,
    which passes is_contiguous()) is refused by the C entry before anything is launched."""
    from vbx_b200 import VbxError
    from vbx_b200.batch import VbxBatch
    x = inputs([40, 24], 128, 4, seed=3)
    vb = VbxBatch(x['lens'], 128, 4, device=dev())
    N, S, R, B = vb.N, vb.S, vb.R, vb.B
    lib, h = vb.lib, vb._h
    P = lambda t, shift=0: ctypes.c_void_p(t.data_ptr() + shift)
    fea, Phi = cuda(x['fea']), cuda(x['Phi'])
    # shifted views with room behind them: nothing outside an allocation is named even by a refused call
    fbuf = torch.zeros(N * R + 4, device=dev())
    gbuf = torch.zeros(N * S + 4, device=dev())
    p = torch.zeros((B, S), device=dev())
    Li = torch.empty((B, 2), dtype=torch.float64, device=dev())
    ni = torch.empty(B, dtype=torch.int32, device=dev())
    fl = torch.empty(B, dtype=torch.int32, device=dev())
    st = vb._stream()
    for shift in (4, 8):
        assert lib.vbx_prepare_scale(h, P(fbuf, shift), P(Phi), P(fbuf), st) == -1
        assert b'fea must be 16-byte aligned' in lib.vbx_last_error(h)
        assert lib.vbx_prepare_scale(h, P(fea), P(Phi), P(fbuf, shift), st) == -1
        assert b'rho_out must be 16-byte aligned' in lib.vbx_last_error(h)
    rho = vb.prepare_scale(fea, Phi)
    for shift in (4, 8, 12):
        assert lib.vbx_run(h, P(fbuf, shift), P(Phi), P(gbuf), P(p), None, FA, FB, 0.9, 2, -np.inf, None, None, 0, P(Li), P(ni),
                           P(fl), st) == -1
        assert b'rho must be 16-byte aligned' in lib.vbx_last_error(h)
        assert lib.vbx_run(h, P(rho), P(Phi), P(gbuf, shift), P(p), None, FA, FB, 0.9, 2, -np.inf, None, None, 0, P(Li), P(ni),
                           P(fl), st) == -1
        assert b'gamma_io must be 16-byte aligned' in lib.vbx_last_error(h)
        hyper = torch.full((3, B), 0.5, dtype=torch.float64, device=dev())
        assert lib.vbx_run_per_recording(h, P(rho), P(Phi), P(gbuf, shift), P(p), None, P(hyper[0]), P(hyper[1]), P(hyper[2]), 2,
                                         -np.inf, None, None, 0, P(Li), P(ni), P(fl), st) == -1
        assert b'gamma_io must be 16-byte aligned' in lib.vbx_last_error(h)
        lab = torch.empty(N, dtype=torch.int32, device=dev())
        assert lib.vbx_hard_labels(h, P(gbuf, shift), None, P(lab), None, st) == -1
        assert b'gamma must be 16-byte aligned' in lib.vbx_last_error(h)
        keep = torch.ones(B, dtype=torch.int32, device=dev())
        mass = torch.empty((B, S), dtype=torch.float64, device=dev())
        assert lib.vbx_hard_labels_keep(h, P(gbuf, shift), None, P(keep), P(lab), P(lab), P(mass), st) == -1
        assert b'gamma must be 16-byte aligned' in lib.vbx_last_error(h)
    # through the Python API: a contiguous view that starts one float into its storage
    g = gbuf[1:1 + N * S].view(N, S)
    assert g.is_contiguous()
    with pytest.raises(VbxError, match='16-byte aligned'):
        vb.run(g, p, maxIters=2)
    # the handle stays usable: an aligned call afterwards runs
    g = torch.zeros((N, S), device=dev())
    g[:, :4] = cuda(x['gamma0'])
    p[:] = 0.25
    out = vb.run(g, p, Fa=FA, Fb=FB, maxIters=2, epsilon=-np.inf)
    torch.cuda.synchronize()
    assert int(out['n_iters'].min()) == 2
    vb.close()
