"""The float64 finishing round (vbx_exact64.cu) against a float64 emulation, one hand-over at a time, at every state tier,
tile edge and feature width (DESIGN.md section 3).

A recording's fate under a finite epsilon is decided by elbo_kernel from float32 ELBO values alone, and a run with
epsilon = -inf executes the same float32 iterations bit for bit.  So the -inf trace predicts, for any epsilon, whether a
recording keeps going, stops at iteration j, or hands over at iteration k (d_k inside [eps - 4 nb, eps + 16 nb)), and the
state the finishing round restores -- the one that entered iteration k - 1 -- is the output of a -inf run with
maxIters = k - 1.  From that state tests/test_stop_rule_math.py's finish64 emulates the finishing round in numpy
float64 with the kernels' storage points (device rho and G, gamma float32 between rounds, pi float32 at the restore and
float64 after, the forward variables parked in float32), and the device must agree:

  * recordings that never hand over: bit-identical to the -inf run truncated where they stop;
  * a handed-over recording: Li[0 .. k-2] bit-identical to the float32 trace, the first float64 ELBO to rtol 1e-13 and
    later ones to 1e-11 (a 1-ulp flip of a stored gamma value propagates), gamma, pi, alpha and invL within one float32
    ulp of the emulation's rounding, n_iters and flags exact where the emulated step is >= 1e-9 from epsilon (and, for the
    'ELBO decreased' flag, from 0), Li NaN past n_iters.

epsilon is placed on purpose: eps = d_k - 2 nb_k hands recording b over at iteration k (after checking that its earlier
steps stay above eps + 16 nb_j).  Every non-empty recording is handed over at k = 1 (the state is the exact inputs) and at
a later k wherever its trace allows one, and each case asserts that all of these hand-overs happened; the recipes' 1e-4
and 1e-6 run as well.  Predictions within 1e-12 relative of a threshold are skipped (nvcc may contract
the threshold into an FMA).  Every batch holds T = 1, 2, 3, empty recordings first, mid-batch and last, the 64-frame
blocks' 31 / 32 / 33 and 63 / 64 / 65, the 512-frame M-tiles' 511 / 512 / 513 and 1023 / 1024 / 1025, dead columns and a
recording with one live state; the workspace is poisoned with 0xFF and gamma is followed by NaN guard rows.

The float64 mode (vbx_run_f64) at its layout limits is tested in test_f64_mode_gpu.py."""
import numpy as np
import pytest
import torch

from test_em_stages_gpu import GUARD, cuda, dev, inputs, mstep_model
from test_enroll_prior_gpu import make_prior
from test_stop_rule_math import GUARD as GUARD_MULT
from test_stop_rule_math import NOISE_C, SAFE_STOP, f32, f64, finish64

pytestmark = pytest.mark.gpu
FA, FB, LOOP = 0.3, 17.0, 0.99
EDGES = [0, 1, 2, 3, 31, 32, 33, 0, 63, 64, 65, 511, 512, 513, 1023, 1024, 1025]
LONG = [4095, 4096, 4097]         # the fused schedule's chunked float32 sweep, then the sequential float64 one
LI_FIRST, LI_LATER, STEP_MARGIN = 1e-13, 1e-11, 1e-9


def batch(S_user, R, seed, long=False):
    lens = np.array(EDGES + (LONG if long else []) + [0], dtype=np.int64)
    x = inputs(lens, R, S_user, seed)
    b1 = 9                        # T = 64: one live state
    lo, hi = x['offsets'][b1], x['offsets'][b1 + 1]
    x['ns'][b1] = 1
    x['gamma0'][lo:hi] = 0
    x['gamma0'][lo:hi, 0] = 1
    x['pi0'][b1] = 0
    x['pi0'][b1, 0] = 1
    return x


def device_run(x, maxIters, eps, fb_split=0, gemm=0, hyper=None, warm=None, prior=None, parts=1, graph=None):
    """One run over the batch with the guards checked; numpy results (S_user columns) plus rho and G of the device."""
    from vbx_b200.parts import make_batch
    lens, ns, S_user, R = x['lens'], x['ns'], x['S_user'], x['R']
    vb = make_batch(lens, R, ns, device=dev(), parts=parts, fb_split=fb_split)
    for c in getattr(vb, 'children', [vb]):
        c.workspace.fill_(0xFF)   # NaN in float32 and float64: nothing may be read before it is written
    vb.set_option('gemm', gemm)
    if graph is not None:
        vb.set_option('graph', graph)
    S, N, B = vb.S, vb.N, vb.B
    buf = torch.full((N + GUARD, S), float('nan'), device=dev())
    g, p = buf[:N], torch.zeros((B, S), device=dev())
    rho = vb.prepare_scale(cuda(x['fea']), cuda(x['Phi']))
    hp = dict(Fa=FA, Fb=FB, loopProb=LOOP) if hyper is None else {k: cuda(v, torch.float64) for k, v in hyper.items()}
    kw = dict(maxIters=maxIters, epsilon=eps, return_model=True, **hp)
    if prior is not None:
        kw['prior'] = tuple(cuda(np.pad(v, [(0, 0), (0, S - S_user)] + [(0, 0)] * (v.ndim - 2)), torch.float64)
                            for v in prior)
    if warm is not None:
        a, il = torch.zeros((B, S, R), device=dev()), torch.zeros((B, S, R), device=dev())
        kw.update(alpha=a, invL=il, warm_start=True)
    calls = 3 if graph == 1 else 1            # graph: call 0 runs directly, call 1 is captured, call 2 replays
    if graph == 1:
        kw['buffers'] = vb.output_buffers(maxIters)
    for _ in range(calls):
        g.zero_()
        g[:, :S_user] = cuda(x['gamma0'])
        p.zero_()
        p[:, :S_user] = cuda(x['pi0'])
        if warm is not None:
            kw['alpha'].zero_()
            kw['invL'].zero_()
            kw['alpha'][:, :S_user] = cuda(warm[0])
            kw['invL'][:, :S_user] = cuda(warm[1])
        out = vb.run(g, p, **kw)
        torch.cuda.synchronize()
    assert bool(torch.isnan(buf[N:]).all()), 'gamma written past its last row'
    gam = g.cpu().numpy()
    res = dict(gamma=gam[:, :S_user], pi=p[:, :S_user].cpu().numpy(), Li=out['Li'].cpu().numpy(),
               n_iters=out['n_iters'].cpu().numpy(), flags=out['flags'].cpu().numpy(),
               alpha=out['alpha'][:, :S_user].cpu().numpy(), invL=out['invL'][:, :S_user].cpu().numpy())
    if parts == 1:
        res.update(rho=rho.cpu().numpy(), gsum=vb.g_sum().cpu().numpy())
    vb.close()
    off = x['offsets']
    for b in range(B):
        assert np.all(gam[off[b]:off[b + 1], ns[b]:] == 0), f'recording {b}: a dead or padded column of gamma is not 0'
        n = int(res['n_iters'][b])
        assert np.all(np.isnan(res['Li'][b, n:])) and np.all(np.isfinite(res['Li'][b, :n])), (b, n, res['Li'][b])
        assert x['lens'][b] > 0 or n == 0, f'empty recording {b} ran {n} iterations'
    return res


def near(a, b):
    return abs(a - b) <= 1e-12 * max(abs(a), abs(b), 1e-300)


def predict(Li, M, eps, warm):
    """Fate of one recording under epsilon from its float32 trace Li [M] (elbo_kernel's decision):
    ('run', M) | ('stop', j) | ('hand', k, fresh) | None (too close to a threshold to tell)."""
    for k in range(1, M):
        d, nb = Li[k] - Li[k - 1], NOISE_C * 2.0 ** -24 * abs(Li[k])
        hi, lo = eps + GUARD_MULT * nb, eps - SAFE_STOP * nb
        if near(d, hi) or near(d, lo):
            return None
        if d >= hi:
            continue
        if d < lo:
            return ('stop', k + 1)
        if warm and k == 1:
            if near(d, eps + 4.0 * nb):
                return None
            return ('hand', 1, 1 if d >= eps + 4.0 * nb else 2)
        return ('hand', k, 1)
    return ('run', M)


def targets(Li32, lens, M, warm):
    """Placed epsilons as (key, eps): key = (recording, phase, fresh) of the hand-over eps = d_k - 2 nb_k causes.  Every
    non-empty recording at k = 1 first (warm: both fresh branches, the second with eps = d_1 - 10 nb_1), then at a later k
    wherever the trace allows one (a positive step whose earlier steps all stay above eps + 16 nb_j)."""
    first, later = [], []
    for b in np.flatnonzero(lens > 0):
        L = Li32[b]
        nb = NOISE_C * 2.0 ** -24 * np.abs(L)
        d = np.diff(L)
        first.append(((b, 'k=1', 2 if warm else 1), d[0] - 2 * nb[1]))
        if warm:
            first.append(((b, 'k=1', 1), d[0] - 10 * nb[1]))
        ks = [k for k in range(2, M - 1) if d[k - 1] > 0 and all(d[j - 1] >= d[k - 1] + 16 * nb[j] for j in range(1, k))]
        if ks:
            k = ks[len(ks) // 2]
            later.append(((b, 'k>1', 1), d[k - 1] - 2 * nb[k]))
    return first + later


def ulp_ok(got, want, tag, flips):
    """got (float32, device) within one float32 ulp of f32(want); counts the values that differ."""
    w = np.asarray(want, dtype=f64).astype(f32)
    diff = np.abs(got.astype(f64) - w.astype(f64))
    tol = np.spacing(np.abs(w)).astype(f64)
    assert np.all(diff <= tol), f'{tag}: {int((diff > tol).sum())} values more than one float32 ulp off, max {diff.max():.3g}'
    flips[0] += int((diff > 0).sum())
    flips[1] += diff.size


class Finishing:
    """One batch and its option set, with the -inf runs it needs cached by maxIters."""

    def __init__(self, x, M, warm=None, hyper=None, prior=None, **opts):
        self.x, self.M, self.warm, self.hyper, self.prior, self.opts = x, M, warm, hyper, prior, opts
        self.runs = {}
        self.ref = self.f32_run(M)
        self.stats = dict(li_first=0.0, li_later=0.0, flips=[0, 0], hand=set(), n=0)

    def run(self, maxIters, eps, **kw):
        return device_run(self.x, maxIters, eps, warm=self.warm, hyper=self.hyper, prior=self.prior, **self.opts, **kw)

    def f32_run(self, m):
        if m not in self.runs:
            self.runs[m] = self.run(m, -np.inf)
        return self.runs[m]

    def entering(self, k):
        """gamma, pi entering iteration k (the snapshot the restore reads)."""
        if k == 0:
            return self.x['gamma0'], self.x['pi0']
        r = self.f32_run(k)
        return r['gamma'], r['pi']

    def hp(self, b):
        if self.hyper is None:
            return FA, FB, LOOP
        return tuple(float(self.hyper[k][b]) for k in ('Fa', 'Fb', 'loopProb'))

    def check(self, eps):
        x, M, ref = self.x, self.M, self.ref
        out = self.run(M, eps)
        off, ns, lens = x['offsets'], x['ns'], x['lens']
        for b in range(len(lens)):
            lo, hi, n = off[b], off[b + 1], ns[b]
            if hi == lo:
                assert out['n_iters'][b] == 0
                continue
            fate = predict(ref['Li'][b], M, eps, self.warm is not None)
            if fate is None:
                continue
            tag = f'eps={eps!r} recording {b} (T={hi - lo}, {n} states) {fate}'
            if fate[0] != 'hand':
                j = fate[1]
                tr = self.f32_run(j)
                assert out['n_iters'][b] == j, tag
                assert np.array_equal(out['Li'][b, :j], ref['Li'][b, :j]), tag
                d = ref['Li'][b, j - 1] - ref['Li'][b, j - 2] if j > 1 else 0.0
                want_fl = (4 if j < M else 0) | (2 if j > 1 and d < 0 and fate[0] == 'stop' else 0)
                assert out['flags'][b] == want_fl, (tag, out['flags'][b], want_fl)
                for k in ('gamma', 'alpha', 'invL'):
                    sl = slice(lo, hi) if k == 'gamma' else b
                    assert np.array_equal(out[k][sl], tr[k][sl]), (tag, k)
                assert np.array_equal(out['pi'][b], tr['pi'][b]), tag
                continue
            _, k, fresh = fate
            first = 1 if (self.warm is not None and k == 1) else k - 1
            g_in, p_in = self.entering(first)
            Fa, Fb, P = self.hp(b)
            pr = None if self.prior is None else (self.prior[0][b, :n], self.prior[1][b, :n])
            em = finish64(ref['rho'][lo:hi], float(ref['gsum'][b]), x['Phi'], g_in[lo:hi, :n], p_in[b, :n], Fa, Fb, P,
                          first, M, eps, fresh=fresh, prev=ref['Li'][b, 0], prior=pr)
            self.stats['hand'].add((b, 'k=1' if k == 1 else 'k>1', fresh))
            self.stats['n'] += 1
            assert np.array_equal(out['Li'][b, :first], ref['Li'][b, :first]), f'{tag}: the float32 part of Li changed'
            ni = int(out['n_iters'][b])
            if em['margin'] >= STEP_MARGIN:
                assert ni == em['n_iters'], (tag, ni, em['n_iters'])
                # flag 2 (the step was negative) is exact where the last step is >= 1e-9 from 0: a converged short
                # recording's step can be a few ulps of the ELBO either side of 0
                mask = 7 if abs(em['last_step']) >= STEP_MARGIN else 5
                assert out['flags'][b] & mask == em['flags'] & mask, (tag, out['flags'][b], em['flags'])
            if ni != em['n_iters']:
                continue
            got = out['Li'][b, first:ni]
            rel = np.abs(got - np.array(em['Li'])) / np.abs(np.array(em['Li']))
            self.stats['li_first'] = max(self.stats['li_first'], rel[0])
            assert rel[0] <= LI_FIRST, (tag, rel[0])
            if len(rel) > 1:
                self.stats['li_later'] = max(self.stats['li_later'], rel[1:].max())
                assert rel[1:].max() <= LI_LATER, (tag, rel)
            fl = self.stats['flips']
            ulp_ok(out['gamma'][lo:hi, :n], em['gamma'], tag + ' gamma', fl)
            ulp_ok(out['pi'][b, :n], em['pi'], tag + ' pi', fl)
            ulp_ok(out['alpha'][b, :n], em['alpha'], tag + ' alpha', fl)
            ulp_ok(out['invL'][b, :n], em['invL'], tag + ' invL', fl)
            assert np.all(out['alpha'][b, n:] == 0) and np.all(out['invL'][b, n:] == 0), tag

    def sweep(self, extra=(1e-4, 1e-6)):
        """The recipes' epsilons, then a placed one for every hand-over of `targets` that no earlier run produced; every
        one of them must have happened."""
        for eps in extra:
            self.check(eps)
        want = targets(self.ref['Li'], self.x['lens'], self.M, self.warm is not None)
        for key, eps in want:
            if key not in self.stats['hand']:
                self.check(float(eps))
        s, lens = self.stats, self.x['lens']
        missing = [(int(lens[k[0]]),) + k[1:] for k, _ in want if k not in s['hand']]
        assert not missing, f'placed hand-overs that did not happen (T, phase, fresh): {missing}'
        for phase in ('k=1', 'k>1'):
            print(f'handed over at {phase}: T = {sorted({int(lens[h[0]]) for h in s["hand"] if h[1] == phase})}')
        print(f'{s["n"]} hand-overs ({len(s["hand"])} recording / phase / fresh kinds): Li rel err first {s["li_first"]:.3g}, '
              f'later {s["li_later"]:.3g}; {s["flips"][0]} of {s["flips"][1]} float32 values off by one ulp')
        return s


# ---- every state tier, feature width and schedule ---------------------------------------------------------------------
TIERS = {  # id: (S_user, R, fb_split, gemm, long recordings)
    'S3-R4': (3, 4, 2, 0, False),
    'S4-R12-split': (4, 12, 1, 1, False),
    'S7-R52': (7, 52, 2, 1, True),
    'S8-R100-split': (8, 100, 1, 0, False),
    'S16-R128': (16, 128, 2, 0, False),
    'S31-R12-split': (31, 12, 1, 0, False),
    'S33-R128': (33, 128, 2, 1, True),
    'S64-R52-split': (64, 52, 1, 1, False),
    'S100-R128': (100, 128, 1, 0, False),
    'S100-R4': (100, 4, 1, 1, False),
}


@pytest.mark.parametrize('tier', list(TIERS))
def test_finishing_round(tier):
    S_user, R, fb, gemm, long = TIERS[tier]
    x = batch(S_user, R, seed=S_user * 7 + R, long=long)
    s = Finishing(x, 12, fb_split=fb, gemm=gemm).sweep()
    assert {b for b, p, _ in s['hand'] if p == 'k=1'} == set(np.flatnonzero(x['lens'] > 0)), s['hand']
    assert {int(x['lens'][b]) for b, p, _ in s['hand'] if p == 'k>1'} >= {511, 512, 513, 1023, 1024, 1025}, s['hand']


def test_per_recording_hyperparameters():
    x = batch(16, 128, seed=5)
    B = len(x['lens'])
    rec = [(0.3, 17.0, 0.99), (0.4, 64.0, 0.65), (0.2, 6.0, 0.35), (0.4, 17.0, 0.40)]
    hyper = {k: np.array([rec[b % 4][i] for b in range(B)]) for i, k in enumerate(('Fa', 'Fb', 'loopProb'))}
    Finishing(x, 12, hyper=hyper, fb_split=2).sweep()


@pytest.mark.parametrize('S_user,fb', [(8, 2), (100, 1)])
def test_warm_start_hands_over_at_iteration_1(S_user, fb):
    """A warm start cannot redo iteration 0: iteration 1 alone is redone, tested against the float32 ELBO of iteration 0
    when it was within float32 noise of epsilon (fresh = 2) and not tested otherwise (fresh = 1)."""
    x = batch(S_user, 128, seed=S_user + 3)
    s = Finishing(x, 10, warm=mstep_model(x), fb_split=fb).sweep()
    assert {f for _, p, f in s['hand'] if p == 'k=1'} == {1, 2}, s['hand']


@pytest.mark.parametrize('S_user,R,fb', [(4, 128, 2), (33, 52, 1), (100, 128, 1)])
def test_enrolment_prior(S_user, R, fb):
    x = batch(S_user, R, seed=S_user + R)
    keep = x['lens'] > 0
    d = dict(fea=x['fea'], offsets=np.concatenate([[0], np.cumsum(x['lens'][keep])]))
    pn_k, pF_k = make_prior(d, S_user, S_user, R, seed=S_user)      # the second non-empty recording has no prior
    pn, pF = np.zeros((len(keep), S_user)), np.zeros((len(keep), S_user, R))
    pn[keep], pF[keep] = pn_k, pF_k
    for b, n in enumerate(x['ns']):
        pn[b, n:], pF[b, n:] = 0, 0
    Finishing(x, 12, prior=(pn, pF), fb_split=fb).sweep()


def test_partitioned_batch_and_graph_replay():
    """A two-part batch and a graph replay give the whole batch's bits, with recordings handing over at different
    iterations (warp-mates of fb64 in different phases and of different lengths)."""
    x = batch(16, 128, seed=11)
    f = Finishing(x, 12, fb_split=1)
    t = [eps for key, eps in targets(f.ref['Li'], x['lens'], 12, False) if key[1] == 'k>1']
    for eps in (1e-6, t[len(t) // 2]):
        whole = f.run(12, eps)
        hand = [b for b in range(len(x['lens'])) if (predict(f.ref['Li'][b], 12, eps, False) or ('',))[0] == 'hand']
        assert hand, eps
        for kw in (dict(parts=2), dict(graph=1)):
            got = f.run(12, eps, **kw)
            for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags', 'alpha', 'invL'):
                assert np.array_equal(got[k], whole[k], equal_nan=True), (kw, k)
