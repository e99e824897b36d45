"""The float64 mode (vbx_run_f64, the drop-in's default) at its layout limits against the float64 oracles, at the bars of
test_parity_gpu.py::test_float64_mode_matches_reference_tightly (gamma 1e-7, pi 1e-8, Li rtol 1e-9, alpha 1e-7, invL
1e-9, identical iteration counts):

  * states: S = 1, 2, 31 / 32 / 33 (fb_kernel_small's one / two states per lane), 63 / 64 / 65 (the switch to fb_kernel),
    877 / 878 (the sweep's 7 S doubles pass 48 KB of shared memory) and 3600, the plan's limit; 3601 is refused;
  * widths: R = 1, 3, 127, 128, 129, 256;
  * ragged batches with empty recordings first, mid-batch and last (loglik_kernel's binary search over the offsets) and
    per-recording n_states down to 1;
  * the enrolment prior against oracle/prior_oracle.py at the same bars.
T stays small at large S so that the oracles run in seconds."""
import numpy as np
import pytest
import torch

from oracle import c_oracle, prior_oracle
from vbx_b200 import synth

pytestmark = pytest.mark.gpu
FA, FB, LOOP, ITERS = 0.3, 17.0, 0.99, 5
WIDTHS = [1, 3, 127, 128, 129, 256]
STATES = [1, 2, 31, 32, 33, 63, 64, 65, 877, 878, 3600]


def dev():
    return torch.device('cuda:0')


def case(S, R, seed):
    rng = np.random.default_rng(seed)
    lens = np.array([0, 1, 37, 0, 2, 64, 65, 0] if S <= 65 else [0, 1, 9, 0, 6, 0], dtype=np.int64)
    B, N = len(lens), int(lens.sum())
    ns = rng.integers(1, S + 1, size=B).astype(np.int32)
    ns[1], ns[2], ns[-2] = 1, S, max(1, S // 2)
    Phi = synth.plda_phi(R) if R > 1 else np.array([2.5])
    spk = rng.standard_normal((4, R)) * np.sqrt(Phi)[None, :]
    fea = spk[rng.integers(0, 4, size=N)] + rng.standard_normal((N, R))
    off = np.concatenate([[0], np.cumsum(lens)])
    gamma0, pi0 = np.zeros((N, S)), np.zeros((B, S))
    for b in range(B):
        lo, hi, n = off[b], off[b + 1], ns[b]
        gamma0[lo:hi, :n] = rng.dirichlet(np.ones(n), size=hi - lo)
        pi0[b, :n] = 1.0 / n
    return dict(lens=lens, ns=ns, fea=fea, Phi=Phi, gamma0=gamma0, pi0=pi0, off=off, S=S, R=R)


def run_gpu(x, prior=None):
    from vbx_b200.batch import VbxBatch, run_f64
    vb = VbxBatch(x['lens'], x['R'], x['ns'], device=dev(), f64_only=True)
    assert vb.S == x['S']
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev())
    g, p = c(x['gamma0']), c(x['pi0'])
    pr = None if prior is None else (c(prior[0]), c(prior[1]))
    out = run_f64(vb, c(x['fea']), c(x['Phi']), g, p, Fa=FA, Fb=FB, loopProb=LOOP, maxIters=ITERS, epsilon=-np.inf,
                  return_model=True, prior=pr)
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    vb.close()
    return res


def check(x, out, refs):
    """refs[b]: (gamma, pi, Li, alpha, invL) of recording b's live states, None for an empty recording."""
    off, ns = x['off'], x['ns']
    for b, ref in enumerate(refs):
        lo, hi, n = off[b], off[b + 1], ns[b]
        if ref is None:
            assert out['n_iters'][b] == 0 and np.all(np.isnan(out['Li'][b]))
            continue
        g, pi, Li, alpha, invL = ref
        tag = f'recording {b} (T={hi - lo}, {n} of {x["S"]} states, R={x["R"]})'
        assert out['n_iters'][b] == len(Li), tag
        np.testing.assert_allclose(out['gamma'][lo:hi, :n], g, rtol=0, atol=1e-7, err_msg=tag)
        np.testing.assert_allclose(out['pi'][b, :n], pi, rtol=0, atol=1e-8, err_msg=tag)
        np.testing.assert_allclose(out['Li'][b, :len(Li)], Li, rtol=1e-9, err_msg=tag)
        np.testing.assert_allclose(out['alpha'][b, :n], alpha, rtol=0, atol=1e-7, err_msg=tag)
        np.testing.assert_allclose(out['invL'][b, :n], invL, rtol=0, atol=1e-9, err_msg=tag)
        assert np.all(out['gamma'][lo:hi, n:] == 0) and np.all(out['pi'][b, n:] == 0), tag


def oracle_refs(x):
    keep = x['lens'] > 0
    ko = np.concatenate([[0], np.cumsum(x['lens'][keep])])
    r = c_oracle.vbx_oracle_batch(x['fea'], x['Phi'], ko, x['gamma0'], x['pi0'][keep], FA, FB, LOOP, ITERS, -np.inf,
                                  n_states=x['ns'][keep])
    refs, k = [], 0
    for b in range(len(x['lens'])):
        if not keep[b]:
            refs.append(None)
            continue
        n = x['ns'][b]
        refs.append((r['gamma'][ko[k]:ko[k + 1], :n], r['pi'][k, :n], r['Li'][k, :r['n_iters'][k]], r['alpha'][k, :n],
                     r['invL'][k, :n]))
        k += 1
    return refs


@pytest.mark.parametrize('S', STATES)
def test_states(S):
    x = case(S, WIDTHS[STATES.index(S) % len(WIDTHS)], seed=S)
    check(x, run_gpu(x), oracle_refs(x))


@pytest.mark.parametrize('R', WIDTHS)
def test_widths(R):
    x = case(33, R, seed=100 + R)
    check(x, run_gpu(x), oracle_refs(x))


@pytest.mark.parametrize('S,R', [(33, 128), (65, 3), (878, 129)])
def test_enrolment_prior(S, R):
    """State 0 with many enrolment x-vectors, state 1 with a few, the rest none; recording 4 has no prior at all."""
    x = case(S, R, seed=7 * S + R)
    rng = np.random.default_rng(S)
    B = len(x['lens'])
    pn, pF = np.zeros((B, S)), np.zeros((B, S, R))
    for b in range(B):
        if b == 4:
            continue
        for s, k in ((0, 200), (1, 3)):
            if s < x['ns'][b]:
                pn[b, s] = k
                pF[b, s] = rng.standard_normal((k, R)).sum(0) + k * x['fea'][0]
    refs = []
    for b in range(B):
        lo, hi, n = x['off'][b], x['off'][b + 1], x['ns'][b]
        if hi == lo:
            refs.append(None)
            continue
        g, pi, Li, alpha, invL = prior_oracle.vbx_prior_oracle(
            x['fea'][lo:hi], x['Phi'], pn[b, :n], pF[b, :n], loopProb=LOOP, Fa=FA, Fb=FB, pi=x['pi0'][b, :n],
            gamma=x['gamma0'][lo:hi, :n], maxIters=ITERS, epsilon=-np.inf, return_model=True)
        refs.append((g, pi, np.array([v[0] for v in Li]), alpha, invL))
    check(x, run_gpu(x, prior=(pn, pF)), refs)


def test_more_than_3600_states_is_refused():
    from vbx_b200 import VbxError
    from vbx_b200.batch import VbxBatch
    with pytest.raises(VbxError, match='S <= 3600'):
        VbxBatch([5, 0, 3], 16, 3601, device=dev(), f64_only=True)
