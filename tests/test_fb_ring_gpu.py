"""The fused forward-backward sweep fed from shared-memory rings (option fb_ring = 1, forward_backward_ring_kernel) computes
exactly what the register-burst sweep (fb_ring = 0, forward_backward_la_kernel) computes: same recurrences, same order
of operations, same float64 flushes of N_s and the re-entry sums.  Every (S, states per lane) instantiation, ragged
lengths with frame offsets that are not multiples of 4 (the 1/sigma windows of the bulk copies), fewer live states than
S, recordings that stop early and finish in float64 and per-recording Fa / Fb / loopP.
The launcher takes the ring sweep for plans whose recordings are at most 2048 frames long."""
import numpy as np
import pytest
import torch

from vbx_b200 import synth

pytestmark = pytest.mark.gpu
# (S, states per lane): every instantiation the launcher can pick on the fused sweep
VARIANTS = [(4, 1), (4, 2), (4, 4), (8, 1), (8, 2), (8, 4), (16, 1), (16, 2), (16, 4), (32, 1), (32, 2), (32, 4), (64, 2),
            (64, 4)]


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def lengths(seed, B, tmax, extra=()):
    lens = np.random.default_rng(seed).integers(1, tmax, size=B)
    lens[:5] = [1, 2, 17, 1023, 3]
    return np.concatenate([lens, np.asarray(extra, dtype=lens.dtype)])


def run_both(lens, S, spl, seed, epsilon=-np.inf, per_rec=False, max_iters=8):
    """gamma, pi, Li, n_iters and flags of the same batch with fb_ring = 0 and = 1 on the fused sweep."""
    from vbx_b200.batch import VbxBatch
    rng = np.random.default_rng(seed)
    ns = rng.integers(max(1, S // 2 + 1), S + 1, size=len(lens)).astype(np.int32)   # some recordings below S live states
    ns[0] = S
    d = synth.make_batch(lens, R=128, S=S, seed=seed, dtype=np.float32)
    g0 = d['gamma0'].astype(np.float32)
    for b in range(len(lens)):            # a recording's dead states carry no responsibility
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        g0[lo:hi, ns[b]:] = 0.0
        g0[lo:hi, :ns[b]] /= np.maximum(g0[lo:hi, :ns[b]].sum(1, keepdims=True), 1e-30)
    pi0 = np.zeros((len(lens), S), dtype=np.float32)
    for b in range(len(lens)):
        pi0[b, :ns[b]] = 1.0 / ns[b]
    if per_rec:
        B = len(lens)
        hyper = dict(Fa=cuda(rng.uniform(0.2, 0.4, B), torch.float64), Fb=cuda(rng.uniform(6.0, 64.0, B), torch.float64),
                     loopProb=cuda(rng.uniform(0.35, 0.99, B), torch.float64))
    else:
        hyper = dict(Fa=0.3, Fb=17.0, loopProb=0.99)
    out = []
    for ring in (0, 1):
        vb = VbxBatch(lens, 128, ns, device=dev(), fb_split=2)
        assert vb.S == S
        vb.set_option('fb_states_per_lane', spl)
        vb.set_option('fb_ring', ring)
        vb.prepare_scale(cuda(d['fea']), cuda(d['Phi']))
        g, p = cuda(g0), cuda(pi0)
        o = vb.run(g, p, maxIters=max_iters, epsilon=epsilon, **hyper)
        torch.cuda.synchronize()
        out.append({k: o[k].cpu().numpy() for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags')})
        vb.close()
    return out


def assert_identical(a, b):
    for k in ('gamma', 'pi', 'n_iters', 'flags'):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a['Li'], b['Li'], equal_nan=True)


@pytest.mark.parametrize('S,spl', VARIANTS, ids=[f'S{s}-spl{l}' for s, l in VARIANTS])
def test_ring_sweep_is_bit_identical(S, spl):
    a, b = run_both(lengths(S * 7 + spl, 150, 1200), S, spl, seed=S + spl)
    assert_identical(a, b)


@pytest.mark.parametrize('S,spl', [(16, 2), (8, 1), (64, 4)], ids=['S16-spl2', 'S8-spl1', 'S64-spl4'])
def test_ring_sweep_early_stop_float64_finish(S, spl):
    """epsilon = 1e-5: recordings stop at different iterations (inactive lanes in the sweep) and hand over to float64."""
    a, b = run_both(lengths(S + 11, 120, 900), S, spl, seed=3 * S + spl, epsilon=1e-5, max_iters=20)
    assert_identical(a, b)
    assert (a['n_iters'] < 20).any()


@pytest.mark.parametrize('S,spl', [(16, 2), (32, 1)], ids=['S16-spl2', 'S32-spl1'])
def test_ring_sweep_per_recording_hyperparameters(S, spl):
    a, b = run_both(lengths(S + 5, 100, 1100), S, spl, seed=5 * S + spl, per_rec=True)
    assert_identical(a, b)

