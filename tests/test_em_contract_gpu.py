"""The fused EM contraction (em_contract_kernel, vbx_em_contract.cu) against the three kernels it replaces.

Batches on the fused sweep whose recordings are all <= 1024 frames run M-step, speaker model and log-likelihood as one
cluster kernel; one recording of 1500 frames sends the whole batch back to the three kernels.  A recording's results do
not depend on the rest of its batch, so every recording of batch A must come out bit for bit as in batch B, A plus the
long recording.  Workspace, rho and gamma are surrounded by poison so that a read or write out of bounds shows."""
import subprocess
import shutil

import numpy as np
import pytest
import torch

from vbx_b200 import _lib, synth

EDGES = [0, 1, 2, 3, 7, 8, 9, 31, 32, 33, 487, 488, 511, 512, 513, 1000, 1023, 1024]
# clusters of 8 CTAs (longest recording 513 .. 1024 frames) and of 4 (at most 512 frames)
BATCHES = {'cl8': EDGES + [600, 900, 1024, 257] * 2, 'cl4': [t for t in EDGES if t <= 512] + [100, 257, 400, 512] * 2}
GUARD = 64   # NaN rows after rho and after gamma


def run(lens, d, n, eps, per_rec):
    from vbx_b200.batch import VbxBatch
    dev = torch.device('cuda:0')
    B = len(lens)
    ns = [n - (b % 3 == 1) for b in range(B)]   # dead columns in every third recording
    vb = VbxBatch(lens, 128, ns, device=dev, fb_split=2, allocate=False)
    vb.bind(torch.full((vb.workspace_bytes,), 0xFF, dtype=torch.uint8, device=dev))
    vb.set_option('timing', 1)
    S, N = vb.S, vb.N
    rho_all = torch.full((N + GUARD, 128), float('nan'), device=dev)
    vb.prepare_scale(torch.from_numpy(d['fea'][:N]).to(dev), torch.from_numpy(d['Phi']).to(dev), out=rho_all[:N])
    g_all = torch.full((N + GUARD, S), float('nan'), device=dev)
    g = g_all[:N]
    g.zero_()
    g0 = torch.from_numpy(d['gamma0'][:N]).to(dev)
    for b in range(B):
        lo, hi = int(vb.offsets[b]), int(vb.offsets[b + 1])
        g[lo:hi, :ns[b]] = g0[lo:hi, :ns[b]] / g0[lo:hi, :ns[b]].sum(1, keepdim=True).clamp_min(1e-30)
    pi = torch.zeros((B, S), device=dev)
    for b in range(B):
        pi[b, :ns[b]] = 1.0 / ns[b]
    hyper = dict(Fa=0.3, Fb=17.0, loopProb=0.99)
    if per_rec:
        hyper = {k: torch.full((B,), v, dtype=torch.float64, device=dev) for k, v in hyper.items()}
    vb.timings(reset=True)
    out = vb.run(g, pi, maxIters=12, epsilon=eps, return_model=True, **hyper)
    torch.cuda.synchronize()
    t = vb.timings(reset=True)
    assert torch.isnan(g_all[N:]).all() and torch.isnan(rho_all[N:]).all()
    for b in range(B):
        assert (pi[b, ns[b]:] == 0).all()
        lo, hi = int(vb.offsets[b]), int(vb.offsets[b + 1])
        assert (g[lo:hi, ns[b]:] == 0).all()
    res = dict(gamma=g.cpu(), pi=pi.cpu(), Li=out['Li'].cpu(), n_iters=out['n_iters'].cpu(), alpha=out['alpha'].cpu(),
               invL=out['invL'].cpu(), offsets=vb.offsets.copy(), fused=t['em_contract'][1], mstep=t['mstep_partial'][1])
    vb.close()
    return res


def same(a, b):
    a, b = a.numpy(), b.numpy()
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize('n', [3, 7, 16])
@pytest.mark.parametrize('per_rec', [False, True])
@pytest.mark.parametrize('eps', [-float('inf'), 1e-6])
@pytest.mark.parametrize('batch', sorted(BATCHES))
def test_fused_iteration_is_bit_identical_to_the_three_kernels(n, per_rec, eps, batch):
    lens = list(BATCHES[batch])
    d = synth.make_batch([t for t in lens + [1500] if t], R=128, S=n, seed=11 + n, dtype=np.float32)   # B's inputs
    a = run(lens, d, n, eps, per_rec)                                          # A's: the rows of its recordings
    b = run(lens + [1500], d, n, eps, per_rec)
    assert a['fused'] > 0 and a['mstep'] == 0
    assert b['fused'] == 0 and b['mstep'] > 0
    N = int(a['offsets'][-1])
    B = len(lens)
    assert same(a['gamma'], b['gamma'][:N])
    for k in ('pi', 'Li', 'n_iters', 'alpha', 'invL'):
        assert same(a[k], b[k][:B]), k


def test_fused_kernel_sass():
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    try:
        out = subprocess.run([tool, '-sass', _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip('cuobjdump not available')
    fns = [f for f in out.split('Function : ')[1:] if f.startswith('_ZN3vbx18em_contract_kernel')]
    assert len(fns) == 6                                   # S = 4, 8, 16 x clusters of 4 and 8
    for f in fns:
        for op in ('HMMA', 'UCGABAR_ARV', 'UCGABAR_WAIT', 'UBLKCP'):
            assert op in f, op
