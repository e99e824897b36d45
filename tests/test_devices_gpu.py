"""Handles on two devices in one process.  Kernels that launch with more than 48 KB of dynamic shared memory must be
allowed that much on each device they run on (allow_dynamic_smem); every case here runs on cuda:0 and then on cuda:1 in
the same process, and the second device's outputs must equal the first's bit for bit."""
import pickle

import numpy as np
import pytest
import torch

from test_combine_gpu import _batch as combine_batch
from test_jer_gpu import ragged_case
from test_projection_gpu import xvector_model
from vbx_b200 import api, combine, score, synth
from vbx_b200.batch import VbxBatch, run_f64

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two CUDA devices in one process '
                                                                       '(torch.cuda.device_count() < 2)')]
LENS = [300, 450, 700, 1000]


def cuda(a, dev, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev).to(dtype)


def on_both_devices(case, *args):
    a = case(torch.device('cuda:0'), *args)
    b = case(torch.device('cuda:1'), *args)
    assert pickle.dumps(b) == pickle.dumps(a)
    return a


def vb_run(dev, n, fb_split, gemm, prior=False):
    d = synth.make_batch(LENS, R=128, S=n, seed=5 + n, dtype=np.float32)
    vb = VbxBatch(LENS, 128, n, device=dev, fb_split=fb_split)
    vb.set_option('gemm', gemm)
    vb.set_option('timing', 1)
    S = vb.S
    vb.prepare_scale(cuda(d['fea'], dev), cuda(d['Phi'], dev))
    g = torch.zeros((vb.N, S), device=dev)
    g[:, :n] = cuda(d['gamma0'], dev)
    pi = torch.zeros((vb.B, S), device=dev)
    pi[:, :n] = 1.0 / n
    kw = {}
    if prior:
        rng = np.random.default_rng(3)
        pn = np.zeros((vb.B, S))
        pn[:, :n] = rng.uniform(0.0, 4.0, (vb.B, n))
        pF = rng.standard_normal((vb.B, S, 128)) * pn[..., None]
        kw['prior'] = (cuda(pn, dev, torch.float64), cuda(pF, dev, torch.float64))
    out = vb.run(g, pi, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=10, epsilon=1e-6, return_model=True, **kw)
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res['launches'] = {k: c for k, (_, c) in vb.timings().items()}
    vb.close()
    return res


@pytest.mark.parametrize('gemm', [0, 1])
@pytest.mark.parametrize('fb_split', [0, 2])
def test_run_s16(fb_split, gemm):
    """Float64 finish (loglik64 above 48 KB); fb_split = 2 takes em_contract and the ring sweep, gemm = 1 the FFMA
    mstep_partial and loglik."""
    res = on_both_devices(vb_run, 16, fb_split, gemm)
    assert res['launches']['exact64'] > 0
    assert (res['launches']['em_contract'] > 0) == (fb_split == 2 and gemm == 0)


@pytest.mark.parametrize('gemm', [0, 1])
@pytest.mark.parametrize('n', [64, 100])
def test_run_wide(n, gemm):
    """loglik_mma, mstep_mma<128>, speaker_model<128> and fb_combine; mstep_partial<128> and loglik with gemm = 1."""
    on_both_devices(vb_run, n, 0, gemm)


def test_run_prior():
    """speaker_model_prior<128>"""
    on_both_devices(vb_run, 100, 0, 0, True)


def project(dev):
    d = synth.make_batch([700, 300], R=128, S=4, seed=2, D=256, dtype=np.float32)
    vb = VbxBatch([700, 300], 128, 4, device=dev)
    rho = vb.prepare_project(cuda(d['X'], dev), cuda(d['V'], dev), cuda(d['Phi'], dev)).cpu().numpy()
    model = xvector_model(np.random.default_rng(4), 512)
    x_raw = cuda(np.random.default_rng(5).standard_normal((1000, 512)), dev)
    rho2, x_norm = vb.prepare_xvectors(x_raw, *(cuda(a, dev) for a in model))
    res = dict(rho=rho, rho2=rho2.cpu().numpy(), x_norm=x_norm.cpu().numpy(), g=vb.g_sum().cpu().numpy())
    vb.close()
    return res


def test_projection():
    on_both_devices(project)


def f64_run(dev):
    lens, n = [200, 150], 1000
    d = synth.make_batch(lens, R=128, S=n, seed=6, dtype=np.float64)
    vb = VbxBatch(lens, 128, n, device=dev, f64_only=True, allocate=False)
    g = cuda(d['gamma0'], dev, torch.float64)
    pi = torch.full((vb.B, n), 1.0 / n, dtype=torch.float64, device=dev)
    out = run_f64(vb, cuda(d['fea'], dev, torch.float64), cuda(d['Phi'], dev, torch.float64), g, pi, Fa=0.3, Fb=17.0,
                  loopProb=0.99, maxIters=3, epsilon=-float('inf'))
    res = {k: v.cpu().numpy() for k, v in out.items()}
    vb.close()
    return res


def test_run_f64_many_states():
    """f64::fb_kernel above 48 KB"""
    on_both_devices(f64_run)


def dense_fb(dev):
    rng = np.random.default_rng(7)
    S = 100
    tr = rng.uniform(0.1, 1.0, (S, S))
    tr /= tr.sum(1, keepdims=True)
    with torch.cuda.device(dev):
        return api.forward_backward(rng.standard_normal((400, S)) * 3.0, tr, np.full(S, 1.0 / S))


def test_forward_backward_dense():
    """fb_dense_kernel<true>"""
    on_both_devices(dense_fb)


def test_score_jer_large_block():
    """The score kernel with label time and a block of 64 reference speakers x 128 or 200 labels (above 48 KB)."""
    names, segs, ref_rows, recs, ovl, entries, _ = ragged_case(61, True, False)
    assert any(r.n_ref == 64 for r in recs)
    on_both_devices(lambda dev: score.score_entries(recs, entries, device=dev, jer='full'))


def test_combine():
    intervals, hyps = combine_batch(8, 4, 90, [0, 1, 40, 300, 1200])
    on_both_devices(lambda dev: combine.combine_labels(intervals, hyps, device=dev, strict=False, blocks=True))
