"""Representative runs for compute-sanitizer (memcheck / racecheck / synccheck / initcheck): wgmma projection and
x-vector chain, fused and split forward-backward, chunked scan, the float64 finishing phase (stop rule), state counts
6..64, per-recording state masks, AHC, hard labels, the dense forward_backward() and the ELBO trace.

    compute-sanitizer --tool memcheck --error-exitcode 3 python tools/sanitizer_cases.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vbx_b200 import ahc, api, synth          # noqa: E402
from vbx_b200.batch import VbxBatch           # noqa: E402

dev = torch.device('cuda:0')


def run(lens, S, iters, D=None, ns=None, fb_split=0, eps=-float('inf'), tag=''):
    d = synth.make_batch(lens, R=128, S=S, seed=3, D=D, dtype=np.float32)
    nsa = np.full(len(lens), S, dtype=np.int32) if ns is None else np.asarray(ns, dtype=np.int32)
    vb = VbxBatch(lens, 128, nsa, device=dev, fb_split=fb_split)
    Sp = vb.S
    g = torch.zeros((sum(lens), Sp), device=dev)
    g0 = d['gamma0'].copy()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        g0[offs[b]:offs[b + 1], nsa[b]:] = 0
        g0[offs[b]:offs[b + 1]] /= g0[offs[b]:offs[b + 1]].sum(1, keepdims=True)
    g[:, :S] = torch.from_numpy(g0).to(dev)
    p = torch.zeros((len(lens), Sp), device=dev)
    for b in range(len(lens)):
        p[b, :nsa[b]] = 1.0 / nsa[b]
    if D:
        vb.prepare_project(torch.from_numpy(d['X']).to(dev), torch.from_numpy(d['V']).to(dev), torch.from_numpy(d['Phi']).to(dev))
    else:
        vb.prepare_scale(torch.from_numpy(d['fea']).to(dev), torch.from_numpy(d['Phi']).to(dev))
    out = vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=iters, epsilon=eps, return_model=True)
    lab = vb.hard_labels(g, second=True)
    tr = vb.elbo_trace(out['Li'])
    torch.cuda.synchronize()
    vb.close()
    print(tag, lens[:4], S, 'ok', out['n_iters'].tolist()[:4], float(tr[0]))


run([300, 45, 1, 129, 600], 16, 2, D=256, fb_split=2, tag='fused+projection')
run([300, 45, 1, 129, 600], 16, 2, fb_split=1, tag='split')
run([37, 700, 2], 6, 2, ns=[6, 3, 5], fb_split=2, tag='fused masks')
run([37, 700, 2], 6, 2, ns=[6, 3, 5], fb_split=1, tag='split masks')
run([4100, 300], 8, 2, fb_split=2, tag='chunked scan')
run([4100, 300], 8, 2, fb_split=1, tag='split long')
run([513, 512, 511], 64, 2, fb_split=2, tag='S=64 fused')
run([513, 512, 1], 64, 2, fb_split=1, tag='S=64 split')
run([100, 200], 31, 2, fb_split=1, tag='S=31 split')
run([300, 120, 64], 8, 30, eps=1e-5, tag='stop rule, float64 finish')
run([513, 40], 31, 25, eps=1e-6, fb_split=2, tag='stop rule fused')

# real-data front end + AHC
T = 300
gen = np.random.default_rng(5)
x_raw = gen.standard_normal((T, 256)).astype(np.float32)
q, _ = np.linalg.qr(gen.standard_normal((128, 128)))
model = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev) for a in (
    gen.standard_normal(256) * 0.1, gen.standard_normal((256, 128)) / 16, gen.standard_normal(128) * 0.05,
    gen.standard_normal(128) * 0.02, q * gen.uniform(2, 20, 128)[:, None], np.linspace(8.0, 0.05, 128))]
front = VbxBatch([T], 128, 1, device=dev)
rho, xn = front.prepare_xvectors(torch.from_numpy(x_raw).to(dev), *model)
labels, thr, _ = ahc.ahc_batch(front, xn)
torch.cuda.synchronize()
front.close()
print('front end + AHC ok', int(labels[0].max()) + 1)

# dense forward_backward()
lls = gen.standard_normal((60, 9)) * 5
tr_ = gen.dirichlet(np.ones(9), size=9)
post, tll, lfw, lbw = api.forward_backward(lls, tr_, gen.dirichlet(np.ones(9)))
print('forward_backward ok', tll)
