"""Representative runs for compute-sanitizer (memcheck / racecheck / synccheck / initcheck): wgmma projection at
D = 32 ... 2048 and x-vector chain (Dx = 256, 512), batches holding recordings without frames, fused and split forward-backward, chunked scan, the float64 finishing phase (stop rule, also with the enrolment prior at S = 4 and 128), state counts
6..128 (both contraction modes at S = 128), per-recording state masks, AHC, hard labels (also under a speaker-count bound),
the dense forward_backward(), the ELBO trace, DER / JER scoring, speaker linking across recordings (one problem and
batched), enrolment
against known speakers and score normalisation against a cohort (one problem and batched, and at R = 100), and
verification trials with AS-norm and the error rates.

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


def run(lens, S, iters, D=None, ns=None, fb_split=0, eps=-float('inf'), tag='', gemm=0, per_rec=False):
    d = synth.make_batch([t for t in lens if t], R=128, S=S, seed=3, D=D, dtype=np.float32)   # T = 0: no rows
    nsa = np.full(len(lens), S, dtype=np.int32) if ns is None else np.asarray(ns, dtype=np.int32)
    vb = VbxBatch(lens, 128, nsa, device=dev, fb_split=fb_split)
    vb.set_option('gemm', gemm)
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
    hp = dict(Fa=0.3, Fb=17.0, loopProb=0.99)
    if per_rec:      # per-recording hyperparameters (vbx_run_per_recording): the recipe settings in turn
        rec = [(0.3, 17.0, 0.99), (0.4, 64.0, 0.65), (0.2, 6.0, 0.35), (0.4, 17.0, 0.40)]
        hp = {k: torch.tensor([rec[b % 4][i] for b in range(len(lens))], dtype=torch.float64, device=dev)
              for i, k in enumerate(('Fa', 'Fb', 'loopProb'))}
    out = vb.run(g, p, maxIters=iters, epsilon=eps, return_model=True, **hp)
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
run([0, 300, 45, 0, 129, 0], 8, 30, D=256, eps=1e-5, fb_split=2, tag='empty recordings fused')
run([0, 300, 45, 0, 129, 0], 8, 30, D=256, eps=1e-5, fb_split=1, tag='empty recordings split')
# S = 128 tier (always the split schedule): both contraction modes, per-recording masks, the float64 finish
for gm in (0, 1):
    run([513, 512, 1, 2, 300], 128, 2, ns=[128, 100, 65, 3, 1], gemm=gm, tag=f'S=128 masks gemm={gm}')
    run([4100, 0, 300], 100, 2, D=256, gemm=gm, tag=f'S=128 long + empty gemm={gm}')
    run([300, 120, 64], 100, 30, eps=1e-5, gemm=gm, tag=f'S=128 stop rule, float64 finish gemm={gm}')
# the float64 finishing round with the enrolment prior at S = 4 and S = 128: empty recordings, T = 1 and 65 (a partial
# 64-frame block), 513 (a partial M-tile); states 0 and 2 enrolled from the recording's own frames, recording 1 without a
# prior.  epsilon is placed from a float32-only run (epsilon = -inf) so that recording 3 hands over at iteration 1: its
# Li[0] is then redone in float64 and differs from the float32 value.
for S_, fb_ in ((4, 2), (100, 1)):
    p_lens = [0, 513, 1, 65, 0, 300]
    p_vb = VbxBatch(p_lens, 128, S_, device=dev, fb_split=fb_)
    p_d = synth.make_batch([t for t in p_lens if t], R=128, S=S_, seed=5, dtype=np.float32)
    p_off = np.concatenate([[0], np.cumsum(p_lens)])
    p_n = np.zeros((len(p_lens), p_vb.S))
    p_F = np.zeros((len(p_lens), p_vb.S, 128))
    for b in (2, 3, 5):
        fb = p_d['fea'][p_off[b]:p_off[b + 1]].astype(np.float64)
        p_n[b, 0], p_n[b, 2] = 40.0, 3.0
        p_F[b, 0], p_F[b, 2] = 40.0 * fb.mean(0), fb[:1].sum(0) * 3.0
    p_prior = (torch.from_numpy(p_n).to(dev), torch.from_numpy(p_F).to(dev))
    p_vb.prepare_scale(torch.from_numpy(p_d['fea']).to(dev), torch.from_numpy(p_d['Phi']).to(dev))

    def p_run(eps):
        g = torch.zeros((p_vb.N, p_vb.S), device=dev)
        g[:, :S_] = torch.from_numpy(p_d['gamma0']).to(dev)
        p = torch.zeros((len(p_lens), p_vb.S), device=dev)
        p[:, :S_] = 1.0 / S_
        o = p_vb.run(g, p, Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=30, epsilon=eps, return_model=True, prior=p_prior)
        return o['Li'].cpu().numpy(), o['n_iters'].cpu().numpy()

    li32, _ = p_run(-float('inf'))
    p_eps = float(li32[3, 1] - li32[3, 0] - 4.0 * 2.0 ** -24 * abs(li32[3, 1]))      # d_1 - 2 nb_1
    li, n_it = p_run(p_eps)
    p_vb.close()
    assert li[3, 0] != li32[3, 0], 'recording 3 did not reach the float64 finishing round'
    print('float64 finish with prior ok', S_, n_it.tolist())
# per-recording Fa / Fb / loopP on every schedule, with the float64 finish
run([300, 45, 1, 129, 600], 16, 30, fb_split=1, eps=1e-5, per_rec=True, tag='per-recording split')
run([300, 45, 1, 129, 600], 16, 30, fb_split=2, eps=1e-5, per_rec=True, tag='per-recording fused')
run([4100, 300, 5000, 64], 8, 30, fb_split=2, eps=1e-5, per_rec=True, tag='per-recording chunked scan')
run([513, 512, 1, 2, 300], 128, 30, ns=[128, 100, 65, 3, 1], eps=1e-5, per_rec=True, tag='per-recording S=128')

# labels under a speaker-count bound (vbx_hard_labels_keep) at S = 128: recordings without frames, keep = 1, keep >= n_states
lens = [300, 0, 65, 1, 129, 0]
nsk = np.array([128, 1, 100, 3, 65, 7], dtype=np.int32)
kb = VbxBatch(lens, 128, nsk, device=dev, allocate=False)
gk = torch.rand((kb.N, kb.S), device=dev) * (torch.arange(kb.S, device=dev)[None, :] < 65)
fk, sk, mk = kb.hard_labels_keep(gk.contiguous(), [1, 1, 100, 5, 3, 1])
torch.cuda.synchronize()
kb.close()
print('hard labels keep ok', int(fk.max()), float(mk.sum()))

# speaker linking (link_speakers): recordings without x-vectors, a speaker with one x-vector, padded features, tile
# edges
from vbx_b200 import link  # noqa: E402
gl = np.random.default_rng(3)
l_lens = [0, 40, 1, 300, 0, 77]
l_labels = [gl.integers(0, k, n) for n, k in zip(l_lens, [1, 5, 1, 37, 1, 9])]
l_fea = torch.randn((sum(l_lens), 16), device=dev)
l_fea[:, 13:] = 0
l_phi = torch.rand(16, device=dev) * (torch.arange(16, device=dev) < 13)
l_out = link.link_speakers(l_fea, l_phi, np.concatenate([[0], np.cumsum(l_lens)]), l_labels, 0.3, 17.0, dev, dist=True)
torch.cuda.synchronize()
print('link ok', len(l_out[0].rec), float(l_out[3][:, 2].min()))
# batched linking (vbx_link_batch): a problem without speakers, one with a speaker per recording and the one above, each
# with its own Fa / Fb, in one launch and under a budget that puts the last problem into a launch of its own
lb_labels = [[np.full(n, -1) for n in l_lens], [np.where(np.arange(n) == 0, 0, -1) for n in l_lens], l_labels]
for lb_max in (None, 80000):          # 80 000 bytes: the last problem needs 78 592, the others 5 888
    lb_out = link.link_many(l_fea, l_phi, np.concatenate([[0], np.cumsum(l_lens)]), lb_labels, [0.3, 0.4, 0.2],
                            [17.0, 6.0, 64.0], dev, max_bytes=lb_max, dist=True)
    torch.cuda.synchronize()
    print('link batch ok', [len(o[0].rec) for o in lb_out], float(lb_out[2][3][:, 2].min()))

# enrolment (enroll_speakers): recordings without speakers, E = 1 and E < K_b, a tail tile (M, E not multiples of 32),
# and a recording with 150 speakers (more than 128)
from vbx_b200 import enroll  # noqa: E402
e_lens = l_lens + [600]
e_labels = l_labels + [np.concatenate([np.arange(150), gl.integers(0, 150, 450)])]
e_fea = torch.cat([l_fea, torch.randn((600, 16), device=dev)])
e_fea[:, 13:] = 0
for E in (1, 7, 45):
    e_x = torch.randn((2 * E + 1, 16), device=dev)
    e_x[:, 13:] = 0
    e_spk = np.concatenate([np.arange(E), np.arange(E), [0]])
    e_out = enroll.enroll_speakers(e_fea, l_phi, np.concatenate([[0], np.cumsum(e_lens)]), e_labels, e_x, e_spk, 0.3,
                                   17.0, 0.0, dev, llr=True, max_bytes=8 * E * 100)
    torch.cuda.synchronize()
    print('enroll ok', E, len(e_out.table.rec), int((e_out.assign >= 0).sum()))

# score normalisation against a cohort (cohort_stats, link_speakers and enroll_speakers with norm): C = 45 and M not
# multiples of 32, top_k > C, a run forced into chunks, and the recording with 150 speakers
from vbx_b200 import cohort  # noqa: E402
c_x = torch.randn((100, 16), device=dev)
c_x[:, 13:] = 0
c_spk = np.concatenate([np.arange(45), gl.integers(0, 45, 55)])
e_offs = np.concatenate([[0], np.cumsum(e_lens)])
c_st = cohort.cohort_stats(e_fea, l_phi, e_offs, e_labels, c_x, c_spk, 0.3, 17.0, top_k=50, device=dev,
                           max_bytes=8 * 45 * 40, scores=True)
c_en = cohort.cohort_stats(e_x, l_phi, None, e_spk, c_x, c_spk, 0.3, 17.0, top_k=50, device=dev)
c_link = link.link_speakers(e_fea, l_phi, e_offs, e_labels, 0.3, 17.0, dev, dist=True, norm=c_st[:2])
c_enr = enroll.enroll_speakers(e_fea, l_phi, e_offs, e_labels, e_x, e_spk, 0.3, 17.0, 0.0, dev, llr=True,
                               max_bytes=8 * 45 * 100, norm=c_st[:2] + c_en[:2])
torch.cuda.synchronize()
print('cohort ok', len(c_st.mean), float(c_st.std.min()), float(c_link[3][:, 2].min()), int((c_enr.assign >= 0).sum()))

# batched enrolment and cohort statistics (enroll_many, cohort_stats_many, link_many with norm): a problem
# without speakers, one with a speaker per recording and the one with 150 speakers, each with its own Fa / Fb; E = 45 <
# K_b = 150 and tail tiles; three thresholds; plain and normalised
eb_labels = [[np.full(n, -1) for n in e_lens], [np.where(np.arange(n) == 0, 0, -1) for n in e_lens], e_labels]
eb_fa, eb_fb = [0.3, 0.4, 0.2], [17.0, 6.0, 64.0]
eb_st = cohort.cohort_stats_many(e_fea, l_phi, e_offs, eb_labels, c_x, c_spk, eb_fa, eb_fb, 50, dev)
eb_en = cohort.cohort_stats_many(e_x, l_phi, None, [e_spk] * 3, c_x, c_spk, eb_fa, eb_fb, 50, dev)
for eb_norm in (None, [a[:2] + b[:2] for a, b in zip(eb_st, eb_en)]):
    eb_out = enroll.enroll_many(e_fea, l_phi, e_offs, eb_labels, e_x, e_spk, eb_fa, eb_fb, [-10.0, 0.0, 10.0], dev,
                                llr=True, norm=eb_norm)
    torch.cuda.synchronize()
    print('enroll batch ok', [len(o.table.rec) for o in eb_out], int((eb_out[2].assign >= 0).sum()))
eb_link = link.link_many(e_fea, l_phi, e_offs, eb_labels, eb_fa, eb_fb, dev, dist=True, norm=[a[:2] for a in eb_st])
torch.cuda.synchronize()
print('cohort batch ok', float(eb_st[2].std.min()), float(eb_en[2].std.min()), float(eb_link[2][3][:, 2].min()))

# the speaker-pair scores at R = 100 (a partial last chunk ending in a partial log group): linking, enrolment with
# E = 33 and cohort statistics with C = 33 (tail tiles), the speakers of the archive above
w_fea = torch.randn((sum(e_lens), 100), device=dev)
w_phi = torch.rand(100, device=dev) + 0.01
w_offs = np.concatenate([[0], np.cumsum(e_lens)])
w_x = torch.randn((70, 100), device=dev)
w_spk = np.concatenate([np.arange(33), gl.integers(0, 33, 37)])
w_link = link.link_speakers(w_fea, w_phi, w_offs, e_labels, 0.3, 17.0, dev, dist=True)
w_enr = enroll.enroll_speakers(w_fea, w_phi, w_offs, e_labels, w_x, w_spk, 0.3, 17.0, 0.0, dev, llr=True)
w_st = cohort.cohort_stats(w_fea, w_phi, w_offs, e_labels, w_x, w_spk, 0.3, 17.0, top_k=10, device=dev, scores=True)
torch.cuda.synchronize()
print('R=100 link, enroll, cohort ok', len(w_link[0].rec), int((w_enr.assign >= 0).sum()), float(w_st.std.min()))

# verification trials (vbx_verify_score, vbx_verify_metrics): single and multi-x-vector items at R = 100, trials whose
# count is not a multiple of 32 (a warp with idle lanes), AS-norm against a cohort, and the error rates with ties
from vbx_b200 import verify  # noqa: E402
v_e, v_t = w_x[:40].cpu().numpy(), w_fea[:500].cpu().numpy()
v_ie, v_it = np.arange(40) % 17, gl.integers(0, 61, 500)
v_it[:61] = np.arange(61)
v_phi = w_phi.cpu().numpy()
v_tr = np.stack([gl.integers(0, 17, 1001), gl.integers(0, 61, 1001)], 1)
v_norm = verify.trial_norm(v_e, v_ie, v_t, v_it, v_phi, w_x.cpu().numpy(), w_spk, 0.3, 17.0, top_k=20, device=dev)
v_s = verify.score_trials(v_e, v_ie, v_t, v_it, v_phi, v_tr, Fa=0.3, Fb=17.0, norm=v_norm, device=dev)
v_y = v_tr[:, 0] == v_tr[:, 1] % 17
v_m = verify.error_rates(np.round(v_s, 1), v_y, (0.01, 0.5), device=dev)
torch.cuda.synchronize()
print('verify ok', float(v_s.min()), v_m['eer'], v_m['cllr'])

# wgmma projection at the smallest and largest D, one frame and one frame past a full wave of tiles
sms = torch.cuda.get_device_properties(0).multi_processor_count
gen = np.random.default_rng(7)
for D in (32, 2048):
    for N in (1, 128 * sms + 1):
        pb = VbxBatch([N], 128, 4, device=dev)
        pb.set_option('projection', 2)
        pb.prepare_project(torch.from_numpy(gen.standard_normal((N, D)).astype(np.float32)).to(dev),
                           torch.from_numpy(gen.standard_normal((D, 128)).astype(np.float32)).to(dev),
                           torch.ones(128, device=dev))
        pg = pb.g_sum()
        torch.cuda.synchronize()
        pb.close()
        print('projection ok', D, N, float(pg[0]))

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

# AHC at a feature width with a 1-wide tail tile and a recording of 1056 x-vectors (more than the linkage kernel's
# 1024 threads), once with duplicated x-vectors (ties) and once with a NaN x-vector (the linkage stops early)
for tag in ('duplicates', 'NaN row'):
    lens = [1056, 40, 3]
    xa = gen.standard_normal((sum(lens), 33))
    if tag == 'duplicates':
        xa[gen.choice(1056, 300, replace=False)] = xa[gen.integers(0, 1056, 300)]
    else:
        xa[500, 7] = np.nan
    ab = VbxBatch(lens, 128, 1, device=dev, allocate=False)
    labels, thr, _ = ahc.ahc_batch(ab, torch.from_numpy(xa).to(dev))
    torch.cuda.synchronize()
    ab.close()
    print('AHC dim 33 ' + tag + ' ok', int(labels[0].max()) + 1)

# x-vector chain with Dx = 512 over more than one tile per CTA
T = 128 * sms + 1
front = VbxBatch([T], 128, 1, device=dev)
model512 = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev) for a in (
    gen.standard_normal(512) * 0.1, gen.standard_normal((512, 128)) / 16, gen.standard_normal(128) * 0.05,
    gen.standard_normal(128) * 0.02, q * gen.uniform(2, 20, 128)[:, None], np.linspace(8.0, 0.05, 128))]
rho, xn = front.prepare_xvectors(torch.from_numpy(gen.standard_normal((T, 512)).astype(np.float32)).to(dev), *model512)
torch.cuda.synchronize()
front.close()
print('x-vector chain Dx=512 ok', float(rho[-1, 0]))

# dense forward_backward()
lls = gen.standard_normal((60, 9)) * 5
tr_ = gen.dirichlet(np.ones(9), size=9)
post, tll, lfw, lbw = api.forward_backward(lls, tr_, gen.dirichlet(np.ones(9)))
print('forward_backward ok', tll)

# DER scoring: ragged recordings (1 x-vector, pauses, none) and one with 64 reference speakers (up to 4 overlapping), so
# that one launch takes the 64 KB shared-memory configuration, holds 64 x 128 overlap blocks in shared memory and
# accumulates 64 x 200 blocks in place in global memory
from vbx_b200 import pipeline, score          # noqa: E402
arch = synth.make_scoring_archive([1, 300, 0, 900], seed=4, gap_prob=0.05)
rows = []
for n, (seg, lab) in list(arch.items())[:3]:
    s_, e_, l_ = pipeline.merge_adjacent_labels(seg[:, 0], seg[:, 1], lab)
    rows += [(n, float(a), float(z - a), f'spk{k}') for a, z, k in zip(s_, e_, l_)]
big = list(arch)[3]
span = float(arch[big][0][-1, 1])
for layer in range(4):
    t, k = float(gen.uniform(0, 2)), layer
    while t < span:
        d = float(gen.uniform(0.2, 2.0))
        rows.append((big, round(t, 2), round(d, 2), f'spk{k % 64}'))
        k += 4
        t += d + float(gen.uniform(0, 1.5))
turns = score.reference_turns(rows)
recs = [score.prepare_recording(n, turns.get(n, []), score.owned_intervals(seg)) for n, (seg, _) in arch.items()]
assert recs[3].n_ref == 64, recs[3].n_ref
entries = [(b, gen.integers(0, L, len(seg))) for b, (seg, _) in enumerate(arch.values()) for L in (1, 128, 200)]
res = score.score_entries(recs, entries, device=dev)
print('score ok', res[-1]['full']['ticks'])

# overlap-aware scoring (vbx_score_overlap): the same recordings with their reference overlaps as the overlap regions,
# second labels for the 128-label (shared O block) and 200-label (global O block) entries, and -1 rows (no second label)
recs = [score.prepare_recording(n, turns.get(n, []), score.owned_intervals(seg),
                                overlap=score.oracle_overlaps(turns.get(n, []))) for n, (seg, _) in arch.items()]
entries2 = []
for b, lab in entries:
    L = int(lab.max()) + 1 if len(lab) else 1
    lab2 = (lab + gen.integers(1, max(L, 2), len(lab))) % max(L, 2) if L > 1 else None
    if lab2 is not None:
        lab2[gen.random(len(lab)) < 0.3] = -1
    entries2.append((b, lab, lab2))
res2 = score.score_entries(recs, entries2, device=dev)
print('score overlap ok', res2[-1]['full']['ticks'])

# label time for the Jaccard error rate (vbx_score_jer): single-label entries, 128-label blocks in shared memory and
# 200-label blocks in place in global memory, then two-stream entries
recs = [score.prepare_recording(n, turns.get(n, []), score.owned_intervals(seg)) for n, (seg, _) in arch.items()]
res3 = score.score_entries(recs, entries, device=dev, jer='full')
print('score jer ok', res3[-1]['jer']['jer'])
recs = [score.prepare_recording(n, turns.get(n, []), score.owned_intervals(seg),
                                overlap=score.oracle_overlaps(turns.get(n, []))) for n, (seg, _) in arch.items()]
res4 = score.score_entries(recs, entries2, device=dev, jer='full')
print('score jer overlap ok', res4[-1]['jer']['jer'])
