"""Enrolled speakers as state priors of the VB-HMM (DESIGN.md section 5.23) on the GPU: every state tier against the
float64 oracle (oracle/prior_oracle.py), the all-zero prior bit-identical to the plain entries, the same bits for a
recording alone, in a larger batch, with per-recording Fa / Fb, in a partitioned batch and under graph replay, and
diarize_batch(enroll_prior=True) and the command line on synthetic archives and ES2005a."""
import io
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from oracle import prior_oracle as po
from vbx_b200 import pipeline, score, synth

pytestmark = pytest.mark.gpu
TOL = 1e-4
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
Fa, Fb, LOOP = 0.3, 17.0, 0.99


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def ragged(seed, B, tmax):
    lens = np.random.default_rng(seed).integers(40, tmax, size=B)
    lens[:2] = [2, 513]
    return lens


def make_prior(d, n, S, R, seed, big=300):
    """Per recording: state 0 enrolled with `big` x-vectors near the recording's own frames, state 2 with 3, state 1 of
    recording 1 none at all (recording 1 has no prior)."""
    rng = np.random.default_rng(seed)
    offs = d['offsets']
    B = len(offs) - 1
    pn, pF = np.zeros((B, S)), np.zeros((B, S, R))
    for b in range(B):
        if b == 1:
            continue
        fea = d['fea'][offs[b]:offs[b + 1]].astype(np.float64)
        for s, k in ((0, big), (2, 3)):
            if s >= n:
                continue
            rows = fea[rng.integers(len(fea), size=k)] + rng.normal(0, 0.3, (k, fea.shape[1]))
            pn[b, s] = k
            pF[b, s] = rows.sum(0)
    return pn, pF


class Case:
    """One planned float32 batch with its inputs and a prior."""

    def __init__(self, lens, n, seed, fb_split=0, opts=None, make=None, poison=False):
        from vbx_b200.batch import VbxBatch
        self.d = synth.make_batch(lens, R=128, S=n, seed=seed, dtype=np.float32)
        self.n, self.lens = n, np.asarray(lens)
        self.vb = (make or VbxBatch)(lens, 128, n, device=dev(), fb_split=fb_split)
        for k, v in (opts or {}).items():
            self.vb.set_option(k, v)
        if poison:
            self.vb.workspace.fill_(0xFF)     # NaN in float32 and float64: nothing may be read before it is written
        self.S = self.vb.S
        self.vb.prepare_scale(cuda(self.d['fea']), cuda(self.d['Phi']))
        self.pn, self.pF = make_prior(self.d, n, self.S, 128, seed)

    def fresh(self):
        g = torch.zeros((self.vb.N, self.S), device=dev())
        g[:, :self.n] = cuda(self.d['gamma0'])
        p = torch.zeros((self.vb.B, self.S), device=dev())
        p[:, :self.n] = 1.0 / self.n
        return g, p

    def prior(self, zero=False):
        f = (lambda a: np.zeros_like(a)) if zero else (lambda a: a)
        return cuda(f(self.pn), torch.float64), cuda(f(self.pF), torch.float64)

    def run(self, Fa=Fa, Fb=Fb, loopProb=LOOP, prior=None, **kw):
        g, p = self.fresh()
        out = self.vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopProb, prior=prior, **kw)
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}


def oracle(d, b, n, pn, pF, maxIters, epsilon, alpha=None, invL=None):
    lo, hi = d['offsets'][b], d['offsets'][b + 1]
    trace = []
    g, pi, Li = po.vbx_prior_oracle(d['fea'][lo:hi].astype(np.float64), d['Phi'].astype(np.float64), pn[b, :n],
                                    pF[b, :n], loopProb=LOOP, Fa=Fa, Fb=Fb, pi=n,
                                    gamma=d['gamma0'][lo:hi].astype(np.float64), maxIters=maxIters, epsilon=epsilon,
                                    alpha=alpha, invL=invL, trace=trace)
    return g, pi, np.array([x[0] for x in Li])


def assert_close(out, d, b, n, ref):
    lo, hi = d['offsets'][b], d['offsets'][b + 1]
    g, pi, Li = ref
    assert int(out['n_iters'][b]) == len(Li), (b, out['n_iters'][b], len(Li))
    assert np.abs(out['gamma'][lo:hi, :n] - g).max() <= TOL, b
    assert np.abs(out['pi'][b, :n] - pi).max() <= TOL, b
    np.testing.assert_allclose(out['Li'][b, :len(Li)], Li, rtol=TOL)


# id: (lengths, live states, fb_split)
CASES = {
    'fused-S16': (ragged(1, 10, 500), 12, 2),
    'split-S16': (ragged(2, 8, 500), 12, 1),
    'fused-S64': (ragged(3, 6, 400), 40, 2),
    'S128': (ragged(4, 4, 400), 90, 1),
}


@pytest.mark.parametrize('epsilon', [1e-4, 1e-5, 1e-6])
@pytest.mark.parametrize('case', list(CASES))
def test_float32_tiers_against_the_oracle(case, epsilon):
    lens, n, fb_split = CASES[case]
    c = Case(lens, n, seed=len(case), fb_split=fb_split, poison=True)
    out = c.run(prior=c.prior(), maxIters=25, epsilon=epsilon)
    for b in range(len(lens)):
        assert_close(out, c.d, b, n, oracle(c.d, b, n, c.pn, c.pF, 25, epsilon))


def test_float32_warm_start_against_the_oracle():
    lens, n, fb_split = CASES['split-S16']
    c = Case(lens, n, seed=5, fb_split=fb_split)
    B, S = len(lens), c.S
    rng = np.random.default_rng(3)
    alpha = rng.normal(0, 0.3, (B, S, 128)).astype(np.float32)
    invL = rng.uniform(0.2, 1.0, (B, S, 128)).astype(np.float32)
    alpha[:, n:] = 0
    invL[:, n:] = 0
    out = c.run(prior=c.prior(), maxIters=12, epsilon=1e-6, alpha=cuda(alpha), invL=cuda(invL), warm_start=True)
    for b in range(B):
        assert_close(out, c.d, b, n, oracle(c.d, b, n, c.pn, c.pF, 12, 1e-6, alpha[b, :n].astype(np.float64),
                                            invL[b, :n].astype(np.float64)))


def _f64(lens, n, seed):
    from vbx_b200.batch import VbxBatch
    d = synth.make_batch(lens, R=24, S=n, seed=seed, dtype=np.float64)
    vb = VbxBatch(lens, 24, n, device=dev(), f64_only=True)
    pn, pF = make_prior(d, n, vb.S, 24, seed)
    return d, vb, pn, pF


def _run_f64(d, vb, n, prior, **kw):
    from vbx_b200.batch import run_f64
    g = cuda(d['gamma0'], torch.float64)
    p = torch.full((vb.B, n), 1.0 / n, dtype=torch.float64, device=dev())
    out = run_f64(vb, cuda(d['fea'], torch.float64), cuda(d['Phi'], torch.float64), g, p, Fa=Fa, Fb=Fb, loopProb=LOOP,
                  prior=prior, return_model=True, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def test_float64_tier_against_the_oracle():
    lens, n = np.array([150, 2, 260]), 130
    d, vb, pn, pF = _f64(lens, n, 7)
    for epsilon in (1e-4, 1e-6):
        out = _run_f64(d, vb, n, (cuda(pn, torch.float64), cuda(pF, torch.float64)), maxIters=15, epsilon=epsilon)
        for b in range(len(lens)):
            assert_close(out, d, b, n, oracle(d, b, n, pn, pF, 15, epsilon))
    zero = _run_f64(d, vb, n, (cuda(0 * pn, torch.float64), cuda(0 * pF, torch.float64)), maxIters=15, epsilon=1e-6)
    plain = _run_f64(d, vb, n, None, maxIters=15, epsilon=1e-6)
    for k in plain:
        assert np.array_equal(zero[k], plain[k], equal_nan=True), k
    vb.close()


def test_float64_tier_warm_start_against_the_oracle():
    lens, n = np.array([150, 2, 260]), 130
    d, vb, pn, pF = _f64(lens, n, 8)
    rng = np.random.default_rng(4)
    alpha = rng.normal(0, 0.3, (len(lens), n, 24))
    invL = rng.uniform(0.2, 1.0, (len(lens), n, 24))
    out = _run_f64(d, vb, n, (cuda(pn, torch.float64), cuda(pF, torch.float64)), maxIters=12, epsilon=1e-6,
                   alpha=cuda(alpha, torch.float64), invL=cuda(invL, torch.float64), warm_start=True)
    for b in range(len(lens)):
        assert_close(out, d, b, n, oracle(d, b, n, pn, pF, 12, 1e-6, alpha[b], invL[b]))
    vb.close()


def assert_entry_equal(a, b, ra, rb, offa, offb):
    assert np.array_equal(a['gamma'][offa[ra]:offa[ra + 1]], b['gamma'][offb[rb]:offb[rb + 1]])
    for k in ('pi', 'Li', 'n_iters', 'flags', 'alpha', 'invL'):
        if k in a:
            assert np.array_equal(a[k][ra], b[k][rb], equal_nan=True), k


@pytest.mark.parametrize('case', list(CASES))
def test_zero_prior_is_bit_identical(case):
    lens, n, fb_split = CASES[case]
    c = Case(lens, n, seed=11, fb_split=fb_split)
    for eps in (-np.inf, 1e-6):
        kw = dict(maxIters=15, epsilon=eps, return_model=True)
        plain = c.run(**kw)
        zero = c.run(prior=c.prior(zero=True), **kw)
        for k in plain:
            assert np.array_equal(plain[k], zero[k], equal_nan=True), (k, eps)


def test_same_bits_alone_in_a_batch_per_recording_and_partitioned():
    from vbx_b200.parts import PartitionedBatch, make_batch
    lens, n = ragged(8, 12, 500), 12
    kw = dict(maxIters=15, epsilon=1e-6, return_model=True)
    whole = Case(lens, n, seed=3, fb_split=1)
    ref = whole.run(prior=whole.prior(), **kw)
    offs = whole.d['offsets']
    # per-recording Fa / Fb: a recording with the batch's values keeps its bits
    B = len(lens)
    fa = torch.full((B,), Fa, dtype=torch.float64, device=dev())
    fb = torch.full((B,), Fb, dtype=torch.float64, device=dev())
    fa[1::2], fb[1::2] = 0.4, 64.0
    per = whole.run(Fa=fa, Fb=fb, prior=whole.prior(), **kw)
    for b in range(0, B, 2):
        assert_entry_equal(per, ref, b, b, offs, offs)
    # partitioned: each part takes its rows of the prior
    parts = Case(lens, n, seed=3, fb_split=1, make=lambda *a, **k: make_batch(*a, parts=2, **k))
    assert isinstance(parts.vb, PartitionedBatch)
    got = parts.run(prior=parts.prior(), **kw)
    for b in range(B):
        assert_entry_equal(got, ref, b, b, offs, offs)
    # recording 3 alone
    from vbx_b200.batch import VbxBatch
    b = 3
    one = VbxBatch(lens[b:b + 1], 128, n, device=dev(), fb_split=1)
    one.prepare_scale(cuda(whole.d['fea'][offs[b]:offs[b + 1]]), cuda(whole.d['Phi']))
    g = torch.zeros((int(lens[b]), one.S), device=dev())
    g[:, :n] = cuda(whole.d['gamma0'][offs[b]:offs[b + 1]])
    p = torch.zeros((1, one.S), device=dev())
    p[:, :n] = 1.0 / n
    pr = (cuda(whole.pn[b:b + 1], torch.float64), cuda(whole.pF[b:b + 1], torch.float64))
    out = {k: v.cpu().numpy() for k, v in one.run(g, p, Fa=Fa, Fb=Fb, loopProb=LOOP, prior=pr, **kw).items()}
    assert_entry_equal(out, ref, 0, b, [0, int(lens[b])], offs)
    one.close()


def test_graph_replay_equals_direct_launches():
    lens, n = ragged(9, 8, 400), 8
    r = Case(lens, n, seed=9, fb_split=1, opts=dict(graph=1))
    direct = Case(lens, n, seed=9, fb_split=1, opts=dict(graph=2))
    bufs = r.vb.output_buffers(12)
    pr = r.prior()
    g, p = r.fresh()
    ref = direct.run(prior=direct.prior(), maxIters=12, epsilon=1e-6)
    for call in range(4):      # call 0 runs directly, call 1 is captured, calls 2 and 3 replay the graph
        g0, p0 = r.fresh()
        g.copy_(g0)
        p.copy_(p0)
        out = r.vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=LOOP, maxIters=12, epsilon=1e-6, buffers=bufs, prior=pr)
        torch.cuda.synchronize()
        got = {k: out[k].cpu().numpy() for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags')}
        for b in range(len(lens)):
            assert_entry_equal(got, ref, b, b, r.d['offsets'], r.d['offsets'])
    # a different prior is a different call: no replay of the old one
    pr2 = (pr[0] * 0, pr[1] * 0)
    out = r.vb.run(g.copy_(r.fresh()[0]), p.copy_(r.fresh()[1]), Fa=Fa, Fb=Fb, loopProb=LOOP, maxIters=12,
                   epsilon=1e-6, buffers=bufs, prior=pr2)
    torch.cuda.synchronize()
    plain = direct.run(maxIters=12, epsilon=1e-6)
    assert np.array_equal(out['gamma'].cpu().numpy(), plain['gamma'])


def test_host_checks():
    lens, n = ragged(10, 4, 200), 8
    c = Case(lens, n, seed=1)
    pn, pF = c.prior()
    g, p = c.fresh()
    bad = [(pn.float(), pF), (pn, pF[:, :, :64]), (pn[:2], pF), (pn.cpu(), pF), (pn, pF.clone().fill_(np.nan)),
           (-pn - 1, pF), (pn,)]
    for pr in bad:
        with pytest.raises(ValueError):
            c.vb.run(g, p, prior=pr)


# ---- diarize_batch --------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def es():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return dict(z=z, recs={'ES2005a': (z['x_raw'], z['seg_times'])}, transform=(m['mean1'], m['mean2'], m['lda']),
                plda=(m['plda_mu'], m['plda_tr'], m['plda_psi']),
                kw=dict(Fa=float(z['Fa']), Fb=float(z['Fb']), loopP=float(z['loopProb']), smoothing=float(z['smoothing']),
                        threshold=-0.015, max_iters=40, epsilon=1e-6))


def sessions(es, seed=13, n_rec=8, pool=10, spread=2.0):
    """The multi-session archive of test_enroll_gpu.py (pool speakers at random directions `spread` standard deviations
    around ES2005a's mean x-vector, 2 .. 5 per recording, sticky turns) with 20 held-out x-vectors per pool speaker.
    A smaller spread puts the pool centres closer together."""
    x_es = es['z']['x_raw']
    rng = np.random.default_rng(seed)
    sd = x_es.std(0)
    centres = x_es.mean(0) + spread * sd * rng.standard_normal((pool, x_es.shape[1]))
    recs, rows, truth = {}, [], {}
    for r in range(n_rec):
        T = int(rng.integers(300, 601))
        who = rng.choice(pool, 2 + r % 4, replace=False)
        spk = np.zeros(T, dtype=np.int64)
        for t in range(1, T):
            spk[t] = spk[t - 1] if rng.random() < 0.97 else rng.integers(len(who))
        x = centres[who[spk]] + 0.5 * sd * rng.standard_normal((T, x_es.shape[1]))
        seg = np.stack([np.arange(T) * 0.24, np.arange(T) * 0.24 + 1.5], 1)
        name = f'ses{r:02d}'
        recs[name] = (x, seg)
        truth[name] = who[spk]
        rows += [(name, round(t * 0.24, 2), 0.24, f'p{k}') for t, k in enumerate(who[spk])]
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x_es.shape[1])) for k in range(pool)}
    return recs, rows, truth, held


def rows_of(items, key):
    return [tuple(line.split()[1:2]) + (float(line.split()[3]), float(line.split()[4]), line.split()[7])
            for it in items.values() for line in it[key]]


def der(rows, items, key):
    per, tot = score.score_rttm(rows, rows_of(items, key), 0.25, False, by_name=True, across_files=True)
    return ({n: round(100 * v['der'], 2) for n, v in per.items()} if isinstance(per, dict) else per,
            round(100 * tot['by_name']['der'], 2))


@pytest.mark.parametrize('spread', [2.0, 0.7], ids=['separated', 'close'])
def test_pipeline_on_a_synthetic_archive(es, spread):
    recs, rows, truth, held = sessions(es, spread=spread)
    args = (recs, es['transform'], es['plda'])
    theta = 20.0
    ahc = pipeline.diarize_batch(*args, **dict(es['kw'], max_iters=0), init='AHC')
    post = pipeline.diarize_batch(*args, **es['kw'], enroll=held, enroll_threshold=theta)
    got = pipeline.diarize_batch(*args, **es['kw'], enroll=held, enroll_threshold=theta, enroll_prior=True)
    attached = 0
    for n in recs:
        it = got[n]
        for s, name in it['prior_speakers'].items():
            attached += 1
            a = ahc[n]['labels'] == s
            assert f'p{np.bincount(truth[n][a]).argmax()}' == name, (n, s, name)   # no prior across speakers
            mine = it['labels'] == s
            if mine.any():
                assert it['speaker_names'][s] == name
                # with well-separated speakers the state keeps its speaker; with close ones it is only reported
                if spread >= 2.0:
                    assert f'p{np.bincount(truth[n][mine]).argmax()}' == name, (n, s, name)
                else:
                    print(n, s, name, 'holds', np.bincount(truth[n][mine], minlength=10).tolist())
        assert set(it['speaker_llr']) == set(np.unique(it['labels']).tolist())
        names = list(it['speaker_names'].values())
        assert len(set(names)) == len(names)
        want = [l.split()[:7] + [it['speaker_names'][int(l.split()[7]) - 1]] + l.split()[8:] for l in it['rttm']]
        assert [l.split() for l in it['rttm_named']] == want
    assert attached > 0
    print(f'spread {spread}: {attached} priors attached; DER per file / by name, post-hoc enrolment',
          der(rows, post, 'rttm_named'), 'enroll_prior', der(rows, got, 'rttm_named'))


def test_no_match_changes_nothing(es):
    recs, _, _, held = sessions(es, seed=4, n_rec=4)
    args = (recs, es['transform'], es['plda'])
    ovl = {n: [(10.0, 30.0), (50.0, 55.0)] for n in list(recs)[:3]}
    for kw in (dict(), dict(overlaps=ovl, output_2nd=True), dict(link_threshold=0.0)):
        base = pipeline.diarize_batch(*args, **es['kw'], **kw, enroll=held, enroll_threshold=1e9)
        got = pipeline.diarize_batch(*args, **es['kw'], **kw, enroll=held, enroll_threshold=1e9, enroll_prior=True)
        for n in recs:
            assert got[n].pop('prior_speakers') == {}
            assert got[n].keys() == base[n].keys()
            for k in base[n]:
                v, w = got[n][k], base[n][k]
                assert (np.array_equal(v, w) if isinstance(w, np.ndarray) else v == w), (kw, n, k)


def test_composes_with_overlaps_linking_and_a_cohort(es):
    recs, _, truth, held = sessions(es, seed=6, n_rec=5)
    args = (recs, es['transform'], es['plda'])
    ovl = {n: [(10.0, 30.0), (50.0, 55.0)] for n in recs}
    part = {k: v for k, v in list(held.items())[:6]}
    cohort = {k: v for k, v in list(held.items())[6:]}
    for kw in (dict(overlaps=ovl, link_threshold=0.0, output_2nd=True), dict(cohort=cohort, enroll_threshold=3.0)):
        kw = dict(dict(enroll_threshold=20.0), **kw)
        got = pipeline.diarize_batch(*args, **es['kw'], **kw, enroll=part, enroll_prior=True)
        for n in recs:
            it = got[n]
            key = 'rttm_overlap' if 'overlaps' in kw else 'rttm'
            want = [l.split()[:7] + [it['speaker_names'][int(l.split()[7]) - 1]] + l.split()[8:] for l in it[key]]
            assert [l.split() for l in it['rttm_named']] == want
            for s, name in it['prior_speakers'].items():
                if s in it['speaker_names']:
                    assert it['speaker_names'][s] == name
            assert ('speaker_score' in it) == ('cohort' in kw)


def test_command_line_on_es2005a(es, tmp_path):
    from vbx_b200 import cli, formats
    z = es['z']
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    x, seg, ref = z['x_raw'], z['seg_times'], z['labels']
    keys = [f'ES2005a_{i:04d}' for i in range(len(x))]
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, x)
    (tmp_path / 'x.seg').write_text(''.join(f'{k} ES2005a {float(s)!r} {float(e)!r}\n' for k, (s, e) in zip(keys, seg)))
    # each reference speaker enrolled from a slice of its own x-vectors
    enr = {f'spk{l + 1}': x[ref == l][:15] for l in np.unique(ref).tolist() if (ref == l).sum() >= 30}
    ekeys = [f'{k}-{i:02d}' for k, v in enr.items() for i in range(len(v))]
    formats.write_vec_flt_ark(str(tmp_path / 'e.ark'), ekeys, np.concatenate(list(enr.values())))
    (tmp_path / 'e.utt2spk').write_text(''.join(f'{k} {k.rsplit("-", 1)[0]}\n' for k in ekeys))
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), m['plda_mu'], m['plda_tr'], m['plda_psi'])
    np.savez(str(tmp_path / 'transform.npz'), mean1=m['mean1'], mean2=m['mean2'], lda=m['lda'])
    out = tmp_path / 'out'
    argv = ['--init', 'AHC+VB', '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file', str(tmp_path / 'x.seg'),
            '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file', str(tmp_path / 'plda.txt'),
            '--threshold', '-0.015', '--lda-dim', '128', '--Fa', str(z['Fa']), '--Fb', str(z['Fb']), '--loopP',
            str(z['loopProb']), '--init-smoothing', str(z['smoothing']), '--out-rttm-dir', str(out),
            '--enroll-ark', str(tmp_path / 'e.ark'), '--enroll-utt2spk', str(tmp_path / 'e.utt2spk'),
            '--enroll-threshold', '0', '--enroll-prior']
    with redirect_stdout(io.StringIO()):
        assert cli.main(argv) == 0
    enr_read = formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'e.utt2spk'))
    it = pipeline.diarize_batch(es['recs'], es['transform'], es['plda'], **es['kw'], enroll=enr_read,
                                enroll_threshold=0.0, enroll_prior=True)['ES2005a']
    assert (out / 'ES2005a.rttm').read_text().splitlines() == it['rttm_named']
    assert it['prior_speakers']
    for s, name in it['prior_speakers'].items():
        mine = it['labels'] == s
        if mine.any():
            assert f'spk{np.bincount(ref[mine]).argmax() + 1}' == name, (s, name)
    print('ES2005a prior states', it['prior_speakers'], 'LLRs', {k: round(v, 1) for k, v in it['speaker_llr'].items()})
