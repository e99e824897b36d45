"""The S = 128 state tier (65 .. 128 live states) of the batched float32 VB-HMM against the float64 C oracle, and the
state tiers of diarize_batch on the shipped ES2005a inputs.

Bars as in test_parity_gpu.py: max|d gamma| <= 1e-4, max|d pi| <= 1e-4, per-iteration |d ELBO| <= 1e-4 |ELBO|,
identical iteration counts."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import c_oracle as co
from vbx_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
TOL = 1e-4
HP = dict(Fa=0.3, Fb=17.0, loopProb=0.99)


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def masked_inputs(lens, n, ns, seed, R=128):
    """Batch with n user columns; recording b keeps its first ns[b] states (gamma0 renormalised, pi0 uniform)."""
    d = synth.make_batch(lens, R=R, S=n, seed=seed, dtype=np.float32)
    g0 = d['gamma0'].astype(np.float64)
    pi0 = np.zeros((len(lens), n))
    for b, (lo, hi) in enumerate(zip(d['offsets'][:-1], d['offsets'][1:])):
        g0[lo:hi, ns[b]:] = 0
        g0[lo:hi] /= g0[lo:hi].sum(1, keepdims=True)
        pi0[b, :ns[b]] = 1.0 / ns[b]
    return d, g0, pi0


def run128(fea, Phi, lens, g0, pi0, ns, gemm=0, warm=None, graph=0, **kw):
    from vbx_b200.batch import VbxBatch
    n = g0.shape[1]
    vb = VbxBatch(lens, fea.shape[1], ns, device=dev())
    assert vb.S == 128
    vb.workspace.fill_(0xFF)       # poison (NaN in float32 and float64): nothing may be read before it is written
    vb.set_option('gemm', gemm)
    vb.set_option('graph', graph)
    g = torch.zeros((fea.shape[0], 128), device=dev())
    g[:, :n] = cuda(g0)
    p = torch.zeros((len(lens), 128), device=dev())
    p[:, :n] = cuda(pi0)
    vb.prepare_scale(cuda(fea), cuda(Phi))
    extra = {}
    if warm is not None:
        a = torch.zeros((len(lens), 128, fea.shape[1]), device=dev())
        il = torch.zeros_like(a)
        a[:, :n] = cuda(warm[0])
        il[:, :n] = cuda(warm[1])
        extra = dict(alpha=a, invL=il, warm_start=True)
    out = vb.run(g, p, return_model=True, **extra, **kw)
    torch.cuda.synchronize()
    res = dict(gamma=g[:, :n].double().cpu().numpy(), pi=p[:, :n].double().cpu().numpy(), Li=out['Li'].cpu().numpy(),
               n_iters=out['n_iters'].cpu().numpy(), flags=out['flags'].cpu().numpy(),
               alpha=out['alpha'][:, :n].double().cpu().numpy(), invL=out['invL'][:, :n].double().cpu().numpy(),
               gamma_pad=g[:, n:].cpu().numpy(), ws=vb.workspace_bytes)
    vb.close()
    return res


def check(out, ref, n_iters=None):
    assert np.array_equal(out['n_iters'], ref['n_iters'] if n_iters is None else n_iters), (out['n_iters'], ref['n_iters'])
    assert np.abs(out['gamma'] - ref['gamma']).max() <= TOL
    assert np.abs(out['pi'] - ref['pi']).max() <= TOL
    for b in range(len(out['n_iters'])):
        m = int(out['n_iters'][b])
        np.testing.assert_allclose(out['Li'][b, :m], ref['Li'][b, :m], rtol=TOL)
        assert np.all(np.isnan(out['Li'][b, m:]))
    assert np.all(out['gamma_pad'] == 0)


def ragged_lens(seed, B=12, tmax=900):
    lens = np.random.default_rng(seed).integers(1, tmax, size=B)
    lens[:5] = [1, 2, 511, 512, 513]
    return lens


@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('ragged', [False, True], ids=['uniform', 'ragged'])
@pytest.mark.parametrize('n', [65, 100, 127, 128])
def test_live_states_vs_oracle(n, ragged, gemm):
    lens = ragged_lens(n)
    ns = np.full(len(lens), n, dtype=np.int32)
    if ragged:                         # per-recording live states, including 1 and 3 inside the S = 128 plan
        ns = np.random.default_rng(n + 1).integers(65, n + 1, size=len(lens)).astype(np.int32)
        ns[[1, 5]] = [1, 3]
        ns[2] = n
    d, g0, pi0 = masked_inputs(lens, n, ns, seed=n)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, HP['Fa'], HP['Fb'], HP['loopProb'], 6, -np.inf, n_states=ns)
    out = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, gemm=gemm, maxIters=6, epsilon=-np.inf, **HP)
    check(out, ref)
    assert np.abs(out['alpha'] - ref['alpha']).max() <= TOL * max(1.0, np.abs(ref['alpha']).max())
    assert not np.any(out['flags'] & 1)


def test_long_recordings_take_the_split_schedule():
    """Recordings >= 4096 frames (12 000 as in BASELINE config 4) at S = 128: the plan is the split one whatever fb_split
    says (same workspace as fb_split = 1), and fb_split = 2 is refused."""
    from vbx_b200.batch import VbxBatch
    from vbx_b200._lib import VbxError
    lens = np.array([12000, 4096, 300, 5000])
    n = 100
    ns = np.array([100, 90, 100, 70], dtype=np.int32)
    ws = [VbxBatch(lens, 128, ns, device=dev(), allocate=False, fb_split=f).workspace_bytes for f in (0, 1)]
    assert ws[0] == ws[1]
    with pytest.raises(VbxError, match='split'):
        VbxBatch(lens, 128, ns, device=dev(), allocate=False, fb_split=2)
    d, g0, pi0 = masked_inputs(lens, n, ns, seed=4)
    kw = dict(Fa=0.2, Fb=6.0, loopProb=0.35)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, kw['Fa'], kw['Fb'], kw['loopProb'], 6, -np.inf, n_states=ns)
    out = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, maxIters=6, epsilon=-np.inf, **kw)
    check(out, ref)
    assert np.abs(out['gamma'].sum(1) - 1).max() < 1e-5


@pytest.mark.parametrize('gemm', [0, 1], ids=['mma3xtf32', 'ffma'])
@pytest.mark.parametrize('eps', [1e-4, 1e-6])
def test_stop_rule_at_float64_resolution(eps, gemm):
    """Finite epsilon with exact_stop: recordings finish in the float64 kernels (vbx_exact64.cu at S = 128) and stop at
    exactly the oracle's iteration."""
    lens = ragged_lens(7, B=10, tmax=700)
    ns = np.random.default_rng(8).integers(65, 129, size=len(lens)).astype(np.int32)
    d, g0, pi0 = masked_inputs(lens, 128, ns, seed=11)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, HP['Fa'], HP['Fb'], HP['loopProb'], 40, eps, n_states=ns)
    assert len(set(ref['n_iters'].tolist())) > 1
    out = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, gemm=gemm, maxIters=40, epsilon=eps, **HP)
    check(out, ref)
    for b in range(len(lens)):
        assert bool(out['flags'][b] & 4) == (ref['n_iters'][b] < 40)
    assert np.abs(out['alpha'] - ref['alpha']).max() <= TOL * max(1.0, np.abs(ref['alpha']).max())
    assert np.abs(out['invL'] - ref['invL']).max() <= TOL


def test_warm_start_and_model_output():
    lens = ragged_lens(12, B=6, tmax=600)
    ns = np.array([128, 100, 65, 3, 1, 127], dtype=np.int32)
    d, g0, pi0 = masked_inputs(lens, 128, ns, seed=12)
    start = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, HP['Fa'], HP['Fb'], HP['loopProb'], 2, -np.inf, n_states=ns)
    a0, il0 = start['alpha'], start['invL']
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, HP['Fa'], HP['Fb'], HP['loopProb'], 5, -np.inf,
                              n_states=ns, alpha0=a0, invL0=il0)
    out = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, warm=(a0, il0), maxIters=5, epsilon=-np.inf, **HP)
    check(out, ref)
    assert np.abs(out['alpha'] - ref['alpha']).max() <= TOL * max(1.0, np.abs(ref['alpha']).max())
    assert np.abs(out['invL'] - ref['invL']).max() <= TOL


def test_deterministic_independent_and_partitioned():
    """Two runs are bit-identical; a recording alone (an S = 128 split plan of its own) equals the same recording inside
    the batch; a parts.py-partitioned batch equals the whole batch."""
    from vbx_b200.parts import make_batch
    lens = ragged_lens(21, B=9, tmax=800)
    ns = np.random.default_rng(22).integers(65, 129, size=len(lens)).astype(np.int32)
    d, g0, pi0 = masked_inputs(lens, 128, ns, seed=21)
    kw = dict(maxIters=25, epsilon=1e-5, **HP)
    full = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, **kw)
    again = run128(d['fea'], d['Phi'], lens, g0.astype(np.float32), pi0, ns, **kw)
    for k in ('gamma', 'pi', 'Li', 'n_iters', 'alpha'):
        assert np.array_equal(full[k], again[k], equal_nan=True), k
    for b in (0, 3, 8):
        lo, hi = d['offsets'][b], d['offsets'][b + 1]
        one = run128(d['fea'][lo:hi], d['Phi'], [hi - lo], g0[lo:hi].astype(np.float32), pi0[b:b + 1], ns[b:b + 1], **kw)
        assert np.array_equal(one['gamma'], full['gamma'][lo:hi])
        assert np.array_equal(one['pi'][0], full['pi'][b])
        assert np.array_equal(one['Li'][0], full['Li'][b], equal_nan=True)
    results = []
    for parts in (1, 2):
        vb = make_batch(lens, 128, ns, device=dev(), parts=parts)
        g = torch.zeros((int(lens.sum()), vb.S), device=dev())
        g[:, :128] = cuda(g0)
        p = cuda(pi0)
        vb.prepare_scale(cuda(d['fea']), cuda(d['Phi']))
        out = vb.run(g, p, return_model=True, **kw)
        lab = vb.hard_labels(g)
        torch.cuda.synchronize()
        results.append([t.cpu().numpy() for t in (g, p, out['Li'], out['n_iters'], out['alpha'], lab)])
        vb.close()
    for a, b in zip(*results):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.array_equal(results[0][0][:, :128], full['gamma'].astype(np.float32))


@pytest.mark.parametrize('eps', [-np.inf, 1e-5])
def test_cuda_graph_replay_is_identical(eps):
    from vbx_b200.batch import VbxBatch
    lens = ragged_lens(31, B=7, tmax=400)
    n = 100
    ns = np.full(len(lens), n, dtype=np.int32)
    d, g0, pi0 = masked_inputs(lens, n, ns, seed=31)
    vb = VbxBatch(lens, 128, ns, device=dev())
    vb.set_option('graph', 1)
    gi = torch.zeros((int(lens.sum()), 128), device=dev())
    gi[:, :n] = cuda(g0)
    g, p = torch.empty_like(gi), torch.empty((len(lens), 128), device=dev())
    vb.prepare_scale(cuda(d['fea']), cuda(d['Phi']))
    Li = torch.empty((len(lens), 30), dtype=torch.float64, device=dev())
    ni = torch.empty(len(lens), dtype=torch.int32, device=dev())
    fl = torch.empty(len(lens), dtype=torch.int32, device=dev())
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    outs = []
    for rep in range(4):           # run 0 direct, run 1 captured, runs 2-3 replayed
        g.copy_(gi)
        p.zero_()
        p[:, :n] = 1.0 / n
        vb._check(vb.lib.vbx_run(vb._h, ptr(vb.rho), ptr(vb.Phi), ptr(g), ptr(p), None, HP['Fa'], HP['Fb'], HP['loopProb'], 30,
                                 float(eps), None, None, 0, ptr(Li), ptr(ni), ptr(fl), vb._stream()))
        torch.cuda.synchronize()
        outs.append([t.clone().cpu().numpy() for t in (g, p, Li, ni, fl)])
    vb.close()
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b, equal_nan=True)
    ref = co.vbx_oracle_batch(d['fea'], d['Phi'], d['offsets'], g0, pi0, HP['Fa'], HP['Fb'], HP['loopProb'], 30, eps)
    assert np.array_equal(outs[0][3], ref['n_iters'])
    assert np.abs(outs[0][0][:, :n] - ref['gamma']).max() <= TOL


def test_hard_labels_at_128_states():
    """vbx_hard_labels = argsort(-gamma)[:, :2] over the live states (stable: ties go to the lower state), -1 as the
    runner-up of a one-state recording."""
    from vbx_b200.batch import VbxBatch
    lens = np.array([1, 63, 64, 65, 300, 2])
    ns = np.array([128, 100, 1, 65, 127, 3], dtype=np.int32)
    rng = np.random.default_rng(5)
    N = int(lens.sum())
    g = rng.random((N, 128)).astype(np.float32)
    g[::7, 10] = g[::7, 40] = 2.0               # ties for first place
    g[::5, 3] = g[::5, 90] = g[::5, 100] = 1.5  # ties for second place behind column 0
    g[::5, 0] = 3.0
    vb = VbxBatch(lens, 128, ns, device=dev(), allocate=False)
    first, second = vb.hard_labels(cuda(g), second=True)
    first, second = first.cpu().numpy(), second.cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        rows = g[offs[b]:offs[b + 1], :ns[b]]
        order = np.argsort(-rows, axis=1, kind='stable')
        assert np.array_equal(first[offs[b]:offs[b + 1]], order[:, 0])
        want2 = order[:, 1] if ns[b] > 1 else np.full(len(rows), -1)
        assert np.array_equal(second[offs[b]:offs[b + 1]], want2)
    vb.close()


def test_c_abi_plan():
    import vbx_b200._lib as L
    lib = L.load()
    assert [lib.vbx_padded_states_wide(n) for n in (1, 64, 65, 128, 129)] == [4, 64, 128, 128, -1]
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    offs = np.array([0, 100, 613], dtype=np.int64)
    po = offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    need = ctypes.c_size_t()
    assert lib.vbx_plan(h, po, 2, 128, 128, ctypes.byref(need)) == 0 and need.value > 0
    for S in (96, 256):
        assert lib.vbx_plan(h, po, 2, 128, S, ctypes.byref(need)) == -1
    assert lib.vbx_set_option(h, b'fb_split', 2) == 0
    assert lib.vbx_plan(h, po, 2, 128, 128, ctypes.byref(need)) == -1
    assert b'split' in lib.vbx_last_error(h)
    assert lib.vbx_plan(h, po, 2, 128, 64, ctypes.byref(need)) == 0
    assert lib.vbx_destroy(h) == 0


# ---- diarize_batch on the shipped ES2005a inputs ---------------------------------------------------------------------

def es_model():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return z, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])


def es_oracle(z, threshold, max_iters=40, eps=1e-6):
    from oracle.ahc_oracle import ahc_labels
    lab = ahc_labels(z["x_lda"], threshold)[0]
    S = int(lab.max()) + 1
    q = np.exp(np.eye(S)[lab] * float(z['smoothing']))
    q /= q.sum(1, keepdims=True)
    T = len(lab)
    ref = co.vbx_oracle_batch(z['fea'], z['Phi'], np.array([0, T]), q, np.full(S, 1.0 / S), float(z['Fa']), float(z['Fb']),
                              float(z['loopProb']), max_iters, eps)
    return lab, q, ref


@pytest.mark.parametrize('threshold,clusters', [(0.1, 80), (0.15, 108), (0.2, 144)])
def test_diarize_batch_state_tiers_es2005a(threshold, clusters):
    """80 and 108 AHC clusters run on the S = 128 float32 tier, 144 on the float64 kernels: AHC labels equal the CPU
    oracle's, and VB labels and iteration counts equal the float64 oracle's from the same initialisation."""
    from vbx_b200 import pipeline
    z, transform, plda = es_model()
    lab, q, ref = es_oracle(z, threshold)
    assert lab.max() + 1 == clusters
    T = len(lab)
    res = pipeline.diarize_batch({'ES2005a': (z['x_raw'], z['seg_times'])}, transform, plda, float(z['Fa']), float(z['Fb']),
                                 float(z['loopProb']), threshold=threshold, smoothing=float(z['smoothing']), chain='float64',
                                 device=dev())['ES2005a']
    ahc = pipeline.diarize_batch({'ES2005a': (z['x_raw'], z['seg_times'])}, transform, plda, float(z['Fa']), float(z['Fb']),
                                 float(z['loopProb']), threshold=threshold, init='AHC', chain='float64', device=dev())['ES2005a']
    assert np.array_equal(ahc['labels'], lab)
    assert res['iterations'] == int(ref['n_iters'][0])
    assert np.array_equal(res['labels'], np.argsort(-ref['gamma'], axis=1, kind='stable')[:, 0])
    assert len(res['rttm']) > 0
    if clusters <= 128:              # the float32 tier's gamma from the same initialisation
        out = run128(z['fea'].astype(np.float32), z['Phi'].astype(np.float32), [T], q.astype(np.float32), np.full((1, clusters), 1.0 / clusters),
                     np.array([clusters], dtype=np.int32), maxIters=40, epsilon=1e-6, Fa=float(z['Fa']), Fb=float(z['Fb']),
                     loopProb=float(z['loopProb']))
        check(out, ref)


def test_mixed_archive_keeps_small_recordings_bit_identical():
    """ES2005a at threshold 0.15 (108 clusters) next to short excerpts that stay <= 64 clusters, in one call: the excerpts
    give the same RTTM, labels and iterations as an archive without ES2005a."""
    from vbx_b200 import pipeline
    z, transform, plda = es_model()
    small = {f'part{i}': (z['x_raw'][a:b], z['seg_times'][a:b]) for i, (a, b) in enumerate([(0, 150), (300, 420), (600, 900)])}
    kw = dict(threshold=0.15, smoothing=float(z['smoothing']), device=dev())
    args = (transform, plda, float(z['Fa']), float(z['Fb']), float(z['loopProb']))
    alone = pipeline.diarize_batch(small, *args, **kw)
    mixed = pipeline.diarize_batch({'ES2005a': (z['x_raw'], z['seg_times']), **small}, *args, **kw)
    assert len(set(mixed['ES2005a']['labels'].tolist())) >= 1 and mixed['ES2005a']['rttm']
    for name, want in alone.items():
        assert max(int(np.max(want['labels'])) + 1, 1) <= 64
        got = mixed[name]
        assert got['rttm'] == want['rttm'], name
        assert np.array_equal(got['labels'], want['labels']), name
        assert got['iterations'] == want['iterations'], name


def test_command_line_writes_every_rttm(tmp_path):
    """`python -m vbx_b200.cli ... --threshold 0.15` (108 AHC clusters on ES2005a) writes an RTTM for every recording."""
    from vbx_b200 import cli, formats
    z, transform, plda = es_model()
    keys, seg_lines, rows = [], [], []
    for rec, (a, b) in (('ES2005a', (0, len(z['x_raw']))), ('SHORT', (0, 200))):
        for i in range(a, b):
            s, e = z['seg_times'][i]
            k = f'{rec}_{i:04d}-{int(round(s * 100)):08d}-{int(round(e * 100)):08d}'
            keys.append(k)
            seg_lines.append(f'{k} {rec} {float(s)!r} {float(e)!r}')
            rows.append(z['x_raw'][i])
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, np.stack(rows))
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    rc = cli.main(['--init', 'AHC+VB', '--out-rttm-dir', str(tmp_path / 'out'), '--xvec-ark-file', str(tmp_path / 'x.ark'),
                   '--segments-file', str(tmp_path / 'x.seg'), '--xvec-transform', str(tmp_path / 'transform.npz'),
                   '--plda-file', str(tmp_path / 'plda.txt'), '--threshold', '0.15', '--lda-dim', '128', '--Fa', '0.3',
                   '--Fb', '17', '--loopP', '0.99'])
    assert rc == 0
    for rec in ('ES2005a', 'SHORT'):
        got = formats.read_rttm(str(tmp_path / 'out' / f'{rec}.rttm'))
        assert len(got) > 0 and all(r == rec for r, _, _, _ in got)
