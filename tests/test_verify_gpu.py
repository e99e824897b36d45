"""Speaker-verification trials on the GPU (DESIGN.md section 5.27): trial scores against the float64 oracle and bit for
bit against the cohort scores of the same pairs, AS-norm against the oracle and bit for bit against the normalised
enrolment scores, the error rates bit for bit against the oracle, the refusals of the Python layer and of the C ABI,
and the command line end to end."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import verify_oracle as O
from test_link_gpu import SPEAKER_WIDTHS, width_phi
from vbx_b200 import _lib, cohort, enroll, formats, pipeline, train, verify

DEV = 'cuda:0'
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
ERR_ARG = -1


def side(M, R, Phi, rng, multi, centres=None):
    """fea [N,R] float32 (items packed, in order) and item [N] of M items: 1 x-vector each, or 1 .. 4 with multi."""
    counts = rng.integers(1, 5, M) if multi else np.ones(M, dtype=np.int64)
    y = rng.standard_normal((M, R)) * np.sqrt(Phi) if centres is None else centres
    item = np.repeat(np.arange(M), counts)
    fea = (y[item] + rng.standard_normal((len(item), R))).astype(np.float32)
    return fea, item


def problem(R, multi, seed, M_e=40, M_t=60, T=2500):
    """Seeded sides and trials; Phi from width_phi at the SPEAKER_WIDTHS."""
    rng = np.random.default_rng(seed)
    Phi = width_phi(rng, R) if R in SPEAKER_WIDTHS else np.sort(rng.uniform(0.2, 8.0, R))[::-1].astype(np.float32)
    fe, ie = side(M_e, R, Phi, rng, multi)
    ft, it = side(M_t, R, Phi, rng, multi)
    tr = np.stack([rng.integers(0, M_e, T), rng.integers(0, M_t, T)], 1)
    tr = np.vstack([tr, tr[:5]])                                        # duplicates are scored twice
    return fe, ie, ft, it, Phi, tr


def oracle_llr(fe, ie, ft, it, Phi, tr, c):
    ne, Fe = O.statistics(fe.astype(np.float64), ie, int(ie.max()) + 1)
    nt, Ft = O.statistics(ft.astype(np.float64), it, int(it.max()) + 1)
    return O.llr_trials(ne, Fe, nt, Ft, Phi.astype(np.float64), c, tr[:, 0], tr[:, 1])


def close(got, want, tol=1e-12):
    err = np.abs(got - want) / np.maximum(np.abs(want), 1.0)
    assert err.max() <= tol, err.max()


@pytest.mark.gpu
@pytest.mark.parametrize('R', [8, 16, 128] + SPEAKER_WIDTHS)
@pytest.mark.parametrize('c', [1.0, 0.3 / 17])
@pytest.mark.parametrize('multi', [False, True])
def test_scores_match_the_oracle(R, c, multi):
    fe, ie, ft, it, Phi, tr = problem(R, multi, R + int(multi))
    got = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=c, Fb=1.0, device=DEV)
    close(got, oracle_llr(fe, ie, ft, it, Phi, tr, c))
    assert got[-5:].tobytes() == got[:5].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize('R, multi', [(16, True), (128, False), (128, True)]
                         + [(R, k % 2 == 0) for k, R in enumerate(SPEAKER_WIDTHS)])
def test_scores_are_the_cohort_scores_bit_for_bit(R, multi):
    Fa, Fb = 0.3, 17.0
    fe, ie, ft, it, Phi, _ = problem(R, multi, 7 * R)
    M_e, M_t = int(ie.max()) + 1, int(it.max()) + 1
    L = cohort.cohort_stats(fe, Phi, None, ie, ft, it, Fa, Fb, top_k=2, device=DEV, scores=True).scores
    ii, jj = np.meshgrid(np.arange(M_e), np.arange(M_t), indexing='ij')
    tr = np.stack([ii.ravel(), jj.ravel()], 1)
    got = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=Fa, Fb=Fb, device=DEV)
    assert got.tobytes() == L.ravel().tobytes()
    swapped = verify.score_trials(ft, it, fe, ie, Phi, tr[:, ::-1], Fa=Fa, Fb=Fb, device=DEV)
    assert swapped.tobytes() == got.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize('R, multi', [(16, True), (128, False), (128, True)]
                         + [(R, k % 2 == 0) for k, R in enumerate(SPEAKER_WIDTHS)])
def test_as_norm_is_the_normalised_enrolment_score_bit_for_bit(R, multi):
    """Enrolment items as the speakers of one recording, test items as the enrolled speakers: every trial's AS-norm
    score is the normalised enrolment score of the same pair."""
    Fa, Fb = 0.3, 17.0
    fe, ie, ft, it, Phi, _ = problem(R, multi, 7 * R)
    fc, ic = side(300, R, Phi, np.random.default_rng(5), True)
    norm = verify.trial_norm(fe, ie, ft, it, Phi, fc, ic, Fa, Fb, top_k=50, device=DEV)
    S = enroll.enroll_speakers(fe, Phi, [0, len(ie)], [ie], ft, it, Fa, Fb, 0.0, device=DEV, llr=True, norm=norm).llr
    ii, jj = np.meshgrid(np.arange(S.shape[0]), np.arange(S.shape[1]), indexing='ij')
    tr = np.stack([ii.ravel(), jj.ravel()], 1)
    got = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=Fa, Fb=Fb, norm=norm, device=DEV)
    assert got.tobytes() == S.ravel().tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize('R, multi', [pytest.param(128, m, id=str(m)) for m in (False, True)]
                         + [(R, k % 2 == 1) for k, R in enumerate(SPEAKER_WIDTHS)])
def test_as_norm_matches_the_oracle(R, multi):
    fe, ie, ft, it, Phi, tr = problem(R, multi, 31 if R == 128 else R)
    rng = np.random.default_rng(5)
    fc, ic = side(300, R, Phi, rng, True)
    norm = verify.trial_norm(fe, ie, ft, it, Phi, fc, ic, 0.3, 17.0, top_k=50, device=DEV)
    got = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=0.3, Fb=17.0, norm=norm, device=DEV)
    want = O.as_norm(oracle_llr(fe, ie, ft, it, Phi, tr, 0.3 / 17.0), *norm, tr[:, 0], tr[:, 1])
    close(got, want)


def check_metrics(s, y, ps=(0.01, 0.1, 0.5)):
    got = verify.error_rates(s, y, ps, device=DEV)
    want = O.error_rates(s, y, ps)
    for k in ('n_target', 'n_nontarget', 'eer', 'min_dcf', 'threshold', 'act_dcf'):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), (k, got[k], want[k])
    assert abs(got['cllr'] - want['cllr']) <= 1e-12 * abs(want['cllr'])
    return got


@pytest.mark.gpu
def test_metrics_on_device_scores():
    fe, ie, ft, it, Phi, tr = problem(128, True, 3, M_e=600, M_t=600, T=20000)
    tr[:100, 1] = tr[:100, 0]
    s = verify.score_trials(fe, ie, ft, it, Phi, tr, Fa=0.3, Fb=17.0, device=DEV)
    y = tr[:, 0] == tr[:, 1]
    assert len(np.unique(s)) > 0.9 * len(s)
    check_metrics(s, y)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['ties', 'one_each', 'signed_zero', 'millions'])
def test_metrics_match_the_oracle_bit_for_bit(case):
    rng = np.random.default_rng(11)
    if case == 'ties':
        y = rng.random(50000) < 0.2
        s = np.round(np.where(y, 1.5, -1.0) + rng.standard_normal(len(y)) * 2)
    elif case == 'one_each':
        s, y = np.array([0.25, 0.75]), np.array([False, True])
        check_metrics(s[::-1].copy(), y[::-1].copy())
    elif case == 'signed_zero':
        s = np.array([-0.0, 0.0, 0.0, -0.0, 1.0, -1.0, -0.0, 2.0])
        y = np.array([1, 0, 1, 0, 0, 1, 1, 0], dtype=bool)
    else:
        y = rng.random(3_000_000) < 0.01
        s = np.where(y, 3.0, -3.0) + rng.standard_normal(len(y)) * 2.5
    got = check_metrics(s, y)
    if case == 'signed_zero':
        assert not any(t == 0.0 and np.signbit(t) for t in got['threshold'])     # -0.0 is reported as +0.0


@pytest.mark.gpu
def test_metrics_are_repeatable_and_ignore_the_order_of_the_trials():
    rng = np.random.default_rng(2)
    y = rng.random(200000) < 0.05
    s = np.round(np.where(y, 2.0, -2.0) + rng.standard_normal(len(y)) * 2, 1)
    a = verify.error_rates(s, y, (0.01, 0.05), device=DEV)
    b = verify.error_rates(s, y, (0.01, 0.05), device=DEV)
    p = rng.permutation(len(s))
    c = verify.error_rates(s[p], y[p], (0.01, 0.05), device=DEV)
    assert a == b == c


@pytest.mark.gpu
def test_metrics_refuse_non_finite_scores():
    s = np.array([0.0, 1.0, np.nan, 2.0])
    with pytest.raises(ValueError, match='non-finite'):
        verify.error_rates(s, np.array([1, 0, 1, 0]), device=DEV)
    with pytest.raises(ValueError, match='non-finite'):
        verify.error_rates(np.array([0.0, np.inf]), np.array([1, 0]), device=DEV)


@pytest.fixture(scope='module')
def handle():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    yield lib, h
    lib.vbx_destroy(h)


@pytest.mark.gpu
def test_c_abi_out_of_range_trials_score_nan_and_bad_arguments_are_refused(handle):
    lib, h = handle
    fe, ie, ft, it, Phi, _ = problem(16, False, 1, M_e=3, M_t=4)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    fe, ie, ft, it, Phi = d(fe), d(ie.astype(np.int32)), d(ft), d(it.astype(np.int32)), d(Phi)
    ti, tj = d(np.array([0, 3, -1, 2, 1], dtype=np.int32)), d(np.array([0, 1, 2, 4, 3], dtype=np.int32))
    need = ctypes.c_size_t()
    assert lib.vbx_verify_score_workspace_bytes(h, 3, 4, ctypes.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    out = torch.full((5,), 7.0, dtype=torch.float64, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    base = [h, p(fe), 3, p(ie), 3, p(ft), 4, p(it), 4, 16, p(Phi), 1.0, 1.0, p(ti), p(tj), 5, None, None, None, None,
            p(ws), ws.numel(), p(out), None]
    assert lib.vbx_verify_score(*base) == 0
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isfinite(o[[0, 4]]).all() and np.isnan(o[[1, 2, 3]]).all()
    for k, v in ((9, 129), (9, 0), (11, 0.0), (12, float('nan')), (4, 0), (15, -1), (21, need.value - 1), (16, p(out)),
                 (1, None), (20, ctypes.c_void_p(ws.data_ptr() + 8))):
        a = list(base)
        a[k] = v
        assert lib.vbx_verify_score(*a) == ERR_ARG, k
    s = d(np.array([0.0, 1.0]))
    y = d(np.array([1, 0], dtype=np.uint8))
    assert lib.vbx_verify_metrics_workspace_bytes(h, 2, 1, ctypes.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    res = torch.empty(8, dtype=torch.float64, device=DEV)
    cnt = torch.empty(3, dtype=torch.int64, device=DEV)
    pt = np.array([0.5])
    at = lambda k: ctypes.c_void_p(res.data_ptr() + 8 * k)
    mb = [h, p(s), p(y), 2, 1, pt.ctypes.data_as(ctypes.c_void_p), 1.0, 1.0, p(ws), ws.numel(), p(cnt), at(0), at(1),
          at(2), at(3), at(4), None]
    assert lib.vbx_verify_metrics(*mb) == 0
    bad_p = np.array([1.0])
    for k, v in ((3, 0), (4, 0), (4, 65), (5, bad_p.ctypes.data_as(ctypes.c_void_p)), (6, 0.0), (7, float('inf')),
                 (9, need.value - 1), (1, None), (10, None)):
        a = list(mb)
        a[k] = v
        assert lib.vbx_verify_metrics(*a) == ERR_ARG, k
    assert lib.vbx_verify_metrics_workspace_bytes(h, 0, 1, ctypes.byref(need)) == ERR_ARG
    assert lib.vbx_verify_score_workspace_bytes(h, 0, 1, ctypes.byref(need)) == ERR_ARG


# ---- command line ------------------------------------------------------------------------------------------------------

def raw_speakers(K, Dx, seed, n):
    """{name: x [n, Dx]} of K synthetic speakers in the raw x-vector space."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((Dx, Dx)))
    within = q * np.exp(np.linspace(0, -2, Dx))[None, :] * 0.6
    centres = rng.standard_normal((K, Dx)) * np.exp(np.linspace(0.5, -1.5, Dx))[None, :]
    return {f's{seed}_{k}': centres[k] + rng.standard_normal((n, Dx)) @ within.T for k in range(K)}


def write_side(root, name, sets, per_item):
    """ark (+ utt2spk when per_item is None: items are speakers) of the speakers' x-vectors; each x-vector its own item
    named <speaker>-<k> otherwise.  Returns (ark, utt2spk or None, item names, speaker of each item)."""
    ark = os.path.join(root, f'{name}.ark')
    keys, vecs, spk = [], [], []
    for s, x in sets.items():
        for k, v in enumerate(x):
            keys.append(f'{s}-{k}')
            vecs.append(v)
            spk.append(s)
    formats.write_vec_flt_ark(ark, keys, vecs)
    if per_item:
        return ark, None, keys, spk
    u = os.path.join(root, f'{name}.utt2spk')
    with open(u, 'w') as f:
        f.write(''.join(f'{k} {s}\n' for k, s in zip(keys, spk)))
    return ark, u, list(sets), list(sets)


@pytest.mark.gpu
def test_command_line_end_to_end(tmp_path):
    root = str(tmp_path)
    model = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    tf = os.path.join(root, 'transform.npz')
    np.savez(tf, mean1=model['mean1'], mean2=model['mean2'], lda=model['lda'])
    plda = os.path.join(root, 'plda')
    formats.write_kaldi_plda_binary(plda, model['plda_mu'], model['plda_tr'], model['plda_psi'])
    spk = raw_speakers(40, 256, 1, 5)
    enrol = {s: x[:3] + model['mean1'] for s, x in spk.items()}
    test = {s: x[3:] + model['mean1'] for s, x in spk.items()}
    e_ark, e_u, e_names, _ = write_side(root, 'enrol', enrol, False)
    t_ark, _, t_names, t_spk = write_side(root, 'test', test, True)
    rng = np.random.default_rng(3)
    trials = os.path.join(root, 'trials')
    rows = [(e_names[a], t_names[b]) for a, b in zip(rng.integers(0, len(e_names), 600),
                                                     rng.integers(0, len(t_names), 600))]
    rows += [(t_spk[b], t_names[b]) for b in range(len(t_names))]
    with open(trials, 'w') as f:
        f.write(''.join(f'{a} {b} {"target" if a == t_spk[t_names.index(b)] else "nontarget"}\n' for a, b in rows))
    out, js = os.path.join(root, 'scores'), os.path.join(root, 'm.json')
    args = ['--trials', trials, '--enroll-ark', e_ark, '--enroll-utt2spk', e_u, '--test-ark', t_ark, '--xvec-transform',
            tf, '--plda-file', plda, '--Fa', '0.3', '--Fb', '17', '--p-target', '0.01,0.2', '--device', DEV]
    assert verify.main(args + ['--scores-out', out, '--json', js]) == 0
    lines = [l.split() for l in open(out)]
    assert [(a, b) for a, b, _ in lines] == rows
    got = np.array([float(v) for _, _, v in lines])
    # the same computation through the Python entry points
    en, xe, ie = verify.read_items(e_ark, e_u)
    tn, xt, it = verify.read_items(t_ark)
    transform, pl = formats.read_xvec_transform(tf), formats.read_kaldi_plda(plda)
    x_all = np.concatenate([xe, xt])
    chain = pipeline._resolve_chain('auto', transform, pl, 128, 256)
    front, _, fea, Phi = pipeline._project(x_all, [len(x_all)], transform, pl, 128, chain, torch.device(DEV))
    front.close()
    fea, Phi = fea.cpu().numpy(), Phi.cpu().numpy()
    tr = np.array([[en.index(a), tn.index(b)] for a, b in rows])
    want = verify.score_trials(fea[:len(xe)], ie, fea[len(xe):], it, Phi, tr, Fa=0.3, Fb=17.0, device=DEV)
    assert got.tobytes() == want.tobytes()
    doc = json.load(open(js))
    y = np.array([a == t_spk[t_names.index(b)] for a, b in rows])
    ref = O.error_rates(got, y, (0.01, 0.2))
    assert doc['score_kind'] == 'llr' and doc['n_target'] == int(y.sum()) and doc['n_trials'] == len(rows)
    assert doc['eer'] == ref['eer']
    for k, op in enumerate(doc['operating_points']):
        assert (op['min_dcf'], op['threshold'], op['act_dcf']) == (ref['min_dcf'][k], ref['threshold'][k],
                                                                   ref['act_dcf'][k])
    assert abs(doc['cllr'] - ref['cllr']) <= 1e-12 * ref['cllr']
    # AS-norm against a cohort of other speakers
    c_ark, c_u, _, _ = write_side(root, 'cohort', {s: x + model['mean1'] for s, x in raw_speakers(30, 256, 2, 3).items()},
                                  False)
    assert verify.main(args + ['--cohort-ark', c_ark, '--cohort-utt2spk', c_u, '--cohort-top', '10', '--json', js]) == 0
    assert json.load(open(js))['score_kind'] == 'as-norm'


@pytest.mark.gpu
def test_command_line_takes_trains_output(tmp_path):
    root = str(tmp_path)
    Dx, d = 64, 24
    train_sets = raw_speakers(80, Dx, 5, 8)
    t_ark, t_u, _, _ = write_side(root, 'train', train_sets, False)
    mdir = os.path.join(root, 'model')
    assert train.main(['--xvec-ark-file', t_ark, '--utt2spk', t_u, '--out-dir', mdir, '--lda-dim', str(d),
                       '--device', DEV]) == 0
    held = raw_speakers(20, Dx, 9, 4)
    e_ark, _, e_names, e_spk = write_side(root, 'enrol', held, True)
    trials = os.path.join(root, 'trials')
    with open(trials, 'w') as f:
        f.write(''.join(f'{a} {b}\n' for a in e_names[:10] for b in e_names[10:]))
    out = os.path.join(root, 'scores')
    assert verify.main(['--trials', trials, '--enroll-ark', e_ark, '--test-ark', e_ark, '--xvec-transform',
                        os.path.join(mdir, 'transform.npz'), '--plda-file', os.path.join(mdir, 'plda'), '--lda-dim',
                        str(d), '--device', DEV, '--scores-out', out]) == 0
    v = np.array([float(l.split()[2]) for l in open(out)])
    assert len(v) == 10 * (len(e_names) - 10)
    # the float64 oracle on the trained model's projection of the same x-vectors (both sides read from one ark)
    names, x, item = verify.read_items(e_ark)
    transform = formats.read_xvec_transform(os.path.join(mdir, 'transform.npz'))
    pl = formats.read_kaldi_plda(os.path.join(mdir, 'plda'))
    x_all = np.concatenate([x, x])
    chain = pipeline._resolve_chain('auto', transform, pl, d, Dx)
    front, _, fea, Phi = pipeline._project(x_all, [len(x_all)], transform, pl, d, chain, torch.device(DEV))
    front.close()
    fea, Phi = fea.cpu().numpy(), Phi.cpu().numpy()
    assert fea.shape == (2 * len(x), d)
    tr = np.array([[names.index(a), names.index(b)] for a in e_names[:10] for b in e_names[10:]])
    close(v, oracle_llr(fea[:len(x)], item, fea[len(x):], item, Phi, tr, 1.0))
