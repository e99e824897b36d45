"""Score calibration on the GPU (DESIGN.md section 5.28): vbx_verify_calibrate against the float64 oracle (the fit,
minCllr and the hull), its invariance to the order of the trials, its agreement with vbx_verify_metrics, a 10 M-trial
list with a known answer, the statuses, the C ABI's refusals, and the command lines end to end: verify --calibrate-out
on a trained model, then the diarization command line with --calibration against the raw thresholds."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import calibrate_oracle as O
from test_adapt_gpu import ES, read_dir, write_archive
from test_verify_gpu import write_side
from vbx_b200 import _lib, cli, synth, train, verify

DEV = 'cuda:0'
ERR_ARG = -1


def random_list(seed, T, ties, frac=0.3, sep=1.5):
    rng = np.random.default_rng(seed)
    y = rng.random(T) < frac
    y[:2] = [True, False]
    s = rng.standard_normal(T) * 2.0 + sep * y
    if ties:
        s = np.round(s * 4) / 4
    return s, y


def rel(got, want):
    return abs(got - want) / max(abs(want), 1e-300)


@pytest.mark.gpu
def test_worked_case():
    s = np.array([3.0, 1.0, 1.0, 2.0, 1.0, 0.0, -1.0])
    y = np.array([1, 1, 1, 0, 0, 0, 0], dtype=bool)
    c = verify.calibrate(s, y, device=DEV)
    assert rel(c['a'], 1.0775784972559423) <= 1e-10 and rel(c['b'], -1.1648381046978393) <= 1e-10
    assert rel(c['cllr_prior'], 0.8034306752311062) <= 1e-12
    assert rel(c['min_cllr'], 0.5747164126866467) <= 1e-12
    assert (c['hull_vertices'], c['n_target'], c['n_nontarget']) == (4, 3, 4)
    c = verify.calibrate(s, y, prior=0.01, device=DEV)
    assert rel(c['a'], 1.2683733645220252) <= 1e-10 and rel(c['b'], -1.4891900440709454) <= 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('prior', [0.5, 0.01])
@pytest.mark.parametrize('ties', [False, True])
@pytest.mark.parametrize('T', [50, 3000, 200000])
def test_matches_the_oracle(T, ties, prior):
    s, y = random_list(T + int(ties), T, ties)
    got = verify.calibrate(s, y, prior=prior, device=DEV)
    want = O.calibrate(s, y, prior)
    assert want['status'] == 0
    for k in ('a', 'b', 'cllr_prior'):
        assert rel(got[k], want[k]) <= 1e-10, k
    assert rel(got['min_cllr'], want['min_cllr']) <= 1e-12
    assert got['hull_vertices'] == want['hull_vertices']
    assert got['passes'] == want['passes']
    assert (got['n_target'], got['n_nontarget']) == (int(y.sum()), int((~y).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize('ties', [False, True])
def test_bit_identical_under_permutation_and_repeats(ties):
    s, y = random_list(7, 100000, ties)
    a = verify.calibrate(s, y, device=DEV)
    p = np.random.default_rng(1).permutation(len(s))
    b = verify.calibrate(s[p], y[p], device=DEV)
    c = verify.calibrate(s, y, device=DEV)
    assert a == b == c


@pytest.mark.gpu
@pytest.mark.parametrize('ties', [False, True])
def test_cllr_prior_is_the_cllr_of_the_calibrated_scores(ties):
    s, y = random_list(11, 20000, ties)
    c = verify.calibrate(s, y, device=DEV)
    m = verify.error_rates(c['a'] * s + c['b'], y, device=DEV)
    assert rel(c['cllr_prior'], m['cllr']) <= 1e-12
    assert c['min_cllr'] <= c['cllr_prior']
    # an increasing affine map that keeps the distinct scores distinct leaves EER and minDCF as they are
    raw = verify.error_rates(s, y, p_targets=(0.01, 0.2), device=DEV)
    cal_s = c['a'] * s + c['b']
    assert len(np.unique(cal_s)) == len(np.unique(s))
    cal = verify.error_rates(cal_s, y, p_targets=(0.01, 0.2), device=DEV)
    assert cal['eer'] == raw['eer'] and cal['min_dcf'] == raw['min_dcf']


@pytest.mark.gpu
def test_ten_million_trials_recover_the_true_calibration():
    """Scores N(+mu, sigma^2) for targets and N(-mu, sigma^2) for nontargets: the LLR is (2 mu / sigma^2) s."""
    rng = np.random.default_rng(5)
    T, mu, sigma = 10_000_000, 1.0, 1.5
    y = rng.random(T) < 0.1
    s = np.where(y, mu, -mu) + sigma * rng.standard_normal(T)
    c = verify.calibrate(torch.from_numpy(s).to(DEV), y, device=DEV)
    assert abs(c['a'] / (2 * mu / sigma ** 2) - 1) <= 0.01
    assert abs(c['b']) <= 0.01
    assert 0 < c['min_cllr'] <= c['cllr_prior']


@pytest.mark.gpu
def test_statuses():
    y = np.array([1, 1, 0, 0, 0], dtype=bool)
    with pytest.raises(ValueError, match='separable.*at or above'):
        verify.calibrate(np.array([2.0, 1.0, 1.0, 0.0, -1.0]), y, device=DEV)
    with pytest.raises(ValueError, match='separable.*at or below'):
        verify.calibrate(np.array([-2.0, -1.0, 1.0, 0.0, 3.0]), y, device=DEV)
    with pytest.raises(ValueError, match='non-finite'):
        verify.calibrate(np.array([2.0, np.nan, 1.0, 0.0, -1.0]), y, device=DEV)
    with pytest.raises(ValueError, match='non-finite'):
        verify.calibrate(np.array([2.0, 0.5, 1.0, np.inf, -1.0]), y, device=DEV)


def call(lib, h, s, y, prior=0.5):
    need = ctypes.c_size_t()
    assert lib.vbx_verify_calibrate_workspace_bytes(h, len(s), ctypes.byref(need)) == 0
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    ts, ty = d(s), d(y.astype(np.uint8))
    ws = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    info = torch.full((5,), -7, dtype=torch.int64, device=DEV)
    out = torch.empty(4, dtype=torch.float64, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    args = [h, p(ts), p(ty), len(s), prior, p(ws), ws.numel(), p(info), p(out), None]
    return args, info, out, need.value, (ts, ty, ws)


@pytest.mark.gpu
def test_c_abi_statuses_and_refusals():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    try:
        y = np.array([1, 1, 0, 0, 0], dtype=bool)
        for s, status in (([2.0, 1.0, 1.0, 0.0, -1.0], 1), ([2.0, 1.0, 3.0, 0.0, -1.0], 0),
                          ([2.0, 1.0, np.nan, 0.0, -1.0], 2), ([2.0, 2.0, 2.0, 2.0, 2.0], 1)):
            args, info, out, need, keep = call(lib, h, np.array(s), y)
            assert lib.vbx_verify_calibrate(*args) == 0
            torch.cuda.synchronize()
            i, o = info.cpu().numpy(), out.cpu().numpy()
            assert i[0] == status and (i[2], i[3]) == (2, 3), (s, i)
            if status == 1:
                assert i[1] == 0 and np.isnan(o[:3]).all() and np.isfinite(o[3])
            if status == 2:
                assert np.isnan(o).all()
        # fully separable: minCllr exactly 0
        args, info, out, need, keep = call(lib, h, np.array([2.0, 1.5, 1.0, 0.0, -1.0]), y)
        assert lib.vbx_verify_calibrate(*args) == 0
        torch.cuda.synchronize()
        assert out.cpu().numpy()[3] == 0.0 and info.cpu().numpy()[4] == 3
        # a single trial's class is missing: status 1
        args, info, out, need, keep = call(lib, h, np.array([1.0]), np.array([True]))
        assert lib.vbx_verify_calibrate(*args) == 0
        torch.cuda.synchronize()
        assert info.cpu().numpy()[0] == 1
        args, info, out, need, keep = call(lib, h, np.array([2.0, 1.0, 3.0, 0.0, -1.0]), y)
        for k, v in ((3, 0), (4, 0.0), (4, 1.0), (4, float('nan')), (6, need - 1), (1, None), (7, None), (8, None),
                     (5, ctypes.c_void_p(keep[2].data_ptr() + 8))):
            a = list(args)
            a[k] = v
            assert lib.vbx_verify_calibrate(*a) == ERR_ARG, k
        need_out = ctypes.c_size_t()
        assert lib.vbx_verify_calibrate_workspace_bytes(h, 0, ctypes.byref(need_out)) == ERR_ARG
    finally:
        lib.vbx_destroy(h)


# ---- command lines -----------------------------------------------------------------------------------------------------

HYPER = ['--Fa', str(float(ES['Fa'])), '--Fb', str(float(ES['Fb'])), '--loopP', str(float(ES['loopProb']))]


@pytest.mark.gpu
def test_command_lines_end_to_end(tmp_path):
    root = str(tmp_path)
    d = 24
    # a model trained on one synthetic archive's speakers
    trn, _, truth = synth.multi_session_archive(ES['x_raw'], n_rec=10, pool=60, seed=41)
    sets = {}
    for name, (x, _) in trn.items():
        for k, v in zip(truth[name].tolist(), x):
            sets.setdefault(f'p{k}', []).append(v)
    t_ark, t_u, _, _ = write_side(root, 'train', {k: np.array(v) for k, v in sets.items()}, False)
    mdir = os.path.join(root, 'model')
    assert train.main(['--xvec-ark-file', t_ark, '--utt2spk', t_u, '--out-dir', mdir, '--lda-dim', str(d),
                       '--device', DEV]) == 0
    tf, plda = os.path.join(mdir, 'transform.npz'), os.path.join(mdir, 'plda')
    # trials of held-out speakers at the diarization's Fa / Fb: enrolment items are speakers, test items x-vectors
    held, _, htruth = synth.multi_session_archive(ES['x_raw'], n_rec=6, pool=30, seed=43)
    spk = {}
    for name, (x, _) in held.items():
        for k, v in zip(htruth[name].tolist(), x):
            spk.setdefault(f'h{k}', []).append(v)
    rng = np.random.default_rng(47)                 # extra noise, so that the classes overlap
    spk = {k: np.array(v) + 1.5 * ES['x_raw'].std(0) * rng.standard_normal((len(v), ES['x_raw'].shape[1]))
           for k, v in spk.items() if len(v) >= 8}
    e_ark, e_u, e_names, _ = write_side(root, 'enrol', {k: v[:2] for k, v in spk.items()}, False)
    v_ark, _, v_names, v_spk = write_side(root, 'test', {k: v[4:8] for k, v in spk.items()}, True)
    trials = os.path.join(root, 'trials')
    with open(trials, 'w') as f:
        f.write(''.join(f'{a} {b} {"target" if a == s else "nontarget"}\n' for a in e_names
                        for b, s in zip(v_names, v_spk)))
    cal_path, js = os.path.join(root, 'cal.json'), os.path.join(root, 'm.json')
    vargs = ['--trials', trials, '--enroll-ark', e_ark, '--enroll-utt2spk', e_u, '--test-ark', v_ark,
             '--xvec-transform', tf, '--plda-file', plda, '--lda-dim', str(d), '--device', DEV] + HYPER[:4]
    assert verify.main(vargs + ['--json', os.path.join(root, 'raw.json')]) == 0
    assert verify.main(vargs + ['--calibrate-out', cal_path, '--json', js]) == 0
    cal = verify.read_calibration(cal_path)
    doc = json.load(open(js))
    assert doc['calibration']['self_calibrated'] and doc['calibration']['a'] == cal['a'] > 0
    assert doc['min_cllr'] <= doc['calibration']['cllr'] <= doc['cllr'] + 1e-12
    assert abs(doc['calibration']['cllr'] - doc['calibration']['cllr_prior']) <= 1e-12
    raw = json.load(open(os.path.join(root, 'raw.json')))
    assert {k: v for k, v in doc.items() if k not in ('calibration', 'min_cllr', 'timings_s')} == \
        {k: v for k, v in raw.items() if k != 'timings_s'}
    # applying the file to the same list gives the self-calibrated metrics
    assert verify.main(vargs + ['--calibration', cal_path, '--json', js]) == 0
    app = json.load(open(js))
    assert app['cllr'] == doc['calibration']['cllr'] and app['eer'] == doc['calibration']['eer']
    # diarization with calibrated thresholds against the raw ones
    recs, _, rtruth = synth.multi_session_archive(ES['x_raw'], n_rec=4, pool=10, seed=45)
    ark, seg = write_archive(root, recs)
    first = next(iter(recs))
    enrol = {}
    for k, v in zip(rtruth[first].tolist(), recs[first][0]):
        enrol.setdefault(f'known{k}', []).append(v)
    k_ark, k_u, _, _ = write_side(root, 'known', {k: np.array(v[:10]) for k, v in enrol.items()}, False)
    base = ['--init', 'AHC+VB', '--xvec-ark-file', ark, '--segments-file', seg, '--threshold', '-0.015',
            '--lda-dim', str(d), '--xvec-transform', tf, '--plda-file', plda] + HYPER
    runs = {'link': ['--link-threshold'], 'enrol': ['--enroll-ark', k_ark, '--enroll-utt2spk', k_u,
                                                    '--enroll-threshold']}
    for what, opt in runs.items():
        for t in (0.0, 2.5, -4.0):
            a_dir, b_dir = os.path.join(root, f'{what}{t}a'), os.path.join(root, f'{what}{t}b')
            assert cli.main(base + ['--out-rttm-dir', a_dir, '--calibration', cal_path] + opt + [repr(t)]) == 0
            assert cli.main(base + ['--out-rttm-dir', b_dir] + opt + [repr(verify.raw_threshold(cal, t))]) == 0
            assert read_dir(a_dir) == read_dir(b_dir) and len(read_dir(a_dir)) == len(recs)
    # --enroll-threshold omitted with --calibration: t = 0
    c_dir = os.path.join(root, 'enrol_default')
    assert cli.main(base + ['--out-rttm-dir', c_dir, '--calibration', cal_path] + runs['enrol'][:-1]) == 0
    assert read_dir(c_dir) == read_dir(os.path.join(root, 'enrol0.0a'))
