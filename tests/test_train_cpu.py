"""Back-end training without a GPU (DESIGN.md section 5.24): the float64 oracle against itself (EM never lowers the
objective, the objective is the exact marginal log-likelihood, a known model is recovered, the LDA invariants), the
model files read back bit for bit, the classes taken from reference RTTMs, every refusal, and DMMA in the scatter
kernel's SASS."""
import collections
import re
import shutil
import subprocess

import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import train_oracle as O
from vbx_b200 import _lib, formats, pipeline, score, train


def spd(d, rng, lo, hi):
    q, _ = np.linalg.qr(rng.standard_normal((d, d)))
    return (q * np.exp(np.linspace(np.log(hi), np.log(lo), d))[None, :]) @ q.T


def draw_classes(W, B, n, rng):
    """Vectors z = s_i + e of classes of sizes n from N(0, B) speakers and N(0, W) noise -> (Mc, n, S, classes)."""
    d = W.shape[0]
    Lw, Lb = np.linalg.cholesky(W), np.linalg.cholesky(B)
    classes = [(Lb @ rng.standard_normal(d))[None, :] + rng.standard_normal((k, d)) @ Lw.T for k in n]
    off = np.concatenate([[0], np.cumsum(n)])
    m, S = O.class_stats(np.concatenate(classes), off)
    return m, np.asarray(n, dtype=np.float64), S, classes


def test_em_never_lowers_the_objective():
    rng = np.random.default_rng(3)
    d = 6
    W, B = spd(d, rng, 0.2, 2.0), spd(d, rng, 0.1, 4.0)
    Mc, n, S, _ = draw_classes(W, B, rng.integers(1, 9, 60), rng)
    _, _, trace = O.plda_em(Mc, n, S, 25)
    assert np.all(np.diff(trace) >= -1e-12 * np.abs(trace[1:])), np.diff(trace)
    assert trace[-1] > trace[0]


def test_objective_is_the_marginal_log_likelihood():
    """Small classes: the objective equals the sum of the brute-force log-densities of each class's stacked vectors,
    whose covariance is I (x) W + 1 1^T (x) B."""
    rng = np.random.default_rng(5)
    d = 3
    W, B = spd(d, rng, 0.3, 1.5), spd(d, rng, 0.2, 3.0)
    Mc, n, S, classes = draw_classes(W, B, [1, 2, 3, 4, 2], rng)
    brute = 0.0
    for z in classes:
        k = len(z)
        cov = np.kron(np.eye(k), W) + np.kron(np.ones((k, k)), B)
        brute += multivariate_normal(np.zeros(k * d), cov).logpdf(z.reshape(-1))
    got = O.objective(W, B, Mc, n, S)
    assert abs(got - brute) <= 1e-10 * abs(brute), (got, brute)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_em_recovers_a_known_model(seed):
    rng = np.random.default_rng(100 + seed)
    d, K = 32, 4000
    W, B = spd(d, rng, 0.05, 1.0), spd(d, rng, 0.02, 3.0)
    Mc, n, S, _ = draw_classes(W, B, rng.integers(4, 13, K), rng)
    mu = n @ Mc / n.sum()
    We, Be, trace = O.plda_em(Mc - mu, n, S, 10)
    assert np.linalg.norm(We - W) <= 0.03 * np.linalg.norm(W)
    assert np.linalg.norm(Be - B) <= 0.12 * np.linalg.norm(B)
    # the device's EM (jointly diagonal basis, torch on the CPU here) takes the same steps
    import torch
    W2, B2, trace2 = train.plda_em(torch.from_numpy(Mc - mu), torch.from_numpy(n), S, float(n.sum()), 10)
    assert np.allclose(trace2, trace, rtol=1e-10, atol=0)
    assert np.linalg.norm(W2 - We) <= 1e-9 * np.linalg.norm(We) and np.linalg.norm(B2 - Be) <= 1e-9 * np.linalg.norm(Be)


def test_lda_invariants():
    rng = np.random.default_rng(7)
    D, K, d = 12, 9, 5
    x = np.concatenate([rng.standard_normal(D) * 3 + rng.standard_normal((20, D)) @ spd(D, rng, 0.3, 2) for _ in range(K)])
    off = np.arange(0, 20 * (K + 1), 20)
    m, Sw = O.class_stats(x, off)
    n = np.diff(off).astype(np.float64)
    mu = n @ m / n.sum()
    Sb = ((m - mu).T * n) @ (m - mu) / n.sum()
    lam, A = O.lda(Sw / n.sum(), Sb, d)
    assert np.allclose(A.T @ (Sw / n.sum()) @ A, np.eye(d), atol=1e-10)
    assert np.allclose(A.T @ Sb @ A, np.diag(lam), atol=1e-10 * lam[0])
    assert np.all(np.diff(lam) <= 0)
    assert np.all(A[np.argmax(np.abs(A), 0), np.arange(d)] > 0)


@pytest.mark.parametrize('binary', [True, False])
def test_written_model_reads_back(tmp_path, binary):
    rng = np.random.default_rng(11)
    Dx, d = 16, 6
    W, B = spd(d, rng, 0.1, 1.0), spd(d, rng, 0.05, 2.0)
    tr, psi = O.kaldi_form(W, B)
    transform = (rng.standard_normal(Dx), rng.standard_normal(d), rng.standard_normal((Dx, d)))
    plda = (rng.standard_normal(d), tr, psi)
    paths = train.write_backend(str(tmp_path), transform, plda, dict(N=1, K=2), binary=binary)
    for a, b in zip(formats.read_xvec_transform(paths[0]), transform):
        assert a.dtype == np.float64 and np.array_equal(a, b)
    back = formats.read_kaldi_plda(paths[1])
    for a, b in zip(back, plda):
        assert np.array_equal(a, b)
    _, _, psi2 = pipeline.diagonalise_plda(*back)
    assert np.allclose(psi2, psi, rtol=1e-10, atol=0)
    # the Kaldi form reproduces W and B: W = (tr^T tr)^-1, B = (tr^T diag(1/psi) tr)^-1
    assert np.allclose(np.linalg.inv(tr.T @ tr), W, rtol=0, atol=1e-12)
    assert np.allclose(np.linalg.inv((tr.T / psi) @ tr), B, rtol=0, atol=1e-10)


def rttm_case():
    # 1.5 s segments; A speaks 0-10 s, B 9-10 s (overlap) and 12-20 s; nobody 10-12 s
    seg = np.array([[0.0, 1.5], [8.6, 10.1], [9.0, 10.0], [10.2, 11.7], [11.6, 13.1], [13.0, 14.5], [19.9, 21.4]])
    x = np.arange(7 * 4, dtype=np.float64).reshape(7, 4)
    rows = [('r1', 0.0, 10.0, 'A'), ('r1', 9.0, 1.0, 'B'), ('r1', 12.0, 8.0, 'B'),
            ('r2', 0.0, 10.0, 'A'), ('r2', 9.0, 1.0, 'B'), ('r2', 12.0, 8.0, 'B')]
    return {'r1': (x, seg), 'r2': (x + 100, seg), 'r3': (x + 200, seg)}, rows


def test_speakers_from_rttm():
    recs, rows = rttm_case()
    spk, counts = train.speakers_from_rttm(recs, rows)
    # segment 0 pure A; 1 and 2 overlapped by B; 3 uncovered; 4 B for 1.1 of 1.5 s (below 0.75); 5 pure B; 6 B for
    # 0.1 s and nobody else
    assert list(spk) == [('r1', 'A'), ('r1', 'B'), ('r2', 'A'), ('r2', 'B')]
    assert np.array_equal(spk[('r1', 'A')], recs['r1'][0][[0]])
    assert np.array_equal(spk[('r1', 'B')], recs['r1'][0][[5]])
    assert np.array_equal(spk[('r2', 'B')], recs['r2'][0][[5]])
    assert counts == dict(kept=4, overlapped=4, uncovered=6 + 7)     # r3 has no reference at all
    merged, _ = train.speakers_from_rttm(recs, rows, across_recordings=True)
    assert list(merged) == ['A', 'B']
    assert np.array_equal(merged['A'], np.stack([recs['r1'][0][0], recs['r2'][0][0]]))
    lax, c2 = train.speakers_from_rttm(recs, rows, min_share=0.6)
    assert np.array_equal(lax[('r1', 'B')], recs['r1'][0][[4, 5]]) and c2['kept'] == 6


def test_speaker_shares_match_the_init_definition():
    """c_k = the share of [lo, hi) inside speaker k's merged turns (vbx_init_turns), against a per-tick count."""
    rng = np.random.default_rng(2)
    rows = [('r', float(s), float(rng.integers(1, 40)), f'S{rng.integers(3)}') for s in rng.integers(0, 200, 30)]
    turns = score.named_turns(rows)['r']
    seg = np.sort(rng.integers(0, 260, (50, 2)), 1) * 1_000_000
    c = train.speaker_shares(seg, turns)
    for t, (lo, hi) in enumerate(seg):
        for k, (_, (s, e)) in enumerate(turns):
            cov = sum(max(0, min(hi, b) - max(lo, a)) for a, b in zip(s, e))
            want = cov / (hi - lo) if hi > lo else 0.0
            assert abs(c[t, k] - want) < 1e-15


def good_set(K=6, n=8, D=4, seed=0):
    rng = np.random.default_rng(seed)
    return {f's{i}': rng.standard_normal((n, D)) for i in range(K)}


@pytest.mark.parametrize('change, match', [
    (dict(xvectors={'a': np.ones((5, 4))}), 'at least 2'),
    (dict(xvectors={'a': np.ones((5, 4)), 'b': np.ones((1, 4))}), 'at least 2'),
    (dict(lda_dim=5), 'lda_dim = 5 exceeds Dx = 4'),
    (dict(lda_dim=4, xvectors=good_set(K=3, n=8)), 'K - 1 = 2'),
    (dict(xvectors=good_set(K=3, n=2, D=4), lda_dim=2), 'N - K = 6 - 3 = 3 is below Dx = 4'),
    (dict(xvectors=dict(good_set(), bad=np.full((3, 4), np.nan))), 'non-finite'),
    (dict(min_per_speaker=0), 'min_per_speaker'),
    (dict(em_iters=-1), 'em_iters'),
    (dict(xvectors=dict(good_set(), odd=np.ones((3, 5)))), 'dimension 5'),
])
def test_refusals(change, match):
    kw = dict(xvectors=good_set(), lda_dim=3, em_iters=2, min_per_speaker=2)
    kw.update(change)
    with pytest.raises(ValueError, match=re.escape(match)):
        train.train_backend(kw.pop('xvectors'), **kw)


def test_dropped_speakers_are_counted_before_the_refusals():
    sets = good_set(K=3, n=8, D=2)
    sets.update(tiny=np.ones((1, 2)))
    names, arrays, drop_spk, drop_x, Dx = train.check_training_set(sets, 2, 1, 2)
    assert (drop_spk, drop_x, Dx, len(arrays)) == (1, 1, 2, 3) and 'tiny' not in names


@pytest.mark.parametrize('argv', [
    ['--xvec-ark-file', 'a', '--out-dir', 'o'],
    ['--xvec-ark-file', 'a', '--out-dir', 'o', '--utt2spk', 'u', '--ref-rttm', 'r', '--segments-file', 's'],
    ['--xvec-ark-file', 'a', '--out-dir', 'o', '--ref-rttm', 'r'],
    ['--xvec-ark-file', 'a', '--out-dir', 'o', '--utt2spk', 'u', '--segments-file', 's'],
    ['--xvec-ark-file', 'a', '--out-dir', 'o', '--utt2spk', 'u', '--speakers-across-recordings'],
    ['--xvec-ark-file', 'a', '--out-dir', 'o', '--utt2spk', 'u', '--min-share', '0.5'],
])
def test_parser_refusals(argv):
    with pytest.raises(SystemExit) as e:
        train.main(argv)
    assert e.value.code == 2


def test_scatter_kernel_runs_on_dmma():
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    try:
        out = subprocess.run([tool, '-sass', _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip('cuobjdump not available')
    if out.returncode != 0 or 'Function :' not in out.stdout:
        pytest.skip('cuobjdump could not read the library')
    per_fn, fn = collections.defaultdict(collections.Counter), None
    for line in out.stdout.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            fn = m.group(1)
            continue
        m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)', line)
        if m and fn:
            per_fn[fn][m.group(1)] += 1
    scatter = {f: c for f, c in per_fn.items() if 'train_scatter_kernel' in f}
    assert len(scatter) == 1
    (c,) = scatter.values()
    assert c['DMMA'] >= 16                          # 4 x 4 m8n8k4 tiles per warp and k-step
    assert c['ATOM'] == c['RED'] == 0               # partial tiles are summed in a fixed order
